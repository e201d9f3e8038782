"""CPU: the row-pair conv kernel (conv_rowpair.cu) as ptxas builds it for sm_90a.

It keeps its accumulators and epilogue in registers (no local-memory spills), ptxas does not serialise its wgmma pipeline (no
C75xx advisory), the halo tiles and resident weights arrive by TMA (UTMALDG), the MMAs are m64n128k16 (two output rows of 32
channels x 16 row pairs of 8 pixels), and the epilogue goes through stmatrix (STSM) into the staging tile and out with a TMA
tensor store (UTMASTG)."""
import os
import re

import pytest
from sass_build import compile_sass

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "livetalking_b200", "csrc", "conv_rowpair.cu")


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    return compile_sass(SRC, tmp_path_factory.mktemp("rowpair"))


def test_rowpair_kernel_has_no_spills_or_wgmma_serialisation(compiled):
    log, sass = compiled
    assert "conv_rowpair_kernel" in log, log
    assert re.search(r"\b0 bytes spill stores, 0 bytes spill loads", log), log
    assert not re.search(r"C75\d\d", log), log
    assert not re.search(r"\b(STL|LDL)\b", sass)


def test_rowpair_uses_tma_wgmma_and_stmatrix(compiled):
    _, sass = compiled
    assert "UTMALDG" in sass
    assert "UTMASTG" in sass
    assert "STSM" in sass
    assert len(re.findall(r"HGMMA\.64x128x16\.F32", sass)) == 60   # 4 views x (4 + 1) K steps x 3 tap columns
