"""CPU: the ping-pong conv kernel (conv_pingpong.cu) as ptxas builds it for sm_90a.

It keeps its 64 accumulators, 32 residual words and epilogue in registers (no local-memory spills), ptxas does not serialise
its wgmma pipeline (no C75xx advisory), and the epilogue goes through stmatrix (STSM) into shared memory and out with one TMA
tensor store (UTMASTG) per tile."""
import os
import re

import pytest
from sass_build import compile_sass

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "livetalking_b200", "csrc", "conv_pingpong.cu")


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    return compile_sass(SRC, tmp_path_factory.mktemp("pingpong"))


def test_pingpong_kernel_has_no_spills_or_wgmma_serialisation(compiled):
    log, sass = compiled
    assert "conv_pingpong_kernel" in log, log
    assert re.search(r"\b0 bytes spill stores, 0 bytes spill loads", log), log
    assert not re.search(r"C75\d\d", log), log
    assert not re.search(r"\b(STL|LDL)\b", sass)


def test_pingpong_epilogue_uses_stmatrix_and_tma_store(compiled):
    _, sass = compiled
    assert "STSM" in sass
    assert "UTMASTG" in sass
    assert "HGMMA.64x128x16.F32" in sass
