"""CPU: the small-map split-K conv kernel (conv_smallmap.cu) as ptxas builds it for sm_90a.

All three instances (256, 64 and 16 pixels per tile) keep their accumulators in registers (no local-memory spills), ptxas does
not serialise their wgmma pipeline (no C75xx advisory), operands arrive by TMA (UTMALDG), the MMAs are HGMMA with the pixels on
N, and the split-K partials are reduced across the CTAs of a cluster between cluster barriers."""
import os
import re

import pytest
from sass_build import compile_sass

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "livetalking_b200", "csrc", "conv_smallmap.cu")


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    return compile_sass(SRC, tmp_path_factory.mktemp("smallmap"))


def test_smallmap_kernels_have_no_spills_or_wgmma_serialisation(compiled):
    log, sass = compiled
    for np_ in (256, 64, 16):
        assert f"conv_smallmap_kernelILi{np_}E" in log, log
    assert len(re.findall(r"\b0 bytes spill stores, 0 bytes spill loads", log)) >= 3, log
    assert not re.search(r"C75\d\d", log), log
    assert not re.search(r"\b(STL|LDL)\b", sass)


def test_smallmap_uses_tma_wgmma_and_distributed_shared_memory(compiled):
    _, sass = compiled
    assert "UTMALDG.2D" in sass and "UTMALDG.4D" in sass
    for n in (256, 64, 16):
        assert f"HGMMA.64x{n}x16.F32" in sass, n
    assert "UCGABAR_ARV" in sass and "UCGABAR_WAIT" in sass
