"""CPU: the halo conv kernel's register layout and epilogue accesses, read from the SASS of conv_halo.o.

Every instance keeps its accumulators and epilogue in registers (no local-memory spills), and every instance writes its
output tile with 16-byte stores (8 fp16 channels per lane) and reads a residual with 16-byte loads."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def halo_functions():
    from livetalking_b200 import build
    build.build()
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    obj = os.path.join(ROOT, "livetalking_b200", "build", "conv_halo.o")
    if not os.path.exists(obj):
        pytest.skip("object file not kept")
    sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True).stdout
    funcs = re.split(r"\n\s*Function : ", sass)[1:]
    halo = {f.split("\n", 1)[0].strip(): f for f in funcs if "conv_halo_wgmma_kernel" in f.split("\n", 1)[0]}
    assert len(halo) == 28
    return halo


def test_halo_instances_do_not_spill(halo_functions):
    for name, f in halo_functions.items():
        assert not re.search(r"\b(STL|LDL)\b", f), name


def test_halo_epilogue_uses_16_byte_accesses(halo_functions):
    for name, f in halo_functions.items():
        assert "STG.E.128" in f, name
        assert "LDG.E.128" in f, name       # residual reads
