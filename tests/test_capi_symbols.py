"""CPU: the C-ABI library builds, loads and exports every symbol include/ltb200.h declares (no compute calls)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def built_lib():
    from livetalking_b200 import build
    return build.build()


def _header_functions():
    src = open(os.path.join(ROOT, "include", "ltb200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(ltb_[a-z0-9_]+)\s*\(", src)))


def test_header_and_binding_agree(built_lib):
    from livetalking_b200 import _capi
    names = _header_functions()
    assert len(names) >= 20
    assert sorted(_capi.EXPORTED_SYMBOLS) == names
    lib = ctypes.CDLL(built_lib)
    for n in names:
        assert hasattr(lib, n), n


def test_library_is_sm90a_tensor_core_code(built_lib):
    import shutil
    import subprocess
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", built_lib], capture_output=True, text=True).stdout
    assert "sm_90a" in sass
    assert "HGMMA" in sass            # wgmma.mma_async
    assert "UTMALDG" in sass          # TMA tensor loads


def test_version_and_error_string(built_lib):
    from livetalking_b200 import _capi
    lib = _capi.lib()
    assert lib.ltb_version() >= 100
    # a failing call must set a message and must not abort: null session
    assert lib.ltb_w2l_sync(None) != 0
    assert b"null" in lib.ltb_last_error()


def test_header_constants_match_binding():
    """#define LTB_* values in the header are the ones the ctypes layer uses."""
    from livetalking_b200 import _capi
    src = open(os.path.join(ROOT, "include", "ltb200.h")).read()
    defs = {m.group(1): int(m.group(2), 0) for m in re.finditer(r"#define\s+(LTB_[A-Z0-9_]+)\s+(0x[0-9a-fA-F]+|\d+)\b", src)}
    flags = {k: v for k, v in defs.items() if k.startswith("LTB_SESSION_")}
    assert set(flags) >= {"LTB_SESSION_KEEP_LAYERS", "LTB_SESSION_NO_GRAPH", "LTB_SESSION_NO_HALO", "LTB_SESSION_NO_PDL"}
    for k, v in flags.items():
        assert getattr(_capi, k) == v, k
    vals = sorted(flags.values())
    assert all(a & b == 0 for i, a in enumerate(vals) for b in vals[i + 1:])      # distinct bits


def test_issue_path_has_no_election_loops(built_lib):
    """Regression guard: an MMA issued from divergent code makes ptxas wrap it in an ELECT / BRA.U.ANY loop (~100 cycles per
    MMA).  The halo kernels must contain only the few loops of the TMA producer."""
    import shutil
    import subprocess
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    obj = os.path.join(ROOT, "livetalking_b200", "build", "conv_halo.o")
    if not os.path.exists(obj):
        pytest.skip("object file not kept")
    sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True).stdout
    funcs = re.split(r"\n\s*Function : ", sass)[1:]
    halo = [f for f in funcs if "conv_halo_wgmma_kernel" in f.split("\n", 1)[0]]
    assert len(halo) >= 10
    for f in halo:
        mma = f.count("HGMMA")
        loops = f.count("BRA.U.ANY")
        lines = f.count("\n") // 2
        assert mma >= 4, f.split("\n", 1)[0]
        assert loops <= 12 and loops < mma, (f.split("\n", 1)[0], mma, loops)
        assert lines < 8000, (f.split("\n", 1)[0], lines)     # the fully unrolled 28k-line variant thrashed the instruction cache
