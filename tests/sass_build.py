"""One kernel source compiled on its own with the library's nvcc flags plus -Xptxas -v, for the tests that read what ptxas made of
it: the ptxas log (registers, spills, advisories) and the SASS cuobjdump prints."""
import os
import shutil
import subprocess

import pytest


def compile_sass(src: str, tmpdir) -> tuple:
    """(ptxas log, sass) of `src` compiled into `tmpdir`; skips the calling test when cuobjdump is missing."""
    from livetalking_b200 import build
    nvcc = build._nvcc()
    cuobjdump = shutil.which("cuobjdump") or os.path.join(os.path.dirname(nvcc), "cuobjdump")
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    obj = os.path.join(str(tmpdir), os.path.basename(src)[:-3] + ".o")
    r = subprocess.run([nvcc, *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", src, "-o", obj], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    return r.stdout + r.stderr, sass
