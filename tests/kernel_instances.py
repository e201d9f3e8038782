"""The template instances of a kernel compiled into a built object, read from its SASS with cuobjdump.  Tests that hold one row
per compiled instance compare their tables with this set, so a new instance without a row fails the suite."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "livetalking_b200", "build")


def compiled_instances(obj: str, kernel: str) -> set:
    """{(template arg, ...)} of every ltb::<kernel><int / bool args...> in `obj` (a path under BUILD, or absolute); skips the
    calling test when cuobjdump or the object is missing."""
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    obj = os.path.join(BUILD, obj)
    if not os.path.exists(obj):
        pytest.skip("object file not kept")
    sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    out = set()
    for m in re.finditer(r"Function : _ZN3ltb\d+" + kernel + r"I((?:L[ib]\d+E)+)E", sass):
        out.add(tuple(int(v) for _t, v in re.findall(r"L([ib])(\d+)E", m.group(1))))
    return out
