"""Build libltb200.so (sm_90a only) in-tree with nvcc.

    python -m livetalking_b200.build            # incremental
    python -m livetalking_b200.build --force

The library is written to livetalking_b200/lib/libltb200.so, next to the sources (git-ignored).
There is exactly one target architecture: -gencode arch=compute_90a,code=sm_90a.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
OBJDIR = os.path.join(HERE, "build")
LIB = os.path.join(LIBDIR, "libltb200.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-std=c++17", "-O3", "-lineinfo",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found; libltb200 cannot be built")


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _deps_mtime() -> float:
    mt = 0.0
    for root in (CSRC, os.path.join(HERE, "..", "include")):
        for f in os.listdir(root):
            if f.endswith((".h", ".cuh")):
                mt = max(mt, os.path.getmtime(os.path.join(root, f)))
    return mt


def build(force: bool = False, verbose: bool = False, defines=(), tag: str = "") -> str:
    """defines/tag: diagnostic variants only (e.g. tools/diag_halo.py builds lib/libltb200_diag.so with -DLTB_HALO_DIAG)."""
    LIB = os.path.join(LIBDIR, f"libltb200{tag}.so")
    OBJDIR = os.path.join(HERE, "build" + tag)
    NVCC_FLAGS = [*globals()["NVCC_FLAGS"], *[f"-D{d}" for d in defines]]
    os.makedirs(LIBDIR, exist_ok=True)
    os.makedirs(OBJDIR, exist_ok=True)
    nvcc = _nvcc()
    hdr_mt = _deps_mtime()
    # objects built with other flags (another architecture, other defines) are stale whatever their timestamps
    stamp = os.path.join(OBJDIR, "flags.txt")
    flags = " ".join(NVCC_FLAGS)
    if not os.path.exists(stamp) or open(stamp).read() != flags:
        force = True
    jobs = []
    objs = []
    for src in sources():
        obj = os.path.join(OBJDIR, os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        if force or not os.path.exists(obj) or os.path.getmtime(obj) < max(os.path.getmtime(src), hdr_mt):
            cmd = [nvcc, *NVCC_FLAGS, "-c", src, "-o", obj]
            if verbose:
                cmd.insert(1, "-Xptxas=-v")
            jobs.append(cmd)

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + r.stdout + r.stderr)
        return r.stderr

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            for log in ex.map(run, jobs):
                if verbose and log:
                    print(log)
    if jobs or not os.path.exists(LIB):
        run([nvcc, "-shared", "-o", LIB, *objs, "-gencode", "arch=compute_90a,code=sm_90a", "-lcuda"])
    with open(stamp, "w") as fh:
        fh.write(flags)
    return LIB


if __name__ == "__main__":
    if "--diag" in sys.argv:     # diagnostic library: product kernels + LTB_HALO_DIAG knock-outs
        print(build(force="--force" in sys.argv, defines=("LTB_HALO_DIAG",), tag="_diag"))
        sys.exit(0)
    path = build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(path)
