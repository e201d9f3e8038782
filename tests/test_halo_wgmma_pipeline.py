"""CPU: ptxas keeps the wgmma pipeline of every single-accumulator halo conv instance.

ptxas reports C75xx when it serialises wgmma instructions or injects warpgroup waits (for example when registers the MMAs
write are touched, or a data-dependent branch sits between them).  The 3x3, stride-2 and GEMM instances (NACC == 1) issue their
MMAs back to back and must compile without any such report.  The sub-pixel instances (NACC == 4) wait between fat MMA groups
on purpose and are not checked."""
import os
import re
import subprocess
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_single_accumulator_instances_keep_the_wgmma_pipeline():
    from livetalking_b200 import build
    src = os.path.join(ROOT, "livetalking_b200", "csrc", "conv_halo.cu")
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([build._nvcc(), *build.NVCC_FLAGS, "-Xptxas=-v", "-c", src, "-o", os.path.join(tmp, "conv_halo.o")],
                           capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    log = r.stdout + r.stderr
    instances = {}
    for name in re.findall(r"Compiling entry function '(_ZN3ltb\d+conv_halo_wgmma_kernelI\S+?)'", log):
        args = tuple(int(v) for _t, v in re.findall(r"L([ib])(\d+)E", name))
        instances[name] = args      # (BN, NSUB, NACC, TAPS, RC, GRP)
    assert len(instances) == 28, sorted(instances.values())
    warned = {}
    for code, name in re.findall(r"\((C75\d\d)\)[^\n]*?function '(\S+?)'", log):
        if instances.get(name, (0, 0, 0))[2] == 1:
            warned.setdefault(instances[name], set()).add(code)
    assert not warned, f"wgmma pipeline serialised in: {warned}"
