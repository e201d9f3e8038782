"""CPU: ptxas keeps the wgmma pipeline of every halo conv instance, the sub-pixel ones (NACC == 4) included, without spills.

ptxas reports C75xx when it serialises wgmma instructions or injects warpgroup waits (for example when registers the MMAs
write are touched, or a data-dependent branch sits between them).  The sub-pixel ConvT (TAPS == 9) and upsample + conv
(TAPS == 16) instances issue one N = BN wgmma per (view, phase slot): every MMA of a K chunk writes a register range of one
shape, so they chain like the 3x3 taps and must compile without any such report, within the consumers' register budget."""
import os
import re
import subprocess
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ptxas_log():
    from livetalking_b200 import build
    src = os.path.join(ROOT, "livetalking_b200", "csrc", "conv_halo.cu")
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([build._nvcc(), *build.NVCC_FLAGS, "-Xptxas=-v", "-c", src, "-o", os.path.join(tmp, "conv_halo.o")],
                           capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return r.stdout + r.stderr


def test_every_halo_instance_keeps_the_wgmma_pipeline_without_spills():
    log = _ptxas_log()
    instances, spills, cur = {}, {}, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '(_ZN3ltb\d+conv_halo_wgmma_kernelI\S+?)'", line)
        if m:
            cur = m.group(1)
            instances[cur] = tuple(int(v) for _t, v in re.findall(r"L([ib])(\d+)E", cur))   # (BN, NSUB, NACC, TAPS, RC, GRP)
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur in instances and (int(m.group(1)) or int(m.group(2))):
            spills[instances[cur]] = (int(m.group(1)), int(m.group(2)))
    assert len(instances) == 28, sorted(instances.values())
    subpixel = sorted(a for a in instances.values() if a[2] == 4)
    assert subpixel == [(32, 1, 4, 9, 0, 0), (32, 1, 4, 9, 1, 0), (32, 1, 4, 9, 2, 0), (64, 1, 4, 9, 0, 0), (64, 1, 4, 9, 1, 0),
                        (64, 1, 4, 9, 2, 0), (64, 1, 4, 16, 0, 0)], subpixel
    warned = {}
    for code, name in re.findall(r"\((C75\d\d)\)[^\n]*?function '(\S+?)'", log):
        warned.setdefault(instances.get(name, name), set()).add(code)
    assert not warned, f"wgmma pipeline serialised in: {warned}"
    assert not spills, f"register spills (stores, loads) in: {spills}"
