"""CPU: the evidence tooling reproduces the committed artefacts in profiles/ from the committed raw captures."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_traffic_from_ncu_reproduces_committed_json(tmp_path):
    src = os.path.join(ROOT, "profiles", "r02q_launches_wav2lip.csv")
    out = str(tmp_path / "traffic.json")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "traffic_from_ncu.py"), src, out], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    got = json.load(open(out))
    want = json.load(open(os.path.join(ROOT, "profiles", "conv_traffic.json")))
    assert got["dram_bytes_per_step"] == want["dram_bytes_per_step"]
    # sanity of the figure itself: between the weights-only floor and the no-reuse algorithmic traffic of one B=16 step
    assert 0.107e9 < got["dram_bytes_per_step"] < 2.5e9
    kernels = got["per_kernel"]
    assert any("conv_halo_umma_kernel" in k for k in kernels) and any("stem_umma_kernel" in k for k in kernels)


def test_layer_roofline_table_is_consistent():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "layer_roofline.py"),
                        os.path.join(ROOT, "profiles", "r01n_per_op_wav2lip.json"), "1.2876", "1404.6", "6541.8"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    rows = [l for l in r.stdout.splitlines() if l.startswith("| L")]
    assert len(rows) == 54                                             # 13 audio + 20 face-encoder + 21 decoder conv layers
    total = sum(float(l.split("|")[4]) for l in rows)
    assert abs(total - 889.3) < 1.0                                    # 16 x 55.58 GFLOP (SURVEY App. A)
    assert r.stdout.strip() == open(os.path.join(ROOT, "profiles", "r01n_layer_roofline.md")).read().strip()
