"""Per-layer roofline of the wav2lip256 forward (SURVEY.md §8(d): max(flops/peak, bytes/BW) per layer).

    python tools/layer_roofline.py per_op.json [forward_ms [peak_tflops peak_gbs]] > layer_roofline.md

For every conv op of the B=16 step: algorithmic FLOPs (from the engine's profile pass), algorithmic HBM bytes (fp16 input +
output (+ residual is the input: counted once) + weights), the time the measured peaks allow
(default: H100 SXM data sheet, 989 TFLOP/s dense fp16 and 3350 GB/s; pass the peaks of the GPU the profile came from) and the measured eager-event time.  Eager events include a launch gap
per op (their sum is ~25 % above the graph replay), so the last line also gives the whole-forward figure from the live replay.
"""
import json
import sys

PEAK_TF, PEAK_GBS = 989.0, 3350.0
B = 16


def od(h, k, s, p):
    return (h + 2 * p - k) // s + 1


def layers():
    """(name, cin, cout, k, IH, IW, OH, OW, kind) in the engine's op order (audio branch first)."""
    out = []
    H, W = 80, 16
    audio = [(1, 32, 3, 1, 1, 1), (32, 32, 3, 1, 1, 1), (32, 32, 3, 1, 1, 1), (32, 64, 3, 3, 1, 1), (64, 64, 3, 1, 1, 1), (64, 64, 3, 1, 1, 1),
             (64, 128, 3, 3, 3, 1), (128, 128, 3, 1, 1, 1), (128, 128, 3, 1, 1, 1), (128, 256, 3, 3, 2, 1), (256, 256, 3, 1, 1, 1),
             (256, 512, 3, 1, 1, 0), (512, 512, 1, 1, 1, 0)]
    for i, (ci, co, k, sy, sx, p) in enumerate(audio):
        OH, OW = od(H, k, sy, p), od(W, k, sx, p)
        out.append((f"L{i:02d} audio", ci, co, k, H, W, OH, OW, "c"))
        H, W = OH, OW
    face = [(6, 16, 7, 1, 3), (16, 32, 3, 2, 1), (32, 32, 3, 1, 1), (32, 32, 3, 1, 1), (32, 64, 3, 2, 1), (64, 64, 3, 1, 1), (64, 64, 3, 1, 1),
            (64, 64, 3, 1, 1), (64, 128, 3, 2, 1), (128, 128, 3, 1, 1), (128, 128, 3, 1, 1), (128, 256, 3, 2, 1), (256, 256, 3, 1, 1),
            (256, 256, 3, 1, 1), (256, 512, 3, 2, 1), (512, 512, 3, 1, 1), (512, 512, 3, 2, 1), (512, 512, 3, 1, 1), (512, 512, 4, 1, 0),
            (512, 512, 1, 1, 0)]
    H = 256
    for i, (ci, co, k, s, p) in enumerate(face):
        OH = od(H, k, s, p)
        out.append((f"L{13 + i:02d} enc", ci, co, k, H, H, OH, OH, "c"))
        H = OH
    dec = [("c", 512, 512, 1), ("t4", 1024, 512, 4), ("c", 512, 512, 3), ("t", 1024, 512, 3), ("c", 512, 512, 3), ("t", 1024, 512, 3),
           ("c", 512, 512, 3), ("c", 512, 512, 3), ("t", 768, 384, 3), ("c", 384, 384, 3), ("c", 384, 384, 3), ("t", 512, 256, 3),
           ("c", 256, 256, 3), ("c", 256, 256, 3), ("t", 320, 128, 3), ("c", 128, 128, 3), ("c", 128, 128, 3), ("t", 160, 64, 3),
           ("c", 64, 64, 3), ("c", 64, 64, 3), ("c", 80, 32, 3)]
    H = 1
    for i, (kind, ci, co, k) in enumerate(dec):
        OH = 4 if kind == "t4" else (2 * H if kind == "t" else H)
        out.append((f"L{33 + i:02d} dec{'T' if kind != 'c' else ''}", ci, co, k, H, H, OH, OH, kind))
        H = OH
    return out


def main(path, forward_ms=None):
    ops = json.load(open(path))["ops"]
    conv_ops = [(k, ms, fl) for k, ms, fl in ops if k in (0, 2, 4, 5)]          # audio conv0 (kind 2) is layer 0
    L = layers()
    assert len(conv_ops) == len(L), (len(conv_ops), len(L))
    print("| layer | Cin→Cout k | map | GFLOP | MB | bound µs (tensor / HBM) | measured µs | % of bound |")
    print("|---|---|---|---|---|---|---|---|")
    tot_bound = tot_meas = tot_fl = tot_by = 0.0
    main_bound = main_meas = 0.0
    for (name, ci, co, k, IH, IW, OH, OW, kind), (opk, ms, fl) in zip(L, conv_ops):
        if kind == "c":
            flops = 2.0 * B * OH * OW * co * ci * k * k
        elif kind == "t4":
            flops = 2.0 * B * 16 * co * ci
        else:
            flops = 2.0 * B * IH * IW * 9 * co * ci       # ConvT k3 s2 without zero insertion: 9 taps per INPUT pixel
        by = 2.0 * B * (IH * IW * ci + OH * OW * co) + 2.0 * ci * co * k * k
        t_tc, t_hbm = flops / (PEAK_TF * 1e12) * 1e6, by / (PEAK_GBS * 1e9) * 1e6
        bound = max(t_tc, t_hbm)
        meas = ms * 1e3
        tot_bound += bound
        tot_meas += meas
        tot_fl += flops
        tot_by += by
        if "audio" not in name:
            main_bound += bound
            main_meas += meas
        print(f"| {name} | {ci}→{co} k{k} | {IH}x{IW}→{OH}x{OW} | {flops / 1e9:.2f} | {by / 1e6:.1f} | {bound:.1f} ({t_tc:.1f} / {t_hbm:.1f}) | {meas:.1f} | {100 * bound / meas:.0f} |")
    print()
    print(f"Sum over all {len(L)} conv layers: {tot_fl / 1e9:.1f} GFLOP, {tot_by / 1e9:.2f} GB, per-layer roofline bound {tot_bound:.0f} µs "
          f"(face path only, the audio branch runs concurrently: {main_bound:.0f} µs); eager per-op events sum to {tot_meas:.0f} µs "
          f"(face path {main_meas:.0f} µs).")
    if forward_ms:
        print(f"Live forward-graph replay: {forward_ms * 1e3:.0f} µs per step = {100 * main_bound / (forward_ms * 1e3):.0f} % of the per-layer "
              f"roofline bound of the face path ({100 * (tot_fl / 1e12) / (forward_ms / 1e3) / PEAK_TF:.1f} % of the pure tensor roofline).")


if __name__ == "__main__":
    if len(sys.argv) > 4:
        PEAK_TF, PEAK_GBS = float(sys.argv[3]), float(sys.argv[4])
    main(sys.argv[1], float(sys.argv[2]) if len(sys.argv) > 2 else None)
