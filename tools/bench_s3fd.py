"""S3FD face detection of the wav2lip avatar generator: the engine's captured graph against the torch eager restatement.

    python tools/bench_s3fd.py [--batch 16] [--height 720] [--width 1280] [--iters 20] [--video-seconds 10]

(1) detector: one S3FDDetector graph replay per batch (prep -> 31 convs -> select), CUDA events on the detector's stream after
    warm-up; TFLOP/s from s3fd.gflop_per_frame and the share of the 989 TFLOP/s dense fp16 tensor-core peak of the H100 SXM data
    sheet (the bound quoted).
(2) existing-path proxy, same GPU, same run: oracle/s3fd_ref.forward + select in torch eager, fp32 (TF32 off, as the reference
    runs) and fp16 channels_last.
(3) generate_avatar end to end on a synthetic video made with cv2.VideoWriter (MJPG): decode + watermark, full_imgs PNG writes,
    detection, face crops + PNG writes, avatar.ltbav.
Synthetic seeded weights (oracle.s3fd_ref.synth_state_dict).  Prints one JSON line, with the GPU name and power limit."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_TFLOPS = 989.0


def _gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, pl = [s.strip() for s in out.split(",")]
        return name, pl
    except Exception:
        import torch
        return torch.cuda.get_device_name(0), "unknown"


def _events_ms(torch, stream, fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(iters):
        fn()
    e1.record(stream)
    e1.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--height", type=int, default=720)
    ap.add_argument("--width", type=int, default=1280)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--video-seconds", type=float, default=10.0)
    a = ap.parse_args()
    import torch

    from livetalking_b200 import engine
    from livetalking_b200.plugin import wav2lip_genavatar as G
    from livetalking_b200.s3fd import S3FDDetector, S3FDNet, gflop_per_frame
    from oracle import s3fd_ref as R

    engine.set_device(0)
    N, H, W = a.batch, a.height, a.width
    sd = R.synth_state_dict(0)
    net = S3FDNet.from_state_dict(sd)
    det = S3FDDetector(net, N, H, W)
    frames = R.synth_frames([35 + (i % 3) * 5 for i in range(N)], H, W, seed=1)
    det.run_raw(frames)                                   # uploads the frames; the timed replays reuse them
    stream = torch.cuda.ExternalStream(det.ctx.cuda_stream)
    for _ in range(3):
        det.graph.launch()
    det.ctx.sync()
    ms = _events_ms(torch, stream, det.graph.launch, a.iters)
    gflop = gflop_per_frame(H, W) * N
    tflops = gflop / ms                                  # GFLOP per ms = TFLOP/s

    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.benchmark = True
    x = R.prep(frames, "cuda")
    sd_h = {k: v.cuda().half() for k, v in sd.items()}
    x_h = x.half().contiguous(memory_format=torch.channels_last)
    cur = torch.cuda.current_stream()
    with torch.no_grad():
        def eager32():
            R.select(R.forward(sd, x))

        def eager16():
            R.select(R.forward(sd_h, x_h))
        res = {}
        for name, fn in (("fp32", eager32), ("fp16_channels_last", eager16)):
            for _ in range(2):
                fn()
            torch.cuda.synchronize()
            res[name] = _events_ms(torch, cur, fn, max(3, a.iters // 4))

    tmp = tempfile.mkdtemp(prefix="bench_s3fd_")
    nfr = int(round(a.video_seconds * 25))
    amps = [40 if (i // 25) % 4 else 0 for i in range(nfr)]
    vid = os.path.join(tmp, "clip.avi")
    import cv2
    vw = cv2.VideoWriter(vid, cv2.VideoWriter_fourcc(*"MJPG"), 25, (W, H))
    for i in range(0, nfr, 25):
        for f in R.synth_frames(amps[i:i + 25], H, W, seed=i):
            vw.write(f)
    vw.release()
    wpath = os.path.join(tmp, "s3fd.pth")
    torch.save(sd, wpath)
    G.load_net(wpath)                                     # weights upload outside the timed call (as on a running server)
    t0 = time.perf_counter()
    split = {}
    G.generate_avatar(vid, "bench", save_path=os.path.join(tmp, "avatars"), face_det_batch_size=N, weights_path=wpath, timings=split)
    total = time.perf_counter() - t0
    name, pl = _gpu_info()
    det.close()
    print(json.dumps({
        "gpu": name, "power_limit": pl, "batch": N, "height": H, "width": W,
        "detector_ms_per_batch": round(ms, 3), "gflop_per_frame": round(gflop_per_frame(H, W), 2), "tflops": round(tflops, 1),
        "share_of_peak": round(tflops / PEAK_TFLOPS, 3), "peak_bound": "989 TFLOP/s dense fp16 (H100 SXM data sheet)",
        "torch_eager_fp32_ms_per_batch": round(res["fp32"], 2), "torch_eager_fp16_cl_ms_per_batch": round(res["fp16_channels_last"], 2),
        "e2e_frames": nfr, "e2e_s": round(total, 2), "e2e_split_s": {k: round(v, 2) for k, v in split.items()},
    }))


if __name__ == "__main__":
    main()
