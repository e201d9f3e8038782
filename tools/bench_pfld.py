"""PFLD landmarks of the UltraLight avatar generator: the engine's captured graph against the train-time module in torch eager.

    python tools/bench_pfld.py [--batch 16] [--iters 50] [--video-seconds 10]

(1) landmarker: one PFLDLandmarker graph replay per batch of 192 x 192 crops (prep -> 51 conv and depthwise layers -> head),
    CUDA events on its stream after warm-up; GFLOP/s from pfld.gflop_per_frame.
(2) reference architecture, same GPU, same run: oracle/pfld_ref.forward_train (PFLD_GhostOne's train-time form: six conv + BN
    branches, the scale branch and the skip BatchNorm per MobileOneBlock) in torch eager, fp32 (TF32 off) and fp16, at the same
    batch.  Landmark.detect itself runs it one frame at a time; the batch-1 fp32 time is printed too.
(3) generate_avatar end to end on a synthetic 720p MJPG clip with the replaying detector (oracle.pfld_ref.ReplayDetector: the SCRFD
    ONNX file is not part of the run): decode, full_imgs PNG writes, face_det crops + resize (host), landmarks (device wait), mouth
    crops + PNG writes, avatar.ltbav.
Synthetic seeded weights (oracle.pfld_ref.synth_state_dict).  Prints one JSON line, with the GPU name and power limit."""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

from gpu_bench import events_ms, gpu_info

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--video-seconds", type=float, default=10.0)
    a = ap.parse_args()
    import torch

    from livetalking_b200 import engine
    from livetalking_b200.pfld import PFLDLandmarker, PFLDNet, gflop_per_frame
    from livetalking_b200.plugin import ultralight_genavatar as G
    from oracle import pfld_ref as R

    engine.set_device(0)
    N = a.batch
    sd = R.synth_state_dict(0)
    mean_face = R.read_mean_face(os.path.join(ROOT, "tests", "golden", "pfld_mean_face.txt"))
    net = PFLDNet.from_state_dict(sd, mean_face)
    lm = PFLDLandmarker(net, N)
    crops = R.synth_video_frames(N, 192, 192, seed=1)
    lm.run(crops, np.full((N, 2), 200, np.int32))         # uploads the crops; the timed replays reuse them
    ms = events_ms(lm.graph.launch, a.iters, warmup=5, stream=torch.cuda.ExternalStream(lm.ctx.cuda_stream))

    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    x = R.prep(crops).cuda()
    sd32 = {k: (v.cuda().float() if v.is_floating_point() else v) for k, v in sd.items()}
    sd16 = {k: (v.cuda().half() if v.is_floating_point() else v) for k, v in sd.items()}
    res = {}
    with torch.no_grad():
        for name, fn in (("fp32", lambda: R.forward_train(sd32, x)), ("fp16", lambda: R.forward_train(sd16, x.half())),
                         ("fp32_b1", lambda: R.forward_train(sd32, x[:1]))):
            res[name] = events_ms(fn, max(5, a.iters // 5), warmup=3)

    tmp = tempfile.mkdtemp(prefix="bench_pfld_")
    nfr = int(round(a.video_seconds * 25))
    vid = os.path.join(tmp, "clip.avi")
    import cv2
    H, W = 720, 1280
    vw = cv2.VideoWriter(vid, cv2.VideoWriter_fourcc(*"MJPG"), 25, (W, H))
    for i in range(0, nfr, 25):
        for f in R.synth_video_frames(min(25, nfr - i), H, W, seed=i):
            vw.write(f)
    vw.release()
    boxes = [(480 + 40 * np.sin(i / 10), 200 + 20 * np.cos(i / 7), 300.0, 340.0) for i in range(nfr)]
    split = {}
    t0 = time.perf_counter()
    G.generate_avatar(vid, "bench", save_path=os.path.join(tmp, "avatars"), detector=R.ReplayDetector(R.face_records(boxes)),
                      make_landmarker=lambda n: PFLDLandmarker(net, n), timings=split)
    total = time.perf_counter() - t0
    name, pl = gpu_info()
    lm.close()
    gf = gflop_per_frame() * N
    print(json.dumps({
        "gpu": name, "power_limit": pl, "batch": N,
        "landmarker_ms_per_batch": round(ms, 4), "gflop_per_frame": round(gflop_per_frame(), 4), "gflops": round(gf / ms * 1e3, 1),
        "train_time_eager_fp32_ms_per_batch": round(res["fp32"], 3), "train_time_eager_fp16_ms_per_batch": round(res["fp16"], 3),
        "train_time_eager_fp32_ms_per_frame_b1": round(res["fp32_b1"], 3),
        "e2e_frames": nfr, "e2e_s": round(total, 2), "e2e_split_s": {k: round(v, 2) for k, v in split.items()},
    }))


if __name__ == "__main__":
    main()
