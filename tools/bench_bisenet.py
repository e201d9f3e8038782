"""BiSeNet face parsing on the GPU: the parse graph per batch of 16 crops against the reference network restated in torch eager on the
same GPU in the same run, and generate_avatar's host / device split on a synthetic 10 s 720p clip.  Prints one JSON line.

    python tools/bench_bisenet.py [--iters 50]

Synthetic weights (oracle.bisenet_ref.synth_state_dict).  The eager numbers use oracle.bisenet_ref.forward + the bilinear resize +
arg-max with the folded weights resident on the GPU, in fp32 with TF32 off (as the reference runs), in fp16, and for the single crop
FaceParsing runs per call.  The
generate_avatar run replays detector boxes and landmarks (no S3FD, no dlib) and stands a constant encoder in for the VAE, so its
'latents' entry is host crop + LANCZOS4 time only."""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

import numpy as np
import torch

from gpu_bench import events_ms, gpu_info

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import bisenet_ref as R  # noqa: E402
from oracle import pfld_ref, s3fd_ref  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    from livetalking_b200 import engine
    from livetalking_b200.bisenet import BiSeNetNet, BiSeNetParser, gflop_per_frame
    card = ", ".join(gpu_info())
    engine.set_device(0)
    sd = R.synth_state_dict(0)
    net = BiSeNetNet.from_state_dict(sd)
    B = 16
    p = BiSeNetParser(net, B)
    crops = np.ascontiguousarray(pfld_ref.synth_video_frames(B, 512, 512, seed=1)[..., ::-1])
    p.ctx.h2d(p.buf["rgb"], crops)
    graph_ms = events_ms(p.graph.launch, args.iters, warmup=1, stream=torch.cuda.ExternalStream(p.ctx.cuda_stream))
    t0 = time.perf_counter()
    for _ in range(10):
        p.parse(crops)
    parse_ms = (time.perf_counter() - t0) / 10 * 1e3
    p.close()

    fw = R.folded(sd)
    x32 = R.prep(crops).cuda()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False

    # the oracle converts its host float64 weights on every call; the reference keeps its module on the GPU, so the eager runs
    # take device-resident copies (one per dtype, made before timing) and the timed window holds only forward, resize and arg-max
    resident = {dt: {k: (torch.from_numpy(w).to("cuda", dt), torch.from_numpy(b).to("cuda", dt)) for k, (w, b) in fw.items()}
                for dt in (torch.float32, torch.float16)}
    R._t = lambda fw_, name, like: resident[like.dtype][name]

    def run_dtype(dtype, x):
        xd = x.to(dtype)

        def run():
            with torch.no_grad():
                return R.upsample(R.forward(fw, xd)).argmax(1)
        return run
    it = max(3, args.iters // 10)
    eager32 = events_ms(run_dtype(torch.float32, x32), it, warmup=1)
    eager16 = events_ms(run_dtype(torch.float16, x32), it, warmup=1)
    eager1 = events_ms(run_dtype(torch.float32, x32[:1]), it, warmup=1)

    from livetalking_b200.plugin import musetalk_face_parsing as mfp
    from livetalking_b200.plugin import musetalk_genavatar as G
    n = 250
    tmp = tempfile.mkdtemp(prefix="bench_bisenet_")
    vid = os.path.join(tmp, "clip.avi")
    s3fd_ref.write_video(vid, pfld_ref.synth_video_frames(n, 720, 1280, seed=9))
    boxes = [(500 + (i % 20), 200 + (i % 10), 780 + (i % 20), 560 + (i % 10)) for i in range(n)]
    split = {}
    t0 = time.perf_counter()
    G.generate_avatar(vid, "bench", save_path=os.path.join(tmp, "av"), detect=lambda fr: list(boxes),
                      landmarks=R.ReplayLandmarks([R.synth_landmarks(b, seed=i) for i, b in enumerate(boxes)]),
                      face_parsing=mfp.FaceParsing(90, 90, make_parser=lambda N: BiSeNetParser(net, N)),
                      encode_latents=lambda c: np.zeros((len(c), 8, 32, 32), np.float32), timings=split)
    total = time.perf_counter() - t0
    shutil.rmtree(tmp, ignore_errors=True)
    gf = gflop_per_frame()
    print(json.dumps({"card": card, "gflop_per_crop": round(gf, 2), "batch": B, "graph_ms": round(graph_ms, 3),
                      "graph_tflops": round(gf * B / graph_ms, 1), "parse_call_ms": round(parse_ms, 2),
                      "eager_fp32_ms": round(eager32, 2), "eager_fp16_ms": round(eager16, 2), "eager_single_crop_fp32_ms": round(eager1, 2),
                      "generate_avatar_s": round(total, 2), "frames": n, "split_s": {k: round(v, 3) for k, v in split.items()}}))


if __name__ == "__main__":
    main()
