"""UltraLight cross-session batching: G independent sessions against one grouped launch.

    python tools/bench_ultralight_mux.py [--steps 20] [--warmup 3] [--groups 1,2,4,8] [--frames 4,16]

For G distinct synthetic avatars (each with its own network, oracle.ultralight_ref.synth_state_dict(k)) and Bs frames per session it
times the U-Net + paste-back step
  (a) "sessions": G UltraLightSessions, each on its own stream with its own graph (what LightReal runs without cross-session mode);
  (b) "batched":  one UltraLightBatchSession of G groups (what LightReal runs with LTB_CROSS_SESSION=1), weights in a bank of 2G slots.
HuBERT is left out of both arms: every session runs the same feature extractor in either mode.  Features are resident on the device
in both arms.  Timing: CUDA events around `steps` steps enqueued behind a spin kernel (bench.py's gate), after `warmup` steps.
Prints one JSON line with frames/s of both arms, launches per step, device bytes held per session, the largest u8 difference between
the arms' frames on the same inputs, and the GPU name and power limit read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info(torch) -> dict:
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit"], info["max_sm_clock"] = [v.strip() for v in q.split(",")[:2]]
    except Exception as e:   # noqa: BLE001 - reported, not hidden
        info["power_limit"] = f"unavailable ({e!r})"
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--groups", default="1,2,4,8")
    ap.add_argument("--frames", default="4,16")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_ultralight_mux: no CUDA device (this measurement exists only on the GPU)")
    from bench import Gate, timed_steps
    from livetalking_b200 import engine
    from livetalking_b200.ops import Ctx, DevTensor
    from livetalking_b200.ultralight import UltraLightAvatar, UltraLightBatchSession, UltraLightModel, UltraLightSession
    from oracle import ultralight_ref as U
    engine.set_device(0)
    torch.cuda.init()
    groups = [int(g) for g in args.groups.split(",")]
    frames_per = [int(b) for b in args.frames.split(",")]
    H, W, n_frames = 360, 480, 8
    mctx = Ctx()
    avs = []
    for k in range(max(groups)):
        _i, _a, faces = U.synth_inputs(n_frames, seed=50 + k)
        frames = np.random.default_rng(k).integers(0, 256, (n_frames, H, W, 3), dtype=np.uint8)
        avs.append(UltraLightAvatar(mctx, UltraLightModel(mctx, U.synth_state_dict(k)), frames, faces, [(100 + k, 80, 300 + k, 290)] * n_frames))
    rng = np.random.default_rng(0)
    rows = []
    for Bs in frames_per:
        for G in groups:
            feats = [rng.standard_normal((Bs, 16, 1024)).astype(np.float32) for _ in range(G)]
            # (a) G independent sessions
            free0 = torch.cuda.mem_get_info()[0]
            ss = [UltraLightSession(avs[k], Bs) for k in range(G)]
            for s_, f in zip(ss, feats):
                s_.infer_paste(0, f)
            torch.cuda.synchronize()
            bytes_a = (free0 - torch.cuda.mem_get_info()[0]) / G
            ref = [s_.ctx.download(s_.frames_out) for s_ in ss]
            streams = [torch.cuda.ExternalStream(s_.ctx.cuda_stream) for s_ in ss]

            def step_a(k):
                for s_ in ss:
                    s_.step_async((k * Bs) % n_frames)

            l0 = sum(s_.ctx.launch_count for s_ in ss)
            step_a(0)
            launches_a = sum(s_.ctx.launch_count for s_ in ss) - l0
            for k in range(args.warmup):
                step_a(k)
            torch.cuda.synchronize()
            ms_a = timed_steps(torch, streams[0], Gate(torch, streams[0]), step_a, args.steps, streams[1:]) / args.steps
            for s_ in ss:
                s_.close()
            del ss, streams
            torch.cuda.synchronize()
            # (b) one batched session of G groups
            free0 = torch.cuda.mem_get_info()[0]
            mux = UltraLightBatchSession(avs[0].model, G, Bs)
            got = mux.infer_groups([(avs[k], 0, feats[k]) for k in range(G)])
            torch.cuda.synchronize()
            bytes_b = (free0 - torch.cuda.mem_get_info()[0]) / G
            diff = max(int(np.abs(got[k].astype(np.int16) - ref[k].astype(np.int16)).max()) for k in range(G))
            stream = torch.cuda.ExternalStream(mux.ctx.cuda_stream)

            def step_b(k):
                mux.step_async([(avs[g], (k * Bs) % n_frames, None) for g in range(G)])

            l0 = mux.ctx.launch_count
            step_b(0)
            launches_b = mux.ctx.launch_count - l0
            for k in range(args.warmup):
                step_b(k)
            torch.cuda.synchronize()
            ms_b = timed_steps(torch, stream, Gate(torch, stream), step_b, args.steps) / args.steps
            mux.close()
            del mux, stream
            torch.cuda.synchronize()
            rows.append({"groups": G, "frames_per_session": Bs,
                         "sessions_fps": round(G * Bs * 1000.0 / ms_a, 1), "batched_fps": round(G * Bs * 1000.0 / ms_b, 1),
                         "sessions_ms_per_step": round(ms_a, 3), "batched_ms_per_step": round(ms_b, 3),
                         "sessions_launches_per_step": launches_a, "batched_launches_per_step": launches_b,
                         "sessions_bytes_per_session": int(bytes_a), "batched_bytes_per_session": int(bytes_b),
                         "max_u8_diff": diff})
    mctx.close()
    print(json.dumps({"what": "UltraLight U-Net + paste-back step, G sessions with distinct avatars and networks: G independent sessions "
                              "(own stream / graph each) vs one grouped batch launch (UltraLightBatchSession)",
                      "excluded": "HuBERT feature extraction (identical in both arms)",
                      "timing": f"CUDA events, {args.steps} gated steps after {args.warmup} warm-up steps; features resident",
                      "gpu": gpu_info(torch), "rows": rows}))


if __name__ == "__main__":
    main()
