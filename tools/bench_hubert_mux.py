"""HuBERT cross-session batching: G sessions' windows through one grouped encoder forward against G independent extractors.

    python tools/bench_hubert_mux.py [--groups 1,2,4,8] [--frames 4,16] [--min-ms 2000] [--e2e-groups 4,8] [--e2e-frames 4,16]

hubert-large (24 layers, d 1024, FFN 4096, random weights of the real layout), one (l + r + 2B) x 320-sample window per session and
step (l = r = 10, the plugin's defaults).

  (1) extractor: for every (G, B), G sessions' windows resident on the device
      (a) "sessions": G HubertFeatures graphs, each on its own stream (what every session runs without cross-session mode);
      (b) "grouped":  one HubertBatchFeatures graph of G groups (what cross-session mode runs).
      CUDA events around gated chunks of steps after warm-up, repeated until at least --min-ms of device time per arm.
  (2) end to end, UltraLight cross-session mode with HuBERT included: G sessions with their own avatars, networks and audio, one
      round = every session's HuBERT window (host PCM -> host features) + one UltraLightBatchSession round (host features -> host
      composited 720p frames).  "before" runs the G per-session extractors from G threads (each session's HubertASR thread) and
      "after" runs one HubertBatchFeatures call; the U-Net round is the same object in both arms.  Wall clock over >= --min-ms.
Prints one JSON line with per-arm times, speed-ups, the largest grouped-vs-session feature difference, and the GPU name and power
limit read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def _device_ms_per_step(torch, stream, gate, enqueue, min_ms, extra_streams=()):
    """Chunks of 16 gated steps (short enough that the host enqueues them inside the gate's hold) until min_ms of device time."""
    from bench import timed_steps
    total, steps = 0.0, 0
    while total < min_ms:
        total += timed_steps(torch, stream, gate, enqueue, 16, extra_streams)
        steps += 16
    return total / steps, steps


def extractor_rows(torch, enc, groups, frames, min_ms, warmup):
    from bench import Gate
    from livetalking_b200.hubert import HubertBatchFeatures, HubertFeatures
    rows = []
    for B in frames:
        for G in groups:
            hb = HubertBatchFeatures(enc, B, G)
            rng = np.random.default_rng(B * 100 + G)
            t = np.arange(hb.n) / 16000.0
            pcms = [(0.3 * np.sin(2 * np.pi * (180 + 30 * g) * t) + 0.05 * rng.standard_normal(hb.n)).astype(np.float32) for g in range(G)]
            ss = [HubertFeatures(enc, B) for _ in range(G)]
            ref = [s.run(p) for s, p in zip(ss, pcms)]
            got = hb.run_groups(pcms)
            diff = max(float(np.abs(got[g] - ref[g]).max() / np.abs(ref[g]).max()) for g in range(G))
            streams = [torch.cuda.ExternalStream(s.ctx.cuda_stream) for s in ss]

            def step_a(k):
                for s in ss:
                    s.run_async(None)

            for k in range(warmup):
                step_a(k)
            torch.cuda.synchronize()
            ms_a, n_a = _device_ms_per_step(torch, streams[0], Gate(torch, streams[0]), step_a, min_ms, streams[1:])
            for s in ss:
                s.close()
            del ss, streams
            stream = torch.cuda.ExternalStream(hb.ctx.cuda_stream)

            def step_b(k):
                hb.graph.launch()

            for k in range(warmup):
                step_b(k)
            torch.cuda.synchronize()
            ms_b, n_b = _device_ms_per_step(torch, stream, Gate(torch, stream), step_b, min_ms)
            hb.close()
            del stream
            torch.cuda.synchronize()
            rows.append({"groups": G, "frames_per_session": B, "tokens_per_window": hb.Tc,
                         "sessions_ms_per_step": round(ms_a, 3), "grouped_ms_per_step": round(ms_b, 3),
                         "speedup": round(ms_a / ms_b, 3), "sessions_steps_timed": n_a, "grouped_steps_timed": n_b,
                         "max_rel_feature_diff": float(f"{diff:.3e}")})
            print(json.dumps(rows[-1]), file=sys.stderr, flush=True)
    return rows


def e2e_rows(torch, enc, groups, frames, min_ms, warmup):
    from livetalking_b200 import synth
    from livetalking_b200.hubert import HubertBatchFeatures, HubertFeatures
    from livetalking_b200.ops import Ctx
    from livetalking_b200.ultralight import UltraLightAvatar, UltraLightBatchSession, UltraLightModel
    from oracle import ultralight_ref as U
    rows = []
    mctx = Ctx()
    fr, fa, co = synth.synthetic_ultralight_avatar(n=16)
    avs = [UltraLightAvatar(mctx, UltraLightModel(mctx, U.synth_state_dict(k)), fr, fa, co) for k in range(max(groups))]
    for B in frames:
        audio = [synth.sine_audio(10.0) * (0.5 + 0.1 * k) for k in range(max(groups))]
        for G in groups:
            mux = UltraLightBatchSession(avs[0].model, G, B)
            hb = HubertBatchFeatures(enc, B, G)
            ss = [HubertFeatures(enc, B) for _ in range(G)]
            n = hb.n
            pool = ThreadPoolExecutor(max_workers=G)

            def pcm(k, r):
                o = (r * 2 * B * 320) % (audio[k].size - n)
                return np.ascontiguousarray(audio[k][o:o + n], np.float32)

            def before(r):
                feats = list(pool.map(lambda k: ss[k].run(pcm(k, r)), range(G)))
                return mux.infer_groups([(avs[k], r * B, feats[k]) for k in range(G)])

            def after(r):
                feats = hb.run_groups([pcm(k, r) for k in range(G)])
                return mux.infer_groups([(avs[k], r * B, feats[k]) for k in range(G)])

            res = {}
            for name, fn in (("before", before), ("after", after)) * 2:          # alternated twice, the second pass is reported
                for r in range(warmup):
                    fn(r)
                rounds, t0 = 0, time.perf_counter()
                while (time.perf_counter() - t0) * 1000.0 < min_ms:
                    fn(rounds)
                    rounds += 1
                res[name] = (time.perf_counter() - t0) * 1000.0 / rounds
            a, b = before(3), after(3)
            diff = max(int(np.abs(a[k].astype(np.int16) - b[k].astype(np.int16)).max()) for k in range(G))
            pool.shutdown()
            for o in (*ss, hb, mux):
                o.close()
            torch.cuda.synchronize()
            rows.append({"groups": G, "frames_per_session": B,
                         "before_fps": round(G * B * 1000.0 / res["before"], 1), "after_fps": round(G * B * 1000.0 / res["after"], 1),
                         "before_ms_per_round": round(res["before"], 3), "after_ms_per_round": round(res["after"], 3),
                         "speedup": round(res["before"] / res["after"], 3), "max_u8_frame_diff": diff})
            print(json.dumps(rows[-1]), file=sys.stderr, flush=True)
    mctx.close()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--groups", default="1,2,4,8")
    ap.add_argument("--frames", default="4,16")
    ap.add_argument("--e2e-groups", default="4,8")
    ap.add_argument("--e2e-frames", default="4,16")
    ap.add_argument("--min-ms", type=float, default=2000.0)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_hubert_mux: no CUDA device (this measurement exists only on the GPU)")
    from bench_ultralight_mux import gpu_info
    from livetalking_b200 import engine, synth
    from livetalking_b200.hubert import HubertEncoder
    from livetalking_b200.ops import Ctx
    engine.set_device(0)
    torch.cuda.init()
    ctx = Ctx()
    enc = HubertEncoder(ctx, synth.random_hubert_state_dict())
    ints = lambda s: [int(v) for v in s.split(",") if v]                          # noqa: E731
    ext = extractor_rows(torch, enc, ints(args.groups), ints(args.frames), args.min_ms, args.warmup)
    e2e = e2e_rows(torch, enc, ints(args.e2e_groups), ints(args.e2e_frames), args.min_ms, args.warmup)
    ctx.close()
    print(json.dumps({"what": "hubert-large features for G sessions: G independent HubertFeatures graphs (own streams) vs one "
                              "HubertBatchFeatures graph; and UltraLight cross-session rounds with HuBERT before / after grouping it",
                      "timing": {"extractor": f"CUDA events, gated chunks of 16 steps, >= {args.min_ms} ms per arm, {args.warmup} warm-up steps",
                                 "e2e": f"wall clock over >= {args.min_ms} ms per arm, host PCM in, host frames out"},
                      "gpu": gpu_info(torch), "extractor": ext, "e2e": e2e}))


if __name__ == "__main__":
    main()
