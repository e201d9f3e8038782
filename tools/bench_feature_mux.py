"""Audio-feature cross-session batching: G sessions' windows through one grouped encoder forward against G independent extractors.

    python tools/bench_feature_mux.py --encoder hubert|whisper [--groups 1,2,4,8] [--frames F] [--repeats 5] [--min-ms M]
                                      [--e2e-groups 4,8] [--e2e-frames F]

One (l + r + 2B) x 320-sample window per session and step (l = r = 10, the plugin's defaults), random weights of the real layout:
  hubert:  hubert-large (24 layers, d 1024, FFN 4096); defaults --frames 4,16 --e2e-frames 4,16 --min-ms 2000.
  whisper: Whisper-tiny encoder (4 layers, d 384, FFN 1536), always over the 30-s padded window (1500 tokens); defaults --frames 2,8
           --e2e-frames 2,8 --min-ms 400.

  (1) extractor: for every (G, B), G sessions' windows resident on the device
      (a) "sessions": G HubertFeatures / WhisperFeatures graphs, each on its own stream (what every session runs without
          cross-session mode);
      (b) "grouped":  one HubertBatchFeatures / WhisperBatchFeatures graph of G groups (what cross-session mode runs).
      CUDA events around gated chunks of 16 steps after warm-up, at least --min-ms of device time per measurement.  The two arms
      alternate, --repeats times each; every repeat is reported, so the spread is visible next to the median.
  (2) end to end, the avatar's cross-session mode with the encoder included: G sessions with their own avatars and audio.  A round
      is every session's feature window (host PCM in -> host features out, "features") followed by one batch-session round
      ("round"): for hubert an UltraLightBatchSession round (host features -> host composited 720p frames), for whisper a
      MuseTalkBatchSession round (full-size UNet + VAE decoder, 32x32 latents; host features -> host (B, 256, 256, 3) predictions).
      "before" runs the G per-session extractors from G threads (each session's ASR thread), "after" one grouped extractor call;
      the batch session is the same object in both arms.  Wall clock over >= --min-ms, arms alternated --repeats times.
Prints one JSON line with per-arm times, speed-ups, the largest grouped-vs-session feature difference, and the GPU name and power
limit read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

DEFAULTS = {"hubert": {"frames": "4,16", "e2e_frames": "4,16", "min_ms": 2000.0},
            "whisper": {"frames": "2,8", "e2e_frames": "2,8", "min_ms": 400.0}}


def _extractors(encoder: str):
    """-> (encoder class, random state dict, grouped extractor class, per-session extractor class)."""
    from livetalking_b200 import synth
    if encoder == "hubert":
        from livetalking_b200.hubert import HubertBatchFeatures, HubertEncoder, HubertFeatures
        return HubertEncoder, synth.random_hubert_state_dict(), HubertBatchFeatures, HubertFeatures
    from livetalking_b200.whisper import WhisperBatchFeatures, WhisperEncoder, WhisperFeatures
    return WhisperEncoder, synth.random_whisper_state_dict(), WhisperBatchFeatures, WhisperFeatures


def _round_setup(encoder: str, mctx, n_avatars: int):
    """-> (avatars, per-session audio, make_mux(G, B)): the batch session a cross-session round of this encoder's avatar runs."""
    from livetalking_b200 import synth
    if encoder == "hubert":
        from livetalking_b200.ultralight import UltraLightAvatar, UltraLightBatchSession, UltraLightModel
        from oracle import ultralight_ref as U
        fr, fa, co = synth.synthetic_ultralight_avatar(n=16)
        avs = [UltraLightAvatar(mctx, UltraLightModel(mctx, U.synth_state_dict(k)), fr, fa, co) for k in range(n_avatars)]
        audio = [synth.sine_audio(10.0) * (0.5 + 0.1 * k) for k in range(n_avatars)]
        return avs, audio, lambda G, B: UltraLightBatchSession(avs[0].model, G, B)
    from livetalking_b200 import configs
    from livetalking_b200.musetalk import MuseTalkAvatar, MuseTalkBatchSession, MuseTalkModel
    net = MuseTalkModel(mctx, synth.random_unet_state_dict(configs.UNetConfig()), synth.random_vae_state_dict(configs.VAEConfig()),
                        configs.UNetConfig(), configs.VAEConfig(), with_encoder=False)
    avs = [MuseTalkAvatar(mctx, *synth.synthetic_musetalk_avatar(n=16, hw=32, seed=100 + g)) for g in range(n_avatars)]
    audio = [synth.sine_audio(10.0, freq=220.0 + 40.0 * k) for k in range(n_avatars)]
    return avs, audio, lambda G, B: MuseTalkBatchSession(net, 32, G, B)


def _device_ms_per_step(torch, stream, gate, enqueue, min_ms, extra_streams=()):
    """Chunks of 16 gated steps (short enough that the host enqueues them inside the gate's hold) until min_ms of device time."""
    from bench import timed_steps
    total, steps = 0.0, 0
    while total < min_ms:
        total += timed_steps(torch, stream, gate, enqueue, 16, extra_streams)
        steps += 16
    return total / steps


def _windows(n, G, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(n) / 16000.0
    return [(0.3 * np.sin(2 * np.pi * (180 + 30 * g) * t) + 0.05 * rng.standard_normal(n)).astype(np.float32) for g in range(G)]


def _summary(a, b):
    ma, mb = statistics.median(a), statistics.median(b)
    return {"sessions_ms": [round(v, 3) for v in a], "grouped_ms": [round(v, 3) for v in b],
            "sessions_ms_median": round(ma, 3), "grouped_ms_median": round(mb, 3), "speedup_median": round(ma / mb, 3),
            "speedup_range": [round(min(x / y for x, y in zip(a, b)), 3), round(max(x / y for x, y in zip(a, b)), 3)]}


def extractor_rows(torch, enc, grouped, single, groups, frames, repeats, min_ms, warmup):
    from bench import Gate
    rows = []
    for B in frames:
        for G in groups:
            hb = grouped(enc, B, G)
            ss = [single(enc, B) for _ in range(G)]
            pcms = _windows(hb.n, G, B * 100 + G)
            ref = [s.run(p).astype(np.float32) for s, p in zip(ss, pcms)]
            got = hb.run_groups(pcms)
            diff = max(float(np.abs(got[g].astype(np.float32) - ref[g]).max() / np.abs(ref[g]).max()) for g in range(G))
            streams = [torch.cuda.ExternalStream(s.ctx.cuda_stream) for s in ss]
            gate_a = Gate(torch, streams[0])
            stream_b = torch.cuda.ExternalStream(hb.ctx.cuda_stream)
            gate_b = Gate(torch, stream_b)

            def step_a(k):
                for s in ss:
                    s.run_async(None)

            def step_b(k):
                hb.graph.launch()

            for k in range(warmup):
                step_a(k)
                step_b(k)
            torch.cuda.synchronize()
            a, b = [], []
            for _ in range(repeats):
                a.append(_device_ms_per_step(torch, streams[0], gate_a, step_a, min_ms, streams[1:]))
                b.append(_device_ms_per_step(torch, stream_b, gate_b, step_b, min_ms))
            for o in (*ss, hb):
                o.close()
            del streams, stream_b
            torch.cuda.synchronize()
            rows.append({"groups": G, "frames_per_session": B, **_summary(a, b), "max_rel_feature_diff": float(f"{diff:.3e}")})
            print(json.dumps(rows[-1]), file=sys.stderr, flush=True)
    return rows


def e2e_rows(torch, encoder, enc, grouped, single, groups, frames, repeats, min_ms, warmup):
    from livetalking_b200.ops import Ctx
    rows = []
    mctx = Ctx()
    avs, audio, make_mux = _round_setup(encoder, mctx, max(groups))
    for B in frames:
        for G in groups:
            mux = make_mux(G, B)
            hb = grouped(enc, B, G)
            ss = [single(enc, B) for _ in range(G)]
            n = hb.n
            pool = ThreadPoolExecutor(max_workers=G)

            def pcm(k, r):
                o = (r * 2 * B * 320) % (audio[k].size - n)
                return np.ascontiguousarray(audio[k][o:o + n], np.float32)

            arms = {
                "features_before": lambda r: list(pool.map(lambda k: ss[k].run(pcm(k, r)), range(G))),
                "features_after": lambda r: hb.run_groups([pcm(k, r) for k in range(G)]),
            }
            arms["round_before"] = lambda r: mux.infer_groups([(avs[k], r * B, f) for k, f in enumerate(arms["features_before"](r))])
            arms["round_after"] = lambda r: mux.infer_groups([(avs[k], r * B, f) for k, f in enumerate(arms["features_after"](r))])
            for fn in arms.values():
                for r in range(warmup):
                    fn(r)
            res = {name: [] for name in arms}
            for _ in range(repeats):
                for name, fn in arms.items():
                    rounds, t0 = 0, time.perf_counter()
                    while (time.perf_counter() - t0) * 1000.0 < min_ms:
                        fn(rounds)
                        rounds += 1
                    res[name].append((time.perf_counter() - t0) * 1000.0 / rounds)
            pa, pb = arms["round_before"](3), arms["round_after"](3)
            diff = max(int(np.abs(pa[k].astype(np.int16) - pb[k].astype(np.int16)).max()) for k in range(G))
            pool.shutdown()
            for o in (*ss, hb, mux):
                o.close()
            torch.cuda.synchronize()
            feat, rnd = _summary(res["features_before"], res["features_after"]), _summary(res["round_before"], res["round_after"])
            rows.append({"groups": G, "frames_per_session": B,
                         "features": {k.replace("sessions", "before").replace("grouped", "after"): v for k, v in feat.items()},
                         "round": {k.replace("sessions", "before").replace("grouped", "after"): v for k, v in rnd.items()},
                         "round_fps_median": {"before": round(G * B * 1000.0 / rnd["sessions_ms_median"], 1),
                                              "after": round(G * B * 1000.0 / rnd["grouped_ms_median"], 1)},
                         "max_u8_round_diff": diff})
            print(json.dumps(rows[-1]), file=sys.stderr, flush=True)
    mctx.close()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--encoder", choices=sorted(DEFAULTS), required=True)
    ap.add_argument("--groups", default="1,2,4,8")
    ap.add_argument("--frames")
    ap.add_argument("--e2e-groups", default="4,8")
    ap.add_argument("--e2e-frames")
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--min-ms", type=float)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    for k, v in DEFAULTS[args.encoder].items():
        if getattr(args, k) is None:
            setattr(args, k, v)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_feature_mux: no CUDA device (this measurement exists only on the GPU)")
    from bench_ultralight_mux import gpu_info
    from livetalking_b200 import engine
    from livetalking_b200.ops import Ctx
    engine.set_device(0)
    torch.cuda.init()
    gpu = gpu_info(torch)
    ctx = Ctx()
    encoder_cls, sd, grouped, single = _extractors(args.encoder)
    enc = encoder_cls(ctx, sd)
    ints = lambda s: [int(v) for v in s.split(",") if v]                          # noqa: E731
    ext = extractor_rows(torch, enc, grouped, single, ints(args.groups), ints(args.frames), args.repeats, args.min_ms, args.warmup)
    e2e = (e2e_rows(torch, args.encoder, enc, grouped, single, ints(args.e2e_groups), ints(args.e2e_frames), args.repeats, args.min_ms,
                    args.warmup) if args.e2e_groups else [])
    ctx.close()
    print(json.dumps({"what": f"{args.encoder} features for G sessions: G independent {single.__name__} graphs (own streams) vs one "
                              f"{grouped.__name__} graph; and cross-session rounds with the encoder before / after grouping it",
                      "timing": {"extractor": f"CUDA events, gated chunks of 16 steps, >= {args.min_ms} ms per measurement, arms "
                                              f"alternated x{args.repeats}, {args.warmup} warm-up steps",
                                 "e2e": f"wall clock over >= {args.min_ms} ms per measurement, arms alternated x{args.repeats}, host PCM in"},
                      "gpu": gpu, "extractor": ext, "e2e": e2e}))


if __name__ == "__main__":
    main()
