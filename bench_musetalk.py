#!/usr/bin/env python
"""Secondary benchmark: MuseTalk 256x256, batch 8 (BASELINE.json configs[2]) on one H100.

    python bench_musetalk.py [--steps K] [--warmup W] [--batch 8]

Reports device-timed frames/s for (a) the ONLINE path the reference runs per step (Whisper features -> PE -> UNet ->
VAE decode -> blend paste-back; latents pre-encoded, F7 in SURVEY.md) and (b) the FULL chain of configs[2] (the same plus
VAE encode of masked + reference crops every step), with the algorithmic FLOPs of BASELINE.md §2.
The contract benchmark (`bench.py`) stays on the wav2lip256 workload the BASELINE metric is quoted on."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

GFLOP_ONLINE = 800.0      # UNet 177.8 + VAE decode 622.2 (BASELINE.md §2)
GFLOP_FULL = 1345.4       # + 2 x VAE encode 272.7
GFLOP_WHISPER_STEP = 37.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=8)
    args = ap.parse_args()
    import torch
    from livetalking_b200 import configs, engine, synth
    from livetalking_b200.graph import GraphSession
    from livetalking_b200.musetalk import MuseTalkAvatar, MuseTalkModel, MuseTalkSession
    from livetalking_b200.ops import Ctx
    from livetalking_b200.whisper import WhisperEncoder, WhisperFeatures

    torch.cuda.set_device(0)
    engine.set_device(0)
    B = args.batch
    ucfg, vcfg = configs.UNetConfig(), configs.VAEConfig()
    t0 = time.time()
    ctx = Ctx()
    net = MuseTalkModel(ctx, synth.random_unet_state_dict(ucfg), synth.random_vae_state_dict(vcfg), ucfg, vcfg, with_encoder=True)
    wenc = WhisperEncoder(ctx, synth.random_whisper_state_dict())
    frames, masks, coords, crops, latents = synth.synthetic_musetalk_avatar(n=16)
    av = MuseTalkAvatar(ctx, frames, masks, coords, crops, latents)
    sess = MuseTalkSession(net, av, B, ctx=ctx)      # one stream for the whole timed chain (device-resident benchmark)
    wf = WhisperFeatures(wenc, B, out=sess.audio_in, out_rows=64, ctx=ctx)          # features land directly in the UNet's audio buffer
    load_s = time.time() - t0
    # encoder graph (config 3): B crops -> latents
    crops_u8 = ctx.upload(np.random.default_rng(0).integers(0, 256, (B, 256, 256, 3), dtype=np.uint8))
    enc_out = ctx.alloc((B, 32, 32, 16), np.float16, zero=True)
    enc = GraphSession(ctx)
    enc.capture(lambda b: net.emit_vae_encode(b, crops_u8, enc_out))
    enc_graph = enc.graph

    pcm = synth.sine_audio(5.0)[:wf.n]
    wf.run_async(pcm)
    ctx.sync()
    stream = torch.cuda.ExternalStream(ctx.cuda_stream)

    def timed(fn, steps):
        for _ in range(args.warmup):
            fn(0)
        ctx.sync()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for k in range(steps):
            fn(k * B)
        e1.record(stream)
        ctx.sync()
        return e0.elapsed_time(e1) / steps

    def online(i):
        wf.run_async(None)            # log-mel + Whisper encoder + slicing (PCM resident)
        sess.step_async(i)            # PE + UNet + VAE decode + blend paste-back

    def full(i):
        enc_graph.launch()            # VAE encode (masked + reference) of B crops
        online(i)

    l0 = ctx.launch_count
    ms_online = timed(online, args.steps)
    launches = (ctx.launch_count - l0) // (args.steps + args.warmup)
    ms_full = timed(full, args.steps)
    ms_whisper = timed(lambda i: wf.run_async(None), args.steps)
    ms_unet_vae = timed(lambda i: sess.infer_async(i, None), args.steps)
    ms_paste = timed(lambda i: sess.paste_batch_async(i), args.steps)
    ms_enc = timed(lambda i: enc_graph.launch(), args.steps)
    peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))) if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else {}
    peak = float(peaks.get("bf16_tflops_sustained", 1400.0))
    tf_online = (GFLOP_ONLINE * B + GFLOP_WHISPER_STEP) / ms_online
    tf_full = (GFLOP_FULL * B + GFLOP_WHISPER_STEP) / ms_full
    out = {
        "metric": "lip-sync frames/sec (MuseTalk 256x256, batch %d, fp16)" % B, "unit": "frames/s", "n_gpus": 1, "steps": args.steps,
        "warmup": args.warmup, "dtype": "f16 (fp32 accumulate)", "data": "synthetic",
        "online": {"value": round(1000.0 * B / ms_online, 2), "ms_per_step": round(ms_online, 3),
                   "what": "whisper features + PE + UNet + VAE decode + blend paste-back (latents pre-encoded, as the reference's live path)",
                   "achieved_tflops": round(tf_online, 1), "frac_of_peak": round(tf_online / peak, 4)},
        "full_chain": {"value": round(1000.0 * B / ms_full, 2), "ms_per_step": round(ms_full, 3),
                       "what": "configs[2]: VAE encode x2 + UNet + VAE decode (+ whisper, paste)",
                       "achieved_tflops": round(tf_full, 1), "frac_of_peak": round(tf_full / peak, 4)},
        "breakdown_ms": {"whisper": round(ms_whisper, 3), "unet_plus_vae_decode": round(ms_unet_vae, 3), "blend_paste": round(ms_paste, 3),
                         "vae_encode_x2": round(ms_enc, 3)},
        "gpu_launches_per_step": int(launches), "model_load_s": round(load_s, 1), "peak_tflops": peak,
        "config": {"workload": "MuseTalk 256x256 batch %d, VAE enc -> UNet -> VAE dec, 1xH100, fp16 (BASELINE.json configs[2])" % B},
    }
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()
