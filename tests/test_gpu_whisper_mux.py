"""GPU: cross-session batching for Whisper — the grouped log-mel kernels against the single-window op and transformers'
WhisperFeatureExtractor, WhisperBatchFeatures (G sessions' windows in one encoder forward) against WhisperFeatures on each window alone
and against transformers' WhisperModel, independence of the groups, partial rounds, and MuseReal sessions in cross-session mode whose
Whisper windows go through the shared grouped extractor."""
import os
import sys
import threading

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(__file__))
import stubs  # noqa: E402
from test_gpu_whisper import _reference  # noqa: E402

pytestmark = pytest.mark.gpu


def _model(seed=0):
    """The random-init Whisper-tiny encoder of test_gpu_whisper, widened so the features have some dynamic range."""
    from transformers import WhisperConfig, WhisperModel
    torch.manual_seed(seed)
    cfg = WhisperConfig(d_model=384, encoder_layers=4, encoder_attention_heads=6, encoder_ffn_dim=1536, decoder_layers=1,
                        decoder_attention_heads=6, decoder_ffn_dim=64, num_mel_bins=80, max_source_positions=1500)
    model = WhisperModel(cfg).eval()
    with torch.no_grad():
        for n, p in model.encoder.named_parameters():
            if p.ndim >= 2 and "embed_positions" not in n:
                p.mul_(4.0)
            elif n.endswith("bias"):
                p.add_(torch.randn_like(p) * 0.05)
    return model


def _window(n, seed, amp=0.3):
    """Two tones (distinct per seed) + noise at amplitude `amp`; amp 0 is digital silence."""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / 16000.0
    x = np.sin(2 * np.pi * (180.0 + 45.0 * seed) * t) + 0.33 * np.sin(2 * np.pi * (1500.0 + 110.0 * seed) * t) + 0.17 * rng.standard_normal(n)
    return (amp * x).astype(np.float32)


def _windows(n, G, seed):
    """G distinct windows; with G >= 3 group 1 is silent and group 2 loud (each window is clamped to its own maximum)."""
    amps = [0.3, 0.0, 0.95, 0.05][:G] if G >= 3 else [0.3] * G
    return [_window(n, seed + g, a) for g, a in enumerate(amps)]


@pytest.fixture(scope="module")
def whisper():
    from livetalking_b200 import engine
    from livetalking_b200.ops import Ctx
    from livetalking_b200.whisper import WhisperEncoder
    engine.set_device(0)
    model = _model()
    ctx = Ctx()
    enc = WhisperEncoder(ctx, model.state_dict())
    yield model, enc
    ctx.close()


def test_grouped_logmel_matches_single_window_op_and_transformers():
    from transformers import WhisperFeatureExtractor
    from livetalking_b200 import engine
    from livetalking_b200.ops import Ctx
    from livetalking_b200.whisper import N_FRAMES, N_MELS, slaney_mel_filterbank
    engine.set_device(0)
    ctx = Ctx()
    G, n = 4, (10 + 10 + 2 * 8) * 320
    pcms = _windows(n, G, seed=2)
    fb = ctx.upload(slaney_mel_filterbank())
    pcm = ctx.upload(np.stack(pcms))
    logspec = ctx.alloc((G, N_MELS * N_FRAMES), np.float32, zero=True)
    gmax = ctx.alloc((G,), np.int32, zero=True)
    f16 = ctx.alloc((G, N_FRAMES, N_MELS), np.float16, zero=True)
    f32 = ctx.alloc((G, N_MELS, N_FRAMES), np.float32, zero=True)
    ctx.whisper_logmel(pcm, n, fb, logspec, gmax, f16, f32, G=G)
    got16, got32 = ctx.download(f16), ctx.download(f32)
    ws = ctx.alloc((N_MELS * N_FRAMES,), np.float32, zero=True)
    m1 = ctx.alloc((4,), np.int32, zero=True)
    o16 = ctx.alloc((N_FRAMES, N_MELS), np.float16, zero=True)
    o32 = ctx.alloc((N_MELS, N_FRAMES), np.float32, zero=True)
    fe = WhisperFeatureExtractor()
    for g in range(G):
        ctx.whisper_logmel(ctx.upload(pcms[g]), n, fb, ws, m1, o16, o32)
        assert np.array_equal(got16[g], ctx.download(o16)) and np.array_equal(got32[g], ctx.download(o32)), g
        want = fe(pcms[g], return_tensors="np", sampling_rate=16000).input_features[0]
        np.testing.assert_allclose(got32[g], want, atol=1e-4 if not pcms[g].any() else 2e-3, err_msg=f"window {g}")
    assert not pcms[1].any() and got32[1].max() < got32[2].max()      # the silent window is not clamped by the loud one
    ctx.close()


def _plans(enc, make):
    """make(ctx) builds an extractor on ctx -> (extractor, {layer: conv plan of the kernel instance it runs}).  Layers are named by
    their weights; the unfused attention GEMMs (no weights) are 'attention'."""
    from livetalking_b200.ops import Ctx
    names = {id(enc.conv1): "conv1", id(enc.conv2): "conv2"}
    for i, L in enumerate(enc.layers):
        names.update({id(L["attn"].qkv): f"layers.{i}.qkv", id(L["attn"].out): f"layers.{i}.out_proj", id(L["fc1"]): f"layers.{i}.fc1",
                      id(L["fc2"]): f"layers.{i}.fc2"})
    ctx = Ctx()
    plans, conv = {}, ctx.conv

    def recording_conv(x, w, out, **kw):
        plans.setdefault(names.get(id(w), "attention"), ctx.conv_plan(x, w, out, **kw))
        return conv(x, w, out, **kw)

    ctx.conv = recording_conv
    return ctx, make(ctx), plans


@pytest.mark.parametrize("B", [2, 8])
@pytest.mark.parametrize("G", [1, 3, 4])
def test_grouped_windows_match_single_window_and_transformers(whisper, G, B):
    from livetalking_b200.whisper import WhisperBatchFeatures, WhisperFeatures
    model, enc = whisper
    cg, hb, plans_g = _plans(enc, lambda c: WhisperBatchFeatures(enc, B, G, ctx=c))
    c1, single, plans_1 = _plans(enc, lambda c: WhisperFeatures(enc, B, ctx=c))
    rerouted = {k: {f: (v, plans_g[k][f]) for f, v in plans_1[k].items() if plans_g[k][f] != v} for k in sorted(plans_1)
                if plans_g.get(k) != plans_1[k]}                             # layer -> {plan field: (1 window, G windows)}
    print(f"G={G} B={B}: layers the conv planner routes differently at {G}x1500 rows: {rerouted or 'none'}")
    pcms = _windows(hb.n, G, seed=11 * B + G)
    got = hb.run_groups(pcms)
    assert len(got) == G and hb.batch == G
    worst = 0.0
    for g in range(G):
        alone = single.run(pcms[g])
        assert got[g].shape == alone.shape == (B, 50, 384) and got[g].dtype == np.float16
        a, x = alone.astype(np.float32), got[g].astype(np.float32)
        if G == 1:
            assert np.array_equal(x, a)
        d = np.abs(x - a).max() / np.abs(a).max()
        worst = max(worst, d)
        assert d <= 2e-3, (g, d, f"layers planned differently at {G}x1500 rows: {rerouted or 'none'}")
        _f, _h, want = _reference(pcms[g], model, B)
        err = np.abs(x - want)
        assert err.max() <= 4e-2 * np.abs(want).max() and err.mean() <= 1e-2 * np.abs(want).mean(), (g, err.max(), err.mean(), rerouted)
    print(f"G={G} B={B}: largest grouped vs single-window difference {worst:.2e} of max")
    for o, c in ((single, c1), (hb, cg)):
        o.close()
        c.close()


def test_groups_do_not_see_each_other(whisper):
    from livetalking_b200.whisper import WhisperBatchFeatures
    _model_, enc = whisper
    G, B = 4, 2
    hb = WhisperBatchFeatures(enc, B, G)
    pcms = _windows(hb.n, G, seed=3)
    base = hb.run_groups(pcms)
    for g in (0, 1, 2):
        changed = list(pcms)
        changed[g] = _window(hb.n, 99 + g, 0.6)
        out = hb.run_groups(changed)
        assert not np.array_equal(out[g], base[g])
        for k in range(G):
            if k != g:
                assert np.array_equal(out[k], base[k]), (g, k)
    hb.close()


def test_partial_rounds_match_the_full_round(whisper):
    from livetalking_b200.whisper import WhisperBatchFeatures
    _model_, enc = whisper
    G, B = 4, 2
    hb = WhisperBatchFeatures(enc, B, G)
    pcms = _windows(hb.n, G, seed=5)
    full = hb.run_groups(pcms)
    for k in range(1, G):
        hb.run_groups(_windows(hb.n, G, seed=40 + k))            # other windows left in the groups a partial round does not use
        part = hb.run_groups(pcms[:k])
        assert len(part) == k
        for g in range(k):
            assert np.array_equal(part[g], full[g]), (k, g)
    with pytest.raises(ValueError):
        hb.run_groups(pcms + pcms[:1])
    with pytest.raises(ValueError):
        hb.run_groups([pcms[0][:-320]])
    with pytest.raises(ValueError):
        hb.run_groups([])
    hb.close()


def test_musereal_cross_session_whisper_windows_match_sessions_alone():
    """Three MuseReal sessions in cross-session mode, each with its own audio and avatar, run WhisperASR.run_step and inference_batch
    from their own threads: every feat_queue item matches the one the same session queues alone (2e-3 of max), and the frames match
    the session's own MuseTalkSession on the same features (<= 2 u8 steps, PSNR >= 50 dB: the batched UNet may pick other tiles)."""
    stubs.install()
    from livetalking_b200.plugin import musetalk_avatar as MT
    from oracle import musetalk_ref as M
    from oracle.wav2lip_ref import psnr_u8
    import registry
    us, vs = M.synth_unet_state_dict(M.UNET_SMALL), M.synth_vae_state_dict(M.VAE_SMALL)
    model = MT.make_model(us, vs, _model(seed=1).state_dict(), M.UNET_SMALL, M.VAE_SMALL)
    B, n, S, steps = 2, 3, 3, 3
    rng = np.random.default_rng(8)
    coords = [(60, 30, 190, 170), (50, 20, 200, 180), (70, 40, 180, 160)]
    crops = [(30, 10, 230, 195), (20, 5, 240, 198), (40, 20, 220, 190)]
    masks = [np.repeat((np.linspace(0, 255, (c[3] - c[1]))[:, None] * np.ones((1, c[2] - c[0]))).astype(np.uint8)[..., None], 3, 2) for c in crops]
    avatars = []
    for s in range(S):
        lat, _ = M.synth_latents_and_audio(n, seed=20 + s)
        frames = list(rng.integers(0, 256, (n, 200, 260 + 4 * s, 3), dtype=np.uint8))
        avatars.append(MT.make_avatar(frames, masks, coords, crops, [lat[i:i + 1] for i in range(n)], model))
    audio = [[_window(2 * B * 320, 70 + 10 * k + s, 0.2 + 0.2 * k) for s in range(steps)] for k in range(S)]

    def session(k, cross):
        return registry.create("avatar", "musetalk", opt=stubs.Opt(batch_size=B, ltb_cross_session=cross, sessionid=k), model=model,
                               avatar=avatars[k])

    def drive(av, k, out):
        for s in range(steps):
            for c in range(2 * B):
                av.asr.put_audio_frame(audio[k][s][c * 320:(c + 1) * 320], {})
            av.asr.run_step()
            out.append(av.asr.feat_queue.get(timeout=60))
        out.append(av.inference_batch(k, out[0]))

    alone = []
    for k in range(S):
        av, out = session(k, False), []
        drive(av, k, out)
        alone.append((av, out[:steps]))
    sessions = [session(k, True) for k in range(S)]
    fb = sessions[0].audio_processor.batcher
    assert isinstance(sessions[0].audio_processor, MT.SharedFeatures) and all(a.audio_processor.batcher is fb for a in sessions)
    assert isinstance(fb.mux, MT.WhisperBatchFeatures) and fb.mux.G == int(os.environ.get("LTB_MT_GROUPS", "4"))
    results = [[] for _ in range(S)]
    ths = [threading.Thread(target=drive, args=(sessions[k], k, results[k])) for k in range(S)]
    for t in ths:
        t.start()
    for t in ths:
        t.join(timeout=300)
    assert not any(t.is_alive() for t in ths)
    for k in range(S):
        own, want_feats = alone[k]
        for s in range(steps):
            got, want = results[k][s], want_feats[s]
            assert len(got) == len(want) == B
            for i in range(B):
                g, w = np.asarray(got[i], np.float32), np.asarray(want[i], np.float32)
                assert g.shape == (50, 384) and np.abs(g - w).max() <= 2e-3 * np.abs(w).max(), (k, s, i)
        pred = results[k][steps]
        pred_alone = own.inference_batch(k, results[k][0])
        assert pred.shape == (B, 256, 256, 3) and np.abs(pred.astype(int) - pred_alone.astype(int)).max() <= 2, k
        assert psnr_u8(pred, pred_alone) >= 50.0, (k, psnr_u8(pred, pred_alone))
        own.close()
    assert fb.slots == S * steps
    print(f"Whisper rounds: {fb.batches} for {fb.slots} windows")
    fb.close()
    fb.mux.close()
    sessions[0]._batcher.close()
    sessions[0]._batcher.mux.close()
    for a in sessions:
        a.close()
