"""GPU: cross-session batching for HuBERT — HubertBatchFeatures (G sessions' windows in one encoder forward) against HubertFeatures on
each window alone and against transformers' HubertModel, independence of the groups, partial rounds, and LightReal sessions in
cross-session mode whose HuBERT windows go through the shared grouped extractor."""
import os
import sys
import threading

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(__file__))
import stubs  # noqa: E402
from test_gpu_ultralight import _hubert  # noqa: E402

pytestmark = pytest.mark.gpu


def _window(n, seed, amp=0.3):
    """Tone + noise + DC (the signal of test_gpu_ultralight's HuBERT test) at amplitude `amp`; amp 0 is digital silence."""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / 16000.0
    f0 = 150.0 + 40.0 * seed
    x = np.sin(2 * np.pi * f0 * t) + 0.33 * np.sin(2 * np.pi * 1900 * t) + 0.17 * rng.standard_normal(n) + 0.07
    return (amp * x).astype(np.float32)


def _windows(n, G, seed):
    """G distinct windows; with G >= 3 group 1 is silent and group 2 loud (each window is normalised on its own)."""
    amps = [0.3, 0.0, 0.95, 0.05][:G] if G >= 3 else [0.3] * G
    return [_window(n, seed + g, a) for g, a in enumerate(amps)]


@pytest.fixture(scope="module")
def hubert():
    from livetalking_b200 import engine
    from livetalking_b200.hubert import HubertEncoder
    from livetalking_b200.ops import Ctx
    engine.set_device(0)
    model = _hubert()
    ctx = Ctx()
    enc = HubertEncoder(ctx, model.state_dict())
    yield model, enc
    ctx.close()


def _hf_windows(model, pcm, B):
    from transformers import Wav2Vec2FeatureExtractor
    from oracle import ultralight_ref as U
    fe = Wav2Vec2FeatureExtractor(feature_size=1, sampling_rate=16000, padding_value=0.0, do_normalize=True, return_attention_mask=True)
    with torch.no_grad():
        hid = model(fe(pcm, return_tensors="pt", sampling_rate=16000).input_values).last_hidden_state[0].numpy()
    ref = U.trim_features(hid, pcm.size)
    return ref[U.window_rows(ref.shape[0], B, 5.0)]


@pytest.mark.parametrize("B", [4, 16])
@pytest.mark.parametrize("G", [1, 3, 4])
def test_grouped_windows_match_single_window_and_transformers(hubert, G, B):
    from livetalking_b200.hubert import HubertBatchFeatures, HubertFeatures
    model, enc = hubert
    hb = HubertBatchFeatures(enc, B, G)
    pcms = _windows(hb.n, G, seed=11 * B + G)
    got = hb.run_groups(pcms)
    assert len(got) == G and hb.batch == G
    single = HubertFeatures(enc, B)
    worst = 0.0
    for g in range(G):
        alone = single.run(pcms[g])
        assert got[g].shape == alone.shape == (B, 16, 1024) and got[g].dtype == np.float32
        if G == 1:
            assert np.array_equal(got[g], alone)
        d = np.abs(got[g] - alone).max() / np.abs(alone).max()
        worst = max(worst, d)
        assert d <= 2e-3, (g, d)
        want = _hf_windows(model, pcms[g], B)
        err = np.abs(got[g] - want)
        assert err.max() <= 4e-2 * np.abs(want).max() and err.mean() <= 1e-2 * np.abs(want).mean(), (g, err.max(), np.abs(want).max())
    print(f"G={G} B={B}: largest grouped vs single-window difference {worst:.2e} of max")
    single.close()
    hb.close()


def test_groups_do_not_see_each_other(hubert):
    from livetalking_b200.hubert import HubertBatchFeatures
    _model, enc = hubert
    G, B = 4, 4
    hb = HubertBatchFeatures(enc, B, G)
    pcms = _windows(hb.n, G, seed=3)
    base = hb.run_groups(pcms)
    for g in (0, 2):
        changed = list(pcms)
        changed[g] = _window(hb.n, 99 + g, 0.6)
        out = hb.run_groups(changed)
        assert not np.array_equal(out[g], base[g])
        for k in range(G):
            if k != g:
                assert np.array_equal(out[k], base[k]), (g, k)
    hb.close()


def test_partial_rounds_match_the_full_round(hubert):
    from livetalking_b200.hubert import HubertBatchFeatures
    _model, enc = hubert
    G, B = 4, 4
    hb = HubertBatchFeatures(enc, B, G)
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
    hb.close()


def test_grouped_attention_without_the_fused_kernel(hubert, monkeypatch):
    """Builder.attention with batch G and a key count that is not a multiple of 16 on the GEMM + softmax + GEMM path."""
    from livetalking_b200.hubert import HubertBatchFeatures, HubertFeatures
    from livetalking_b200.graph import Builder
    _model, enc = hubert
    monkeypatch.setattr(Builder, "FUSE_ATTENTION", False)
    G, B = 3, 4
    hb = HubertBatchFeatures(enc, B, G)
    assert hb.Tc % 16
    single = HubertFeatures(enc, B)
    pcms = _windows(hb.n, G, seed=8)
    for g, out in enumerate(hb.run_groups(pcms)):
        alone = single.run(pcms[g])
        assert np.abs(out - alone).max() <= 2e-3 * np.abs(alone).max(), g
    single.close()
    hb.close()


@pytest.fixture(scope="module")
def three_avatars():
    from oracle import ultralight_ref as U
    from test_gpu_ultralight_mux import _assets
    return [(U.synth_state_dict(k), *_assets(3 + k, seed=60 + k)) for k in range(3)]


def test_lightreal_cross_session_hubert_windows_match_sessions_alone(three_avatars):
    """Three LightReal sessions in cross-session mode, each with its own audio and avatar, run HubertASR.run_step and inference_batch
    from their own threads: every feat_queue item equals the one the same session queues alone (to 2e-3 of max), a session whose
    batch and previous batch are silent makes no HuBERT request, and the frames match the oracle on the session's own windows."""
    stubs.install()
    from livetalking_b200.plugin import ultralight_avatar as UL
    from oracle import ultralight_ref as U
    import registry
    model = UL.make_model(_hubert(layers=1, inter=512).state_dict())
    B, S, steps = 4, 3, 3
    speech = [[True, True, True], [True, False, True], [True, False, False]]      # session 2: two silent batches in a row at the end
    audio = [[_window(2 * B * 320, 70 + 10 * k + s) for s in range(steps)] for k in range(S)]

    def session(k, cross):
        sd, fr, fa, co = three_avatars[k]
        payload = UL.make_avatar(sd, list(fr), list(fa), co)
        return registry.create("avatar", "ultralight", opt=stubs.Opt(batch_size=B, ltb_cross_session=cross, sessionid=k), model=model,
                               avatar=payload)

    def drive(av, k, out):
        for s in range(steps):
            if speech[k][s]:
                for c in range(2 * B):
                    av.asr.put_audio_frame(audio[k][s][c * 320:(c + 1) * 320], {})
            av.asr.run_step()
            out.append(av.asr.feat_queue.get(timeout=60))
        out.append(av.inference_batch(k, out[0]))

    alone = []
    for k in range(S):
        av, out = session(k, False), []
        drive(av, k, out)
        alone.append(out[:steps])
        av.close()
    sessions = [session(k, True) for k in range(S)]
    fb = sessions[0].audio_processor.batcher
    assert isinstance(sessions[0].audio_processor, UL.SharedFeatures) and all(a.audio_processor.batcher is fb for a in sessions)
    assert isinstance(fb.mux, UL.HubertBatchFeatures) and fb.mux.G == int(os.environ.get("LTB_UL_GROUPS", "4"))
    results = [[] for _ in range(S)]
    ths = [threading.Thread(target=drive, args=(sessions[k], k, results[k])) for k in range(S)]
    for t in ths:
        t.start()
    for t in ths:
        t.join(timeout=300)
    assert not any(t.is_alive() for t in ths)
    for k in range(S):
        for s in range(steps):
            got, want = results[k][s], alone[k][s]
            assert len(got) == len(want) == B
            for i in range(B):
                if want[i].shape == (10, 1024):                  # the silence default: no HuBERT request
                    assert got[i].shape == (10, 1024) and not got[i].any(), (k, s, i)
                    continue
                assert got[i].shape == (16, 1024) and np.abs(got[i] - want[i]).max() <= 2e-3 * np.abs(want[i]).max(), (k, s, i)
        sd, fr, fa, co = three_avatars[k]
        feats = [np.asarray(f, np.float32) for f in results[k][0]]
        ref = U.lightreal_inference_batch(sd, list(fa), k, feats)
        for i in range(B):
            idx = U.mirror_index(len(fa), k + i)
            frame = sessions[k].paste_back_frame(results[k][steps][i], idx)
            assert U.psnr_u8(frame, U.lightreal_paste(ref[i], fr[idx], fa[idx], co[idx])) >= 40.0, (k, i)
    assert fb.slots == sum(sum(1 for s in range(steps) if speech[k][s] or (s > 0 and speech[k][s - 1])) for k in range(S))
    print(f"HuBERT rounds: {fb.batches} for {fb.slots} windows")
    fb.close()
    fb.mux.close()
    sessions[0]._batcher.close()
    sessions[0]._batcher.mux.close()
    for a in sessions:
        a.close()
