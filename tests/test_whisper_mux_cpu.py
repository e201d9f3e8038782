"""Cross-session Whisper scheduling without a GPU: MuseReal / WhisperASR in cross-session mode routing their PCM windows to one shared
grouped extractor per window layout (a stand-in for WhisperBatchFeatures), with the reference's WhisperASR bookkeeping, a close() that
leaves the shared extractor alive, and sessions outside cross-session mode keeping their own WhisperFeatures."""
import json
import os

import numpy as np

import stubs  # noqa: E402

stubs.install()

L, R = 10, 10


def fake_features(pcm, B):
    """(L + R + 2B) * 320 PCM -> (B, 50, 384) float16: a cheap function of the window, so a window routed to the wrong session shows."""
    pcm = np.asarray(pcm, np.float32)
    assert pcm.size == (L + R + 2 * B) * 320
    return np.broadcast_to(pcm[-B * 50:].reshape(B, 50, 1), (B, 50, 384)).astype(np.float16)


class FakeGroupedFeatures:
    """livetalking_b200.whisper.WhisperBatchFeatures surface: `batch` windows per call, run_groups / infer_slots -> per window features."""
    instances = []

    def __init__(self, enc, batch, groups, stride_left=10, stride_right=10, **kw):
        assert (stride_left, stride_right) == (L, R)
        self.B, self.G, self.batch = batch, groups, groups
        self.sizes, self.calls, self.closed = [], [], False
        FakeGroupedFeatures.instances.append(self)

    def infer_slots(self, pcms):
        assert 1 <= len(pcms) <= self.G and not self.closed
        self.sizes.append(len(pcms))
        self.calls.extend(np.asarray(p, np.float32).copy() for p in pcms)
        return [fake_features(p, self.B) for p in pcms]

    run_groups = infer_slots

    def close(self):
        self.closed = True


class FakeOwnFeatures:
    """livetalking_b200.whisper.WhisperFeatures surface (one session's own extractor)."""
    instances = []

    def __init__(self, enc, batch, l=10, r=10, **kw):
        self.B, self.closed = batch, False
        FakeOwnFeatures.instances.append(self)

    def run(self, pcm):
        return fake_features(pcm, self.B)

    def close(self):
        self.closed = True


class _FakeEncoder:
    D = 384


class _FakeCtx:
    def close(self):
        pass


class _FakeAvatar:
    def __init__(self, ctx, frames, masks, coords, crops, latents):
        self.n, self.lat_hw = len(frames), 32


class _FakeSession:
    def __init__(self, net, avatar, batch, paste_only=False, **kw):
        pass

    def close(self):
        pass


class _FakeUnetMux:
    def __init__(self, net, lat_hw, groups, frames_per_session, **kw):
        self.batch = groups

    def close(self):
        pass


def _patch(monkeypatch):
    from livetalking_b200.plugin import musetalk_avatar as MT
    for name, fake in (("WhisperEncoder", _FakeEncoder), ("WhisperBatchFeatures", FakeGroupedFeatures), ("WhisperFeatures", FakeOwnFeatures),
                       ("MuseTalkBatchSession", _FakeUnetMux), ("MuseTalkAvatar", _FakeAvatar), ("MuseTalkSession", _FakeSession),
                       ("Ctx", _FakeCtx)):
        monkeypatch.setattr(MT, name, fake)
    monkeypatch.setenv("LTB_MT_GROUPS", "3")
    FakeGroupedFeatures.instances.clear()
    FakeOwnFeatures.instances.clear()
    return MT


def _session(MT, model, B, sid, cross=True, l=L, r=R):
    import registry
    z = [np.zeros((4, 4, 3), np.uint8)] * 3
    payload = MT.make_avatar(z, z, [(0, 0, 4, 4)] * 3, [(0, 0, 4, 4)] * 3, [np.zeros((1, 8, 32, 32), np.float32)] * 3)
    return registry.create("avatar", "musetalk", opt=stubs.Opt(batch_size=B, ltb_cross_session=cross, sessionid=sid, l=l, r=r), model=model,
                           avatar=payload)


def _close_all(avs):
    for av in avs:
        for b in {id(x): x for x in (getattr(av.audio_processor, "batcher", None), av._batcher) if x is not None}.values():
            b.close()
        av.close()


def test_cross_session_sessions_share_one_whisper_scheduler_per_layout(monkeypatch):
    MT = _patch(monkeypatch)
    model = MT.EngineModel(_FakeCtx(), net=object(), whisper=_FakeEncoder())
    avs = [_session(MT, model, 2, s) for s in range(3)] + [_session(MT, model, 4, 3)]
    fb = avs[0].audio_processor.batcher
    assert all(isinstance(a.audio_processor, MT.SharedFeatures) for a in avs)
    assert avs[1].audio_processor.batcher is fb and avs[2].audio_processor.batcher is fb
    assert avs[3].audio_processor.batcher is not fb                       # another batch size: another window layout
    assert len(FakeGroupedFeatures.instances) == 2 and not FakeOwnFeatures.instances
    assert fb.mux is FakeGroupedFeatures.instances[0] and fb.mux.G == 3 and fb.mux.B == 2
    assert set(model._ltb_feature_batchers) == {(2, L, R), (4, L, R)}
    # every session's window comes back to that session
    for s, av in enumerate(avs[:3]):
        pcm = np.random.default_rng(s).standard_normal((L + R + 4) * 320).astype(np.float32)
        assert np.array_equal(av.audio_processor.run(pcm), fake_features(pcm, 2))
    _close_all(avs[3:])
    for av in avs[:3]:
        av.close()
    fb.close()


def test_close_leaves_the_shared_extractor_alive(monkeypatch):
    MT = _patch(monkeypatch)
    model = MT.EngineModel(_FakeCtx(), net=object(), whisper=_FakeEncoder())
    a, b = _session(MT, model, 2, 0), _session(MT, model, 2, 1)
    fb = b.audio_processor.batcher
    a.close()
    assert a.audio_processor is None and not fb.mux.closed
    pcm = np.ones((L + R + 4) * 320, np.float32)
    assert np.array_equal(b.audio_processor.run(pcm), fake_features(pcm, 2))
    c = _session(MT, model, 2, 2)                                     # a later session joins the same scheduler
    assert c.audio_processor.batcher is fb and len(FakeGroupedFeatures.instances) == 1
    b.close()
    c.close()
    fb.close()


def _golden(name):
    with open(os.path.join(os.path.dirname(__file__), "golden", "reference_host_golden.json")) as f:
        return json.load(f)[name]


def _idx(a, chunks):
    """index of the input chunk an audio frame equals, -1 for synthesised silence (the golden file's encoding)"""
    a = np.asarray(a, np.float32)
    return -1 if not a.any() else next(i for i, c in enumerate(chunks) if np.array_equal(a, c))


def test_run_step_through_the_shared_extractor_matches_the_reference_bookkeeping(monkeypatch):
    """The chunk sequence of the reference WhisperASR recording (tests/golden/reference_host_golden.json): the same PCM context reaches
    the grouped extractor, the same B (50, 384) items are queued and the same chunks are forwarded and kept."""
    MT = _patch(monkeypatch)
    want = _golden("whisper_asr")
    B = 3
    model = MT.EngineModel(_FakeCtx(), net=object(), whisper=_FakeEncoder())
    av = _session(MT, model, B, 0)
    mux = av.audio_processor.batcher.mux
    asr = av.asr
    asr.frames.clear()                                               # MuseReal warmed its ASR up on silence: start where the recording did
    while asr.output_queue.qsize():
        asr.output_queue.get()
    rng = np.random.default_rng(2)
    chunks = [rng.standard_normal(320).astype(np.float32) for _ in range(20 + 2 * B + 2)]
    for i, c in enumerate(chunks):
        asr.put_audio_frame(c, {"i": i})
    asr.warm_up()
    asr.run_step()
    feats = asr.feat_queue.get(timeout=5)
    assert [list(np.asarray(f).shape) for f in feats] == want["feat_shapes"]
    assert [[_idx(p, chunks) for p in c.reshape(-1, 320)] for c in mux.calls] == want["calls"]
    assert np.array_equal(np.stack(feats), fake_features(mux.calls[0], B))
    assert [_idx(f, chunks) for f in asr.frames] == want["frames"]
    q = asr.output_queue
    assert [[f.type, _idx(f.data, chunks)] for f in (q.get() for _ in range(q.qsize()))] == want["output_queue"]
    assert mux.sizes == [1]
    _close_all([av])


def test_sessions_outside_cross_session_mode_keep_their_own_extractor(monkeypatch):
    MT = _patch(monkeypatch)
    model = MT.EngineModel(_FakeCtx(), net=object(), whisper=_FakeEncoder())
    avs = [_session(MT, model, 2, s, cross=False) for s in range(2)]
    assert [a.audio_processor for a in avs] == FakeOwnFeatures.instances and len(FakeOwnFeatures.instances) == 2
    assert not FakeGroupedFeatures.instances and not hasattr(model, "_ltb_feature_batchers")
    own = avs[0].audio_processor
    avs[0].close()
    assert own.closed
    # a stand-in encoder (no device weights) keeps its own extractor in cross-session mode too
    stand_in = MT.EngineModel(_FakeCtx(), net=object(), whisper=object())
    c = _session(MT, stand_in, 2, 5)
    assert isinstance(c.audio_processor, FakeOwnFeatures) and not FakeGroupedFeatures.instances
    _close_all([avs[1], c])
