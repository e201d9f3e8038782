"""Cross-session HuBERT scheduling without a GPU: CrossSessionBatcher serving HuBERT group requests (one PCM window per session step)
through a stand-in grouped extractor — order, the latency rule, errors and close() — and LightReal / HubertASR in cross-session mode
routing their windows to one shared extractor, with no request for a silent session."""
import threading
import time

import numpy as np
import pytest

import stubs  # noqa: E402

stubs.install()

B, L, R = 2, 10, 10
N = (L + R + 2 * B) * 320


def fake_features(pcm):
    """(N,) PCM -> (B, 16, 1024): a cheap function of the window, so a window routed to the wrong session is visible."""
    pcm = np.asarray(pcm, np.float32)
    assert pcm.size == N
    return np.broadcast_to(pcm[-B * 16:].reshape(B, 16, 1), (B, 16, 1024)).astype(np.float32)


class FakeGroupedFeatures:
    """livetalking_b200.hubert.HubertBatchFeatures surface: `batch` windows per call, run_groups / infer_slots -> per window features."""
    instances = []

    def __init__(self, enc, batch, groups, stride_left=10, stride_right=10, **kw):
        assert (batch, stride_left, stride_right) == (B, L, R)
        self.G = self.batch = groups
        self.sizes, self.seen, self.latency, self.fail, self.gate = [], [], 0.002, None, None
        FakeGroupedFeatures.instances.append(self)

    def infer_slots(self, pcms):
        assert 1 <= len(pcms) <= self.G
        if self.gate is not None:
            self.gate.wait(10)
        time.sleep(self.latency)
        if self.fail is not None:
            raise self.fail
        self.sizes.append(len(pcms))
        self.seen.extend(float(p[0]) for p in pcms)
        return [fake_features(p) for p in pcms]

    run_groups = infer_slots

    def close(self):
        pass


def _pcm(tag):
    x = np.random.default_rng(int(tag)).standard_normal(N).astype(np.float32)
    x[0] = tag
    return x


def _batcher(groups=4, wait_ms=20.0):
    from livetalking_b200.plugin.batcher import CrossSessionBatcher
    return CrossSessionBatcher(FakeGroupedFeatures(None, B, groups), wait_ms)


def test_windows_of_many_sessions_are_grouped_in_order_and_routed_back():
    from livetalking_b200.plugin.ultralight_avatar import SharedFeatures
    b = _batcher(groups=4)
    errors, order = [], {}

    def session(sid):
        try:
            f = SharedFeatures(b)
            for k in range(20):
                pcm = _pcm(1000 * sid + k)
                assert np.array_equal(f.run(pcm), fake_features(pcm)), (sid, k)
        except Exception as e:                                  # noqa: BLE001
            errors.append(e)

    ths = [threading.Thread(target=session, args=(s,)) for s in range(6)]
    for t in ths:
        t.start()
    for t in ths:
        t.join(timeout=60)
    b.close()
    assert not errors, errors
    mux = b.mux
    assert b.slots == sum(mux.sizes) == 6 * 20 and max(mux.sizes) == 4 and b.batches < 6 * 20
    for tag in mux.seen:                                        # every session's steps reached the extractor in the order it made them
        order.setdefault(int(tag) // 1000, []).append(int(tag) % 1000)
    assert all(v == list(range(20)) for v in order.values()) and len(order) == 6


def test_latency_rule_full_rounds_go_at_once_a_lone_window_after_the_wait():
    b = _batcher(groups=3, wait_ms=60.0)
    t0 = time.monotonic()
    got = b.submit([_pcm(1)])
    dt = time.monotonic() - t0
    assert np.array_equal(got[0], fake_features(_pcm(1))) and 0.06 <= dt < 0.5 and b.mux.sizes == [1]
    b.close()
    b = _batcher(groups=3, wait_ms=5000.0)                     # a full round does not wait for the deadline
    out = [None] * 3
    ths = [threading.Thread(target=lambda k=k: out.__setitem__(k, b.submit([_pcm(10 + k)])[0])) for k in range(3)]
    t0 = time.monotonic()
    for t in ths:
        t.start()
    for t in ths:
        t.join(timeout=10)
    assert time.monotonic() - t0 < 2.0 and b.mux.sizes == [3]
    assert all(np.array_equal(out[k], fake_features(_pcm(10 + k))) for k in range(3))
    b.close()


def test_an_error_reaches_every_session_of_the_round_and_close_releases_waiters():
    b = _batcher(groups=3, wait_ms=5000.0)
    b.mux.fail = RuntimeError("extractor failure")
    errs = []

    def waiter(k):
        try:
            b.submit([_pcm(k)])
        except RuntimeError as e:
            errs.append(str(e))

    ths = [threading.Thread(target=waiter, args=(k,)) for k in range(3)]
    for t in ths:
        t.start()
    for t in ths:
        t.join(timeout=10)
    assert errs == ["extractor failure"] * 3
    # one round in the extractor (held by the gate), two windows queued behind it: close() fails the queued ones, the round in
    # flight still completes
    b.mux.fail, b.mux.gate = None, threading.Event()
    b.max_wait = 0.0
    errs.clear()
    ths = [threading.Thread(target=waiter, args=(k,)) for k in range(3)]
    ths[0].start()
    time.sleep(0.2)
    for t in ths[1:]:
        t.start()
    time.sleep(0.2)
    assert b.mux.sizes == [] and len(b._q) == 2
    threading.Timer(0.3, b.mux.gate.set).start()               # close() joins the dispatcher: let the round in flight finish
    b.close()
    for t in ths:
        t.join(timeout=10)
    assert not any(t.is_alive() for t in ths)
    assert errs == ["CrossSessionBatcher closed"] * 2 and b.mux.sizes == [1]
    with pytest.raises(RuntimeError, match="closed"):
        b.submit([_pcm(0)])


class _FakeEncoder:
    D = 1024


class _FakeUnetMux:
    def __init__(self, template, groups, frames_per_session, slots=None, return_pred=False, **kw):
        self.batch = groups

    def close(self):
        pass


class _FakeAvatar:
    def __init__(self, ctx, model, frames, faces, coords):
        self.model, self.n = model, len(frames)


class _FakeSession:
    def __init__(self, avatar, batch, **kw):
        pass

    def close(self):
        pass


def test_lightreal_cross_session_windows_go_to_one_shared_extractor(monkeypatch):
    from livetalking_b200.plugin import ultralight_avatar as UL
    import registry

    class FakeCtx:
        def close(self):
            pass

    for name, fake in (("HubertEncoder", _FakeEncoder), ("HubertBatchFeatures", FakeGroupedFeatures), ("UltraLightBatchSession", _FakeUnetMux),
                       ("UltraLightAvatar", _FakeAvatar), ("UltraLightModel", lambda ctx, sd: sd), ("UltraLightSession", _FakeSession),
                       ("Ctx", FakeCtx)):
        monkeypatch.setattr(UL, name, fake)
    monkeypatch.setenv("LTB_UL_GROUPS", "3")
    FakeGroupedFeatures.instances.clear()
    model = (UL.EngineAudio(FakeCtx(), _FakeEncoder()), None)
    avs = []
    for s in range(2):
        payload = UL.make_avatar({"w": s}, [np.zeros((4, 4, 3), np.uint8)] * 3, [np.zeros((4, 4, 3), np.uint8)] * 3, [(0, 0, 4, 4)] * 3)
        avs.append(registry.create("avatar", "ultralight", opt=stubs.Opt(batch_size=B, ltb_cross_session=True, sessionid=s), model=model,
                                   avatar=payload))
    assert len(FakeGroupedFeatures.instances) == 1
    mux = FakeGroupedFeatures.instances[0]
    fb = avs[0].audio_processor.batcher
    assert isinstance(avs[0].audio_processor, UL.SharedFeatures) and avs[1].audio_processor.batcher is fb and fb.mux is mux and mux.G == 3
    # session 0 speaks, session 1 stays silent: its batch and the previous one are silence, so it makes no request
    speech = np.random.default_rng(0).standard_normal(2 * B * 320).astype(np.float32)
    for c in range(2 * B):
        avs[0].asr.put_audio_frame(speech[c * 320:(c + 1) * 320], {})
    for av in avs:
        av.asr.run_step()
    feats0, feats1 = avs[0].asr.feat_queue.get(timeout=5), avs[1].asr.feat_queue.get(timeout=5)
    window = np.concatenate([np.zeros((L + R) * 320, np.float32), speech])
    assert np.array_equal(np.stack(feats0), fake_features(window))
    assert len(feats1) == B and all(f.shape == (10, 1024) and not f.any() for f in feats1)
    assert fb.slots == 1 and mux.sizes == [1]
    fb.close()
    avs[0]._batcher.close()
    for av in avs:
        av.close()
