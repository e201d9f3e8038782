"""UltraLight cross-session batching without a GPU: ``LightReal`` in cross-session mode under the reference's REAL three-thread driving
(unmodified ``avatars/base_avatar.py``, deterministic engine stand-ins of tests/test_ultralight_threads.py, one shared scheduler for
two sessions with their own avatars and audio), and the slot policy of ``UltraLightBank`` (hits, least-recently-used eviction, never
evicting a slot the current batch uses) on a fake context that records the device copies."""
import threading
import time

import numpy as np
import pytest

import ref_runtime as RR
import test_ultralight_threads as T
from livetalking_b200.ops import DevTensor


class FakeBatchSession:
    """livetalking_b200.ultralight.UltraLightBatchSession surface: the mux of the cross-session scheduler (oracle arithmetic)."""
    instances = []

    def __init__(self, template, groups, frames_per_session, slots=None, return_pred=False, **kw):
        self.batch, self.Bs, self.return_pred, self.sizes = groups, frames_per_session, return_pred, []
        assert slots == 2 * groups
        FakeBatchSession.instances.append(self)

    def infer_slots(self, requests):
        from oracle import ultralight_ref as U
        assert 1 <= len(requests) <= self.batch
        time.sleep(0.004)
        self.sizes.append(len(requests))
        outs = []
        for av, index, feats in requests:
            feats = np.asarray(feats, np.float32)
            idxs = [U.mirror_index(av.n, index + i) for i in range(self.Bs)]
            pred = np.stack([T.fake_net(av.faces[j], feats[i]) for i, j in enumerate(idxs)])
            outs.append(pred if self.return_pred else
                        np.stack([U.lightreal_paste(pred[i], av.frames[j], av.faces[j], av.coords[j]) for i, j in enumerate(idxs)]))
        return outs

    def close(self):
        pass


def _assets(seed):
    rng = np.random.default_rng(seed)
    faces = [rng.integers(0, 256, (168, 168, 3), dtype=np.uint8) for _ in range(T.N_AV)]
    frames = [rng.integers(0, 256, (T.H, T.W, 3), dtype=np.uint8) for _ in range(T.N_AV)]
    coords = [(20 + i, 10 + 2 * i, 140 + i, 150 + 2 * i) for i in range(T.N_AV - 1)] + [(40, 30, 208, 198)]
    return faces, frames, coords


@pytest.mark.skipif(not RR.available(), reason="reference checkout not present (GPU box)")
@pytest.mark.parametrize("return_pred", [False, True], ids=["fused", "reference_pred"])
def test_lightreal_cross_session_mode_under_the_real_render_loops(tmp_path, monkeypatch, return_pred):
    """opt.ltb_cross_session: two LightReal sessions (own avatars, own audio) with the reference's own three threads each; their
    inference_batch calls are group requests to ONE shared scheduler; every emitted frame matches its own audio window and index."""
    all_assets = [_assets(30 + s) for s in range(2)]
    pristine = [[f.copy() for f in a[1]] for a in all_assets]
    FakeBatchSession.instances.clear()
    with RR.reference_runtime(str(tmp_path)) as rt:
        UL = rt.load_ultralight()
        for name, fake in (("UltraLightSession", T.FakeSession), ("UltraLightAvatar", T.FakeAvatar), ("UltraLightModel", T.FakeModel),
                           ("HubertFeatures", T.FakeHubertFeatures), ("Ctx", T.FakeCtx), ("UltraLightBatchSession", FakeBatchSession)):
            monkeypatch.setattr(UL, name, fake)
        model = (UL.EngineAudio(T.FakeCtx(), encoder=object()), None)
        avatars = []
        for s in range(2):
            faces, frames, coords = all_assets[s]
            payload = UL.make_avatar({"weights": s}, frames, faces, coords)
            opt = RR.make_opt(batch_size=T.B, ltb_return_pred=return_pred, ltb_cross_session=True, sessionid=s)
            avatars.append(rt.registry.create("avatar", "ultralight", opt=opt, model=model, avatar=payload))
        assert avatars[0]._batcher is not None and avatars[0]._batcher is avatars[1]._batcher
        sinks, spies, threads = [], [], []
        quit_event = threading.Event()
        for s, av in enumerate(avatars):
            sink = RR.RecordingSink()
            av.output, av.tts = sink, RR.NullTTS()
            pulled = [rt.AudioFrameData(data=np.zeros(320, np.float32), type=1, userdata={}) for _ in range(20)]
            RR.spy_audio_frames(av.asr, pulled)
            sinks.append(sink)
            spies.append(pulled)
            threads.append(threading.Thread(target=av.render, args=(quit_event,)))
            threads.append(threading.Thread(target=RR.feed_bursts, args=(av, [90, 70, 110, 50]), kwargs={"seed": s}))
        for t in threads:
            t.start()
        t0 = time.time()
        while min(len(s.frames) for s in sinks) < 220 and time.time() - t0 < 150:
            time.sleep(0.02)
        quit_event.set()
        for t in threads:
            t.join(timeout=40)
        assert not any(t.is_alive() for t in threads), "render() did not stop"
        for s in range(2):
            faces, _frames, coords = all_assets[s]
            n = len(sinks[s].frames)
            assert n >= 200, f"session {s}: only {n} frames emitted"
            exp = T.replay_expected(spies[s], n, faces, pristine[s], coords)
            assert len(exp) >= n - T.B
            n_speech = 0
            for j in range(min(n, len(exp))):
                assert np.array_equal(sinks[s].frames[j], exp[j]), f"session {s} frame {j}: not the frame of its own audio window / index"
                n_speech += int(not np.array_equal(exp[j], T.watermark(pristine[s][rt.mirror_index(T.N_AV, j)].copy())))
            assert 40 <= n_speech <= min(n, len(exp)) - 20, (s, n_speech)
        mux = FakeBatchSession.instances[0]
        assert len(FakeBatchSession.instances) == 1 and sum(mux.sizes) == avatars[0]._batcher.slots and max(mux.sizes) <= mux.batch
        avatars[0]._batcher.close()
        for av in avatars:
            av.close()


# ---------------------------------------------------------------------------------------------------------------- bank slot policy
class _RecordingCtx:
    """alloc / d2d of livetalking_b200.ops.Ctx without a device: fake addresses, copies recorded."""

    def __init__(self):
        self.next, self.copies = 1 << 20, []

    def alloc(self, shape, dtype=np.float16, zero=False):
        t = DevTensor(self.next, shape, dtype)
        self.next += (t.nbytes + 255) // 256 * 256
        return t

    def d2d(self, dst, src, nbytes):
        self.copies.append((dst, src, nbytes))


class _Net:
    def __init__(self, ctx, cout=32):
        self.ts = [ctx.alloc((cout, 16)), ctx.alloc((cout,), np.float32)]

    def weight_tensors(self):
        return self.ts


def test_bank_slots_hit_evict_least_recently_used_and_keep_the_batch():
    from livetalking_b200.ultralight import UltraLightBank
    ctx = _RecordingCtx()
    nets = [_Net(ctx) for _ in range(5)]
    bank = UltraLightBank(ctx, nets[0], 3)
    w_buf, b_buf = bank.stacked(nets[0].ts[0]), bank.stacked(nets[0].ts[1])
    assert w_buf.shape == (3, 32, 16) and b_buf.shape == (3, 32) and bank.nbytes == w_buf.nbytes + b_buf.nbytes
    # misses fill the empty slots in order; each load copies every tensor into its slot
    assert [bank.slot_of(nets[i]) for i in range(3)] == [0, 1, 2] and bank.loads == 3
    assert ctx.copies[2:4] == [(w_buf.ptr + 1 * 1024, nets[1].ts[0].ptr, 1024), (b_buf.ptr + 1 * 128, nets[1].ts[1].ptr, 128)]
    # hits copy nothing
    n = len(ctx.copies)
    assert bank.slot_of(nets[1]) == 1 and bank.slot_of(nets[0]) == 0 and bank.loads == 3 and len(ctx.copies) == n
    # a miss evicts the least recently used slot (2: net 2, untouched since it was loaded)
    assert bank.slot_of(nets[3]) == 2 and bank.loads == 4 and ctx.copies[-1][1] == nets[3].ts[1].ptr
    # ... unless the current batch uses it: slots 1 (LRU now) and 0 are kept, so slot 2 goes
    assert bank.slot_of(nets[4], keep=[1, 0]) == 2
    assert bank.slot_of(nets[3], keep=[2]) == 1                  # net 3 was evicted above; LRU outside the batch is slot 1
    assert bank.slot_of(nets[0], keep=[0, 1, 2]) == 0           # a hit is served even when every slot is in the batch
    with pytest.raises(RuntimeError):
        bank.slot_of(nets[1], keep=[0, 1, 2])                   # a miss with every slot in the batch
    with pytest.raises(ValueError):
        bank.slot_of(_Net(ctx, cout=48))                        # another architecture


def test_bank_batch_of_distinct_networks_never_evicts_its_own_slots():
    """Every call of a batch session asks for its groups' networks in turn with the slots taken so far kept: within one call no
    slot is handed out twice, whatever the bank held before."""
    from livetalking_b200.ultralight import UltraLightBank
    ctx = _RecordingCtx()
    nets = [_Net(ctx) for _ in range(7)]
    bank = UltraLightBank(ctx, nets[0], 4)
    rng = np.random.default_rng(0)
    for _call in range(200):
        picks = rng.choice(len(nets), size=int(rng.integers(1, 5)), replace=False)
        keep = []
        for k in picks:
            s = bank.slot_of(nets[k], keep)
            assert s not in keep
            keep.append(s)
        for k, s in zip(picks, keep):                           # every group's network is in its slot after the call
            assert bank.slot_of(nets[k], keep) == s
