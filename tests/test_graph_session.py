"""The captured-graph session lifecycle (livetalking_b200.graph.GraphSession): capture on the eager pass's buffers, and close()
giving back exactly what the session allocated.

Without a GPU every session class is built on a recording stand-in for ``Ctx`` (fake addresses, ops recorded as no-ops) from the
synthetic weights the GPU tests use: on a borrowed ctx close() frees the session's builder temporaries, its own buffers, its lazily
made outputs and its weight bank, and nothing it was handed; on an owned ctx it closes every context it made.  The GPU test builds
every class on one shared real ``Ctx`` and checks its live allocations the same way, then that a session built afterwards on that
ctx computes what the first one did."""
import contextlib
import os
import threading
import types
from functools import lru_cache

import numpy as np
import pytest

from livetalking_b200.graph import GraphSession
from livetalking_b200.ops import DevTensor

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


class _Graph:
    def __init__(self):
        self.closed, self.launches = False, 0

    def launch(self):
        self.launches += 1

    def close(self):
        self.closed = True


class _RecordingCtx:
    """livetalking_b200.ops.Ctx without a device: fake addresses, the live allocations, every op (a no-op) recorded in order."""

    def __init__(self):
        self.next, self.live, self.ops = 1 << 20, {}, []
        self.closed = self.capturing = False
        self.lock = threading.RLock()

    def alloc(self, shape, dtype=np.float16, zero=False):
        assert not self.closed
        t = DevTensor(self.next, shape, dtype)
        self.next += (t.nbytes + 255) // 256 * 256
        self.live[t.ptr] = t
        return t

    def upload(self, arr, dtype=None):
        arr = np.ascontiguousarray(arr, dtype=dtype)
        return self.alloc(arr.shape, arr.dtype)

    def free(self, t):
        del self.live[t.ptr]                           # a pointer this ctx does not hold is an error, as in ltb_dev_free

    def download(self, t, out=None, sync=True):
        return np.zeros(t.shape, t.dtype) if out is None else out

    def close(self):
        self.closed = True

    @contextlib.contextmanager
    def capture(self):
        holder = types.SimpleNamespace(graph=None)
        self.capturing = True
        try:
            yield holder
        finally:
            self.capturing = False
        holder.graph = _Graph()

    def __getattr__(self, name):                       # sync, h2d, d2d and every op
        if name.startswith("_"):
            raise AttributeError(name)
        return lambda *a, **kw: self.ops.append((name, self.capturing))


# ---------------------------------------------------------------------------------------------------------------- capture
class _Session(GraphSession):
    """A session whose graph is `emit`, with one buffer of its own."""

    def __init__(self, emit, ctx=None):
        super().__init__(ctx)
        try:
            self.own = self.alloc((4,), np.float32)
            self.capture(emit)
        except BaseException:
            self.close()
            raise


def test_captured_pass_gets_the_eager_pass_buffers_in_order():
    ctx = _RecordingCtx()
    passes = []

    def emit(b):
        got = [b.new(2, 3, 4, 16), b.new(5, 32), b.new(1, 1, 1, 16)]
        b.ctx.conv(*got)
        passes.append([t.ptr for t in got])

    s = _Session(emit, ctx)
    assert len(passes) == 2 and passes[0] == passes[1]
    assert [op for op in ctx.ops if op[0] == "conv"] == [("conv", False), ("conv", True)]
    assert isinstance(s.graph, _Graph)


@pytest.mark.parametrize("shapes", [[(2, 3, 4, 16), (5, 31)], [(2, 3, 4, 16)], [(2, 3, 4, 16), (5, 32), (16,)]],
                         ids=["other-shape", "fewer", "more"])
def test_a_replay_that_differs_from_the_eager_pass_raises(shapes):
    ctx = _RecordingCtx()
    before = dict(ctx.live)
    calls = []

    def emit(b):
        calls.append(1)
        for s in (shapes if len(calls) == 2 else [(2, 3, 4, 16), (5, 32)]):
            b.new(*s)

    with pytest.raises(RuntimeError):
        _Session(emit, ctx)
    assert ctx.live == before and not ctx.closed


@pytest.mark.parametrize("failing_pass", [1, 2], ids=["eager", "captured"])
@pytest.mark.parametrize("borrowed", [True, False], ids=["borrowed", "owned"])
def test_an_emit_that_raises_leaves_nothing_behind(monkeypatch, failing_pass, borrowed):
    made = _patch_ctx(monkeypatch)
    ctx = _RecordingCtx() if borrowed else None
    calls = []

    def emit(b):
        calls.append(1)
        b.new(8, 16)
        if len(calls) == failing_pass:
            raise KeyError("emit")
        b.new(4, 16)

    with pytest.raises(KeyError):
        _Session(emit, ctx)
    if borrowed:
        assert ctx.live == {} and not ctx.closed and made == []
    else:
        assert len(made) == 1 and made[0].closed                 # closing the owned ctx frees everything on it


# ---------------------------------------------------------------------------------------------------------------- every session class
def _patch_ctx(monkeypatch):
    """Ctx() in the session base makes recording stand-ins; returns the list of those made."""
    import livetalking_b200.graph as G
    made = []

    def make():
        made.append(_RecordingCtx())
        return made[-1]
    monkeypatch.setattr(G, "Ctx", make)
    return made


@lru_cache(None)
def _weights(name):
    from livetalking_b200 import synth
    if name == "ultralight":
        return synth.random_ultralight_state_dict()
    if name == "hubert":
        return synth.random_hubert_state_dict(layers=1)
    if name == "whisper":
        return synth.random_whisper_state_dict()       # 4 layers: the feature slice reads all 5 hidden states
    if name == "musetalk":
        from oracle import musetalk_ref as M
        return M.UNET_SMALL, M.VAE_SMALL, M.synth_unet_state_dict(M.UNET_SMALL, fast=True), M.synth_vae_state_dict(M.VAE_SMALL, fast=True)
    if name == "s3fd":
        from oracle import s3fd_ref as R
        return R.synth_state_dict(0)
    if name == "bisenet":
        from oracle import bisenet_ref as R
        return R.synth_state_dict(0)
    from oracle import pfld_ref as R
    return R.synth_state_dict(0), R.read_mean_face(os.path.join(GOLDEN, "pfld_mean_face.txt"))


def _ul_avatars(mctx, k=2):
    from livetalking_b200 import synth
    from livetalking_b200.ultralight import UltraLightAvatar, UltraLightModel
    model = UltraLightModel(mctx, _weights("ultralight"))
    return model, [UltraLightAvatar(mctx, model, *synth.synthetic_ultralight_avatar(n=2, H=240, W=320, bbox=(40, 30, 200, 190), seed=s))
                   for s in range(k)]


def _mt(mctx):
    from livetalking_b200 import synth
    from livetalking_b200.musetalk import MuseTalkAvatar, MuseTalkModel
    ucfg, vcfg, us, vs = _weights("musetalk")
    model = MuseTalkModel(mctx, us, vs, ucfg, vcfg, with_encoder=False)
    return model, [MuseTalkAvatar(mctx, *synth.synthetic_musetalk_avatar(n=2, H=400, W=500, bbox=(150, 100, 350, 300), seed=s))
                   for s in range(2)]


def _feats(*shape, seed=0):
    return np.random.default_rng(seed).standard_normal(shape).astype(np.float32) * 0.5


def _u8(*shape, seed=0):
    return np.random.default_rng(seed).integers(0, 256, shape, dtype=np.uint8)


# name -> case(model ctx) -> (make(session ctx or None) -> session, tensors handed to the session, exercise(session) -> outputs): the
# case uploads weights and avatars; exercise runs the session on seeded inputs and makes what a session makes lazily (paste contexts,
# per-group outputs, bank loads)
def _case_ultralight(mctx):
    from livetalking_b200.ultralight import FACE, UltraLightSession
    _m, (av, _) = _ul_avatars(mctx)
    return lambda ctx: UltraLightSession(av, 2, ctx=ctx), [], \
        lambda s: (s.infer_paste(0, _feats(2, 16, 1024)), s.paste_pred(_feats(FACE, FACE, 3) * 255, 1))


def _case_ultralight_paste_only(mctx):
    from livetalking_b200.ultralight import FACE, UltraLightSession
    _m, (av, _) = _ul_avatars(mctx)
    return lambda ctx: UltraLightSession(av, 2, ctx=ctx, paste_only=True), [], lambda s: s.paste_pred(_feats(FACE, FACE, 3) * 255, 0)


def _case_ultralight_batch(mctx):
    from livetalking_b200.ultralight import UltraLightBatchSession
    model, avs = _ul_avatars(mctx)
    return lambda ctx: UltraLightBatchSession(model, 2, 2, ctx=ctx), [], \
        lambda s: s.infer_groups([(avs[0], 0, _feats(2, 16, 1024)), (avs[1], 1, _feats(2, 16, 1024, seed=1))])


def _case_hubert(mctx):
    from livetalking_b200.hubert import HubertEncoder, HubertFeatures
    enc = HubertEncoder(mctx, _weights("hubert"))
    audio16 = mctx.alloc((2, 32, 32, 16), np.float16)
    return lambda ctx: HubertFeatures(enc, 2, out_nhwc=audio16, ctx=ctx), [audio16], lambda s: s.run(_feats(s.n))


def _case_hubert_batch(mctx):
    from livetalking_b200.hubert import HubertBatchFeatures, HubertEncoder
    enc = HubertEncoder(mctx, _weights("hubert"))
    return lambda ctx: HubertBatchFeatures(enc, 2, 2, ctx=ctx), [], lambda s: s.run_groups([_feats(s.n), _feats(s.n, seed=1)])


def _case_musetalk(mctx):
    from livetalking_b200.musetalk import MuseTalkSession
    model, (av, _) = _mt(mctx)
    return lambda ctx: MuseTalkSession(model, av, 2, ctx=ctx), [], \
        lambda s: (s.infer(0, _feats(2, 50, 384)), s.paste_batch(0), s.paste_pred(_u8(256, 256, 3), 1))


def _case_musetalk_paste_only(mctx):
    from livetalking_b200.musetalk import MuseTalkSession
    model, (av, _) = _mt(mctx)
    return lambda ctx: MuseTalkSession(model, av, 2, ctx=ctx, paste_only=True), [], lambda s: s.paste_pred(_u8(256, 256, 3), 0)


def _case_musetalk_batch(mctx):
    from livetalking_b200.musetalk import MuseTalkBatchSession
    model, avs = _mt(mctx)
    return lambda ctx: MuseTalkBatchSession(model, 32, 2, 2, ctx=ctx), [], \
        lambda s: s.step([(avs[0], 0, _feats(2, 50, 384)), (avs[1], 1, _feats(2, 50, 384, seed=1))])


def _case_whisper(mctx):
    from livetalking_b200.whisper import WhisperEncoder, WhisperFeatures
    enc = WhisperEncoder(mctx, _weights("whisper"))
    out = mctx.alloc((2, 64, 384), np.float16)
    return lambda ctx: WhisperFeatures(enc, 2, out=out, out_rows=64, ctx=ctx), [out], lambda s: s.run(_feats(s.n))


def _case_s3fd(mctx):
    from livetalking_b200.s3fd import S3FDDetector, S3FDNet
    net = S3FDNet.from_state_dict(_weights("s3fd"), mctx)
    return lambda ctx: S3FDDetector(net, 2, 64, 96, ctx=ctx), [], lambda s: s.run_raw(_u8(2, 64, 96, 3))


def _case_pfld(mctx):
    from livetalking_b200.pfld import PFLDLandmarker, PFLDNet
    sd, mean_face = _weights("pfld")
    net = PFLDNet.from_state_dict({"pfld_backbone": sd}, mean_face, mctx)
    return lambda ctx: PFLDLandmarker(net, 2, ctx=ctx), [], lambda s: s.run(_u8(2, 192, 192, 3), [[100, 100], [120, 90]])


def _case_bisenet(mctx):
    from livetalking_b200.bisenet import BiSeNetNet, BiSeNetParser
    net = BiSeNetNet.from_state_dict(_weights("bisenet"), mctx)
    return lambda ctx: BiSeNetParser(net, 2, ctx=ctx), [], lambda s: s.parse(_u8(2, 512, 512, 3))


CASES = {f.__name__[len("_case_"):]: f for f in (_case_ultralight, _case_ultralight_batch, _case_hubert, _case_hubert_batch,
                                                   _case_musetalk, _case_musetalk_batch, _case_whisper, _case_s3fd, _case_pfld,
                                                   _case_bisenet)}
PASTE_ONLY = {"ultralight_paste_only": _case_ultralight_paste_only, "musetalk_paste_only": _case_musetalk_paste_only}


@pytest.mark.parametrize("name", list(CASES))
def test_close_on_a_borrowed_ctx_frees_exactly_what_the_session_allocated(monkeypatch, name):
    made = _patch_ctx(monkeypatch)
    ctx = _RecordingCtx()
    make, handed, exercise = CASES[name](ctx)
    before = dict(ctx.live)                                # weights, avatars and the tensors handed to the session
    sess = make(ctx)
    exercise(sess)
    assert sess.ctx is ctx and len(ctx.live) > len(before)
    sess.close()
    assert ctx.live == before and not ctx.closed
    assert all(t.ptr in ctx.live for t in handed)
    assert all(c.closed for c in made)                     # paste contexts
    sess.close()                                           # twice is harmless
    assert ctx.live == before


@pytest.mark.parametrize("name", list(CASES) + list(PASTE_ONLY))
def test_close_on_an_owned_ctx_closes_it(monkeypatch, name):
    made = _patch_ctx(monkeypatch)
    mctx = _RecordingCtx()
    make, _handed, exercise = {**CASES, **PASTE_ONLY}[name](mctx)
    before = dict(mctx.live)
    sess = make(None)
    exercise(sess)
    assert made and sess.ctx is (None if name in PASTE_ONLY else made[0])
    sess.close()
    assert all(c.closed for c in made) and sess.ctx is None and sess.graph is None
    assert mctx.live == before and not mctx.closed
    sess.close()


@pytest.mark.parametrize("failing_pass", [1, 2], ids=["eager", "captured"])
def test_a_session_constructor_that_raises_releases_its_allocations(monkeypatch, failing_pass):
    from livetalking_b200.ultralight import UltraLightModel
    calls = []
    emit = UltraLightModel.emit

    def failing(self, *a, **kw):
        calls.append(1)
        if len(calls) == failing_pass:
            raise RuntimeError("emit")
        return emit(self, *a, **kw)
    monkeypatch.setattr(UltraLightModel, "emit", failing)
    ctx = _RecordingCtx()
    before = dict(ctx.live)
    from livetalking_b200.ultralight import UltraLightSession
    _m, (av, _) = _ul_avatars(ctx)
    models = dict(ctx.live)
    with pytest.raises(RuntimeError):
        UltraLightSession(av, 2, ctx=ctx)
    assert ctx.live == models and set(before) <= set(ctx.live) and not ctx.closed


def test_a_layer_plan_that_reads_an_overwritten_arena_buffer_raises():
    """Buffers of one arena share memory: a step that reads one after another of them was written is refused at construction,
    before anything is allocated."""
    from livetalking_b200.layerplan import LayerSession, Step
    ctx = _RecordingCtx()
    bufs = {name: ((1, 4, 4, 16), np.float16) for name in ("in", "a", "b", "c")}
    copy = lambda s, x, y: s.ctx.copy_channels(x, y)                # noqa: E731
    ok = [Step("a", src=("in", 0, 16), dst=("a", 0, 16), run=copy), Step("b", src=("a", 0, 16), dst=("b", 0, 16), run=copy)]
    LayerSession(1, bufs, ok, ctx, arenas={"a": 0, "b": 0}).close()
    assert ctx.live == {}
    bad = ok + [Step("c", src=("a", 0, 16), dst=("c", 0, 16), run=copy)]
    with pytest.raises(ValueError, match="reads a after b"):
        LayerSession(1, bufs, bad, ctx, arenas={"a": 0, "b": 0})
    assert ctx.live == {} and not ctx.closed
    LayerSession(1, bufs, bad, ctx, arenas={"a": 0, "b": 1}).close()


# ---------------------------------------------------------------------------------------------------------------- GPU
def _flat(x):
    return [a for v in x for a in _flat(v)] if isinstance(x, (list, tuple)) else [np.asarray(x)]


@pytest.mark.gpu
def test_sessions_on_a_shared_ctx_give_back_every_allocation():
    """Every session class on ONE shared ctx (weights on their own): the ctx's live allocations after close() are those from before
    the session was built; a session built afterwards on the same ctx computes what the first one did (last-bit float jitter of the
    atomics in GroupNorm statistics / split-K allowed)."""
    from livetalking_b200 import engine
    from livetalking_b200.ops import Ctx
    engine.set_device(0)
    mctx, ctx = Ctx(), Ctx()
    live = set()
    alloc, free = ctx.alloc, ctx.free

    def traced_alloc(*a, **kw):
        t = alloc(*a, **kw)
        live.add(t.ptr)
        return t

    def traced_free(t):
        live.discard(t.ptr)
        return free(t)

    ctx.alloc, ctx.free = traced_alloc, traced_free
    for name, case in CASES.items():
        make, _handed, exercise = case(mctx)
        before = set(live)
        outs = []
        for _ in range(2):
            s = make(ctx)
            outs.append(_flat(exercise(s)))
            assert live > before, name
            s.close()
            assert live == before, f"{name}: {len(live - before)} allocations left on the shared ctx after close()"
        for a, b in zip(*outs):
            assert a.shape == b.shape and a.dtype == b.dtype, name
            if a.dtype.kind in "iu":
                assert np.abs(a.astype(np.int64) - b).max(initial=0) <= 2, name
            else:
                assert np.isfinite(a).all() and np.abs(a - b).max(initial=0) <= 1e-2 * max(1.0, float(np.abs(a).max())), name
    ctx.close()
    mctx.close()
