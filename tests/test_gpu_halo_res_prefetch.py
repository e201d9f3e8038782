"""GPU: the prefetched global residual of the halo conv instance <128, 2, 1> (L45/L46/L48/L49 of wav2lip256).

That instance reads its residual from global memory; it loads sub-tile 0's residual into shared memory at the start of each
tile and sub-tile 1's into registers under the tile's last MMAs.  The residual it adds must be exactly the residual of each
output pixel: the conv with a residual must equal, value for value, the same conv without one (ReLU off, so the fp16 value is
the one the residual is added to) plus the residual in one correctly rounded fp16 add, clamped to [0 or -65504, 65504].
Rows cover overhanging tiles, several tiles per CTA (the shared-memory slots are reused), two N tiles, ReLU on and off, and the
residual both as the input slice itself and as a separate copy.  Nothing may be written outside the output slice."""
import types

import numpy as np
import pytest
import torch

H100_SMS = 132
SENT_IN = 512.0
SENT_OUT = -3.25

ROWS = [  # N, H, W, C
    (16, 64, 64, 128),    # 256 tiles: two per CTA
    (16, 64, 60, 128),    # the same with the last tile column 4 pixels past the map
    (5, 128, 36, 256),    # 200 tiles, 2 N tiles, overhanging columns
]


@pytest.fixture(scope="module")
def ctx():
    from livetalking_b200 import engine
    from livetalking_b200.ops import Ctx
    engine.set_device(0)
    c = Ctx()
    yield c
    c.close()


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint16)


def _slice_buf(ctx, dense, pitch, off, fill):
    from livetalking_b200.ops import DevTensor
    buf = np.full(dense.shape[:-1] + (pitch,), fill, np.float16)
    buf[..., off:off + dense.shape[-1]] = dense
    t = ctx.upload(buf)
    return DevTensor(t.ptr, dense.shape, pitch=pitch, c_off=off), t, buf


@pytest.mark.gpu
@pytest.mark.parametrize("relu", [True, False], ids=["relu", "norelu"])
@pytest.mark.parametrize("row", ROWS, ids=["x".join(map(str, r)) for r in ROWS])
def test_prefetched_residual_is_each_pixels_own(ctx, row, relu):
    N, IH, IW, Cch = row
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    g = torch.Generator().manual_seed(N * 1000 + IW + relu)
    x = (torch.randn(N, IH, IW, Cch, generator=g) * 0.7 + 0.4 + torch.randn(Cch, generator=g) * 0.3).half()
    w = (torch.randn(Cch, Cch, 3, 3, generator=g) * (2.0 / (Cch * 9)) ** 0.5).half()
    b = torch.randn(Cch, generator=g) * 0.2
    ICtot, OCtot, RCtot = Cch + 24, Cch + 16, Cch + 8
    xv, xt, xbuf = _slice_buf(ctx, x.numpy(), ICtot, 8, SENT_IN)
    rv, rt, rbuf = _slice_buf(ctx, x.numpy(), RCtot, 8, SENT_IN)
    wt = ctx.upload(w.permute(0, 2, 3, 1).reshape(Cch, 9 * Cch).numpy())
    bt = ctx.upload(b.numpy().astype(np.float32))
    wtap = ctx.alloc((9, Cch, Cch))
    ctx.w_tap_major(wt, wtap, Cch, Cch)
    cw = types.SimpleNamespace(cout=Cch, cin=Cch, kh=3, kw=3, ktot=9 * Cch, w=wt, w_tap=wtap, bias=bt)
    temps = [xt, rt, wt, bt, wtap]
    want = dict(kernel=1, taps=9, bn=128, nsub=2, nacc=1, resident_chunks=0, kb=0, ksplit=0, grouped=0)
    outs = {}
    try:
        for name, res, rl in (("plain", None, False), ("self", xv, relu), ("copy", rv, relu)):
            ov, ot, obuf = _slice_buf(ctx, np.full((N, IH, IW, Cch), np.nan, np.float16), OCtot, 8, SENT_OUT)
            temps.append(ot)
            geo = dict(N=N, IH=IH, IW=IW, OH=IH, OW=IW, pad=(1, 1), relu=rl, res=res)
            variant = ctx.conv_plan(xv, cw, ov, **geo)
            assert variant == want and sms == H100_SMS, f"{name}: planned {variant}, expected {want} on {sms} SMs"
            assert not ctx.conv_res_halo(xv, cw, ov, **geo), name
            ctx.conv(xv, cw, ov, **geo)
            full = ctx.download(ot)
            outside = np.ones(obuf.shape, bool)
            outside[..., 8:8 + Cch] = False
            assert np.array_equal(_bits(full)[outside], _bits(obuf)[outside]), f"{name}: wrote outside the output slice"
            outs[name] = full[..., 8:8 + Cch]
        assert np.array_equal(_bits(ctx.download(xt)), _bits(xbuf)), "the conv changed its input buffer"
        assert np.array_equal(_bits(ctx.download(rt)), _bits(rbuf)), "the conv changed its residual buffer"
        assert np.isfinite(outs["plain"]).all(), "unwritten outputs"
        # fp16 + fp16 is exact in float64; one rounding to fp16 is the correctly rounded __hadd2
        ref = (outs["plain"].astype(np.float64) + x.numpy().astype(np.float64)).astype(np.float16)
        ref = np.minimum(np.maximum(ref, np.float16(0.0 if relu else -65504.0)), np.float16(65504.0))
        for name in ("self", "copy"):
            diff = outs[name] != ref     # value comparison: max(-0, 0) may keep either zero
            assert not diff.any(), f"{name}: {int(diff.sum())} outputs differ from conv + residual, first at {np.argwhere(diff)[0]}"
    finally:
        for t in temps:
            ctx.free(t)
