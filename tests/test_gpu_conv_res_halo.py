"""GPU: the halo conv kernel's residual-from-shared-memory path (HaloParams::res_halo).

When a 3x3 stride-1 conv adds its own input (res is the input slice, Cin == Cout: the wav2lip residual blocks), the TMA kernel
takes the residual from the centre view of the halo tiles it already holds in shared memory instead of reading res from global
memory.  Each row runs one instance twice in the same binary: once with res = the input slice itself, once with res = a
separate copy of it, which takes the global-load path.  Both must report the path they take (Ctx.conv_res_halo), produce
bit-identical outputs (the same fp16 add and clamp on the same operands) and pass conv_check.py against float64 with the halo
rounding order: fp16(acc + b), then the fp16 add of the residual and the ReLU.  Inputs are channel slices (ic_off = 8, ICtot = Cin + 24) whose neighbours hold sentinels.

<128, 2, 1> keeps the global-load path (its registers have no room for the residual words); its row checks that it says so."""
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import conv_check as cc

H100_SMS = 132
SENT_IN = 512.0
SENT_OUT = -3.25

# (BN, NSUB, NACC, TAPS, resident chunks) -> (N, H, W, C, takes the residual from the halo); the expected variants are those
# of the 132-SM H100 SXM
ROWS = {
    # 216 tiles, 20 columns overhang; C = 96: ragged second K chunk, N tiles n0 = 0, 32 (n0 % 64 = 32), 64 (chunk 1)
    (32, 2, 1, 9, 0): ((6, 128, 20, 96), True),
    # 216 tiles, 3 N tiles (chunks 0, 1, 2)
    (64, 2, 1, 9, 0): ((6, 128, 20, 192), True),
    # resident weights: one chunk, one N tile, 272 tiles, 132 columns overhang
    (64, 2, 1, 9, 1): ((4, 128, 132, 64), True),
    # 144 tiles, 20 x 20 overhangs rows and columns, 3 N tiles of two residual chunks each (0/1, 2/3, 4/5)
    (128, 1, 1, 9, 0): ((8, 20, 20, 384), True),
    # 200 tiles, 2 N tiles: global residual path
    (128, 2, 1, 9, 0): ((5, 128, 36, 256), False),
}


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
@pytest.mark.parametrize("key", list(ROWS), ids=[f"halo<{','.join(map(str, k))}>" for k in ROWS])
def test_residual_from_halo_matches_global_residual(ctx, key):
    (N, IH, IW, Cch), from_halo = ROWS[key]
    bn, nsub, nacc, taps, rc = key
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    g = torch.Generator().manual_seed(sum(key))
    x = (torch.randn(N, IH, IW, Cch, generator=g) * 0.7 + 0.4 + torch.randn(Cch, generator=g) * 0.3).half()
    w = (torch.randn(Cch, Cch, 3, 3, generator=g) * (2.0 / (Cch * 9)) ** 0.5).half()
    b = torch.randn(Cch, generator=g) * 0.2
    ICtot, OCtot, RCtot = Cch + 24, Cch + 16, Cch + 8
    xv, xt, xbuf = _slice_buf(ctx, x.numpy(), ICtot, 8, SENT_IN)
    rv, rt, rbuf = _slice_buf(ctx, x.numpy(), RCtot, 8, SENT_IN)     # the same values in a separate buffer
    wt = ctx.upload(w.permute(0, 2, 3, 1).reshape(Cch, 9 * Cch).numpy())
    bt = ctx.upload(b.numpy().astype(np.float32))
    wtap = ctx.alloc((9, Cch, Cch))
    ctx.w_tap_major(wt, wtap, Cch, Cch)
    cw = types.SimpleNamespace(cout=Cch, cin=Cch, kh=3, kw=3, ktot=9 * Cch, w=wt, w_tap=wtap, bias=bt)
    temps = [xt, rt, wt, bt, wtap]
    outs = {}
    try:
        want = dict(kernel=1, taps=taps, bn=bn, nsub=nsub, nacc=nacc, resident_chunks=rc, kb=0, ksplit=0, grouped=0)
        for name, res in (("halo", xv), ("copy", rv)):
            ov, ot, obuf = _slice_buf(ctx, np.full((N, IH, IW, Cch), np.nan, np.float16), OCtot, 8, SENT_OUT)
            temps.append(ot)
            geo = dict(N=N, IH=IH, IW=IW, OH=IH, OW=IW, pad=(1, 1), relu=True, res=res)
            variant = ctx.conv_plan(xv, cw, ov, **geo)
            assert variant == want and sms == H100_SMS, f"{name}: planned {variant}, expected {want} on {sms} SMs"
            assert ctx.conv_res_halo(xv, cw, ov, **geo) == (from_halo and name == "halo"), name
            ctx.conv(xv, cw, ov, **geo)
            full = ctx.download(ot)
            outside = np.ones(obuf.shape, bool)
            outside[..., 8:8 + Cch] = False
            assert np.array_equal(_bits(full)[outside], _bits(obuf)[outside]), f"{name}: wrote outside the output slice"
            outs[name] = full[..., 8:8 + Cch]
        assert np.array_equal(_bits(ctx.download(xt)), _bits(xbuf)), "the conv changed its input buffer"
        assert np.array_equal(_bits(ctx.download(rt)), _bits(rbuf)), "the conv changed its residual buffer"
        diff = _bits(outs["halo"]) != _bits(outs["copy"])
        assert not diff.any(), f"{int(diff.sum())} outputs differ between the two residual paths, first at {np.argwhere(diff)[0]}"
        x64 = x.double().permute(0, 3, 1, 2)
        conv = F.conv2d(F.pad(x64, (1, 1, 1, 1)), w.double()).permute(0, 2, 3, 1).numpy()
        A = F.conv2d(F.pad(x64.abs(), (1, 1, 1, 1)), w.double().abs()).permute(0, 2, 3, 1).numpy()
        cc.check(outs["halo"], conv, A, b.numpy(), K=9 * Cch, order="halo", relu=True, r=x.numpy(),
                 what=f"halo<{','.join(map(str, key))}> residual from {'shared memory' if from_halo else 'global memory'}")
    finally:
        for t in temps:
            ctx.free(t)
