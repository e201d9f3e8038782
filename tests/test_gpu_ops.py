"""GPU: the bandwidth-bound device ops of the C ABI (csrc/ops.cu through ltb_op_*) against plain float64 references computed from
the same fp16 inputs.

Channel-sliced inputs sit between neighbours that hold SENT_IN (512: large enough to wreck a statistic if it is read, small
enough not to overflow an fp32 accumulator); outputs are pre-filled with SENT_OUT, and every element outside the written
slice must keep its bits.  Pure data movement and fp16 rounding ops are compared bit for bit; norms and activations with fp16
output within TOL_ABS + TOL_REL * |ref| (a few fp16 half-ulps: a biased / unbiased variance swap on a 2x2 map is ~6 %)."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

SENT_IN = 512.0
SENT_OUT = -3.25
TOL_ABS, TOL_REL = 1e-3, 2e-3


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


def _sliced(ctx, dense: np.ndarray, pitch: int, off: int, fill=SENT_IN):
    """Upload `dense` (..., C) fp16 as channels [off, off+C) of a (..., pitch) buffer whose other channels hold `fill`."""
    from livetalking_b200.ops import DevTensor
    buf = np.full(dense.shape[:-1] + (pitch,), fill, np.float16)
    buf[..., off:off + dense.shape[-1]] = dense
    t = ctx.upload(buf)
    return DevTensor(t.ptr, dense.shape, pitch=pitch, c_off=off), t, buf


def _check_close(got, ref, what, tol_abs=TOL_ABS, tol_rel=TOL_REL):
    got = got.astype(np.float64)
    assert np.isfinite(got).all(), f"{what}: non-finite output"
    err = np.abs(got - ref)
    tol = tol_abs + tol_rel * np.abs(ref)
    bad = err > tol
    assert not bad.any(), (f"{what}: {int(bad.sum())} of {bad.size} outside tolerance; worst err/tol {(err / tol).max():.2f} at "
                           f"{np.unravel_index((err / tol).argmax(), err.shape)} (err {err.max():.3g})")


def _untouched(buf_after, buf_before, mask_written, what):
    a, b = _bits(buf_after), _bits(buf_before)
    changed = (a != b) & ~mask_written
    assert not changed.any(), f"{what}: {int(changed.sum())} elements outside the written range changed, first at {np.argwhere(changed)[0]}"


# ------------------------------------------------------------------------------------------------ GroupNorm
def _gn_ref(x, groups, eps, gamma, beta, silu):
    """x (N, HW, C) float64 -> GroupNorm (biased variance, like torch) [+ SiLU]."""
    N, HW, Cc = x.shape
    g = x.reshape(N, HW, groups, Cc // groups)
    m = g.mean(axis=(1, 3), keepdims=True)
    v = ((g - m) ** 2).mean(axis=(1, 3), keepdims=True)
    y = ((g - m) / np.sqrt(v + eps)).reshape(N, HW, Cc) * gamma + beta
    return y / (1.0 + np.exp(-y)) if silu else y


GN_CASES = [
    # N, H, W, C, groups, silu, offset: what it targets
    (2, 1, 1, 64, 64, False, "chan"),     # one-warp stats block, 64 groups: groups 32..63 zeroed / flushed by nobody (defect 1)
    (3, 2, 1, 128, 64, True, "chan"),     # C=128, HW=2: same one-warp block (defect 1)
    (2, 2, 2, 64, 64, False, "chan"),     # C=64, HW=4: still one warp (defect 1)
    (4, 2, 2, 128, 64, True, "chan"),     # HW=4: two warps, 2 channels per group, biased variance over 8 values
    (4, 2, 2, 128, 32, False, "chan"),
    (2, 4, 4, 320, 32, True, "chan"),     # 10 channels per group: 16-byte vectors straddle groups
    (48, 8, 8, 320, 32, True, "chan"),    # large batch: one grid row per image
    (5, 3, 5, 640, 64, False, "chan"),    # odd HW, 10 channels per group
    (2, 16, 16, 1280, 64, True, "chan"),  # C/8 = 160 vectors per pixel, 20 channels per group
    (48, 2, 2, 1280, 64, False, "chan"),  # N * groups = 3072
    (2, 64, 64, 320, 32, True, "chan"),   # many splits per image: cross-block atomics
    (1, 32, 32, 640, 32, False, "chan"),
    (2, 32, 32, 320, 32, False, "big"),   # mean ~4, std ~0.1: the E[x^2] - m^2 form in fp32
]


@pytest.mark.parametrize("case", GN_CASES, ids=[f"N{c[0]}_{c[1]}x{c[2]}_C{c[3]}_g{c[4]}{'_silu' if c[5] else ''}_{c[6]}" for c in GN_CASES])
def test_groupnorm_slices_match_float64(ctx, case):
    """ltb_op_groupnorm (gn_stats_kernel + gn_apply_kernel) on a channel slice into a channel slice.  Every channel has its own
    offset and scale, so a channel counted in the wrong group moves that group's mean and shows."""
    from livetalking_b200.ops import DevTensor
    N, H, W, Cc, groups, silu, kind = case
    HW = H * W
    rng = np.random.default_rng(N * 1000003 + HW * 1009 + Cc * 7 + groups + silu)
    if kind == "big":
        x = (4.0 + 0.1 * rng.standard_normal((N, H, W, Cc))).astype(np.float16)
    else:
        x = (rng.uniform(-2, 2, Cc) + rng.uniform(0.3, 1.5, Cc) * rng.standard_normal((N, H, W, Cc))).astype(np.float16)
    gamma = rng.uniform(0.5, 1.5, Cc).astype(np.float32)
    beta = rng.uniform(-0.5, 0.5, Cc).astype(np.float32)
    eps = 1e-6 if kind == "big" else 1e-5
    xv, xt, xbuf = _sliced(ctx, x, Cc + 16, 8)
    opitch, ooff = Cc + 24, 16
    obuf = np.full((N, H, W, opitch), SENT_OUT, np.float16)
    ot = ctx.upload(obuf)
    ctx.groupnorm(xv, N, HW, groups, eps, ctx.upload(gamma), ctx.upload(beta), silu, DevTensor(ot.ptr, (N, H, W, Cc), pitch=opitch, c_off=ooff))
    got = ctx.download(ot)
    written = np.zeros(obuf.shape, bool)
    written[..., ooff:ooff + Cc] = True
    _untouched(got, obuf, written, "groupnorm output neighbours")
    _untouched(ctx.download(xt), xbuf, np.zeros(xbuf.shape, bool), "groupnorm input")
    ref = _gn_ref(x.astype(np.float64).reshape(N, HW, Cc), groups, eps, gamma.astype(np.float64), beta.astype(np.float64), silu)
    _check_close(got[..., ooff:ooff + Cc].reshape(N, HW, Cc), ref, "groupnorm")


def test_groupnorm_rejects_batch_beyond_stats_workspace(ctx):
    """N * groups > 4096 would overflow the context's statistics workspace: the op must refuse instead of writing past it."""
    from livetalking_b200._capi import LtbError
    x = ctx.alloc((65, 1, 1, 64), np.float16, zero=True)
    out = ctx.alloc((65, 1, 1, 64), np.float16)
    g = ctx.upload(np.ones(64, np.float32))
    b = ctx.upload(np.zeros(64, np.float32))
    with pytest.raises(LtbError, match="statistics workspace"):
        ctx.groupnorm(x, 65, 1, 64, 1e-5, g, b, False, out)
    ctx.groupnorm(ctx.alloc((64, 1, 1, 64), np.float16, zero=True), 64, 1, 64, 1e-5, g, b, False, out)   # exactly 4096: accepted
    ctx.sync()


# ------------------------------------------------------------------------------------------------ LayerNorm
@pytest.mark.parametrize("Cc,rows", [(8, 13), (264, 37), (320, 301), (384, 77), (1280, 19), (2048, 45)])
def test_layernorm_matches_float64(ctx, Cc, rows):
    """layernorm_kernel (warp per row, up to 8 vectors per lane): C = 8 (one vector), 264 (C/8 not a multiple of 32: lanes own
    different vector counts), 2048 (the register limit); row counts that leave the last 8-row block partly empty."""
    rng = np.random.default_rng(Cc * 1000 + rows)
    x = (rng.uniform(-1, 1, (rows, 1)) + rng.standard_normal((rows, Cc)) * rng.uniform(0.2, 3, (rows, 1))).astype(np.float16)
    gamma = rng.uniform(0.5, 1.5, Cc).astype(np.float32)
    beta = rng.uniform(-0.5, 0.5, Cc).astype(np.float32)
    xt = ctx.upload(x)
    obuf = np.full((rows + 3, Cc), SENT_OUT, np.float16)      # 3 rows past the end must stay untouched
    ot = ctx.upload(obuf)
    ctx.layernorm(xt, rows, Cc, 1e-5, ctx.upload(gamma), ctx.upload(beta), ot)
    got = ctx.download(ot)
    written = np.zeros(obuf.shape, bool)
    written[:rows] = True
    _untouched(got, obuf, written, "layernorm tail")
    xd = x.astype(np.float64)
    m = xd.mean(1, keepdims=True)
    ref = (xd - m) / np.sqrt(((xd - m) ** 2).mean(1, keepdims=True) + 1e-5) * gamma + beta
    _check_close(got[:rows], ref, "layernorm")


# ------------------------------------------------------------------------------------------------ softmax
def _softmax_call(ctx, x_ptr, rows, cols, ld, valid, scale, out_ptr):
    from livetalking_b200._capi import check, lib
    check(lib().ltb_op_softmax(ctx._h, C.c_void_p(x_ptr), rows, cols, ld, valid, C.c_float(scale), C.c_void_p(out_ptr)))


SOFTMAX_CASES = [
    # rows, cols, ld, valid, scale, in_place: kernel
    (11, 8, 8, 1, 0.5, True),            # narrow: a single valid key
    (37, 200, 200, 77, 0.158, True),     # narrow: valid not a multiple of 8, padded columns zeroed
    (9, 1536, 1536, 1536, 0.125, False), # narrow kernel's widest row, out of place
    (13, 64, 80, 50, 0.25, True),        # ld > cols in place: columns [cols, ld) are not the op's
    (13, 64, 80, 64, 0.25, False),       # ld > cols out of place
    (5, 1544, 1552, 1001, 0.1, False),   # wide kernel: first width past 1536, ld > cols
    (3, 4096, 4096, 4096, 0.0625, True), # wide: 64x64-latent self-attention
    (2, 8192, 8192, 1, 1.0, True),       # wide: the register limit, one valid key
    (4, 8192, 8200, 6007, 0.2, False),   # wide: ragged valid, ld > cols
]


@pytest.mark.parametrize("case", SOFTMAX_CASES, ids=[f"r{c[0]}_c{c[1]}_ld{c[2]}_v{c[3]}{'_inplace' if c[5] else ''}" for c in SOFTMAX_CASES])
def test_softmax_matches_float64(ctx, case):
    """softmax_kernel (cols <= 1536) / softmax_wide_kernel: probabilities over the first `valid` columns, padded columns exactly 0,
    columns past `cols` untouched, every row sums to 1.  Two rows hold logits near the fp16 limits."""
    rows, cols, ld, valid, scale, in_place = case
    rng = np.random.default_rng(rows * 7 + cols + valid)
    x = np.full((rows, ld), SENT_IN, np.float16)
    x[:, :cols] = (rng.standard_normal((rows, cols)) * 6).astype(np.float16)
    x[0, :cols] = rng.choice(np.array([65504, -65504, 64000, -60000, 0], np.float16), cols)
    if rows > 1:
        x[1, :cols] = (65504 - 32 * rng.integers(0, 4, cols)).astype(np.float16)   # every logit within 96 of the fp16 max
    xt = ctx.upload(x)
    if in_place:
        ot, obuf = xt, x
    else:
        obuf = np.full((rows, ld), SENT_OUT, np.float16)
        ot = ctx.upload(obuf)
    _softmax_call(ctx, xt.ptr, rows, cols, ld, valid, scale, ot.ptr)
    got = ctx.download(ot)
    written = np.zeros(obuf.shape, bool)
    written[:, :cols] = True
    _untouched(got, obuf, written, "softmax columns past cols")
    if not in_place:
        _untouched(ctx.download(xt), x, np.zeros(x.shape, bool), "softmax input")
    assert not _bits(got[:, valid:cols]).any(), "padded columns must be exactly +0"
    lg = x[:, :valid].astype(np.float64) * float(np.float32(scale))
    e = np.exp(lg - lg.max(1, keepdims=True))
    ref = e / e.sum(1, keepdims=True)
    p = got[:, :valid].astype(np.float64)
    _check_close(p, ref, "softmax", tol_abs=1e-5, tol_rel=2e-3)
    assert np.abs(p.sum(1) - 1).max() < 1e-3, p.sum(1)


def test_softmax_rejects_bad_shapes(ctx):
    from livetalking_b200._capi import LtbError
    t = ctx.alloc((8, 8200), np.float16, zero=True)
    for cols, ld, valid in ((8200, 8200, 8), (64, 64, 0), (64, 64, 65), (60, 64, 8), (64, 68, 8)):
        with pytest.raises(LtbError):
            _softmax_call(ctx, t.ptr, 8, cols, ld, valid, 1.0, t.ptr)


# ------------------------------------------------------------------------------------------------ GEGLU / eltwise
def _gelu(v):
    from scipy.special import erf
    return 0.5 * v * (1.0 + erf(v / np.sqrt(2.0)))


@pytest.mark.parametrize("rows,H", [(5, 8), (37, 1280), (64, 2560)])
def test_geglu_matches_float64(ctx, rows, H):
    """geglu_kernel: out = h[:, :H] * gelu_erf(h[:, H:]) (diffusers GEGLU), rows x 2H -> rows x H."""
    rng = np.random.default_rng(rows + H)
    h = (rng.standard_normal((rows, 2 * H)) * 2.5).astype(np.float16)
    obuf = np.full((rows + 1, H), SENT_OUT, np.float16)
    ot = ctx.upload(obuf)
    ctx.geglu(ctx.upload(h), rows, H, ot)
    got = ctx.download(ot)
    written = np.zeros(obuf.shape, bool)
    written[:rows] = True
    _untouched(got, obuf, written, "geglu tail")
    hd = h.astype(np.float64)
    _check_close(got[:rows], hd[:, :H] * _gelu(hd[:, H:]), "geglu")


ELT_CASES = [
    # n, period, act, with_y, in_place: what it models
    (4096, 0, 0, False, False),       # copy through fp16 (act none)
    (4096, 0, 1, False, True),        # in-place GELU (whisper.py conv stem)
    (4104, 0, 2, False, False),       # SiLU, n not a multiple of 256 vectors
    (64 * 384 * 3, 64 * 384, 0, True, True),   # positional encoding: (B*KEY_PAD, 384) += pe (KEY_PAD, 384), in place
    (1500 * 384, 1500 * 384, 1, True, True),   # whisper residual + GELU, y not broadcast, in place
    (77 * 320, 320, 2, True, False),  # bias-like broadcast of one row + SiLU
]


@pytest.mark.parametrize("case", ELT_CASES, ids=[f"n{c[0]}_p{c[1]}_act{c[2]}{'_y' if c[3] else ''}{'_inplace' if c[4] else ''}" for c in ELT_CASES])
def test_eltwise_matches_float64(ctx, case):
    """eltwise_kernel: out = act(x + y[i % period]), act 0 none / 1 gelu(erf) / 2 silu.  act 0 is bit-exact against the same add
    in torch fp16 on the CPU (fp32 add, one rounding)."""
    n, period, act, with_y, in_place = case
    rng = np.random.default_rng(n + period + act)
    x = (rng.standard_normal(n) * 3).astype(np.float16)
    x[:8] = np.array([0, -0.0, 65504, -65504, 6e-8, -20, 20, 11.5], np.float16)
    y = (rng.standard_normal(period) * 2).astype(np.float16) if with_y else None
    xt = ctx.upload(x)
    yt = ctx.upload(y) if with_y else None
    if in_place:
        ot, obuf = xt, x
    else:
        obuf = np.full(n + 8, SENT_OUT, np.float16)
        ot = ctx.upload(obuf)
    ctx.eltwise(xt, yt, n, period, act, ot)
    got = ctx.download(ot)
    written = np.zeros(obuf.shape, bool)
    written[:n] = True
    _untouched(got, obuf, written, "eltwise tail")
    got = got[:n]
    yb = np.tile(y, n // period) if with_y else np.zeros(n, np.float16)
    if act == 0:
        want = (torch.from_numpy(x) + torch.from_numpy(yb)).numpy()
        assert np.array_equal(_bits(got), _bits(want)), "act 0 must be the fp16 rounding of the fp32 sum"
        return
    v = x.astype(np.float64) + yb.astype(np.float64)
    with np.errstate(over="ignore"):
        ref = _gelu(v) if act == 1 else v / (1.0 + np.exp(-v))
    _check_close(got, ref, f"eltwise act {act}")


# ------------------------------------------------------------------------------------------------ bit-exact data movement
@pytest.mark.parametrize("N,H,W,Cc", [(1, 1, 1, 8), (2, 5, 3, 40), (3, 16, 16, 320)])
def test_upsample2x_is_nearest_bit_exact(ctx, N, H, W, Cc):
    """upsample2x_kernel against F.interpolate(nearest), every output element."""
    x = (np.random.default_rng(H * W + Cc).standard_normal((N, H, W, Cc)) * 4).astype(np.float16)
    obuf = np.full((N * 4 * H * W + 5, Cc), SENT_OUT, np.float16)
    ot = ctx.upload(obuf)
    ctx.upsample2x(ctx.upload(x), N, H, W, ot)
    got = ctx.download(ot)
    want = F.interpolate(torch.from_numpy(x).permute(0, 3, 1, 2).float(), scale_factor=2, mode="nearest").half().permute(0, 2, 3, 1)
    assert np.array_equal(_bits(got[:N * 4 * H * W]), _bits(want.reshape(-1, Cc).numpy()))
    assert np.array_equal(_bits(got[N * 4 * H * W:]), _bits(obuf[N * 4 * H * W:])), "rows past the output changed"


@pytest.mark.parametrize("rows,Cc,spitch,soff,dpitch,doff", [(7, 8, 24, 16, 16, 0), (301, 320, 640, 320, 960, 320), (64, 1280, 1288, 8, 2560, 1280)])
def test_copy_channels_between_slices_bit_exact(ctx, rows, Cc, spitch, soff, dpitch, doff):
    """copy_channels_kernel (the concat of the UNet skip connections): slice -> slice, neighbours on both sides untouched."""
    from livetalking_b200.ops import DevTensor
    x = (np.random.default_rng(rows + Cc).standard_normal((rows, Cc)) * 4).astype(np.float16)
    sv, st, sbuf = _sliced(ctx, x, spitch, soff)
    dbuf = np.full((rows, dpitch), SENT_OUT, np.float16)
    dt = ctx.upload(dbuf)
    ctx.copy_channels(sv, DevTensor(dt.ptr, (rows, Cc), pitch=dpitch, c_off=doff))
    got = ctx.download(dt)
    assert np.array_equal(_bits(got[:, doff:doff + Cc]), _bits(x))
    written = np.zeros(dbuf.shape, bool)
    written[:, doff:doff + Cc] = True
    _untouched(got, dbuf, written, "copy_channels destination neighbours")
    _untouched(ctx.download(st), sbuf, np.zeros(sbuf.shape, bool), "copy_channels source")


@pytest.mark.parametrize("B,n_keys,heads,d,c_off,n_pad", [(2, 50, 8, 40, 320, 64), (1, 77, 5, 48, 8, 80), (3, 64, 2, 80, 16, 64),
                                                          (2, 33, 2, 160, 160, 48)])
def test_transpose_heads_bit_exact(ctx, B, n_keys, heads, d, c_off, n_pad):
    """transpose_heads_kernel: V [B, n_keys, Ctot] (head h = channels c_off + h*d ...) -> VT [B, heads, d, n_pad], keys >= n_keys
    written as 0 (the P.V GEMM runs over the padded key count), nothing written past VT."""
    from livetalking_b200._capi import check, lib
    Ctot = c_off + heads * d + 24
    v = (np.random.default_rng(B * n_keys + d).standard_normal((B, n_keys, Ctot)) * 3).astype(np.float16)
    v[..., :c_off] = SENT_IN
    v[..., c_off + heads * d:] = SENT_IN
    vbuf = np.full(B * heads * d * n_pad + 64, SENT_OUT, np.float16)
    vt = ctx.upload(vbuf)
    check(lib().ltb_op_transpose_heads(ctx._h, C.c_void_p(ctx.upload(v).ptr), B, n_keys, Ctot, c_off, heads, d, n_pad, C.c_void_p(vt.ptr)))
    got = ctx.download(vt)
    want = np.zeros((B, heads, d, n_pad), np.float16)
    want[..., :n_keys] = v[..., c_off:c_off + heads * d].reshape(B, n_keys, heads, d).transpose(0, 2, 3, 1)
    n = want.size
    assert np.array_equal(_bits(got[:n]), _bits(want.reshape(-1))), "VT differs (padding must be +0)"
    assert np.array_equal(_bits(got[n:]), _bits(vbuf[n:])), "written past VT"


@pytest.mark.parametrize("n,index,B", [(1, 0, 4), (1, 5, 3), (5, 7, 12), (4, 13, 9), (3, 0, 7)])
def test_gather_rows_mirror_index_bit_exact(ctx, n, index, B):
    """gather_rows_kernel: out[i] = table[mirror_index(n, index + i)], indices past 2n (a second forward turn) and n = 1."""
    from oracle.paste_ref import mirror_index
    row = 8 * 37
    table = (np.random.default_rng(n * 100 + index).standard_normal((n, row)) * 3).astype(np.float16)
    d_index = ctx.upload(np.array([index], np.int32))
    obuf = np.full((B + 1, row), SENT_OUT, np.float16)
    ot = ctx.upload(obuf)
    ctx.gather_rows(ctx.upload(table), n, d_index, B, row, ot)
    got = ctx.download(ot)
    want = np.stack([table[mirror_index(n, index + i)] for i in range(B)])
    assert np.array_equal(_bits(got[:B]), _bits(want))
    assert np.array_equal(_bits(got[B]), _bits(obuf[B])), "written past the batch"


@pytest.mark.parametrize("N,H,W", [(2, 7, 10), (1, 33, 16), (3, 256, 256)])
@pytest.mark.parametrize("half_mask", [False, True], ids=["full", "masked"])
def test_vae_pre_matches_preprocess_img_bit_exact(ctx, N, H, W, half_mask):
    """vae_pre_kernel against oracle.musetalk_ref.preprocess_img(...).half(): BGR->RGB, /255, lower half zeroed (H // 2 rows kept,
    odd H), Normalize(0.5, 0.5); channels 3..15 of the 16-channel output written as 0."""
    from oracle.musetalk_ref import preprocess_img
    img = np.random.default_rng(N * H * W).integers(0, 256, (N, H, W, 3), dtype=np.uint8)
    img[0, 0, :3] = [[0, 0, 0], [255, 255, 255], [127, 128, 1]]
    obuf = np.full((N, H, W, 16), SENT_OUT, np.float16)
    ot = ctx.upload(obuf)
    ctx.vae_pre(ctx.upload(img), N, H, W, half_mask, ot)
    got = ctx.download(ot)
    want = np.zeros((N, H, W, 16), np.float16)
    for i in range(N):
        want[i, ..., :3] = preprocess_img(img[i], half_mask).half()[0].permute(1, 2, 0).numpy()
    assert np.array_equal(_bits(got), _bits(want))


def test_vae_post_matches_torch_fp16_bit_exact(ctx):
    """vae_post_kernel against the same arithmetic in torch fp16 on the CPU: (x/2 + 0.5).clamp(0, 1) in half, *255 in fp32,
    round-half-even, RGB -> BGR.  Every fp16 value in [-1.5, 1.5] appears (so every rounding boundary of the u8 scale is crossed),
    read from a 8-channel pitch whose channels 3..7 hold a sentinel."""
    from livetalking_b200.ops import DevTensor
    vals = np.arange(0, 1 << 16, dtype=np.uint32).astype(np.uint16).view(np.float16)
    vals = vals[np.isfinite(vals) & (np.abs(vals.astype(np.float32)) <= 1.5)]
    rng = np.random.default_rng(0)
    npix = (vals.size + 2) // 3 + 1
    rgb = np.concatenate([vals, rng.permutation(vals)[:npix * 3 - vals.size]]).reshape(npix, 3).astype(np.float16)
    rgb[-1] = [0, -1, 1]
    Ctot = 8
    x = np.full((npix, Ctot), SENT_IN, np.float16)
    x[:, :3] = rgb
    obuf = np.full((npix + 2, 3), 77, np.uint8)
    ot = ctx.upload(obuf)
    xt = ctx.upload(x)
    ctx.vae_post(DevTensor(xt.ptr, (npix, 3), pitch=Ctot), npix, ot)
    got = ctx.download(ot)
    t = (torch.from_numpy(rgb) / 2 + 0.5).clamp(0, 1).float().numpy()
    want = np.round(t * np.float32(255)).astype(np.uint8)[:, ::-1]
    assert np.array_equal(got[:npix], want), f"{int((got[:npix] != want).sum())} bytes differ"
    assert (got[npix:] == 77).all(), "written past the image"
