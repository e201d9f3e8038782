"""GPU: the UltraLight leaf kernels (csrc/ultralight.cu: dwconv3x3, upsample_bilinear2x, ul_prep; csrc/w2l_small.cu: the
sigmoid * 255 head) against float64 references computed from the same inputs.

Channel-sliced inputs sit between neighbours that hold SENT_IN; outputs are pre-filled with SENT_OUT and every element outside the
written slice must keep its bits.  ul_prep is bit-exact; the others are within a bound derived in each test's docstring, multiplied
by SAFETY = 1.25 for second-order terms, with the worst err / bound printed.  Both grid-stride kernels cap their grid at 148 x 16
blocks of 256 threads (606,208 work items of 8 channels); the BIG shapes have more work items than that, so the loop takes a
second trip."""
import numpy as np
import pytest

SENT_IN = 512.0
SENT_OUT = -3.25
SAFETY = 1.25
GRID_ITEMS = 148 * 16 * 256


@pytest.fixture(scope="module")
def ctx():
    from livetalking_b200 import engine
    from livetalking_b200.ops import Ctx
    engine.set_device(0)
    c = Ctx()
    yield c
    c.close()


def _bits(a):
    return np.ascontiguousarray(a).view({2: np.uint16, 4: np.uint32, 1: np.uint8}[a.dtype.itemsize])


def _check(got, ref, bound, what):
    got = np.asarray(got, np.float64)
    assert np.isfinite(got).all(), f"{what}: non-finite output"
    ratio = np.abs(got - ref) / (SAFETY * bound)
    worst = float(ratio.max())
    print(f"{what}: worst err/bound {worst:.3f}")
    assert worst <= 1.0, (f"{what}: {int((ratio > 1).sum())} of {ratio.size} outside the bound; worst err/bound {worst:.2f} at "
                          f"{np.unravel_index(ratio.argmax(), ratio.shape)}")


def _sliced(ctx, dense, pitch, off):
    from livetalking_b200.ops import DevTensor
    buf = np.full(dense.shape[:-1] + (pitch,), SENT_IN, np.float16)
    buf[..., off:off + dense.shape[-1]] = dense
    t = ctx.upload(buf)
    return DevTensor(t.ptr, dense.shape, pitch=pitch, c_off=off)


def _out_slice(ctx, shape, pitch, off):
    from livetalking_b200.ops import DevTensor
    buf = np.full(shape[:-1] + (pitch,), SENT_OUT, np.float16)
    t = ctx.upload(buf)
    return DevTensor(t.ptr, shape, pitch=pitch, c_off=off), t, buf


def _slice_result(ctx, t, buf, off, Cc, what):
    got = ctx.download(t)
    written = np.zeros(buf.shape, bool)
    written[..., off:off + Cc] = True
    changed = (_bits(got) != _bits(buf)) & ~written
    assert not changed.any(), f"{what}: {int(changed.sum())} elements outside the output slice changed"
    return got[..., off:off + Cc]


# ------------------------------------------------------------------------------------------------ depthwise 3x3
def _dw_ref(x, w9, b, stride, relu):
    """x (N, IH, IW, C) -> float64 (ref, bound): pad 1, stride s, + bias, ReLU, clamp to the fp16 range.
    Bound: nine fmas onto the fp32 bias, 10 2^-24 (|b| + sum |x w|), and fp16 rounding 2^-11 |ref| + 2^-25."""
    N, IH, IW, Cc = x.shape
    OH, OW = (IH - 1) // stride + 1, (IW - 1) // stride + 1
    xp = np.zeros((N, IH + 2, IW + 2, Cc))
    xp[:, 1:-1, 1:-1] = x.astype(np.float64)
    acc = np.zeros((N, OH, OW, Cc)) + b
    mag = np.zeros((N, OH, OW, Cc)) + np.abs(b)
    for ky in range(3):
        for kx in range(3):
            tap = xp[:, ky:ky + stride * (OH - 1) + 1:stride, kx:kx + stride * (OW - 1) + 1:stride]
            acc += tap * w9[ky * 3 + kx]
            mag += np.abs(tap * w9[ky * 3 + kx])
    ref = np.clip(np.maximum(acc, 0) if relu else acc, -65504, 65504)
    return ref, 10 * 2.0 ** -24 * mag + 2.0 ** -11 * np.abs(ref) + 2.0 ** -25


DW_CASES = [
    # N, IH, IW, C, stride, relu
    (2, 1, 7, 8, 1, False),        # IH = 1
    (3, 6, 1, 8, 2, True),         # IW = 1, stride 2
    (2, 5, 5, 16, 2, False),       # 5 -> 3
    (2, 9, 13, 192, 1, True),      # ragged, C = 192
    (1, 7, 4, 192, 2, False),
    (8, 80, 80, 192, 1, False),    # BIG: 1,228,800 work items
    (16, 160, 160, 64, 2, True),   # BIG at stride 2: 819,200 work items
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", DW_CASES, ids=[f"N{c[0]}_{c[1]}x{c[2]}_C{c[3]}_s{c[4]}{'_relu' if c[5] else ''}" for c in DW_CASES])
def test_dwconv3x3_matches_float64(ctx, case):
    """dwconv3x3_kernel<false> from a channel slice into a channel slice (bound: _dw_ref)."""
    N, IH, IW, Cc, stride, relu = case
    rng = np.random.default_rng(sum(case))
    x = (2 * rng.standard_normal((N, IH, IW, Cc))).astype(np.float16)
    w9 = rng.standard_normal((9, Cc)).astype(np.float16)
    b = rng.standard_normal(Cc).astype(np.float32)
    OH, OW = (IH - 1) // stride + 1, (IW - 1) // stride + 1
    if N >= 8:   # the BIG rows
        assert N * OH * OW * Cc // 8 > GRID_ITEMS
    ov, ot, obuf = _out_slice(ctx, (N, OH, OW, Cc), Cc + 24, 16)
    ctx.dwconv3x3(_sliced(ctx, x, Cc + 16, 8), N, IH, IW, ctx.upload(w9), ctx.upload(b), stride, relu, ov)
    got = _slice_result(ctx, ot, obuf, 16, Cc, "dwconv3x3")
    ref, bound = _dw_ref(x, w9.astype(np.float64), b.astype(np.float64), stride, relu)
    _check(got, ref, bound, f"dwconv3x3 {case}")


@pytest.mark.gpu
def test_dwconv3x3_grouped_matches_float64_per_slot(ctx):
    """dwconv3x3_kernel<true>: slot table [2, 0, 2] over three weight slots, two images per group; every group against float64 with
    its own slot's weights and bias."""
    table, images, slots = [2, 0, 2], 2, 3
    N, IH, IW, Cc, stride, relu = len(table) * images, 11, 9, 64, 2, True
    rng = np.random.default_rng(202)
    x = (2 * rng.standard_normal((N, IH, IW, Cc))).astype(np.float16)
    w = rng.standard_normal((slots, 9, Cc)).astype(np.float16)
    b = rng.standard_normal((slots, Cc)).astype(np.float32)
    OH, OW = (IH - 1) // stride + 1, (IW - 1) // stride + 1
    ov, ot, obuf = _out_slice(ctx, (N, OH, OW, Cc), Cc + 8, 8)
    ctx.dwconv3x3(_sliced(ctx, x, Cc + 16, 8), N, IH, IW, ctx.upload(w), ctx.upload(b), stride, relu, ov,
                  group=(ctx.upload(np.array(table, np.int32)), images, 9 * Cc, Cc))
    got = _slice_result(ctx, ot, obuf, 8, Cc, "dwconv3x3 grouped")
    for g, s in enumerate(table):
        sl = slice(g * images, (g + 1) * images)
        ref, bound = _dw_ref(x[sl], w[s].astype(np.float64), b[s].astype(np.float64), stride, relu)
        _check(got[sl], ref, bound, f"dwconv3x3 grouped group {g} (slot {s})")


# ------------------------------------------------------------------------------------------------ bilinear x2
UP_CASES = [(2, 1, 5, 8), (1, 7, 1, 16), (3, 5, 9, 40), (2, 13, 6, 192), (4, 80, 80, 64)]   # the last: 819,200 work items


@pytest.mark.gpu
@pytest.mark.parametrize("N,H,W,Cc", UP_CASES)
def test_upsample_bilinear2x_matches_float64(ctx, N, H, W, Cc):
    """F.interpolate(scale_factor=2, bilinear, align_corners=True) in float64 into the upper channel half of a concat buffer.
    Bound: the kernel's source coordinate sy * oy (sy = (H-1)/(2H-1), two fp32 roundings) is off by at most 2^-23 (H - 1), which
    moves a value by that times the largest step 2M between neighbours (M = max |x| of the image channel); the four products and
    three adds of the lerp and the weight roundings 10 2^-24 M; fp16 rounding 2^-11 |ref| + 2^-25."""
    import torch
    import torch.nn.functional as F
    rng = np.random.default_rng(N * 100 + H * 10 + W + Cc)
    x = (3 * rng.standard_normal((N, H, W, Cc))).astype(np.float16)
    ov, ot, obuf = _out_slice(ctx, (N, 2 * H, 2 * W, Cc), 2 * Cc, Cc)
    ctx.upsample_bilinear2x(_sliced(ctx, x, Cc + 8, 8), N, H, W, ov)
    got = _slice_result(ctx, ot, obuf, Cc, Cc, "upsample_bilinear2x")
    ref = F.interpolate(torch.from_numpy(x.astype(np.float64)).permute(0, 3, 1, 2), scale_factor=2, mode="bilinear",
                        align_corners=True).permute(0, 2, 3, 1).numpy()
    M = np.abs(x.astype(np.float64)).max(axis=(1, 2), keepdims=True)
    bound = 2.0 ** -11 * np.abs(ref) + 2.0 ** -25 + (10 * 2.0 ** -24 + 2.0 ** -22 * (H + W)) * M
    if N == 4:   # the BIG row
        assert N * 4 * H * W * Cc // 8 > GRID_ITEMS
    _check(got, ref, bound, f"upsample_bilinear2x N{N} {H}x{W} C{Cc}")


# ------------------------------------------------------------------------------------------------ 32 -> 3 head, sigmoid * 255
def _head_ref(x, w, b):
    """float64 255 * sigmoid(b + x w^T) and its bound in x255 units: the 32 fp32 fmas onto the bias, 33 2^-24 (|b| + sum |x w|),
    through sigmoid' <= 1/4; expf (2 ulp) moves sigmoid by at most sigma (1 - sigma) 2^-22 and the division and the * 255 add
    2 2^-24 sigma."""
    a = x.astype(np.float64) @ w.T + b
    sig = 1.0 / (1.0 + np.exp(-a))
    mag = np.abs(x.astype(np.float64)) @ np.abs(w).T + np.abs(b)
    return 255 * sig, 255 * (33 * 2.0 ** -24 * mag / 4 + sig * (1 - sig) * 2.0 ** -22 + 2 * 2.0 ** -24 * sig)


def _head_inputs(rng, npix):
    x = rng.standard_normal((npix, 32)).astype(np.float16)
    w = (0.5 * rng.standard_normal((3, 32))).astype(np.float32)
    w[:, 0] = 1.0
    b = np.array([0.25, -0.5, 0.125], np.float32)
    # saturation pixels: logits 40 + b (1 + expf(-40) rounds to 1: exactly 255) and -100 + b (expf(100) = inf: exactly 0)
    x[3] = 0
    x[3, 0] = 40
    x[npix - 2] = 0
    x[npix - 2, 0] = -100
    return x, w, b


@pytest.mark.gpu
def test_head_sigmoid255_matches_float64(ctx):
    """w2l_head_kernel<false> with npix % 256 != 0: three pixels past npix must keep their bits."""
    npix = 3 * 256 + 77
    x, w, b = _head_inputs(np.random.default_rng(845), npix)
    pbuf = np.full((npix + 3, 3), SENT_OUT, np.float32)
    pt = ctx.upload(pbuf)
    ctx.head_sigmoid255(ctx.upload(x), ctx.upload(w), ctx.upload(b), npix, pt)
    got = ctx.download(pt)
    assert np.array_equal(_bits(got[npix:]), _bits(pbuf[npix:])), "written past npix"
    assert (got[3] == 255.0).all() and (got[npix - 2] == 0.0).all(), (got[3], got[npix - 2])
    ref, bound = _head_ref(x, w.astype(np.float64), b.astype(np.float64))
    _check(got[:npix], ref, bound, "head_sigmoid255")


@pytest.mark.gpu
def test_head_sigmoid255_grouped_matches_float64_per_slot(ctx):
    """w2l_head_kernel<true>: slot table [2, 0, 2], two images of 512 pixels per group, each group against its own slot's weights."""
    table, images, hw = [2, 0, 2], 2, 512
    npix = len(table) * images * hw
    rng = np.random.default_rng(3)
    x, _w, _b = _head_inputs(rng, npix)
    w = (0.5 * rng.standard_normal((3, 3, 32))).astype(np.float32)
    w[:, :, 0] = 1.0
    b = np.tile(np.array([0.25, -0.5, 0.125], np.float32), (3, 1)) + np.arange(3, dtype=np.float32)[:, None] * 0.0625
    pbuf = np.full((npix + 3, 3), SENT_OUT, np.float32)
    pt = ctx.upload(pbuf)
    ctx.head_sigmoid255(ctx.upload(x), ctx.upload(w), ctx.upload(b), npix, pt, group=(ctx.upload(np.array(table, np.int32)), images, 96, 3),
                        hw=hw)
    got = ctx.download(pt)
    assert np.array_equal(_bits(got[npix:]), _bits(pbuf[npix:])), "written past npix"
    for g, s in enumerate(table):
        sl = slice(g * images * hw, (g + 1) * images * hw)
        ref, bound = _head_ref(x[sl], w[s].astype(np.float64), b[s].astype(np.float64))
        _check(got[sl], ref, bound, f"head_sigmoid255 grouped group {g} (slot {s})")
    assert (got[3] == 255.0).all() and (got[npix - 2] == 0.0).all()


# ------------------------------------------------------------------------------------------------ LightReal input glue
@pytest.mark.gpu
@pytest.mark.parametrize("nf,index,B", [(3, 5, 4), (1, 0, 2), (4, 1, 3)])
def test_ul_prep_bit_exact(ctx, nf, index, B):
    """ul_prep_kernel<false>: crop [4:164, 4:164] of faces[mirror_index(nf, index + b)] (indices past 2 nf included); channels 0-2
    are fp16(np.float32(p) / np.float32(255)) for every one of the 256 byte values, channels 3-5 the same with columns [5, 154] x
    rows [5, 149] zeroed (edges 4/5/154/155 and 4/5/149/150 checked by name), channels 6-15 exactly +0.  One image past B must
    keep its bits."""
    from oracle.paste_ref import mirror_index
    rng = np.random.default_rng(nf * 100 + index * 10 + B)
    faces = rng.integers(0, 256, (nf, 168, 168, 3), dtype=np.uint8)
    faces[0, 10, 4:90] = (np.arange(258) % 256).reshape(86, 3)
    obuf = np.full((B + 1, 160, 160, 16), SENT_OUT, np.float16)
    ot = ctx.upload(obuf)
    ctx.ul_prep(ctx.upload(faces), nf, ctx.upload(np.array([index], np.int32)), B, ot)
    got = ctx.download(ot)
    assert np.array_equal(_bits(got[B]), _bits(obuf[B])), "written past the batch"
    lut = (np.arange(256, dtype=np.float32) / np.float32(255)).astype(np.float16)
    want = np.zeros((B, 160, 160, 16), np.float16)
    for b in range(B):
        crop = lut[faces[mirror_index(nf, index + b), 4:164, 4:164]]
        want[b, ..., 0:3] = crop
        want[b, ..., 3:6] = crop
        want[b, 5:150, 5:155, 3:6] = 0
    assert np.array_equal(_bits(got[:B]), _bits(want)), f"{int((_bits(got[:B]) != _bits(want)).sum())} halves differ"
    used = np.unique(np.concatenate([faces[mirror_index(nf, index + b), 4:164, 4:164].ravel() for b in range(B)]))
    assert used.size == 256, "not every byte value was converted"
    for y, x, masked in ((4, 80, False), (5, 80, True), (149, 80, True), (150, 80, False),
                         (80, 4, False), (80, 5, True), (80, 154, True), (80, 155, False)):
        if masked:
            assert not _bits(got[:B, y, x, 3:6]).any(), (y, x)
        else:
            assert np.array_equal(_bits(got[:B, y, x, 3:6]), _bits(got[:B, y, x, 0:3])), (y, x)
    assert not _bits(got[:B, ..., 6:]).any(), "channels 6-15 must be exactly +0"
