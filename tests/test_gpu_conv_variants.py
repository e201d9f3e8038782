"""Every compiled instance of the two conv kernels against a float64 reference, each test proving which instance it ran.

conv_halo.cu builds conv_halo_wgmma_kernel<BN, NSUB, NACC, TAPS, RC, GRP> and conv_gather.cu conv_gather_wgmma_kernel<BN, KB, GRP>;
which one runs is decided by the host planner from the shape (and, for the resident-weight halo variants, the SM count).  VARIANTS
has one row per instance, keyed by its template arguments: an ltb_op_conv2d geometry that Ctx.conv_plan (ltb_op_conv2d_plan) must
map to exactly that instance, then the op itself against float64 PyTorch on the same fp16 inputs and fp16 weights, held to
conv_check.py: the hard error bound and the rounding model of the instance's kernel.  Inputs, outputs and residuals are channel slices whose neighbours hold sentinels; every
byte outside the output slice must keep its bits and the inputs must not change.  Rows reach, where the instance admits them: a
ragged last M tile or overhanging halo tiles, Cin that is not a multiple of 64 (zero-filled last K chunk), several N tiles (the
resident variants need exactly one), more tiles than SMs (persistent halo CTAs run a second tile, the mbarrier phases wrap), and
relu in every other row on inputs with a non-zero mean.

Grouped rows run three groups with the slot table [S-1, 0, S-1] over a bank of S = 5 weight slots (the last slot used, one slot
repeated), with group rows that are not a multiple of the M tile; each group is compared with float64 on its own slot's weights
and, where the ungrouped op on that group plans the same instance, bit for bit with it.

The expected variants are those of the 132-SM H100 SXM.  test_variants_cover_every_compiled_instance (CPU) checks that VARIANTS
lists exactly the instances in the built objects, so a new instance without a row fails the suite."""
import os
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from kernel_instances import compiled_instances

import conv_check as cc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H100_SMS = 132
SLOTS, TABLE = 5, [4, 0, 4]
SENT_IN = 512.0
SENT_OUT = -3.25


def H(bn, nsub, nacc, taps, rc=0, grp=False):
    return ("halo", bn, nsub, nacc, taps, rc, grp)


def G(bn, kb, grp=False):
    return ("gather", bn, kb, grp)


def _conv(N, IH, IW, Cin, Cout, k=3, stride=1, pad=1, **kw):
    return dict(kind="conv", N=N, IH=IH, IW=IW, Cin=Cin, Cout=Cout, k=k, stride=stride, pad=pad, **kw)


def _convT(N, IH, IW, Cin, Cout):
    return dict(kind="convT", N=N, IH=IH, IW=IW, Cin=Cin, Cout=Cout, k=3, stride=1, pad=1)


def _up(N, IH, IW, Cin, Cout):
    return dict(kind="up", N=N, IH=IH, IW=IW, Cin=Cin, Cout=Cout, k=3, stride=1, pad=1)


def _gemm(N, IH, IW, Cin, Cout, **kw):
    return _conv(N, IH, IW, Cin, Cout, k=1, pad=0, **kw)


# key: geometry.  gi = images per group (grouped rows: N = 3 gi); no_halo = 1 forces the gather kernel where the halo kernel
# would take the shape.  The comment gives the tiles (halo: persistent tiles vs 132 SMs) or the gather grid (M tiles x N tiles).
VARIANTS = {
    # halo 3x3, streamed weights: 80 channels = a full and a zero-filled K chunk
    H(128, 2, 1, 9): _conv(5, 128, 36, 80, 256),             # 200 tiles, 36 columns: overhanging column tiles, 2 N tiles
    H(128, 1, 1, 9): _conv(8, 20, 20, 80, 384),              # 144 tiles, 20 x 20: overhanging row and column tiles
    H(64, 2, 1, 9): _conv(6, 128, 20, 80, 192),              # 216 tiles, 3 N tiles
    H(64, 1, 1, 9): _conv(6, 20, 12, 80, 384),               # 144 tiles, 6 N tiles
    H(32, 2, 1, 9): _conv(6, 128, 20, 80, 96),               # 216 tiles
    H(32, 1, 1, 9): _conv(8, 20, 20, 80, 96),                # 144 tiles
    # halo 3x3, resident weights: one N tile, >= 2 x 132 tiles, 40 channels (one chunk) or 80 (two)
    H(64, 2, 1, 9, 1): _conv(4, 128, 132, 40, 64),           # 272 tiles, overhanging column tiles
    H(32, 2, 1, 9, 1): _conv(4, 128, 132, 40, 32),
    H(32, 2, 1, 9, 2): _conv(4, 128, 132, 80, 32),
    # halo ConvT (four phase accumulators): 8 x 20 / 8 x 132 maps overhang the 16-row tile
    H(64, 1, 4, 9): _convT(16, 8, 20, 40, 192),              # 144 tiles, 3 N tiles
    H(32, 1, 4, 9): _convT(16, 8, 20, 40, 96),
    H(64, 1, 4, 9, 1): _convT(16, 8, 132, 40, 64),           # 272 tiles, resident
    H(64, 1, 4, 9, 2): _convT(16, 8, 132, 80, 64),
    H(32, 1, 4, 9, 1): _convT(16, 8, 132, 40, 32),
    H(32, 1, 4, 9, 2): _convT(16, 8, 132, 80, 32),
    # halo stride-2 parity planes: 36 x 36 output overhangs the 16 x 8 tile, 135 tiles
    H(64, 1, 1, 10): _conv(3, 72, 72, 80, 192, stride=2),
    H(32, 1, 1, 10): _conv(3, 72, 72, 80, 96, stride=2),
    # halo fused nearest-2x upsample + 3x3: 24 x 60 low-resolution map, 144 tiles
    H(64, 1, 4, 16): _up(3, 24, 60, 40, 192),
    # halo GEMM mode (1x1): ragged M, 40 channels
    H(128, 1, 1, 1): _gemm(2, 36, 120, 40, 256),             # 136 tiles
    H(64, 2, 1, 1): _gemm(1, 100, 120, 40, 192),             # 141 tiles
    H(64, 1, 1, 1): _gemm(1, 24, 120, 40, 384),              # 138 tiles
    H(32, 2, 1, 1): _gemm(1, 100, 120, 40, 96),              # 141 tiles
    H(32, 1, 1, 1): _gemm(3, 10, 70, 40, 256),               # 136 tiles
    # halo grouped GEMM mode: group rows 400 / 3888 / 1800 are not multiples of 128 * NSUB
    H(128, 1, 1, 1, 0, True): _gemm(3, 36, 50, 40, 384, gi=1),   # 135 tiles
    H(64, 2, 1, 1, 0, True): _gemm(9, 36, 36, 40, 192, gi=3),    # 144 tiles
    H(64, 1, 1, 1, 0, True): _gemm(3, 36, 50, 40, 192, gi=1),    # 135 tiles
    H(32, 2, 1, 1, 0, True): _gemm(9, 36, 36, 40, 96, gi=3),     # 144 tiles
    H(32, 1, 1, 1, 0, True): _gemm(3, 10, 40, 40, 384, gi=1),    # 144 tiles
    # gather, ungrouped (no split-K: either more than 8 M tiles or fewer than 32 K blocks)
    G(128, 64): _conv(2, 66, 66, 64, 256, no_halo=1),                # 69 x 2
    G(128, 32): _conv(2, 132, 132, 96, 256, stride=2, no_halo=1),    # 69 x 2, stride 2
    G(128, 16): _gemm(2, 66, 66, 48, 256, no_halo=1),                # 69 x 2, 1x1
    G(64, 64): _conv(2, 54, 54, 128, 192, k=2, pad=0),               # 44 x 3, 2x2 valid
    G(64, 32): _conv(3, 44, 44, 96, 192, no_halo=1),                 # 46 x 3
    G(64, 16): _conv(3, 96, 96, 48, 192, k=4, stride=2),             # 54 x 3, 4x4 stride 2 pad 1
    G(32, 64): _conv(2, 20, 22, 64, 64, no_halo=1),                  # 7 x 2
    G(32, 32): _gemm(2, 12, 13, 96, 96),                             # 3 x 3, M = 312 is too small for the GEMM mode
    G(32, 16): _conv(2, 16, 16, 48, 128, stride=2, pad=3),           # 2 x 4, UltraLight conv5 padding
    G(16, 64): _conv(2, 15, 17, 128, 48, no_halo=1),                 # 4 x 3
    G(16, 32): _gemm(1, 20, 23, 32, 80),                             # 4 x 5
    G(16, 16): _conv(2, 30, 30, 16, 48),                             # 15 x 3, Cout = 48 is no halo geometry
    # gather, grouped: group rows 2888 / 1922 / 240 / 200 / 198 / 81 / 260 are not multiples of 128
    G(128, 64, True): _conv(6, 38, 38, 64, 256, gi=2),
    G(128, 32, True): _conv(6, 76, 76, 96, 256, stride=2, gi=2),
    G(128, 16, True): _gemm(6, 38, 38, 48, 256, gi=2, no_halo=1),
    G(64, 64, True): _conv(6, 32, 32, 128, 192, k=2, pad=0, gi=2),
    G(64, 32, True): _conv(6, 31, 31, 96, 192, gi=2),
    G(64, 16, True): _conv(6, 62, 62, 48, 192, k=4, stride=2, gi=2),
    G(32, 64, True): _conv(6, 12, 10, 64, 64, gi=2),
    G(32, 32, True): _conv(6, 24, 20, 96, 96, stride=2, gi=2),
    G(32, 16, True): _conv(6, 16, 16, 48, 128, stride=2, pad=3, gi=2),
    G(16, 64, True): _conv(6, 9, 11, 128, 48, gi=2),
    G(16, 32, True): _conv(3, 9, 9, 32, 80, gi=1),                   # one image per group, 81 rows: less than one M tile
    G(16, 16, True): _conv(6, 10, 13, 16, 48, gi=2),
}

# split-K: 8 x 8 map, 36 K blocks in one M tile -> four K slices and the finalize kernel
SPLITK = (_conv(2, 8, 8, 256, 64, no_halo=1), dict(kernel=0, taps=0, bn=64, nsub=0, nacc=0, resident_chunks=0, kb=64, ksplit=4, grouped=0))

# UltraLight audio branch at 4 groups of 4 images (cross-session batching): a3 128 -> 256 at 32 -> 16 (s2 p1) and a5 256 -> 512 at
# 16 -> 10 (s2 p3), both on the grouped gather kernel
SHIPPED_GROUPED = {
    "ultralight_a3": (_conv(16, 32, 32, 128, 256, stride=2, gi=4, table=[4, 0, 4, 2]), G(32, 64, True)),
    "ultralight_a5": (_conv(16, 16, 16, 256, 512, stride=2, pad=3, gi=4, table=[4, 0, 4, 2]), G(32, 64, True)),
}


def _expected(key):
    if key[0] == "halo":
        _, bn, nsub, nacc, taps, rc, grp = key
        return dict(kernel=1, taps=taps, bn=bn, nsub=nsub, nacc=nacc, resident_chunks=rc, kb=0, ksplit=0, grouped=int(grp))
    _, bn, kb, grp = key
    return dict(kernel=0, taps=0, bn=bn, nsub=0, nacc=0, resident_chunks=0, kb=kb, ksplit=1, grouped=int(grp))


def _key_id(key):
    return f"{key[0]}<{','.join(str(int(a)) for a in key[1:])}>"


# ------------------------------------------------------------------------------------------------ completeness (CPU)
def test_variants_cover_every_compiled_instance():
    halo = compiled_instances("conv_halo.o", "conv_halo_wgmma_kernel")
    gather = compiled_instances("conv_gather.o", "conv_gather_wgmma_kernel")
    compiled = {H(bn, ns, na, t, rc, bool(g)) for bn, ns, na, t, rc, g in halo} | {G(bn, kb, bool(g)) for bn, kb, g in gather}
    assert len(halo) == 28 and len(gather) == 24, (len(halo), len(gather))
    missing = sorted(map(_key_id, compiled - set(VARIANTS)))
    stale = sorted(map(_key_id, set(VARIANTS) - compiled))
    assert not missing and not stale, f"instances without a test row: {missing}; rows for instances that are not compiled: {stale}"


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def ctx():
    from livetalking_b200 import engine
    from livetalking_b200.ops import Ctx
    engine.set_device(0)
    c = Ctx()
    yield c
    c.close()


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint16)


def _slice_buf(ctx, dense, pitch, off, fill):
    """dense (..., C) placed at channels [off, off + C) of a (..., pitch) buffer whose other channels hold `fill`."""
    from livetalking_b200.ops import DevTensor
    buf = np.full(dense.shape[:-1] + (pitch,), fill, np.float16)
    buf[..., off:off + dense.shape[-1]] = dense
    t = ctx.upload(buf)
    return DevTensor(t.ptr, dense.shape, pitch=pitch, c_off=off), t, buf


def _shape_weight(cout, cin, k, w=None, w_tap=None, bias=None):
    """The geometry (and optionally the device tensors) Ctx.conv reads from a ConvWeight."""
    return types.SimpleNamespace(cout=cout, cin=cin, kh=k, kw=k, ktot=k * k * cin, w=w, w_tap=w_tap, bias=bias)


# ConvTranspose2d(k3, s2, p1, op1) as sub-pixel phases: phase a of a dimension reads kernel taps kTk[a] at input offsets 0, +1
_T_TAPS = {0: [1], 1: [2, 0]}


def _pack_convT(w):
    """(Cin, Cout, 3, 3) -> phase-major rows (Cout, 9 Cin) and the TMA kernel's view-major slices (9, Cout, Cin)
    (ltb_conv_op.transposed)."""
    slices = [w[:, :, kh, kw].T for a in (0, 1) for b in (0, 1) for kh in _T_TAPS[a] for kw in _T_TAPS[b]]
    rows = np.concatenate(slices, axis=1)
    view = np.stack([slices[i] for i in (0, 1, 5, 2, 6, 8, 7, 4, 3)])
    return np.ascontiguousarray(rows), np.ascontiguousarray(view)


def _reference(row, x, w):
    """float64 NHWC parts of the row's op on x (N, Cin, H, W) and w (Cout, Cin, k, k), ConvT (Cin, Cout, 3, 3): (conv without
    bias, conv of the absolute values, the fused upsample's sum with its pre-summed fp16 weights or None)."""
    def op(a, b):
        if row["kind"] == "convT":
            return F.conv_transpose2d(a, b, stride=2, padding=1, output_padding=1)
        if row["kind"] == "up":
            a = F.interpolate(a, scale_factor=2, mode="nearest")
        p = row["pad"]
        return F.conv2d(F.pad(a, (p, p, p, p)), b, stride=row["stride"])
    nhwc = lambda t: t.permute(0, 2, 3, 1).numpy()
    up = nhwc(cc.upsample_presummed(x, w.float().numpy())) if row["kind"] == "up" else None
    return nhwc(op(x, w)), nhwc(op(x.abs(), w.abs())), up


def _chain_k(row):
    return 4 * row["Cin"] if row["kind"] in ("convT", "up") else row["k"] ** 2 * row["Cin"]


def _check_model(got, parts, b, r, relu, row, variant, what, ks=None):
    """conv_check.check of the row's output: parts = (conv, A, conv_model) of _reference, b the bias per element."""
    conv, A, up = parts
    return cc.check(got, conv, A, b, K=_chain_k(row), order=cc.order_of(variant), relu=relu, r=r,
                    ks=cc.ksplit_of(variant) if ks is None else ks, conv_model=up, upsample=up is not None, what=what)


def _run_row(ctx, row, seed, relu, with_res):
    """Plan and run one row through Ctx.conv_plan / Ctx.conv.  Returns (variant, output slice, float64 reference, ungrouped
    check) where the last is a callable (group g, slot s) -> (variant, output) of the ungrouped op on that group's images."""
    from livetalking_b200._capi import LtbError
    from livetalking_b200.ops import DevTensor
    kind, N, IH, IW, Cin, Cout, k = (row[n] for n in ("kind", "N", "IH", "IW", "Cin", "Cout", "k"))
    gi, table = row.get("gi"), row.get("table", TABLE)
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(N, IH, IW, Cin, generator=g) * 0.7 + 0.4 + torch.randn(Cin, generator=g) * 0.3).half()
    nslot = SLOTS if gi else 1
    if kind == "convT":
        w = torch.randn(nslot, Cin, Cout, 3, 3, generator=g) * (2.0 / (Cin * 9 / 4)) ** 0.5
    else:
        w = torch.randn(nslot, Cout, Cin, k, k, generator=g) * (2.0 / (Cin * k * k)) ** 0.5
    w = w.half()
    b = torch.randn(nslot, Cout, generator=g) * 0.2
    x64 = x.double().permute(0, 3, 1, 2)
    OH, OW = (2 * IH, 2 * IW) if kind in ("convT", "up") else ((IH + 2 * row["pad"] - k) // row["stride"] + 1,
                                                               (IW + 2 * row["pad"] - k) // row["stride"] + 1)
    ICtot, OCtot, RCtot = Cin + 24, Cout + 16, Cout + 8
    xv, xt, xbuf = _slice_buf(ctx, x.numpy(), ICtot, 8, SENT_IN)
    ov, ot, obuf = _slice_buf(ctx, np.full((N, OH, OW, Cout), np.nan, np.float16), OCtot, 8, SENT_OUT)
    rv = r = None
    if with_res:
        r = (torch.randn(N, OH, OW, Cout, generator=g) * 0.5).half()
        rv, rt, rbuf = _slice_buf(ctx, r.numpy(), RCtot, 8, SENT_IN)
    geo = dict(N=N, IH=IH, IW=IW, OH=OH, OW=OW, stride=(row["stride"], row["stride"]), pad=(row["pad"], row["pad"]), relu=relu,
               no_halo=row.get("no_halo", 0), res=rv, upsample2x=kind == "up", transposed=kind == "convT")
    temps = [xt, ot] + ([rt] if with_res else [])
    if kind == "convT":
        packed = [_pack_convT(w[s].numpy()) for s in range(nslot)]
        wrows = np.stack([p[0] for p in packed])
        wview = ctx.upload(packed[0][1])
        temps.append(wview)
    else:
        wrows = w.permute(0, 1, 3, 4, 2).reshape(nslot, Cout, k * k * Cin).numpy()
        wview = None
    wt, bt = ctx.upload(wrows), ctx.upload(b.numpy().astype(np.float32))
    temps += [wt, bt]
    if kind == "up":                            # the 16-slice weights of ConvWeight.upconv()
        from livetalking_b200.ops import ConvWeight
        cw = ConvWeight(ctx, w[0].float().numpy(), b[0].numpy(), tap_major=False)
        temps += [cw.w, cw.bias] + list(cw.upconv(ctx))
    elif gi:
        cw = _shape_weight(Cout, Cin, k)
        tab = ctx.upload(np.asarray(table, np.int32))
        temps.append(tab)
        geo.update(w_ptr=wt.ptr, bias_ptr=bt.ptr, group=(tab, gi, SLOTS, Cout * k * k * Cin, Cout))
    else:
        wtap = wview
        if kind == "conv" and k == 3:
            wtap = ctx.alloc((9, Cout, Cin))
            ctx.w_tap_major(wt, wtap, Cout, Cin)
            temps.append(wtap)
        cw = _shape_weight(Cout, Cin, k, wt, wtap, bt)
    variant = ctx.conv_plan(xv, cw, ov, **geo)
    ctx.conv(xv, cw, ov, **geo)
    full = ctx.download(ot)
    written = np.zeros(obuf.shape, bool)
    written[..., 8:8 + Cout] = True
    changed = (_bits(full) != _bits(obuf)) & ~written
    assert not changed.any(), f"{variant}: wrote {int(changed.sum())} elements outside the output slice, first at {np.argwhere(changed)[0]}"
    assert np.array_equal(_bits(ctx.download(xt)), _bits(xbuf)), "the conv changed its input buffer"
    if with_res:
        assert np.array_equal(_bits(ctx.download(rt)), _bits(rbuf)), "the conv changed its residual buffer"
    got = full[..., 8:8 + Cout]
    slots = [table[n // gi] for n in range(N)] if gi else [0] * N
    # each group's float64 parts with its own slot's weights and bias
    parts = [np.empty(got.shape, np.float64) for _ in range(3 if kind == "up" else 2)]
    bias = np.empty((N, 1, 1, Cout), np.float64)
    for s in sorted(set(slots)):
        idx = [n for n in range(N) if slots[n] == s]
        for dst, src in zip(parts, _reference(row, x64[idx], w[s].double())):
            dst[idx] = src
        bias[idx] = b[s].double().numpy()
    ref = (parts[0], parts[1], parts[2] if kind == "up" else None), bias, (r.numpy() if with_res else None)

    def ungrouped(grp, s):
        """The ungrouped op on group grp's images with slot s's weights, into a fresh output slice."""
        lo = grp * gi
        xg = DevTensor(xv.offset(lo * IH * IW * ICtot), (gi, IH, IW, Cin), pitch=ICtot, c_off=8)
        og, ogt, _ = _slice_buf(ctx, np.full((gi, OH, OW, Cout), np.nan, np.float16), OCtot, 8, SENT_OUT)
        gg = dict(geo, N=gi, group=None, w_ptr=wt.ptr + s * Cout * k * k * Cin * 2, bias_ptr=bt.ptr + s * Cout * 4)
        if with_res:
            gg["res"] = DevTensor(rv.offset(lo * OH * OW * RCtot), (gi, OH, OW, Cout), pitch=RCtot, c_off=8)
        try:
            v = ctx.conv_plan(xg, cw, og, **gg)
        except LtbError:        # e.g. 400 rows of 40 channels: too few rows for the GEMM mode, a Cin the gather kernel cannot take
            v = None
        out = None
        if v is not None:
            ctx.conv(xg, cw, og, **gg)
            out = ctx.download(ogt)[..., 8:8 + Cout]
        ctx.free(ogt)
        return v, out

    ctx.sync()
    return (variant, got, ref, ungrouped if gi else None, slots), temps


def _assert_variant(variant, want, sms, what):
    assert variant == want and sms == H100_SMS, (
        f"{what}: planned {variant}, expected {want} (the expected variants assume the {H100_SMS}-SM H100 SXM; this device has "
        f"{sms} SMs)")


def _check_row(ctx, sms, what, row, want, seed, relu, with_res):
    (variant, got, (parts, bias, r), ungrouped, slots), temps = _run_row(ctx, row, seed, relu, with_res)
    try:
        _check_model(got, parts, bias, r, relu, row, variant, f"{what} (planned {variant})")
        _assert_variant(variant, want, sms, what)
        if ungrouped is not None:
            gi = row["gi"]
            same = 0
            for grp in range(row["N"] // gi):
                v, alone = ungrouped(grp, slots[grp * gi])
                if v is not None and dict(v, grouped=1) == want:
                    assert np.array_equal(_bits(alone), _bits(got[grp * gi:(grp + 1) * gi])), \
                        f"{what}: group {grp} differs from the ungrouped op on the same instance {v}"
                    same += 1
            print(f"{what}: {same} of {row['N'] // gi} groups bit-identical to the ungrouped op on the same instance")
    finally:
        for t in temps:
            ctx.free(t)


ROWS = list(VARIANTS.items())


@pytest.mark.gpu
@pytest.mark.parametrize("key,row", ROWS, ids=[_key_id(k) for k, _ in ROWS])
def test_conv_variant_matches_float64(ctx, sms, key, row):
    i = ROWS.index((key, row))
    _check_row(ctx, sms, _key_id(key), row, _expected(key), seed=1000 + i, relu=i % 2 == 0, with_res=i % 3 != 2)


@pytest.mark.gpu
def test_splitk_variant_matches_float64(ctx, sms):
    row, want = SPLITK
    _check_row(ctx, sms, "split-K", row, want, seed=7, relu=True, with_res=True)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SHIPPED_GROUPED))
def test_shipped_grouped_stride2_convs_match_float64(ctx, sms, name):
    row, key = SHIPPED_GROUPED[name]
    _check_row(ctx, sms, name, row, _expected(key), seed=len(name), relu=True, with_res=False)
