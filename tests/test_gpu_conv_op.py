"""GPU: the features of ltb_op_conv2d that the MuseTalk / Whisper / UltraLight graphs use and the dense ltb_conv2d_f16 descriptor of
test_gpu_conv.py never reaches: channel-sliced input / output / residual, asymmetric padding, batched GEMMs (zbatch / zdiv), Ktot
larger than the taps times Cin with a NULL bias, and the GroupNorm statistics output (fused into the conv epilogue or a separate
pass) consumed by ltb_op_groupnorm_apply.

References are float64 PyTorch on the same fp16 inputs and fp16 weights.  Conv outputs are held to conv_check.py: the hard error
bound and the rounding model of the kernel Ctx.conv_plan reports (K = kh kw Cin, 4 Cin for the fused upsample, the padded head
dim or key count for the batched GEMMs).  Slice neighbours of inputs hold 512 and of outputs a second sentinel; a kernel that
reads a neighbour channel or writes one fails the comparison or the bit check."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import conv_check as cc

pytestmark = pytest.mark.gpu

SENT_IN = 512.0
SENT_OUT = -3.25


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


def _check_conv(r, what):
    """conv_check.check on a _run_conv result."""
    return cc.check(r["out"], r["conv"], r["A"], r["b"], K=r["K"], order=cc.order_of(r["variant"]), relu=r["relu"], r=r["res"],
                    ks=cc.ksplit_of(r["variant"]), conv_model=r["conv_model"], upsample=r["conv_model"] is not None,
                    what=f"{what} (planned {r['variant']})")


def _run_conv(ctx, *, N, IH, IW, Cin, Cout, k=3, stride=1, pad=(1, 1), ref_pad=None, ic=None, oc=None, rc=None, no_halo=False,
              upsample=False, relu=False, gn=None, seed=0):
    """One ltb_op_conv2d through ops.Ctx.conv.  ic / oc / rc = (pitch, offset) of the input / output / residual slice (None: dense,
    no residual).  gn = (groups, guard_floats) asks for GroupNorm statistics.  ref_pad: F.pad (left, right, top, bottom) of the
    reference (default: the symmetric `pad`).  Returns a dict with the dense output, the float64 reference, the launch count and
    the downloaded statistics buffer; conv, A, b, res, K, conv_model and variant for _check_conv."""
    from livetalking_b200.ops import ConvWeight, DevTensor
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(N, IH, IW, Cin, generator=g) * 0.7 + torch.randn(Cin, generator=g) * 0.3).half()
    w = (torch.randn(Cout, Cin, k, k, generator=g) * (2.0 / (Cin * k * k)) ** 0.5).half()
    b = torch.randn(Cout, generator=g) * 0.2
    x0 = x.double().permute(0, 3, 1, 2)
    xd = F.interpolate(x0, scale_factor=2, mode="nearest") if upsample else x0
    if ref_pad is None:
        ref_pad = (pad[1], pad[1], pad[0], pad[0])
    conv = F.conv2d(F.pad(xd, ref_pad), w.double(), stride=stride)
    A = F.conv2d(F.pad(xd.abs(), ref_pad), w.double().abs(), stride=stride).permute(0, 2, 3, 1).numpy()
    conv_model = cc.upsample_presummed(x0, w.float().numpy()).permute(0, 2, 3, 1).numpy() if upsample else None
    OH, OW = conv.shape[2], conv.shape[3]
    conv = conv.permute(0, 2, 3, 1).numpy()
    ic, oc = ic or (Cin, 0), oc or (Cout, 0)
    xv, xt, xbuf = _slice_buf(ctx, x.numpy(), ic[0], ic[1], SENT_IN)
    ov, ot, obuf = _slice_buf(ctx, np.full((N, OH, OW, Cout), SENT_OUT, np.float16), oc[0], oc[1], SENT_OUT)
    rv = r = None
    if rc is not None:
        r = (torch.randn(N, OH, OW, Cout, generator=g) * 0.5).half().numpy()
        rv, _rt, _rbuf = _slice_buf(ctx, r, rc[0], rc[1], SENT_IN)
    cw = ConvWeight(ctx, w.float().numpy(), b.numpy())
    st = None
    if gn is not None:
        groups, guard = gn
        st = ctx.upload(np.full(N * groups * 2 + guard, -0.0, np.float32))
    geo = dict(N=N, IH=IH, IW=IW, OH=OH, OW=OW, stride=(stride, stride), pad=pad, res=rv, relu=relu, no_halo=no_halo,
               upsample2x=upsample)
    variant = ctx.conv_plan(xv, cw, ov, **geo)
    before = ctx.launch_count
    ctx.conv(xv, cw, ov, gn_stats=st, gn_groups=gn[0] if gn else 0, gn_hw=OH * OW if gn else 0, **geo)
    launches = ctx.launch_count - before
    full = ctx.download(ot)
    written = np.zeros(obuf.shape, bool)
    written[..., oc[1]:oc[1] + Cout] = True
    changed = (_bits(full) != _bits(obuf)) & ~written
    assert not changed.any(), f"conv wrote {int(changed.sum())} elements outside its output slice, first at {np.argwhere(changed)[0]}"
    assert np.array_equal(_bits(ctx.download(xt)), _bits(xbuf)), "conv changed its input buffer"
    return dict(out=full[..., oc[1]:oc[1] + Cout], conv=conv, A=A, b=b.numpy(), res=r, relu=relu, variant=variant,
                K=4 * Cin if upsample else k * k * Cin, conv_model=conv_model, launches=launches,
                stats=ctx.download(st) if st is not None else None, view=ov, OH=OH, OW=OW)


# ------------------------------------------------------------------------------------------------ slices, padding
SLICE_CASES = [
    # id, kwargs: kernel reached / what it would catch
    ("halo_cin80_of160", dict(N=2, IH=32, IW=16, Cin=80, Cout=64, ic=(160, 40), oc=(96, 16), rc=(80, 8))),
    #   3x3 halo (TMA): the second 64-channel chunk must be zero-filled past Cin, not read from the neighbour slice
    ("halo_overhang", dict(N=3, IH=12, IW=20, Cin=64, Cout=64, ic=(128, 64), oc=(192, 128), rc=(64, 0), relu=True)),
    #   3x3 halo with overhanging tiles: masked rows / columns must not write the sliced output
    ("s2_parity_planes", dict(N=2, IH=64, IW=32, Cin=64, Cout=64, stride=2, ic=(192, 64), oc=(128, 64))),
    #   stride-2 parity-plane TMA path (TAPS = 10) on a slice
    ("gemm_tma", dict(N=2, IH=16, IW=24, Cin=96, Cout=64, k=1, pad=(0, 0), ic=(128, 16), oc=(128, 32), rc=(96, 24))),
    #   TMA GEMM mode (1x1, M = 768): 2-D tensor map over a channel slice, slice epilogue
    ("gather_no_halo", dict(N=2, IH=12, IW=12, Cin=48, Cout=32, ic=(64, 8), oc=(64, 24), rc=(48, 16), no_halo=True)),
    #   cp.async gather kernel (no_halo = 1): ic_off in the gather, oc_off / rc_off in its epilogue
    ("upsample2x_fused", dict(N=2, IH=8, IW=8, Cin=64, Cout=64, upsample=True, ic=(128, 64), oc=(192, 64))),
    #   fused nearest-2x upsample + 3x3 (sub-pixel phases, TAPS = 16) reading a slice, writing a slice
    ("splitk_finalize", dict(N=2, IH=4, IW=4, Cin=1280, Cout=640, ic=(1280 + 64, 32), oc=(1280, 640), rc=(1280, 320))),
    #   split-K gather (180 K blocks, M = 32): the finalize kernel writes the output slice and reads the residual slice
    ("vae_down_pad00", dict(N=2, IH=16, IW=16, Cin=64, Cout=64, stride=2, pad=(0, 0), ref_pad=(0, 1, 0, 1), ic=(128, 0), oc=(64, 0))),
    #   VAE Downsample2D: pad (0, 0) at stride 2 with the implicit bottom / right zero row (gather kernel)
    ("ultralight_pad33", dict(N=2, IH=16, IW=16, Cin=16, Cout=16, stride=2, pad=(3, 3), oc=(32, 16), no_halo=True, relu=True)),
    #   UltraLight conv5: pad (3, 3) at stride 2, 16 -> 10
]


@pytest.mark.parametrize("name,kw", SLICE_CASES, ids=[c[0] for c in SLICE_CASES])
def test_conv_op_slices_and_padding(ctx, name, kw):
    r = _run_conv(ctx, seed=len(name), **kw)
    _check_conv(r, name)


# ------------------------------------------------------------------------------------------------ Ktot > taps * Cin, NULL bias
@pytest.mark.parametrize("rows", [37, 640], ids=["gather", "gemm_tma"])
def test_conv_op_weight_koff_and_null_bias(ctx, rows):
    """A 1x1 conv whose weight rows are longer than Cin (Ktot = Cin + 40) and start at column w_koff = 16, with bias = NULL (the
    context's zero bias): the gather kernel (37 rows) and the TMA GEMM mode (640 rows) must read exactly w[:, 16:16+Cin]."""
    from livetalking_b200._capi import ConvOp, check, lib
    Cin, Cout, koff, Ktot = 64, 96, 16, 64 + 40
    rng = np.random.default_rng(rows)
    x = (rng.standard_normal((rows, Cin)) * 0.7).astype(np.float16)
    w = np.full((Cout, Ktot), SENT_IN, np.float16)
    w[:, koff:koff + Cin] = (rng.standard_normal((Cout, Cin)) / 8).astype(np.float16)
    xt, wt = ctx.upload(x), ctx.upload(w)
    ot = ctx.upload(np.full((rows, Cout), SENT_OUT, np.float16))
    d = ConvOp()
    d.in_, d.w, d.w_tap, d.bias, d.res, d.out = xt.ptr, wt.ptr, None, None, None, ot.ptr
    d.N, d.IH, d.IW, d.ICtot, d.ic_off, d.Cin = 1, 1, rows, Cin, 0, Cin
    d.OH, d.OW, d.Cout, d.OCtot, d.oc_off = 1, rows, Cout, Cout, 0
    d.KH = d.KW = d.sy = d.sx = 1
    d.Ktot, d.w_koff, d.zdiv = Ktot, koff, 1
    check(lib().ltb_op_conv2d(ctx._h, C.byref(d)))
    got = ctx.download(ot)
    wk = w[:, koff:koff + Cin].astype(np.float64).T
    x64 = x.astype(np.float64)
    # no residual: the gather and the halo GEMM epilogue both round acc + 0 once
    cc.check(got, x64 @ wk, np.abs(x64) @ np.abs(wk), 0.0, K=Cin, order="gather", ks=cc.ks_ceiling(Cin), what=f"koff rows={rows}")


# ------------------------------------------------------------------------------------------------ batched GEMMs (attention, unfused)
@pytest.mark.parametrize("mode", ["self_padded_keys", "cross_key_pad"])
def test_batched_gemms_of_unfused_attention(ctx, mode):
    """The two zbatch / zdiv GEMMs of Builder.attention's unfused branch (LTB_FUSE_ATTENTION=0) with exactly its arguments:
    S = Q K^T per (batch, head) with Ktot = kv_pitch and a NULL bias, then O = P V^T-transposed into the heads' column slices of O.
    Self-attention pads 40 keys to 48 (the padded K rows are zero rows of the qkv buffer); cross-attention has KEY_PAD = 64 keys
    per batch item.  Compared with torch.bmm in float64."""
    from livetalking_b200.musetalk import KEY_PAD
    from livetalking_b200.ops import DevTensor
    rng = np.random.default_rng(7 if mode.startswith("self") else 8)
    H, d = 2, 40
    dp = 48
    Hdp = H * dp
    if mode == "self_padded_keys":
        B, nq = 1, 40
        nk, kv_rows = 48, nq
        qkv = np.zeros((B * nq + (nk - nq), 3 * Hdp), np.float16)
        qkv[:B * nq] = (rng.standard_normal((B * nq, 3 * Hdp)) * 0.5).astype(np.float16)
        buf = ctx.upload(qkv)
        q_ptr, q_pitch = buf.ptr, 3 * Hdp
        k_ptr, kv_pitch = buf.offset(Hdp), 3 * Hdp
        Q = qkv[:, :Hdp]
        K = qkv[:, Hdp:2 * Hdp]
    else:
        B, nq = 2, 64
        nk = kv_rows = KEY_PAD
        q = (rng.standard_normal((B * nq, Hdp)) * 0.5).astype(np.float16)
        kv = (rng.standard_normal((B * nk, 2 * Hdp)) * 0.5).astype(np.float16)
        qt, kvt = ctx.upload(q), ctx.upload(kv)
        q_ptr, q_pitch = qt.ptr, Hdp
        k_ptr, kv_pitch = kvt.ptr, 2 * Hdp
        Q, K = q, kv[:, :Hdp]
    S = ctx.upload(np.full((B * H, nq, nk), SENT_OUT, np.float16))
    qv = DevTensor(q_ptr, (nq, dp), pitch=q_pitch)
    sv = DevTensor(S.ptr, (nq, nk), pitch=nk)
    ctx.conv(qv, None, sv, N=1, IH=1, IW=nq, OH=1, OW=nq, cin=dp, cout=nk, w_ptr=k_ptr, ktot=kv_pitch,
             zbatch=B * H, zdiv=H, in_z=(nq * q_pitch, dp), w_z=(kv_rows * kv_pitch, dp), out_z=(H * nq * nk, nq * nk))
    got_s = ctx.download(S).astype(np.float64)
    Qh = Q[:B * nq].astype(np.float64).reshape(B, nq, H, dp).transpose(0, 2, 1, 3)
    if mode == "self_padded_keys":
        Kh = K[:nk].astype(np.float64).reshape(1, nk, H, dp).transpose(0, 2, 1, 3)           # rows 40..47: the zero padding rows
    else:
        Kh = K.astype(np.float64).reshape(B, nk, H, dp).transpose(0, 2, 1, 3)
    def bmm(a, b):
        return torch.bmm(torch.from_numpy(a), torch.from_numpy(b).transpose(1, 2)).numpy()
    Qh, Kh = Qh.reshape(B * H, nq, dp), Kh.reshape(B * H, nk, dp)
    # no bias, no residual: one rounding of the exact sum over the padded head dim
    cc.check(got_s, bmm(Qh, Kh), bmm(np.abs(Qh), np.abs(Kh)), 0.0, K=dp, order="gather", ks=cc.ks_ceiling(dp), what=f"{mode} Q K^T")
    # P V: probabilities (zero in padded key columns) times V^T laid out [B, H, dp, nk] by transpose_heads
    P = rng.uniform(0, 1, (B * H, nq, nk))
    P[..., 50 if mode != "self_padded_keys" else nq:] = 0
    P = (P / P.sum(-1, keepdims=True)).astype(np.float16)
    VT = (rng.standard_normal((B * H, dp, nk)) * 0.8).astype(np.float16)
    S2, VTt = ctx.upload(P), ctx.upload(VT)
    O = ctx.upload(np.full((B * nq, Hdp), SENT_OUT, np.float16))
    sv2 = DevTensor(S2.ptr, (nq, nk), pitch=nk)
    ov = DevTensor(O.ptr, (nq, dp), pitch=Hdp)
    ctx.conv(sv2, None, ov, N=1, IH=1, IW=nq, OH=1, OW=nq, cin=nk, cout=dp, w_ptr=VTt.ptr, ktot=nk,
             zbatch=B * H, zdiv=H, in_z=(H * nq * nk, nq * nk), w_z=(H * dp * nk, dp * nk), out_z=(nq * Hdp, dp))
    got_o = ctx.download(O).astype(np.float64)
    def heads(a):
        return a.reshape(B, H, nq, dp).transpose(0, 2, 1, 3).reshape(B * nq, Hdp)
    P64, VT64 = P.astype(np.float64), VT.astype(np.float64)
    cc.check(got_o, heads(bmm(P64, VT64)), heads(bmm(np.abs(P64), np.abs(VT64))), 0.0, K=nk, order="gather", ks=cc.ks_ceiling(nk),
             what=f"{mode} P V")


# ------------------------------------------------------------------------------------------------ GroupNorm statistics
GN_CASES = [
    # id, kwargs, groups, fused (1 launch) or separate pass (2): kernel / table reached
    ("halo_cpg4", dict(N=2, IH=16, IW=16, Cin=64, Cout=64), 16, True),              # halo 3x3, lane-pair reduction, smem table
    ("halo_cpg8", dict(N=2, IH=32, IW=16, Cin=32, Cout=128), 16, True),             # halo 3x3, 8-column blocks
    ("halo_cpg16", dict(N=1, IH=16, IW=16, Cin=64, Cout=512, rc=(512, 0)), 32, True),   # two 8-column blocks per group, residual
    ("halo_overhang", dict(N=3, IH=12, IW=20, Cin=64, Cout=64), 16, True),          # overhanging tiles: masked rows must not count
    ("halo_12_images", dict(N=12, IH=16, IW=16, Cin=32, Cout=128), 32, True),       # 12 x 32 groups: global-atomic table
    ("s2_cpg4", dict(N=2, IH=64, IW=32, Cin=64, Cout=64, stride=2), 16, True),      # stride-2 parity-plane path
    ("gemm_smem", dict(N=4, IH=16, IW=16, Cin=64, Cout=128, k=1, pad=(0, 0)), 32, True),    # TMA GEMM mode, shared table
    ("sep_cpg10", dict(N=2, IH=16, IW=16, Cin=64, Cout=320), 32, False),            # 10 channels per group: separate pass
    ("sep_cpg40", dict(N=2, IH=4, IW=4, Cin=64, Cout=1280), 32, False),             # 40 channels per group: separate pass
    ("sep_gather", dict(N=2, IH=8, IW=8, Cin=64, Cout=64, no_halo=True), 16, False),   # gather kernel: separate pass
    ("sep_oc_off", dict(N=2, IH=16, IW=16, Cin=64, Cout=64, oc=(128, 32)), 16, False),  # output slice: separate pass over the slice
]


def _check_stats_and_apply(ctx, r, groups, what, apply=True):
    """apply=False: only the statistics (groupnorm_apply takes at most 64 groups)."""
    from livetalking_b200.ops import DevTensor
    out = r["out"].astype(np.float64)
    N, OH, OW, Cout = out.shape
    g = out.reshape(N, OH * OW, groups, Cout // groups)
    s_ref, q_ref = g.sum(axis=(1, 3)), (g * g).sum(axis=(1, 3))
    st = r["stats"][:N * groups * 2].reshape(N, groups, 2).astype(np.float64)
    abs_sum = np.abs(g).sum(axis=(1, 3))
    assert (np.abs(st[..., 0] - s_ref) <= 1e-4 * abs_sum + 1e-3).all(), \
        f"{what}: group sums off by {np.abs(st[..., 0] - s_ref).max():.4g} (worst at {np.unravel_index(np.abs(st[..., 0] - s_ref).argmax(), s_ref.shape)})"
    assert (np.abs(st[..., 1] - q_ref) <= 1e-4 * q_ref + 1e-3).all(), \
        f"{what}: group sums of squares off by {np.abs(st[..., 1] - q_ref).max():.4g}"
    if not apply:
        return
    # groupnorm_apply on these statistics against F.group_norm in float64
    rng = np.random.default_rng(Cout + groups)
    gamma = rng.uniform(0.5, 1.5, Cout).astype(np.float32)
    beta = rng.uniform(-0.5, 0.5, Cout).astype(np.float32)
    stt = ctx.upload(r["stats"])
    yt = ctx.upload(np.full((N, OH, OW, Cout), SENT_OUT, np.float16))
    ctx.groupnorm_apply(r["view"], N, OH * OW, groups, 1e-5, stt, ctx.upload(gamma), ctx.upload(beta), True,
                        DevTensor(yt.ptr, (N, OH, OW, Cout)))
    y = ctx.download(yt).astype(np.float64)
    ref = F.silu(F.group_norm(torch.from_numpy(out).permute(0, 3, 1, 2), groups, torch.from_numpy(gamma).double(),
                              torch.from_numpy(beta).double(), 1e-5)).permute(0, 2, 3, 1).numpy()
    err = np.abs(y - ref)
    assert (err <= 1e-3 + 2e-3 * np.abs(ref)).all(), f"{what}: groupnorm_apply max err {err.max():.4g}"


@pytest.mark.parametrize("name,kw,groups,fused", GN_CASES, ids=[c[0] for c in GN_CASES])
def test_conv_op_groupnorm_statistics(ctx, name, kw, groups, fused):
    """(sum, sum of squares) per (image, group) of the conv's fp16 output, against float64 sums of the downloaded output; then
    groupnorm_apply on them against F.group_norm.  The launch count tells the fused epilogue (1) from the separate pass (2).
    The 2*groups floats after the table hold -0.0 and must keep their bits."""
    r = _run_conv(ctx, seed=len(name) + 100, gn=(groups, 2 * groups), **kw)
    _check_conv(r, name)
    assert r["launches"] == (1 if fused else 2), f"{name}: {r['launches']} launches"
    N = kw["N"]
    guard = r["stats"][N * groups * 2:]
    assert np.array_equal(guard.view(np.uint32), np.full(guard.shape, 0x80000000, np.uint32)), \
        f"{name}: statistics written past the table at {np.flatnonzero(guard.view(np.uint32) != 0x80000000)[:8]}"
    _check_stats_and_apply(ctx, r, groups, name)


def test_fused_gemm_statistics_stay_inside_the_table(ctx):
    """TMA GEMM mode with NSUB = 2 and an odd number of 128-row blocks (19 images of 16x24, 64 -> 320 channels, 80 groups of 4:
    BN = 64, 29 x 5 tiles): the second sub-tile of the last tile lies wholly past M.  Its warps must not add their (zero) partial
    sums at image index 19, one table past the end; the -0.0 guard would turn +0.0 there."""
    groups = 80
    r = _run_conv(ctx, seed=19, N=19, IH=16, IW=24, Cin=64, Cout=320, k=1, pad=(0, 0), gn=(groups, 2 * groups))
    _check_conv(r, "gemm nsub2")
    assert r["launches"] == 1, "expected the statistics fused into the GEMM epilogue"
    guard = r["stats"][19 * groups * 2:]
    bad = np.flatnonzero(guard.view(np.uint32) != 0x80000000)
    assert bad.size == 0, f"fused GEMM statistics wrote {bad.size} floats past the table (guard offsets {bad[:8]})"
    _check_stats_and_apply(ctx, r, groups, "gemm nsub2", apply=False)
