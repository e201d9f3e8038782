"""GPU: the small-map split-K conv kernel (csrc/conv_smallmap.cu, ltb_conv_variant kernel 4) against float64 on its own fp16 inputs.

Every wav2lip256 bottleneck geometry it supports (3x3 s1 with a residual on 8x8 and 4x4 maps, 3x3 s2 to 8x8 and 4x4, the
k3 s2 ConvT on 4x4 and 8x8 grids, the 4x4 valid conv to 1x1 and the 1x1 GEMM on a 1x1 map) at B = 16, 3 and 1, through
ltb_op_conv2d with the opt-in flag.  Inputs, outputs and residuals are channel slices whose neighbours hold sentinels that must
keep their bits.  Each output is held to conv_check.py with the gather rounding order (the split partials summed in fp32 with
the bias and residual, one fp16 rounding): the bound of test_gpu_w2l_layers.py with the planned split count, and the rounding
model.  Also: two launches are
bit-identical, the planner routes the wav2lip256 bottleneck geometries here only when asked, and the wav2lip256 forward with
LTB_CONV_SMALLMAP on and off agrees within the layers' bounds."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from conv_cases import bits, ctx, slice_buf

import conv_check as cc

pytestmark = pytest.mark.gpu

SENT = -3.25

# id: (IH, Cin, Cout, k, stride, pad, transposed, residual)
CASES = {
    "res3x3_8x8": (8, 512, 512, 3, 1, 1, False, True),       # L28 / L37
    "res3x3_4x4": (4, 512, 512, 3, 1, 1, False, True),       # L30 / L35
    "s2_16to8": (16, 256, 512, 3, 2, 1, False, False),       # L27
    "s2_8to4": (8, 512, 512, 3, 2, 1, False, False),         # L29
    "convT_4x4": (4, 1024, 512, 3, 2, 1, True, False),       # L36
    "convT_8x8": (8, 1024, 512, 3, 2, 1, True, False),       # L38
    "k4_valid": (4, 512, 512, 4, 1, 0, False, False),        # L31
    "gemm_1x1": (1, 512, 512, 1, 1, 0, False, False),        # L32 / L33
    "gemm_1x1_wide": (1, 1024, 8192, 1, 1, 0, False, False),  # L34 (the k4 ConvT on the 1x1 map)
}
# ConvTranspose2d(k3, s2, p1, op1) sub-pixel packing (conv_plan.cu kTk / kTn): phase (a, b) reads kernel rows kTk[a][:kTn[a]]
KTK, KTN = ((1, 0), (2, 0)), (1, 2)


def _pack(w, transposed):
    """fp16 K-major rows [Cout][Ktot] in the kernels' order (dense: [kh][kw][ci]; ConvT: the four sub-pixel phases in turn)."""
    if not transposed:
        cout, cin, kh, kw = w.shape
        return np.ascontiguousarray(w.permute(0, 2, 3, 1).reshape(cout, kh * kw * cin).numpy()).astype(np.float16)
    cin, cout = w.shape[:2]
    cols = [w[:, :, KTK[a][i], KTK[b][j]].t() for a in (0, 1) for b in (0, 1) for i in range(KTN[a]) for j in range(KTN[b])]
    return np.ascontiguousarray(torch.cat(cols, 1).numpy()).astype(np.float16)


def _problem(name, B, seed):
    IH, cin, cout, k, s, p, tr, res = CASES[name]
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(B, IH, IH, cin, generator=g) * 0.7).half()
    shape = (cin, cout, k, k) if tr else (cout, cin, k, k)
    w = (torch.randn(*shape, generator=g) * (2.0 / (cin * k * k)) ** 0.5).half().double()
    b = torch.randn(cout, generator=g).double() * 0.2
    xd = x.double().permute(0, 3, 1, 2)
    if tr:
        conv = F.conv_transpose2d(xd, w, stride=2, padding=1, output_padding=1)
        A = F.conv_transpose2d(xd.abs(), w.abs(), stride=2, padding=1, output_padding=1)
    else:
        conv = F.conv2d(xd, w, stride=s, padding=p)
        A = F.conv2d(xd.abs(), w.abs(), stride=s, padding=p)
    OH = conv.shape[2]
    r = (torch.randn(B, OH, OH, cout, generator=g) * 0.5).half() if res else None
    return dict(x=x, w=w, b=b, conv=conv, A=A, r=r, OH=OH, IH=IH, cin=cin, cout=cout, k=k, s=s, p=p, tr=tr)


def _launch(ctx, P, B, smallmap=True, plan_only=False, slices=True):
    from livetalking_b200.ops import DevTensor
    cin, cout = P["cin"], P["cout"]
    ic = (cin + 64, 32) if slices else (cin, 0)
    oc = (cout + 128, 64) if slices else (cout, 0)
    rc = (cout + 32, 16) if slices else (cout, 0)
    xv, xt, xbuf = slice_buf(ctx, P["x"].numpy(), ic[0], ic[1], 512.0)
    ov, ot, obuf = slice_buf(ctx, np.full((B, P["OH"], P["OH"], cout), SENT, np.float16), oc[0], oc[1], SENT)
    rv = slice_buf(ctx, P["r"].numpy(), rc[0], rc[1], 512.0)[0] if P["r"] is not None else None
    k = P["k"]
    wt = SimpleNamespace(w=ctx.upload(_pack(P["w"].float(), P["tr"])), w_tap=None, bias=ctx.upload(P["b"].float().numpy()),
                         cin=cin, cout=cout, kh=k, kw=k, ktot=k * k * cin)
    kw = dict(N=B, IH=P["IH"], IW=P["IH"], OH=P["OH"], OW=P["OH"], stride=(P["s"], P["s"]), pad=(P["p"], P["p"]), res=rv, relu=True,
              transposed=P["tr"], smallmap=smallmap)
    if plan_only:
        return ctx.conv_plan(xv, wt, ov, **kw)
    ctx.conv(xv, wt, ov, **kw)
    full = ctx.download(ot)
    outside = np.ones(obuf.shape, bool)
    outside[..., oc[1]:oc[1] + cout] = False
    assert np.array_equal(bits(full)[outside], bits(obuf)[outside]), "the conv wrote outside its output slice"
    assert np.array_equal(bits(ctx.download(xt)), bits(xbuf)), "the conv changed its input buffer"
    return full[..., oc[1]:oc[1] + cout]


def _check(P, got, ks, what):
    K = 4 * P["cin"] if P["tr"] else P["cin"] * P["k"] ** 2
    assert ks <= min(32, K // 128)
    nhwc = lambda t: t.permute(0, 2, 3, 1).numpy()
    return cc.check(got, nhwc(P["conv"]), nhwc(P["A"]), P["b"].numpy(), K=K, order=cc.order_of(dict(kernel=4)), relu=True,
                    r=None if P["r"] is None else P["r"].numpy(), ks=ks, what=what)


@pytest.mark.parametrize("B", [16, 3, 1])
@pytest.mark.parametrize("name", list(CASES))
def test_smallmap_against_float64(ctx, name, B):
    P = _problem(name, B, seed=len(name) + B)
    v = _launch(ctx, P, B, plan_only=True)
    assert v["kernel"] == 4 and v["bn"] == 128 and v["kb"] == 64, v
    assert v["taps"] == (9 if P["tr"] else P["k"] ** 2), v
    got = _launch(ctx, P, B, slices=(B != 1))
    _check(P, got, v["ksplit"], f"smallmap {name} B={B}")


@pytest.mark.parametrize("name", ["res3x3_8x8", "convT_8x8", "k4_valid"])
def test_two_launches_bit_identical(ctx, name):
    P = _problem(name, 16, seed=7)
    a = _launch(ctx, P, 16)
    b = _launch(ctx, P, 16)
    assert np.array_equal(bits(a), bits(b))


def test_routing_is_opt_in(ctx):
    """The bottleneck geometries at B = 16 take the kernel with the flag (and these split counts), and never without it."""
    want_ks = {"res3x3_8x8": 8, "res3x3_4x4": 8, "s2_16to8": 8, "s2_8to4": 8, "convT_4x4": 8, "convT_8x8": 8, "k4_valid": 8,
               "gemm_1x1": 4, "gemm_1x1_wide": 2}
    for name, ks in want_ks.items():
        P = _problem(name, 16, seed=1)
        v = _launch(ctx, P, 16, plan_only=True)
        assert v["kernel"] == 4 and v["ksplit"] == ks, (name, v)
        assert _launch(ctx, P, 16, smallmap=False, plan_only=True)["kernel"] != 4, name


def test_w2l_forward_switch_on_and_off(monkeypatch):
    """The batch-16 wav2lip256 forward with the bottleneck on this kernel and on the halo / gather kernels: pred agrees to well
    inside the layers' rounding (split-K reorders fp32 sums, then every later layer rounds to fp16)."""
    from livetalking_b200 import engine, synth
    from livetalking_b200.w2l_pack import pack_state_dict
    engine.set_device(0)
    model = engine.W2LModel(pack_state_dict(synth.random_state_dict(0)))
    av = engine.W2LAvatar(*synth.synthetic_avatar(n=16, H=720, W=1280, bbox=(200, 520, 480, 800)))
    rng = np.random.default_rng(3)
    mel = rng.standard_normal((16, 80, 16)).astype(np.float32)
    preds, times = {}, {}
    for val in ("1", "0"):
        monkeypatch.setenv("LTB_CONV_SMALLMAP", val)
        s = engine.W2LSession(model, av, 16)
        try:
            preds[val] = s.infer(0, mel).astype(np.float64)
            ms = np.median(np.stack([s.profile_ops(0)[0] for _ in range(3)]), axis=0)
            times[val] = float(ms[29:41].sum()) * 1e3
        finally:
            s.close()
    d = np.abs(preds["1"] - preds["0"])
    print(f"\npred |diff| max {d.max():.4f} mean {d.mean():.6f} (of 255); L27-L38 {times['1']:.1f} us on, {times['0']:.1f} us off")
    assert np.isfinite(preds["1"]).all()
    assert d.max() < 2.0 and d.mean() < 0.1
