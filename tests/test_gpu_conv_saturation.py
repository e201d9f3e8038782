"""GPU: every conv epilogue at the edge of the fp16 range.

One row per epilogue implementation: the gather kernel's direct epilogue and its split-K finalize, the halo kernel with no
residual, with the residual from shared memory and from global memory, its GEMM mode, the ping-pong, row-pair and small-map
kernels.  Half of the output channels get a bias of +-(65504 + U(-3000, 3000)) on inputs scaled by 32, so that their
pre-activations straddle +-65504: some saturate, others land just below.  Residuals are large (N(0, 1) x 600, or the scaled
input itself) so that the two rounding orders part.  Each row runs with ReLU on and off.  The output must hold no inf and no
NaN, must pass conv_check.py (the in-range elements), and must equal the rounding model bit for bit on the saturated elements.

The two kernel families differ there, and the rows pin both: where acc + b > 65504 and r < 0, the halo family (halo,
ping-pong) returns fp16(65504 + r), because it saturates fp16(acc + b) before the fp16 residual add, while the gather family
(gather, split-K finalize, small-map) returns min(acc + b + r, 65504) rounded once.  The difference is acceptable: both are
the saturating fp16 result of a value beyond the fp16 range, and the shipped models keep their activations below 2^14
(test_gpu_s3fd.py asserts it), far from either."""
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from conv_cases import ctx, slice_buf  # noqa: F401  (fixture)

import conv_check as cc

pytestmark = pytest.mark.gpu

SCALE = 32.0

# id: (N, H, W, Cin, Cout, k, residual: None / "sep" / "input" / "copy", extra conv kwargs, expected variant fields)
ROWS = {
    "gather_direct": ((2, 20, 22, 64, 64, 3), "sep", dict(no_halo=1), dict(kernel=0, ksplit=1)),
    "gather_splitk": ((2, 8, 8, 256, 64, 3), "sep", dict(no_halo=1), dict(kernel=0, ksplit=4)),
    "halo_no_res": ((6, 128, 20, 96, 96, 3), None, {}, dict(kernel=1)),
    "halo_res_smem": ((6, 128, 20, 96, 96, 3), "input", {}, dict(kernel=1)),
    "halo_res_gmem": ((6, 128, 20, 96, 96, 3), "copy", {}, dict(kernel=1)),
    "halo_gemm": ((2, 36, 120, 40, 256, 1), "sep", {}, dict(kernel=1, taps=1)),
    "pingpong": ((16, 64, 64, 64, 64, 3), "input", {}, dict(kernel=2)),
    "rowpair": ((16, 72, 80, 80, 32, 3), None, {}, dict(kernel=3)),
    "smallmap": ((16, 8, 8, 512, 512, 3), "sep", dict(smallmap=True), dict(kernel=4)),
}


@pytest.mark.parametrize("relu", [False, True], ids=["no_relu", "relu"])
@pytest.mark.parametrize("name", list(ROWS))
def test_saturating_epilogue_matches_model(ctx, name, relu):
    (N, H, W, Cin, Cout, k), res, extra, want = ROWS[name]
    g = torch.Generator().manual_seed(len(name) * 7 + relu)
    x = ((torch.randn(N, H, W, Cin, generator=g) * 0.7 + 0.4 + torch.randn(Cin, generator=g) * 0.3) * SCALE).half()
    w = (torch.randn(Cout, Cin, k, k, generator=g) * (2.0 / (Cin * k * k)) ** 0.5).half()
    b = torch.randn(Cout, generator=g) * 0.2
    edge = torch.arange(Cout) % 2 == 1          # odd channels straddle the fp16 limit, with both signs
    sign = torch.where(torch.arange(Cout) % 4 == 1, 1.0, -1.0)
    b = torch.where(edge, sign * (65504.0 + (torch.rand(Cout, generator=g) * 2 - 1) * 3000.0), b).float()
    pad = k // 2
    temps = []
    try:
        xv, xt, _ = slice_buf(ctx, x.numpy(), Cin, 0, 0.0)
        ov, ot, _ = slice_buf(ctx, np.full((N, H, W, Cout), np.nan, np.float16), Cout, 0, 0.0)
        temps += [xt, ot]
        r = rv = None
        if res == "sep":
            r = (torch.randn(N, H, W, Cout, generator=g) * 600.0).half().numpy()
        elif res in ("input", "copy"):
            r = x.numpy()
        if res == "input":
            rv = xv
        elif r is not None:
            rv, rt, _ = slice_buf(ctx, r, Cout, 0, 0.0)
            temps.append(rt)
        wt = ctx.upload(w.permute(0, 2, 3, 1).reshape(Cout, k * k * Cin).numpy())
        bt = ctx.upload(b.numpy())
        temps += [wt, bt]
        wtap = None
        if k == 3:
            wtap = ctx.alloc((9, Cout, Cin))
            ctx.w_tap_major(wt, wtap, Cout, Cin)
            temps.append(wtap)
        cw = types.SimpleNamespace(cout=Cout, cin=Cin, kh=k, kw=k, ktot=k * k * Cin, w=wt, w_tap=wtap, bias=bt)
        geo = dict(N=N, IH=H, IW=W, OH=H, OW=W, pad=(pad, pad), relu=relu, res=rv, **extra)
        v = ctx.conv_plan(xv, cw, ov, **geo)
        assert all(v[f] == want[f] for f in want), (name, v)
        if name.startswith("halo_res"):
            assert ctx.conv_res_halo(xv, cw, ov, **geo) == (res == "input"), name
        ctx.conv(xv, cw, ov, **geo)
        got = ctx.download(ot)
    finally:
        for t in temps:
            ctx.free(t)

    x64 = x.double().permute(0, 3, 1, 2)
    conv = F.conv2d(x64, w.double(), padding=pad).permute(0, 2, 3, 1).numpy()
    A = F.conv2d(x64.abs(), w.double().abs(), padding=pad).permute(0, 2, 3, 1).numpy()
    order = cc.order_of(v)
    what = f"saturation {name} relu={relu}"
    assert np.isfinite(got.astype(np.float32)).all(), f"{what}: inf / NaN in the output"
    pre = conv + b.double().numpy()
    tot = pre + (r.astype(np.float64) if r is not None else 0.0)
    hi = tot > cc.F16_MAX if r is None or order == "gather" else pre > cc.F16_MAX
    assert hi.any() and ((tot > 60000) & (tot < cc.F16_MAX)).any(), f"{what}: the inputs do not straddle +65504"
    if not relu:
        assert (tot < -cc.F16_MAX).any(), f"{what}: no element saturates at -65504"
    cc.check(got, conv, A, b.double().numpy(), K=k * k * Cin, order=order, relu=relu, r=r, ks=cc.ksplit_of(v), what=what)
    n = cc.check_saturated(got, conv, b.double().numpy(), order=order, relu=relu, r=r, what=what)
    if r is not None:
        # the two orders part on the saturated elements: the row pins which one the kernel follows
        other = cc.model(pre, r.astype(np.float64), relu, "gather" if order == "halo" else "halo")
        mine = cc.model(pre, r.astype(np.float64), relu, order)
        assert (other != mine)[np.abs(pre) > cc.F16_MAX].any(), f"{what}: the two orders agree on every saturated element"
    print(f"{what}: {n} saturated elements equal the {order} model")
