"""GPU: the row-pair 80 -> 32 channel 3x3 conv (conv_rowpair.cu) and its fused head against the halo kernel it replaces.

The planner sends a 3x3 stride-1 conv with Cin = 80, Cout = 32 and no residual, with at least three 32 x 8 pixel tiles per SM, to
conv_rowpair_kernel (ltb_conv_variant.kernel = 3); LTB_CONV_ROWPAIR=0 keeps it on the halo kernel.  Each case runs the same op
on the same inputs and weights both ways in one process and requires bit-identical outputs: the new kernel issues its MMAs in
the halo kernel's order (its extra products are exact zeros) and rounds in the halo kernel's order.  The input is an 80-channel
slice whose neighbours hold sentinels, the output goes into a channel slice of a wider buffer, and nothing outside it may
change.  The fused head is checked through the whole wav2lip256 forward, whose pred it writes."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F
from conv_cases import bits, ctx, slice_buf, weights

import conv_check as cc

pytestmark = pytest.mark.gpu

SENT_IN = 512.0
SENT_OUT = -3.25
ROWPAIR = dict(kernel=3, taps=9, bn=32, nsub=1, nacc=1, resident_chunks=2, kb=0, ksplit=0, grouped=0)

# (N, H, W): 72 and 200 rows overhang the 32-row tile and 204 columns the 8-pixel tile (the output TMA store clips them)
CASES = [(16, 72, 80), (16, 96, 72), (3, 200, 204)]


@pytest.fixture
def switch(monkeypatch):
    def set_(on):
        monkeypatch.setenv("LTB_CONV_ROWPAIR", "1" if on else "0")
    return set_


@pytest.mark.parametrize("relu", [True, False], ids=["relu", "no_relu"])
@pytest.mark.parametrize("shape", CASES, ids=[f"b{n}_{h}x{w}" for n, h, w in CASES])
def test_rowpair_equals_halo_kernel(ctx, switch, shape, relu):
    N, H, W = shape
    g = torch.Generator().manual_seed(N * 1000 + H + W + relu)
    x = (torch.randn(N, H, W, 80, generator=g) * 0.7 + 0.2 + torch.randn(80, generator=g) * 0.3).half()
    w, b, cw, temps = weights(ctx, g, 80, 32)
    xv, xt, xbuf = slice_buf(ctx, x.numpy(), 96, 8, SENT_IN)
    temps.append(xt)
    outs = {}
    try:
        for on in (False, True):
            switch(on)
            ov, ot, obuf = slice_buf(ctx, np.full((N, H, W, 32), np.nan, np.float16), 48, 8, SENT_OUT)
            temps.append(ot)
            geo = dict(N=N, IH=H, IW=W, OH=H, OW=W, pad=(1, 1), relu=relu)
            variant = ctx.conv_plan(xv, cw, ov, **geo)
            if on:
                assert variant == ROWPAIR, variant
            else:
                assert variant["kernel"] == 1 and variant["bn"] == 32, variant
            ctx.conv(xv, cw, ov, **geo)
            full = ctx.download(ot)
            outside = np.ones(obuf.shape, bool)
            outside[..., 8:40] = False
            assert np.array_equal(bits(full)[outside], bits(obuf)[outside]), f"rowpair={on}: wrote outside the output slice"
            outs[on] = full[..., 8:40]
        assert np.array_equal(bits(ctx.download(xt)), bits(xbuf)), "the conv changed its input buffer"
        assert np.isfinite(outs[True].astype(np.float32)).all(), "unwritten outputs"
        diff = bits(outs[True]) != bits(outs[False])
        assert not diff.any(), f"{int(diff.sum())} of {diff.size} outputs differ from the halo kernel, first at {np.argwhere(diff)[0]}"
        # and against float64 on the first image (conv_check.py; no residual: one rounding of acc + b)
        x64 = x[:1].double().permute(0, 3, 1, 2)
        conv = F.conv2d(F.pad(x64, (1, 1, 1, 1)), w.double()).permute(0, 2, 3, 1).numpy()
        A = F.conv2d(F.pad(x64.abs(), (1, 1, 1, 1)), w.double().abs()).permute(0, 2, 3, 1).numpy()
        cc.check(outs[True][:1], conv, A, b.numpy(), K=9 * 80, order=cc.order_of(ROWPAIR), relu=relu,
                 what=f"rowpair b{N}_{H}x{W} relu={relu}")
    finally:
        for t in temps:
            ctx.free(t)


def test_plans_route_only_the_output_conv(ctx, switch):
    """L53 (cat7's 80 channels -> a 32-channel temporary at B = 16, 256 x 256) plans the row-pair kernel, and the halo
    kernel's <32,2,1,9,2> with the switch off.  A residual, other channel counts and layers with fewer than three tiles per SM
    keep their halo plans."""
    from livetalking_b200.ops import DevTensor
    g = torch.Generator().manual_seed(53)
    _, _, cw, temps = weights(ctx, g, 80, 32)
    N, S = 16, 256
    cat7 = ctx.alloc((N, S, S, 80))
    h = ctx.alloc((N, S, S, 32))
    temps += [cat7, h]
    try:
        x_v, h_v = DevTensor(cat7.ptr, (N, S, S, 80)), DevTensor(h.ptr, (N, S, S, 32))
        geo = dict(N=N, IH=S, IW=S, OH=S, OW=S, pad=(1, 1), relu=True)
        switch(True)
        assert ctx.conv_plan(x_v, cw, h_v, **geo) == ROWPAIR
        # 4 x 128 x 132: 272 tiles, fewer than three per SM (test_gpu_conv_variants' <32,2,1,9,2> row)
        small = dict(geo, N=4, IH=128, IW=132, OH=128, OW=132)
        assert ctx.conv_plan(DevTensor(cat7.ptr, (4, 128, 132, 80)), cw, DevTensor(h.ptr, (4, 128, 132, 32)), **small)["kernel"] == 1
        # a residual
        assert ctx.conv_plan(x_v, cw, h_v, **dict(geo, res=h_v))["kernel"] == 1
        switch(False)
        assert ctx.conv_plan(x_v, cw, h_v, **geo) == dict(ROWPAIR, kernel=1, nsub=2)
    finally:
        for t in temps:
            ctx.free(t)


@pytest.mark.parametrize("keep_layers", [False, True], ids=["fused_head", "keep_layers"])
def test_wav2lip_forward_unchanged(w2l_state_dict, switch, keep_layers):
    """The whole wav2lip256 forward at B = 16 gives the same pred, bit for bit, with L53 on the row-pair kernel as on the halo
    kernel: with the head fused into L53 (the production plan), and with L53's activations stored and the separate head kernel
    (keep_layers)."""
    from livetalking_b200 import engine
    from oracle import wav2lip_ref as R
    engine.set_device(0)
    model = engine.W2LModel.from_state_dict(w2l_state_dict)
    mel, img = R.synth_inputs(2, seed=7)
    f = (img[:, 3:6].permute(0, 2, 3, 1).numpy() * 255.0).round().astype(np.uint8)
    faces = [f[i % 2] for i in range(16)]
    frames = np.random.default_rng(4).integers(0, 256, (16, 360, 640, 3), np.uint8)
    boxes = [(20 + 3 * i, 20 + 3 * i + 200, 100 + i, 100 + i + 190) for i in range(16)]
    av = engine.W2LAvatar(faces, frames, boxes)
    melB = np.tile(mel.numpy().reshape(2, 80, 16), (8, 1, 1))
    got = {}
    for on in (False, True):
        switch(on)
        s = engine.W2LSession(model, av, 16, keep_layers=keep_layers)
        got[on] = s.infer(0, melB)
        s.close()
    av.close()
    model.close()
    assert np.isfinite(got[True]).all()
    assert np.array_equal(got[True].view(np.uint32), got[False].view(np.uint32))
