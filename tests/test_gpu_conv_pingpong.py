"""GPU: the ping-pong 64-channel residual 3x3 conv (conv_pingpong.cu) against the halo kernel it replaces.

The planner sends a 3x3 stride-1 conv with Cin = Cout = 64 whose residual is its own input slice, on a map whose width is a
multiple of 8, with at least three 16 x 8 pixel tiles per SM, to conv_pingpong_kernel (ltb_conv_variant.kernel = 2); LTB_CONV_PINGPONG=0 keeps it on the halo kernel.
Each case runs the same op on the same inputs and weights both ways in one process and requires bit-identical outputs: the
new kernel issues its MMAs in the halo kernel's order and rounds in the halo kernel's order.  Inputs are channel slices whose
neighbours hold sentinels, outputs go into a channel slice of a wider buffer, and nothing outside it may change.

Convs without a residual, or whose residual is another tensor, stay on the halo kernel (the S3FD, BiSeNet and UltraLight plans
pin that), as do maps whose width is not a multiple of 8 and layers with fewer tiles (the wav2lip256 audio encoder)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F
from conv_cases import bits, ctx, slice_buf, weights

import conv_check as cc

pytestmark = pytest.mark.gpu

SENT_IN = 512.0
SENT_OUT = -3.25
PINGPONG = dict(kernel=2, taps=9, bn=64, nsub=1, nacc=1, resident_chunks=1, kb=0, ksplit=0, grouped=0)

# (N, H, W): 64 x 64 = L18-L20 at B = 16 (512 tiles); 72 and 150 rows overhang the 16-row tile (the output TMA store clips them)
CASES = [(16, 64, 64), (16, 72, 80), (3, 150, 152)]


@pytest.fixture
def switch(monkeypatch):
    def set_(on):
        monkeypatch.setenv("LTB_CONV_PINGPONG", "1" if on else "0")
    return set_


@pytest.mark.parametrize("relu", [True, False], ids=["relu", "no_relu"])
@pytest.mark.parametrize("shape", CASES, ids=[f"b{n}_{h}x{w}" for n, h, w in CASES])
def test_pingpong_equals_halo_kernel(ctx, switch, shape, relu):
    N, H, W = shape
    g = torch.Generator().manual_seed(N * 1000 + H + W + relu)
    x = (torch.randn(N, H, W, 64, generator=g) * 0.7 + 0.2 + torch.randn(64, generator=g) * 0.3).half()
    w, b, cw, temps = weights(ctx, g, 64, 64)
    xv, xt, xbuf = slice_buf(ctx, x.numpy(), 88, 8, SENT_IN)
    temps.append(xt)
    outs = {}
    try:
        for on in (False, True):
            switch(on)
            ov, ot, obuf = slice_buf(ctx, np.full((N, H, W, 64), np.nan, np.float16), 80, 8, SENT_OUT)
            temps.append(ot)
            geo = dict(N=N, IH=H, IW=W, OH=H, OW=W, pad=(1, 1), relu=relu, res=xv)
            variant = ctx.conv_plan(xv, cw, ov, **geo)
            if on:
                assert variant == PINGPONG, variant
            else:
                assert variant["kernel"] == 1 and ctx.conv_res_halo(xv, cw, ov, **geo), variant
            ctx.conv(xv, cw, ov, **geo)
            full = ctx.download(ot)
            outside = np.ones(obuf.shape, bool)
            outside[..., 8:72] = False
            assert np.array_equal(bits(full)[outside], bits(obuf)[outside]), f"pingpong={on}: wrote outside the output slice"
            outs[on] = full[..., 8:72]
        assert np.array_equal(bits(ctx.download(xt)), bits(xbuf)), "the conv changed its input buffer"
        assert np.isfinite(outs[True].astype(np.float32)).all(), "unwritten outputs"
        diff = bits(outs[True]) != bits(outs[False])
        assert not diff.any(), f"{int(diff.sum())} of {diff.size} outputs differ from the halo kernel, first at {np.argwhere(diff)[0]}"
        # and both against float64 on the first image, with the halo kernel's rounding order (conv_check.py)
        x64 = x[:1].double().permute(0, 3, 1, 2)
        conv = F.conv2d(F.pad(x64, (1, 1, 1, 1)), w.double()).permute(0, 2, 3, 1).numpy()
        A = F.conv2d(F.pad(x64.abs(), (1, 1, 1, 1)), w.double().abs()).permute(0, 2, 3, 1).numpy()
        cc.check(outs[True][:1], conv, A, b.numpy(), K=9 * 64, order=cc.order_of(PINGPONG), relu=relu, r=x[:1].numpy(),
                 what=f"pingpong b{N}_{H}x{W} relu={relu}")
    finally:
        for t in temps:
            ctx.free(t)


def test_wav2lip_decoder_layers_plan_pingpong(ctx, switch):
    """L51 (64-channel temporary -> temporary) and L52 (temporary -> cat7[0:64] of the 80-channel concat buffer) at B = 16 and
    256 x 256, each with its input as residual, plan the ping-pong kernel; with the switch off, the halo kernel."""
    from livetalking_b200.ops import DevTensor
    g = torch.Generator().manual_seed(51)
    _, _, cw, temps = weights(ctx, g, 64, 64)
    N, S = 16, 256
    a = ctx.alloc((N, S, S, 64))
    cat7 = ctx.alloc((N, S, S, 80))
    temps += [a, cat7]
    try:
        a_v = DevTensor(a.ptr, (N, S, S, 64))
        c_v = DevTensor(cat7.ptr, (N, S, S, 64), pitch=80, c_off=0)
        geo = dict(N=N, IH=S, IW=S, OH=S, OW=S, pad=(1, 1), relu=True, res=a_v)
        for on in (True, False):
            switch(on)
            for name, out in (("L51", a_v), ("L52", c_v)):
                v = ctx.conv_plan(a_v, cw, out, **geo)
                if on:
                    assert v == PINGPONG, (name, v)
                else:
                    assert v == dict(PINGPONG, kernel=1, nsub=2), (name, v)
        switch(True)
        # no residual, or a residual that is not the input: the halo kernel
        assert ctx.conv_plan(a_v, cw, c_v, **dict(geo, res=None))["kernel"] == 1
        assert ctx.conv_plan(a_v, cw, a_v, **dict(geo, res=c_v))["kernel"] == 1
        # a map width that is not a multiple of 8 (test_gpu_conv_res_halo's <64,2,1,9,1> row)
        x_v = DevTensor(a.ptr, (4, 128, 132, 64))
        assert ctx.conv_plan(x_v, cw, x_v, **dict(geo, N=4, IH=128, IW=132, OH=128, OW=132, res=x_v))["kernel"] == 1
    finally:
        for t in temps:
            ctx.free(t)


def test_wav2lip_forward_unchanged(w2l_state_dict, switch):
    """The whole wav2lip256 forward at B = 16 (L18-L20, L51, L52 on the ping-pong kernel) gives the same frames, byte for byte,
    as with those layers on the halo kernel."""
    from livetalking_b200 import engine
    from oracle import wav2lip_ref as R
    engine.set_device(0)
    model = engine.W2LModel.from_state_dict(w2l_state_dict)
    mel, img = R.synth_inputs(2, seed=5)
    f = (img[:, 3:6].permute(0, 2, 3, 1).numpy() * 255.0).round().astype(np.uint8)
    faces = [f[i % 2] for i in range(16)]
    frames = np.random.default_rng(3).integers(0, 256, (16, 360, 640, 3), np.uint8)
    boxes = [(20 + 3 * i, 20 + 3 * i + 200, 100 + i, 100 + i + 190) for i in range(16)]
    av = engine.W2LAvatar(faces, frames, boxes)
    melB = np.tile(mel.numpy().reshape(2, 80, 16), (8, 1, 1))
    got = {}
    for on in (False, True):
        switch(on)
        s = engine.W2LSession(model, av, 16)
        got[on] = s.infer(0, melB)
        s.close()
    av.close()
    model.close()
    assert np.array_equal(got[True], got[False])
