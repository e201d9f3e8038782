"""GPU: the wgmma implicit-GEMM conv kernels against a float64 PyTorch reference of the same op, called through the C ABI
(ltb_conv2d_f16).  Every output is held to conv_check.py: the hard error bound and the rounding model of the kernel that ran
(the gather kernel rounds acc + b + r once; the halo kernel rounds fp16(acc + b) and then adds the residual in fp16).  Which
kernel the automatic path takes is read from the planner (Ctx.conv_plan on the same geometry).  The test names keep their
`torch_fp32` suffix from when the reference was fp32 PyTorch, so that their ids stay stable."""
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from conv_cases import ctx  # noqa: F401  (fixture)

import conv_check as cc

pytestmark = pytest.mark.gpu

CASES = [
    # N, H, W, Cin, Cout, k, (sy,sx), pad, transposed, res
    (2, 16, 16, 64, 64, 3, (1, 1), 1, False, True),      # halo BN=32, residual
    (1, 12, 10, 32, 32, 3, (1, 1), 1, False, True),      # halo BN=32, overhanging tile (120 pixels)
    (2, 20, 20, 16, 32, 3, (2, 2), 1, False, False),     # KB=16, stride 2
    (1, 12, 10, 128, 256, 3, (2, 2), 1, False, False),   # stride 2, 8 N tiles of 32
    (3, 80, 16, 32, 64, 3, (3, 1), 1, False, False),     # audio encoder stride (3,1)
    (3, 27, 16, 64, 128, 3, (3, 3), 1, False, False),    # audio encoder stride 3
    (3, 9, 6, 128, 256, 3, (3, 2), 1, False, False),     # audio encoder stride (3,2)
    (16, 1, 1, 512, 512, 1, (1, 1), 0, False, False),    # 1x1 on the bottleneck (M = 16)
    (4, 4, 4, 512, 512, 4, (1, 1), 0, False, False),     # 4x4 valid conv -> 1x1 (16 taps)
    (4, 3, 3, 256, 512, 3, (1, 1), 0, False, False),     # 3x3 valid conv -> 1x1
    (1, 5, 7, 64, 32, 3, (2, 2), 1, True, False),        # ConvT phases, ragged
    (2, 8, 8, 160, 64, 3, (2, 2), 1, True, False),       # ConvT KB=32
    (2, 4, 4, 1024, 512, 3, (2, 2), 1, True, False),     # ConvT deep K
    (1, 16, 16, 384, 384, 3, (1, 1), 1, False, True),    # 12 N tiles of 32
    (1, 24, 24, 80, 32, 3, (1, 1), 1, False, False),     # head conv: halo BN=32, ragged second K chunk
    (1, 64, 64, 64, 64, 3, (1, 1), 1, False, True),      # many M tiles
    (1, 32, 32, 320, 128, 3, (2, 2), 1, True, False),    # ConvT 320 -> 128
    (8, 8, 8, 512, 512, 3, (1, 1), 1, False, True),      # M = 512, 8 K chunks: halo BN=32 over overhanging tiles, residual
    (8, 4, 4, 1280, 640, 3, (1, 1), 1, False, False),    # split-K: M = 128, 180 K blocks
    (2, 8, 8, 256, 512, 3, (2, 2), 1, False, False),     # split-K with stride 2 (M = 32)
    (16, 16, 16, 768, 384, 3, (2, 2), 1, True, False),   # ConvT with 384 outputs: six 64-wide N tiles, fat-N issue up to N = 192
    (16, 32, 32, 384, 384, 3, (1, 1), 1, False, True),   # 384 channels @32x32, batch 16: the cost model picks BN=128, NSUB=1 (3 waves)
    # stride-2 parity-plane TMA path (conv_halo.cu TAPS = 10): four planes loaded with traversal stride 2, nine taps as views
    (2, 64, 64, 80, 32, 3, (2, 2), 1, False, False),     # BN = 32, ragged second K chunk (80 channels)
    (2, 32, 48, 64, 128, 3, (2, 2), 1, False, False),    # 2 N tiles of 64, non-square, output 16 x 24
    (1, 64, 32, 128, 256, 3, (2, 2), 1, False, False),   # 2 K chunks, 4 N tiles
    (3, 40, 36, 64, 64, 3, (2, 2), 1, False, False),     # ragged output 20 x 18: overhanging tile rows / columns
    # narrow 3x3 layers on the halo kernel: streamed and resident weights, ragged chunks, overhanging tiles
    (2, 64, 64, 64, 64, 3, (1, 1), 1, False, True),      # BN=32: residual, streamed weights
    (5, 256, 64, 64, 64, 3, (1, 1), 1, False, True),     # enough tiles for the weights-resident variant (BN=64, NSUB=2)
    (1, 96, 40, 80, 32, 3, (1, 1), 1, False, False),     # BN=32: 80 -> 32 (ragged second K chunk)
    (3, 128, 128, 32, 32, 3, (1, 1), 1, False, True),    # 32 -> 32 + residual @128: BN=32, NSUB=2, streamed (192 tiles)
    (2, 50, 21, 64, 64, 3, (1, 1), 1, False, False),     # ragged height and width: masked last row tile / column tile
    (4, 256, 256, 80, 32, 3, (1, 1), 1, False, False),   # the output conv's geometry (2 chunks resident)
]


def _reference(x, w, stride, pad, transposed):
    """float64 NHWC conv (no bias) and conv of the absolute values.  x: fp16 NCHW; w: fp16-rounded PyTorch-layout weights."""
    x64, w64 = x.double(), w.half().double()
    if transposed:
        f = lambda a, b: F.conv_transpose2d(a, b, stride=2, padding=1, output_padding=1)
    else:
        f = lambda a, b: F.conv2d(a, b, stride=stride, padding=pad)
    return f(x64, w64).permute(0, 2, 3, 1).numpy(), f(x64.abs(), w64.abs()).permute(0, 2, 3, 1).numpy()


def _chain(Cin, k, transposed):
    return 4 * Cin if transposed else Cin * k * k


def _planned(ctx, N, H, W, Cin, Cout, k, s, pad, transposed, res):
    """The variant ltb_op_conv2d plans for this dense geometry: ltb_conv2d_f16 plans through the same conv_plan."""
    OH, OW = (2 * H, 2 * W) if transposed else ((H + 2 * pad - k) // s[0] + 1, (W + 2 * pad - k) // s[1] + 1)
    x, o = ctx.alloc((N, H, W, Cin)), ctx.alloc((N, OH, OW, Cout))
    r = ctx.alloc((N, OH, OW, Cout)) if res else None
    wt, bt = ctx.alloc((Cout, 9 * Cin if transposed else k * k * Cin)), ctx.alloc((Cout,), np.float32)
    wtap = ctx.alloc((9, Cout, Cin)) if k == 3 else None
    cw = types.SimpleNamespace(cout=Cout, cin=Cin, kh=k, kw=k, ktot=9 * Cin if transposed else k * k * Cin, w=wt, w_tap=wtap, bias=bt)
    try:
        return ctx.conv_plan(x, cw, o, N=N, IH=H, IW=W, OH=OH, OW=OW, stride=s, pad=(pad, pad), res=r, relu=True,
                             transposed=transposed)
    finally:
        for t in (x, o, r, wt, bt, wtap):
            if t is not None:
                ctx.free(t)


@pytest.mark.parametrize("case", CASES, ids=[f"c{i}" for i in range(len(CASES))])
def test_conv_matches_torch_fp32(ctx, case):
    from livetalking_b200 import engine
    engine.set_device(0)
    N, H, W, Cin, Cout, k, s, pad, transposed, res = case
    g = torch.Generator().manual_seed(hash(case) % (2 ** 31))
    x = (torch.randn(N, Cin, H, W, generator=g) * 0.7).half()
    fan = Cin * k * k
    if transposed:
        w = torch.randn(Cin, Cout, k, k, generator=g) * (2.0 / (fan / 4)) ** 0.5
    else:
        w = torch.randn(Cout, Cin, k, k, generator=g) * (2.0 / fan) ** 0.5
    b = torch.randn(Cout, generator=g) * 0.2
    conv, A = _reference(x, w, s, pad, transposed)
    r = (torch.randn(conv.shape, generator=g) * 0.5).half() if res else None    # NHWC
    out = engine.conv2d_f16(x.permute(0, 2, 3, 1).contiguous().numpy(), w.numpy(), b.numpy(), stride=s, pad=pad,
                            transposed=transposed, relu=True, res=None if r is None else r.numpy())
    assert out.shape == conv.shape
    v = _planned(ctx, N, H, W, Cin, Cout, k, s, pad, transposed, res)
    K = _chain(Cin, k, transposed)
    ks = cc.ks_ceiling(K) if v["kernel"] == 0 else 0      # the C ABI's split-K workspace differs from the context's
    cc.check(out, conv, A, b.numpy(), K=K, order=cc.order_of(v), relu=True, r=None if r is None else r.numpy(), ks=ks,
             what=f"c{CASES.index(case)} (planned {v})")


def test_conv_no_relu_negative_outputs():
    from livetalking_b200 import engine
    engine.set_device(0)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(1, 64, 8, 8, generator=g).half()
    w = torch.randn(32, 64, 3, 3, generator=g) * 0.05
    b = torch.randn(32, generator=g)
    conv, A = _reference(x, w, (1, 1), 1, False)
    out = engine.conv2d_f16(x.permute(0, 2, 3, 1).contiguous().numpy(), w.numpy(), b.numpy(), pad=1, relu=False)
    assert ((conv + b.numpy()) < 0).any()
    # no residual: both kernels' epilogues are one rounding of acc + b
    cc.check(out, conv, A, b.numpy(), K=576, order="gather", relu=False, ks=cc.ks_ceiling(576), what="no relu")


# ---- halo-resident TMA kernel (conv_halo.cu): 3x3 s1 p1 convs and k3 s2 ConvT with H % 16 == 0, W % 8 == 0
HALO_CASES = [
    # N, H, W, Cin, Cout, transposed, res
    (1, 16, 16, 64, 64, False, True),       # NSUB=1
    (1, 64, 64, 64, 64, False, True),       # NSUB=1, BN=32
    (2, 32, 32, 128, 128, False, True),     # 2 chunks
    (1, 32, 16, 256, 384, False, False),    # 12 N tiles, 4 chunks
    (1, 32, 32, 80, 32, False, False),      # Cin=80: second chunk zero-filled beyond channel 80
    (2, 32, 8, 32, 32, False, True),        # Cin=32: half a chunk
    (16, 16, 16, 512, 512, False, True),    # deep K, BN=128: 128 tiles
    (3, 48, 24, 64, 128, False, False),     # non power-of-two tiling
    (1, 16, 16, 64, 64, True, False),       # ConvT, 4 accumulators
    (2, 32, 32, 160, 64, True, False),      # ConvT Cin=160 (2.5 chunks)
    (1, 16, 8, 128, 32, True, False),       # ConvT BN=32
    (1, 32, 32, 320, 128, True, False),     # ConvT 320->128
    (1, 128, 128, 64, 64, False, True),     # BN=64, NSUB=1: 128 tiles
    (16, 8, 8, 512, 512, False, True),      # map smaller than a tile: overhanging rows masked (w2l L28/L37)
    (16, 4, 4, 512, 512, False, True),      # 4x4 map: rows and columns masked (w2l L30/L35)
    (4, 4, 4, 1024, 512, True, False),      # ConvT 4x4 -> 8x8 (w2l L36)
    (2, 8, 8, 1024, 512, True, False),      # ConvT 8x8 -> 16x16 (w2l L38)
    (2, 27, 16, 64, 64, False, True),       # odd height (audio encoder 27x16)
    (3, 9, 6, 128, 128, False, True),       # odd height and width
    (2, 20, 12, 64, 32, True, False),       # ConvT over an odd-sized map
    (3, 64, 64, 544, 128, True, False),     # ConvT, 128 outputs in two BN=64 tiles, ragged last K chunk
    (3, 64, 32, 512, 256, True, False),     # ConvT BN=64, four N tiles
]


@pytest.mark.parametrize("case", HALO_CASES, ids=[f"h{i}" for i in range(len(HALO_CASES))])
def test_halo_kernel_matches_torch_fp32(case):
    from livetalking_b200 import engine
    engine.set_device(0)
    N, H, W, Cin, Cout, transposed, res = case
    g = torch.Generator().manual_seed(1234 + hash(case) % 1000)
    x = (torch.randn(N, Cin, H, W, generator=g) * 0.7).half()
    if transposed:
        w = torch.randn(Cin, Cout, 3, 3, generator=g) * (2.0 / (Cin * 9 / 4)) ** 0.5
    else:
        w = torch.randn(Cout, Cin, 3, 3, generator=g) * (2.0 / (Cin * 9)) ** 0.5
    b = torch.randn(Cout, generator=g) * 0.2
    conv, A = _reference(x, w, (1, 1), 1, transposed)
    r = (torch.randn(conv.shape, generator=g) * 0.5).half().numpy() if res else None
    xn = x.permute(0, 2, 3, 1).contiguous().numpy()
    K = _chain(Cin, 3, transposed)
    what = f"h{HALO_CASES.index(case)}"
    out = engine.conv2d_f16(xn, w.numpy(), b.numpy(), stride=(1, 1), pad=1, transposed=transposed, relu=True, res=r, force_path=2)
    cc.check(out, conv, A, b.numpy(), K=K, order="halo", relu=True, r=r, what=f"{what} halo")
    # the gather kernel on the same op, held to its own rounding order
    out_g = engine.conv2d_f16(xn, w.numpy(), b.numpy(), stride=(1, 1), pad=1, transposed=transposed, relu=True, res=r, force_path=1)
    cc.check(out_g, conv, A, b.numpy(), K=K, order="gather", relu=True, r=r, ks=cc.ks_ceiling(K), what=f"{what} gather")


# ---- TMA GEMM mode of the halo kernel (1x1 convs / linears with M >= 512)
GEMM_CASES = [
    # N, H, W, Cin, Cout, res
    (1, 32, 32, 320, 2560, False),      # FF1 of the 32x32 transformer block (5 K chunks, 20 N tiles)
    (1, 64, 128, 64, 128, True),        # 8192 rows, residual
    (1, 25, 40, 96, 64, False),         # ragged M = 1000, partial K chunk (96 = 64 + 32)
    (2, 16, 16, 1280, 320, True),       # FF2-like: deep K
    (1, 32, 32, 384, 96, False),        # Cout = 96 -> BN 32
]


@pytest.mark.parametrize("case", GEMM_CASES, ids=[f"g{i}" for i in range(len(GEMM_CASES))])
def test_tma_gemm_mode_matches_torch_fp32(case):
    from livetalking_b200 import engine
    engine.set_device(0)
    N, H, W, Cin, Cout, res = case
    g = torch.Generator().manual_seed(77 + Cin + Cout)
    x = (torch.randn(N, Cin, H, W, generator=g) * 0.7).half()
    w = torch.randn(Cout, Cin, 1, 1, generator=g) * (1.0 / Cin) ** 0.5
    b = torch.randn(Cout, generator=g) * 0.2
    conv, A = _reference(x, w, (1, 1), 0, False)
    r = (torch.randn(conv.shape, generator=g) * 0.5).half().numpy() if res else None
    xn = x.permute(0, 2, 3, 1).contiguous().numpy()
    what = f"g{GEMM_CASES.index(case)}"
    out = engine.conv2d_f16(xn, w.numpy(), b.numpy(), relu=False, res=r, force_path=2)
    cc.check(out, conv, A, b.numpy(), K=Cin, order="halo", r=r, what=f"{what} halo gemm")
    out_g = engine.conv2d_f16(xn, w.numpy(), b.numpy(), relu=False, res=r, force_path=1)
    cc.check(out_g, conv, A, b.numpy(), K=Cin, order="gather", r=r, ks=cc.ks_ceiling(Cin), what=f"{what} gather")
