"""GPU: the wgmma implicit-GEMM conv kernels against a plain PyTorch fp32 reference of the same op,
called through the C ABI (ltb_conv2d_f16).  Tolerance: fp16 in/out, fp32 accumulate -> |err| <= 2e-2 + 1e-2*|ref|."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

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


@pytest.mark.parametrize("case", CASES, ids=[f"c{i}" for i in range(len(CASES))])
def test_conv_matches_torch_fp32(case):
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
    wq = w.half().float()
    if transposed:
        ref = F.conv_transpose2d(x.float(), wq, b, stride=2, padding=1, output_padding=1)
    else:
        ref = F.conv2d(x.float(), wq, b, stride=s, padding=pad)
    r = None
    if res:
        r = (torch.randn(ref.shape, generator=g) * 0.5).half()
        ref = ref + r.float()
    ref = F.relu(ref).permute(0, 2, 3, 1).contiguous().numpy()
    out = engine.conv2d_f16(x.permute(0, 2, 3, 1).contiguous().numpy(), w.numpy(), b.numpy(), stride=s, pad=pad,
                            transposed=transposed, relu=True,
                            res=None if r is None else r.permute(0, 2, 3, 1).contiguous().numpy())
    assert out.shape == ref.shape
    out = out.astype(np.float32)
    assert np.isfinite(out).all(), "unwritten / non-finite outputs"
    err = np.abs(out - ref)
    tol = 2e-2 + 1e-2 * np.abs(ref)
    assert (err <= tol).all(), f"max err {err.max():.4f} at {np.unravel_index(err.argmax(), err.shape)}; mean {err.mean():.5f}"
    assert err.mean() < 2e-3


def test_conv_no_relu_negative_outputs():
    from livetalking_b200 import engine
    engine.set_device(0)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(1, 64, 8, 8, generator=g).half()
    w = torch.randn(32, 64, 3, 3, generator=g) * 0.05
    b = torch.randn(32, generator=g)
    ref = F.conv2d(x.float(), w.half().float(), b, padding=1).permute(0, 2, 3, 1).numpy()
    out = engine.conv2d_f16(x.permute(0, 2, 3, 1).contiguous().numpy(), w.numpy(), b.numpy(), pad=1, relu=False).astype(np.float32)
    assert (ref < 0).any()
    assert np.abs(out - ref).max() < 2e-2


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
    wq = w.half().float()
    if transposed:
        ref = F.conv_transpose2d(x.float(), wq, b, stride=2, padding=1, output_padding=1)
    else:
        ref = F.conv2d(x.float(), wq, b, padding=1)
    r = None
    if res:
        r = (torch.randn(ref.shape, generator=g) * 0.5).half()
        ref = ref + r.float()
    ref = F.relu(ref).permute(0, 2, 3, 1).contiguous().numpy()
    xn = x.permute(0, 2, 3, 1).contiguous().numpy()
    rn = None if r is None else r.permute(0, 2, 3, 1).contiguous().numpy()
    out = engine.conv2d_f16(xn, w.numpy(), b.numpy(), stride=(1, 1), pad=1, transposed=transposed, relu=True, res=rn,
                            force_path=2).astype(np.float32)
    assert np.isfinite(out).all(), "unwritten / non-finite outputs"
    err = np.abs(out - ref)
    tol = 2e-2 + 1e-2 * np.abs(ref)
    assert (err <= tol).all(), f"max err {err.max():.4f} at {np.unravel_index(err.argmax(), err.shape)}; mean {err.mean():.5f}"
    # both tensor-core paths accumulate the same K order in fp32: they must agree to the last fp16 bit almost everywhere
    out_g = engine.conv2d_f16(xn, w.numpy(), b.numpy(), stride=(1, 1), pad=1, transposed=transposed, relu=True, res=rn,
                              force_path=1).astype(np.float32)
    assert np.abs(out - out_g).max() <= 2e-2


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
    ref = F.conv2d(x.float(), w.half().float(), b)
    r = None
    if res:
        r = (torch.randn(ref.shape, generator=g) * 0.5).half()
        ref = ref + r.float()
    ref = ref.permute(0, 2, 3, 1).contiguous().numpy()
    xn = x.permute(0, 2, 3, 1).contiguous().numpy()
    rn = None if r is None else r.permute(0, 2, 3, 1).contiguous().numpy()
    out = engine.conv2d_f16(xn, w.numpy(), b.numpy(), relu=False, res=rn, force_path=2).astype(np.float32)
    assert np.isfinite(out).all()
    err = np.abs(out - ref)
    assert (err <= 2e-2 + 1e-2 * np.abs(ref)).all(), f"max err {err.max():.4f} at {np.unravel_index(err.argmax(), err.shape)}"
    out_g = engine.conv2d_f16(xn, w.numpy(), b.numpy(), relu=False, res=rn, force_path=1).astype(np.float32)
    assert np.abs(out - out_g).max() <= 2e-2

