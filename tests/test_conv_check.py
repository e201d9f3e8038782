"""CPU: the conv checker of conv_check.py against numpy emulations of right and wrong conv kernels.

Each emulation computes 8000 outputs (250 pixels x 32 channels) of a K-long fp16 dot product at the GPU conv tests' input
statistics (x ~ 0.7 N(0, 1) + 0.4 + per-channel offsets, He-scaled fp16 weights, bias ~ 0.2 N(0, 1), residual ~ 0.5 N(0, 1)):

  * correct: the k16 steps' products summed exactly and added to an fp32 accumulator (one rounding per step), then the
    epilogue of the gather order (fp32 acc + b + r, one fp16 rounding) or of the halo order (fp16(acc + b), then the fp16 add
    of the residual).  Both must pass every gate with the committed thresholds.
  * wrong: an fp16 accumulator rounded after every k16 step; activations rounded to bf16; four split-K partials stored as fp16;
    the residual added in fp32 before the one rounding where the halo order is claimed.  Each must be rejected.
  * a result that drops one input channel at 1 % of the pixels (K = 720) must be rejected by the hard bound, as the old flat
    tolerance would have.

These keep P_NEQ and R_MAX honest: loosening either until a wrong kernel passes fails here."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import conv_check as cc

KS = [64, 720, 4608]
NPIX, NOUT = 250, 32


def _problem(K, seed):
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal((NPIX, K)) * 0.7 + 0.4 + rng.standard_normal(K) * 0.3).astype(np.float16).astype(np.float64)
    w = (rng.standard_normal((K, NOUT)) * math.sqrt(2.0 / K)).astype(np.float16).astype(np.float64)
    b = (rng.standard_normal(NOUT) * 0.2).astype(np.float32).astype(np.float64)
    r = (rng.standard_normal((NPIX, NOUT)) * 0.5).astype(np.float16).astype(np.float64)
    return x, w, b, r


def _accumulate(x, w, steps=None, fp16_acc=False):
    """fp32 (or fp16) accumulator over the k16 steps in `steps` (default: all), each step's 16 products summed exactly."""
    K = x.shape[1]
    acc = np.zeros((x.shape[0], w.shape[1]), np.float64)
    for s in (range(K // 16) if steps is None else steps):
        step = x[:, 16 * s:16 * s + 16] @ w[16 * s:16 * s + 16]
        acc = cc.f16(acc + step) if fp16_acc else (acc + step).astype(np.float32).astype(np.float64)
    return acc


def _f32(a):
    return np.asarray(a, np.float64).astype(np.float32).astype(np.float64)


def _epilogue(acc, b, r, order):
    if order == "gather":
        return cc.f16(_f32(_f32(acc + b) + r))
    return cc.f16(cc.f16(_f32(acc + b)) + r)


def _emulate(K, kind, order, seed=1):
    x, w, b, r = _problem(K, seed)
    conv, A = x @ w, np.abs(x) @ np.abs(w)
    ks = 0
    if kind == "correct":
        got = _epilogue(_accumulate(x, w), b, r, order)
    elif kind == "fp16_acc":
        got = _epilogue(_accumulate(x, w, fp16_acc=True), b, r, order)
    elif kind == "bf16_act":
        xb = torch.from_numpy(x).to(torch.bfloat16).double().numpy()
        got = _epilogue(_accumulate(xb, w), b, r, order)
    elif kind == "fp16_splitk":
        ks, n = 4, K // 16
        parts = [cc.f16(_accumulate(x, w, range(i * n // ks, (i + 1) * n // ks))) for i in range(ks)]
        f = _f32(np.broadcast_to(b, parts[0].shape))
        for p in parts:
            f = _f32(f + p)
        got = cc.f16(_f32(f + r))
        order = "gather"
    elif kind == "fp32_residual":      # claims the halo order, adds the residual in fp32 before one rounding
        got = _epilogue(_accumulate(x, w), b, r, "gather")
        order = "halo"
    else:
        raise ValueError(kind)
    return got, conv, A, b, r, ks, order


@pytest.mark.parametrize("order", ["gather", "halo"])
@pytest.mark.parametrize("K", KS)
def test_correct_kernel_passes(K, order):
    got, conv, A, b, r, ks, order = _emulate(K, "correct", order)
    s = cc.check(got, conv, A, b, K=K, order=order, r=r, ks=ks, what=f"correct K={K}")
    assert s["worst"] <= 1.0 and s["neq"] <= cc.P_NEQ and s["rms"] <= cc.R_MAX


@pytest.mark.parametrize("kind", ["fp16_acc", "bf16_act", "fp16_splitk", "fp32_residual"])
@pytest.mark.parametrize("K", KS)
def test_wrong_kernel_is_rejected(K, kind):
    got, conv, A, b, r, ks, order = _emulate(K, kind, "halo")
    with pytest.raises(AssertionError):
        cc.check(got, conv, A, b, K=K, order=order, r=r, ks=ks, what=f"{kind} K={K}", negative_control=False)


def test_dropped_channel_fails_the_bound():
    K = 720
    x, w, b, r = _problem(K, 5)
    rng = np.random.default_rng(6)
    rows = rng.choice(NPIX, NPIX // 100 + 1, replace=False)
    xd = x.copy()
    xd[rows, 357] = 0.0
    got = _epilogue(_accumulate(xd, w), b, r, "gather")
    with pytest.raises(AssertionError, match="outside the bound"):
        cc.check(got, x @ w, np.abs(x) @ np.abs(w), b, K=K, order="gather", r=r, what="dropped channel")


def test_thresholds_sit_between_measured_and_rejected():
    """The committed thresholds: above what the H100 measured, and below every rate a wrong kernel reaches above."""
    assert cc.MEASURED_NEQ_MAX is not None and cc.MEASURED_RMS_MAX is not None
    assert cc.MEASURED_NEQ_MAX <= cc.P_NEQ <= 0.05
    assert cc.MEASURED_RMS_MAX <= cc.R_MAX <= 1.1


def test_model_orders_and_saturation():
    """The two rounding orders on hand-picked values, saturation included."""
    pre = np.array([1.0 + 3 * 2.0 ** -13, 70000.0, 70000.0, -70000.0, 65000.0, -0.3])
    r = np.array([3 * 2.0 ** -13, -1000.0, 0.0, 1000.0, 1000.0, 0.1])
    # gather: one rounding of the exact sum, clamped
    assert list(cc.model(pre, r, order="gather")) == [1.0 + 2.0 ** -10, 65504.0, 65504.0, -65504.0, 65504.0,
                                                     float(np.float16(-0.2))]
    # halo: fp16(pre) first (1 + 3 2^-13 rounds to 1, 70000 saturates), then the fp16 add
    assert list(cc.model(pre, r, order="halo")) == [1.0, float(np.float16(64504.0)), 65504.0, float(np.float16(-64504.0)), 65504.0,
                                                   float(np.float16(float(np.float16(-0.3)) + 0.1))]
    assert list(cc.model(pre, r, relu=True, order="halo"))[3] == 0.0
    assert cc.ulp16(np.array([0.0, 1.0, 65504.0, 2.0 ** -20]))[[0, 1, 2, 3]].tolist() == [2.0 ** -24, 2.0 ** -10, 32.0, 2.0 ** -24]


def test_upsample_presummed_is_the_upsampled_conv():
    """The fused upsample's model differs from conv3x3(nearest 2x) only by the fp16 rounding of the pre-summed weights."""
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 16, 5, 7, generator=g, dtype=torch.float64)
    w = (torch.randn(8, 16, 3, 3, generator=g) * 0.1).half().float().numpy()
    got = cc.upsample_presummed(x, w)
    want = F.conv2d(F.interpolate(x, scale_factor=2, mode="nearest"), torch.from_numpy(w).double(), padding=1)
    A = F.conv2d(F.interpolate(x.abs(), scale_factor=2, mode="nearest"), torch.from_numpy(np.abs(w)).double(), padding=1)
    assert ((got - want).abs() <= cc.U16 * A + 1e-12).all()
    assert (got - want).abs().max() > 0
