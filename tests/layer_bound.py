"""The float64 per-element bound of the avatar-creation layer tests (test_gpu_s3fd.py, test_gpu_pfld.py, test_gpu_bisenet.py): one
planner conv or depthwise conv on its own fp16 GPU input, with A = conv(|x|, |w|), K the accumulation chain and the constants of
conv_check.py:

    1.25 (18 ceil(K/16) 2^-23 A + (3 + min(32, K // 128)) 2^-24 (A + |b| + extra) [+ 2^-11 A if up] + 2^-11 |ref| + 2^-25)

The min(32, K // 128) term covers a split-K gather plan.  extra (residual only): |r| + 2^13 |conv + b|, the epilogue may round
conv + bias to fp16 before it adds r.  up (the fused nearest-2x convs): the summed sub-pixel weights are rounded to fp16 once."""
import torch
import torch.nn.functional as F

from conv_check import SAFETY, SUB16, U16, V32, eps_acc, ks_ceiling


def conv_bound(x, w, b, stride, pad, relu, groups=1, r=None, up=False):
    """float64 NCHW input x, weights w [cout, cin / groups, k, k], bias b [cout], residual r -> (ref, bound)."""
    if up:
        x = F.interpolate(x, scale_factor=2, mode="nearest")
    conv = F.conv2d(x, w, stride=stride, padding=pad, groups=groups)
    A = F.conv2d(x.abs(), w.abs(), stride=stride, padding=pad, groups=groups)
    bb = b[None, :, None, None]
    pre = conv + bb
    extra = torch.zeros_like(A)
    if r is not None:
        extra = r.abs() + (U16 / V32) * pre.abs()
        pre = pre + r
    ref = torch.relu(pre) if relu else pre
    K = w.shape[1] * w.shape[2] * w.shape[3]
    acc = eps_acc(K) * A + (3 + ks_ceiling(K)) * V32 * (A + bb.abs() + extra)
    if up:
        acc = acc + U16 * A
    return ref, SAFETY * (acc + U16 * ref.abs() + SUB16)
