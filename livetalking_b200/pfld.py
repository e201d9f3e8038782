"""PFLD_GhostOne landmark network on the device: the landmark step of the UltraLight avatar generator (avatars/ultralight/genavatar.py
-> face_detect_utils/get_landmark.py Landmark.detect -> pfld_mobileone.PFLD_GhostOne(0.5, 192, 110)), as one captured CUDA graph
per batch size.

    net = PFLDNet.from_state_dict(torch.load("checkpoint_epoch_335.pth.tar"), mean_face)   # train-time or re-parameterised keys
    lm = PFLDLandmarker(net, 16)
    lm.run(crops_192_bgr_u8, crop_wh)      # -> (float32 [n,110,2] pixel landmarks, int32 [n,110,2] = Landmark.detect's result)

Weights.  Every MobileOneBlock is folded on the host in float64 by the reference's own reparameterize arithmetic (BN-fold each of
the six conv branches, the 1x1 scale branch padded to k x k, an identity kernel for the skip BatchNorm) and cast once to fp16;
biases stay fp32 (the epilogues add them in fp32).  conv8 (a 12 x 12 valid conv on the 12 x 12 map, no BN) is a 1x1 conv with
Cin = 12 * 12 * 16 = 2304 over the NHWC-flattened map: its weight is reordered to (ky, kx, c) on the host.

Graph: pfld_prep (u8 BGR -> fp16 v / 255, 16 channels) -> conv1 (3x3 s2) on the conv planner -> conv2 depthwise (dwconv3x3) ->
per GhostOneModule the primary 1x1 on the planner into channels [0, half_p) of its output and the cheap depthwise 3x3 into
[half_p, 2 half_p) (torch.cat costs nothing), the stride-2 depthwise of the down-sampling bottlenecks on dwconv3x3(stride 2) ->
conv7 (3x3) and conv8 on the planner -> pfld_head (one CTA per image: the four AvgPool2d taps and conv8's output, conv_out in fp32,
+ mean_face, times the crop width / height, truncation).

Channel padding.  The planner's kernels need Cin % 16 == 0 and Cout % 16 == 0 (conv_gather_pick: the halo kernel needs more, so
every conv here may fall back to the gather kernel) and 8-aligned pitches and channel offsets; dwconv3x3 needs C, pitches and
offsets % 8 == 0.  At width 0.5 the GhostOneModule halves are 20, 24, 30, 36, 50, 54, 60, 84, 126 and 4 channels, so each half is
stored padded to a multiple of 16 (half_p), which satisfies both.  The padded channels hold exact zeros: their weights and biases are
zero, so ReLU or not, they compute 0.  The consumers' weights are zero at the padded input positions, and pfld_head reads each tap's
real channels only.

fp16 range.  Weights are checked to stay below 2^14 after folding (a 4x margin to the fp16 range); activations are stored in fp16
with fp32 accumulation and the epilogues saturate.  The published checkpoint has not been run here; the tests assert the largest
activation of every layer on their synthetic weights."""
from __future__ import annotations

import math
from typing import List, Optional, Tuple

import numpy as np

from .graph import _ceil16
from .layerplan import Layer, LayerSession, Step, _f64, fp16_weights
from .ops import Ctx

INPUT, LANDMARKS, IN_C = 192, 110, 16
BRANCHES, BN_EPS = 6, 1e-5
# GhostOneBottleneck(in, hidden, out, stride) of PFLD_GhostOne at width_factor 0.5 (pfld_mobileone.py:59-72)
BOTTLENECKS = [("conv3_1", 32, 48, 40, 2), ("conv3_2", 40, 60, 40, 1), ("conv3_3", 40, 60, 40, 1),
               ("conv4_1", 40, 100, 48, 2), ("conv4_2", 48, 120, 48, 1), ("conv4_3", 48, 120, 48, 1),
               ("conv5_1", 48, 168, 72, 2), ("conv5_2", 72, 252, 72, 1), ("conv5_3", 72, 252, 72, 1), ("conv5_4", 72, 252, 72, 1),
               ("conv6", 72, 108, 8, 1)]
TAPS = ("conv2", "conv3_3", "conv4_3", "conv5_4")           # x1..x4; x5 is conv8


def gflop_per_frame() -> float:
    """2 x the multiply-accumulates of the reference's convs (unpadded), conv8 and conv_out for one 192 x 192 crop."""
    mac, h = 0, INPUT
    for _, cin, cout, k, s, g, _ in _blocks():
        h = (h + 2 * (k // 2) - k) // s + 1
        mac += h * h * cout * (cin // g) * k * k
    return 2.0 * (mac + 64 * 16 * 144 + 220 * 256) / 1e9


def _blocks():
    """Every MobileOneBlock in forward order: (prefix, cin, cout, kernel, stride, groups, relu)."""
    def ghost(p, cin, cout, relu):
        h = math.ceil(cout / 2)
        return [(p + ".primary_conv", cin, h, 1, 1, 1, relu), (p + ".cheap_operation", h, h, 3, 1, h, relu)]
    out = [("conv1", 3, 32, 3, 2, 1, True), ("conv2", 32, 32, 3, 1, 32, True)]
    for name, cin, hid, cout, s in BOTTLENECKS:
        out += ghost(name + ".ghost_conv.0", cin, hid, True)
        if s == 2:
            out.append((name + ".ghost_conv.1", hid, hid, 3, 2, hid, False))
        out += ghost(name + ".ghost_conv.2", hid, cout, False)
    out.append(("conv7", 8, 16, 3, 1, 1, True))
    return out


def fold_block(sd, p: str, cin: int, cout: int, k: int, groups: int) -> Tuple[np.ndarray, np.ndarray]:
    """MobileOneBlock._get_kernel_bias in float64 (or p.reparam_conv as stored) -> (kernel [cout, cin/groups, k, k], bias [cout])."""
    if p + ".reparam_conv.weight" in sd:
        return _f64(sd[p + ".reparam_conv.weight"]), _f64(sd[p + ".reparam_conv.bias"])

    def fuse(kernel, bn):
        std = np.sqrt(_f64(sd[bn + ".running_var"]) + BN_EPS)
        g = _f64(sd[bn + ".weight"])
        return kernel * (g / std).reshape(-1, 1, 1, 1), _f64(sd[bn + ".bias"]) - _f64(sd[bn + ".running_mean"]) * g / std

    kern = np.zeros((cout, cin // groups, k, k))
    bias = np.zeros(cout)
    if k > 1:
        ks, bs = fuse(_f64(sd[p + ".rbr_scale.conv.weight"]), p + ".rbr_scale.bn")
        kern, bias = kern + np.pad(ks, ((0, 0), (0, 0), (k // 2, k // 2), (k // 2, k // 2))), bias + bs
    if p + ".rbr_skip.weight" in sd:
        idk = np.zeros((cin, cin // groups, k, k))
        for i in range(cin):
            idk[i, i % (cin // groups), k // 2, k // 2] = 1
        ki, bi = fuse(idk, p + ".rbr_skip")
        kern, bias = kern + ki, bias + bi
    for i in range(BRANCHES):
        kc, bc = fuse(_f64(sd[f"{p}.rbr_conv.{i}.conv.weight"]), f"{p}.rbr_conv.{i}.bn")
        kern, bias = kern + kc, bias + bc
    return kern, bias


def plan(sd) -> Tuple[List[Layer], dict, list]:
    """Host-side plan from a PFLD_GhostOne state dict: (layers, buffers {name: (H, W, pitch)}, taps [(buffer, real channel list)] x 5).
    Buffer 'in' is the prepared crop [192, 192, 16], 'c7' conv7's output [12, 12, 16] which conv8 reads as [1, 1, 2304]."""
    sd = sd["pfld_backbone"] if "pfld_backbone" in sd else sd
    blocks = {b[0]: b for b in _blocks()}
    bufs = {"in": (INPUT, INPUT, IN_C)}
    layers: List[Layer] = []

    def dense(name, src, src_idx, dst, relu):
        _, cin, cout, k, s, g, _ = blocks[name]
        w16, b32 = fp16_weights(f"PFLD {name}", *fold_block(sd, name, cin, cout, k, g))
        cin_p, cout_p = bufs[src][2], _ceil16(cout)
        w, b = np.zeros((cout_p, cin_p, k, k), np.float32), np.zeros(cout_p, np.float32)
        w[:cout, src_idx], b[:cout] = w16, b32
        layers.append(Layer(name, "conv", w, b, s, k // 2, relu, (src, 0, cin_p), (dst, 0, cout_p)))
        return list(range(cout))

    def depthwise(name, buf, c_in, c_out, idx, C, relu):
        _, cin, cout, k, s, g, _ = blocks[name]
        w16, b32 = fp16_weights(f"PFLD {name}", *fold_block(sd, name, cin, cout, k, g))
        w, b = np.zeros((C, 1, 3, 3), np.float32), np.zeros(C, np.float32)
        w[idx], b[idx] = w16, b32
        layers.append(Layer(name, "dw", w, b, s, 1, relu, (buf[0], c_in, C), (buf[1], c_out, C)))

    H = INPUT // 2
    bufs["c1"] = (H, H, 32)
    dense("conv1", "in", slice(0, 3), "c1", True)
    bufs["x1"] = (H, H, 32)
    depthwise("conv2", ("c1", "x1"), 0, 0, list(range(32)), 32, True)
    cur, cur_idx = "x1", list(range(32))
    taps = [("x1", cur_idx)]

    def ghost(p, src, src_idx, cout, H, relu):
        h = math.ceil(cout / 2)
        hp = _ceil16(h)
        bufs[p] = (H, H, 2 * hp)
        assert len(src_idx) == blocks[p + ".primary_conv"][1], p
        dense(p + ".primary_conv", src, src_idx, p, relu)
        depthwise(p + ".cheap_operation", (p, p), 0, hp, list(range(h)), hp, relu)
        return p, list(range(h)) + list(range(hp, hp + h))

    for name, cin, hid, cout, s in BOTTLENECKS:
        g0, g0_idx = ghost(name + ".ghost_conv.0", cur, cur_idx, hid, H, True)
        if s == 2:
            H //= 2
            dwn = name + ".ghost_conv.1"
            C = bufs[g0][2]
            bufs[dwn] = (H, H, C)
            depthwise(dwn, (g0, dwn), 0, 0, g0_idx, C, False)
            g0 = dwn
        cur, cur_idx = ghost(name + ".ghost_conv.2", g0, g0_idx, cout, H, False)
        if name in TAPS:
            taps.append((cur, cur_idx))
    bufs["c7"] = (H, H, 16)
    dense("conv7", cur, cur_idx, "c7", True)
    # conv8: weight (64, 16, 12, 12) -> (64, 12 * 12 * 16) in the (ky, kx, c) order of the NHWC-flattened map
    w8 = _f64(sd["conv8.0.weight"])
    k8 = w8.shape[-1]
    assert w8.shape == (64, 16, H, H) and k8 == H, w8.shape
    bufs["x5"] = (1, 1, 64)
    w8, b8 = fp16_weights("PFLD conv8", w8.transpose(0, 2, 3, 1).reshape(64, -1, 1, 1), np.zeros(64))
    layers.append(Layer("conv8", "conv", w8, b8, 1, 0, True, ("c7", 0, H * H * 16), ("x5", 0, 64)))
    taps.append(("x5", list(range(64))))
    return layers, bufs, taps


class PFLDNet:
    """Device-resident PFLD_GhostOne: the plan's conv / depthwise weights, conv_out (fp32, transposed [256][220]) and mean_face."""

    def __init__(self, ctx: Ctx, layers, bufs, taps, wt, bias, mean):
        self.ctx, self.layers, self.bufs, self.taps, self.wt, self.bias, self.mean = ctx, layers, bufs, taps, wt, bias, mean

    @classmethod
    def from_state_dict(cls, sd, mean_face: np.ndarray, ctx: Optional[Ctx] = None) -> "PFLDNet":
        """sd: checkpoint['pfld_backbone'] (or the checkpoint itself) of PFLD_GhostOne, train-time or re-parameterised keys;
        mean_face: the 220 floats of mean_face.txt."""
        sd = sd["pfld_backbone"] if "pfld_backbone" in sd else sd
        layers, bufs, taps = plan(sd)
        mean = np.asarray(mean_face, np.float32).reshape(-1)
        wo = _f64(sd["conv_out.weight"]).reshape(2 * LANDMARKS, -1)
        if mean.shape != (2 * LANDMARKS,) or wo.shape[1] != sum(len(c) for _, c in taps):
            raise ValueError(f"PFLD: mean_face {mean.shape} / conv_out {wo.shape} do not match 110 landmarks over 256 features")
        ctx = ctx or Ctx()
        for L in layers:
            L.upload(ctx)
        wt = ctx.upload(np.ascontiguousarray(wo.T).astype(np.float32))
        bias = ctx.upload(_f64(sd["conv_out.bias"]).astype(np.float32))
        net = cls(ctx, layers, bufs, taps, wt, bias, ctx.upload(mean))
        ctx.sync()
        return net


class PFLDLandmarker(LayerSession):
    """One captured graph for batches of N crops of 192 x 192.  Every layer writes its own buffer (the layer tests read them)."""

    def __init__(self, net: PFLDNet, N: int, ctx: Optional[Ctx] = None):
        self.net, N = net, int(N)
        bufs = {"crops": ((N, INPUT, INPUT, 3), np.uint8), "crop_wh": ((N, 2), np.int32),
                **{name: ((N,) + hwc, np.float16) for name, hwc in net.bufs.items()},
                "out_f": ((N, 2 * LANDMARKS), np.float32), "out_i": ((N, 2 * LANDMARKS), np.int32)}
        taps, chans = [name for name, _ in net.taps], [c for _, c in net.taps]
        steps = [Step("prep", src=("crops", 0, 3), dst=("in", 0, IN_C), run=lambda s, x, y: s.ctx.pfld_prep(x, s.N, INPUT, INPUT, y)),
                 *[Step(L.name, L) for L in net.layers],
                 Step("head", run=lambda s, x, y: s.ctx.pfld_head([s.buf[t] for t in taps], chans, s.N, net.wt, net.bias, net.mean,
                                                                  s.buf["crop_wh"], s.buf["out_f"], s.buf["out_i"]))]
        super().__init__(N, bufs, steps, ctx, zero=True)

    def run(self, crops_u8: np.ndarray, crop_wh) -> Tuple[np.ndarray, np.ndarray]:
        """crops u8 BGR [n <= N, 192, 192, 3] (cv2.resize of the face crops), crop_wh [n, 2] = the crops' width and height before the
        resize -> (float32 [n, 110, 2] scaled landmarks, int32 [n, 110, 2] their truncation: Landmark.detect's pre_landmark)."""
        crops_u8 = np.ascontiguousarray(crops_u8, np.uint8)
        wh = np.ascontiguousarray(crop_wh, np.int32).reshape(-1, 2)
        n = crops_u8.shape[0]
        if crops_u8.shape[1:] != (INPUT, INPUT, 3) or not 1 <= n <= self.N or wh.shape[0] != n:
            raise ValueError(f"expected up to {self.N} crops of 192x192x3 and their sizes, got {crops_u8.shape} / {wh.shape}")
        of, oi = self.replay({"crops": crops_u8, "crop_wh": wh}, ("out_f", "out_i"))
        return of.reshape(n, LANDMARKS, 2), oi.reshape(n, LANDMARKS, 2)
