"""BiSeNet face parser on the device: the mask step of the MuseTalk avatar generator (avatars/musetalk/utils/face_parsing
FaceParsing -> model.BiSeNet(n_classes=19) over ResNet-18), as one captured CUDA graph per batch size.

    net = BiSeNetNet.from_state_dict(torch.load("79999_iter.pth"))
    parser = BiSeNetParser(net, 16)
    labels = parser.parse(rgb512_u8)        # u8 [n, 512, 512] = FaceParsing's out.argmax(0) per crop

Weights.  Every conv's BatchNorm is folded on the host in float64 and the result cast once to fp16; biases stay fp32 (the conv
epilogues add them in fp32).  The 7x7 stride-2 stem is rearranged in float64 to a 4x4 valid conv over the space-to-depth input
that bisenet_prep writes (s2d_stem), so it runs on the planner's gather kernel with 16 taps and Cin = 16.
conv_out's 19 classes are zero-padded to 32 output channels.  The attention / pooling 1x1s (ARM conv_atten + BN, conv_avg + BN,
FFM conv1 / conv2) act on one pooled vector per image and stay fp32 for chan_gate.  conv_out16 / conv_out32 are dead code in
FaceParsing (it reads output [0] only); their keys are accepted and ignored.

Graph: bisenet_prep -> stem (4x4 conv + ReLU) -> maxpool3x3s2 -> the eight BasicBlocks (conv1 + ReLU; conv2 with the shortcut as
the epilogue's residual, ReLU after the add; 1x1 stride-2 downsample convs) -> ARM32 (3x3 conv, chan_gate sigmoid, chan_scale_add
of the broadcast conv_avg vector from chan_gate ReLU) -> nearest 2x + conv_head32 as one sub-pixel conv (ConvWeight.upconv) ->
ARM16 (+ the conv_head32 map) -> nearest 2x + conv_head16 -> FFM: layer2 and conv_head16 write the two channel halves of one
256-channel map (torch.cat costs nothing), convblk 1x1, chan_gate (1x1 -> ReLU -> 1x1 -> sigmoid), feat * att + feat ->
conv_out (3x3 + ReLU, 1x1 to 32 channels) -> bisenet_upsample_argmax (bilinear align_corners=True to 512 x 512 and the arg-max over
the 19 classes; the interpolated logits are never written).

fp16 range.  Folded weights and biases of 2^14 or more are rejected (a 4x margin to the fp16 range).  The published 79999_iter.pth
has not been run here; the tests assert the largest activation of every layer on their synthetic weights."""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import numpy as np

from .layerplan import Layer, LayerSession, Step, _f64, check_fp16_margin, fp16_weights
from .ops import Ctx

INPUT, S2D, IN_C = 512, 259, 16
N_CLASSES, OUT_C = 19, 32
BN_EPS = 1e-5
# (layer, blocks, cin, cout, stride, output map size) of Resnet18 at 512 x 512
LAYERS = [("layer1", 2, 64, 64, 1, 128), ("layer2", 2, 64, 128, 2, 64), ("layer3", 2, 128, 256, 2, 32), ("layer4", 2, 256, 512, 2, 16)]


def _fold(sd, wk: str, bn: Optional[str]) -> Tuple[np.ndarray, np.ndarray]:
    w = _f64(sd[wk])
    if bn is None:
        return w, np.zeros(w.shape[0])
    s = _f64(sd[bn + ".weight"]) / np.sqrt(_f64(sd[bn + ".running_var"]) + BN_EPS)
    return w * s[:, None, None, None], _f64(sd[bn + ".bias"]) - _f64(sd[bn + ".running_mean"]) * s


def s2d_stem(w7: np.ndarray) -> np.ndarray:
    """[cout, 3, 7, 7] -> [cout, 16, 4, 4] in float64: s2d channel (2 by + bx) * 3 + c at tap (a, b) is kernel element
    (2 a + by - 1, 2 b + bx - 1) (bisenet_prep puts input pixel (2 (j - 2) + by, 2 (i - 2) + bx) at s2d pixel (j, i))."""
    w4 = np.zeros((w7.shape[0], IN_C, 4, 4))
    for a in range(4):
        for b in range(4):
            for by in range(2):
                for bx in range(2):
                    ky, kx = 2 * a + by - 1, 2 * b + bx - 1
                    if 0 <= ky < 7 and 0 <= kx < 7:
                        w4[:, (by * 2 + bx) * 3: (by * 2 + bx) * 3 + 3, a, b] = w7[:, :, ky, kx]
    return w4


class Gate:
    """chan_gate weights: w1t fp32 [C, n1] (+ b1), optional second layer w2t [n1, n2] (+ b2); act codes of Ctx.ACT_*."""

    def __init__(self, name, w1, b1, act1, w2=None, b2=None, act2=0):
        self.name, self.act1, self.act2 = name, act1, act2
        self.w1t = np.ascontiguousarray(w1.reshape(w1.shape[0], -1).T, np.float32)
        self.b1 = None if b1 is None else np.asarray(b1, np.float32)
        self.w2t = None if w2 is None else np.ascontiguousarray(w2.reshape(w2.shape[0], -1).T, np.float32)
        self.b2 = None if b2 is None else np.asarray(b2, np.float32)
        self.dev = None


def gflop_per_frame() -> float:
    """2 x the multiply-accumulates of the live convs of the reference's BiSeNet (7x7 stem, 19 classes) for one 512 x 512 crop."""
    mac = 256 * 256 * 64 * 3 * 49
    for _, nb, cin, cout, s, hw in LAYERS:
        for b in range(nb):
            ci = cin if b == 0 else cout
            mac += hw * hw * cout * (ci + cout) * 9 + (hw * hw * cout * cin if b == 0 and (cin != cout or s != 1) else 0)
    mac += 16 * 16 * 128 * 512 * 9 + 128 * 128 + 512 * 128                 # ARM32 conv, conv_atten, conv_avg
    mac += 32 * 32 * 128 * 128 * 9 + 32 * 32 * 128 * 256 * 9 + 128 * 128     # conv_head32, ARM16 conv, conv_atten
    mac += 64 * 64 * 128 * 128 * 9 + 64 * 64 * 256 * 256 + 2 * 256 * 64       # conv_head16, FFM convblk, conv1 / conv2
    mac += 64 * 64 * 256 * 256 * 9 + 64 * 64 * 256 * N_CLASSES               # conv_out
    return 2.0 * mac / 1e9


def plan(sd) -> Tuple[List[Layer], Dict[str, Gate], Dict[str, Tuple[int, int, int]]]:
    """Host-side plan from a BiSeNet state dict: (convs in forward order, gates, buffers {name: (H, W, C)})."""
    layers: List[Layer] = []
    bufs = {"in": (S2D, S2D, IN_C)}

    def conv(name, wk, bn, stride, relu, src, dst, res=None, up=False, w64=None, pad=None):
        w, b = _fold(sd, wk, bn)
        if w64 is not None:
            w = w64(w)
            b = np.concatenate([b, np.zeros(w.shape[0] - b.shape[0])])
        w, b = fp16_weights(f"BiSeNet {name}", w, b)
        layers.append(Layer(name, "conv", w, b, stride, w.shape[-1] // 2 if pad is None else pad, relu, src, dst, res, up))

    bufs["stem"] = (256, 256, 64)
    conv("stem", "cp.resnet.conv1.weight", "cp.resnet.bn1", 1, True, ("in", 0, IN_C), ("stem", 0, 64), w64=s2d_stem, pad=0)
    bufs["pool"] = (128, 128, 64)
    cur = ("pool", 0, 64)
    for name, nb, cin, cout, s, hw in LAYERS:
        for b in range(nb):
            p = f"cp.resnet.{name}.{b}"
            st = s if b == 0 else 1
            bufs[p + ".conv1"] = (hw, hw, cout)
            conv(p + ".conv1", p + ".conv1.weight", p + ".bn1", st, True, cur, (p + ".conv1", 0, cout))
            short = cur
            if p + ".downsample.0.weight" in sd:
                bufs[p + ".downsample"] = (hw, hw, cout)
                conv(p + ".downsample", p + ".downsample.0.weight", p + ".downsample.1", st, False, cur, (p + ".downsample", 0, cout))
                short = (p + ".downsample", 0, cout)
            if name == "layer2" and b == nb - 1:         # feat8: channels [0, 128) of FFM's concatenated input
                bufs["fcat"] = (64, 64, 256)
                dst = ("fcat", 0, 128)
            else:
                bufs[p] = (hw, hw, cout)
                dst = (p, 0, cout)
            conv(p + ".conv2", p + ".conv2.weight", p + ".bn2", 1, True, (p + ".conv1", 0, cout), dst, res=short)
            cur = dst
        if name == "layer3":
            feat16 = cur
    feat32 = cur

    bufs["arm32"] = (16, 16, 128)
    conv("arm32", "cp.arm32.conv.conv.weight", "cp.arm32.conv.bn", 1, True, feat32, ("arm32", 0, 128))
    bufs["sum32"] = (16, 16, 128)
    bufs["head32"] = (32, 32, 128)
    conv("conv_head32", "cp.conv_head32.conv.weight", "cp.conv_head32.bn", 1, True, ("sum32", 0, 128), ("head32", 0, 128), up=True)
    bufs["arm16"] = (32, 32, 128)
    conv("arm16", "cp.arm16.conv.conv.weight", "cp.arm16.conv.bn", 1, True, feat16, ("arm16", 0, 128))
    bufs["sum16"] = (32, 32, 128)
    conv("conv_head16", "cp.conv_head16.conv.weight", "cp.conv_head16.bn", 1, True, ("sum16", 0, 128), ("fcat", 128, 128), up=True)
    bufs["ffm"] = (64, 64, 256)
    conv("ffm", "ffm.convblk.conv.weight", "ffm.convblk.bn", 1, True, ("fcat", 0, 256), ("ffm", 0, 256))
    bufs["fuse"] = (64, 64, 256)
    bufs["head"] = (64, 64, 256)
    conv("conv_out", "conv_out.conv.conv.weight", "conv_out.conv.bn", 1, True, ("fuse", 0, 256), ("head", 0, 256))
    bufs["logits"] = (64, 64, OUT_C)
    conv("classes", "conv_out.conv_out.weight", None, 1, False, ("head", 0, 256), ("logits", 0, OUT_C),
         w64=lambda w: np.concatenate([w, np.zeros((OUT_C - w.shape[0],) + w.shape[1:])], 0))

    gates = {}

    def gate(name, wk, bn, act, *second):
        w, b = _fold(sd, wk, bn)
        check_fp16_margin(f"BiSeNet {name}", w, b)
        if second:
            w2 = _f64(sd[second[0]])
            check_fp16_margin(f"BiSeNet {name}", w2)
            gates[name] = Gate(name, w, None, Ctx.ACT_RELU, w2, None, act)
        else:
            gates[name] = Gate(name, w, b, act)

    gate("avg", "cp.conv_avg.conv.weight", "cp.conv_avg.bn", Ctx.ACT_RELU)
    gate("att32", "cp.arm32.conv_atten.weight", "cp.arm32.bn_atten", Ctx.ACT_SIGMOID)
    gate("att16", "cp.arm16.conv_atten.weight", "cp.arm16.bn_atten", Ctx.ACT_SIGMOID)
    gate("attffm", "ffm.conv1.weight", None, Ctx.ACT_SIGMOID, "ffm.conv2.weight")
    return layers, gates, bufs


class BiSeNetNet:
    """Device-resident BiSeNet: the plan's conv weights (ConvWeight) and the gates' fp32 weights."""

    def __init__(self, ctx: Ctx, layers, gates, bufs):
        self.ctx, self.layers, self.gates, self.bufs = ctx, layers, gates, bufs

    @classmethod
    def from_state_dict(cls, sd, ctx: Optional[Ctx] = None) -> "BiSeNetNet":
        """sd: the reference's BiSeNet state dict (79999_iter.pth: cp.resnet.*, cp.arm*, cp.conv_*, ffm.*, conv_out.*)."""
        sd = {k[len("module."):] if k.startswith("module.") else k: v for k, v in sd.items()}
        layers, gates, bufs = plan(sd)
        ctx = ctx or Ctx()
        for L in layers:
            L.upload(ctx)
        for g in gates.values():
            g.dev = tuple(None if a is None else ctx.upload(a) for a in (g.w1t, g.b1, g.w2t, g.b2))
        net = cls(ctx, layers, gates, bufs)
        ctx.sync()
        return net


class BiSeNetParser(LayerSession):
    """One captured graph for batches of N RGB crops of 512 x 512.  Every conv writes its own buffer (the layer tests read them);
    labels: the u8 [N, 512, 512] label map the graph writes."""

    def __init__(self, net: BiSeNetNet, N: int, ctx: Optional[Ctx] = None):
        self.net, N = net, int(N)
        bufs = {"rgb": ((N, INPUT, INPUT, 3), np.uint8), **{name: ((N,) + hwc, np.float16) for name, hwc in net.bufs.items()},
                **{name: ((N, (g.w1t if g.w2t is None else g.w2t).shape[1]), np.float32) for name, g in net.gates.items()},
                "labels": ((N, INPUT, INPUT), np.uint8)}

        def gate(name, src):
            g = net.gates[name]
            return Step(name, run=lambda s, x, y: s.ctx.chan_gate(s.buf[src], s.N, g.dev[0], g.dev[1], g.act1, s.buf[name], g.dev[2],
                                                                  g.dev[3], g.act2))

        def scale_add(src, g, out, **y):            # out = src * gate g + (yvec: a gate vector, y: a map, neither: src)
            return Step(out, run=lambda s, x_, y_: s.ctx.chan_scale_add(s.buf[src], s.N, s.buf[g], s.buf[out],
                                                                         **{k: s.buf[v] for k, v in y.items()}))
        before = {"cp.resnet.layer1.0.conv1": [Step("pool", src=("stem", 0, 64), dst=("pool", 0, 64),
                                                    run=lambda s, x, y: s.ctx.maxpool3x3s2(x, s.N, 256, 256, y))],
                  "arm32": [gate("avg", "cp.resnet.layer4.1")]}
        after = {"arm32": [gate("att32", "arm32"), scale_add("arm32", "att32", "sum32", yvec="avg")],
                 "arm16": [gate("att16", "arm16"), scale_add("arm16", "att16", "sum16", y="head32")],
                 "ffm": [gate("attffm", "ffm"), scale_add("ffm", "attffm", "fuse")]}
        steps = [Step("prep", src=("rgb", 0, 3), dst=("in", 0, IN_C), run=lambda s, x, y: s.ctx.bisenet_prep(x, s.N, y))]
        for L in net.layers:
            steps += before.get(L.name, []) + [Step(L.name, L)] + after.get(L.name, [])
        steps.append(Step("argmax", src=("logits", 0, OUT_C),
                          run=lambda s, x, y: s.ctx.bisenet_upsample_argmax(x, s.N, N_CLASSES, s.buf["labels"])))
        super().__init__(N, bufs, steps, ctx, zero=True)
        self.labels = self.buf["labels"]

    def parse(self, rgb512_u8: np.ndarray) -> np.ndarray:
        """u8 RGB [n <= N, 512, 512, 3] (FaceParsing's PIL resize of each crop) -> u8 labels [n, 512, 512]."""
        x = np.ascontiguousarray(rgb512_u8, np.uint8)
        n = x.shape[0]
        if x.shape[1:] != (INPUT, INPUT, 3) or not 1 <= n <= self.N:
            raise ValueError(f"expected up to {self.N} RGB crops of 512x512x3, got {x.shape}")
        return self.replay({"rgb": x}, ("labels",))[0]
