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

from .graph import GraphSession
from .ops import ConvWeight, Ctx, DevTensor

INPUT, S2D, IN_C = 512, 259, 16
N_CLASSES, OUT_C = 19, 32
BN_EPS = 1e-5
FP16_LIMIT = 2.0 ** 14
# (layer, blocks, cin, cout, stride, output map size) of Resnet18 at 512 x 512
LAYERS = [("layer1", 2, 64, 64, 1, 128), ("layer2", 2, 64, 128, 2, 64), ("layer3", 2, 128, 256, 2, 32), ("layer4", 2, 256, 512, 2, 16)]


def _f64(t) -> np.ndarray:
    return t.detach().cpu().double().numpy() if hasattr(t, "detach") else np.asarray(t, np.float64)


def _fold(sd, wk: str, bn: Optional[str]) -> Tuple[np.ndarray, np.ndarray]:
    w = _f64(sd[wk])
    if bn is None:
        return w, np.zeros(w.shape[0])
    s = _f64(sd[bn + ".weight"]) / np.sqrt(_f64(sd[bn + ".running_var"]) + BN_EPS)
    return w * s[:, None, None, None], _f64(sd[bn + ".bias"]) - _f64(sd[bn + ".running_mean"]) * s


def _check(name: str, *arrs):
    for a in arrs:
        m = float(np.abs(a).max(initial=0.0))
        if not m < FP16_LIMIT:
            raise ValueError(f"BiSeNet {name}: largest folded value {m:g} leaves less than a 4x margin to the fp16 range")


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


class Layer:
    """One planner conv: w the fp16-rounded kernel as float32 [cout, cin, k, k], b fp32 [cout]; src / dst / res: (buffer, c_off, C)
    (res None: no residual).  up: nearest 2x upsample fused in front (ConvWeight.upconv)."""

    def __init__(self, name, w, b, stride, relu, src, dst, res=None, up=False):
        self.name, self.w, self.b, self.stride, self.relu = name, w, b, stride, relu
        self.src, self.dst, self.res, self.up = src, dst, res, up
        self.dev: Optional[ConvWeight] = None

    @property
    def pad(self) -> int:
        return 0 if self.name == "stem" else self.w.shape[-1] // 2


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

    def conv(name, wk, bn, stride, relu, src, dst, res=None, up=False, w64=None):
        w, b = _fold(sd, wk, bn)
        if w64 is not None:
            w = w64(w)
            b = np.concatenate([b, np.zeros(w.shape[0] - b.shape[0])])
        _check(name, w, b)
        layers.append(Layer(name, w.astype(np.float16).astype(np.float32), b.astype(np.float32), stride, relu, src, dst, res, up))

    bufs["stem"] = (256, 256, 64)
    conv("stem", "cp.resnet.conv1.weight", "cp.resnet.bn1", 1, True, ("in", 0, IN_C), ("stem", 0, 64), w64=s2d_stem)
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
        _check(name, w, b)
        if second:
            w2 = _f64(sd[second[0]])
            _check(name, w2)
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
            L.dev = ConvWeight(ctx, L.w, L.b)
            if L.up:
                L.dev.upconv(ctx)
        for g in gates.values():
            g.dev = tuple(None if a is None else ctx.upload(a) for a in (g.w1t, g.b1, g.w2t, g.b2))
        net = cls(ctx, layers, gates, bufs)
        ctx.sync()
        return net


class BiSeNetParser(GraphSession):
    """One captured graph for batches of N RGB crops of 512 x 512.  Every conv writes its own buffer (the layer tests read them)."""

    def __init__(self, net: BiSeNetNet, N: int, ctx: Optional[Ctx] = None):
        super().__init__(ctx)
        self.net, self.N = net, int(N)
        try:
            self._build()
        except BaseException:
            self.close()
            raise

    def _build(self):
        N, net = self.N, self.net
        self.rgb = self.alloc((N, INPUT, INPUT, 3), np.uint8, zero=True)
        self.buf = {name: self.alloc((N, h, w, c), zero=True) for name, (h, w, c) in net.bufs.items()}
        self.vec = {name: self.alloc((N, g.w2t.shape[1] if g.w2t is not None else g.w1t.shape[1]), np.float32, zero=True)
                    for name, g in net.gates.items()}
        self.labels = self.alloc((N, INPUT, INPUT), np.uint8, zero=True)
        conv = {L.name: L for L in net.layers}
        self.ops = [("prep", None)]
        for L in net.layers:
            if L.name == "cp.resnet.layer1.0.conv1":
                self.ops.append(("pool", None))
            if L.name == "arm32":
                self.ops.append(("gate", ("avg", "cp.resnet.layer4.1")))
            self.ops.append(("conv", L))
            if L.name == "arm32":
                self.ops += [("gate", ("att32", "arm32")), ("scale_add", ("arm32", "att32", "sum32", ("vec", "avg")))]
            elif L.name == "arm16":
                self.ops += [("gate", ("att16", "arm16")), ("scale_add", ("arm16", "att16", "sum16", ("map", "head32")))]
            elif L.name == "ffm":
                self.ops += [("gate", ("attffm", "ffm")), ("scale_add", ("ffm", "attffm", "fuse", ("self", None)))]
        self.ops.append(("argmax", conv["classes"]))
        self.ctx.sync()
        with self.ctx.capture() as g:
            for op in self.ops:
                self._run(op)
        self.graph = g.graph

    def view(self, ref) -> DevTensor:
        """(buffer, c_off, C) -> the channel-slice view."""
        name, c_off, C = ref
        t = self.buf[name]
        n, h, w, pitch = t.shape
        return DevTensor(t.ptr, (n, h, w, C), pitch=pitch, c_off=c_off)

    def _conv_kw(self, L: Layer) -> dict:
        x, y = self.view(L.src), self.view(L.dst)
        kw = dict(N=self.N, IH=x.shape[1], IW=x.shape[2], OH=y.shape[1], OW=y.shape[2], stride=(L.stride, L.stride), pad=(L.pad, L.pad),
                  relu=L.relu, upsample2x=L.up)
        if L.res is not None:
            kw["res"] = self.view(L.res)
        return kw

    def _run(self, op):
        kind, a = op
        ctx, N = self.ctx, self.N
        if kind == "prep":
            ctx.bisenet_prep(self.rgb, N, self.buf["in"])
        elif kind == "pool":
            ctx.maxpool3x3s2(self.buf["stem"], N, 256, 256, self.buf["pool"])
        elif kind == "conv":
            ctx.conv(self.view(a.src), a.dev, self.view(a.dst), **self._conv_kw(a))
        elif kind == "gate":
            g, src = self.net.gates[a[0]], a[1]
            w1t, b1, w2t, b2 = g.dev
            ctx.chan_gate(self.buf[src], N, w1t, b1, g.act1, self.vec[a[0]], w2t, b2, g.act2)
        elif kind == "scale_add":
            x, g, out, (ykind, y) = a
            kw = {"yvec": self.vec[y]} if ykind == "vec" else ({"y": self.buf[y]} if ykind == "map" else {})
            ctx.chan_scale_add(self.buf[x], N, self.vec[g], self.buf[out], **kw)
        elif kind == "argmax":
            ctx.bisenet_upsample_argmax(self.view(a.dst), N, N_CLASSES, self.labels)
        else:
            raise ValueError(kind)

    def conv_variants(self) -> dict:
        """name -> the kernel instance (Ctx.conv_plan) each planner conv runs in this graph."""
        return {L.name: self.ctx.conv_plan(self.view(L.src), L.dev, self.view(L.dst), **self._conv_kw(L)) for L in self.net.layers}

    def parse(self, rgb512_u8: np.ndarray) -> np.ndarray:
        """u8 RGB [n <= N, 512, 512, 3] (FaceParsing's PIL resize of each crop) -> u8 labels [n, 512, 512]."""
        x = np.ascontiguousarray(rgb512_u8, np.uint8)
        n = x.shape[0]
        if x.shape[1:] != (INPUT, INPUT, 3) or not 1 <= n <= self.N:
            raise ValueError(f"expected up to {self.N} RGB crops of 512x512x3, got {x.shape}")
        if n < self.N:   # images are independent: pad with copies of the last crop
            x = np.concatenate([x, np.repeat(x[-1:], self.N - n, 0)], 0)
        with self.ctx.lock:
            self.ctx.h2d(self.rgb, x)
            self.graph.launch()
            out = self.ctx.download(self.labels)
        return out[:n]
