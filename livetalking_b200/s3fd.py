"""S3FD face detector on the device: the detector of the wav2lip avatar generator (avatars/wav2lip/genavatar.py ->
face_detection.FaceAlignment.get_detections_for_batch -> detection/sfd), as one captured CUDA graph per (batch, height, width).

    net = S3FDNet.from_state_dict(torch.load("s3fd.pth"))       # the reference's key scheme
    det = S3FDDetector(net, 16, 720, 1280)
    det.detect(frames_bgr_u8)                                   # -> [(x1, y1, x2, y2) | None] * n, get_detections_for_batch's contract

Graph: s3fd_prep (u8 BGR -> fp16 NHWC, RGB minus the means, 16 channels) -> the VGG-16 trunk on the conv planner (ltb_op_conv2d,
bias + ReLU in the epilogue; fc6's padding 3 and the two stride-2 convs take whatever kernel the planner picks) with maxpool2x2
between the stages -> l2norm (in place, after the pool has read the tensor) on conv3_3 / conv4_3 / conv5_3 -> one head conv per
level with conf and loc stacked (8 output channels on conv3_3, 6 elsewhere, zero-padded to 16) -> s3fd_select (one CTA per image).

Selection.  The reference keeps the first box of nms(candidates, 0.3) whose score is above 0.5, where the candidates are the
anchors at which any image of the batch scores above 0.05.  NMS keeps the highest-scoring candidate first, and an anchor where an
image scores above 0.5 is always a candidate, so per image the result is the box of its arg-max anchor over all six levels when that
score is above 0.5, and None otherwise: s3fd_select computes exactly that, without NMS.  Exactly equal scores (implementation-defined
in the reference) go to the lowest anchor number (level, row, column).  The box is clipped at 0 and truncated, as np.clip + int().

fp16 range.  Activations are stored in fp16 with fp32 accumulation, and the conv epilogue saturates (an overflow would be clamped
to 65504 silently).  The weights of the published s3fd.pth have not been measured here; the tests assert the largest activation
of every layer on their synthetic weights.  Should a checkpoint come close to the fp16 range there is an exact remedy: scale the
input and every trunk bias by 2^-k and the fc7 / conv6_2 / conv7_2 head weights by 2^k (ReLU and max-pool commute with the
scale, L2Norm is scale-free apart from its 1e-10)."""
from __future__ import annotations

from typing import List, Optional, Tuple

import numpy as np

from .graph import _np
from .layerplan import Layer, LayerSession, Step
from .ops import Ctx

IN_C = 16            # channels of the prepared image (both conv kernels need Cin >= 16)
HEAD_C = 16          # fused conf + loc head outputs, zero-padded (the gather kernel needs Cout % 16 == 0)
L2_EPS = 1e-10
THRESH = 0.5

# (name, Cin, Cout, kernel, stride, padding) or "pool" (F.max_pool2d(h, 2, 2))
TRUNK = [("conv1_1", 3, 64, 3, 1, 1), ("conv1_2", 64, 64, 3, 1, 1), "pool",
         ("conv2_1", 64, 128, 3, 1, 1), ("conv2_2", 128, 128, 3, 1, 1), "pool",
         ("conv3_1", 128, 256, 3, 1, 1), ("conv3_2", 256, 256, 3, 1, 1), ("conv3_3", 256, 256, 3, 1, 1), "pool",
         ("conv4_1", 256, 512, 3, 1, 1), ("conv4_2", 512, 512, 3, 1, 1), ("conv4_3", 512, 512, 3, 1, 1), "pool",
         ("conv5_1", 512, 512, 3, 1, 1), ("conv5_2", 512, 512, 3, 1, 1), ("conv5_3", 512, 512, 3, 1, 1), "pool",
         ("fc6", 512, 1024, 3, 1, 3), ("fc7", 1024, 1024, 1, 1, 0),
         ("conv6_1", 1024, 256, 1, 1, 0), ("conv6_2", 256, 512, 3, 2, 1),
         ("conv7_1", 512, 128, 1, 1, 0), ("conv7_2", 128, 256, 3, 2, 1)]
# detection levels, finest first: (feature layer, channels, has L2Norm, conf channels)
LEVELS = [("conv3_3", 256, True, 4), ("conv4_3", 512, True, 2), ("conv5_3", 512, True, 2), ("fc7", 1024, False, 2),
          ("conv6_2", 512, False, 2), ("conv7_2", 256, False, 2)]


def _head_name(src: str, normed: bool) -> str:
    return src + "_norm" if normed else src


def _out_dim(i: int, k: int, s: int, p: int) -> int:
    return (i + 2 * p - k) // s + 1


def gflop_per_frame(H: int, W: int) -> float:
    """2 x the multiply-accumulates of the 31 convolutions for one H x W frame (the reference's, without head padding)."""
    mac, h, w, shapes = 0, H, W, {}
    for e in TRUNK:
        if e == "pool":
            h, w = h // 2, w // 2
            continue
        name, cin, cout, k, s, p = e
        h, w = _out_dim(h, k, s, p), _out_dim(w, k, s, p)
        mac += h * w * cout * cin * k * k
        shapes[name] = (h, w)
    for src, cin, _, nconf in LEVELS:
        h, w = shapes[src]
        mac += h * w * (nconf + 4) * cin * 9
    return 2.0 * mac / 1e9


class S3FDNet:
    """Device-resident S3FD weights: the trunk convs and the six fused heads as Layers, and the L2Norm scales."""

    def __init__(self, ctx: Ctx, convs: List[Layer], norms: dict, heads: List[Layer]):
        self.ctx, self.convs, self.norms, self.heads = ctx, convs, norms, heads

    @classmethod
    def from_state_dict(cls, sd, ctx: Optional[Ctx] = None) -> "S3FDNet":
        """sd: the reference's s3fd state dict (conv1_1.weight ... conv3_3_norm.weight ... conv7_2_mbox_loc.bias)."""
        missing = [k for k in _expected_keys() if k not in sd]
        if missing:
            raise KeyError(f"S3FD state dict lacks {len(missing)} keys, e.g. {missing[:3]}")
        ctx = ctx or Ctx()
        convs, src = [], "in"
        for e in TRUNK:
            if e == "pool":
                src += "_pool"
                continue
            name, _, _, _, s, p = e
            convs.append(_layer(name, _np(sd[name + ".weight"]), _np(sd[name + ".bias"]), s, p, True, src, name))
            src = name
        heads = []
        for src, _, normed, _ in LEVELS:
            pre = _head_name(src, normed)
            w = np.concatenate([_np(sd[pre + "_mbox_conf.weight"]), _np(sd[pre + "_mbox_loc.weight"])], 0)
            b = np.concatenate([_np(sd[pre + "_mbox_conf.bias"]), _np(sd[pre + "_mbox_loc.bias"])], 0)
            heads.append(_layer(pre + "_mbox", w, b, 1, 1, False, pre, pre + "_mbox"))
        for L in convs:
            L.upload(ctx)
        norms = {src: ctx.upload(_np(sd[src + "_norm.weight"]).astype(np.float32)) for src, _, normed, _ in LEVELS if normed}
        for L in heads:
            L.upload(ctx)
        ctx.sync()
        return cls(ctx, convs, norms, heads)


def _layer(name, w, b, stride, pad, relu, src, dst) -> Layer:
    """A trunk conv or head, zero-padded to at least IN_C inputs (conv1_1) and HEAD_C outputs (the heads), rounded to fp16 once."""
    cout, cin = max(w.shape[0], HEAD_C), max(w.shape[1], IN_C)
    wp = np.zeros((cout, cin) + w.shape[2:], np.float32)
    wp[:w.shape[0], :w.shape[1]] = w
    bp = np.zeros(cout, np.float32)
    bp[:b.shape[0]] = b
    return Layer(name, "conv", wp.astype(np.float16).astype(np.float32), bp, stride, pad, relu, (src, 0, cin), (dst, 0, cout))


def _expected_keys():
    keys = [f"{e[0]}.{p}" for e in TRUNK if e != "pool" for p in ("weight", "bias")]
    keys += [src + "_norm.weight" for src, _, normed, _ in LEVELS if normed]
    keys += [f"{_head_name(src, normed)}_mbox_{h}.{p}" for src, _, normed, _ in LEVELS for h in ("conf", "loc") for p in ("weight", "bias")]
    return keys


class S3FDDetector(LayerSession):
    """One captured graph for batches of N frames of H x W.  keep_layers: every op writes its own buffer (the layer tests read
    them back); otherwise the trunk ping-pongs between two arenas, only the six level features have their own buffers and
    L2Norm runs in place on them."""

    def __init__(self, net: S3FDNet, N: int, H: int, W: int, keep_layers: bool = False, ctx: Optional[Ctx] = None):
        if H < 32 or W < 32:
            raise ValueError(f"S3FD needs frames of at least 32 x 32, got {H} x {W}")
        self.net, self.H, self.W = net, int(H), int(W)
        N, H, W = int(N), self.H, self.W
        bufs = {"frames": ((N, H, W, 3), np.uint8), "in": ((N, H, W, IN_C), np.float16)}
        steps = [Step("prep", src=("frames", 0, 3), dst=("in", 0, IN_C), run=lambda s, x, y: s.ctx.s3fd_prep(x, s.N, s.H, s.W, y))]
        feats = {src for src, _, _, _ in LEVELS}
        arenas, nxt, convs, cur, h, w, c = {}, 0, iter(net.convs), "in", H, W, IN_C
        for e in TRUNK:
            if e == "pool":
                name, h, w = cur + "_pool", h // 2, w // 2
                steps.append(Step(name, src=(cur, 0, c), dst=(name, 0, c),
                                  run=lambda s, x, y: s.ctx.maxpool2x2(x, s.N, x.shape[1], x.shape[2], y)))
            else:
                L = next(convs)
                name, c = L.name, L.w.shape[0]
                h, w = _out_dim(h, L.w.shape[-1], L.stride, L.pad), _out_dim(w, L.w.shape[-1], L.stride, L.pad)
                steps.append(Step(name, L))
            bufs[name] = ((N, h, w, c), np.float16)
            if not keep_layers and name not in feats:     # the next arena that does not hold the input
                if arenas.get(cur) == nxt:
                    nxt ^= 1
                arenas[name], nxt = nxt, nxt ^ 1
            cur = name
        for (src, _, normed, _), L in zip(LEVELS, net.heads):
            shape = bufs[src][0]
            f = (src, 0, shape[3])
            if normed:                                      # in place unless keep_layers: the pool has already read f
                if keep_layers:
                    bufs[L.src[0]] = bufs[src]
                steps.append(Step(L.src[0], src=f, dst=L.src if keep_layers else f,
                                  run=lambda s, x, y, g=net.norms[src]: s.ctx.l2norm(x, x.rows, g, L2_EPS, y)))
            bufs[L.name] = (shape[:3] + (HEAD_C,), np.float16)
            steps.append(Step(L.name, L, src=None if keep_layers else f))
        bufs["out_i"], bufs["out_s"] = ((N, 6), np.int32), ((N,), np.float32)
        heads = [L.name for L in net.heads]
        steps.append(Step("select", run=lambda s, x, y: s.ctx.s3fd_select([s.buf[n] for n in heads], s.N, THRESH, s.buf["out_i"],
                                                                            s.buf["out_s"])))
        super().__init__(N, bufs, steps, ctx, arenas=arenas)
        self.heads = [self.buf[n] for n in heads]

    def run_raw(self, frames_u8: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
        """frames u8 BGR [n <= N, H, W, 3] -> (int32 [n, 6] = found, x1, y1, x2, y2, anchor; float32 [n] winning score)."""
        frames_u8 = np.ascontiguousarray(frames_u8, np.uint8)
        n = frames_u8.shape[0]
        if frames_u8.shape[1:] != (self.H, self.W, 3) or not 1 <= n <= self.N:
            raise ValueError(f"expected up to {self.N} frames of {self.H}x{self.W}x3, got {frames_u8.shape}")
        return tuple(self.replay({"frames": frames_u8}, ("out_i", "out_s")))

    def detect(self, frames_u8: np.ndarray) -> List[Optional[Tuple[int, int, int, int]]]:
        oi, _ = self.run_raw(frames_u8)
        return [tuple(int(v) for v in r[1:5]) if r[0] else None for r in oi]
