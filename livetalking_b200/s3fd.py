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

from .ops import ConvWeight, Ctx, DevTensor

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


def _np(t) -> np.ndarray:
    return t.detach().cpu().float().numpy() if hasattr(t, "detach") else np.asarray(t, np.float32)


class S3FDNet:
    """Device-resident S3FD weights: trunk convs, L2Norm scales and the six fused heads."""

    def __init__(self, ctx: Ctx, convs: dict, norms: dict, heads: list):
        self.ctx, self.convs, self.norms, self.heads = ctx, convs, norms, heads

    @classmethod
    def from_state_dict(cls, sd, ctx: Optional[Ctx] = None) -> "S3FDNet":
        """sd: the reference's s3fd state dict (conv1_1.weight ... conv3_3_norm.weight ... conv7_2_mbox_loc.bias)."""
        missing = [k for k in _expected_keys() if k not in sd]
        if missing:
            raise KeyError(f"S3FD state dict lacks {len(missing)} keys, e.g. {missing[:3]}")
        ctx = ctx or Ctx()
        convs = {}
        for e in TRUNK:
            if e == "pool":
                continue
            name = e[0]
            convs[name] = ConvWeight(ctx, _np(sd[name + ".weight"]), _np(sd[name + ".bias"]), pad_cin=IN_C if name == "conv1_1" else None)
        norms = {src: ctx.upload(_np(sd[src + "_norm.weight"]).astype(np.float32)) for src, _, normed, _ in LEVELS if normed}
        heads = []
        for src, _, normed, _ in LEVELS:
            pre = _head_name(src, normed)
            w = np.concatenate([_np(sd[pre + "_mbox_conf.weight"]), _np(sd[pre + "_mbox_loc.weight"])], 0)
            b = np.concatenate([_np(sd[pre + "_mbox_conf.bias"]), _np(sd[pre + "_mbox_loc.bias"])], 0)
            heads.append(ConvWeight(ctx, w, b, pad_cout=HEAD_C))
        ctx.sync()
        return cls(ctx, convs, norms, heads)


def _expected_keys():
    keys = [f"{e[0]}.{p}" for e in TRUNK if e != "pool" for p in ("weight", "bias")]
    keys += [src + "_norm.weight" for src, _, normed, _ in LEVELS if normed]
    keys += [f"{_head_name(src, normed)}_mbox_{h}.{p}" for src, _, normed, _ in LEVELS for h in ("conf", "loc") for p in ("weight", "bias")]
    return keys


class S3FDDetector:
    """One captured graph for batches of N frames of H x W.  keep_layers: every op writes its own buffer (the layer tests read
    them back); otherwise the trunk ping-pongs between two buffers and only the six level features have their own."""

    def __init__(self, net: S3FDNet, N: int, H: int, W: int, keep_layers: bool = False, ctx: Optional[Ctx] = None):
        if H < 32 or W < 32:
            raise ValueError(f"S3FD needs frames of at least 32 x 32, got {H} x {W}")
        self.net, self.N, self.H, self.W = net, int(N), int(H), int(W)
        self.ctx = ctx or Ctx()
        self._owned = []
        try:
            self._build(keep_layers)
        except Exception:
            self.close()
            raise

    def _alloc(self, shape, dtype=np.float16) -> DevTensor:
        t = self.ctx.alloc(shape, dtype)
        self._owned.append(t)
        return t

    def _build(self, keep: bool):
        N, H, W = self.N, self.H, self.W
        self.frames = self._alloc((N, H, W, 3), np.uint8)
        x0 = self._alloc((N, H, W, IN_C))
        self.ops: List[tuple] = [("prep", "prep", self.frames, x0, {})]
        feats = {src for src, _, _, _ in LEVELS}
        # pass 1: shapes, so that the ping-pong buffers can be sized
        plan, h, w, c = [], H, W, IN_C
        for e in TRUNK:
            if e == "pool":
                plan.append(("pool", plan[-1][1] + "_pool", (N, h // 2, w // 2, c), dict(N=N, H=h, W=w)))
                h, w = h // 2, w // 2
                continue
            name, _, cout, k, s, p = e
            oh, ow = _out_dim(h, k, s, p), _out_dim(w, k, s, p)
            plan.append(("conv", name, (N, oh, ow, cout), dict(N=N, IH=h, IW=w, OH=oh, OW=ow, stride=(s, s), pad=(p, p), relu=True)))
            h, w, c = oh, ow, cout
        pp = []
        if not keep:
            big = max(int(np.prod(shape)) for kind, name, shape, _ in plan if name not in feats)
            pp = [self._alloc((big,)), self._alloc((big,))]
        cur, nxt, fmap = x0, 0, {}
        for kind, name, shape, kw in plan:
            if keep or name in feats:
                out = self._alloc(shape)
            else:
                if cur.ptr == pp[nxt].ptr:
                    nxt ^= 1
                out = DevTensor(pp[nxt].ptr, shape)
                nxt ^= 1
            self.ops.append((kind, name, cur, out, kw))
            if name in feats:
                fmap[name] = out
            cur = out
        self.heads = []
        for lv, (src, _, normed, _) in enumerate(LEVELS):
            f = fmap[src]
            n_, fh, fw, fc = f.shape
            if normed:
                g = self._alloc(f.shape) if keep else f          # in place: the pool has already read f
                self.ops.append(("l2norm", src + "_norm", f, g, dict(npix=n_ * fh * fw, w=self.net.norms[src])))
                f = g
            hd = self._alloc((N, fh, fw, HEAD_C))
            self.ops.append(("head", _head_name(src, normed) + "_mbox", f, hd,
                             dict(N=N, IH=fh, IW=fw, OH=fh, OW=fw, stride=(1, 1), pad=(1, 1), relu=False, level=lv)))
            self.heads.append(hd)
        self.out_i = self._alloc((N, 6), np.int32)
        self.out_s = self._alloc((N,), np.float32)
        self.ops.append(("select", "select", None, self.out_i, {}))
        self.ctx.sync()
        with self.ctx.capture() as g:
            for op in self.ops:
                self._run(op)
        self.graph = g.graph

    def _weights(self, kind: str, name: str, kw: dict) -> ConvWeight:
        return self.net.heads[kw["level"]] if kind == "head" else self.net.convs[name]

    def _conv_kw(self, kw: dict) -> dict:
        return {k: v for k, v in kw.items() if k != "level"}

    def _run(self, op):
        kind, name, x, y, kw = op
        ctx = self.ctx
        if kind == "prep":
            ctx.s3fd_prep(self.frames, self.N, self.H, self.W, y)
        elif kind in ("conv", "head"):
            ctx.conv(x, self._weights(kind, name, kw), y, **self._conv_kw(kw))
        elif kind == "pool":
            ctx.maxpool2x2(x, kw["N"], kw["H"], kw["W"], y)
        elif kind == "l2norm":
            ctx.l2norm(x, kw["npix"], kw["w"], L2_EPS, y)
        elif kind == "select":
            ctx.s3fd_select(self.heads, self.N, THRESH, self.out_i, self.out_s)
        else:
            raise ValueError(kind)

    def conv_variants(self) -> dict:
        """name -> the kernel instance (Ctx.conv_plan) each conv and head runs in this graph."""
        return {name: self.ctx.conv_plan(x, self._weights(kind, name, kw), y, **self._conv_kw(kw))
                for kind, name, x, y, kw in self.ops if kind in ("conv", "head")}

    def run_raw(self, frames_u8: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
        """frames u8 BGR [n <= N, H, W, 3] -> (int32 [n, 6] = found, x1, y1, x2, y2, anchor; float32 [n] winning score)."""
        frames_u8 = np.ascontiguousarray(frames_u8, np.uint8)
        n = frames_u8.shape[0]
        if frames_u8.shape[1:] != (self.H, self.W, 3) or not 1 <= n <= self.N:
            raise ValueError(f"expected up to {self.N} frames of {self.H}x{self.W}x3, got {frames_u8.shape}")
        if n < self.N:   # images are independent: pad with copies of the last frame
            frames_u8 = np.concatenate([frames_u8, np.repeat(frames_u8[-1:], self.N - n, 0)], 0)
        with self.ctx.lock:
            self.ctx.h2d(self.frames, frames_u8)
            self.graph.launch()
            oi = self.ctx.download(self.out_i)
            os_ = self.ctx.download(self.out_s)
        return oi[:n], os_[:n]

    def detect(self, frames_u8: np.ndarray) -> List[Optional[Tuple[int, int, int, int]]]:
        oi, _ = self.run_raw(frames_u8)
        return [tuple(int(v) for v in r[1:5]) if r[0] else None for r in oi]

    def close(self):
        g = getattr(self, "graph", None)
        if g is not None:
            g.close()
            self.graph = None
        for t in self._owned:
            try:
                self.ctx.free(t)
            except Exception:
                pass
        self._owned = []
