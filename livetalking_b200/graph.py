"""Graph building and the session lifecycle shared by every captured-graph model leg.

``Builder`` emits the generic engine ops (convs, linears, norms, attention, upsampling, concatenation) on NHWC fp16 ``DevTensor``s
and allocates every intermediate it needs.  ``GraphSession`` is the base of the per-stream session classes: it owns the device
memory a session allocates, captures the session's op sequence into one CUDA graph and gives everything back on ``close()``."""
from __future__ import annotations

import os
from typing import Callable, List, Optional, Tuple

import numpy as np

from .ops import ConvWeight, Ctx, DevTensor, Graph


def _np(t) -> np.ndarray:
    if hasattr(t, "detach"):
        t = t.detach().cpu().float().numpy()
    return np.asarray(t, dtype=np.float32)


def _ceil16(x: int) -> int:
    return (x + 15) // 16 * 16


class _Norm:
    def __init__(self, ctx: Ctx, sd, p):
        self.gamma = ctx.upload(_np(sd[p + ".weight"]))
        self.beta = ctx.upload(_np(sd[p + ".bias"]))


class Builder:
    """Emits engine ops for generic network building blocks.  Tensors are NHWC fp16 ``DevTensor``s of shape (N,H,W,C)."""

    GN_GROUPS = 32   # every GroupNorm of the diffusers UNet / VAE uses 32 groups
    # Fusing the GroupNorm statistics into the producing conv's epilogue (ltb_conv_op.gn_stats) is implemented and tested per kernel
    # path against float64 sums (tests/test_gpu_conv_op.py::test_conv_op_groupnorm_statistics), but off by default: the extra
    # shuffles/atomics load the conv epilogue, and whether that beats the separate statistics pass has not been measured on H100.
    FUSE_GN_STATS = os.environ.get("LTB_FUSE_GN", "0") == "1"

    def __init__(self, ctx: Ctx, alloc: Optional[Callable[..., DevTensor]] = None):
        """alloc(shape, dtype, zero=...): where the intermediates come from (ctx.alloc unless given; GraphSession passes its own)."""
        self.ctx, self._alloc = ctx, alloc
        self.temps: List[DevTensor] = []

    def _stats_for(self, out: DevTensor, n_img: int):
        """Ask the producing conv to also emit the GroupNorm statistics of `out` (fused into its epilogue when possible)."""
        if not self.FUSE_GN_STATS or out.C % self.GN_GROUPS or out.pitch != out.C or out.c_off:
            return None
        st = self.new(n_img * self.GN_GROUPS * 4)                  # n_img * groups * 2 floats
        out.stats = (st, self.GN_GROUPS)
        return st

    def new(self, *shape) -> DevTensor:
        t = (self._alloc or self.ctx.alloc)(shape, np.float16, zero=True)
        self.temps.append(t)
        return t

    # -- primitives
    def conv3(self, x: DevTensor, w: ConvWeight, res: Optional[DevTensor] = None, stride: int = 1, pad=(1, 1), out: Optional[DevTensor] = None,
              stats: bool = False):
        N, H, W, _ = x.shape
        OH = (H + (2 if pad == (1, 1) else 1) - 3) // stride + 1
        OW = (W + (2 if pad == (1, 1) else 1) - 3) // stride + 1
        if out is None:
            out = self.new(N, OH, OW, w.cout)
        st = self._stats_for(out, N) if stats else None
        self.ctx.conv(x, w, out, N=N, IH=H, IW=W, OH=OH, OW=OW, stride=(stride, stride), pad=pad, res=res,
                      gn_stats=st, gn_groups=self.GN_GROUPS if st is not None else 0, gn_hw=OH * OW)
        return out

    def linear(self, x: DevTensor, w: ConvWeight, res: Optional[DevTensor] = None, out: Optional[DevTensor] = None, stats_imgs: int = 0):
        """x (..., Cin) -> (..., Cout) ; also 1x1 convs.  stats_imgs > 0: also produce GroupNorm statistics (rows/stats_imgs pixels per image)."""
        rows = x.rows
        if out is None:
            out = self.new(*x.shape[:-1], w.cout)
        st = self._stats_for(out, stats_imgs) if stats_imgs else None
        self.ctx.conv(x, w, out, N=1, IH=1, IW=rows, OH=1, OW=rows, res=res,
                      gn_stats=st, gn_groups=self.GN_GROUPS if st is not None else 0, gn_hw=(rows // stats_imgs) if stats_imgs else 0)
        return out

    def groupnorm(self, x: DevTensor, n: _Norm, groups: int, eps: float, silu: bool):
        N, H, W, C = x.shape
        out = self.new(N, H, W, C)
        if x.stats is not None and x.stats[1] == groups:
            self.ctx.groupnorm_apply(x, N, H * W, groups, eps, x.stats[0], n.gamma, n.beta, silu, out)
        else:
            self.ctx.groupnorm(x, N, H * W, groups, eps, n.gamma, n.beta, silu, out)
        return out

    def layernorm(self, x: DevTensor, n: _Norm, eps: float = 1e-5):
        out = self.new(*x.shape)
        self.ctx.layernorm(x, x.rows, x.C, eps, n.gamma, n.beta, out)
        return out

    # softmax(QK^T)V as one tcgen05 kernel (scores never reach HBM); LTB_FUSE_ATTENTION=0 restores GEMM + softmax + GEMM
    FUSE_ATTENTION = os.environ.get("LTB_FUSE_ATTENTION", "1") == "1"

    def attention(self, a, xq: DevTensor, B: int, nq: int, res: DevTensor, kv_src: Optional[DevTensor] = None, n_keys: Optional[int] = None,
                  n_valid: Optional[int] = None, stats_imgs: int = 0):
        """xq: (B*nq, C) normalised tokens.  Self-attention when kv_src is None, else keys/values from kv_src (B*n_keys, kv_dim).
        Key counts are padded to a multiple of 16 (tensor-core N / K granularity); padded keys get probability 0."""
        ctx, H, dp, d = self.ctx, a.heads, a.dp, a.d
        Hdp = H * dp
        if a.self_attn:
            nk = _ceil16(nq)
            valid = nq
            # batch b's padded keys [nq, nk) are rows of batch b + 1 (the zero rows below for the last batch) on the unfused path and
            # TMA zero fill on the fused one: both are masked to probability 0, and VT (transpose_heads) is zero for keys >= nq
            qkv = self.new(B * nq + (nk - nq), 3 * Hdp)                   # padded key rows stay zero
            self.linear(xq, a.qkv, out=DevTensor(qkv.ptr, (B * nq, 3 * Hdp)))
            q_ptr, q_pitch = qkv.ptr, 3 * Hdp
            k_ptr, v_ptr, kv_pitch = qkv.offset(Hdp), qkv.offset(2 * Hdp), 3 * Hdp
            kv_rows = nq
        else:
            q = self.linear(xq, a.q)                                      # (B*nq, Hdp)
            kv = self.linear(kv_src, a.kv)                                # (B*n_keys, 2*Hdp)
            q_ptr, q_pitch = q.ptr, Hdp
            k_ptr, v_ptr, kv_pitch = kv.ptr, kv.offset(Hdp), 2 * Hdp
            nk, valid, kv_rows = n_keys, n_valid, n_keys
        if self.FUSE_ATTENTION and dp % 16 == 0 and dp <= 160:
            VT = self.new(B * H, dp, nk)
            ctx.transpose_heads(v_ptr, B, kv_rows, kv_pitch, H, dp, nk, VT)
            O = self.new(B * nq, Hdp)
            ctx.attention(q_ptr, q_pitch, k_ptr, kv_pitch, kv_rows, VT, nk, B, H, nq, valid, dp, float(d) ** -0.5, O)
            return self.linear(O, a.out, res=res, stats_imgs=stats_imgs)
        S = self.new(B * H, nq, nk)
        qv = DevTensor(q_ptr, (nq, dp), pitch=q_pitch)
        sv = DevTensor(S.ptr, (nq, nk), pitch=nk)
        ctx.conv(qv, None, sv, N=1, IH=1, IW=nq, OH=1, OW=nq, cin=dp, cout=nk, w_ptr=k_ptr, ktot=kv_pitch,
                 zbatch=B * H, zdiv=H, in_z=(nq * q_pitch, dp), w_z=(kv_rows * kv_pitch, dp), out_z=(H * nq * nk, nq * nk))
        ctx.softmax(S, B * H * nq, nk, valid, float(d) ** -0.5)
        VT = self.new(B * H, dp, nk)
        ctx.transpose_heads(v_ptr, B, kv_rows, kv_pitch, H, dp, nk, VT)
        O = self.new(B * nq, Hdp)
        ov = DevTensor(O.ptr, (nq, dp), pitch=Hdp)
        ctx.conv(sv, None, ov, N=1, IH=1, IW=nq, OH=1, OW=nq, cin=nk, cout=dp, w_ptr=VT.ptr, ktot=nk,
                 zbatch=B * H, zdiv=H, in_z=(H * nq * nk, nq * nk), w_z=(H * dp * nk, dp * nk), out_z=(nq * Hdp, dp))
        return self.linear(O, a.out, res=res, stats_imgs=stats_imgs)

    # Upsample2D (nearest 2x + conv3x3) as ONE kernel: four 2x2 sub-pixel convs over the low-res map (ops.ConvWeight.upconv).
    FUSE_UPSAMPLE = os.environ.get("LTB_FUSE_UPSAMPLE", "1") == "1"

    def upsample(self, x: DevTensor, w: ConvWeight):
        N, H, W, C = x.shape
        if self.FUSE_UPSAMPLE and w.upconv_supported() and x.pitch % 8 == 0 and x.c_off % 8 == 0:
            out = self.new(N, 2 * H, 2 * W, w.cout)
            self.ctx.conv(x, w, out, N=N, IH=H, IW=W, OH=2 * H, OW=2 * W, pad=(1, 1), upsample2x=True)
            return out
        up = self.new(N, 2 * H, 2 * W, C)
        self.ctx.upsample2x(x, N, H, W, up)
        return self.conv3(up, w, stats=True)

    def concat(self, a: DevTensor, b: DevTensor):
        N, H, W, _ = a.shape
        out = self.new(N, H, W, a.C + b.C)
        self.ctx.copy_channels(a, DevTensor(out.ptr, (N, H, W, a.C), pitch=out.C, c_off=0))
        self.ctx.copy_channels(b, DevTensor(out.ptr, (N, H, W, b.C), pitch=out.C, c_off=a.C))
        return out


class _Replay:
    """Hands back the buffers of the eager pass, in order, while the same op sequence is being captured."""

    def __init__(self, temps):
        self.temps, self.i = temps, 0

    def __call__(self, *shape):
        if self.i == len(self.temps):
            raise RuntimeError(f"the captured pass asks for more than the eager pass's {len(self.temps)} buffers")
        t = self.temps[self.i]
        self.i += 1
        if t.shape != tuple(shape):
            raise RuntimeError(f"captured pass buffer {self.i - 1}: shape {tuple(shape)}, the eager pass made {t.shape}")
        return t

    def finish(self):
        if self.i != len(self.temps):
            raise RuntimeError(f"the captured pass took {self.i} of the eager pass's {len(self.temps)} buffers")


class GraphSession:
    """A session that runs captured CUDA graphs on one device context and owns the memory it allocates there.

    ctx=None: the session creates its own Ctx and close() closes it, which frees everything on it.  A given ctx is borrowed:
    close() frees exactly the tensors the session made through alloc() and capture(), and neither the ctx nor any tensor the
    session was handed.  with_ctx=False: no session ctx at all (a paste-only session).  A constructor that raises calls close()."""

    def __init__(self, ctx: Optional[Ctx] = None, with_ctx: bool = True):
        self.graph: Optional[Graph] = None
        self._owned: List[DevTensor] = []
        self._ctxs: List[Ctx] = []                       # contexts close() closes
        self._paste: Optional[Tuple[Ctx, DevTensor, DevTensor]] = None
        self._borrowed = with_ctx and ctx is not None
        self.ctx = None
        if with_ctx:
            self.ctx = ctx if ctx is not None else self.new_ctx()

    def new_ctx(self) -> Ctx:
        """Another context owned by the session (its own stream and memory): close() closes it."""
        c = Ctx()
        self._ctxs.append(c)
        return c

    def paste_ctx(self, pred_shape, pred_dtype, frame_shape) -> Tuple[Ctx, DevTensor, DevTensor]:
        """(ctx, prediction scratch, uint8 output frame) for pasting one host prediction, made on first use.  The ctx is the session's
        own (new_ctx), so a paste runs while the session's graph is in flight (the reference's process_frames thread)."""
        if self._paste is None:
            c = self.new_ctx()
            self._paste = (c, c.alloc(pred_shape, pred_dtype), c.alloc(frame_shape, np.uint8))
        return self._paste

    def alloc(self, shape, dtype=np.float16, zero: bool = False) -> DevTensor:
        t = self.ctx.alloc(shape, dtype, zero=zero)
        self._owned.append(t)
        return t

    def capture(self, emit: Callable[[Builder], None]):
        """self.graph := the ops emit(builder) enqueues on self.ctx.  emit runs twice: an eager pass that allocates every intermediate
        (owned by the session) and warms the kernels up, then the captured pass, which gets exactly the same buffers in the same order."""
        b = Builder(self.ctx, self.alloc)
        emit(b)
        self.ctx.sync()
        replay = b.new = _Replay(b.temps)
        with self.ctx.capture() as cap:
            emit(b)
            replay.finish()
        self.graph = cap.graph

    def close(self):
        """Release the graph, then the session's memory.  Idempotent."""
        if self.graph is not None:
            self.graph.close()
            self.graph = None
        owned, self._owned = self._owned, []
        if self._borrowed and owned:
            self.ctx.sync()
            for t in owned:
                self.ctx.free(t)
        ctxs, self._ctxs, self._paste = self._ctxs, [], None
        for c in ctxs:
            c.close()
        self.ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
