"""The layer-plan graph session of the avatar-creation networks (S3FD, PFLD, BiSeNet): a named buffer table and a list of steps,
captured once into one CUDA graph and replayed on batches of up to N images.

A plan is host data.  ``Layer`` is one planner conv or depthwise conv with its host weights and its (buffer, c_off, C) references;
``Step`` is one op of the graph: a Layer, which the session runs generically, or a closure over its ``Ctx`` op.  Each network
builds its own plan and keeps its own input validation; ``LayerSession`` allocates the buffers, captures the steps and replays."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Any, Callable, Dict, List, Optional, Tuple

import numpy as np

from .graph import GraphSession
from .ops import ConvWeight, Ctx, DevTensor

FP16_LIMIT = 2.0 ** 14
Ref = Tuple[str, int, int]                 # (buffer, c_off, C): a channel slice of a buffer of the table


def _f64(t) -> np.ndarray:
    return t.detach().cpu().double().numpy() if hasattr(t, "detach") else np.asarray(t, np.float64)


def check_fp16_margin(what: str, *arrs):
    """Reject folded values of 2^14 or more (less than a 4x margin to the fp16 range), and NaN."""
    for a in arrs:
        m = float(np.abs(a).max(initial=0.0))
        if not m < FP16_LIMIT:
            raise ValueError(f"{what}: largest folded value {m:g} leaves less than a 4x margin to the fp16 range")


def fp16_weights(what: str, w: np.ndarray, b: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """Folded float64 (w, b) -> (w rounded once to fp16, as float32; b as float32), after check_fp16_margin."""
    check_fp16_margin(what, w, b)
    return w.astype(np.float16).astype(np.float32), b.astype(np.float32)


@dataclass
class Layer:
    """kind "conv" (Ctx.conv, the planner) or "dw" (Ctx.dwconv3x3).  w: the padded kernel in PyTorch layout, fp16-rounded values
    as float32 ([cout, cin, k, k], [C, 1, 3, 3] for "dw"); b: fp32 [cout].  res: the residual the epilogue adds (None: none);
    up: nearest 2x upsample fused in front (ConvWeight.upconv).  dev: the device weights, set by upload()."""
    name: str
    kind: str
    w: np.ndarray
    b: np.ndarray
    stride: int
    pad: int
    relu: bool
    src: Ref
    dst: Ref
    res: Optional[Ref] = None
    up: bool = False
    dev: Any = None

    def upload(self, ctx: Ctx):
        if self.kind == "dw":
            C = self.w.shape[0]
            self.dev = (ctx.upload(np.ascontiguousarray(self.w.reshape(C, 9).T).astype(np.float16)), ctx.upload(self.b))
        else:
            self.dev = ConvWeight(ctx, self.w, self.b)
            if self.up:
                self.dev.upconv(ctx)


@dataclass
class Step:
    """One op of the graph: a Layer, run on the views of src and dst (the layer's own unless given), or run(session, x, y) with
    x, y the views of src and dst (None where not given).  src and dst are what the arena check sees a step read and write."""
    name: str
    layer: Optional[Layer] = None
    src: Optional[Ref] = None
    dst: Optional[Ref] = None
    run: Optional[Callable] = None

    def __post_init__(self):
        if self.layer is not None:
            self.src, self.dst = self.src or self.layer.src, self.dst or self.layer.dst


class LayerSession(GraphSession):
    """One captured graph of a plan for batches of N images.

    buffers {name: (shape, dtype)} are allocated in table order (zero-filled when zero).  arenas {name: key}: buffers of one key
    share one allocation, sized to the largest and made where the first of them comes in the table; a step may not read such a
    buffer once another buffer of its arena has been written (checked at construction)."""

    def __init__(self, N: int, buffers: Dict[str, tuple], steps: List[Step], ctx: Optional[Ctx] = None, zero: bool = False,
                 arenas: Optional[Dict[str, Any]] = None):
        super().__init__(ctx)
        self.N, self.steps = int(N), steps
        try:
            self._build(buffers, arenas or {}, zero)
        except BaseException:
            self.close()
            raise

    def _build(self, buffers, arenas, zero):
        last = {}
        for st in self.steps:
            for ref in (st.src, st.layer.res if st.layer else None):
                if ref is not None and ref[0] in arenas and last.get(arenas[ref[0]], ref[0]) != ref[0]:
                    raise ValueError(f"step {st.name} reads {ref[0]} after {last[arenas[ref[0]]]} has overwritten its arena")
            if st.dst is not None and st.dst[0] in arenas:
                last[arenas[st.dst[0]]] = st.dst[0]
        size, store, self.buf = {}, {}, {}
        for name, (shape, _) in buffers.items():
            if name in arenas:
                size[arenas[name]] = max(size.get(arenas[name], 0), int(np.prod(shape)))
        for name, (shape, dtype) in buffers.items():
            key = arenas.get(name)
            if key is None:
                self.buf[name] = self.alloc(shape, dtype, zero=zero)
                continue
            if key not in store:
                store[key] = self.alloc((size[key],), dtype, zero=zero)
            self.buf[name] = DevTensor(store[key].ptr, shape, dtype)
        self.ctx.sync()
        with self.ctx.capture() as g:
            for st in self.steps:
                x = None if st.src is None else self.view(st.src)
                y = None if st.dst is None else self.view(st.dst)
                if st.layer is None:
                    st.run(self, x, y)
                elif st.layer.kind == "dw":
                    self.ctx.dwconv3x3(x, self.N, x.shape[1], x.shape[2], *st.layer.dev, st.layer.stride, st.layer.relu, y)
                else:
                    self.ctx.conv(x, st.layer.dev, y, **self._conv_kw(st.layer, x, y))
        self.graph = g.graph

    def view(self, ref: Ref) -> DevTensor:
        """(buffer, c_off, C) -> the channel-slice view; C wider than the buffer's pitch: the whole map seen as [N, 1, 1, H W pitch]
        (PFLD's conv8 reads conv7's map as one 2304-wide pixel)."""
        name, c_off, C = ref
        t = self.buf[name]
        n, h, w, pitch = t.shape
        if C > pitch:
            return DevTensor(t.ptr, (n, 1, 1, h * w * pitch), t.dtype)
        return DevTensor(t.ptr, (n, h, w, C), t.dtype, pitch=pitch, c_off=c_off)

    def _conv_kw(self, L: Layer, x: DevTensor, y: DevTensor) -> dict:
        kw = dict(N=self.N, IH=x.shape[1], IW=x.shape[2], OH=y.shape[1], OW=y.shape[2], stride=(L.stride, L.stride), pad=(L.pad, L.pad),
                  relu=L.relu)
        if L.res is not None:
            kw["res"] = self.view(L.res)
        if L.up:
            kw["upsample2x"] = True
        return kw

    def conv_variants(self) -> dict:
        """name -> the kernel instance (Ctx.conv_plan) each planner conv runs in this graph."""
        out = {}
        for st in self.steps:
            if st.layer is not None and st.layer.kind == "conv":
                x, y = self.view(st.src), self.view(st.dst)
                out[st.name] = self.ctx.conv_plan(x, st.layer.dev, y, **self._conv_kw(st.layer, x, y))
        return out

    def replay(self, inputs: Dict[str, np.ndarray], outputs) -> List[np.ndarray]:
        """inputs {buffer: n <= N images}: a partial batch is padded with copies of its last image (images are independent); one
        launch; returns the first n images of each output buffer."""
        n = len(next(iter(inputs.values())))
        if n < self.N:
            inputs = {k: np.concatenate([a, np.repeat(a[-1:], self.N - n, 0)], 0) for k, a in inputs.items()}
        with self.ctx.lock:
            for k, a in inputs.items():
                self.ctx.h2d(self.buf[k], a)
            self.graph.launch()
            return [self.ctx.download(self.buf[k])[:n] for k in outputs]
