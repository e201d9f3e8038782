"""Op tracer for the device-op layer: wraps the op methods of ONE ``livetalking_b200.ops.Ctx`` instance (instance attributes, the
class is untouched) so that an eager pass records every op it launches together with the data the op actually read and wrote.

For every traced call the tracer
  * syncs the stream and reads each input view back BEFORE the op runs, so an in-place op (eltwise GELU) is seen with its input;
  * for ``conv``, records ``ctx.conv_plan(...)`` with the same arguments: the kernel instance that ran;
  * reads the whole allocation under each output view before and after the op and records every byte outside the view that
    changed (an output whose allocation the tracer did not see being made is checked over the span of its view, pitch gaps
    included);
  * keeps the dense contents of the input and output views, passed through ``keep`` (e.g. to keep some images of a batch).
Channel-sliced views are read at full pitch and sliced on the host: no kernel runs for a read-back.  Ops that take raw pointers
(``attention``, ``transpose_heads``) get their views rebuilt from the pointer, pitch and row arguments.  Entering
``ctx.capture()`` stops tracing (a sync inside stream capture is illegal); ``stop()`` restores the plain methods."""
from __future__ import annotations

import inspect
from typing import Callable, Dict, List, Optional

import numpy as np

UL_OPS = ("conv", "dwconv3x3", "upsample_bilinear2x", "head_sigmoid255", "ul_prep", "ul_prep_grouped")
HUBERT_OPS = ("conv", "layernorm", "eltwise", "hubert_conv0", "hubert_pos_conv", "transpose_heads", "attention")


class OpRecord:
    __slots__ = ("index", "op", "args", "inputs", "outputs", "plan")

    def __init__(self, index, op, args, inputs, outputs, plan):
        self.index, self.op, self.args, self.inputs, self.outputs, self.plan = index, op, args, inputs, outputs, plan

    def __repr__(self):
        return f"#{self.index} {self.op}"


def _io(op: str, a: dict):
    """The op's bound arguments -> ({input name: view}, {output name: view}) as DevTensors."""
    from livetalking_b200.ops import DevTensor as T
    if op == "conv":
        kw = a["kw"]
        x, out = a["x"], a["out"]
        if kw.get("in_ptr") is not None:
            x = T(kw["in_ptr"], x.shape, x.dtype, x.pitch, x.c_off)
        if kw.get("out_ptr") is not None:
            out = T(kw["out_ptr"], out.shape, out.dtype, out.pitch, out.c_off)
        ins = {"x": x}
        if kw.get("res") is not None:
            ins["res"] = kw["res"]
        if kw.get("group") is not None:
            ins["slot"] = kw["group"][0]
        return ins, {"out": out}
    if op == "dwconv3x3":
        ins = {"x": a["x"]}
        if a["group"] is not None:
            ins["slot"] = a["group"][0]
        return ins, {"out": a["out"]}
    if op == "upsample_bilinear2x":
        return {"x": a["x"]}, {"out": a["out"]}
    if op == "head_sigmoid255":
        ins = {"x": a["x"]}
        if a["group"] is not None:
            ins["slot"] = a["group"][0]
        return ins, {"pred": a["pred"]}
    if op == "ul_prep":
        return {"faces": a["faces_u8"], "index": a["d_index"]}, {"out": a["out"]}
    if op == "ul_prep_grouped":
        return {"groups": a["groups"]}, {"out": a["out"]}
    if op == "layernorm":
        return {"x": T(a["x"].ptr, (a["rows"], a["Cc"]))}, {"out": T(a["out"].ptr, (a["rows"], a["Cc"]))}
    if op == "eltwise":
        ins = {"x": T(a["x"].ptr, (a["n"],))}
        if a["y"] is not None:
            ins["y"] = T(a["y"].ptr, (a["period"],))
        return ins, {"out": T(a["out"].ptr, (a["n"],))}
    if op == "hubert_conv0":
        G, n = a["G"], a["n"]
        return ({"pcm": T(a["pcm"].ptr, (G, n), np.float32)},
                {"stats": T(a["stats"].ptr, (G, 4), np.float32), "out": T(a["out"].ptr, (G * ((n - 10) // 5 + 1), a["Cc"]))})
    if op == "hubert_pos_conv":
        rows = a["G"] * a["T"]
        return {"h": T(a["h"].ptr, (rows, a["D"]))}, {"out": T(a["out"].ptr, (rows, a["D"]))}
    if op == "transpose_heads":
        hd = a["heads"] * a["d"]
        return ({"v": T(a["v_ptr"], (a["B"] * a["n_keys"], hd), pitch=a["Ctot"])},
                {"vt": T(a["vt"].ptr, (a["B"] * a["heads"], a["d"], a["n_pad"]))})
    if op == "attention":
        hd, B = a["heads"] * a["d"], a["B"]
        out = a["out"]
        return ({"q": T(a["q_ptr"], (B * a["nq"], hd), pitch=a["q_pitch"]), "k": T(a["k_ptr"], (B * a["kv_rows"], hd), pitch=a["kv_pitch"]),
                 "vt": T(a["vt"].ptr, (B * a["heads"], a["d"], a["n_pad"]))},
                {"out": T(out.ptr, (B * a["nq"], hd), pitch=out.pitch, c_off=out.c_off)})
    raise ValueError(f"op_trace: no views defined for op {op!r}")


def _span(v):
    """(first byte, byte count) of the memory a view covers, from its first element to its last."""
    isz = v.dtype.itemsize
    return v.ptr + v.c_off * isz, ((v.rows - 1) * v.pitch + v.C) * isz


def _rows_of(buf: np.ndarray, off: int, v) -> np.ndarray:
    """Writable (rows, C * itemsize) byte view of `v` inside the byte array `buf` whose first byte is `off` bytes before v's first."""
    isz = v.dtype.itemsize
    need = off + ((v.rows - 1) * v.pitch + v.C) * isz
    assert off >= 0 and need <= buf.size, (off, need, buf.size)
    return np.lib.stride_tricks.as_strided(buf[off:], shape=(v.rows, v.C * isz), strides=(v.pitch * isz, 1))


def _dense(rows: np.ndarray, v) -> np.ndarray:
    return np.ascontiguousarray(rows).view(v.dtype).reshape(v.shape)


class OpTrace:
    """Trace the ops `ops` of `ctx` until stop().  records: OpRecord per call; errors: writes outside an output view."""

    def __init__(self, ctx, ops=UL_OPS + HUBERT_OPS, keep: Optional[Callable[[np.ndarray], np.ndarray]] = None):
        self.ctx, self.keep = ctx, keep or (lambda arr: arr)
        self.records: List[OpRecord] = []
        self.errors: List[str] = []
        self._allocs: Dict[int, int] = {}                  # ptr -> nbytes of the allocations made through ctx while tracing
        self._orig = {}
        self.active = True
        for name in dict.fromkeys(ops):
            self._wrap_op(name)
        alloc, free, capture = ctx.alloc, ctx.free, ctx.capture

        def traced_alloc(*args, **kw):
            t = alloc(*args, **kw)
            self._allocs[t.ptr] = t.nbytes
            return t

        def traced_free(t):
            self._allocs.pop(t.ptr, None)
            return free(t)

        def traced_capture(*args, **kw):
            self.stop()
            return capture(*args, **kw)

        for name, f in (("alloc", traced_alloc), ("free", traced_free), ("capture", traced_capture)):
            self._orig[name] = None
            setattr(ctx, name, f)

    def stop(self):
        """Restore the plain methods of the ctx; later ops are not traced."""
        if not self.active:
            return
        self.active = False
        for name in self._orig:
            delattr(self.ctx, name)

    def _wrap_op(self, name: str):
        orig = getattr(self.ctx, name)
        sig = inspect.signature(orig)

        def traced(*args, **kw):
            if not self.active:
                return orig(*args, **kw)
            bound = sig.bind(*args, **kw)
            bound.apply_defaults()
            self._record(name, dict(bound.arguments), lambda: orig(*args, **kw))

        self._orig[name] = orig
        setattr(self.ctx, name, traced)

    # ---- read-back without kernels
    def _read_bytes(self, ptr: int, nbytes: int) -> np.ndarray:
        from livetalking_b200.ops import DevTensor
        return self.ctx.download(DevTensor(ptr, (nbytes,), np.uint8))

    def _read_view(self, v) -> np.ndarray:
        start, n = _span(v)
        return _dense(_rows_of(self._read_bytes(start, n), 0, v), v)

    def _allocation(self, v):
        start, n = _span(v)
        for base, size in self._allocs.items():
            if base <= start and start + n <= base + size:
                return base, size
        return start, n

    def _record(self, name: str, args: dict, run):
        ctx = self.ctx
        ins, outs = _io(name, args)
        ctx.sync()
        inputs = {k: self.keep(self._read_view(v)) for k, v in ins.items()}
        plan = None
        if name == "conv":
            plan = ctx.conv_plan(args["x"], args["w"], args["out"], **args["kw"])
        before = {}
        for k, v in outs.items():
            base, size = self._allocation(v)
            before[k] = (base, size, self._read_bytes(base, size))
        run()
        ctx.sync()
        index = len(self.records)
        outputs = {}
        for k, v in outs.items():
            base, size, old = before[k]
            new = self._read_bytes(base, size)
            first = _span(v)[0] - base
            mask = np.zeros(size, bool)
            _rows_of(mask, first, v)[...] = True
            changed = (old != new) & ~mask
            if changed.any():
                at = int(np.argmax(changed))
                self.errors.append(f"#{index} {name}: {int(changed.sum())} bytes outside output {k!r} changed, first at byte {at} of "
                                   f"the {size}-byte allocation (the view starts at byte {first})")
            outputs[k] = self.keep(_dense(_rows_of(new, first, v), v))
        self.records.append(OpRecord(index, name, args, inputs, outputs, plan))
