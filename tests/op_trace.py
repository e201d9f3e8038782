"""Op tracer for the device-op layer: wraps the op methods of ONE ``livetalking_b200.ops.Ctx`` instance (instance attributes, the
class is untouched) so that an eager pass records every op it launches together with the data the op actually read and wrote.

For every traced call the tracer
  * syncs the stream and reads each input view back BEFORE the op runs, so an in-place op (eltwise GELU) is seen with its input;
  * for ``conv``, records ``ctx.conv_plan(...)`` with the same arguments: the kernel instance that ran;
  * reads the whole allocation under each output view before and after the op and records every byte outside the view that
    changed (an output whose allocation the tracer did not see being made is checked over the span of its view, pitch gaps
    included);
  * keeps the dense contents of the input and output views, passed through ``keep`` (e.g. to keep some images of a batch), or,
    with ``on_record``, hands each finished record to that callback and then drops its dense data (a traced full-width decoder
    would otherwise hold many GB of host copies);
  * with ``data=False`` records only the op sequence (arguments and conv plans): no sync and no read-back.
Channel-sliced views are read at full pitch and sliced on the host: no kernel runs for a read-back.  Ops that take raw pointers
(``attention``, ``transpose_heads``, ``softmax``, ...) get their views rebuilt from the pointer, pitch and row arguments.  A
z-batched conv (``w=None``, ``zbatch > 1``: the GEMMs of the unfused attention) has one view per z slice for its input, its
weight operand (activation data: K or V^T) and its output; the outside-write check of an allocation uses the union of every
output view that lies in it.  Entering ``ctx.capture()`` stops tracing (a sync inside stream capture is illegal); ``stop()``
restores the plain methods."""
from __future__ import annotations

import inspect
from typing import Callable, Dict, List, Optional

import numpy as np

UL_OPS = ("conv", "dwconv3x3", "upsample_bilinear2x", "head_sigmoid255", "ul_prep", "ul_prep_grouped")
HUBERT_OPS = ("conv", "layernorm", "eltwise", "hubert_conv0", "hubert_pos_conv", "transpose_heads", "attention")
MT_OPS = ("conv", "groupnorm", "groupnorm_apply", "layernorm", "geglu", "eltwise", "softmax", "copy_channels", "upsample2x",
          "transpose_heads", "attention", "vae_post", "vae_pre", "gather_rows")
WHISPER_OPS = ("conv", "layernorm", "eltwise", "transpose_heads", "attention", "softmax", "whisper_logmel", "whisper_slice")
WHISPER_FRAMES, WHISPER_MELS, WHISPER_HOP, WHISPER_NFFT = 3000, 80, 160, 400


class OpRecord:
    __slots__ = ("index", "op", "args", "inputs", "outputs", "plan")

    def __init__(self, index, op, args, inputs, outputs, plan):
        self.index, self.op, self.args, self.inputs, self.outputs, self.plan = index, op, args, inputs, outputs, plan

    def __repr__(self):
        return f"#{self.index} {self.op}"


def _zviews(v, ptr, n, zdiv, zo, zi, shape=None, pitch=None):
    """The n z slices of a z-batched conv operand: slice z starts (z // zdiv) zo + (z % zdiv) zi elements after ptr."""
    from livetalking_b200.ops import DevTensor as T
    return [T(ptr + ((z // zdiv) * zo + (z % zdiv) * zi) * 2, shape or v.shape, pitch=pitch or v.pitch, c_off=0 if shape else v.c_off)
            for z in range(n)]


def _io(op: str, a: dict):
    """The op's bound arguments -> ({input name: view}, {output name: view}) as DevTensors; a list of views (the z slices of a
    z-batched conv) is kept as one stacked array."""
    from livetalking_b200.ops import DevTensor as T
    if op == "conv" and a["w"] is None and a["kw"].get("zbatch", 0) > 1:
        kw = a["kw"]
        x, out, n, zdiv = a["x"], a["out"], kw["zbatch"], kw.get("zdiv", 1)
        cin, cout = kw["cin"], kw["cout"]
        assert kw.get("in_ptr") is None and kw.get("out_ptr") is None and kw.get("res") is None, "z-batched conv with extra pointers"
        return ({"x": _zviews(x, x.ptr + x.c_off * 2, n, zdiv, *kw["in_z"], shape=(x.rows, cin), pitch=x.pitch),
                 "w": _zviews(None, kw["w_ptr"], n, zdiv, *kw["w_z"], shape=(cout, cin), pitch=kw["ktot"])},
                {"out": _zviews(out, out.ptr + out.c_off * 2, n, zdiv, *kw["out_z"], shape=(out.rows, cout), pitch=out.pitch)})
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
    if op == "groupnorm":
        return {"x": a["x"]}, {"out": a["out"]}
    if op == "groupnorm_apply":
        st = a["stats"]
        return {"x": a["x"], "stats": T(st.ptr, (a["N"], a["groups"], 2), np.float32)}, {"out": a["out"]}
    if op == "geglu":
        rows, H = a["rows"], a["H"]
        return {"h": T(a["h"].ptr, (rows, 2 * H))}, {"out": T(a["out"].ptr, (rows, H))}
    if op == "softmax":                                    # in place: the input is read before the op runs
        v = T(a["x"].ptr, (a["rows"], a["cols"]))
        return {"x": v}, {"out": v}
    if op == "copy_channels":
        src, dst = a["src"], a["dst"]
        if a["rows"] is not None and a["rows"] != src.rows:
            src = T(src.ptr, (a["rows"], src.C), pitch=src.pitch, c_off=src.c_off)
            dst = T(dst.ptr, (a["rows"], dst.C), pitch=dst.pitch, c_off=dst.c_off)
        return {"src": src}, {"dst": dst}
    if op == "upsample2x":
        N, H, W, x = a["N"], a["H"], a["W"], a["x"]
        return {"x": T(x.ptr, (N, H, W, x.C))}, {"out": T(a["out"].ptr, (N, 2 * H, 2 * W, x.C))}
    if op == "vae_post":
        x, n = a["x"], a["npix"]
        return {"x": T(x.ptr, (n, 3), pitch=x.pitch)}, {"out": T(a["out_u8"].ptr, (n, 3), np.uint8)}
    if op == "vae_pre":
        N, H, W = a["N"], a["H"], a["W"]
        return {"img": T(a["img_u8"].ptr, (N, H, W, 3), np.uint8)}, {"out": T(a["out"].ptr, (N, H, W, 16))}
    if op == "gather_rows":
        n, B, r = a["n"], a["B"], a["row_elems"]
        return ({"table": T(a["table"].ptr, (n, r)), "index": T(a["d_index"].ptr, (1,), np.int32)},
                {"out": T(a["out"].ptr, (B, r))})
    if op == "whisper_logmel":
        G, n = a["G"], a["n"]
        t_active = min(WHISPER_FRAMES, (n + WHISPER_NFFT // 2 + WHISPER_HOP - 1) // WHISPER_HOP + 1)
        outs = {"feats16": T(a["feats16"].ptr, (G, WHISPER_FRAMES, WHISPER_MELS)),
                "logspec": T(a["logspec"].ptr, (G, WHISPER_MELS, t_active), np.float32),
                "gmax": T(a["gmax"].ptr, (G,), np.int32)}
        if a["feats32"] is not None:
            outs["feats32"] = T(a["feats32"].ptr, (G, WHISPER_MELS, WHISPER_FRAMES), np.float32)
        return {"pcm": T(a["pcm"].ptr, (G, n), np.float32)}, outs
    if op == "whisper_slice":
        G, T_, D, B, rows = a["G"], a["T"], a["D"], a["B"], a["out_rows"]
        ins = {f"h{i}": T(h.ptr, (G * T_, D)) for i, h in enumerate(a["hidden"])}
        return ins, {"out": T(a["out"].ptr, (G * B, 50 * D), pitch=rows * D)}
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

    def __init__(self, ctx, ops=UL_OPS + HUBERT_OPS, keep: Optional[Callable[[np.ndarray], np.ndarray]] = None,
                 on_record: Optional[Callable[[OpRecord], None]] = None, data: bool = True):
        self.ctx, self.keep = ctx, keep or (lambda arr: arr)
        self.on_record, self.data = on_record, data
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
        plan = None
        if name == "conv":
            kw = args["kw"]
            plan = ctx.conv_plan(args["x"], args["w"], args["out"], **kw)
        if not self.data:
            run()
            self.records.append(OpRecord(len(self.records), name, args, None, None, plan))
            return
        ins, outs = _io(name, args)
        ctx.sync()
        inputs = {k: (np.stack([self._read_view(u) for u in v]) if isinstance(v, list) else self.keep(self._read_view(v)))
                  for k, v in ins.items()}
        # every output view, grouped by the allocation it lies in: each allocation is read once before and once after
        views = [(k, u) for k, v in outs.items() for u in (v if isinstance(v, list) else [v])]
        allocs = {}
        for k, u in views:
            allocs.setdefault(self._allocation(u), []).append((k, u))
        before = {key: self._read_bytes(*key) for key in allocs}
        run()
        ctx.sync()
        index = len(self.records)
        dense = {}
        for (base, size), members in allocs.items():
            new = self._read_bytes(base, size)
            mask = np.zeros(size, bool)
            for k, u in members:
                first = _span(u)[0] - base
                _rows_of(mask, first, u)[...] = True
                dense.setdefault(k, []).append(_dense(_rows_of(new, first, u), u))
            changed = (before[(base, size)] != new) & ~mask
            if changed.any():
                at = int(np.argmax(changed))
                names = sorted({k for k, _ in members})
                self.errors.append(f"#{index} {name}: {int(changed.sum())} bytes outside output {'/'.join(names)!r} changed, first at "
                                   f"byte {at} of the {size}-byte allocation")
        outputs = {k: (np.stack(dense[k]) if isinstance(v, list) else self.keep(dense[k][0])) for k, v in outs.items()}
        rec = OpRecord(index, name, args, inputs, outputs, plan)
        if self.on_record is not None:
            self.on_record(rec)
            rec.inputs = rec.outputs = None
        self.records.append(rec)
