"""GPU: every op of the Whisper-tiny feature path — log-mel, the encoder (WhisperEncoder.emit) and the per-frame
slicing — against float64, each op recomputed from the input the GPU read.

The test drives an eager pass on a fresh Ctx whose op methods are wrapped by `op_trace.OpTrace` (see
test_gpu_ultralight_layers.py): the tracer reads every op's inputs back before it runs, records the conv plan, and checks that
the op changed nothing in its output allocation outside the output view.  The weights are `synth.random_whisper_state_dict()`'s,
in the HF layout (conv1d [Cout, Cin, 3] evaluated as F.conv2d on [Cout, Cin, 1, 3], q/k/v/out/fc as [out, in]), rounded to fp16
as ConvWeight holds them.  Every op is checked on every row of every window:

  * conv / linear: the conv bound of test_gpu_ultralight_layers.py (tensor-core accumulation, epilogue adds, fp16 rounding,
    halo-residual and split-K terms).  The 1x3 convs run with N = G images of 1 x 3000, so F.conv2d's per-image zero padding
    is the per-window padding the encoder must apply;
  * GELU, LayerNorm: the bounds of test_gpu_ultralight_layers.py;
  * the positional add (eltwise with period T2 D): an fp32 add of two fp16 values and one fp16 rounding,
    |out - ref| <= 1.25 (v |ref| + u |ref| + 2^-25); the reference adds position rows 0..1499 to every window's rows;
  * attention: test_gpu_attention._reference, and the op must run with batch G (one window per batch entry);
  * transpose_heads and whisper_slice: bit-exact.  Frame i of window g takes steps clamp(int((i + start) 2) + j, 0, 1499),
    j < 10, from the five hidden states, step-major (row 5 j + layer), start = stride_left / 2 = 5;
  * whisper_logmel: the kernel runs the STFT (periodic Hann rounded to fp32, centre reflect padding of the zero-padded 30-s
    signal) and the Slaney mel sum in double, then log10f of the fp32 value, the per-window clamp max(v, max - 8) and
    (v + 4) / 4 in fp32, and rounds to fp16.  The float64 reference does the same with the same fp32 window.  With
    S = sum_j |frame_j| (the frame after windowing) the real and imaginary parts of bin k are each off by at most
    d = 420 2^-53 S (400 fmas, the rounded product and table terms), |re| + |im| <= sqrt 2 S, so the power is off by at most
    2 sqrt 2 S d + 2 d^2 + 3 2^-53 S^2 <= 1200 2^-53 S^2, and the mel value m by 201 2^-53 m + 1200 2^-53 S^2 sum_k fb[m, k];
    the fp32 rounding of m adds 2^-24 relative.  dlog = rel(m) / ln 10 + 2 ulp(log10f) per element.  An element that is surely
    below the clamp floor carries the floor's error (the dlog of the window's maximum + the fp32 rounding of max - 8), any
    other the larger of its own and the floor's; the fp32 add and divide add 2^-23 (|v| + 4) / 4; fp16 adds u |ref| + 2^-25.

Runs: g1_b8 (WhisperEncoder.emit, one window, B = 8 frames) and g4_b2 (emit over G = 4 windows: a tone, digital silence,
a window near full scale with clipped peaks, and a quiet one).  The Whisper path has no float atomics (the only atomic is the
integer atomicMax of the log-mel maximum), so WhisperFeatures.run / WhisperBatchFeatures.run_groups must reproduce the traced
features bit for bit."""
import math
import os
import sys
import time

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
from op_trace import WHISPER_OPS, OpTrace  # noqa: E402
from test_gpu_ultralight_layers import (SUB16, U16, V32, _bits, _conv_check, _conv_w, _gelu_check, _kernel,  # noqa: E402
                                        _ln_check, _ratio, _Report, _t64, _vt_as_v)

pytestmark = pytest.mark.gpu

STRIDE_L = STRIDE_R = 10
RUNS = {"g1_b8": (1, 8), "g4_b2": (4, 2)}
T_IN, T2, MELS, NFFT, HOP, NSAMP = 3000, 1500, 80, 400, 160, 480000


def _pcm(n, kind, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(n) / 16000.0
    x = 0.3 * np.sin(2 * np.pi * 230 * t) + 0.1 * np.sin(2 * np.pi * 1900 * t) + 0.05 * rng.standard_normal(n)
    if kind == "silence":
        x = np.zeros(n)
    elif kind == "full":
        x = np.clip(3.5 * x, -1.0, 1.0)
    elif kind == "quiet":
        x = 2e-4 * x
    return x.astype(np.float32)


# ------------------------------------------------------------------------------------------------ weights
class _WhisperWeights:
    def __init__(self, enc, sd):
        f = lambda k: np.asarray(sd["encoder." + k], np.float32)  # noqa: E731
        self.conv = {id(enc.conv1): ("conv1", lambda: _conv_w(f("conv1.weight")[:, :, None, :], f("conv1.bias"))),
                     id(enc.conv2): ("conv2", lambda: _conv_w(f("conv2.weight")[:, :, None, :], f("conv2.bias")))}
        self.norm = {id(enc.ln_post.gamma): "layer_norm"}
        D = enc.D
        for i, L in enumerate(enc.layers):
            p = f"layers.{i}"
            qkv = lambda p=p: _conv_w(np.concatenate([f(f"{p}.self_attn.{n}_proj.weight") for n in "qkv"])[:, :, None, None],  # noqa: E731
                                      np.concatenate([f(f"{p}.self_attn.q_proj.bias"), np.zeros(D, np.float32), f(f"{p}.self_attn.v_proj.bias")]))
            lin = lambda k, p=p: _conv_w(f(f"{p}.{k}.weight")[:, :, None, None], f(f"{p}.{k}.bias"))  # noqa: E731
            self.conv[id(L["attn"].qkv)] = (f"L{i} qkv", qkv)
            self.conv[id(L["attn"].out)] = (f"L{i} out_proj", lambda lin=lin: lin("self_attn.out_proj"))
            self.conv[id(L["fc1"])] = (f"L{i} fc1", lambda lin=lin: lin("fc1"))
            self.conv[id(L["fc2"])] = (f"L{i} fc2", lambda lin=lin: lin("fc2"))
            self.norm[id(L["ln1"].gamma)] = f"{p}.self_attn_layer_norm"
            self.norm[id(L["ln2"].gamma)] = f"{p}.final_layer_norm"
        self.f = f
        self.pos = f("embed_positions.weight").astype(np.float16)

    def norm_weights(self, gamma):
        p = self.norm[id(gamma)]
        return p, _t64(self.f(p + ".weight")), _t64(self.f(p + ".bias"))


# ------------------------------------------------------------------------------------------------ references
def _logmel_ref(pcm, fb):
    """-> (log10 mel power (80, 3000) float64, the error bound of that value per element) for one window."""
    n = pcm.size
    i = np.arange(NFFT)
    win = (0.5 - 0.5 * np.cos(np.pi * i / 200.0)).astype(np.float32).astype(np.float64)
    idx = HOP * np.arange(T_IN)[:, None] + i[None, :] - NFFT // 2
    idx = np.where(idx < 0, -idx, idx)
    idx = np.where(idx >= NSAMP, 2 * (NSAMP - 1) - idx, idx)
    x = np.where(idx < n, pcm.astype(np.float64)[np.minimum(idx, n - 1)], 0.0)
    fr = x * win[None, :]
    spec = np.fft.rfft(fr, axis=1)
    pw = spec.real ** 2 + spec.imag ** 2                       # (3000, 201)
    fbd = fb.astype(np.float64)
    mel = pw @ fbd.T                                           # (3000, 80)
    S = np.abs(fr).sum(1)[:, None]
    dmel = 201 * 2.0 ** -53 * mel + 1200 * 2.0 ** -53 * S ** 2 * fbd.sum(1)[None, :]
    m = np.maximum(mel, 1e-10)
    rel = np.where(mel > 1e-10, dmel / m, dmel / 1e-10) + 2.0 ** -24
    lg = np.log10(m)
    dlog = rel / math.log(10.0) + 2 * 2.0 ** -23 * np.abs(lg)
    return lg.T, dlog.T


def _logmel_check(rec, fb, rep):
    G, n = rec.args["G"], rec.args["n"]
    pcm = rec.inputs["pcm"]
    t_active = rec.outputs["logspec"].shape[-1]
    res_f16, res_log = [], []
    for g in range(G):
        lg, dlog = _logmel_ref(pcm[g], fb)
        got_log = rec.outputs["logspec"][g]
        r, info = _ratio(got_log, _t64(lg[:, :t_active]), _t64(dlog[:, :t_active]), f"logspec window {g}")
        res_log.append((r, f"window {g} {info}"))
        at = np.unravel_index(np.argmax(lg), lg.shape)
        floor = lg[at] - 8.0
        v = np.maximum(lg, floor)
        ref = (v + 4.0) / 4.0
        dfloor = dlog[at] + 2.0 ** -23 * abs(floor)
        dv = np.where(lg + dlog < floor - dfloor, dfloor, np.maximum(dlog, dfloor))
        bound = (dv + 2.0 ** -23 * (np.abs(v) + 4.0)) / 4.0 + U16 * np.abs(ref) + SUB16
        r, info = _ratio(rec.outputs["feats16"][g].T, _t64(ref), _t64(bound), f"feats16 window {g}")
        res_f16.append((r, f"window {g} {info}"))
        if "feats32" in rec.outputs:
            r, info = _ratio(rec.outputs["feats32"][g], _t64(ref), _t64(bound - U16 * np.abs(ref) - SUB16), f"feats32 window {g}")
            res_f16.append((r, f"window {g} feats32 {info}"))
    rep.add(f"#{rec.index:<3} whisper_logmel log10 mel (fp32)", *max(res_log, key=lambda t: t[0]))
    rep.add(f"#{rec.index:<3} whisper_logmel features", *max(res_f16, key=lambda t: t[0]))


def _pe_check(rec, pos, G):
    a = rec.args
    D = pos.shape[1]
    assert a["act"] == 0 and a["period"] == T2 * D and a["n"] == G * T2 * D, a
    x = rec.inputs["x"].astype(np.float64).reshape(G, T2, D)
    ref = x + pos.astype(np.float64)[None]                     # position rows 0..1499 in every window
    assert np.array_equal(_bits(rec.inputs["y"].reshape(T2, D)), _bits(pos)), "positional table read back differs"
    bound = (V32 + U16) * np.abs(ref) + SUB16
    return _ratio(rec.outputs["out"].reshape(G, T2, D), _t64(ref), _t64(bound), "positional add")


def _slice_want(hidden, G, B, start, out_rows=50):
    """hidden: 5 arrays (G*T2, D) -> (G*B, 50*D): frame i takes steps clamp(int((i + start) * 2) + j), j < 10, step-major."""
    D = hidden[0].shape[1]
    want = np.zeros((G, B, out_rows, D), np.float16)
    for g in range(G):
        for i in range(B):
            c = int((i + start) * 2)
            for j in range(10):
                s = min(max(c + j, 0), T2 - 1)
                for layer in range(5):
                    want[g, i, 5 * j + layer] = hidden[layer][g * T2 + s]
    return want.reshape(G * B, out_rows * D)


def _check_whisper(run, recs, W, G, B, fb):
    from test_gpu_attention import _reference
    rep = _Report(run)
    counts = {}
    for rec in recs:
        counts[rec.op] = counts.get(rec.op, 0) + 1
    nl = sum(1 for k in W.norm.values() if k.endswith(".final_layer_norm"))
    # conv1, conv2, per layer qkv / out / fc1 / fc2; GELU after both convs and every fc1, the positional add; LN 2 per layer + 1
    assert counts == {"whisper_logmel": 1, "conv": 2 + 4 * nl, "eltwise": 3 + nl, "layernorm": 2 * nl + 1, "transpose_heads": nl,
                      "attention": nl, "whisper_slice": 1}, counts
    t0 = time.time()
    n_pe = 0
    for rec in recs:
        op, a = rec.op, rec.args
        if op == "whisper_logmel":
            assert a["G"] == G
            _logmel_check(rec, fb, rep)
        elif op == "conv":
            name, build = W.conv[id(a["w"])]
            assert rec.plan["grouped"] == 0
            if name.startswith("conv"):
                assert a["kw"]["N"] == G and a["kw"]["IH"] == 1 and tuple(a["kw"]["pad"]) == (0, 1), a["kw"]
            r, info = _conv_check(rec, *build())
            rep.add(f"#{rec.index:<3} conv {name} [{_kernel(rec)}]", r, info)
        elif op == "layernorm":
            p, gamma, beta = W.norm_weights(a["gamma"])
            r, info = _ln_check(rec, gamma, beta)
            rep.add(f"#{rec.index:<3} layernorm {p}", r, info)
        elif op == "eltwise":
            if a["y"] is not None:
                n_pe += 1
                r, info = _pe_check(rec, W.pos, G)
                rep.add(f"#{rec.index:<3} positional add", r, info)
            else:
                r, info = _gelu_check(rec)
                rep.add(f"#{rec.index:<3} gelu", r, info)
        elif op == "transpose_heads":
            Bz, H, d, nk = a["B"], a["heads"], a["d"], a["n_pad"]
            vt = _vt_as_v(rec.outputs["vt"], Bz, H, d, nk)
            v = rec.inputs["v"].reshape(Bz, a["n_keys"], H, d)
            ok = np.array_equal(_bits(vt[:, :a["n_keys"]]), _bits(v)) and not _bits(vt[:, a["n_keys"]:]).any()
            rep.add(f"#{rec.index:<3} transpose_heads", 0.0 if ok else math.inf, "V^T is not V transposed with zero padding")
        elif op == "attention":
            Bz, H, d, nq, kv, valid = a["B"], a["heads"], a["d"], a["nq"], a["kv_rows"], a["valid"]
            assert (Bz, nq, kv, valid) == (G, T2, T2, T2), (Bz, nq, kv, valid)
            assert abs(a["scale"] - d ** -0.5) < 1e-12, a["scale"]
            Q = rec.inputs["q"].reshape(Bz, nq, H, d)
            K = rec.inputs["k"].reshape(Bz, kv, H, d)
            V = _vt_as_v(rec.inputs["vt"], Bz, H, d, a["n_pad"])
            ref, bound = _reference(Q, K, V, valid, a["scale"])
            r, info = _ratio(rec.outputs["out"].reshape(Bz, nq, H, d), _t64(ref), _t64(bound), "attention")
            rep.add(f"#{rec.index:<3} attention", r, info)
        else:
            assert op == "whisper_slice" and a["G"] == G and a["B"] == B and a["T"] == T2, a
            assert a["start"] == STRIDE_L / 2.0 and a["mult"] == 2.0, (a["start"], a["mult"])
            want = _slice_want([rec.inputs[f"h{i}"] for i in range(5)], G, B, STRIDE_L / 2.0)
            same = _bits(rec.outputs["out"]) == _bits(want)
            rep.add(f"#{rec.index:<3} whisper_slice", 0.0 if same.all() else math.inf, f"{int((~same).sum())} halves differ")
    assert n_pe == 1
    return rep, time.time() - t0


@pytest.fixture(scope="module")
def whisper():
    from livetalking_b200 import engine, synth
    from livetalking_b200.ops import Ctx
    from livetalking_b200.whisper import WhisperEncoder
    engine.set_device(0)
    ctx = Ctx()
    sd = synth.random_whisper_state_dict()
    enc = WhisperEncoder(ctx, sd)
    yield enc, sd
    ctx.close()


@pytest.mark.parametrize("run", list(RUNS))
def test_whisper_every_op_against_float64(whisper, run):
    """log-mel + WhisperEncoder.emit (G = 1 / G = 4) + whisper_slice traced eagerly, every op on every row against
    float64; WhisperFeatures / WhisperBatchFeatures must give the traced features bit for bit."""
    from livetalking_b200.graph import Builder
    from livetalking_b200.ops import Ctx
    from livetalking_b200.whisper import WhisperBatchFeatures, WhisperFeatures, slaney_mel_filterbank
    enc, sd = whisper
    G, B = RUNS[run]
    n = (STRIDE_L + STRIDE_R + 2 * B) * 320
    kinds = ["tone"] if G == 1 else ["tone", "silence", "full", "quiet"]
    pcms = np.stack([_pcm(n, k, seed=30 + g) for g, k in enumerate(kinds)])
    t0 = time.time()
    ctx = Ctx()
    tr = OpTrace(ctx, WHISPER_OPS)
    pcm = ctx.alloc((G, n), np.float32, zero=True)
    logspec = ctx.alloc((G, MELS * T_IN), np.float32, zero=True)
    gmax = ctx.alloc((G,), np.int32, zero=True)
    feats16 = ctx.alloc((G, T_IN, MELS), np.float16, zero=True)
    feats32 = ctx.alloc((G, MELS, T_IN), np.float32, zero=True) if G == 1 else None
    out = ctx.alloc((G, B, 50, enc.D), np.float16, zero=True)
    ctx.h2d(pcm, pcms)
    ctx.whisper_logmel(pcm, n, enc.fb, logspec, gmax, feats16, feats32, G=G)
    b = Builder(ctx)
    hidden = enc.emit(b, feats16, G=G)
    ctx.whisper_slice(hidden, T2, enc.D, B, STRIDE_L / 2.0, 2.0, out, 50, G=G)
    tr.stop()
    traced = ctx.download(out)
    assert not tr.errors, tr.errors[:5]
    t_gpu = time.time() - t0
    ctx.close()

    if G == 1:
        wf = WhisperFeatures(enc, B)
        prod = [wf.run(pcms[0])]
    else:
        wf = WhisperBatchFeatures(enc, B, G)
        prod = wf.run_groups(list(pcms))
    wf.close()
    for g in range(G):
        diff = _bits(prod[g]) != _bits(traced[g])
        assert not diff.any(), f"[{run}] window {g}: production features differ from the traced pass in {int(diff.sum())} values"

    rep, t_ref = _check_whisper(run, tr.records, _WhisperWeights(enc, sd), G, B, slaney_mel_filterbank())
    rep.finish(t_gpu, t_ref)
