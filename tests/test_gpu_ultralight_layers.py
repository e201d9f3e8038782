"""GPU: every op of the UltraLight leg — the UltraLight U-Net (single session and grouped across sessions) and HuBERT-large (one
window and G windows) — against float64, each op recomputed from the fp16 input the GPU read.

The test drives an eager pass itself on a fresh Ctx whose op methods are wrapped by `op_trace.OpTrace`: before every op the
tracer reads the op's inputs back, records which conv kernel the planner picked, and after it checks that the op changed no
byte of its output allocation outside the output view (so `upsample_bilinear2x` leaves the skip half of a concat buffer
alone and producers writing into `cat5` stay in their slice).  Each op is then recomputed in float64 with PyTorch in the
reference's own layout: `F.conv2d` on [Cout, Cin, k, k] (the depthwise convs on [C, 1, 3, 3], groups = C, evaluated as nine
shifted products), never the engine's packed layouts.
Conv weights are the BatchNorm-folded weights of `ultralight._fold` (HuBERT: the state_dict weights) rounded to fp16, the bias
fp32: what `ConvWeight` holds.  In a grouped run every image uses the weights of the network its group's bank slot holds.

Conv bound per output element, A = sum |w| |x| (a second float64 conv on absolute values), b the bias, r the residual,
pre = conv + b, ref = relu(pre (+ r)), u = 2^-11 (fp16), v = 2^-24 (fp32):

    |out - ref| <= 1.25 * ( eps_acc(K) A                     tensor-core accumulation over the op's K chain
                          + 3 v (A + |b| + |r|)              fp32 adds of bias and residual in the epilogue
                          + u |ref| + 2^-25                  the fp16 output rounding (normal / subnormal)
                          [+ u |pre| + 2^-25]                halo kernel with a residual (the pw2 of res=True blocks, HuBERT's
                                                             out_proj / fc2): it rounds fp16(acc + b) first and then adds the
                                                             residual in fp16 (conv_halo.cu, add_res)
                          [+ ks v (A + |b|)] )               gather kernel with split-K: the finalize sums the plan's ks fp32
                                                             partial slices onto the bias

  * eps_acc(K) = 18 ceil(K / 16) 2^-23, K = kh kw Cin (padded Cin).  Assumption, as in test_gpu_w2l_layers.py and not measured
    on the H100: each k16 wgmma step forms its 16 fp16 products exactly and adds them and the fp32 accumulator after aligning
    all 17 addends to the largest, truncating each aligned addend and the normalised result by at most one fp32 ulp.
  * 1.25 (SAFETY) absorbs the second-order terms the linearisation drops.

The other ops use the bounds of their kernel tests: depthwise 3x3, bilinear 2x and the sigmoid head those of
test_gpu_ultralight_ops.py, fused attention that of test_gpu_attention.py, conv0 and the positional conv those of
test_gpu_hubert_ops.py; `ul_prep` and `transpose_heads` are bit-exact.  LayerNorm (layernorm_kernel: one warp per row, lane
partial sums of L = 8 ceil(C / 256) values then a 5-level butterfly, mean = s / C, d = x - mean, rstd = rsqrtf(sum d^2 / C + eps),
out = fp16(d rstd gamma + beta)), with z = d rstd gamma:

    |out - ref| <= 1.25 * ( rstd |gamma| dm                  dm = (L + 5) v sum|x| / C + v |mean|: the fp32 mean
                          + ((L + 10) / 2 + 7) v |z|          variance sum, /C, + eps (relative, halved by the square root),
                                                             rsqrtf (2 ulp) and the roundings of d, d rstd and * gamma
                          + v |ref| + u |ref| + 2^-25 )      + beta, fp16 output

and eltwise GELU (gelu_erf: 0.5 x (1 + erff(x / sqrt 2)) in fp32) the GELU terms of the positional-conv bound:
0.5 |x| 2^-22 (erff's absolute error where 1 + erf cancels) + 2^-20 |gelu| (the fp32 products) + u |ref| + 2^-25.

Runs (the table of the module's RUNS and HUBERT_RUNS): the UltraLightSession plan at B = 16 as bench.py runs it, B = 3 (ragged
M tiles at 10x10 and 20x20, other split-K choices), an UltraLightBatchSession of 4 groups x 4 frames whose slot table holds
three networks, one slot twice and a network loaded after an eviction, HuBERT-large with the benchmark's 24-layer weights on a
B = 16 window (16640 samples, T = 51) and the same encoder over G = 3 windows of very different loudness.  The production graph
(UltraLightSession / UltraLightBatchSession / HubertFeatures / HubertBatchFeatures) must reproduce the traced pass bit for bit:
the only float atomics in csrc are in GroupNorm statistics paths neither network uses, and split-K writes per-split slices.
The U-Net runs also assert the routing the planner reports (the single-session `a3` on the halo kernel, every grouped 3x3 conv
on the gather kernel, `grouped` set on every grouped conv), that the padded hidden channels 12..15 of `inc` are exactly zero
after its pw1 and its depthwise conv, and at B = 16 that a depthwise and a bilinear op have more work items than the kernels'
grid cap, so their grid-stride loops take a second trip."""
import math
import os
import sys
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(__file__))
from op_trace import HUBERT_OPS, UL_OPS, OpTrace  # noqa: E402

pytestmark = pytest.mark.gpu

SAFETY = 1.25
U16 = 2.0 ** -11
SUB16 = 2.0 ** -25
V32 = 2.0 ** -24
ULP32 = 2.0 ** -23
GRID_ITEMS = 148 * 16 * 256          # the grid-stride cap of the depthwise / bilinear kernels (work items of 8 channels)
GATHER, HALO = 0, 1                  # ltb_conv_variant.kernel

# run -> (batch, first frame index, checked images): mirror_index(3, index + b) turns inside the batch
RUNS = {"b16": (16, 2, (0, 7, 15)), "b3": (3, 4, (0, 1, 2))}
GROUPS, FRAMES = 4, 4
# at least one image per group, the last image of the batch included; n % FRAMES and n // FRAMES name different slots for
# images 1, 6, 11 and 12, so a slot looked up with the wrong index shows
GROUP_IMAGES = (1, 6, 11, 12, 15)
HUBERT_RUNS = {"hubert_g1": 1, "hubert_g3": 3}


# ------------------------------------------------------------------------------------------------ inputs
def _faces():
    """One full-range random u8 crop and two smooth ones (168 x 168 BGR)."""
    rng = np.random.default_rng(160)
    rnd = rng.integers(0, 256, (168, 168, 3), dtype=np.uint8)
    rnd[4, 4], rnd[163, 163], rnd[5, 154], rnd[149, 5] = 255, 0, (255, 0, 255), (0, 255, 0)
    yy, xx = np.mgrid[0:168, 0:168] / 167.0
    smooth = []
    for k in range(2):
        ch = [127.5 + 127.5 * np.sin(2 * np.pi * ((1 + k) * yy + (0.5 + c) * xx) + c + k) for c in range(3)]
        smooth.append(np.clip(np.stack(ch, -1), 0, 255).round().astype(np.uint8))
    return [rnd] + smooth


def _feats(B, seed):
    """HuBERT windows (B, 16, 1024): randn x 3 with some entries at exactly +-8."""
    rng = np.random.default_rng(seed)
    f = (3 * rng.standard_normal((B, 16, 1024))).astype(np.float32)
    f[:, ::5, ::37] = 8.0
    f[:, 3::7, 11::53] = -8.0
    return f


def _pcm(n, kind, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(n) / 16000.0
    x = 0.3 * np.sin(2 * np.pi * 230 * t) + 0.1 * np.sin(2 * np.pi * 1900 * t) + 0.05 * rng.standard_normal(n)
    if kind == "quiet":
        # near-silent: digital silence around a short burst at 1e-3 of the tone.  The silent stretches reach conv0 as one constant,
        # so their conv-stack LayerNorm rows hold little more than the bias vector: a spread of ~0.02, where eps = 1e-5 matters.
        x = np.where(np.abs(t - t[n // 2]) < 0.05, 1e-3 * x, 0.0)
    elif kind == "full":
        x = np.clip(3.5 * x, -1.0, 1.0)                                   # full scale, clipped peaks
    return x.astype(np.float32)


# ------------------------------------------------------------------------------------------------ float64 weights
def _prefixes(model):
    """(block, state_dict prefix) for every InvertedResidual, in UltraLightModel.blocks() order."""
    a = "audio_model"
    names = [f"{a}.conv1", f"{a}.conv2", f"{a}.conv4", f"{a}.conv6", f"{a}.conv7"]
    names += [f"fuse_conv.{i}.double_conv.{j}" for i in range(2) for j in range(2)]
    names += ["inc.inconv.0"]
    names += [f"down{i + 1}.maxpool_conv.0.double_conv.{j}" for i in range(4) for j in range(2)]
    names += [f"up{i + 1}.conv.double_conv.{j}" for i in range(4) for j in range(2)]
    blocks = model.blocks()
    assert len(blocks) == len(names) == 26
    return list(zip(blocks, names))


def _t64(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64))


def _conv_w(w, b, cout_p=None, cin_p=None):
    """Folded weights -> (float64 [Cout, Cin, kh, kw] as fp16, float64 of the fp32 bias), zero-padded like ConvWeight."""
    w = np.asarray(w, np.float32)
    cout, cin = w.shape[:2]
    wp = np.zeros((cout_p or cout, cin_p or cin) + w.shape[2:], np.float32)
    wp[:cout, :cin] = w
    bp = np.zeros(cout_p or cout, np.float32)
    if b is not None:
        bp[:cout] = b
    return _t64(wp.astype(np.float16)), _t64(bp)


class _UlNet:
    """The float64 weights of one UltraLight network, by op name, and the names of the template's weight objects."""

    def __init__(self, model, sd):
        from livetalking_b200.ultralight import _fold
        from livetalking_b200.graph import _np
        self.model, self.w, self.names = model, {}, {}
        for blk, p in _prefixes(model):
            hid = int(_np(sd[p + ".conv.0.weight"]).shape[0])
            self.w[p + ".pw1"] = _conv_w(*_fold(sd, _np(sd[p + ".conv.0.weight"]), None, p + ".conv.1"), blk.hid_p, blk.inp_p)
            wd, bd = _fold(sd, _np(sd[p + ".conv.3.weight"]), None, p + ".conv.4")
            self.w[p + ".dw"] = _conv_w(wd, bd, blk.hid_p)
            self.w[p + ".pw2"] = _conv_w(*_fold(sd, _np(sd[p + ".conv.6.weight"]), None, p + ".conv.7"), None, blk.hid_p)
            self.names.update({id(blk.pw1): p + ".pw1", id(blk.dw_w): p + ".dw", id(blk.pw2): p + ".pw2"})
            assert hid <= blk.hid_p
        a = "audio_model"
        for k, cw in (("3", model.a3), ("5", model.a5)):
            self.w["a" + k] = _conv_w(*_fold(sd, _np(sd[f"{a}.conv{k}.weight"]), _np(sd[f"{a}.conv{k}.bias"]), f"{a}.bn{k}"))
            self.names[id(cw)] = "a" + k
        self.w["head"] = (_t64(_np(sd["outc.conv.weight"]).reshape(3, 32)), _t64(_np(sd["outc.conv.bias"])))
        self.names[id(model.head_w)] = "head"
        self.inc = "inc.inconv.0"

    def bank_names(self, bank):
        """Names of the bank buffers the grouped depthwise and head ops read (UltraLightBank.stacked of this template's tensors)."""
        out = {}
        for blk, p in _prefixes(self.model):
            out[id(bank.stacked(blk.dw_w))] = p + ".dw"
        out[id(bank.stacked(self.model.head_w))] = "head"
        return out


# ------------------------------------------------------------------------------------------------ per-op references
def _ratio(got, ref, bound, what):
    """-> (worst err / bound, description of the worst element); non-finite output fails at once."""
    got = torch.as_tensor(np.asarray(got, np.float64))
    assert torch.isfinite(got).all(), f"{what}: non-finite output"
    r = (got - ref).abs() / (SAFETY * bound)
    i = int(r.argmax())
    where = np.unravel_index(i, tuple(r.shape))
    return float(r.max()), f"{where}: got {float(got[where]):.6g} want {float(ref[where]):.6g} bound {SAFETY * float(bound[where]):.3g}"


def _nchw(a, *shape):
    return _t64(np.asarray(a).reshape(shape)).permute(0, 3, 1, 2)


def _conv_check(rec, w, b):
    """One conv (any kernel, grouped or not) against F.conv2d on its traced fp16 input; bound of the module docstring."""
    kw = rec.args["kw"]
    x, got = rec.inputs["x"], rec.outputs["out"]
    cout, cin, kh, kwid = w.shape
    assert x.shape[-1] == cin and got.shape[-1] == cout, (x.shape, got.shape, tuple(w.shape))
    stride, pad = tuple(kw.get("stride", (1, 1))), tuple(kw.get("pad", (0, 0)))
    if (kh, kwid, stride, pad) == (1, 1, (1, 1), (0, 0)):
        X = _nchw(x, 1, 1, -1, cin)                      # a 1x1 conv over all pixels: one image of 1 x rows
    else:
        X = _nchw(x, -1, kw["IH"], kw["IW"], cin)
    conv = F.conv2d(X, w, stride=stride, padding=pad).permute(0, 2, 3, 1).reshape(-1, cout)
    A = F.conv2d(X.abs(), w.abs(), stride=stride, padding=pad).permute(0, 2, 3, 1).reshape(-1, cout)
    bb = b[None, :]
    pre = conv + bb
    r = _t64(rec.inputs["res"]).reshape(-1, cout) if "res" in rec.inputs else torch.zeros_like(pre)
    ref = pre + r
    if kw.get("relu"):
        ref = torch.relu(ref)
    ref = ref.clamp(-65504, 65504)
    K = cin * kh * kwid
    bound = 18 * math.ceil(K / 16) * ULP32 * A + 3 * V32 * (A + bb.abs() + r.abs()) + U16 * ref.abs() + SUB16
    if rec.plan["kernel"] == HALO and "res" in rec.inputs:
        bound = bound + U16 * pre.abs() + SUB16
    if rec.plan["ksplit"] > 1:
        bound = bound + rec.plan["ksplit"] * V32 * (A + bb.abs())
    return _ratio(got.reshape(-1, cout), ref, bound, f"conv #{rec.index}")


def _depthwise(X, w, stride):
    """F.conv2d(X, w, stride, padding=1, groups=C) for w [C, 1, 3, 3], as the sum of nine shifted products (the same float64
    arithmetic; PyTorch's grouped float64 conv on the CPU is ~50x slower at 160 x 160 x 128)."""
    _n, _c, H, W = X.shape
    OH, OW = (H - 1) // stride + 1, (W - 1) // stride + 1
    cl = torch.channels_last
    Xp = F.pad(X, (1, 1, 1, 1)).contiguous(memory_format=cl)
    out = torch.zeros(X.shape[:2] + (OH, OW), dtype=X.dtype).contiguous(memory_format=cl)
    for ky in range(3):
        for kx in range(3):
            out.addcmul_(Xp[:, :, ky:ky + stride * (OH - 1) + 1:stride, kx:kx + stride * (OW - 1) + 1:stride], w[None, :, 0, ky, kx, None, None])
    return out


def _dw_check(rec, w, b, x=None, got=None):
    """depthwise 3x3 (pad 1): nine fmas onto the fp32 bias, 10 v (|b| + sum |x w|), fp16 rounding (test_gpu_ultralight_ops)."""
    a = rec.args
    x = rec.inputs["x"] if x is None else x
    got = rec.outputs["out"] if got is None else got
    C = x.shape[-1]
    X = _nchw(x, -1, a["IH"], a["IW"], C)
    conv = _depthwise(X, w, a["stride"]) + b[None, :, None, None]
    mag = _depthwise(X.abs(), w.abs(), a["stride"]) + b.abs()[None, :, None, None]
    ref = (torch.relu(conv) if a["relu"] else conv).clamp(-65504, 65504).permute(0, 2, 3, 1)
    bound = 10 * V32 * mag.permute(0, 2, 3, 1) + U16 * ref.abs() + SUB16
    return _ratio(got, ref, bound, f"dwconv3x3 #{rec.index}")


def _upsample_check(rec):
    """bilinear 2x, align_corners=True: coordinate rounding 2^-23 (H - 1) times the largest step 2M, the lerp 10 v M, fp16 rounding."""
    x, got = rec.inputs["x"], rec.outputs["out"]
    H, W = rec.args["H"], rec.args["W"]
    X = _nchw(x, -1, H, W, x.shape[-1])
    ref = F.interpolate(X, scale_factor=2, mode="bilinear", align_corners=True).permute(0, 2, 3, 1)
    M = X.abs().amax(dim=(2, 3))[:, None, None, :]
    bound = U16 * ref.abs() + SUB16 + (10 * V32 + 2.0 ** -22 * (H + W)) * M
    return _ratio(got, ref, bound, f"upsample #{rec.index}")


def _head_check(x, got, w, b):
    """255 sigmoid(b + x w^T): 33 fp32 fmas through sigmoid' <= 1/4, expf 2 ulp, the division and * 255 (test_gpu_ultralight_ops)."""
    xd = _t64(x).reshape(-1, 32)
    a = xd @ w.T + b
    sig = torch.sigmoid(a)
    mag = xd.abs() @ w.abs().T + b.abs()
    bound = 255 * (33 * V32 * mag / 4 + sig * (1 - sig) * 2.0 ** -22 + 2 * V32 * sig)
    return _ratio(np.asarray(got).reshape(-1, 3), 255 * sig, bound, "head")


def _prep_want(faces, nf, index, images):
    """ul_prep for the images `images` (positions counted from `index`), as test_gpu_ultralight_ops' bit-exact test builds it."""
    from oracle.paste_ref import mirror_index
    lut = (np.arange(256, dtype=np.float32) / np.float32(255)).astype(np.float16)
    want = np.zeros((len(images), 160, 160, 16), np.float16)
    for i, b in enumerate(images):
        crop = lut[faces[mirror_index(nf, index + b)][4:164, 4:164]]
        want[i, ..., 0:3] = crop
        want[i, ..., 3:6] = crop
        want[i, 5:150, 5:155, 3:6] = 0
    return want


def _bits(a):
    return np.ascontiguousarray(a).view({1: np.uint8, 2: np.uint16, 4: np.uint32}[a.dtype.itemsize])


class _Report:
    def __init__(self, run):
        self.run, self.rows, self.bad = run, [], []

    def add(self, label, worst, info):
        self.rows.append((label, worst))
        if worst > 1.0:
            self.bad.append(f"{label}: {worst:.2f} at {info}")

    def finish(self, t_gpu, t_ref):
        print(f"\n[{self.run}] traced pass + read-back {t_gpu:.1f} s, float64 references {t_ref:.1f} s, {len(self.rows)} checks")
        for label, worst in self.rows:
            print(f"  {label:<58} worst err/bound {worst:.3f}")
        top = max(self.rows, key=lambda r: r[1])
        print(f"  [{self.run}] largest err/bound {top[1]:.3f} at {top[0]}")
        assert not self.bad, f"[{self.run}] outside the bound: " + "; ".join(self.bad[:10])


def _kernel(rec):
    p = rec.plan
    if p["kernel"] == HALO:
        return f"halo taps{p['taps']}"
    return f"gather ks{p['ksplit']}" if p["ksplit"] > 1 else "gather"


# ------------------------------------------------------------------------------------------------ fixtures
@pytest.fixture(scope="module")
def ul():
    """Five UltraLight networks (network 0 has the benchmark's weights) and one avatar per network on one model ctx; avatars 0-2
    hold the test faces (nf = 3), the others smooth faces of their own."""
    from livetalking_b200 import engine, synth
    from livetalking_b200.ops import Ctx
    from livetalking_b200.ultralight import UltraLightAvatar, UltraLightModel
    engine.set_device(0)
    ctx = Ctx()
    faces = np.stack(_faces())
    frames = np.random.default_rng(5).integers(0, 256, (3, 64, 64, 3), dtype=np.uint8)
    nets, avs = [], []
    for k in range(5):
        sd = synth.random_ultralight_state_dict(seed=4 + k)
        m = UltraLightModel(ctx, sd)
        nets.append(_UlNet(m, sd))
        f = faces if k == 0 else np.roll(faces, 17 * k, axis=(1, 2))[::-1].copy()
        avs.append((UltraLightAvatar(ctx, m, frames, f, [(0, 0, 64, 64)] * 3), f))
    yield nets, avs
    ctx.close()


@pytest.fixture(scope="module")
def hubert():
    from livetalking_b200 import engine, synth
    from livetalking_b200.hubert import HubertEncoder
    from livetalking_b200.ops import Ctx
    engine.set_device(0)
    ctx = Ctx()
    sd = synth.random_hubert_state_dict()
    enc = HubertEncoder(ctx, sd)
    yield enc, sd
    ctx.close()


def _keep(B, imgs):
    idx = list(imgs)
    return lambda a: a[idx] if a.ndim >= 2 and a.shape[0] == B else a


# ------------------------------------------------------------------------------------------------ U-Net
def _check_unet(run, recs, net_of_image, names, imgs, B, prep_want, grouped):
    """Every traced U-Net op of `recs` against float64 (images `imgs`; net_of_image(n) -> that image's _UlNet)."""
    rep = _Report(run)
    counts = {}
    for rec in recs:
        counts[rec.op] = counts.get(rec.op, 0) + 1
    template = net_of_image(None)
    nblk = len(template.model.blocks())
    assert counts == {"ul_prep_grouped" if grouped else "ul_prep": 1, "conv": 2 * nblk + 2, "dwconv3x3": nblk, "upsample_bilinear2x": 4,
                      "head_sigmoid255": 1}, counts
    big_dw = big_up = False
    t0 = time.time()
    for rec in recs:
        op = rec.op
        if op in ("ul_prep", "ul_prep_grouped"):
            got = rec.outputs["out"]
            same = _bits(got) == _bits(prep_want)
            rep.add(f"#{rec.index:<3} {op}", 0.0 if same.all() else math.inf, f"{int((~same).sum())} halves differ")
            continue
        if op == "conv":
            name = names[id(rec.args["w"])]
            p = rec.plan
            assert p["grouped"] == int(grouped), (name, p)
            if grouped and rec.args["w"].kh == 3:
                assert p["kernel"] == GATHER, f"grouped 3x3 conv {name} on the halo kernel: {p}"
            if name == "a3":
                assert p["kernel"] == (GATHER if grouped else HALO), (run, p)
            worst, info = 0.0, ""
            for i, n in enumerate(imgs):     # the checked images may use different networks
                w, b = net_of_image(n).w[name]
                sub = _Sub(rec, i)
                r, inf = _conv_check(sub, w, b)
                if r >= worst:
                    worst, info = r, f"image {n} {inf}"
            rep.add(f"#{rec.index:<3} conv {name} [{_kernel(rec)}]", worst, info)
            if name == template.inc + ".pw1":
                assert not _bits(rec.outputs["out"][..., 12:]).any(), "inc: padded hidden channels 12..15 not zero after pw1"
            continue
        if op == "dwconv3x3":
            name = names[id(rec.args["w_tap"])]
            a = rec.args
            OH = (a["IH"] - 1) // a["stride"] + 1
            big_dw |= a["N"] * OH * OH * a["x"].C // 8 > GRID_ITEMS
            worst, info = 0.0, ""
            for i, n in enumerate(imgs):
                w, b = net_of_image(n).w[name]
                r, inf = _dw_check(rec, w.reshape(-1, 1, 3, 3), b, rec.inputs["x"][i:i + 1], rec.outputs["out"][i:i + 1])
                if r >= worst:
                    worst, info = r, f"image {n} {inf}"
            rep.add(f"#{rec.index:<3} dwconv3x3 {name} s{a['stride']}", worst, info)
            if name == template.inc + ".dw":
                assert not _bits(rec.outputs["out"][..., 12:]).any(), "inc: padded hidden channels 12..15 not zero after the depthwise conv"
            continue
        if op == "upsample_bilinear2x":
            a = rec.args
            big_up |= a["N"] * 4 * a["H"] * a["W"] * a["x"].C // 8 > GRID_ITEMS
            r, inf = _upsample_check(rec)
            rep.add(f"#{rec.index:<3} upsample_bilinear2x {a['H']}x{a['W']} C{a['x'].C}", r, inf)
            continue
        assert op == "head_sigmoid255", op
        assert names[id(rec.args["w3x32"])] == "head"
        worst, info = 0.0, ""
        for i, n in enumerate(imgs):
            w, b = net_of_image(n).w["head"]
            r, inf = _head_check(rec.inputs["x"][i], rec.outputs["pred"][i], w, b)
            if r >= worst:
                worst, info = r, f"image {n} {inf}"
        rep.add(f"#{rec.index:<3} head_sigmoid255", worst, info)
    if B == 16:   # the 160x160 depthwise / bilinear layers take a second trip through the grid-stride loop
        assert big_dw and big_up
    return rep, time.time() - t0


class _Sub:
    """The record restricted to the i-th kept image (inputs and outputs of a conv)."""

    def __init__(self, rec, i):
        self.index, self.args, self.plan = rec.index, rec.args, rec.plan
        self.inputs = {k: v[i:i + 1] for k, v in rec.inputs.items() if k in ("x", "res")}
        self.outputs = {"out": rec.outputs["out"][i:i + 1]}


@pytest.mark.parametrize("run", list(RUNS))
def test_unet_every_op_against_float64(ul, run):
    """UltraLightSession's op sequence (set_i32 + h2d + ul_prep + UltraLightModel.emit) traced eagerly; every op of the checked
    images against float64, and UltraLightSession.infer must give the traced pass's pred bit for bit."""
    from livetalking_b200.graph import Builder
    from livetalking_b200.ops import Ctx
    from livetalking_b200.ultralight import UltraLightSession
    nets, avs = ul
    B, index, imgs = RUNS[run]
    net = nets[0]
    av, faces = avs[0]
    feats = _feats(B, seed=B)
    t0 = time.time()
    ctx = Ctx()
    tr = OpTrace(ctx, UL_OPS, keep=_keep(B, imgs))
    d_index = ctx.alloc((4,), np.int32, zero=True)
    audio16 = ctx.alloc((B, 32, 32, 16), np.float16, zero=True)
    img16 = ctx.alloc((B, 160, 160, 16), np.float16, zero=True)
    pred = ctx.alloc((B, 160, 160, 3), np.float32, zero=True)
    ctx.set_i32(d_index, index)
    ctx.h2d(audio16, np.ascontiguousarray(feats.transpose(0, 2, 1)).astype(np.float16))
    ctx.ul_prep(av.faces, av.n, d_index, B, img16)
    net.model.emit(Builder(ctx), img16, audio16, pred)
    tr.stop()
    traced = ctx.download(pred)
    assert not tr.errors, tr.errors[:5]
    t_gpu = time.time() - t0
    ctx.close()

    sess = UltraLightSession(av, B)
    prod = sess.infer(index, feats)
    sess.close()
    diff = _bits(prod) != _bits(traced)
    assert not diff.any(), f"[{run}] production pred differs from the traced pass in {int(diff.sum())} values, first at {np.argwhere(diff)[0]}"

    rep, t_ref = _check_unet(run, tr.records, lambda n: net, net.names, imgs, B, _prep_want(faces, av.n, index, imgs), grouped=False)
    rep.finish(t_gpu, t_ref)


def test_grouped_unet_every_op_against_float64(ul):
    """UltraLightBatchSession(G = 4, Bs = 4) with a bank of 4 slots.  A first call loads networks 0-3; the checked call asks for
    networks [4, 1, 4, 2], so network 4 is loaded after evicting network 0 and the slot table is [0, 1, 0, 2]: three networks,
    one slot used by two groups.  The grouped op sequence (ul_prep_grouped + emit with the session's _Grouping) is traced
    eagerly over the session's bank and tables; every op of GROUP_IMAGES (each group's) against float64 with that image's network,
    and the session's pred (return_pred) must equal the traced pass's bit for bit."""
    from livetalking_b200.graph import Builder
    from livetalking_b200.ops import Ctx
    from livetalking_b200.ultralight import UltraLightBatchSession, _Grouping
    nets, avs = ul
    G, Bs = GROUPS, FRAMES
    B = G * Bs
    feats = [_feats(Bs, seed=70 + g) for g in range(G)]
    template = nets[0]
    s = UltraLightBatchSession(template.model, G, Bs, slots=G, return_pred=True)
    s.infer_groups([(avs[k][0], k, feats[k]) for k in range(G)])
    want_nets = [4, 1, 4, 2]
    requests = [(avs[k][0], 3 + 2 * g, feats[g]) for g, k in enumerate(want_nets)]
    prod = np.concatenate(s.infer_groups(requests))
    table = s.ctx.download(s.d_slot)
    assert s.bank.loads == 5 and table.tolist() == [0, 1, 0, 2], (s.bank.loads, table)
    by_model = {id(n.model): n for n in nets}
    slot_net = [by_model[id(s.bank._model[t])] for t in table]
    assert [nets.index(n) for n in slot_net] == want_nets

    t0 = time.time()
    ctx = Ctx()
    tr = OpTrace(ctx, UL_OPS, keep=_keep(B, GROUP_IMAGES))
    audio16 = ctx.alloc((B, 32, 32, 16), np.float16, zero=True)
    img16 = ctx.alloc((B, 160, 160, 16), np.float16, zero=True)
    pred = ctx.alloc((B, 160, 160, 3), np.float32, zero=True)
    ctx.h2d(audio16, np.ascontiguousarray(np.concatenate(feats).transpose(0, 2, 1)).astype(np.float16))
    ctx.ul_prep_grouped(s.d_prep, Bs, B, img16)
    template.model.emit(Builder(ctx), img16, audio16, pred, None, _Grouping(s.bank, s.d_slot, Bs))
    tr.stop()
    traced = ctx.download(pred)
    assert not tr.errors, tr.errors[:5]
    t_gpu = time.time() - t0
    ctx.close()
    s.close()
    diff = _bits(prod) != _bits(traced)
    assert not diff.any(), f"[grouped] production pred differs from the traced pass in {int(diff.sum())} values, first at {np.argwhere(diff)[0]}"

    names = dict(template.names)
    names.update(template.bank_names(s.bank))
    # image n of group g = n // Bs is frame n - g Bs of that group's request (avatar avs[want_nets[g]], first index 3 + 2 g)
    prep = np.concatenate([_prep_want(avs[want_nets[n // Bs]][1], 3, 3 + 2 * (n // Bs), [n % Bs]) for n in GROUP_IMAGES])
    rep, t_ref = _check_unet("grouped", tr.records, lambda n: template if n is None else slot_net[n // Bs], names, GROUP_IMAGES, B, prep,
                             grouped=True)
    rep.finish(t_gpu, t_ref)


# ------------------------------------------------------------------------------------------------ HuBERT
class _HubertWeights:
    """float64 references of the encoder's weights by weight object, built on demand from the state_dict."""

    def __init__(self, enc, sd):
        from livetalking_b200.hubert import CONV_KERNEL
        fe = "feature_extractor.conv_layers"
        f = lambda k: np.asarray(sd[k], np.float32)  # noqa: E731
        self.conv = {id(enc.convs[i - 1]): (f"conv{i}", lambda i=i: _conv_w(f(f"{fe}.{i}.conv.weight")[:, :, None, :], f(f"{fe}.{i}.conv.bias")))
                     for i in range(1, len(CONV_KERNEL))}
        self.conv[id(enc.proj)] = ("proj", lambda: _conv_w(f("feature_projection.projection.weight")[:, :, None, None],
                                                           f("feature_projection.projection.bias")))
        self.norm = {id(enc.conv_ln[i].gamma): f"{fe}.{i}.layer_norm" for i in range(len(CONV_KERNEL))}
        self.norm[id(enc.proj_ln.gamma)] = "feature_projection.layer_norm"
        self.norm[id(enc.ln_post.gamma)] = "encoder.layer_norm"
        for li, L in enumerate(enc.layers):
            p = f"encoder.layers.{li}"
            qkv = lambda p=p: _conv_w(np.concatenate([f(f"{p}.attention.{n}_proj.weight") for n in "qkv"])[:, :, None, None],  # noqa: E731
                                      np.concatenate([f(f"{p}.attention.{n}_proj.bias") for n in "qkv"]))
            lin = lambda k, p=p: _conv_w(f(f"{p}.{k}.weight")[:, :, None, None], f(f"{p}.{k}.bias"))  # noqa: E731
            self.conv[id(L["attn"].qkv)] = (f"L{li} qkv", qkv)
            self.conv[id(L["attn"].out)] = (f"L{li} out_proj", lambda lin=lin: lin("attention.out_proj"))
            self.conv[id(L["fc1"])] = (f"L{li} fc1", lambda lin=lin: lin("feed_forward.intermediate_dense"))
            self.conv[id(L["fc2"])] = (f"L{li} fc2", lambda lin=lin: lin("feed_forward.output_dense"))
            self.norm[id(L["ln1"].gamma)] = f"{p}.layer_norm"
            self.norm[id(L["ln2"].gamma)] = f"{p}.final_layer_norm"
        self.sd, self.f = sd, f

    def norm_weights(self, gamma):
        p = self.norm[id(gamma)]
        return p, _t64(self.f(p + ".weight")), _t64(self.f(p + ".bias"))

    def pos(self):
        """The positional conv's weight_norm weights in PyTorch layout [D, D/16, K] as the engine computes them (fp32), fp16."""
        pc = "encoder.pos_conv_embed.conv"
        g, v = self.f(f"{pc}.parametrizations.weight.original0"), self.f(f"{pc}.parametrizations.weight.original1")
        w = v * (g / np.sqrt((v.astype(np.float64) ** 2).sum((0, 1), keepdims=True))).astype(np.float32)
        return _t64(w.astype(np.float16)), _t64(self.f(f"{pc}.bias"))


def _gelu(v):
    return 0.5 * v * (1.0 + torch.special.erf(v / math.sqrt(2.0)))


def _ln_check(rec, gamma, beta):
    x = _t64(rec.inputs["x"])
    got = rec.outputs["out"]
    C = x.shape[1]
    L = 8 * math.ceil(C / 256)
    m = x.mean(1, keepdim=True)
    d = x - m
    eps = float(np.float32(rec.args["eps"]))
    rstd = 1.0 / torch.sqrt((d * d).mean(1, keepdim=True) + eps)
    z = d * rstd * gamma
    ref = z + beta
    dm = (L + 5) * V32 * x.abs().sum(1, keepdim=True) / C + V32 * m.abs()
    bound = rstd * gamma.abs() * dm + ((L + 10) / 2 + 7) * V32 * z.abs() + V32 * ref.abs() + U16 * ref.abs() + SUB16
    return _ratio(got, ref, bound, f"layernorm #{rec.index}")


def _gelu_check(rec):
    assert rec.args["act"] == 1 and rec.args["y"] is None, rec.args
    x = _t64(rec.inputs["x"])
    ref = _gelu(x)
    bound = 0.5 * x.abs() * 2.0 ** -22 + 2.0 ** -20 * ref.abs() + U16 * ref.abs() + SUB16
    return _ratio(rec.outputs["out"], ref, bound, f"gelu #{rec.index}")


def _conv0_check(rec, w, bias):
    """test_gpu_hubert_ops.test_conv0_matches_float64's statistics and output bounds, per window."""
    G, n = rec.args["G"], rec.args["n"]
    x = rec.inputs["pcm"].astype(np.float64)
    stats, out = rec.outputs["stats"], rec.outputs["out"]
    T0 = (n - 10) // 5 + 1
    mean = x.mean(1)
    ex2 = (x ** 2).mean(1)
    var = ((x - mean[:, None]) ** 2).mean(1)
    inv = 1.0 / np.sqrt(var + 1e-7)
    tol_m = 2.0 ** -24 * np.abs(mean) + n * 2.0 ** -53 * np.abs(x).mean(1)
    tol_i = inv * (2.0 ** -24 + (n + 2) * 2.0 ** -54 * ex2 / (var + 1e-7))
    res = [_ratio(stats[:, 0], _t64(mean), _t64(tol_m / SAFETY + 1e-300), "conv0 mean"),
           _ratio(stats[:, 1], _t64(inv), _t64(tol_i / SAFETY), "conv0 inv_std")]
    idx = 5 * np.arange(T0)[:, None] + np.arange(10)[None, :]
    wd, b = w.numpy(), bias.numpy()
    for g in range(G):
        xn = (x[g] - mean[g]) * inv[g]
        dxn = 2.0 ** -22 * inv[g] * (np.abs(x[g] - mean[g]) + abs(mean[g])) + np.abs(xn) * tol_i[g] / inv[g]
        ref = xn[idx] @ wd.T + b
        bound = dxn[idx] @ np.abs(wd).T + 10 * 2.0 ** -24 * (np.abs(b) + np.abs(xn[idx]) @ np.abs(wd).T) + U16 * np.abs(ref) + SUB16
        r, info = _ratio(out[g * T0:(g + 1) * T0], _t64(ref), _t64(bound), f"conv0 window {g}")
        res.append((r, f"window {g} {info}"))
    return max(res, key=lambda t: t[0])


def _pos_check(rec, w, b):
    """out = h + gelu(b + conv1d(h, padding 64, groups 16)[:T]) per window; test_gpu_hubert_ops.test_pos_conv_matches_float64's bound."""
    G, T, D, K = rec.args["G"], rec.args["T"], rec.args["D"], rec.args["K"]
    h, got = rec.inputs["h"], rec.outputs["out"]
    res = []
    for g in range(G):
        hd = _t64(h[g * T:(g + 1) * T])
        X = hd.T[None]
        conv = F.conv1d(X, w, padding=K // 2, groups=rec.args["groups"])[0, :, :T].T
        mag = F.conv1d(X.abs(), w.abs(), padding=K // 2, groups=rec.args["groups"])[0, :, :T].T
        pre = conv + b
        v = _gelu(pre)
        ref = hd + v
        bound = (1.13 * 8192 * V32 * (mag + b.abs()) + 0.5 * pre.abs() * 2.0 ** -22 + 2.0 ** -20 * v.abs() + V32 * ref.abs()
                 + U16 * ref.abs() + SUB16)
        r, info = _ratio(got[g * T:(g + 1) * T], ref, bound, f"pos_conv window {g}")
        res.append((r, f"window {g} {info}"))
    assert D == w.shape[0]
    return max(res, key=lambda t: t[0])


def _vt_as_v(vt, B, H, d, n_pad):
    """[B*H][d][n_pad] -> (B, n_pad, H, d)."""
    return vt.reshape(B, H, d, n_pad).transpose(0, 3, 1, 2)


def _check_hubert(run, recs, W, G, T):
    from test_gpu_attention import _reference
    rep = _Report(run)
    counts = {}
    for rec in recs:
        counts[rec.op] = counts.get(rec.op, 0) + 1
    nl = sum(1 for k in W.norm.values() if k.endswith(".final_layer_norm"))
    assert counts == {"hubert_conv0": 1, "conv": 7 + 4 * nl, "layernorm": 9 + 2 * nl, "eltwise": 7 + nl, "hubert_pos_conv": 1,
                      "transpose_heads": nl, "attention": nl}, counts
    t0 = time.time()
    last_ln = None
    for rec in recs:
        op = rec.op
        if op == "conv":
            name, build = W.conv[id(rec.args["w"])]
            assert rec.plan["grouped"] == 0
            r, info = _conv_check(rec, *build())
            rep.add(f"#{rec.index:<3} conv {name} [{_kernel(rec)}]", r, info)
        elif op == "layernorm":
            p, gamma, beta = W.norm_weights(rec.args["gamma"])
            r, info = _ln_check(rec, gamma, beta)
            last_ln = p
            rep.add(f"#{rec.index:<3} layernorm {p}", r, info)
        elif op == "eltwise":
            r, info = _gelu_check(rec)
            rep.add(f"#{rec.index:<3} gelu (after {last_ln})", r, info)
        elif op == "hubert_conv0":
            w = _t64(np.asarray(W.sd["feature_extractor.conv_layers.0.conv.weight"], np.float32).reshape(-1, 10))
            b = _t64(np.asarray(W.sd["feature_extractor.conv_layers.0.conv.bias"], np.float32))
            assert rec.args["G"] == G
            r, info = _conv0_check(rec, w, b)
            rep.add(f"#{rec.index:<3} hubert_conv0", r, info)
        elif op == "hubert_pos_conv":
            assert rec.args["G"] == G and rec.args["T"] == T
            r, info = _pos_check(rec, *W.pos())
            rep.add(f"#{rec.index:<3} hubert_pos_conv", r, info)
        elif op == "transpose_heads":
            a = rec.args
            B, H, d, nk = a["B"], a["heads"], a["d"], a["n_pad"]
            vt = _vt_as_v(rec.outputs["vt"], B, H, d, nk)
            v = rec.inputs["v"].reshape(B, a["n_keys"], H, d)
            ok = np.array_equal(_bits(vt[:, :a["n_keys"]]), _bits(v)) and not _bits(vt[:, a["n_keys"]:]).any()
            rep.add(f"#{rec.index:<3} transpose_heads", 0.0 if ok else math.inf, "V^T is not V transposed with zero padding")
        else:
            a = rec.args
            B, H, d, nq, kv, valid = a["B"], a["heads"], a["d"], a["nq"], a["kv_rows"], a["valid"]
            assert (B, nq, valid) == (G, T, T)
            Q = rec.inputs["q"].reshape(B, nq, H, d)
            K = rec.inputs["k"].reshape(B, kv, H, d)
            V = _vt_as_v(rec.inputs["vt"], B, H, d, a["n_pad"])
            ref, bound = _reference(Q, K, V, valid, a["scale"])
            r, info = _ratio(rec.outputs["out"].reshape(B, nq, H, d), _t64(ref), _t64(bound), "attention")
            rep.add(f"#{rec.index:<3} attention", r, info)
    return rep, time.time() - t0


@pytest.mark.parametrize("run", list(HUBERT_RUNS))
def test_hubert_every_op_against_float64(hubert, run):
    """HubertEncoder.emit with G = 1 / G = 3 over B = 16 windows traced eagerly, every op on every row against float64;
    the production graph (HubertFeatures / HubertBatchFeatures) must give the traced hidden states bit for bit."""
    from livetalking_b200.hubert import HubertBatchFeatures, HubertFeatures, window_samples
    from livetalking_b200.graph import Builder
    from livetalking_b200.ops import Ctx
    enc, sd = hubert
    G = HUBERT_RUNS[run]
    n, Tc, _T = window_samples(16, 10, 10)
    kinds = ["tone", "quiet", "full"][:G]
    pcms = np.stack([_pcm(n, k, seed=50 + g) for g, k in enumerate(kinds)])
    t0 = time.time()
    ctx = Ctx()
    tr = OpTrace(ctx, HUBERT_OPS)
    pcm = ctx.alloc((G, n), np.float32, zero=True)
    stats = ctx.alloc((G, 4), np.float32, zero=True)
    ctx.h2d(pcm, pcms)
    hidden = enc.emit(Builder(ctx), pcm, n, stats, G=G)
    tr.stop()
    traced = ctx.download(hidden)
    assert not tr.errors, tr.errors[:5]
    t_gpu = time.time() - t0
    ctx.close()
    assert traced.shape == (G * Tc, enc.D)

    if G == 1:
        hf = HubertFeatures(enc, 16)
        hf.run(pcms[0])
        prod = hf.hidden_states()
    else:
        hf = HubertBatchFeatures(enc, 16, G)
        hf.run_groups(list(pcms))
        prod = hf.ctx.download(hf.hidden)
    hf.close()
    diff = _bits(prod) != _bits(traced)
    assert not diff.any(), f"[{run}] production hidden states differ from the traced pass in {int(diff.sum())} values"

    rep, t_ref = _check_hubert(run, tr.records, _HubertWeights(enc, sd), G, Tc)
    rep.finish(t_gpu, t_ref)


def test_tracer_stops_at_capture():
    """Entering ctx.capture() restores the plain methods: the op inside the capture is not traced (no sync in a capture)."""
    from livetalking_b200 import engine
    from livetalking_b200.ops import Ctx
    engine.set_device(0)
    ctx = Ctx()
    tr = OpTrace(ctx, HUBERT_OPS)
    x = ctx.upload(np.linspace(-4, 4, 64).astype(np.float16))
    ctx.eltwise(x, None, 64, 64, 1, x)
    assert len(tr.records) == 1 and tr.active
    with ctx.capture() as cap:
        ctx.eltwise(x, None, 64, 64, 1, x)
    assert not tr.active and len(tr.records) == 1 and "eltwise" not in vars(ctx)
    cap.graph.launch()
    ctx.sync()
    cap.graph.close()
    ctx.close()


def test_tracer_checks_writes_outside_channel_slices():
    """copy_channels into a channel slice of a wider buffer is traced with a clean report and the data it wrote; when the tracer
    is handed a narrower output view than the op writes (an ordinary in-bounds write into the neighbouring channels of the same
    buffer), it reports the bytes outside the view."""
    from livetalking_b200 import engine
    from livetalking_b200.ops import Ctx, DevTensor
    from op_trace import MT_OPS
    engine.set_device(0)
    ctx = Ctx()
    tr = OpTrace(ctx, MT_OPS)
    src = ctx.upload((np.arange(7 * 16).reshape(7, 16) % 97).astype(np.float16))
    wide = ctx.alloc((7, 48), np.float16, zero=True)
    ctx.copy_channels(src, DevTensor(wide.ptr, (7, 16), pitch=48, c_off=16))
    assert not tr.errors, tr.errors
    rec = tr.records[0]
    assert rec.op == "copy_channels" and np.array_equal(_bits(rec.outputs["dst"]), _bits(rec.inputs["src"]))
    # the op copies src.C = 16 channels, the tracer is told the output is 8 channels wide
    ctx.copy_channels(src, DevTensor(wide.ptr, (7, 8), pitch=48, c_off=24))
    tr.stop()
    assert len(tr.errors) == 1 and "#1 copy_channels" in tr.errors[0] and "outside output 'dst'" in tr.errors[0], tr.errors
    ctx.close()
