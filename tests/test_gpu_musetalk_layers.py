"""GPU: every op of the MuseTalk leg — the UNet, the VAE decoder and the VAE encoder — against float64, each op recomputed from
the fp16 input the GPU read.

An eager pass of MuseTalkSession's op sequence (gather_rows + positional add + emit_unet + emit_vae_decode) runs on a fresh Ctx
whose op methods are wrapped by `op_trace.OpTrace` (see test_gpu_ultralight_layers.py).  Each record is handed to the checks as
it is made and its data dropped, so a full-width batch-8 pass never holds more than one op's tensors.  References use the
layout of the reference architecture (oracle/musetalk_ref.py, diffusers keys), never the engine's packed layouts: F.conv2d on
[Cout, Cin, k, k]; attention on the unpadded head dim (the engine pads every head to a multiple of 16: 8 -> 16, 40 -> 48) with
scale d^-0.5 of that dim; the encoder's downsample as F.pad(x, (0, 1, 0, 1)) + a stride-2 conv; the fused upsample conv as
nearest 2x + a 3x3 conv.  Weights are the state_dict weights with musetalk.py's load-time rewrites redone in float64 (the t = 0
time embedding folded into conv1's bias, 1 / scaling_factor into post_quant_conv, scaling_factor into the quant conv's mean rows),
rounded to fp16 (biases to fp32) as ConvWeight holds them.

Bounds (u = 2^-11, v = 2^-24, each multiplied by SAFETY = 1.25 when checked):
  * conv / linear: the conv bound of test_gpu_ultralight_layers.py, K = kh kw Cin; the z-batched GEMMs of the unfused attention
    use K = padded head dim (Q K^T) or the padded key count (P V).  The fused upsample conv accumulates 4 sub-pixel taps
    (K = 4 Cin) whose pre-summed weights are rounded to fp16 once (ConvWeight.upconv): its reference uses the unrounded 3x3
    weights and the bound adds u A;
  * GroupNorm (+SiLU), gn_stats_kernel + gn_apply_kernel.  The fp32 sums of x and x^2 over a group run along chains of at most
    Ls = ceil(per / R) + 1 (one thread's pixels, pairs summed first) + 8 (the channel fold) + R ceil(cpg / 8 + 1) (shared-memory
    atomics) + splits (global atomics) additions, R / splits / per as launch_gn_stats picks them, so with n = HW cpg
        dm = Ls v sum|x| / n + v |m|,   dq = Ls v sum x^2 / n + v q,   dvar = dq + 2 |m| dm + v m^2 + v |var|
    (the E[x^2] - m^2 cancellation term is dq: it grows with m^2 / var), rstd relative error
    dr = dvar / (2 (var + eps)) + 2^-22 + v, pre-activation y = z gamma + beta off by
        dy = rstd |gamma| dm + |z gamma| dr + 3 v (|z gamma| + |beta| + |m rstd gamma|),
    SiLU (__expf, __fdividef) adds 1.1 dy + (4 + 2 |y|) 2^-23 |silu(y)|, then u |ref| + 2^-25.  Tightness rule: on these
    activations SAFETY times the bound may not exceed 8 fp16 ulps of |ref| + 1 at any element;
  * LayerNorm, GELU: the bounds of test_gpu_ultralight_layers.py;
  * GEGLU a gelu(g): |a| (0.5 |g| 2^-22 + 2^-20 |gelu(g)|) + v |ref| (the product) + u |ref| + 2^-25;
  * positional add: fp32 add of fp16 values and one fp16 rounding, v |ref| + u |ref| + 2^-25, plus the fp16 / fp32 rounding of
    the table against float64 sin / cos (u |pe| + 2^-18); the table is the reference's 50 rows, rows 50..63 zero;
  * softmax on fp16 scores s (unfused attention): p = e_j / sum e, e_j = __expf(scale s_j - max).  Relative error of p_j:
    v (|scale s_j| + |max|) (the scaling) + 2^-21 + 1.5 2^-23 |scale s_j - max| (ex2.approx and its argument) + cols v (the
    sum) + 2 v (reciprocal, product); then u p + 2^-25;
  * attention (fused): test_gpu_attention._reference;
  * bit-exact: vae_pre (oracle.musetalk_ref.preprocess_img), vae_post (test_gpu_ops' torch fp16 arithmetic), gather_rows
    (mirror index), copy_channels, upsample2x, transpose_heads.
Padding invariants, bit for bit zero: the head-padding columns of every qkv / q / kv output and of every attention output,
channels 4..31 of the UNet's conv_out, 4..15 of post_quant_conv, 3..31 of the decoder's conv_out (8..31 of the encoder's), and
V^T beyond the real keys.  Op counts per run are derived from the configs and state_dict keys.

Maps of more than 64 rows (the decoder's 128 x 128 and 256 x 256 levels at full width and in small_64) are checked on a 64-row
band at the top and one at the bottom, full width; GroupNorm statistics are always taken over the whole map.

Production: GroupNorm accumulates with float atomics, so the captured graph is not compared bit for bit.  (a) A data-free tracer
on the Ctx handed to MuseTalkSession records the session's own eager pass: its op names, shapes, scalar arguments and conv
plans must equal the traced pass's.  (b) infer() must be within 2 u8 steps and PSNR >= 55 dB of the traced image, and pred16
within PRED_TOL (absolute, on the 4 real channels) of the traced latents.  Measured on an H100 80 GB (default power limit): every
run, full_b8 included, at most 1 u8 step, PSNR 58.4-58.8 dB, pred16 within 0.0049 (full_b8: 1 step, 58.8 dB, 0.0039); the
GroupNorm bound reached at most 0.16 of the 8-ulp tightness limit."""
import math
import os
import sys
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(__file__))
from op_trace import MT_OPS, OpTrace  # noqa: E402
from test_gpu_ultralight_layers import (GATHER, HALO, SAFETY, SUB16, U16, ULP32, V32, _bits, _gelu, _gelu_check, _kernel,  # noqa: E402,F401
                                        _ln_check, _ratio, _Report, _t64, _vt_as_v)

pytestmark = pytest.mark.gpu

BAND = 64
PRED_TOL = 2e-2
# run -> (nets, B, latent size, avatar frames, first index, checked images, band large maps, fused attention)
RUNS = {"small_b2": ("small", 2, 32, 3, 4, (0, 1), False, True),        # mirror_index(3, 4..5) = 1, 0: the index turns
        "small_64": ("small", 1, 64, 3, 1, (0,), True, True),
        "small_unfused": ("small", 2, 32, 3, 4, (0,), False, False),
        "full_b8": ("full", 8, 32, 3, 2, (0, 7), True, True)}


# ------------------------------------------------------------------------------------------------ float64 weights
def _f64(t):
    return np.asarray(t.detach().cpu().double().numpy() if hasattr(t, "detach") else t, np.float64)


def _real_cols(H, d, dp, off=0):
    return np.array([off + h * dp + j for h in range(H) for j in range(d)])


class _Weights:
    """Per engine weight object: (name, float64 [Cout, Cin, kh, kw] rounded to fp16, float64 of the fp32 bias, input channel
    selection, output channel selection) in the reference layout; per norm gamma: (name, eps, silu, gamma, beta)."""

    def __init__(self, model, us, vs, ucfg, vcfg):
        self.conv, self.norm, self.attn = {}, {}, {}
        self.us, self.vs = us, vs
        boc, heads = ucfg.block_out_channels, ucfg.num_heads
        # t = 0 time embedding in float64 (diffusers get_timestep_embedding, flip_sin_to_cos: [cos 0] * half + [sin 0] * half)
        half = boc[0] // 2
        temb = np.concatenate([np.ones(half), np.zeros(half)])
        lin = lambda p, x: _f64(us[p + ".weight"]) @ x + _f64(us[p + ".bias"])  # noqa: E731
        silu = lambda x: x / (1 + np.exp(-x))  # noqa: E731
        self.ta = silu(lin("time_embedding.linear_2", silu(lin("time_embedding.linear_1", temb))))
        self._unet(model, us, ucfg, heads)
        self._vae(model, vs, vcfg)

    def _w(self, key, sd, obj, w, b, in_sel=None, out_sel=None, raw=False):
        w = np.asarray(w, np.float64)
        if w.ndim == 2:
            w = w[:, :, None, None]
        b = np.zeros(w.shape[0]) if b is None else np.asarray(b, np.float64)
        self.conv[id(obj)] = (key, _t64(w if raw else w.astype(np.float16)), _t64(b.astype(np.float32)), in_sel, out_sel)

    def _plain(self, sd, obj, p, **kw):
        self._w(p, sd, obj, _f64(sd[p + ".weight"]), _f64(sd[p + ".bias"]) if (p + ".bias") in sd else None, **kw)

    def _norm(self, sd, obj, p, eps, silu):
        self.norm[id(obj.gamma)] = (p, eps, silu, _t64(_f64(sd[p + ".weight"])), _t64(_f64(sd[p + ".bias"])))

    def _resnet(self, sd, r, p, eps, temb):
        self._norm(sd, r.norm1, p + ".norm1", eps, True)
        self._norm(sd, r.norm2, p + ".norm2", eps, True)
        b1 = _f64(sd[p + ".conv1.bias"])
        if temb:
            b1 = b1 + _f64(sd[p + ".time_emb_proj.weight"]) @ self.ta + _f64(sd[p + ".time_emb_proj.bias"])
        self._w(p + ".conv1", sd, r.conv1, _f64(sd[p + ".conv1.weight"]), b1)
        self._plain(sd, r.conv2, p + ".conv2")
        if r.shortcut is not None:
            self._plain(sd, r.shortcut, p + ".conv_shortcut")

    def _attn(self, sd, a, p):
        H, d, dp = a.heads, a.d, a.dp
        self.attn[id(a)] = (p, H, d, dp)
        g = lambda n: _f64(sd[f"{p}.{n}.weight"])  # noqa: E731
        gb = lambda n: _f64(sd[f"{p}.{n}.bias"]) if f"{p}.{n}.bias" in sd else np.zeros(H * d)  # noqa: E731
        if a.self_attn:
            self._w(p + ".to_qkv", sd, a.qkv, np.concatenate([g("to_q"), g("to_k"), g("to_v")]), np.concatenate([gb("to_q"), gb("to_k"), gb("to_v")]),
                    out_sel=np.concatenate([_real_cols(H, d, dp, k * H * dp) for k in range(3)]))
        else:
            self._w(p + ".to_q", sd, a.q, g("to_q"), gb("to_q"), out_sel=_real_cols(H, d, dp))
            self._w(p + ".to_kv", sd, a.kv, np.concatenate([g("to_k"), g("to_v")]), np.concatenate([gb("to_k"), gb("to_v")]),
                    out_sel=np.concatenate([_real_cols(H, d, dp, k * H * dp) for k in range(2)]))
        self._plain(sd, a.out, p + ".to_out.0", in_sel=_real_cols(H, d, dp))

    def _transformer(self, sd, t, p):
        self._norm(sd, t.norm, p + ".norm", 1e-6, False)
        self._plain(sd, t.proj_in, p + ".proj_in")
        self._plain(sd, t.proj_out, p + ".proj_out")
        b = p + ".transformer_blocks.0"
        self.ln = getattr(self, "ln", {})
        for i, n in enumerate((t.ln1, t.ln2, t.ln3)):
            self.ln[id(n.gamma)] = (f"{b}.norm{i + 1}", _t64(_f64(sd[f"{b}.norm{i + 1}.weight"])), _t64(_f64(sd[f"{b}.norm{i + 1}.bias"])))
        self._attn(sd, t.attn1, b + ".attn1")
        self._attn(sd, t.attn2, b + ".attn2")
        self._plain(sd, t.ff1, b + ".ff.net.0.proj")
        self._plain(sd, t.ff2, b + ".ff.net.2")

    def _unet(self, m, sd, cfg, heads):
        eps = cfg.norm_eps
        self._plain(sd, m.u_conv_in, "conv_in", in_sel=np.arange(cfg.in_channels))
        for i, blk in enumerate(m.u_down):
            for j, r in enumerate(blk["res"]):
                self._resnet(sd, r, f"down_blocks.{i}.resnets.{j}", eps, True)
            for j, t in enumerate(blk["attn"]):
                self._transformer(sd, t, f"down_blocks.{i}.attentions.{j}")
            if blk["down"] is not None:
                self._plain(sd, blk["down"], f"down_blocks.{i}.downsamplers.0.conv")
        self._resnet(sd, m.u_mid[0], "mid_block.resnets.0", eps, True)
        self._transformer(sd, m.u_mid[1], "mid_block.attentions.0")
        self._resnet(sd, m.u_mid[2], "mid_block.resnets.1", eps, True)
        for i, blk in enumerate(m.u_up):
            for j, r in enumerate(blk["res"]):
                self._resnet(sd, r, f"up_blocks.{i}.resnets.{j}", eps, True)
            for j, t in enumerate(blk["attn"]):
                self._transformer(sd, t, f"up_blocks.{i}.attentions.{j}")
            if blk["up"] is not None:
                self._plain(sd, blk["up"], f"up_blocks.{i}.upsamplers.0.conv")
                self.raw_up = getattr(self, "raw_up", {})
                self.raw_up[id(blk["up"])] = _t64(_f64(sd[f"up_blocks.{i}.upsamplers.0.conv.weight"]).astype(np.float32))
        self._norm(sd, m.u_norm_out, "conv_norm_out", eps, True)
        self._plain(sd, m.u_conv_out, "conv_out")

    def _vae_mid(self, sd, mid, p, eps):
        r0, gn, attn, r1 = mid
        self._resnet(sd, r0, p + ".resnets.0", eps, False)
        self._norm(sd, gn, p + ".attentions.0.group_norm", eps, False)
        self._attn(sd, attn, p + ".attentions.0")
        self._resnet(sd, r1, p + ".resnets.1", eps, False)

    def _vae(self, m, sd, cfg):
        eps, sf, L = cfg.norm_eps, cfg.scaling_factor, cfg.latent_channels
        self._w("post_quant_conv", sd, m.v_post_quant, _f64(sd["post_quant_conv.weight"]) / sf, _f64(sd["post_quant_conv.bias"]),
                in_sel=np.arange(L))
        self._plain(sd, m.v_dec_in, "decoder.conv_in", in_sel=np.arange(L))
        self._vae_mid(sd, m.v_dec_mid, "decoder.mid_block", eps)
        for i, blk in enumerate(m.v_dec_up):
            for j, r in enumerate(blk["res"]):
                self._resnet(sd, r, f"decoder.up_blocks.{i}.resnets.{j}", eps, False)
            if blk["up"] is not None:
                p = f"decoder.up_blocks.{i}.upsamplers.0.conv"
                self._plain(sd, blk["up"], p)
                self.raw_up = getattr(self, "raw_up", {})
                self.raw_up[id(blk["up"])] = _t64(_f64(sd[p + ".weight"]).astype(np.float32))
        self._norm(sd, m.v_dec_norm_out, "decoder.conv_norm_out", eps, True)
        self._plain(sd, m.v_dec_out, "decoder.conv_out")
        if m.with_encoder:
            self._plain(sd, m.v_enc_in, "encoder.conv_in", in_sel=np.arange(3))
            for i, blk in enumerate(m.v_enc_down):
                for j, r in enumerate(blk["res"]):
                    self._resnet(sd, r, f"encoder.down_blocks.{i}.resnets.{j}", eps, False)
                if blk["down"] is not None:
                    self._plain(sd, blk["down"], f"encoder.down_blocks.{i}.downsamplers.0.conv")
            self._vae_mid(sd, m.v_enc_mid, "encoder.mid_block", eps)
            self._norm(sd, m.v_enc_norm_out, "encoder.conv_norm_out", eps, True)
            self._plain(sd, m.v_enc_out, "encoder.conv_out")
            qw, qb = _f64(sd["quant_conv.weight"])[:L, :, 0, 0] * sf, _f64(sd["quant_conv.bias"])[:L] * sf
            for obj, lo in ((m.v_quant_masked, 0), (m.v_quant_ref, L)):
                w = np.zeros((16, 16))
                b = np.zeros(16)
                w[lo:lo + L, :2 * L] = qw
                b[lo:lo + L] = qb
                self._w("quant_conv[mean]" + (" ref" if lo else " masked"), sd, obj, w, b)


# ------------------------------------------------------------------------------------------------ per-op checks
def _band_rows(OH, band):
    return [(0, OH)] if not band or OH <= BAND else [(0, BAND), (OH - BAND, OH)]


def _conv_check(rec, W, band, imgs):
    """conv / linear (possibly banded); -> (worst, info, name, padded output channels)."""
    kw, a = rec.args["kw"], rec.args
    name, w, b, in_sel, out_sel = W.conv[id(a["w"])]
    x, got = rec.inputs["x"], rec.outputs["out"]
    res = rec.inputs.get("res")
    cout_e = got.shape[-1]
    up = bool(kw.get("upsample2x"))
    if up:
        w = W.raw_up[id(a["w"])]
    cout, cin, kh, kwid = w.shape
    cin_e = x.shape[-1]                                    # the engine's (padded) input channels: its K chain
    if in_sel is not None:
        x = x[..., in_sel]
    assert x.shape[-1] == cin, (name, x.shape, tuple(w.shape))
    stride, pad = tuple(kw.get("stride", (1, 1))), tuple(kw.get("pad", (0, 0)))
    linear = (kh, kwid) == (1, 1) and kw["IH"] == 1
    nimg = len(imgs)
    if linear:
        X = _t64(np.asarray(x).reshape(nimg, -1, cin)).permute(0, 2, 1)[:, :, None, :]
        gotv = np.asarray(got).reshape(nimg, 1, -1, cout_e)
        if res is not None:
            res = np.asarray(res).reshape(nimg, 1, -1, cout_e)
    else:
        X = _t64(np.asarray(x).reshape(nimg, kw["IH"], kw["IW"], cin)).permute(0, 3, 1, 2)
        gotv = np.asarray(got).reshape(nimg, kw["OH"], kw["OW"], cout_e)
        if res is not None:
            res = np.asarray(res).reshape(nimg, kw["OH"], kw["OW"], cout_e)
    if up:
        X = F.interpolate(X, scale_factor=2, mode="nearest")
    if kh == 3 and pad == (0, 0):                       # diffusers Downsample2D(padding=0): F.pad(x, (0, 1, 0, 1))
        Xp = F.pad(X, (0, 1, 0, 1))
    else:
        Xp = F.pad(X, (pad[1], pad[1], pad[0], pad[0]))
    OH = gotv.shape[1]
    K = 4 * cin_e if up else cin_e * kh * kwid
    worst, info = 0.0, ""
    sel = out_sel if out_sel is not None else np.arange(cout_e)[:cout]
    for r0, r1 in _band_rows(OH, band):
        Xb = Xp[:, :, r0 * stride[0]:(r1 - 1) * stride[0] + kh]
        conv = F.conv2d(Xb, w, stride=stride).permute(0, 2, 3, 1)
        A = F.conv2d(Xb.abs(), w.abs(), stride=stride).permute(0, 2, 3, 1)
        pre = conv + b
        r = _t64(res[:, r0:r1][..., sel]) if res is not None else torch.zeros_like(pre)
        ref = (pre + r).clamp(-65504, 65504)
        bound = 18 * math.ceil(K / 16) * ULP32 * A + 3 * V32 * (A + b.abs() + r.abs()) + U16 * ref.abs() + SUB16
        if up:
            bound = bound + U16 * A
        if rec.plan["kernel"] == HALO and res is not None:
            bound = bound + U16 * pre.abs() + SUB16
        if rec.plan["ksplit"] > 1:
            bound = bound + rec.plan["ksplit"] * V32 * (A + b.abs())
        rr, inf = _ratio(gotv[:, r0:r1][..., sel], ref, bound, f"conv {name}")
        if rr >= worst:
            worst, info = rr, f"rows {r0}..{r1} {inf}"
    pad_cols = np.setdiff1d(np.arange(cout_e), sel)
    return worst, info, name, (gotv[..., pad_cols] if pad_cols.size else None)


def _gn_launch(N, HW, C, groups):
    """R, splits and pixels per split of launch_gn_stats."""
    vpr = C // 8
    R = min(512 // vpr, HW)
    splits = min((592 + N - 1) // N, (HW + 4 * R - 1) // (4 * R))
    splits = max(splits, 1)
    return R, splits, (HW + splits - 1) // splits


def _gn_check(rec, W, band, nimg):
    a = rec.args
    name, eps, silu, gamma, beta = W.norm[id(a["gamma"])]
    x = _t64(rec.inputs["x"])
    got = rec.outputs["out"]
    N_all, HW, groups = a["N"], a["HW"], a["groups"]
    C = x.shape[-1]
    cpg = C // groups
    xg = x.reshape(nimg, HW, groups, cpg)
    n = HW * cpg
    m = xg.mean((1, 3), keepdim=True)
    q = (xg * xg).mean((1, 3), keepdim=True)
    var = ((xg - m) ** 2).mean((1, 3), keepdim=True)
    R, splits, per = _gn_launch(N_all, HW, C, groups)
    Ls = math.ceil(per / R) + 1 + 8 + R * math.ceil(cpg / 8 + 1) + splits
    dm = Ls * V32 * xg.abs().sum((1, 3), keepdim=True) / n + V32 * m.abs()
    dq = Ls * V32 * q + V32 * q
    dvar = dq + 2 * m.abs() * dm + V32 * m * m + V32 * var
    rstd = 1.0 / torch.sqrt(var + eps)
    dr = dvar / (2 * (var + eps)) + 2.0 ** -22 + V32
    g4, b4 = gamma.reshape(1, 1, groups, cpg), beta.reshape(1, 1, groups, cpg)
    zg = (xg - m) * rstd * g4
    y = zg + b4
    dy = rstd * g4.abs() * dm + zg.abs() * dr + 3 * V32 * (zg.abs() + b4.abs() + (m * rstd * g4).abs())
    if silu:
        sg = torch.sigmoid(y)
        ref = y * sg
        dy = 1.1 * dy + (4 + 2 * y.abs()) * 2.0 ** -23 * ref.abs()
    else:
        ref = y
    bound = (dy + U16 * ref.abs() + SUB16).reshape(nimg, HW, C)
    ref = ref.reshape(nimg, HW, C)
    r, info = _ratio(np.asarray(got).reshape(nimg, HW, C), ref, bound, f"groupnorm {name}")
    # tightness: the bound may not exceed 8 fp16 ulps of |ref| + 1
    mag = ref.abs() + 1
    ulp = torch.exp2(torch.floor(torch.log2(mag)) - 10)
    tight = float((SAFETY * bound / (8 * ulp)).max())
    assert tight <= 1.0, f"groupnorm {name}: the bound is {tight:.2f} x 8 fp16 ulps of |ref| + 1 (eps {eps})"
    return r, info, name, tight


def _softmax_check(rec, d_ref):
    a = rec.args
    x = _t64(rec.inputs["x"])
    got = rec.outputs["out"]
    valid, cols = a["valid"], a["cols"]
    scale = float(np.float32(d_ref ** -0.5))
    lg = x[:, :valid] * scale
    mx = lg.max(1, keepdim=True).values
    e = torch.exp(lg - mx)
    p = e / e.sum(1, keepdim=True)
    rel = V32 * (lg.abs() + mx.abs()) + 2.0 ** -21 + 1.5 * 2.0 ** -23 * (lg - mx).abs() + cols * V32 + 2 * V32
    bound = p * rel + U16 * p + SUB16
    r, info = _ratio(np.asarray(got)[:, :valid], p, bound, "softmax")
    pad_zero = not _bits(np.asarray(got)[:, valid:]).any()
    return r, info, pad_zero


def _zgemm_check(rec, kind, d, dp):
    """The z-batched GEMMs of the unfused attention: kind 'qk' S = Q K^T over the real head dims, 'pv' O = P V."""
    xs, ws, outs = _t64(rec.inputs["x"]), _t64(rec.inputs["w"]), rec.outputs["out"]
    if kind == "qk":
        Xr, Wr, K = xs[..., :d], ws[..., :d], dp
    else:
        Xr, Wr, K = xs, ws[:, :d], ws.shape[-1]
    ref = Xr @ Wr.transpose(1, 2)
    A = Xr.abs() @ Wr.abs().transpose(1, 2)
    bound = 18 * math.ceil(K / 16) * ULP32 * A + U16 * ref.abs() + SUB16
    got = np.asarray(outs)
    r, info = _ratio(got[..., :ref.shape[-1]], ref, bound, f"z-gemm {kind}")
    pad_zero = True if kind == "qk" else not _bits(got[..., d:]).any()
    return r, info, pad_zero


def _geglu_check(rec):
    h = _t64(rec.inputs["h"])
    H = h.shape[1] // 2
    av, g = h[:, :H], h[:, H:]
    gl = _gelu(g)
    ref = av * gl
    bound = av.abs() * (0.5 * g.abs() * 2.0 ** -22 + 2.0 ** -20 * gl.abs()) + V32 * ref.abs() + U16 * ref.abs() + SUB16
    return _ratio(rec.outputs["out"], ref, bound, "geglu")


def _pe_table(D):
    pos = np.arange(50, dtype=np.float64)[:, None]
    div = np.exp(np.arange(0, D, 2, dtype=np.float64) * (-math.log(10000.0) / D))
    pe = np.zeros((64, D))
    pe[:50, 0::2] = np.sin(pos * div)
    pe[:50, 1::2] = np.cos(pos * div)
    return pe


def _pe_check(rec, B):
    a = rec.args
    D = 384
    assert a["act"] == 0 and a["n"] == B * 64 * D
    x = np.asarray(rec.inputs["x"], np.float64).reshape(B, 64, D)
    pe = _pe_table(D)
    ref = x + pe[None]
    bound = (V32 + U16) * np.abs(ref) + SUB16 + U16 * np.abs(pe)[None] + 2.0 ** -18
    return _ratio(np.asarray(rec.outputs["out"]).reshape(B, 64, D), _t64(ref), _t64(bound), "positional add")


def _attn_check(rec, W, H, d, dp, imgs):
    from test_gpu_attention import _reference
    a = rec.args
    nimg = len(imgs)
    nq, kv, valid = a["nq"], a["kv_rows"], a["valid"]
    Q = np.asarray(rec.inputs["q"]).reshape(nimg, nq, H, dp)[..., :d]
    K = np.asarray(rec.inputs["k"]).reshape(nimg, kv, H, dp)[..., :d]
    V = _vt_as_v(np.asarray(rec.inputs["vt"]), nimg, H, dp, a["n_pad"])[..., :d]
    ref, bound = _reference(Q, K, V, valid, float(d) ** -0.5)
    got = np.asarray(rec.outputs["out"]).reshape(nimg, nq, H, dp)
    r, info = _ratio(got[..., :d], _t64(ref), _t64(bound), "attention")
    return r, info, not _bits(got[..., d:]).any()


def _keep(B, imgs):
    """Keep the checked images of any array whose leading dimension is a multiple of B (image-major rows)."""
    idx = list(imgs)
    if len(idx) == B:
        return None

    def keep(arr):
        if arr.ndim >= 2 and arr.shape[0] % B == 0:
            return arr.reshape((B, arr.shape[0] // B) + arr.shape[1:])[idx].reshape((len(idx) * (arr.shape[0] // B),) + arr.shape[1:])
        return arr
    return keep


class _Checker:
    """on_record callback: checks every record against float64 as the tracer makes it."""

    def __init__(self, run, W, B, imgs, band, model):
        self.rep, self.W, self.B, self.imgs, self.band = _Report(run), W, B, imgs, band
        self.t = 0.0
        self.counts = {}
        self.tight = 0.0
        self.attn_of_qkv = {}
        self.cur_attn = None
        self.model = model
        self.pads = []
        self.zgemms = 0

    def __call__(self, rec):
        t0 = time.time()
        op, a = rec.op, rec.args
        self.counts[op] = self.counts.get(op, 0) + 1
        nimg = len(self.imgs)
        label = f"#{rec.index:<3} {op}"
        if op == "conv" and a["w"] is None:
            p, H, d, dp = self.cur_attn
            kind = "pv" if self.zgemms % 2 else "qk"           # Q K^T, softmax, transpose_heads, P V
            self.zgemms += 1
            assert a["kw"]["zdiv"] == H and a["kw"]["zbatch"] == self.B * H, a["kw"]
            r, info, ok = _zgemm_check(rec, kind, d, dp)
            self.rep.add(f"{label} {p} {'Q K^T' if kind == 'qk' else 'P V'} [{_kernel(rec)}]", r, info)
            assert ok, f"{p}: padded head columns of the P V output are not zero"
        elif op == "conv":
            r, info, name, padded = _conv_check(rec, self.W, self.band, self.imgs)
            self.rep.add(f"{label} {name} [{_kernel(rec)}]", r, info)
            if padded is not None:
                assert not _bits(np.ascontiguousarray(padded)).any(), f"{name}: padded output channels are not zero"
                self.pads.append(name)
            key = id(a["w"])
            if key in self.attn_of_qkv:
                self.cur_attn = self.attn_of_qkv[key]
        elif op in ("groupnorm", "groupnorm_apply"):
            r, info, name, tight = _gn_check(rec, self.W, self.band, nimg)
            self.tight = max(self.tight, tight)
            self.rep.add(f"{label} {name}", r, info)
        elif op == "layernorm":
            p, gamma, beta = self.W.ln[id(a["gamma"])]
            assert a["eps"] == 1e-5
            r, info = _ln_check(rec, gamma, beta)
            self.rep.add(f"{label} {p}", r, info)
        elif op == "geglu":
            self.rep.add(label, *_geglu_check(rec))
        elif op == "eltwise":
            assert a["y"] is not None and a["period"] % 384 == 0, "the MuseTalk graph's only eltwise is the positional add"
            self.rep.add(f"{label} positional add", *_pe_check(rec, self.B))
        elif op == "softmax":
            p, H, d, dp = self.cur_attn
            r, info, ok = _softmax_check(rec, d)
            assert ok, f"{p}: softmax padded key columns are not zero"
            self.rep.add(f"{label} {p}", r, info)
        elif op == "transpose_heads":
            Bz, H, d, nk = nimg, a["heads"], a["d"], a["n_pad"]
            vt = _vt_as_v(np.asarray(rec.outputs["vt"]), Bz, H, d, nk)
            v = np.asarray(rec.inputs["v"]).reshape(Bz, a["n_keys"], H, d)
            ok = np.array_equal(_bits(vt[:, :a["n_keys"]]), _bits(v)) and not _bits(vt[:, a["n_keys"]:]).any()
            self.rep.add(label, 0.0 if ok else math.inf, "V^T is not V transposed with zero keys beyond the real ones")
        elif op == "attention":
            p, H, d, dp = self.cur_attn
            assert a["heads"] == H and a["d"] == dp
            if p.endswith("attn2"):
                assert a["valid"] == 50 and a["kv_rows"] == 64 and a["n_pad"] == 64, a
            r, info, ok = _attn_check(rec, self.W, H, d, dp, self.imgs)
            assert ok, f"{p}: padded head columns of the attention output are not zero"
            self.rep.add(f"{label} {p}", r, info)
        elif op == "copy_channels":
            ok = np.array_equal(_bits(rec.outputs["dst"]), _bits(rec.inputs["src"]))
            self.rep.add(label, 0.0 if ok else math.inf, "concat copy differs")
        elif op == "upsample2x":
            x = torch.from_numpy(np.asarray(rec.inputs["x"]).astype(np.float32)).permute(0, 3, 1, 2)
            want = F.interpolate(x, scale_factor=2, mode="nearest").permute(0, 2, 3, 1).numpy().astype(np.float16)
            ok = np.array_equal(_bits(rec.outputs["out"]), _bits(want))
            self.rep.add(label, 0.0 if ok else math.inf, "nearest 2x differs")
        elif op == "gather_rows":
            from oracle.paste_ref import mirror_index
            table, index = rec.inputs["table"], int(rec.inputs["index"][0])
            want = np.stack([table[mirror_index(a["n"], index + i)] for i in self.imgs])
            ok = np.array_equal(_bits(rec.outputs["out"]), _bits(want))
            self.rep.add(label, 0.0 if ok else math.inf, "gathered latents differ")
        elif op == "vae_post":
            rgb = np.asarray(rec.inputs["x"])
            t = (torch.from_numpy(rgb) / 2 + 0.5).clamp(0, 1).float().numpy()
            want = np.round(t * np.float32(255)).astype(np.uint8)[:, ::-1]
            ok = np.array_equal(rec.outputs["out"], want)
            self.rep.add(label, 0.0 if ok else math.inf, f"{int((rec.outputs['out'] != want).sum())} bytes differ")
        elif op == "vae_pre":
            from oracle.musetalk_ref import preprocess_img
            img = rec.inputs["img"]
            want = np.zeros(img.shape[:3] + (16,), np.float16)
            for i in range(img.shape[0]):
                want[i, ..., :3] = preprocess_img(img[i], bool(a["half_mask"])).half()[0].permute(1, 2, 0).numpy()
            ok = np.array_equal(_bits(rec.outputs["out"]), _bits(want))
            self.rep.add(f"{label} {'masked' if a['half_mask'] else 'full'}", 0.0 if ok else math.inf, "preprocessed image differs")
        else:
            raise AssertionError(f"unexpected op {op}")
        self.t += time.time() - t0


def _attn_objects(model):
    """(UNet or decoder, attention block) for every attention block of the UNet and the VAE decoder."""
    blocks = []
    for blk in model.u_down + model.u_up:
        blocks += blk.get("attn", [])
    blocks.append(model.u_mid[1])
    return [("unet", a) for t in blocks for a in (t.attn1, t.attn2)] + [("vae", model.v_dec_mid[2])]


def _register_attn(chk, W, model):
    """The qkv / q weights that start each attention block -> (name, heads, d, dp) of that block."""
    attns = [a for _k, a in _attn_objects(model)] + ([model.v_enc_mid[2]] if model.with_encoder else [])
    for a in attns:
        p, H, d, dp = W.attn[id(a)]
        chk.attn_of_qkv[id(a.qkv if a.self_attn else a.q)] = (p, H, d, dp)


def _expected_counts(model, us, vs, ucfg, vcfg, fused, decode=True, encode=False):
    from livetalking_b200.graph import Builder
    c = {}

    def add(op, k=1):
        c[op] = c.get(op, 0) + k

    def resnet(sd, p):
        add("groupnorm", 2)
        add("conv", 2 + int(p + ".conv_shortcut.weight" in sd))

    def attention(a, cross):
        add("conv", 2 + int(cross))                            # qkv (q and kv) and out
        if fused and a.dp % 16 == 0 and a.dp <= 160:
            add("transpose_heads")
            add("attention")
        else:
            add("conv", 2)
            add("softmax")
            add("transpose_heads")

    def transformer(t):
        add("groupnorm")
        add("conv", 4)                                         # proj_in, ff1, ff2, proj_out
        add("layernorm", 3)
        add("geglu")
        attention(t.attn1, False)
        attention(t.attn2, True)

    def upsampler(w):
        add("conv")
        if not (Builder.FUSE_UPSAMPLE and w.upconv_supported()):
            add("upsample2x")

    if not encode:
        add("gather_rows")
        add("eltwise")
        boc, L = ucfg.block_out_channels, ucfg.layers_per_block
        add("conv")                                            # conv_in
        for i in range(len(boc)):
            for j in range(L):
                resnet(us, f"down_blocks.{i}.resnets.{j}")
                if ucfg.down_has_attn[i]:
                    transformer(model.u_down[i]["attn"][j])
            if i < len(boc) - 1:
                add("conv")
        resnet(us, "mid_block.resnets.0")
        transformer(model.u_mid[1])
        resnet(us, "mid_block.resnets.1")
        for i in range(len(boc)):
            for j in range(L + 1):
                add("copy_channels", 2)
                resnet(us, f"up_blocks.{i}.resnets.{j}")
                if ucfg.up_has_attn[i]:
                    transformer(model.u_up[i]["attn"][j])
            if i < len(boc) - 1:
                upsampler(model.u_up[i]["up"])
        add("groupnorm")
        add("conv")
    vb, L = vcfg.block_out_channels, vcfg.layers_per_block

    def vmid(p, mid):
        resnet(vs, p + ".resnets.0")
        add("groupnorm")
        attention(mid[2], False)
        resnet(vs, p + ".resnets.1")

    if decode:
        add("conv", 2)                                         # post_quant_conv, conv_in
        vmid("decoder.mid_block", model.v_dec_mid)
        for i in range(len(vb)):
            for j in range(L + 1):
                resnet(vs, f"decoder.up_blocks.{i}.resnets.{j}")
            if i < len(vb) - 1:
                upsampler(model.v_dec_up[i]["up"])
        add("groupnorm")
        add("conv")
        add("vae_post")
    if encode:
        add("vae_pre", 2)
        add("conv")
        for i in range(len(vb)):
            for j in range(L):
                resnet(vs, f"encoder.down_blocks.{i}.resnets.{j}")
            if i < len(vb) - 1:
                add("conv")
        vmid("encoder.mid_block", model.v_enc_mid)
        add("groupnorm")
        add("conv", 3)                                         # conv_out, the two quant convs
    return c


def _sig(rec):
    """An op's name, shapes, scalar arguments and conv plan (no pointers)."""
    from livetalking_b200.ops import DevTensor

    def s(v):
        if isinstance(v, DevTensor):
            return ("T", v.shape, v.dtype.str, v.pitch, v.c_off)
        if isinstance(v, dict):
            return tuple((k, s(x)) for k, x in sorted(v.items()) if not k.endswith("_ptr"))
        if isinstance(v, (list, tuple)):
            return tuple(s(x) for x in v)
        if isinstance(v, (bool, int, float, str)) or v is None:
            return v
        return ("obj", id(v))
    args = tuple((k, s(v)) for k, v in rec.args.items() if not k.endswith("_ptr"))
    return rec.op, args, tuple(sorted(rec.plan.items())) if rec.plan else None


# ------------------------------------------------------------------------------------------------ fixtures
@pytest.fixture(scope="module")
def small():
    from livetalking_b200 import engine
    from livetalking_b200.musetalk import MuseTalkModel
    from livetalking_b200.ops import Ctx
    from oracle import musetalk_ref as M
    engine.set_device(0)
    us, vs = M.synth_unet_state_dict(M.UNET_SMALL), M.synth_vae_state_dict(M.VAE_SMALL)
    ctx = Ctx()
    model = MuseTalkModel(ctx, us, vs, M.UNET_SMALL, M.VAE_SMALL)
    yield model, us, vs, M.UNET_SMALL, M.VAE_SMALL, _Weights(model, us, vs, M.UNET_SMALL, M.VAE_SMALL)
    ctx.close()


@pytest.fixture(scope="module")
def full():
    from livetalking_b200 import engine
    from livetalking_b200.musetalk import MuseTalkModel
    from livetalking_b200.ops import Ctx
    from oracle import musetalk_ref as M
    engine.set_device(0)
    us = M.synth_unet_state_dict(M.UNET_FULL, fast=True)
    vs = M.synth_vae_state_dict(M.VAE_FULL, fast=True)
    ctx = Ctx()
    model = MuseTalkModel(ctx, us, vs, M.UNET_FULL, M.VAE_FULL, with_encoder=False)
    yield model, us, vs, M.UNET_FULL, M.VAE_FULL, _Weights(model, us, vs, M.UNET_FULL, M.VAE_FULL)
    ctx.close()


def _emit(ctx, model, av, B, index, aud, b):
    from livetalking_b200.musetalk import KEY_PAD
    hw = av.lat_hw
    d_index = ctx.alloc((4,), np.int32, zero=True)
    audio_in = ctx.alloc((B, KEY_PAD, 384), np.float16, zero=True)
    audio_pe = ctx.alloc((B * KEY_PAD, 384), np.float16, zero=True)
    lat16 = ctx.alloc((B, hw, hw, 16), np.float16, zero=True)
    img_u8 = ctx.alloc((B, hw * 8, hw * 8, 3), np.uint8, zero=True)
    ctx.set_i32(d_index, index)
    host = np.zeros((B, KEY_PAD, 384), np.float16)
    host[:, :50] = aud.astype(np.float16)
    ctx.h2d(audio_in, host)
    ctx.gather_rows(av.latents, av.latents.shape[0], d_index, B, hw * hw * 16, lat16)
    ctx.eltwise(audio_in, model.pe, audio_in.rows * audio_in.C, KEY_PAD * audio_in.C, 0, audio_pe)
    pred16 = model.emit_unet(b, lat16, audio_pe)
    model.emit_vae_decode(b, pred16, img_u8)
    return pred16, img_u8


@pytest.mark.parametrize("run", list(RUNS))
def test_musetalk_every_op_against_float64(request, run):
    """MuseTalkSession's op sequence traced eagerly, every op of the checked images against float64 as it is recorded; the
    session's own eager pass must emit the same op sequence and its captured graph must reproduce the traced output within the
    GroupNorm-atomics jitter."""
    from livetalking_b200 import engine
    from livetalking_b200.graph import Builder
    from livetalking_b200.musetalk import MuseTalkSession
    from livetalking_b200.ops import Ctx
    from oracle import musetalk_ref as M
    from oracle.wav2lip_ref import psnr_u8
    from test_gpu_musetalk import _avatar
    nets, B, hw, nf, index, imgs, band, fused = RUNS[run]
    model, us, vs, ucfg, vcfg, W = request.getfixturevalue(nets)
    engine.set_device(0)
    lat, _ = M.synth_latents_and_audio(nf, hw=hw, seed=20 + B)
    _, aud = M.synth_latents_and_audio(B, hw=8, seed=40 + B)
    aud = aud.numpy()
    mctx = model.ctx
    av, *_ = _avatar(mctx, lat.numpy(), nf)
    saved = Builder.FUSE_ATTENTION
    Builder.FUSE_ATTENTION = fused
    try:
        t0 = time.time()
        ctx = Ctx()
        chk = _Checker(run, W, B, imgs, band, model)
        _register_attn(chk, W, model)
        tr = OpTrace(ctx, MT_OPS, keep=_keep(B, imgs), on_record=chk)
        pred16, img_u8 = _emit(ctx, model, av, B, index, aud, Builder(ctx))
        tr.stop()
        traced_pred = ctx.download(pred16)
        traced_img = ctx.download(img_u8)
        assert not tr.errors, tr.errors[:5]
        t_all = time.time() - t0
        ctx.close()
        chk.rep.finish(t_all - chk.t, chk.t)
        assert chk.counts == _expected_counts(model, us, vs, ucfg, vcfg, fused), (chk.counts, _expected_counts(model, us, vs, ucfg, vcfg, fused))
        # zero-padded output channels checked: the head padding of every q / kv / qkv projection with d < dp, and the conv outs
        n_head_pad = sum(1 + int(not a.self_attn) for _k, a in _attn_objects(model) if a.dp > a.d)
        conv_outs = [p for p in chk.pads if ".attn" not in p]
        assert conv_outs == ["conv_out", "post_quant_conv", "decoder.conv_out"] and len(chk.pads) == n_head_pad + 3, chk.pads

        # production: the session's own eager pass (a data-free tracer on its ctx) and its captured graph
        sctx = Ctx()
        str_ = OpTrace(sctx, MT_OPS, data=False)
        sess = MuseTalkSession(model, av, B, ctx=sctx)
        assert not str_.active
        prod = sess.infer(index, aud)
        prod_pred = sctx.download(sess.pred16)
        sess.close()
        sctx.close()
    finally:
        Builder.FUSE_ATTENTION = saved
    got_sig = [_sig(r) for r in str_.records]
    want_sig = [_sig(r) for r in tr.records]
    assert len(got_sig) == len(want_sig), (len(got_sig), len(want_sig))
    for i, (g, w) in enumerate(zip(got_sig, want_sig)):
        assert g == w, f"[{run}] op #{i}: the session emits {g[0]} {g[1]} plan {g[2]}, the traced pass {w[0]} {w[1]} plan {w[2]}"
    step = int(np.abs(prod.astype(int) - traced_img.astype(int)).max())
    psnr = psnr_u8(prod, traced_img)
    dpred = float(np.abs(prod_pred[..., :4].astype(np.float64) - traced_pred[..., :4].astype(np.float64)).max())
    print(f"\n[{run}] production vs traced pass: image max step {step}, PSNR {psnr:.1f} dB, pred16 max |diff| {dpred:.3g}; "
          f"GroupNorm bound tightness {chk.tight:.3f} of 8 ulps")
    assert step <= 2 and psnr >= 55.0, (step, psnr)
    assert dpred <= PRED_TOL, dpred


def test_vae_encode_every_op_against_float64(small):
    """emit_vae_encode on the small VAE, B = 2 images (4 encoder images: masked and reference copies): vae_pre, the asymmetric-pad
    stride-2 convs and the quant convs that write the two halves of the latent buffer, every op against float64."""
    from livetalking_b200.graph import Builder
    from livetalking_b200.ops import Ctx
    model, us, vs, ucfg, vcfg, W = small
    B = 2
    rng = np.random.default_rng(2)
    low = rng.integers(0, 256, (B, 32, 32, 3)).astype(np.float32)
    imgs = np.clip(np.kron(low, np.ones((1, 8, 8, 1), np.float32)) + rng.integers(-6, 7, (B, 256, 256, 3)), 0, 255).astype(np.uint8)
    t0 = time.time()
    ctx = Ctx()
    chk = _Checker("encode_small", W, 2 * B, tuple(range(2 * B)), False, model)
    _register_attn(chk, W, model)
    tr = OpTrace(ctx, MT_OPS, on_record=chk)
    d_img = ctx.alloc(imgs.shape, np.uint8)
    ctx.h2d(d_img, imgs)
    out = ctx.alloc((B, 32, 32, 16), np.float16, zero=True)
    model.emit_vae_encode(Builder(ctx), d_img, out)
    tr.stop()
    assert not tr.errors, tr.errors[:5]
    lat = ctx.download(out)
    t_all = time.time() - t0
    ctx.close()
    assert chk.counts == _expected_counts(model, us, vs, ucfg, vcfg, True, decode=False, encode=True), chk.counts
    assert chk.pads == ["encoder.conv_out"], chk.pads
    assert not _bits(lat[..., 8:]).any()
    chk.rep.finish(t_all - chk.t, chk.t)
