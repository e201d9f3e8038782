"""MuseTalk on the H100 engine: VAE-encode -> audio-conditioned UNet -> VAE-decode -> blend paste-back.

The reference only *wraps* these networks (diffusers ``UNet2DConditionModel`` / ``AutoencoderKL``:
avatars/musetalk/models/unet.py:29-48, vae.py:10-38) and drives them from ``MuseReal.inference_batch``
(avatars/musetalk_avatar.py:130-152).  Here the host code (this file) assembles the same graphs out of the engine's
device operators — tcgen05 implicit-GEMM convs / linears / attention GEMMs, GroupNorm, LayerNorm, softmax, GEGLU ... —
captures them ONCE into a CUDA graph per batch size and replays the graph per step.  Weights are taken from state_dicts
with the diffusers key scheme (so a real ``unet.pth`` / ``sd-vae`` loads by name).

``MuseTalkBatchSession`` runs G sessions' frames through one graph, each group's latents gathered from its own avatar before the
launch (cross-session mode); ``MuseTalkSession`` is its one-group form bound to one avatar, one session's own stream.

Load-time rewrites (exact up to fp16 rounding):
  * timestep is the constant 0 (musetalk_avatar.py:61): ``time_emb_proj(silu(time_embedding(t=0)))`` is folded into the
    bias of every ResnetBlock's conv1;
  * ``latents / scaling_factor`` (vae.py:102) is folded into ``post_quant_conv``; ``scaling_factor * mean`` (vae.py:93)
    into ``quant_conv``;
  * q/k/v projections are fused and every head is zero-padded to a multiple of 16 channels (head_dim 40 -> 48) so the
    attention GEMMs meet the tensor-core K granularity; ``to_out`` gets the matching zero columns.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence

import numpy as np

from . import _capi
from .graph import Builder, GraphSession, _ceil16, _Norm, _np
from .ops import ConvWeight, Ctx, DevTensor

KEY_PAD = 64  # cross-attention keys (50 audio tokens) padded to a multiple of 16


def _silu(x):
    return x / (1.0 + np.exp(-x))


def _pad_heads_rows(w: np.ndarray, heads: int, d: int, dp: int) -> np.ndarray:
    """[heads*d, cin] -> [heads*dp, cin] with zero rows after each head."""
    out = np.zeros((heads * dp, w.shape[1]), np.float32)
    for h in range(heads):
        out[h * dp:h * dp + d] = w[h * d:(h + 1) * d]
    return out


def _pad_heads_vec(b: np.ndarray, heads: int, d: int, dp: int) -> np.ndarray:
    out = np.zeros(heads * dp, np.float32)
    for h in range(heads):
        out[h * dp:h * dp + d] = b[h * d:(h + 1) * d]
    return out


def _pad_heads_cols(w: np.ndarray, heads: int, d: int, dp: int) -> np.ndarray:
    """[cout, heads*d] -> [cout, heads*dp] with zero columns after each head."""
    out = np.zeros((w.shape[0], heads * dp), np.float32)
    for h in range(heads):
        out[:, h * dp:h * dp + d] = w[:, h * d:(h + 1) * d]
    return out


class _Attn:
    """One diffusers ``Attention`` block (self or cross) in engine layout."""

    def __init__(self, ctx: Ctx, sd, p: str, C: int, heads: int, kv_dim: Optional[int]):
        d = C // heads
        dp = _ceil16(d)
        self.C, self.heads, self.d, self.dp = C, heads, d, dp
        self.self_attn = kv_dim is None
        bias = (p + ".to_q.bias") in sd
        wq, wk, wv = (_pad_heads_rows(_np(sd[f"{p}.{n}.weight"]), heads, d, dp) for n in ("to_q", "to_k", "to_v"))
        bq = bk = bv = None
        if bias:
            bq, bk, bv = (_pad_heads_vec(_np(sd[f"{p}.{n}.bias"]), heads, d, dp) for n in ("to_q", "to_k", "to_v"))
        if self.self_attn:
            self.qkv = ConvWeight(ctx, np.concatenate([wq, wk, wv], 0), np.concatenate([bq, bk, bv]) if bias else None, tap_major=False)
        else:
            self.q = ConvWeight(ctx, wq, bq, tap_major=False)
            self.kv = ConvWeight(ctx, np.concatenate([wk, wv], 0), np.concatenate([bk, bv]) if bias else None, tap_major=False)
        self.out = ConvWeight(ctx, _pad_heads_cols(_np(sd[p + ".to_out.0.weight"]), heads, d, dp), _np(sd[p + ".to_out.0.bias"]),
                              tap_major=False)


class _Resnet:
    def __init__(self, ctx: Ctx, sd, p: str, temb_act: Optional[np.ndarray]):
        w1 = _np(sd[p + ".conv1.weight"])
        b1 = _np(sd[p + ".conv1.bias"]).copy()
        if temb_act is not None:   # constant timestep: time_emb_proj(silu(emb)) is a per-channel bias after conv1
            b1 += _np(sd[p + ".time_emb_proj.weight"]) @ temb_act + _np(sd[p + ".time_emb_proj.bias"])
        self.cin, self.cout = w1.shape[1], w1.shape[0]
        self.norm1, self.norm2 = _Norm(ctx, sd, p + ".norm1"), _Norm(ctx, sd, p + ".norm2")
        self.conv1 = ConvWeight(ctx, w1, b1)
        self.conv2 = ConvWeight(ctx, _np(sd[p + ".conv2.weight"]), _np(sd[p + ".conv2.bias"]))
        self.shortcut = None
        if (p + ".conv_shortcut.weight") in sd:
            self.shortcut = ConvWeight(ctx, _np(sd[p + ".conv_shortcut.weight"]), _np(sd[p + ".conv_shortcut.bias"]), tap_major=False)


class _Transformer:
    def __init__(self, ctx: Ctx, sd, p: str, C: int, heads: int, ctx_dim: int):
        self.C = C
        self.norm = _Norm(ctx, sd, p + ".norm")
        self.proj_in = ConvWeight(ctx, _np(sd[p + ".proj_in.weight"]), _np(sd[p + ".proj_in.bias"]), tap_major=False)
        self.proj_out = ConvWeight(ctx, _np(sd[p + ".proj_out.weight"]), _np(sd[p + ".proj_out.bias"]), tap_major=False)
        b = p + ".transformer_blocks.0"
        self.ln1, self.ln2, self.ln3 = (_Norm(ctx, sd, f"{b}.norm{i}") for i in (1, 2, 3))
        self.attn1 = _Attn(ctx, sd, b + ".attn1", C, heads, None)
        self.attn2 = _Attn(ctx, sd, b + ".attn2", C, heads, ctx_dim)
        self.ff1 = ConvWeight(ctx, _np(sd[b + ".ff.net.0.proj.weight"]), _np(sd[b + ".ff.net.0.proj.bias"]), tap_major=False)
        self.ff2 = ConvWeight(ctx, _np(sd[b + ".ff.net.2.weight"]), _np(sd[b + ".ff.net.2.bias"]), tap_major=False)


class MuseTalkModel:
    """Device-resident UNet + VAE weights (replaces load_model()'s vae/unet/pe, musetalk_avatar.py:57-67)."""

    def __init__(self, ctx: Ctx, unet_sd: Dict, vae_sd: Dict, ucfg, vcfg, with_encoder: bool = True):
        self.ctx, self.ucfg, self.vcfg = ctx, ucfg, vcfg
        sd = unet_sd
        boc = ucfg.block_out_channels
        heads = ucfg.num_heads
        # constant timestep embedding (t = 0): [cos(0)..., sin(0)...] = [1]*half + [0]*half
        half = boc[0] // 2
        temb = np.concatenate([np.ones(half, np.float32), np.zeros(half, np.float32)])
        temb = _np(sd["time_embedding.linear_1.weight"]) @ temb + _np(sd["time_embedding.linear_1.bias"])
        temb = _np(sd["time_embedding.linear_2.weight"]) @ _silu(temb) + _np(sd["time_embedding.linear_2.bias"])
        ta = _silu(temb)
        self.u_conv_in = ConvWeight(ctx, _np(sd["conv_in.weight"]), _np(sd["conv_in.bias"]), pad_cin=16)
        self.u_down = []
        for i in range(len(boc)):
            blk = {"res": [], "attn": [], "down": None}
            for j in range(ucfg.layers_per_block):
                blk["res"].append(_Resnet(ctx, sd, f"down_blocks.{i}.resnets.{j}", ta))
                if ucfg.down_has_attn[i]:
                    blk["attn"].append(_Transformer(ctx, sd, f"down_blocks.{i}.attentions.{j}", boc[i], heads, ucfg.cross_attention_dim))
            if i < len(boc) - 1:
                p = f"down_blocks.{i}.downsamplers.0.conv"
                blk["down"] = ConvWeight(ctx, _np(sd[p + ".weight"]), _np(sd[p + ".bias"]), tap_major=False)
            self.u_down.append(blk)
        self.u_mid = (_Resnet(ctx, sd, "mid_block.resnets.0", ta),
                      _Transformer(ctx, sd, "mid_block.attentions.0", boc[-1], heads, ucfg.cross_attention_dim),
                      _Resnet(ctx, sd, "mid_block.resnets.1", ta))
        rev = list(reversed(boc))
        self.u_up = []
        for i in range(len(boc)):
            blk = {"res": [], "attn": [], "up": None}
            for j in range(ucfg.layers_per_block + 1):
                blk["res"].append(_Resnet(ctx, sd, f"up_blocks.{i}.resnets.{j}", ta))
                if ucfg.up_has_attn[i]:
                    blk["attn"].append(_Transformer(ctx, sd, f"up_blocks.{i}.attentions.{j}", rev[i], heads, ucfg.cross_attention_dim))
            if i < len(boc) - 1:
                p = f"up_blocks.{i}.upsamplers.0.conv"
                blk["up"] = ConvWeight(ctx, _np(sd[p + ".weight"]), _np(sd[p + ".bias"]))
            self.u_up.append(blk)
        self.u_norm_out = _Norm(ctx, sd, "conv_norm_out")
        self.u_conv_out = ConvWeight(ctx, _np(sd["conv_out.weight"]), _np(sd["conv_out.bias"]), pad_cout=32)   # 32: TMA halo kernel

        # ---- VAE decoder
        sd = vae_sd
        sf = vcfg.scaling_factor
        self.v_post_quant = ConvWeight(ctx, _np(sd["post_quant_conv.weight"]) / sf, _np(sd["post_quant_conv.bias"]), pad_cin=16, pad_cout=16,
                                       tap_major=False)
        self.v_dec_in = ConvWeight(ctx, _np(sd["decoder.conv_in.weight"]), _np(sd["decoder.conv_in.bias"]), pad_cin=16)
        self.v_dec_mid = self._vae_mid(ctx, sd, "decoder.mid_block")
        vrev = list(reversed(vcfg.block_out_channels))
        self.v_dec_up = []
        for i in range(len(vrev)):
            blk = {"res": [_Resnet(ctx, sd, f"decoder.up_blocks.{i}.resnets.{j}", None) for j in range(vcfg.layers_per_block + 1)], "up": None}
            if i < len(vrev) - 1:
                p = f"decoder.up_blocks.{i}.upsamplers.0.conv"
                blk["up"] = ConvWeight(ctx, _np(sd[p + ".weight"]), _np(sd[p + ".bias"]))
            self.v_dec_up.append(blk)
        self.v_dec_norm_out = _Norm(ctx, sd, "decoder.conv_norm_out")
        self.v_dec_out = ConvWeight(ctx, _np(sd["decoder.conv_out.weight"]), _np(sd["decoder.conv_out.bias"]), pad_cout=32)
        # ---- VAE encoder (BASELINE config 3; offline in the reference: avatars/musetalk/genavatar.py:126-128)
        self.with_encoder = with_encoder
        if with_encoder:
            vb = vcfg.block_out_channels
            self.v_enc_in = ConvWeight(ctx, _np(sd["encoder.conv_in.weight"]), _np(sd["encoder.conv_in.bias"]), pad_cin=16)
            self.v_enc_down = []
            for i in range(len(vb)):
                blk = {"res": [_Resnet(ctx, sd, f"encoder.down_blocks.{i}.resnets.{j}", None) for j in range(vcfg.layers_per_block)], "down": None}
                if i < len(vb) - 1:
                    p = f"encoder.down_blocks.{i}.downsamplers.0.conv"
                    blk["down"] = ConvWeight(ctx, _np(sd[p + ".weight"]), _np(sd[p + ".bias"]), tap_major=False)
                self.v_enc_down.append(blk)
            self.v_enc_mid = self._vae_mid(ctx, sd, "encoder.mid_block")
            self.v_enc_norm_out = _Norm(ctx, sd, "encoder.conv_norm_out")
            self.v_enc_out = ConvWeight(ctx, _np(sd["encoder.conv_out.weight"]), _np(sd["encoder.conv_out.bias"]), pad_cout=32)
            L = vcfg.latent_channels
            qw, qb = _np(sd["quant_conv.weight"])[:L, :, 0, 0] * sf, _np(sd["quant_conv.bias"])[:L] * sf   # mean rows, x scaling_factor
            w_lo = np.zeros((16, 16), np.float32)
            b_lo = np.zeros(16, np.float32)
            w_lo[:L, :2 * L] = qw
            b_lo[:L] = qb
            w_hi = np.zeros((16, 16), np.float32)
            b_hi = np.zeros(16, np.float32)
            w_hi[L:2 * L, :2 * L] = qw
            b_hi[L:2 * L] = qb
            self.v_quant_masked = ConvWeight(ctx, w_lo, b_lo, tap_major=False)    # masked latents -> channels [0, L)
            self.v_quant_ref = ConvWeight(ctx, w_hi, b_hi, tap_major=False)       # reference latents -> channels [L, 2L)
        # positional encoding table (unet.py:12-27), rows >= 50 zero (key padding)
        pe = np.zeros((KEY_PAD, ucfg.cross_attention_dim), np.float32)
        pos = np.arange(50, dtype=np.float32)[:, None]
        D = ucfg.cross_attention_dim
        div = np.exp(np.arange(0, D, 2, dtype=np.float32) * np.float32(-math.log(10000.0) / D))
        pe[:50, 0::2] = np.sin(pos * div)
        pe[:50, 1::2] = np.cos(pos * div)
        self.pe = ctx.upload(pe.astype(np.float16))
        ctx.sync()

    @staticmethod
    def _vae_mid(ctx, sd, p):
        a = p + ".attentions.0"
        C = _np(sd[a + ".to_q.weight"]).shape[0]
        return (_Resnet(ctx, sd, p + ".resnets.0", None), _Norm(ctx, sd, a + ".group_norm"), _Attn(ctx, sd, a, C, 1, None),
                _Resnet(ctx, sd, p + ".resnets.1", None))

    # ------------------------------------------------------------------------------------------ graph emitters
    @staticmethod
    def _resnet(b: Builder, x: DevTensor, r: _Resnet, groups: int, eps: float) -> DevTensor:
        h = b.conv3(b.groupnorm(x, r.norm1, groups, eps, True), r.conv1, stats=True)
        h = b.groupnorm(h, r.norm2, groups, eps, True)
        skip = b.linear(x, r.shortcut) if r.shortcut is not None else x
        return b.conv3(h, r.conv2, res=skip, stats=True)

    @staticmethod
    def _transformer(b: Builder, x: DevTensor, t: _Transformer, audio: DevTensor, groups: int) -> DevTensor:
        N, H, W, C = x.shape
        tok = b.linear(b.groupnorm(x, t.norm, groups, 1e-6, False), t.proj_in)          # (N,H,W,C) == tokens (N*HW, C)
        tok = b.attention(t.attn1, b.layernorm(tok, t.ln1), N, H * W, res=tok)
        tok = b.attention(t.attn2, b.layernorm(tok, t.ln2), N, H * W, res=tok, kv_src=audio, n_keys=KEY_PAD, n_valid=50)
        g = b.linear(b.layernorm(tok, t.ln3), t.ff1)                                    # (.., 8C)
        gg = b.new(N, H, W, 4 * C)
        b.ctx.geglu(g, N * H * W, 4 * C, gg)
        tok = b.linear(gg, t.ff2, res=tok)
        return b.linear(tok, t.proj_out, res=x)

    def emit_unet(self, b: Builder, latents16: DevTensor, audio_pe: DevTensor, taps: Optional[dict] = None) -> DevTensor:
        """latents16 (B,h,w,16) [8 real channels], audio_pe (B*64, 384) -> predicted latents (B,h,w,16) [4 real channels]."""
        cfg = self.ucfg
        G, eps = cfg.norm_groups, cfg.norm_eps
        h = b.conv3(latents16, self.u_conv_in, stats=True)
        skips = [h]
        for i, blk in enumerate(self.u_down):
            for j, r in enumerate(blk["res"]):
                h = self._resnet(b, h, r, G, eps)
                if blk["attn"]:
                    h = self._transformer(b, h, blk["attn"][j], audio_pe, G)
                skips.append(h)
            if blk["down"] is not None:
                h = b.conv3(h, blk["down"], stride=2)
                skips.append(h)
            if taps is not None:
                taps[f"down{i}"] = h
        h = self._resnet(b, h, self.u_mid[0], G, eps)
        h = self._transformer(b, h, self.u_mid[1], audio_pe, G)
        h = self._resnet(b, h, self.u_mid[2], G, eps)
        if taps is not None:
            taps["mid"] = h
        for i, blk in enumerate(self.u_up):
            for j, r in enumerate(blk["res"]):
                h = self._resnet(b, b.concat(h, skips.pop()), r, G, eps)
                if blk["attn"]:
                    h = self._transformer(b, h, blk["attn"][j], audio_pe, G)
            if blk["up"] is not None:
                h = b.upsample(h, blk["up"])
            if taps is not None:
                taps[f"up{i}"] = h
        return b.conv3(b.groupnorm(h, self.u_norm_out, G, eps, True), self.u_conv_out)

    def _emit_vae_mid(self, b: Builder, h: DevTensor, mid, G, eps):
        r0, gn, attn, r1 = mid
        h = self._resnet(b, h, r0, G, eps)
        N, H, W, C = h.shape
        h = b.attention(attn, b.groupnorm(h, gn, G, eps, False), N, H * W, res=h, stats_imgs=N)
        st = h.stats
        h = DevTensor(h.ptr, (N, H, W, C))
        h.stats = st
        return self._resnet(b, h, r1, G, eps)

    def emit_vae_decode(self, b: Builder, pred16: DevTensor, out_u8: DevTensor, taps: Optional[dict] = None) -> DevTensor:
        """pred16 (B,h,w,16) latents [4 real channels] -> uint8 BGR image written to out_u8 (B,8h,8w,3)."""
        cfg = self.vcfg
        G, eps = cfg.norm_groups, cfg.norm_eps
        h = b.conv3(b.linear(DevTensor(pred16.ptr, (*pred16.shape[:-1], 16), pitch=pred16.pitch), self.v_post_quant), self.v_dec_in, stats=True)
        h = self._emit_vae_mid(b, h, self.v_dec_mid, G, eps)
        if taps is not None:
            taps["dec_mid"] = h
        for i, blk in enumerate(self.v_dec_up):
            for r in blk["res"]:
                h = self._resnet(b, h, r, G, eps)
            if blk["up"] is not None:
                h = b.upsample(h, blk["up"])
            if taps is not None:
                taps[f"dec_up{i}"] = h
        img = b.conv3(b.groupnorm(h, self.v_dec_norm_out, G, eps, True), self.v_dec_out)   # (B,H,W,16), RGB in channels 0..2
        N, H, W, _ = img.shape
        b.ctx.vae_post(img, N * H * W, out_u8)
        return img

    def emit_vae_encode(self, b: Builder, img_u8: DevTensor, out_latents16: DevTensor):
        """img_u8 (B,H,W,3) uint8 BGR -> get_latents_for_unet (vae.py:110-122, latent_dist.mode()): (B,H/8,W/8,16) [8 real]."""
        assert self.with_encoder
        cfg = self.vcfg
        G, eps = cfg.norm_groups, cfg.norm_eps
        B, H, W, _ = img_u8.shape
        x = b.new(2 * B, H, W, 16)
        b.ctx.vae_pre(img_u8, B, H, W, True, DevTensor(x.ptr, (B, H, W, 16)))                                  # masked copies
        b.ctx.vae_pre(img_u8, B, H, W, False, DevTensor(x.offset(B * H * W * 16), (B, H, W, 16)))              # reference copies
        h = b.conv3(x, self.v_enc_in, stats=True)
        for blk in self.v_enc_down:
            for r in blk["res"]:
                h = self._resnet(b, h, r, G, eps)
            if blk["down"] is not None:
                h = b.conv3(h, blk["down"], stride=2, pad=(0, 0), stats=True)     # F.pad(x,(0,1,0,1)) + conv s2 p0
        h = self._emit_vae_mid(b, h, self.v_enc_mid, G, eps)
        m = b.conv3(b.groupnorm(h, self.v_enc_norm_out, G, eps, True), self.v_enc_out)   # (2B,h,w,16): moments in 0..7
        _, lh, lw, mc = m.shape
        half = B * lh * lw * mc
        tmp = b.linear(DevTensor(m.ptr, (B, lh, lw, 16), pitch=mc), self.v_quant_masked)
        b.linear(DevTensor(m.offset(half), (B, lh, lw, 16), pitch=mc), self.v_quant_ref, res=tmp, out=out_latents16)
        return out_latents16


class MuseTalkAvatar:
    """Avatar assets resident in HBM (replaces load_avatar's lists, musetalk_avatar.py:69-91): full frames, bbox
    (x1,y1,x2,y2), mask crop boxes (x_s,y_s,x_e,y_e), 3-channel blend masks and the pre-computed UNet input latents."""

    def __init__(self, ctx: Ctx, frames, masks, coords, crop_boxes, latents):
        self.ctx = ctx
        frames = np.ascontiguousarray(np.asarray(frames), np.uint8)
        self.n, self.H, self.W = frames.shape[0], frames.shape[1], frames.shape[2]
        self.frames_host = frames
        self.coords_host = np.ascontiguousarray(np.asarray(coords), np.int32).reshape(self.n, 4)
        self.crop_host = np.ascontiguousarray(np.asarray(crop_boxes), np.int32).reshape(self.n, 4)
        offs, blobs, o = [], [], 0
        for i in range(self.n):
            xs, ys, xe, ye = self.crop_host[i]
            x1, y1, x2, y2 = self.coords_host[i]
            m = np.ascontiguousarray(masks[i], np.uint8)
            if m.shape != (ye - ys, xe - xs, 3):
                raise ValueError(f"mask {i} has shape {m.shape}, crop box needs {(ye - ys, xe - xs, 3)}")
            if not (0 <= xs <= x1 < x2 <= xe <= self.W and 0 <= ys <= y1 < y2 <= ye <= self.H):
                raise ValueError(f"avatar frame {i}: bbox / crop box outside the frame")
            offs.append(o)
            blobs.append(m.reshape(-1))
            o += m.size
        self.masks_host = [np.asarray(m, np.uint8) for m in masks]
        self.frames = ctx.upload(frames)
        self.coords = ctx.upload(self.coords_host)
        self.crop = ctx.upload(self.crop_host)
        self.masks = ctx.upload(np.concatenate(blobs))
        self.mask_off = ctx.upload(np.asarray(offs, np.int64))
        # latents: list of (1,8,h,w) arrays (latents.pt) -> NHWC fp16 padded to 16 channels
        lat = np.concatenate([_np(l) for l in latents], 0)
        self.lat_hw = lat.shape[2]
        lat16 = np.zeros((lat.shape[0], lat.shape[2], lat.shape[3], 16), np.float16)
        lat16[..., :8] = lat.transpose(0, 2, 3, 1)
        self.latents = ctx.upload(lat16)


class MuseTalkBatchSession(GraphSession):
    """Cross-session batching for MuseTalk (SURVEY 8(f) rank 1, the MuseTalk twin of ltb_w2l_infer_slots): up to G sessions x Bs
    frames run as ONE captured PE + UNet + VAE-decode graph of batch G*Bs.  A *group request* is (avatar, first frame index,
    Whisper features (Bs, 50, 384) or None): group g's latents are gathered from ITS avatar's table (mirror-indexed, outside the
    graph, so any session may occupy any group of any round), its features occupy rows [g*Bs, (g+1)*Bs) of audio_in.
    The reference serves every session with its own B-frame forward (avatars/musetalk_avatar.py:130-152 under app.py:76-100's
    max_session connections); at batch 8 the UNet is launch-latency bound (64 M-tiles per layer), so four sessions per
    launch cost far less than four launches.  `batch` / `infer_slots` make it a mux for plugin.batcher.CrossSessionBatcher.

    keep_taps: `taps` holds the UNet's and the VAE decoder's intermediate activations (else None).
    avatar: bind the session to this one avatar — every request must use it, and its output frames are allocated here.
    ctx: the session's own stream + scratch (created here unless given).  Sessions never share a ctx: the reference opens up to
    max_session of them concurrently (app.py:76-100), each driven by its own three threads, and capturing / synchronising a stream
    another session is using would corrupt both."""

    def __init__(self, model: MuseTalkModel, lat_hw: int, groups: int, frames_per_session: int, *, ctx: Optional[Ctx] = None,
                 keep_taps: bool = False, avatar: Optional[MuseTalkAvatar] = None):
        super().__init__(ctx)
        self.model, self.lat_hw, self.Bs, self.G, self.avatar = model, int(lat_hw), int(frames_per_session), int(groups), avatar
        self.batch = self.G                                  # CrossSessionBatcher: requests per engine call
        self.B = B = self.G * self.Bs
        try:
            ctx, Bs, hw, cad = self.ctx, self.Bs, self.lat_hw, model.ucfg.cross_attention_dim
            self._d_index = self.alloc((4 * self.G,), np.int32, zero=True)
            self.d_index = [DevTensor(self._d_index.ptr + 16 * g, (4,), np.int32) for g in range(self.G)]
            self.audio_in = self.alloc((B, KEY_PAD, cad), np.float16, zero=True)
            self.audio_in_of = [DevTensor(self.audio_in.ptr + g * Bs * KEY_PAD * cad * 2, (Bs, KEY_PAD, cad)) for g in range(self.G)]
            self.audio_pe = self.alloc((B * KEY_PAD, cad), np.float16, zero=True)
            self.latents16 = self.alloc((B, hw, hw, 16), np.float16, zero=True)
            self.latents16_of = [DevTensor(self.latents16.ptr + g * Bs * hw * hw * 16 * 2, (Bs, hw, hw, 16)) for g in range(self.G)]
            self.image_u8 = self.alloc((B, hw * 8, hw * 8, 3), np.uint8, zero=True)
            self._frames_out: Dict[tuple, DevTensor] = {}
            if avatar is not None:
                if self.G != 1:
                    raise ValueError("a session bound to an avatar has one group")
                self.frames_out = self._out(0, avatar)
                # the warm-up pass below runs on the avatar's frame-0 latents (d_index is 0), not on zeros
                ctx.gather_rows(avatar.latents, avatar.latents.shape[0], self.d_index[0], Bs, hw * hw * 16, self.latents16_of[0])
            self.taps = {} if keep_taps else None
            self._audio_host = np.zeros((B, KEY_PAD, cad), np.float16)

            def emit(b: Builder):
                ctx.eltwise(self.audio_in, model.pe, self.audio_in.rows * self.audio_in.C, KEY_PAD * self.audio_in.C, 0, self.audio_pe)
                self.pred16 = model.emit_unet(b, self.latents16, self.audio_pe, self.taps)
                self.image16 = model.emit_vae_decode(b, self.pred16, self.image_u8, self.taps)

            self.capture(emit)
        except BaseException:
            self.close()
            raise

    def _check(self, requests):
        if not 1 <= len(requests) <= self.G:
            raise ValueError(f"1..{self.G} group requests per call, got {len(requests)}")
        for r in requests:
            if r[0].lat_hw != self.lat_hw:
                raise ValueError("avatar latent size does not match the batch session")
            if self.avatar is not None and r[0] is not self.avatar:
                raise ValueError("the session is bound to another avatar")

    def _launch(self, requests: Sequence[tuple]):
        """requests[g] = (MuseTalkAvatar, first frame index, features (Bs,50,384) | None = resident in audio_in_of[g]): stage the
        features, gather every group's latents (set_i32 + gather_rows before the launch) and launch the graph."""
        if self.graph is None:
            raise RuntimeError(f"{type(self).__name__}: paste-only (or closed) session has no network graph")
        self._check(requests)
        ctx, Bs, row = self.ctx, self.Bs, self.lat_hw * self.lat_hw * 16
        stage = False
        for g, (av, index, feats) in enumerate(requests):
            if feats is not None:
                a = np.asarray(feats)
                if a.shape != (Bs, 50, self._audio_host.shape[2]):
                    raise ValueError(f"audio features must be ({Bs},50,{self._audio_host.shape[2]}), got {a.shape}")
                self._audio_host[g * Bs:(g + 1) * Bs, :50] = a.astype(np.float16)
                stage = True
            ctx.set_i32(self.d_index[g], int(index))
            ctx.gather_rows(av.latents, av.latents.shape[0], self.d_index[g], Bs, row, self.latents16_of[g])
        if stage:
            n = len(requests) * Bs
            ctx.h2d(DevTensor(self.audio_in.ptr, (n,) + self.audio_in.shape[1:]), self._audio_host[:n], sync=False)
        self.graph.launch()

    def _out(self, g: int, av: MuseTalkAvatar) -> DevTensor:
        key = (g, av.H, av.W)
        if key not in self._frames_out:
            self._frames_out[key] = self.alloc((self.Bs, av.H, av.W, 3), np.uint8, zero=True)
        return self._frames_out[key]

    def paste_async(self, requests: Sequence[tuple]) -> List[DevTensor]:
        """Blend paste-back of every group's predictions into its own avatar frames (device resident; MuseReal.paste_back_frame x Bs)."""
        self._check(requests)
        outs = []
        for g, (a, index, _f) in enumerate(requests):
            out = self._out(g, a)
            self.ctx.mt_paste(_paste_op(a, self.image_u8, out, g * self.Bs, int(index), -1, self.Bs))
            outs.append(out)
        return outs

    infer_async = _launch

    def infer_groups(self, requests: Sequence[tuple]) -> List[np.ndarray]:
        """-> per request its (Bs, S, S, 3) uint8 BGR predictions (what MuseReal.inference_batch returns for that session)."""
        with self.ctx.lock:
            self._launch(requests)
            n = len(requests) * self.Bs
            S = self.lat_hw * 8
            pred = self.ctx.download(DevTensor(self.image_u8.ptr, (n, S, S, 3), np.uint8))
        return [pred[g * self.Bs:(g + 1) * self.Bs] for g in range(len(requests))]

    infer_slots = infer_groups

    def step_async(self, requests: Sequence[tuple]):
        self._launch(requests)
        self.paste_async(requests)

    def step(self, requests: Sequence[tuple]) -> List[np.ndarray]:
        """One batched round: returns, per session, its Bs composited frames (Bs, H, W, 3) uint8."""
        with self.ctx.lock:
            self._launch(requests)
            outs = [self.ctx.download(t, sync=False) for t in self.paste_async(requests)]
            self.ctx.sync()
            return outs


class MuseTalkSession(MuseTalkBatchSession):
    """One avatar stream at a fixed batch size: MuseTalkBatchSession with one group, bound to `avatar`."""

    def __init__(self, model: MuseTalkModel, avatar: MuseTalkAvatar, batch: int, keep_taps: bool = False, ctx: Optional[Ctx] = None,
                 paste_only: bool = False):
        """paste_only: no ctx, network graph or activation arena — only paste_pred() works (cross-session mode: the UNet / VAE pass
        of this session's frames runs in a shared MuseTalkBatchSession)."""
        if paste_only:
            GraphSession.__init__(self, ctx, with_ctx=False)
            self.model, self.avatar, self.B = model, avatar, int(batch)
            return
        super().__init__(model, avatar.lat_hw, 1, batch, ctx=ctx, keep_taps=keep_taps, avatar=avatar)

    # ---- MuseReal.inference_batch (musetalk_avatar.py:130-152)
    def infer_async(self, index: int, audio_feats: Optional[np.ndarray] = None):
        self._launch([(self.avatar, index, audio_feats)])

    def infer(self, index: int, audio_feats: Optional[np.ndarray] = None, want_pred: bool = True):
        with self.ctx.lock:       # h2d -> index -> graph -> d2h is one critical section (inference vs process_frames thread)
            self.infer_async(index, audio_feats)
            if want_pred:
                return self.ctx.download(self.image_u8)          # uint8 (B,hw*8,hw*8,3) BGR, as vae.decode_latents returns
            self.ctx.sync()
            return None

    # ---- MuseReal.paste_back_frame (musetalk_avatar.py:154-164)
    def paste(self, slot: int, idx: int) -> np.ndarray:
        if not (0 <= slot < self.B and 0 <= idx < self.avatar.n):
            raise ValueError("paste: slot / idx out of range")
        with self.ctx.lock:
            self.ctx.mt_paste(_paste_op(self.avatar, self.image_u8, self.frames_out, slot, 0, idx, 1))
            one = DevTensor(self.frames_out.ptr, (self.avatar.H, self.avatar.W, 3), np.uint8)
            return self.ctx.download(one)

    def paste_pred(self, pred_u8: np.ndarray, idx: int) -> np.ndarray:
        """paste_back_frame for a host prediction (S,S,3) uint8 — the reference's exact argument, on the session's paste ctx."""
        a = self.avatar
        S = a.lat_hw * 8
        pred_u8 = np.ascontiguousarray(pred_u8, np.uint8)
        if pred_u8.shape != (S, S, 3):
            raise ValueError(f"paste_pred: prediction must be ({S},{S},3) uint8, got {pred_u8.shape}")
        if not 0 <= idx < a.n:
            raise ValueError("paste_pred: idx out of range")
        pc, pred, out = self.paste_ctx((1, S, S, 3), np.uint8, (a.H, a.W, 3))
        with pc.lock:
            pc.h2d(pred, pred_u8, sync=False)
            pc.mt_paste(_paste_op(a, pred, out, 0, 0, idx, 1))
            return pc.download(out)

    def paste_batch_async(self, index: int):
        self.paste_async([(self.avatar, index, None)])

    def paste_batch(self, index: int, out: Optional[np.ndarray] = None) -> np.ndarray:
        with self.ctx.lock:
            self.paste_batch_async(index)
            return self.ctx.download(self.frames_out, out)

    def step_async(self, index: int):
        """Everything resident (audio features already on the device): latent gather + UNet + VAE decode + blend paste-back."""
        self.infer_async(index, None)
        self.paste_batch_async(index)


def _paste_op(a: MuseTalkAvatar, pred: DevTensor, out: DevTensor, slot0: int, index: int, explicit_idx: int, count: int) -> _capi.MtPasteOp:
    """The blend paste-back of `count` predictions from pred slot `slot0` into avatar `a`'s frames (index / explicit_idx as ltb_mt_paste_op)."""
    op = _capi.MtPasteOp()
    op.frames, op.coords, op.crop, op.masks, op.mask_off = a.frames.ptr, a.coords.ptr, a.crop.ptr, a.masks.ptr, a.mask_off.ptr
    op.pred, op.out = pred.ptr, out.ptr
    op.nf, op.H, op.W = a.n, a.H, a.W
    op.index, op.explicit_idx, op.slot0, op.count = index, explicit_idx, slot0, count
    op.pred_hw = a.lat_hw * 8
    return op


def encode_avatar_latents(model: MuseTalkModel, images_u8: np.ndarray) -> np.ndarray:
    """GPU get_latents_for_unet for a stack of (n,256,256,3) uint8 BGR crops -> (n,8,h,w) float16 (latents.pt content,
    avatars/musetalk/genavatar.py:126-128 with the deterministic latent_dist.mode())."""
    ctx = model.ctx
    imgs = np.ascontiguousarray(images_u8, np.uint8)
    n, H, W, _ = imgs.shape
    run = GraphSession(ctx)                      # owns the buffers of this one eager pass
    try:
        d_img = run.alloc(imgs.shape, np.uint8)
        ctx.h2d(d_img, imgs)
        out = run.alloc((n, H // 8, W // 8, 16), np.float16, zero=True)
        model.emit_vae_encode(Builder(ctx, run.alloc), d_img, out)
        lat = ctx.download(out)
    finally:
        run.close()
    return np.ascontiguousarray(lat[..., :8].transpose(0, 3, 1, 2))
