"""HuBERT audio features on the B200 engine (SURVEY §8 row f4) — replaces ``Audio2Feature.get_hubert_from_16k_speech``
(avatars/ultralight/audio2feature.py:14-56: ``Wav2Vec2Processor`` + ``HubertModel(...).last_hidden_state``) and the window gather of
``HubertASR.run_step`` (avatars/audio_features/hubert.py:27-51).

Weights come from the HF ``HubertModel`` state_dict of the checkpoint the reference loads (hubert-large-ls960-ft: 7 conv layers with
per-layer LayerNorm and bias, 1024-d stable-LayerNorm transformer, 16-group positional conv with weight norm).  Conv layers 1-6, the
projections, attention and MLPs run on the tcgen05 conv / fused-attention kernels; conv layer 0 (+ the processor's utterance
normalisation), the grouped positional conv and the window gather are csrc/hubert.cu.  One CUDA graph per extractor.

``HubertBatchFeatures`` runs G sessions' windows stacked on the row dimension, one encoder forward for all (cross-session mode);
``HubertFeatures`` is its one-window form, one session's own extractor."""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import numpy as np

from .graph import Builder, GraphSession, _Norm, _np
from .ops import ConvWeight, Ctx, DevTensor

CONV_KERNEL = (10, 3, 3, 3, 3, 2, 2)
CONV_STRIDE = (5, 2, 2, 2, 2, 2, 2)
POS_K, POS_GROUPS = 128, 16
WIN = (4, 4)            # HubertASR(audio_feat_length=[4,4]) (ultralight_avatar.py:137)
ROWS = 16               # (4 + 4) * 2 feature rows per frame -> reshape(16, 32, 32)


def conv_frames(n: int) -> int:
    for k, s in zip(CONV_KERNEL, CONV_STRIDE):
        n = (n - k) // s + 1
    return n


class _HAttn:
    self_attn = True

    def __init__(self, ctx: Ctx, sd, p: str, d_model: int, heads: int):
        self.heads, self.d, self.dp = heads, d_model // heads, d_model // heads
        if self.d % 16:
            raise ValueError("HuBERT head dim must be a multiple of 16")
        w = np.concatenate([_np(sd[f"{p}.{n}.weight"]) for n in ("q_proj", "k_proj", "v_proj")], 0)
        b = np.concatenate([_np(sd[f"{p}.{n}.bias"]) for n in ("q_proj", "k_proj", "v_proj")])
        self.qkv = ConvWeight(ctx, w, b, tap_major=False)
        self.out = ConvWeight(ctx, _np(sd[p + ".out_proj.weight"]), _np(sd[p + ".out_proj.bias"]), tap_major=False)


class HubertEncoder:
    """Device-resident ``HubertModel`` (large layout: feat_extract_norm='layer', conv_bias, do_stable_layer_norm)."""

    def __init__(self, ctx: Ctx, sd: Dict, heads: int = 16, eps: float = 1e-5):
        sd = {k[len("hubert."):] if k.startswith("hubert.") else k: v for k, v in sd.items()}
        if "feature_extractor.conv_layers.1.layer_norm.weight" not in sd or "feature_extractor.conv_layers.0.conv.bias" not in sd:
            raise ValueError("HubertEncoder supports the hubert-large layout (feat_extract_norm='layer', conv_bias=True) the reference loads")
        self.ctx, self.heads, self.eps = ctx, heads, eps
        fe = "feature_extractor.conv_layers"
        self.C = int(_np(sd[f"{fe}.0.conv.weight"]).shape[0])
        self.conv0_w = ctx.upload(_np(sd[f"{fe}.0.conv.weight"]).reshape(self.C, CONV_KERNEL[0]).astype(np.float32))
        self.conv0_b = ctx.upload(_np(sd[f"{fe}.0.conv.bias"]).astype(np.float32))
        # conv1d(k) as 1 x k convs over a (1, 1, T, C) NHWC tensor
        self.convs = [ConvWeight(ctx, _np(sd[f"{fe}.{i}.conv.weight"])[:, :, None, :], _np(sd[f"{fe}.{i}.conv.bias"]), tap_major=False)
                      for i in range(1, 7)]
        self.conv_ln = [_Norm(ctx, sd, f"{fe}.{i}.layer_norm") for i in range(7)]
        self.proj_ln = _Norm(ctx, sd, "feature_projection.layer_norm")
        self.proj = ConvWeight(ctx, _np(sd["feature_projection.projection.weight"]), _np(sd["feature_projection.projection.bias"]), tap_major=False)
        self.D = self.proj.cout
        pc = "encoder.pos_conv_embed.conv"
        if f"{pc}.parametrizations.weight.original0" in sd:
            g, v = _np(sd[f"{pc}.parametrizations.weight.original0"]), _np(sd[f"{pc}.parametrizations.weight.original1"])
        elif f"{pc}.weight_g" in sd:
            g, v = _np(sd[f"{pc}.weight_g"]), _np(sd[f"{pc}.weight_v"])
        else:
            g, v = None, _np(sd[f"{pc}.weight"])
        if g is not None:                                              # weight_norm(dim=2): w[:, :, k] = g[k] * v[:, :, k] / ||v[:, :, k]||
            v = v * (g / np.sqrt((v.astype(np.float64) ** 2).sum((0, 1), keepdims=True))).astype(np.float32)
        if v.shape != (self.D, self.D // POS_GROUPS, POS_K) or self.D // POS_GROUPS != 64:
            raise ValueError(f"positional conv must be ({self.D},{self.D // POS_GROUPS},{POS_K}) with 64 channels per group, got {v.shape}")
        self.pos_w = ctx.upload(np.ascontiguousarray(v.transpose(0, 2, 1)).astype(np.float16))      # [D][K][D/G]
        self.pos_b = ctx.upload(_np(sd[f"{pc}.bias"]).astype(np.float32))
        if "encoder.layers.0.attention.q_proj.weight" not in sd:
            raise ValueError("no encoder layers in the state_dict")
        self.layers = []
        i = 0
        while f"encoder.layers.{i}.attention.q_proj.weight" in sd:
            p = f"encoder.layers.{i}"
            self.layers.append({
                "ln1": _Norm(ctx, sd, p + ".layer_norm"), "attn": _HAttn(ctx, sd, p + ".attention", self.D, heads),
                "ln2": _Norm(ctx, sd, p + ".final_layer_norm"),
                "fc1": ConvWeight(ctx, _np(sd[p + ".feed_forward.intermediate_dense.weight"]), _np(sd[p + ".feed_forward.intermediate_dense.bias"]),
                                  tap_major=False),
                "fc2": ConvWeight(ctx, _np(sd[p + ".feed_forward.output_dense.weight"]), _np(sd[p + ".feed_forward.output_dense.bias"]),
                                  tap_major=False)})
            i += 1
        self.ln_post = _Norm(ctx, sd, "encoder.layer_norm")
        ctx.sync()

    def emit(self, b: Builder, pcm: DevTensor, n: int, stats: DevTensor, G: int = 1) -> DevTensor:
        """pcm: float32 [G][n] raw 16 kHz samples of G windows, stats [G][4] -> last_hidden_state (G * conv_frames(n), D) fp16, window g
        in rows [g*T, (g+1)*T) (HubertModel.forward on the processor-normalised input; stable-LayerNorm encoder: hidden +=
        pos_conv(hidden); pre-LN layers; final LayerNorm).  Each window is normalised with its own statistics, the conv stack runs
        with N = G images, row-wise ops run over G*T rows and attention with batch G, so no window sees another's samples or keys."""
        ctx, C, D = b.ctx, self.C, self.D
        T = (n - CONV_KERNEL[0]) // CONV_STRIDE[0] + 1
        h = b.new(G, 1, T, C)
        ctx.hubert_conv0(pcm, n, self.conv0_w, self.conv0_b, C, stats, h, G=G)
        for i in range(7):
            if i > 0:
                k, s = CONV_KERNEL[i], CONV_STRIDE[i]
                T2 = (T - k) // s + 1
                h2 = b.new(G, 1, T2, C)
                ctx.conv(h, self.convs[i - 1], h2, N=G, IH=1, IW=T, OH=1, OW=T2, stride=(1, s), pad=(0, 0))
                h, T = h2, T2
            y = b.new(G, 1, T, C)
            ctx.layernorm(h, G * T, C, self.eps, self.conv_ln[i].gamma, self.conv_ln[i].beta, y)  # HubertLayerNormConvLayer
            ctx.eltwise(y, None, G * T * C, 8, 1, y)                                              # GELU
            h = y
        x = DevTensor(h.ptr, (G * T, C))
        x = b.linear(b.layernorm(x, self.proj_ln, self.eps), self.proj)                           # HubertFeatureProjection
        xp = b.new(G * T, D)
        ctx.hubert_pos_conv(x, T, D, POS_GROUPS, POS_K, self.pos_w, self.pos_b, xp, G=G)          # + positional conv embedding
        x = xp
        for L in self.layers:                                                                     # HubertEncoderLayerStableLayerNorm
            x = b.attention(L["attn"], b.layernorm(x, L["ln1"], self.eps), G, T, res=x)
            f = b.linear(b.layernorm(x, L["ln2"], self.eps), L["fc1"])
            ctx.eltwise(f, None, f.rows * f.C, 8, 1, f)
            x = b.linear(f, L["fc2"], res=x)
        return b.layernorm(x, self.ln_post, self.eps)


def window_samples(batch: int, stride_left: int, stride_right: int) -> tuple:
    """HubertASR's window of (stride_left + stride_right + 2 * batch) 20 ms chunks -> (samples n, conv frames Tc, expected rows T).
    Always below the reference's 320000-sample clip length, so the single-clip branch of audio2feature.py:38-47 applies."""
    n = (stride_left + stride_right + 2 * int(batch)) * 320
    if not 400 <= n < 320000:
        raise ValueError("audio window must be 400 .. 319999 samples")
    Tc, T = conv_frames(n), (n - 80) // 320
    if abs(Tc - T) > 1:
        raise ValueError("conv frame count and expected_T differ by more than one (audio2feature.py:52)")
    return n, Tc, T


class HubertBatchFeatures(GraphSession):
    """get_hubert_from_16k_speech + HubertASR's window gather for up to G sessions at once: G PCM windows of the same layout -> G x
    (B, 16, D) features, ONE CUDA graph of one encoder forward over the G windows stacked on the row dimension.  The window is
    (stride_left + stride_right + 2 * batch) 20 ms chunks (HubertASR keeps exactly that many, hubert.py:30-48).  At B = 16 a window
    is ~51 tokens, under half of one 128-row GEMM tile, and every window re-reads the encoder's weights: G windows per forward share
    both.  Each window keeps its own normalisation statistics, positional-conv padding and attention keys, so a session's features do
    not depend on which other windows share its round.  A call with k < G windows is a partial round: groups [k, G) keep their
    last window (zeros before the first call) and their output is not read.  out_nhwc (optional): fp16 [G][B][D][16], written
    besides the float32 features.  `batch` / `infer_slots` make it a mux for plugin.batcher.CrossSessionBatcher (a request is one
    session's PCM window)."""

    def __init__(self, enc: HubertEncoder, batch: int, groups: int, stride_left: int = 10, stride_right: int = 10, *,
                 out_nhwc: Optional[DevTensor] = None, ctx: Optional[Ctx] = None):
        self.enc, self.B, self.G = enc, int(batch), int(groups)
        if self.G < 1:
            raise ValueError("groups must be >= 1")
        self.batch = self.G                                  # CrossSessionBatcher: requests per engine call
        super().__init__(ctx)
        try:
            ctx = self.ctx
            self.n, self.Tc, self.T = window_samples(self.B, stride_left, stride_right)
            self.pcm = self.alloc((self.G, self.n), np.float32, zero=True)
            self.stats = self.alloc((self.G, 4), np.float32, zero=True)
            self.out = self.alloc((self.G, self.B, ROWS, enc.D), np.float32, zero=True)
            self.out_nhwc = out_nhwc
            self.start = stride_left / 2.0

            def emit(b: Builder):
                self.hidden = enc.emit(b, self.pcm, self.n, self.stats, G=self.G)
                ctx.hubert_slice(self.hidden, self.Tc, self.T, enc.D, self.B, ROWS, self.start, 2.0, WIN[0], self.out, self.out_nhwc,
                                 G=self.G)

            self.capture(emit)
        except BaseException:
            self.close()
            raise

    def _stage(self, pcms: Sequence[np.ndarray]) -> int:
        """Copy windows 0 .. k-1 to the device; -> k."""
        k = len(pcms)
        if not 1 <= k <= self.G:
            raise ValueError(f"1..{self.G} windows per call, got {k}")
        x = np.stack([np.ascontiguousarray(p, np.float32).reshape(-1) for p in pcms])
        if x.shape[1] != self.n:
            raise ValueError(f"expected windows of {self.n} samples, got {x.shape[1]}")
        self.ctx.h2d(DevTensor(self.pcm.ptr, (k, self.n), np.float32), x, sync=False)
        return k

    def run_async(self, pcms: Sequence[np.ndarray]) -> int:
        """Stage windows 0 .. k-1 and launch the graph; -> k."""
        k = self._stage(pcms)
        self.graph.launch()
        return k

    def run_groups(self, pcms: Sequence[np.ndarray]) -> List[np.ndarray]:
        """-> per window its (B, 16, D) float32 features: the list HubertASR.run_step queues (stacked) for that window alone."""
        with self.ctx.lock:
            k = self._stage(pcms)
            self.graph.launch()
            out = self.ctx.download(DevTensor(self.out.ptr, (k, self.B, ROWS, self.enc.D), np.float32))
        return [out[g] for g in range(k)]

    infer_slots = run_groups

    def hidden_states(self) -> np.ndarray:
        """-> the encoder's last hidden state (G * Tc, D) fp16 of the last launch."""
        with self.ctx.lock:
            return self.ctx.download(self.hidden)


class HubertFeatures(HubertBatchFeatures):
    """HubertBatchFeatures for one session (G = 1): PCM buffer -> (B, 16, D) features, one CUDA graph."""

    def __init__(self, enc: HubertEncoder, batch: int, stride_left: int = 10, stride_right: int = 10, out_nhwc: Optional[DevTensor] = None,
                 ctx: Optional[Ctx] = None):
        super().__init__(enc, batch, 1, stride_left, stride_right, out_nhwc=out_nhwc, ctx=ctx)

    def run_async(self, pcm: Optional[np.ndarray] = None):
        """Stage `pcm` (None: keep the last window) and launch the graph."""
        if pcm is not None:
            self._stage([pcm])
        self.graph.launch()

    def run(self, pcm: np.ndarray) -> np.ndarray:
        """-> (B, 16, D) float32: the list HubertASR.run_step queues (stacked)."""
        return self.run_groups([pcm])[0]


def gflop_per_window(n_samples: int, layers: int = 24, d_model: int = 1024, ffn: int = 4096, conv_dim: int = 512) -> float:
    """Algorithmic GFLOP (2 x MAC) of one HubertModel forward over n_samples of 16 kHz audio."""
    fl, t, cin = 0.0, n_samples, 1
    for k, s in zip(CONV_KERNEL, CONV_STRIDE):
        t = (t - k) // s + 1
        fl += 2.0 * t * conv_dim * cin * k
        cin = conv_dim
    fl += 2.0 * t * conv_dim * d_model + 2.0 * t * d_model * (d_model // POS_GROUPS) * POS_K
    fl += layers * (2.0 * t * (4 * d_model * d_model + 2 * d_model * ffn) + 4.0 * t * t * d_model)
    return fl / 1e9
