"""Whisper-tiny audio features on the B200 engine — replaces ``Audio2Feature.audio2feat``
(avatars/musetalk/whisper/audio2feature.py:106-117: HF ``WhisperFeatureExtractor`` + ``WhisperModel.encoder(...,
output_hidden_states=True)``) and the slicing of ``WhisperASR.run_step`` (avatars/audio_features/whisper.py:58-76).

Weights come from the HF ``WhisperModel`` state_dict (``encoder.*`` keys).  The encoder (2 conv1d + 4 pre-LN transformer
layers over 1500 steps) is assembled from the same engine ops as the UNet and captured into one CUDA graph together with
the log-mel kernels and the per-frame (50, 384) slicing.

``WhisperBatchFeatures`` runs G sessions' windows stacked on the row dimension, one encoder forward for all (cross-session mode);
``WhisperFeatures`` is its one-window form, one session's own extractor."""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import numpy as np

from .graph import Builder, GraphSession, _Norm, _np
from .ops import ConvWeight, Ctx, DevTensor

N_FRAMES, N_MELS, N_BINS, N_SAMPLES = 3000, 80, 201, 480000


def slaney_mel_filterbank() -> np.ndarray:
    """transformers.audio_utils.mel_filter_bank(201, 80, 0, 8000, 16000, norm='slaney', mel_scale='slaney').T -> (80, 201) f32."""
    def hz_to_mel(f):
        f = np.asarray(f, np.float64)
        return np.where(f >= 1000.0, 15.0 + np.log(np.maximum(f, 1e-12) / 1000.0) * (27.0 / np.log(6.4)), 3.0 * f / 200.0)

    def mel_to_hz(m):
        m = np.asarray(m, np.float64)
        return np.where(m >= 15.0, 1000.0 * np.exp(np.log(6.4) / 27.0 * (m - 15.0)), 200.0 * m / 3.0)

    fft_freqs = np.linspace(0, 8000, N_BINS)
    filt = mel_to_hz(np.linspace(hz_to_mel(0.0), hz_to_mel(8000.0), N_MELS + 2))
    fd = np.diff(filt)
    slopes = filt[None, :] - fft_freqs[:, None]
    down = -slopes[:, :-2] / fd[:-1]
    up = slopes[:, 2:] / fd[1:]
    fb = np.maximum(0.0, np.minimum(down, up))
    fb *= (2.0 / (filt[2:N_MELS + 2] - filt[:N_MELS]))[None, :]
    return np.ascontiguousarray(fb.T.astype(np.float32))


class _WAttn:
    self_attn = True

    def __init__(self, ctx: Ctx, sd, p: str, d_model: int, heads: int):
        self.heads, self.d, self.dp = heads, d_model // heads, d_model // heads
        assert self.d % 16 == 0
        w = np.concatenate([_np(sd[f"{p}.{n}.weight"]) for n in ("q_proj", "k_proj", "v_proj")], 0)
        b = np.concatenate([_np(sd[f"{p}.q_proj.bias"]), np.zeros(d_model, np.float32), _np(sd[f"{p}.v_proj.bias"])])   # k_proj has no bias
        self.qkv = ConvWeight(ctx, w, b, tap_major=False)
        self.out = ConvWeight(ctx, _np(sd[p + ".out_proj.weight"]), _np(sd[p + ".out_proj.bias"]), tap_major=False)


class WhisperEncoder:
    def __init__(self, ctx: Ctx, sd: Dict, d_model: int = 384, heads: int = 6, layers: int = 4):
        sd = {k[len("encoder."):] if k.startswith("encoder.") else k: v for k, v in sd.items() if not k.startswith("decoder.")}
        self.ctx, self.D, self.heads, self.L = ctx, d_model, heads, layers
        # conv1d(k=3) as 1x3 convs over a (1, 1, T, C) NHWC tensor
        self.conv1 = ConvWeight(ctx, _np(sd["conv1.weight"])[:, :, None, :], _np(sd["conv1.bias"]), tap_major=False)
        self.conv2 = ConvWeight(ctx, _np(sd["conv2.weight"])[:, :, None, :], _np(sd["conv2.bias"]), tap_major=False)
        self.pos = ctx.upload(_np(sd["embed_positions.weight"]).astype(np.float16))          # (1500, D)
        self.layers = []
        for i in range(layers):
            p = f"layers.{i}"
            self.layers.append({
                "ln1": _Norm(ctx, sd, p + ".self_attn_layer_norm"), "attn": _WAttn(ctx, sd, p + ".self_attn", d_model, heads),
                "ln2": _Norm(ctx, sd, p + ".final_layer_norm"),
                "fc1": ConvWeight(ctx, _np(sd[p + ".fc1.weight"]), _np(sd[p + ".fc1.bias"]), tap_major=False),
                "fc2": ConvWeight(ctx, _np(sd[p + ".fc2.weight"]), _np(sd[p + ".fc2.bias"]), tap_major=False)})
        self.ln_post = _Norm(ctx, sd, "layer_norm")
        self.fb = ctx.upload(slaney_mel_filterbank())
        ctx.sync()

    def emit(self, b: Builder, feats16: DevTensor, G: int = 1):
        """feats16: fp16 (G, 3000, 80) log-mel features of G windows -> the 5 hidden states HF returns, each (G * 1500, D) fp16, window
        g in rows [g*1500, (g+1)*1500).  The convs run with N = G images of 1 x 3000 (each zero-padded on its own), the positional add
        repeats per window, row-wise ops run over G*1500 rows and attention with batch G, so no op mixes rows of different windows.
        Ops are enqueued on the builder's ctx (the session's own stream); the weights live in self.ctx (read-only)."""
        ctx, D = b.ctx, self.D
        T = N_FRAMES
        x = DevTensor(feats16.ptr, (G, 1, T, N_MELS))
        h = b.new(G, 1, T, D)
        ctx.conv(x, self.conv1, h, N=G, IH=1, IW=T, OH=1, OW=T, pad=(0, 1))
        ctx.eltwise(h, None, G * T * D, 8, 1, h)                                         # GELU
        T2 = T // 2
        h2 = b.new(G, 1, T2, D)
        ctx.conv(h, self.conv2, h2, N=G, IH=1, IW=T, OH=1, OW=T2, stride=(1, 2), pad=(0, 1))
        ctx.eltwise(h2, None, G * T2 * D, 8, 1, h2)                                      # GELU
        x = b.new(G * T2, D)
        ctx.eltwise(h2, self.pos, G * T2 * D, T2 * D, 0, x)                              # + embed_positions
        hidden = [x]
        for i, L in enumerate(self.layers):
            x = b.attention(L["attn"], b.layernorm(x, L["ln1"]), G, T2, res=x)
            f = b.linear(b.layernorm(x, L["ln2"]), L["fc1"])
            ctx.eltwise(f, None, f.rows * f.C, 8, 1, f)
            x = b.linear(f, L["fc2"], res=x)
            hidden.append(x)
        hidden[-1] = b.layernorm(x, self.ln_post)                                         # HF applies the final LN to the last state
        return hidden


class WhisperBatchFeatures(GraphSession):
    """audio2feat + WhisperASR slicing for up to G sessions at once: G PCM windows of the same layout -> G x (B, 50, D) features, ONE
    CUDA graph (log-mel, one encoder forward over the G windows stacked on the row dimension, slice).  The encoder always runs over
    the 30-s padded window (1500 tokens), whatever B, so at small B each session's forward is mostly fixed cost: G windows per forward
    share the weights and fill wider GEMMs.  Each window keeps its own log-mel clamp, conv padding and attention keys, so a session's
    features do not depend on which other windows share its round.  A call with k < G windows is a partial round: groups [k, G) keep
    their last window (zeros before the first call) and their output is not read.  `batch` / `infer_slots` make it a mux for
    plugin.batcher.CrossSessionBatcher (a request is one session's PCM window).

    out (optional): fp16 [G][B][out_rows][D] the features are written to (50 of every out_rows rows), allocated here unless given.
    keep_hidden: also keep the float32 log-mel features in feats32, (G * 80, 3000) with window g in rows [g*80, (g+1)*80) like the
    hidden states (which are in `hidden` either way).
    ctx: this extractor's own stream + scratch (created here unless given): WhisperASR.run_step runs on the render thread
    concurrently with inference_batch on the inference thread (avatars/base_avatar.py:483-489 vs :366)."""

    def __init__(self, enc: WhisperEncoder, batch: int, groups: int, stride_left: int = 10, stride_right: int = 10, *,
                 out: Optional[DevTensor] = None, out_rows: int = 50, keep_hidden: bool = False, ctx: Optional[Ctx] = None):
        self.enc, self.B, self.G = enc, int(batch), int(groups)
        if self.G < 1:
            raise ValueError("groups must be >= 1")
        self.batch = self.G                                  # CrossSessionBatcher: requests per engine call
        self.n = (stride_left + stride_right + 2 * self.B) * 320
        if self.n > N_SAMPLES:
            raise ValueError("audio window longer than 30 s")
        super().__init__(ctx)
        try:
            ctx = self.ctx
            self.pcm = self.alloc((self.G, self.n), np.float32, zero=True)
            self.logspec = self.alloc((self.G, N_MELS * N_FRAMES), np.float32, zero=True)
            self.gmax = self.alloc((self.G,), np.int32, zero=True)
            self.feats16 = self.alloc((self.G, N_FRAMES, N_MELS), np.float16, zero=True)
            self.feats32 = self.alloc((self.G * N_MELS, N_FRAMES), np.float32, zero=True) if keep_hidden else None
            self.out_rows = out_rows
            self.out = out if out is not None else self.alloc((self.G, self.B, out_rows, enc.D), np.float16, zero=True)
            self.start = stride_left / 2.0

            def emit(b: Builder):
                ctx.whisper_logmel(self.pcm, self.n, enc.fb, self.logspec, self.gmax, self.feats16, self.feats32, G=self.G)
                self.hidden = enc.emit(b, self.feats16, G=self.G)
                ctx.whisper_slice(self.hidden, N_FRAMES // 2, enc.D, self.B, self.start, 2.0, self.out, self.out_rows, G=self.G)

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
        """-> per window its (B, 50, D) float16 features: the list WhisperASR.run_step queues (stacked) for that window alone."""
        with self.ctx.lock:
            k = self._stage(pcms)
            self.graph.launch()
            out = self.ctx.download(DevTensor(self.out.ptr, (k, self.B, self.out_rows, self.enc.D), np.float16))
        return [out[g, :, :50] for g in range(k)]

    infer_slots = run_groups


class WhisperFeatures(WhisperBatchFeatures):
    """WhisperBatchFeatures for one session (G = 1): PCM buffer -> (B, 50, D) features, one CUDA graph."""

    def __init__(self, enc: WhisperEncoder, batch: int, stride_left: int = 10, stride_right: int = 10, out: Optional[DevTensor] = None,
                 out_rows: int = 50, keep_hidden: bool = False, ctx: Optional[Ctx] = None):
        super().__init__(enc, batch, 1, stride_left, stride_right, out=out, out_rows=out_rows, keep_hidden=keep_hidden, ctx=ctx)

    def run_async(self, pcm: Optional[np.ndarray] = None):
        """Stage `pcm` (None: keep the last window) and launch the graph."""
        if pcm is not None:
            self._stage([pcm])
        self.graph.launch()

    def run(self, pcm: np.ndarray) -> np.ndarray:
        """-> (B, 50, D) float16, the list WhisperASR.run_step queues (stacked)."""
        return self.run_groups([pcm])[0]
