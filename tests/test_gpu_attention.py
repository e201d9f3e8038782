"""GPU: the fused attention kernel (csrc/attn_fused.cu through ltb_op_attention, V^T produced by transpose_heads) against
softmax(s Q K^T) V in float64 over the keys [0, valid) of every (batch, head), computed from the same fp16 inputs.

Error bound per output element (query i, channel c), p_j the exact probabilities and v_j the fp16 V rows of the valid keys:

    |out - ref| <= 1.25 * ( 2^-11 |ref| + 2^-25                                   fp16 output rounding (normal / subnormal)
                          + (2^-11 + expm1(2 eps_s) + eps_f) sum_j p_j |v_jc|    P rounded to fp16 before the PV wgmma; scores
                          + n_valid 2^-25 max_j |v_jc| )                           probabilities in the fp16 subnormal range

  * eps_s = s d 2^-23 max_j sum_i |q_i k_ji| is twice the worst case of the d-term fp32 score accumulation, in scaled-logit units.
    A logit off by at most eps_s moves its exp() by a factor exp(+-eps_s) and the row sum l by the same factor, so every
    probability is within a factor exp(+-2 eps_s) of p_j.
  * eps_f = (9 nkt + 50) 2^-24 + (nkt + 1) 2^-22 + 2^-17 covers the rest of the fp32 work over nkt 128-key tiles: the PV
    accumulation (8 nkt + 16 sequential adds) and the running sum l (at most 34 + nkt adds) at 2^-24 each, ex2.approx (relative
    2^-22) for the numerator and each rescale of l, and the roundings of scale*log2(e) and of (s - m) * scale*log2(e).
  * 1.25 absorbs the second-order terms the linearisation drops.

Sliced inputs: pitch padding and the channels before the first head hold SENT_IN; the output is a channel slice of a wider
buffer pre-filled with SENT_OUT, and every element outside [0, B*nq) x [off, off + H*d) must keep its bits.  V channel 0 is 1.0
for every key, so that output channel is sum_j P_j and must be within 2^-10 + n_valid 2^-25 of 1."""
import math

import numpy as np
import pytest

SENT_IN = 512.0
SENT_OUT = -3.25
OUT_OFF = 8           # the output slice starts 16 bytes into each row
SAFETY = 1.25


def _ceil16(x):
    return (x + 15) // 16 * 16


# B, H, nq, kv_rows, valid, d, n_pad, layout, scale: every instance with B > 1, nq % 128 != 0, valid < kv_rows, valid % 16 != 0 and
# at least three key tiles (D 144 / 160: the one-stage K ring wraps between pass 1 and pass 2)
GENERIC = [
    (3, 4, 261, 405, 389, 16, 408, "sep", 0.37),
    (2, 3, 390, 390, 357, 32, 400, "fused", 0.21),
    (2, 8, 333, 300, 291, 48, 304, "sep", 40 ** -0.5),      # MuseTalk pads d 40 to 48 and keeps 40^-0.5
    (4, 2, 129, 520, 515, 64, 528, "sep", 0.125),
    (2, 5, 257, 385, 383, 80, 392, "sep", 0.1),
    (3, 2, 300, 300, 297, 96, 304, "fused", 0.102),
    (2, 3, 200, 401, 387, 112, 408, "sep", 0.0945),
    (2, 2, 383, 383, 370, 128, 384, "fused", 0.0884),
    (2, 2, 250, 530, 517, 144, 536, "sep", 0.0833),
    (3, 2, 420, 420, 401, 160, 432, "fused", 0.079),
]
# the shapes the engine launches
PRODUCTION = (
    [(G, 16, T, T, T, 64, _ceil16(T), "fused", 0.125) for G in (1, 3, 8) for T in (27, 51, 83)]   # HuBERT grouped, batch 4 / 16 / 32
    + [(1, 6, 1500, 1500, 1500, 64, 1504, "fused", 0.125),                                        # Whisper encoder
       (2, 8, 1024, 1024, 1024, 48, 1024, "fused", 40 ** -0.5),                                    # MuseTalk self-attention, 32x32
       (1, 8, 4096, 4096, 4096, 48, 4096, "fused", 40 ** -0.5),                                    # MuseTalk self-attention, 64x64
       (2, 8, 256, 64, 50, 80, 64, "sep", 80 ** -0.5),                                             # MuseTalk cross-attention
       (2, 8, 64, 64, 64, 160, 64, "fused", 160 ** -0.5),                                          # 1280-channel levels
       (2, 8, 256, 256, 256, 160, 256, "fused", 160 ** -0.5)])
CASES = GENERIC + PRODUCTION
INSTANCES = (16, 32, 48, 64, 80, 96, 112, 128, 144, 160)


def _case_id(c):
    B, H, nq, kv, valid, d, n_pad, layout, _s = c
    return f"d{d}_B{B}_H{H}_nq{nq}_kv{kv}_v{valid}_pad{n_pad}_{layout}"


# ------------------------------------------------------------------------------------------------ completeness (CPU)
def test_cases_cover_every_compiled_instance():
    """Every attn_fused_kernel<D> in the built object has a row in CASES, and CASES names no instance that is not compiled."""
    from kernel_instances import compiled_instances
    compiled = {v[0] for v in compiled_instances("attn_fused.o", "attn_fused_kernel")}
    assert compiled == {c[5] for c in CASES} == set(INSTANCES), (sorted(compiled), sorted({c[5] for c in CASES}))


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def ctx():
    from livetalking_b200 import engine
    from livetalking_b200.ops import Ctx
    engine.set_device(0)
    c = Ctx()
    yield c
    c.close()


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint16)


def _inputs(rng, B, H, nq, kv_rows, d):
    Q = rng.standard_normal((B, nq, H, d)).astype(np.float16)
    K = rng.standard_normal((B, kv_rows, H, d)).astype(np.float16)
    V = (2 * rng.standard_normal((B, kv_rows, H, d))).astype(np.float16)
    V[..., 0] = 1.0                      # row-sum channel
    return Q, K, V


class _Attn:
    """Host buffers of one launch in either layout, uploaded; run() launches transpose_heads (unless vt is given) + attention."""

    def __init__(self, ctx, Q, K, V, layout, pad=8):
        B, nq, H, d = Q.shape
        kv_rows = K.shape[1]
        self.ctx, self.B, self.H, self.nq, self.kv_rows, self.d = ctx, B, H, nq, kv_rows, d
        Hd = H * d
        if layout == "fused":
            assert nq == kv_rows
            self.q_pitch = self.kv_pitch = 3 * Hd + pad
            buf = np.full((B * nq, self.q_pitch), SENT_IN, np.float16)
            buf[:, :Hd], buf[:, Hd:2 * Hd], buf[:, 2 * Hd:3 * Hd] = (a.reshape(B * nq, Hd) for a in (Q, K, V))
            self.bufs = [buf]
            t = ctx.upload(buf)
            self.dev = [t]
            self.q_ptr, self.k_ptr, self.v_ptr = t.offset(0), t.offset(Hd), t.offset(2 * Hd)
        else:
            self.q_pitch, self.kv_pitch = 8 + Hd + pad, 8 + 2 * Hd + pad
            qb = np.full((B * nq, self.q_pitch), SENT_IN, np.float16)
            qb[:, 8:8 + Hd] = Q.reshape(B * nq, Hd)
            kvb = np.full((B * kv_rows, self.kv_pitch), SENT_IN, np.float16)
            kvb[:, 8:8 + Hd], kvb[:, 8 + Hd:8 + 2 * Hd] = K.reshape(B * kv_rows, Hd), V.reshape(B * kv_rows, Hd)
            self.bufs = [qb, kvb]
            qt, kvt = ctx.upload(qb), ctx.upload(kvb)
            self.dev = [qt, kvt]
            self.q_ptr, self.k_ptr, self.v_ptr = qt.offset(8), kvt.offset(8), kvt.offset(8 + Hd)
        self.out_pitch = Hd + 16
        self.obuf = np.full((B * nq + 2, self.out_pitch), SENT_OUT, np.float16)     # two rows past B*nq must stay untouched
        self.out = ctx.upload(self.obuf)

    def run(self, valid, n_pad, scale, vt_host=None):
        from livetalking_b200.ops import DevTensor
        ctx, B, H, d = self.ctx, self.B, self.H, self.d
        if vt_host is None:
            vt = ctx.alloc((B * H, d, n_pad), np.float16, zero=True)
            ctx.transpose_heads(self.v_ptr, B, self.kv_rows, self.kv_pitch, H, d, n_pad, vt)
        else:
            vt = ctx.upload(vt_host)
        ctx.h2d(self.out, self.obuf)
        o = DevTensor(self.out.offset(OUT_OFF), (B * self.nq, H * d), pitch=self.out_pitch)
        ctx.attention(self.q_ptr, self.q_pitch, self.k_ptr, self.kv_pitch, self.kv_rows, vt, n_pad, B, H, self.nq, valid, d, scale, o)
        got = ctx.download(self.out)
        ctx.free(vt)
        for t, b in zip(self.dev, self.bufs):
            assert np.array_equal(_bits(ctx.download(t)), _bits(b)), "attention or transpose_heads wrote into its input"
        written = np.zeros(got.shape, bool)
        written[:B * self.nq, OUT_OFF:OUT_OFF + H * d] = True
        changed = (_bits(got) != _bits(self.obuf)) & ~written
        assert not changed.any(), f"{int(changed.sum())} elements outside the output slice changed, first at {np.argwhere(changed)[0]}"
        return got[:B * self.nq, OUT_OFF:OUT_OFF + H * d].reshape(B, self.nq, H, d)

    def close(self):
        for t in self.dev + [self.out]:
            self.ctx.free(t)


def _reference(Q, K, V, valid, scale, eps_s_zero=False, eps_s_extra=None):
    """float64 softmax(s Q K^T) V over keys [0, valid) and the bound of the module docstring (without SAFETY), both (B, nq, H, d).
    eps_s_zero: the scores are exact in fp32 (see test_extreme_rows); eps_s_extra(q, k) -> per-row logit error added to eps_s."""
    B, nq, H, d = Q.shape
    s = float(np.float32(scale))
    nkt = (valid + 127) // 128
    eps_f = (9 * nkt + 50) * 2.0 ** -24 + (nkt + 1) * 2.0 ** -22 + 2.0 ** -17
    ref = np.empty(Q.shape)
    bound = np.empty(Q.shape)
    for b in range(B):
        for h in range(H):
            q = Q[b, :, h].astype(np.float64)
            k = K[b, :valid, h].astype(np.float64)
            v = V[b, :valid, h].astype(np.float64)
            lg = s * (q @ k.T)
            e = np.exp(lg - lg.max(1, keepdims=True))
            p = e / e.sum(1, keepdims=True)
            r = p @ v
            eps_s = np.zeros(nq) if eps_s_zero else s * d * 2.0 ** -23 * (np.abs(q) @ np.abs(k).T).max(1)
            if eps_s_extra is not None:
                eps_s = eps_s + eps_s_extra(q, k)
            ref[b, :, h] = r
            bound[b, :, h] = (2.0 ** -11 * np.abs(r) + 2.0 ** -25 + (2.0 ** -11 + np.expm1(2 * eps_s) + eps_f)[:, None] * (p @ np.abs(v))
                              + valid * 2.0 ** -25 * np.abs(v).max(0))
    return ref, bound


def _check(got, ref, bound, what):
    got = got.astype(np.float64)
    assert np.isfinite(got).all(), f"{what}: non-finite output"
    ratio = np.abs(got - ref) / (SAFETY * bound)
    worst = float(ratio.max())
    print(f"{what}: worst err/bound {worst:.3f}")
    assert worst <= 1.0, (f"{what}: {int((ratio > 1).sum())} of {ratio.size} outside the bound; worst err/bound {worst:.2f} at "
                          f"{np.unravel_index(ratio.argmax(), ratio.shape)}")
    return worst


def _check_row_sum(got, valid, what):
    err = float(np.abs(got[..., 0].astype(np.float64) - 1.0).max())
    assert err <= 2.0 ** -10 + valid * 2.0 ** -25, f"{what}: sum_j P_j off by {err:.3g}"


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[_case_id(c) for c in CASES])
def test_attention_matches_float64(ctx, case):
    B, H, nq, kv_rows, valid, d, n_pad, layout, scale = case
    rng = np.random.default_rng(B * 7919 + H * 131 + nq * 17 + kv_rows + valid * 3 + d)
    Q, K, V = _inputs(rng, B, H, nq, kv_rows, d)
    a = _Attn(ctx, Q, K, V, layout, pad=8 if (nq + d) % 2 else 0)
    got = a.run(valid, n_pad, scale)
    a.close()
    ref, bound = _reference(Q, K, V, valid, scale)
    _check(got, ref, bound, _case_id(case))
    _check_row_sum(got, valid, _case_id(case))


def _needle_positions(valid):
    """Keys 0, 127, 128, valid - 1 and the middle of the last tile's valid keys (five distinct keys when valid > 384)."""
    last = (valid - 1) // 128 * 128
    return sorted({0, 127, 128, valid - 1, (last + valid - 1) // 2})


@pytest.mark.gpu
@pytest.mark.parametrize("d", INSTANCES)
def test_needle_keys_return_their_value_row(ctx, d):
    """Query row i_c has Q[i_c, c] = A and key j_c has K[j_c, c] = A in needle channel c (every other Q / K entry of the needle
    channels is 0), with s A^2 more than 40 above every other logit of the row: every other probability is below e^-40, flushes to
    0 in fp16, l rounds to exactly 1, and the output row must be V[j_c] bit for bit.  Needles at keys 0, 127, 128 (first key of the
    second tile), valid - 1 and inside the last tile."""
    B, H, nq, kv_rows, valid, n_pad, scale = 2, 2, 300, 520, 517, 528, 0.11
    rng = np.random.default_rng(d)
    Q, K, V = _inputs(rng, B, H, nq, kv_rows, d)
    needles = _needle_positions(valid)
    assert len(needles) == 5 and needles[-2] // 128 == needles[-1] // 128 == (valid - 1) // 128 and needles[-2] != valid - 1
    rows = [0, 77, 128, 255, 299]
    nc = len(needles)
    Q[..., :nc] = 0
    K[..., :nc] = 0
    rest = scale * np.abs(np.einsum("bihc,bjhc->bhij", Q.astype(np.float32), K.astype(np.float32))).max()
    A = np.float16(math.ceil(math.sqrt((40 + 2 * rest) / scale)))
    for c, (i, j) in enumerate(zip(rows, needles)):
        Q[:, i, :, c] = A
        K[:, j, :, c] = A
    a = _Attn(ctx, Q, K, V, "sep")
    got = a.run(valid, n_pad, scale)
    a.close()
    for i, j in zip(rows, needles):
        assert np.array_equal(_bits(got[:, i]), _bits(V[:, j])), f"needle at key {j} (query {i}): output is not V[{j}]"
    ref, bound = _reference(Q, K, V, valid, scale)
    _check(got, ref, bound, f"needles d{d}")


@pytest.mark.gpu
@pytest.mark.parametrize("case", [(2, 2, 150, 400, 333, 64, 416), (2, 2, 150, 400, 334, 64, 416), (2, 2, 150, 400, 333, 160, 416),
                                  (2, 2, 150, 400, 334, 160, 416), (2, 8, 256, 64, 50, 80, 64)],
                         ids=["d64_3tiles_odd", "d64_3tiles_even", "d160_3tiles_odd", "d160_3tiles_even", "d80_cross"])
def test_masked_keys_get_probability_zero(ctx, case):
    """Keys [valid, kv_rows) carry the largest logits of every row (channel 1: Q = 4, K = 2000 there), and V^T, uploaded
    directly, holds 3e4 in columns [valid, n_pad).  A masked key that leaks into either pass, or into P V, moves the output far out
    of the bound (and the row sum off 1).  Each thread handles an even and an odd key column with separate compares, so the first
    masked key of the last tile is put at both parities."""
    B, H, nq, kv_rows, valid, d, n_pad = case
    scale = 0.09
    rng = np.random.default_rng(sum(case))
    Q, K, V = _inputs(rng, B, H, nq, kv_rows, d)
    Q[..., 1] = 4
    K[:, valid:, :, 1] = 2000
    vt = np.full((B, H, d, n_pad), 3e4, np.float16)
    vt[..., :valid] = V[:, :valid].transpose(0, 2, 3, 1)
    a = _Attn(ctx, Q, K, V, "sep")
    got = a.run(valid, n_pad, scale, vt_host=vt.reshape(B * H, d, n_pad))
    a.close()
    ref, bound = _reference(Q, K, V, valid, scale)
    _check(got, ref, bound, f"mask {case}")
    _check_row_sum(got, valid, f"mask {case}")


EXTREMES = ["fp16_limits", "uniform_keys", "zero_q", "valid_1", "nq_1"]


@pytest.mark.gpu
@pytest.mark.parametrize("d", [64, 160])
@pytest.mark.parametrize("kind", EXTREMES)
def test_extreme_rows(ctx, kind, d):
    """fp16_limits: Q entries +-65504, K entries in {+-32768, +-16384, 0}.  Every product is 2047 * 2^19 * {0, +-1, +-2} and every
    partial sum of a score is a multiple of 2^19 below 2^39, so the fp32 scores (up to 3.4e11) are exact and eps_s = 0; distinct
    scores differ by at least 1.07e9, so P is exactly uniform over the row's maxima.  uniform_keys: every key equal (P = 1/valid).
    zero_q: Q = 0 (uniform P).  valid_1: one valid key of 17 rows, the output is V[0] bit for bit.  nq_1: one query per batch."""
    B, H, nq, kv_rows, valid, n_pad, scale = 2, 2, 200, 300, 290, 304, 0.125
    if kind == "valid_1":
        nq, kv_rows, valid, n_pad = 40, 17, 1, 32
    if kind == "nq_1":
        B, nq = 3, 1
    rng = np.random.default_rng(EXTREMES.index(kind) * 1000 + d)
    Q, K, V = _inputs(rng, B, H, nq, kv_rows, d)
    if kind == "fp16_limits":
        Q = rng.choice(np.array([65504, -65504], np.float16), Q.shape)
        K = rng.choice(np.array([32768, -32768, 16384, -16384, 0], np.float16), K.shape)
    elif kind == "uniform_keys":
        K[:] = K[:, :1]
    elif kind == "zero_q":
        Q[:] = 0
    a = _Attn(ctx, Q, K, V, "sep")
    got = a.run(valid, n_pad, scale)
    a.close()
    if kind == "valid_1":
        assert np.array_equal(_bits(got), _bits(np.broadcast_to(V[:, :1], got.shape))), "one valid key: the output must be V[0]"
    ref, bound = _reference(Q, K, V, valid, scale, eps_s_zero=(kind == "fp16_limits"))
    _check(got, ref, bound, f"{kind} d{d}")
    _check_row_sum(got, valid, f"{kind} d{d}")


@pytest.mark.gpu
def test_batches_are_independent_and_launches_deterministic(ctx):
    """HuBERT grouped layout (G = 8 windows, T = 83): two launches give identical bits, and new Q / K / V rows for batch 1 change
    batch 1's output and leave every other batch's bits alone."""
    B, H, T, d = 8, 16, 83, 64
    rng = np.random.default_rng(83)
    Q, K, V = _inputs(rng, B, H, T, T, d)
    a = _Attn(ctx, Q, K, V, "fused", pad=0)
    first = a.run(T, _ceil16(T), 0.125)
    assert np.array_equal(_bits(first), _bits(a.run(T, _ceil16(T), 0.125))), "two launches differ"
    a.close()
    Q2, K2, V2 = Q.copy(), K.copy(), V.copy()
    Qn, Kn, Vn = _inputs(np.random.default_rng(84), 1, H, T, T, d)
    Q2[1], K2[1], V2[1] = Qn[0], Kn[0], Vn[0]
    a = _Attn(ctx, Q2, K2, V2, "fused", pad=0)
    second = a.run(T, _ceil16(T), 0.125)
    a.close()
    assert not np.array_equal(_bits(second[1]), _bits(first[1]))
    for b in range(B):
        if b != 1:
            assert np.array_equal(_bits(second[b]), _bits(first[b])), f"batch {b} changed with batch 1's inputs"


@pytest.mark.gpu
@pytest.mark.parametrize("fused", [True, False], ids=["fused", "unfused"])
def test_builder_attention_hubert_grouped(ctx, monkeypatch, fused):
    """Builder.attention for a HuBERT _HAttn (16 heads x 64) at B = G = 3 windows of nq = 27 tokens, on the fused kernel and on the
    GEMM + softmax + GEMM path, against float64 multi-head attention with the same fp16 weights.

    The inputs make the qkv projection exact: x in {-4..4} / 4, W in {-128..128} / 1024, bias in multiples of 2^-12, so every
    product and partial sum is a multiple of 2^-12 below 2^7 and the fp32 accumulation is exact; the engine's fp16 qkv is then
    the float64 projection rounded to fp16, which is what the reference uses.  The attention output O (the Builder's temporary
    before the output projection) must be within the module bound; the unfused path stores the unscaled scores in fp16 first,
    which adds s 2^-11 max_j |q k_j| to eps_s.  Each window's keys [27, 32) are padding (TMA zero fill on the fused path, the next
    window's rows on the unfused one): a padded key that is not masked breaks that bound.  The block output must then equal
    O W_o^T + b_o + res from the engine's own fp16 O within 1024 2^-23 (|O| |W_o|^T + |b_o| + |res|) (fp32 accumulation) plus
    2^-11 |ref| + 2^-25 (fp16 rounding)."""
    from livetalking_b200.hubert import _HAttn
    from livetalking_b200.graph import Builder
    monkeypatch.setattr(Builder, "FUSE_ATTENTION", fused)
    G, T, H, d = 3, 27, 16, 64
    D = H * d
    rng = np.random.default_rng(27)
    sd = {}
    for n in ("q_proj", "k_proj", "v_proj"):
        sd[f"a.{n}.weight"] = (rng.integers(-128, 129, (D, D)) / 1024.0).astype(np.float32)
        sd[f"a.{n}.bias"] = (rng.integers(-512, 513, D) / 4096.0).astype(np.float32)
    sd["a.out_proj.weight"] = (rng.standard_normal((D, D)) / 32).astype(np.float32)
    sd["a.out_proj.bias"] = (0.1 * rng.standard_normal(D)).astype(np.float32)
    attn = _HAttn(ctx, sd, "a", D, H)
    x = (rng.integers(-4, 5, (G * T, D)) / 4.0).astype(np.float16)
    res = rng.standard_normal((G * T, D)).astype(np.float16)
    b = Builder(ctx)
    out_t = b.attention(attn, ctx.upload(x), G, T, res=ctx.upload(res))
    got = ctx.download(out_t).astype(np.float64)
    O_t = b.temps[b.temps.index(out_t) - 1]                  # the attention output the output projection reads
    assert O_t.shape == (G * T, D)
    O = ctx.download(O_t)
    for t in b.temps:
        ctx.free(t)

    xd = x.astype(np.float64)
    qkv = [(xd @ sd[f"a.{n}.weight"].astype(np.float64).T + sd[f"a.{n}.bias"]).astype(np.float16).reshape(G, T, H, d)
           for n in ("q_proj", "k_proj", "v_proj")]
    s = float(np.float32(d ** -0.5))
    extra = None if fused else (lambda q, k: s * 2.0 ** -11 * np.abs(q @ k.T).max(1))
    O_ref, bound = _reference(*qkv, T, s, eps_s_extra=extra)
    _check(O.reshape(G, T, H, d), O_ref, bound, f"Builder.attention {'fused' if fused else 'unfused'}: O")
    Od = O.astype(np.float64)
    Wo = sd["a.out_proj.weight"].astype(np.float16).astype(np.float64)
    bo = sd["a.out_proj.bias"].astype(np.float64)
    ref = Od @ Wo.T + bo + res
    bound = D * 2.0 ** -23 * (np.abs(Od) @ np.abs(Wo).T + np.abs(bo) + np.abs(res)) + 2.0 ** -11 * np.abs(ref) + 2.0 ** -25
    _check(got, ref, bound, f"Builder.attention {'fused' if fused else 'unfused'}: output projection")


@pytest.mark.gpu
def test_attention_refuses_unsupported_arguments(ctx):
    """Host-side checks: an unsupported head dim or pitch, valid outside [1, min(kv_rows, n_pad)], n_pad or out_pitch not a
    multiple of 8 must raise LtbError and launch nothing."""
    from livetalking_b200._capi import LtbError
    from livetalking_b200.ops import DevTensor
    buf = ctx.alloc((1 << 20,), np.float16, zero=True)
    vt = ctx.alloc((1 << 20,), np.float16, zero=True)
    ob = ctx.alloc((1 << 16,), np.float16, zero=True)
    ok =dict(d=64, q_pitch=3 * 128, kv_pitch=3 * 128, kv_rows=80, n_pad=80, valid=70, out_pitch=128)
    bad = [dict(d=8, q_pitch=24, kv_pitch=24, out_pitch=16), dict(d=40, q_pitch=240, kv_pitch=240, out_pitch=80),
           dict(d=176, q_pitch=3 * 352, kv_pitch=3 * 352, out_pitch=352),
           dict(q_pitch=3 * 128 + 4), dict(kv_pitch=3 * 128 + 4), dict(valid=0), dict(valid=81), dict(kv_rows=96, valid=88),
           dict(n_pad=84, valid=70), dict(out_pitch=132)]

    def call(a):
        o = DevTensor(ob.ptr, (2 * 50, 128), pitch=a["out_pitch"])
        ctx.attention(buf.ptr, a["q_pitch"], buf.ptr, a["kv_pitch"], a["kv_rows"], vt, a["n_pad"], 2, 2, 50, a["valid"], a["d"], 0.125, o)

    for change in bad:
        before = ctx.launch_count
        with pytest.raises(LtbError):
            call({**ok, **change})
        assert ctx.launch_count == before, change
    call(ok)
    ctx.sync()
