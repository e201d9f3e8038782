"""GPU: the HuBERT front-end kernels (csrc/hubert.cu through the grouped ltb_op_hubert_* entry points, G = 1 included) against
float64 references computed from the same inputs.

  * conv0: per-window statistics (Wav2Vec2's zero_mean_unit_var_norm) and conv layer 0 (1 -> 512, k 10, s 5) of the normalised window.
  * pos_conv: the 16-group, 128-tap positional convolution + SamePad trim + bias + erf-GELU + residual.
  * slice: HubertASR's window gather, bit for bit.

Every tolerance is derived in the test's docstring and multiplied by SAFETY = 1.25 for the second-order terms; the worst err / bound
is printed.  Outputs are pre-filled with SENT_OUT and one window past the last must keep its bits."""
import numpy as np
import pytest

SENT_IN = 512.0
SENT_OUT = -3.25
SAFETY = 1.25
C0 = 512


@pytest.fixture(scope="module")
def ctx():
    from livetalking_b200 import engine
    from livetalking_b200.ops import Ctx
    engine.set_device(0)
    c = Ctx()
    yield c
    c.close()


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint16 if a.dtype == np.float16 else np.uint32)


def _check(got, ref, bound, what):
    got = np.asarray(got, np.float64)
    assert np.isfinite(got).all(), f"{what}: non-finite output"
    ratio = np.abs(got - ref) / (SAFETY * bound)
    worst = float(ratio.max())
    print(f"{what}: worst err/bound {worst:.3f}")
    assert worst <= 1.0, (f"{what}: {int((ratio > 1).sum())} of {ratio.size} outside the bound; worst err/bound {worst:.2f} at "
                          f"{np.unravel_index(ratio.argmax(), ratio.shape)}")


# ------------------------------------------------------------------------------------------------ conv0 + statistics
def _window(kind, n, rng):
    if kind == "tone":
        t = np.arange(n) / 16000.0
        return (0.4 * np.sin(2 * np.pi * 230 * t) + 0.05 * rng.standard_normal(n)).astype(np.float32)
    if kind == "silence":
        return np.zeros(n, np.float32)
    if kind == "dc":
        return np.full(n, 0.3, np.float32)                 # variance zero, mean non-zero
    return rng.choice(np.array([1.0, -1.0], np.float32), n)   # full scale


KINDS = ["tone", "silence", "dc", "fullscale"]


def _conv0_ns():
    from livetalking_b200.hubert import window_samples
    return [window_samples(1, 10, 10)[0], window_samples(16, 10, 10)[0], 10, 1237]


CONV0_CASES = [(G, n, True) for n in _conv0_ns() for G in (1, 3)] + [(3, 1237, False)]


@pytest.mark.gpu
@pytest.mark.parametrize("G,n,with_bias", CONV0_CASES, ids=[f"G{c[0]}_n{c[1]}{'' if c[2] else '_nobias'}" for c in CONV0_CASES])
def test_conv0_matches_float64(ctx, G, n, with_bias):
    """stats[4g + 0] = mean and stats[4g + 1] = 1 / sqrt(var + 1e-7) of window g, accumulated in double and rounded to fp32: within
    2^-24 |ref| plus the double accumulation error, n 2^-53 mean|x| for the mean and (n + 2) 2^-54 E[x^2] / (var + 1e-7) relative for
    1/sqrt (half the relative error of var + 1e-7).  stats[4g + 2..3] are not written.

    out[g][t][c] = bias[c] + sum_k w[c][k] xn[5t + k], xn = (x - mean) * inv_std in fp32 from the fp32 statistics:
    |xn - xn_exact| <= 2^-22 inv_std (|x - mean| + |mean|) (the two statistics roundings and the two fp32 operations) plus |xn| times
    the relative error of inv_std above; ten fmas add
    10 2^-24 (|bias| + sum_k |w xn|); fp16 rounding 2^-11 |ref| + 2^-25.  (n = 10: one frame; n = 1237: (n - 10) % 5 != 0.)"""
    rng = np.random.default_rng(n * 10 + G)
    ci = _conv0_ns().index(n)
    x = np.stack([_window(KINDS[(ci + g) % 4], n, rng) for g in range(G)])
    w = (0.3 * rng.standard_normal((C0, 10))).astype(np.float32)
    bias = (0.2 * rng.standard_normal(C0)).astype(np.float32)
    T0 = (n - 10) // 5 + 1
    sbuf = np.full(4 * (G + 1), SENT_OUT, np.float32)
    obuf = np.full(((G + 1) * T0, C0), SENT_OUT, np.float16)
    st, ot = ctx.upload(sbuf), ctx.upload(obuf)
    ctx.hubert_conv0(ctx.upload(x), n, ctx.upload(w), ctx.upload(bias) if with_bias else None, C0, st, ot, G=G)
    stats, out = ctx.download(st), ctx.download(ot)
    written = np.zeros(sbuf.shape, bool)
    written[[4 * g + k for g in range(G) for k in (0, 1)]] = True
    assert np.array_equal(_bits(stats[~written]), _bits(sbuf[~written])), "statistics slots 2..3 or past the last window changed"
    assert np.array_equal(_bits(out[G * T0:]), _bits(obuf[G * T0:])), "written past the last window"
    xd = x.astype(np.float64)
    mean = xd.mean(1)
    ex2 = (xd ** 2).mean(1)
    var = ((xd - mean[:, None]) ** 2).mean(1)
    inv = 1.0 / np.sqrt(var + 1e-7)
    tol_m = 2.0 ** -24 * np.abs(mean) + n * 2.0 ** -53 * np.abs(xd).mean(1)
    tol_i = inv * (2.0 ** -24 + (n + 2) * 2.0 ** -54 * ex2 / (var + 1e-7))
    _check(stats[0:4 * G:4], mean, tol_m / SAFETY + 1e-300, f"conv0 mean G{G} n{n}")
    _check(stats[1:4 * G:4], inv, tol_i / SAFETY, f"conv0 inv_std G{G} n{n}")
    idx = 5 * np.arange(T0)[:, None] + np.arange(10)[None, :]             # (T0, 10)
    b = bias.astype(np.float64) if with_bias else np.zeros(C0)
    wd = w.astype(np.float64)
    for g in range(G):
        xn = (xd[g] - mean[g]) * inv[g]
        dxn = 2.0 ** -22 * inv[g] * (np.abs(xd[g] - mean[g]) + abs(mean[g])) + np.abs(xn) * tol_i[g] / inv[g]
        ref = xn[idx] @ wd.T + b                                          # (T0, C)
        mag = np.abs(xn[idx]) @ np.abs(wd).T
        bound = dxn[idx] @ np.abs(wd).T + 10 * 2.0 ** -24 * (np.abs(b) + mag) + 2.0 ** -11 * np.abs(ref) + 2.0 ** -25
        _check(out[g * T0:(g + 1) * T0], ref, bound, f"conv0 out G{G} n{n} window {g} ({KINDS[(ci + g) % 4]})")


# ------------------------------------------------------------------------------------------------ positional conv
D, GROUPS, K = 1024, 16, 128


@pytest.fixture(scope="module")
def pos_weights(ctx):
    rng = np.random.default_rng(128)
    w = (0.02 * rng.standard_normal((D, K, D // GROUPS))).astype(np.float16)     # engine layout [D][K][D/G]
    b = (0.3 * rng.standard_normal(D)).astype(np.float32)
    return w, b, ctx.upload(w), ctx.upload(b)


def _gelu(v):
    from scipy.special import erf
    return 0.5 * v * (1.0 + erf(v / np.sqrt(2.0)))


def _pos_ref(h, w, b):
    """h (T, D) -> float64 (ref, bound) of the test's docstring: conv1d(padding=64, groups=16) with the last step dropped."""
    T = h.shape[0]
    hd = h.astype(np.float64)
    pad = np.zeros((T + K, D))
    pad[K // 2:K // 2 + T] = hd
    acc = np.empty((T, D))
    mag = np.empty((T, D))
    cg = D // GROUPS
    cols = np.stack([pad[k:k + T] for k in range(K)], 1)                          # (T, K, D): row t, tap k = h[t + k - 64]
    for g in range(GROUPS):
        xg = cols[:, :, g * cg:(g + 1) * cg].reshape(T, K * cg)
        wg = w[g * cg:(g + 1) * cg].astype(np.float64).reshape(cg, K * cg)
        acc[:, g * cg:(g + 1) * cg] = xg @ wg.T
        mag[:, g * cg:(g + 1) * cg] = np.abs(xg) @ np.abs(wg).T
    pre = acc + b
    v = _gelu(pre)
    ref = hd + v
    bound = (1.13 * 8192 * 2.0 ** -24 * (mag + np.abs(b)) + 0.5 * np.abs(pre) * 2.0 ** -22 + 2.0 ** -20 * np.abs(v)
             + 2.0 ** -24 * np.abs(ref) + 2.0 ** -11 * np.abs(ref) + 2.0 ** -25)
    return ref, bound


POS_CASES = [(G, T) for T in (1, 27, 51, 64, 65, 150) for G in (1, 3)]


@pytest.mark.gpu
@pytest.mark.parametrize("G,T", POS_CASES, ids=[f"G{g}_T{t}" for g, t in POS_CASES])
def test_pos_conv_matches_float64(ctx, pos_weights, G, T):
    """out = h + gelu(bias + conv), per window with its own zero padding.  Bound: two fp32 chains of 4096 fmas each, so at most
    8192 2^-24 (sum |h w| + |bias|) on the pre-activation, times max |gelu'| = 1.13; erff's absolute error (at most 2^-22) enters
    gelu as 0.5 |pre| 2^-22, which matters where 1 + erf cancels (strongly negative pre-activations), and the remaining fp32 GELU
    arithmetic adds 2^-20 |gelu|; the residual add 2^-24 |ref|; fp16 rounding 2^-11 |ref| + 2^-25.  T > 64 runs the kernel's t0
    loop.  Windows other than 1 hold 64x larger values, so a tap that reaches across a window boundary shows in window 1; changing
    window 0 changes no other window's bits."""
    w, b, wt, bt = pos_weights
    rng = np.random.default_rng(G * 1000 + T)
    scale = np.where(np.arange(G) == 1, 1.0, 64.0) if G > 1 else np.ones(1)
    h = (rng.standard_normal((G, T, D)) * scale[:, None, None]).astype(np.float16)
    hbuf = np.full(((G + 1) * T, D), SENT_IN, np.float16)
    hbuf[:G * T] = h.reshape(G * T, D)
    obuf = np.full(((G + 1) * T, D), SENT_OUT, np.float16)
    ht, ot = ctx.upload(hbuf), ctx.upload(obuf)
    ctx.hubert_pos_conv(ht, T, D, GROUPS, K, wt, bt, ot, G=G)
    out = ctx.download(ot)
    assert np.array_equal(_bits(out[G * T:]), _bits(obuf[G * T:])), "written past the last window"
    assert np.array_equal(_bits(ctx.download(ht)), _bits(hbuf)), "input changed"
    for g in range(G):
        ref, bound = _pos_ref(h[g], w, b)
        _check(out[g * T:(g + 1) * T], ref, bound, f"pos_conv G{G} T{T} window {g}")
    if G > 1:
        h2 = hbuf.copy()
        h2[:T] = (rng.standard_normal((T, D)) * 64).astype(np.float16)
        ctx.h2d(ht, h2)
        ctx.h2d(ot, obuf)
        ctx.hubert_pos_conv(ht, T, D, GROUPS, K, wt, bt, ot, G=G)
        out2 = ctx.download(ot)
        assert not np.array_equal(_bits(out2[:T]), _bits(out[:T]))
        assert np.array_equal(_bits(out2[T:]), _bits(out[T:])), "changing window 0 changed another window's bits"


@pytest.mark.gpu
def test_pos_conv_refuses_unsupported_arguments(ctx, pos_weights):
    """In-place (h == out), K != 128 and D / groups != 64 are refused without a launch."""
    from livetalking_b200._capi import LtbError
    _w, _b, wt, bt = pos_weights
    h = ctx.alloc((64, D), np.float16, zero=True)
    out = ctx.alloc((64, D), np.float16, zero=True)
    for args in ((h, 64, D, GROUPS, K, wt, bt, h), (h, 64, D, GROUPS, 64, wt, bt, out), (h, 64, D, 32, K, wt, bt, out),
                 (h, 64, 1000, GROUPS, K, wt, bt, out)):
        before = ctx.launch_count
        with pytest.raises(LtbError):
            ctx.hubert_pos_conv(*args)
        assert ctx.launch_count == before
    ctx.hubert_pos_conv(h, 64, D, GROUPS, K, wt, bt, out)
    ctx.sync()


# ------------------------------------------------------------------------------------------------ window gather
SLICE_CASES = [(G, B, dt, mode) for G in (1, 3) for B in (1, 4, 16) for dt in (-1, 0, 1) for mode in ("both", "f32", "nhwc")]
EDGE_CASES = [(G, B, dt, st) for G in (1, 3) for B in (1, 4, 16) for dt in (-1, 0, 1) for st in ("zero", "end")]


def _slice_start(kind, T):
    """HubertASR's start = stride_left / 2: 0 (no left context: windows reach below row 0) or T / 2 (little right context: the
    last windows reach past row T - 1)."""
    return {"zero": 0.0, "end": T / 2.0}[kind]


def _slice_raw_rows(B, start):
    """The rows hubert_slice_kernel gathers before its clamp (fp32 arithmetic, exact for these starts)."""
    from livetalking_b200.hubert import ROWS, WIN
    return np.array([[int(int((b + start) * 2.0) - WIN[0] * 2.0) + r for r in range(ROWS)] for b in range(B)])


def _run_slice(ctx, G, B, dt, start, modes, seed):
    """Launch hubert_slice once per mode in `modes` and compare with window_rows applied to each window's zero-padded rows."""
    from livetalking_b200.hubert import ROWS, WIN, window_samples
    from oracle.ultralight_ref import window_rows
    _n, _tc, T = window_samples(B, 10, 10)
    Tc = T + dt
    rows = window_rows(T, B, start)
    assert np.array_equal(rows, np.clip(_slice_raw_rows(B, start), 0, T - 1))
    rng = np.random.default_rng(seed)
    hid = (rng.standard_normal((G, Tc, D)) * 3).astype(np.float16)
    hbuf = np.full(((G + 1) * Tc, D), SENT_IN, np.float16)
    hbuf[:G * Tc] = hid.reshape(G * Tc, D)
    ht = ctx.upload(hbuf)
    wants = []
    for g in range(G):
        padded = np.zeros((T, D), np.float16)
        m = min(T, Tc)
        padded[:m] = hid[g, :m]
        wants.append(padded[rows])                                                 # (B, 16, D)
    f_buf = np.full((G + 1, B, ROWS, D), SENT_OUT, np.float32)
    n_buf = np.full((G + 1, B, D, ROWS), SENT_OUT, np.float16)
    for mode in modes:
        ft, nt = ctx.upload(f_buf), ctx.upload(n_buf)
        ctx.hubert_slice(ht, Tc, T, D, B, ROWS, start, 2.0, WIN[0], ft if mode != "nhwc" else None, nt if mode != "f32" else None, G=G)
        got_f, got_n = ctx.download(ft), ctx.download(nt)
        ctx.free(ft)
        ctx.free(nt)
        for g, want in enumerate(wants):
            if mode != "nhwc":
                assert np.array_equal(_bits(got_f[g]), _bits(want.astype(np.float32))), f"{mode}: out_f32 window {g}"
            if mode != "f32":
                assert np.array_equal(_bits(got_n[g]), _bits(np.ascontiguousarray(want.transpose(0, 2, 1)))), f"{mode}: out_nhwc window {g}"
        if mode == "nhwc":
            assert np.array_equal(_bits(got_f), _bits(f_buf)), "out_f32 written although not requested"
        else:
            assert np.array_equal(_bits(got_f[G]), _bits(f_buf[G])), f"{mode}: out_f32 written past the last window"
        if mode == "f32":
            assert np.array_equal(_bits(got_n), _bits(n_buf)), "out_nhwc written although not requested"
        else:
            assert np.array_equal(_bits(got_n[G]), _bits(n_buf[G])), f"{mode}: out_nhwc written past the last window"
    ctx.free(ht)


@pytest.mark.gpu
@pytest.mark.parametrize("G,B,dt,mode", SLICE_CASES, ids=[f"G{c[0]}_B{c[1]}_Tc{c[2]:+d}_{c[3]}" for c in SLICE_CASES])
def test_slice_bit_exact(ctx, G, B, dt, mode):
    """hubert_slice at the default start (stride_left 10: start 5) against oracle.ultralight_ref.window_rows(T, B, start) applied
    to window g's fp16 hidden rows: out_f32 [G][B][16][D] and out_nhwc [G][B][D][16], together and each alone.  At this start every
    gathered row lies inside [0, T - 1) (the clamp and the zero rows are test_slice_clamps_at_window_edges').  The hidden buffer
    holds SENT_IN one window past the last, and both outputs are one window longer than written: that window must keep its bits."""
    _run_slice(ctx, G, B, dt, 5.0, (mode,), seed=G * 100 + B * 3 + dt)


@pytest.mark.gpu
@pytest.mark.parametrize("G,B,dt,start_kind", EDGE_CASES, ids=[f"G{c[0]}_B{c[1]}_Tc{c[2]:+d}_{c[3]}" for c in EDGE_CASES])
def test_slice_clamps_at_window_edges(ctx, G, B, dt, start_kind):
    """hubert_slice where the windows run off the hidden rows, for Tc = T - 1, T, T + 1 and all three output modes.  start 0 (no
    left context) makes the gather clamp rows below 0 to row 0; start T / 2 (little right context) makes it clamp rows past T - 1
    to row T - 1, which at Tc = T - 1 is one of the zero rows [Tc, T).  The test asserts that its windows reach the edge it is
    there for, then compares bit for bit as test_slice_bit_exact does."""
    from livetalking_b200.hubert import window_samples
    T = window_samples(B, 10, 10)[2]
    start = _slice_start(start_kind, T)
    raw = _slice_raw_rows(B, start)
    if start_kind == "zero":
        assert raw.min() < 0, "no gathered row is clamped to row 0"
    else:
        assert raw.max() > T - 1, "no gathered row is clamped to row T - 1"
        if dt == -1:
            assert (raw >= T + dt).any(), "no gathered row falls in the zero rows [Tc, T)"
    _run_slice(ctx, G, B, dt, start, ("both", "f32", "nhwc"), seed=G * 100 + B * 3 + dt + (7 if start_kind == "end" else 11))
