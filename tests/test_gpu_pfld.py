"""GPU: the PFLD landmark network (livetalking_b200/pfld.py, csrc/pfld.cu) against float64 and the oracle (oracle/pfld_ref.py, pinned
to the unmodified reference by tests/test_pfld_oracle.py).

* pfld_prep bit-exact against numpy's fp16(fp32(v) / 255).
* Every conv (planner) and depthwise layer, conv8 as a 2304-wide GEMM included, against float64 computed from that layer's own fp16
  GPU input and the padded fp16 weights, with the per-element bound of tests/layer_bound.py (A = sum |w||x|, u = 2^-11,
  v = 2^-24, K the accumulation length): 1.25 (18 ceil(K/16) 2^-23 A + 3 v (A + |b|) + u |ref| + 2^-25 + min(32, K/128) v (A + |b|)).
  For the depthwise kernel (an fp32 FMA chain of 9 taps) the same formula is a loose bound.  Every padded channel must be exactly 0,
  every activation below 2^14 (a 4x margin to the fp16 range), and the test asserts which planner kernel each conv ran.
* pfld_head against float64 on constructed fp16 taps: the fp32 averages (ceil(hw / T) + T sequential adds, T = 512 / (pitch / 8)
  slots: (chain + 1) v mean|x|), conv_out's
  fp32 FMA chain over 256 features, + mean, x crop size: bound 1.25 ((sum_j |W_oj| e_j + 258 v (sum |W||f| + |b| + |mean|)) s
  + v |out|).  The int output is the truncation of the float output, and equals the truncated float64 value wherever that lies
  farther than the bound from an integer.
* End to end at B = 16 and B = 5 against the oracle in float64: landmarks (pixels) within TOL_NORM x crop size; int landmarks
  equal wherever the float64 value lies farther than that from an integer.
* generate_avatar with the replaying detector on a synthetic 720p clip: coords and face PNGs equal to the oracle-driven path on every
  frame whose three mouth-box landmarks are clear of integers; the result loads through the UltraLight plugin (PNG and .ltbav)."""
import math
import os
import pickle
import sys
import zlib

import cv2
import numpy as np
import pytest
import torch

from conv_check import SAFETY, V32
from layer_bound import conv_bound
from oracle import pfld_ref as R

pytestmark = pytest.mark.gpu

TOL_NORM = 2e-4          # end to end, fp16 network vs float64 oracle, in units of the crop size (4x the largest error measured)
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
GATHER, HALO = 0, 1
CONV1_KERNEL = GATHER


def _want_kernel(L, N):
    """The planner's choice (conv_halo_supported): a 1x1 conv takes the halo kernel's GEMM mode when Cout % 32 == 0, Cin >= 32 and
    M >= 512 pixels; conv7 (Cout 16) and conv8 (M = N rows) take the gather kernel."""
    if L.name == "conv1":
        return CONV1_KERNEL
    cout, cin, k, _ = L.w.shape
    return HALO if k == 1 and L.name != "conv8" and cout % 32 == 0 and cin >= 32 else GATHER


@pytest.fixture(scope="module")
def sd():
    return R.synth_state_dict(0)


@pytest.fixture(scope="module")
def mean_face():
    return R.read_mean_face(os.path.join(GOLDEN, "pfld_mean_face.txt"))


@pytest.fixture(scope="module")
def net(sd, mean_face):
    from livetalking_b200 import engine
    from livetalking_b200.pfld import PFLDNet
    engine.set_device(0)
    return PFLDNet.from_state_dict({"pfld_backbone": sd}, mean_face)


def _crops(n, seed):
    c = R.synth_video_frames(n, 192, 192, seed=seed)
    c[-1] = np.random.default_rng(seed).integers(0, 256, (192, 192, 3), dtype=np.uint8)
    return c


def test_prep_bit_exact():
    from livetalking_b200.ops import Ctx
    ctx = Ctx()
    fr = np.random.default_rng(3).integers(0, 256, (3, 192, 192, 3), dtype=np.uint8)
    fr[0, 0, :256 // 3 + 1] = np.arange(256).repeat(3)[:(256 // 3 + 1) * 3].reshape(-1, 3)
    d_fr = ctx.upload(fr)
    out = ctx.alloc((3, 192, 192, 16))
    ctx.pfld_prep(d_fr, 3, 192, 192, out)
    got = ctx.download(out)
    want = np.zeros_like(got)
    want[..., :3] = (fr.astype(np.float32) / np.float32(255.0)).astype(np.float16)
    np.testing.assert_array_equal(got.view(np.uint16), want.view(np.uint16))
    ctx.close()


def _nchw(a):
    return torch.from_numpy(np.asarray(a, np.float32)).permute(0, 3, 1, 2).to("cuda", torch.float64)


@pytest.mark.parametrize("N", [16, 5])
def test_every_step_against_float64(net, N):
    from livetalking_b200.pfld import PFLDLandmarker
    lm = PFLDLandmarker(net, N)
    crops = _crops(N, 11 + N)
    lm.run(crops, np.full((N, 2), 150, np.int32))
    variants = lm.conv_variants()
    ctx, bad, report = lm.ctx, [], []
    imgs = [0, N - 1]
    for L in [st.layer for st in lm.steps if st.layer]:
        xb = ctx.download(lm.buf[L.src[0]])[imgs]
        yb = ctx.download(lm.buf[L.dst[0]])[imgs]
        assert np.isfinite(yb).all(), L.name
        if L.name == "conv8":
            xin = _nchw(xb.reshape(len(imgs), 1, 1, -1))
        else:
            xin = _nchw(xb[..., L.src[1]:L.src[1] + L.src[2]])
        got = _nchw(yb[..., L.dst[1]:L.dst[1] + L.dst[2]])
        w = torch.from_numpy(L.w).to("cuda", torch.float64)
        b = torch.from_numpy(L.b).to("cuda", torch.float64)
        ref, bound = conv_bound(xin, w, b, L.stride, L.pad, L.relu, groups=L.w.shape[0] if L.kind == "dw" else 1)
        ratio = ((got - ref).abs() / bound).max().item()
        real = np.abs(L.w).reshape(L.w.shape[0], -1).max(1) > 0
        assert torch.all(got[:, torch.from_numpy(~real).cuda()] == 0), f"{L.name}: a padded channel is not zero"
        amax = got.abs().max().item()
        report.append((L.name, L.kind, variants.get(L.name), ratio, amax))
        if ratio > 1.0:
            bad.append((L.name, ratio))
        assert amax < 2.0 ** 14, f"{L.name}: largest activation {amax}"
    for r in report:
        print("  %-36s %-4s %-60s err/bound %.3f  max|act| %.2f" % (r[0], r[1], r[2], r[3], r[4]))
    ran = {name: v["kernel"] for name, v in variants.items()}
    assert set(ran) == {L.name for L in net.layers if L.kind == "conv"}
    want = {L.name: _want_kernel(L, N) for L in net.layers if L.kind == "conv"}
    assert ran == want, {n: (ran[n], want[n]) for n in ran if ran[n] != want[n]}
    assert not bad, bad
    lm.close()


def _head64(taps, chans, wt, bias, mean, wh):
    feats = [t.astype(np.float64).reshape(t.shape[0], -1, t.shape[-1])[..., c] for t, c in zip(taps, chans)]
    f = np.concatenate([x.mean(1) for x in feats], 1)
    # chain of one feature: ceil(hw / T) pixel adds per thread, then the T partials (T = 512 threads / (pitch / 8))
    chain = [math.ceil(x.shape[1] / (512 // (t.shape[-1] // 8))) + 512 // (t.shape[-1] // 8) for x, t in zip(feats, taps)]
    e = np.concatenate([(k + 1) * V32 * np.abs(x).mean(1) for k, x in zip(chain, feats)], 1)
    lm = f @ wt.astype(np.float64) + bias + mean
    s = np.where(np.arange(wt.shape[1]) % 2 == 0, wh[:, :1], wh[:, 1:2]).astype(np.float64)
    absum = np.abs(f) @ np.abs(wt.astype(np.float64)) + np.abs(bias) + np.abs(mean)
    bound = SAFETY * ((e @ np.abs(wt.astype(np.float64)) + 258 * V32 * absum) * s + V32 * np.abs(lm * s))
    return lm * s, bound


def test_head_against_float64(net):
    from livetalking_b200.ops import Ctx
    ctx = Ctx()
    rng = np.random.default_rng(7)
    N = 6
    shapes = [(96, 96, 32), (48, 48, 64), (24, 24, 64), (12, 12, 96), (1, 1, 64)]
    taps, chans = [], [c for _, c in net.taps]
    for (h, w, p), c in zip(shapes, chans):
        t = np.zeros((N, h, w, p), np.float32)
        t[..., c] = rng.uniform(0, 4, (N, h, w, len(c))) * (rng.uniform(0, 1, (N, 1, 1, len(c))) > 0.2)
        t[..., [i for i in range(p) if i not in c]] = 1e4         # padded channels must not be read
        taps.append(t.astype(np.float16))
    wt = (rng.standard_normal((256, 220)) * 0.01).astype(np.float32)
    bias = (rng.standard_normal(220) * 0.01).astype(np.float32)
    mean = np.asarray(R.read_mean_face(os.path.join(GOLDEN, "pfld_mean_face.txt")), np.float32)
    wh = np.stack([rng.integers(60, 700, N), rng.integers(60, 700, N)], 1).astype(np.int32)
    d = [ctx.upload(t) for t in taps]
    d_wt, d_b, d_m, d_wh = ctx.upload(wt), ctx.upload(bias), ctx.upload(mean), ctx.upload(wh)
    of, oi = ctx.alloc((N, 220), np.float32), ctx.alloc((N, 220), np.int32)
    ctx.pfld_head(d, chans, N, d_wt, d_b, d_m, d_wh, of, oi)
    gf, gi = ctx.download(of), ctx.download(oi)
    ctx.close()
    ref, bound = _head64(taps, chans, wt, bias, mean, wh)
    ratio = np.abs(gf - ref) / bound
    print(f"  head err/bound {ratio.max():.3f}")
    assert ratio.max() <= 1.0
    np.testing.assert_array_equal(gi, np.trunc(gf).astype(np.int32))
    clear = np.abs(ref - np.round(ref)) > bound
    assert clear.mean() > 0.9
    np.testing.assert_array_equal(gi[clear], np.trunc(ref[clear]).astype(np.int32))


def _oracle64(sd, mean_face, crops, wh):
    fw = R.folded(sd)
    with torch.no_grad():
        raw = R.forward(fw, R.prep(crops).double().cuda()).cpu().numpy()
    v = (raw + mean_face.astype(np.float64)).reshape(len(crops), -1, 2) * wh[:, None, :].astype(np.float64)
    return v


@pytest.mark.parametrize("N", [16, 5])
def test_end_to_end_against_oracle(net, sd, mean_face, N):
    from livetalking_b200.pfld import PFLDLandmarker
    lm = PFLDLandmarker(net, N)
    crops = _crops(N, 21 + N)
    wh = np.stack([np.arange(N) * 37 % 500 + 90, np.arange(N) * 53 % 500 + 90], 1).astype(np.int32)
    gf, gi = lm.run(crops, wh)
    gf2, gi2 = lm.run(crops[: N - 2], wh[: N - 2])      # partial batch: the same per-image result
    np.testing.assert_array_equal(gf2, gf[: N - 2])
    want = _oracle64(sd, mean_face, crops, wh)
    tol = TOL_NORM * wh[:, None, :].astype(np.float64)
    err = np.abs(gf - want)
    print(f"  [B={N}] largest landmark error {(err / wh[:, None, :]).max():.2e} of the crop size")
    assert np.all(err <= tol)
    np.testing.assert_array_equal(gi, np.trunc(gf).astype(np.int32))
    clear = np.abs(want - np.round(want)) > tol
    np.testing.assert_array_equal(gi[clear], np.trunc(want[clear]).astype(np.int32))   # astype(int32) truncates toward zero
    assert clear.mean() > 0.8
    lm.close()


def test_generate_avatar_on_the_engine(net, sd, mean_face, tmp_path, monkeypatch):
    sys.path.insert(0, os.path.dirname(__file__))
    import stubs
    stubs.install()
    from livetalking_b200.plugin import ultralight_avatar
    from livetalking_b200.plugin import ultralight_genavatar as G
    from livetalking_b200.pfld import PFLDLandmarker
    from oracle import s3fd_ref
    from oracle import ultralight_ref as U

    n = 20
    frames = R.synth_video_frames(n, 720, 1280, seed=9)
    vid = str(tmp_path / "clip.avi")
    s3fd_ref.write_video(vid, frames)
    boxes = [(300 + 13.3 * i, 180 + 7.7 * i, 260 + 3 * i, 300 - 2 * i) for i in range(n)]
    boxes[3] = (2.6, -30.2, 280.0, 310.0)           # face_det's border shift makes x1 and y1 negative
    boxes[7] = (1050.4, 200.6, 250.0, 280.0)
    ckpt = tmp_path / "ul.pth"
    torch.save(U.synth_state_dict(0), ckpt)
    split = {}
    save = tmp_path / "data" / "avatars"
    G.generate_avatar(vid, "eng", save_path=str(save), checkpoint=str(ckpt), detector=R.ReplayDetector(R.face_records(boxes)),
                      make_landmarker=lambda N: PFLDLandmarker(net, N), timings=split)
    assert {"decode", "full_png", "detect", "landmarks", "face_png", "pack"} == set(split)
    fw = R.folded(sd)
    clear = []

    class Oracle:
        def __init__(self, N):
            pass

        def run(self, crops, wh):
            with torch.no_grad():
                raw = R.forward(fw, R.prep(crops).cuda()).cpu().numpy()
            out = np.stack([R.landmarks(r, mean_face, int(w), int(h)) for r, (w, h) in zip(raw, wh)])
            v64 = (raw.astype(np.float64) + mean_face).reshape(len(crops), -1, 2) * wh[:, None, :]
            for i in range(len(crops)):
                pts = np.array([v64[i, 1, 0], v64[i, 31, 0], v64[i, 52, 1]])
                clear.append(bool(np.all(np.abs(pts - np.round(pts)) > TOL_NORM * wh[i].max())))
            return out.astype(np.float32), out

        def close(self):
            pass
    G.generate_avatar(vid, "ora", save_path=str(save), checkpoint=str(ckpt), detector=R.ReplayDetector(R.face_records(boxes)),
                      make_landmarker=Oracle)
    with open(save / "eng" / "coords.pkl", "rb") as f1, open(save / "ora" / "coords.pkl", "rb") as f2:
        ce, co = pickle.load(f1), pickle.load(f2)
    crc = lambda d: [zlib.crc32((d / f).read_bytes()) for f in sorted(os.listdir(d))]  # noqa: E731
    fe, fo = crc(save / "eng" / "face_imgs"), crc(save / "ora" / "face_imgs")
    assert sum(clear) >= n // 2, clear
    for i in range(n):
        if clear[i]:
            assert ce[i] == co[i] and fe[i] == fo[i], (i, ce[i], co[i])
    assert ce[3][0] >= 0 and ce[7][2] == 1280
    monkeypatch.chdir(tmp_path)
    packed = ultralight_avatar.load_avatar("eng")
    os.remove(save / "eng" / "avatar.ltbav")
    from_dir = ultralight_avatar.load_avatar("eng")
    for p in (packed, from_dir):
        assert len(p[1]) == len(p[2]) == len(p[3]) == n
        assert [tuple(int(v) for v in c) for c in p[3]] == [tuple(int(v) for v in c) for c in ce]
        assert p.engine_avatar is not None
    for a, b in zip(packed[2], from_dir[2]):
        np.testing.assert_array_equal(a, b)
    assert cv2.imread(str(save / "eng" / "face_imgs" / "00000000.png")).shape == (168, 168, 3)
