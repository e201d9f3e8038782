"""GPU: the S3FD face detector (livetalking_b200/s3fd.py, csrc/s3fd.cu) against float64 and the fp32 oracle (oracle/s3fd_ref.py).

* s3fd_prep and maxpool2x2 bit-exact (odd map sizes included).
* Every conv, L2Norm and fused head of a keep_layers detector against float64 computed from that op's own fp16 GPU input, with
  the per-element bound of tests/test_gpu_w2l_layers.py (A = sum |w||x|, u = 2^-11, v = 2^-24, K the accumulation chain):
  1.25 (18 ceil(K/16) 2^-23 A + 3 v (A + |b|) + u |ref| + 2^-25 + min(32, K/128) v (A + |b|)).  The last term covers a split-K
  gather plan; the halo plans have no residual here.  L2Norm: fp32 sum of C squares, sqrt, divide and scale: 1.25 ((C/2 + 8) v |ref|
  + u |ref| + 2^-25).  Runs at B = 2 160 x 288, B = 1 119 x 213 and the production size B = 16 720p (images 0 and 15 checked),
  each asserting which kernel (halo or gather) the planner ran for every conv; the largest |activation| per layer is asserted to
  stay below 2^14 (a 4x margin to the fp16 range; the epilogue saturates silently).
* s3fd_select against a float64 restatement on constructed fp16 head maps (720p and 477 x 851 layouts) whose arg-max sits on
  each of the six levels, at both map corners and inside, with max-out backgrounds and a max-out decoy on level 0, found and not
  found, and boxes whose negative corners the clip zeroes: anchor, found and box integers bit-exact (+-1 only where the float64
  coordinate is within 1e-3 of an integer), score within 1e-6.  Also on the detector's own head maps in the end-to-end runs.
* End to end at B = 16, 720p and at 477 x 851 against the oracle in fp32 (TF32 off): the same found flags, a winning anchor whose
  oracle score is within 2 * delta of the oracle's maximum (delta = the largest conf-logit difference of the two runs, the slope of
  the softmax being at most 1/4 on each of the two logits), boxes within 1 px of the oracle's decode of that anchor.
* generate_avatar on a generated video (img_size 256, the engine's wav2lip256 face size): coords.pkl and face PNGs equal to the host path driven by the oracle's detections, and
  the wav2lip plugin loading the result from the directory and from avatar.ltbav."""
import os
import pickle
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conv_check import SAFETY, SUB16, U16, V32
from layer_bound import conv_bound
from oracle import s3fd_ref as R

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def no_tf32():
    c, m = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = c, m


@pytest.fixture(scope="module")
def sd():
    return R.synth_state_dict(0)


@pytest.fixture(scope="module")
def net(sd):
    from livetalking_b200 import engine
    from livetalking_b200.s3fd import S3FDNet
    engine.set_device(0)
    return S3FDNet.from_state_dict(sd)


def _nchw64(a):
    return torch.from_numpy(np.asarray(a, np.float32)).permute(0, 3, 1, 2).to("cuda", torch.float64)


def test_prep_and_maxpool_bit_exact():
    from livetalking_b200.ops import Ctx
    ctx = Ctx()
    rng = np.random.default_rng(3)
    fr = rng.integers(0, 256, (2, 37, 53, 3), dtype=np.uint8)
    d_fr = ctx.upload(fr)
    out = ctx.alloc((2, 37, 53, 16))
    ctx.s3fd_prep(d_fr, 2, 37, 53, out)
    got = ctx.download(out).astype(np.float32)
    want = np.zeros_like(got)
    want[..., :3] = fr[..., ::-1].astype(np.float32) - np.array([104, 117, 123], np.float32)
    np.testing.assert_array_equal(got, want)
    for (H, W, C) in ((37, 53, 64), (46, 80, 256), (7, 11, 512)):
        x = (rng.standard_normal((3, H, W, C)) * 100).astype(np.float16)
        dx = ctx.upload(x)
        dy = ctx.alloc((3, H // 2, W // 2, C))
        ctx.maxpool2x2(dx, 3, H, W, dy)
        want = F.max_pool2d(torch.from_numpy(x.astype(np.float32)).permute(0, 3, 1, 2), 2, 2).permute(0, 2, 3, 1).numpy().astype(np.float16)
        np.testing.assert_array_equal(ctx.download(dy), want)
    ctx.close()


HALO, GATHER = 1, 0
_TRUNK_3X3 = ["conv1_1", "conv1_2", "conv2_1", "conv2_2", "conv3_1", "conv3_2", "conv3_3", "conv4_1", "conv4_2", "conv4_3", "conv5_1",
              "conv5_2", "conv5_3"]
# run -> (N, H, W, checked images, layers the planner puts on the halo kernel; every other conv and all heads run on the gather
# kernel).  At 720p the 3x3 maps from 360 x 640 down are not multiples of 16 rows and too long for the overhanging-tile rule, so
# they take the gather kernel; the 1x1 convs have M >= 512 there and take the halo kernel's GEMM mode.
LAYER_RUNS = {
    "b2_160x288": (2, 160, 288, (0, 1), set(_TRUNK_3X3)),
    "b1_119x213": (1, 119, 213, (0,), set(_TRUNK_3X3)),
    "b16_720p": (16, 720, 1280, (0, 15), {"conv1_1", "conv1_2", "fc7", "conv6_1", "conv7_1"}),
}


def _images(ctx, t, imgs):
    """fp16 NHWC images `imgs` of device tensor t -> float64 NCHW on the GPU (reads back only those images)."""
    from livetalking_b200.ops import DevTensor
    per = int(np.prod(t.shape[1:]))
    out = [ctx.download(DevTensor(t.offset(i * per), (1,) + t.shape[1:])) for i in imgs]
    return _nchw64(np.concatenate(out, 0))


@pytest.mark.parametrize("run", list(LAYER_RUNS))
def test_every_step_against_float64(net, sd, run):
    from livetalking_b200.s3fd import S3FDDetector, LEVELS
    N, H, W, imgs, halo = LAYER_RUNS[run]
    frames = R.synth_frames(([35, 50, 0, 45] * 4)[:N], H, W, seed=11)
    det = S3FDDetector(net, N, H, W, keep_layers=True)
    det.run_raw(frames)
    variants = det.conv_variants()
    ctx, bad, report = det.ctx, [], []
    head_src = {f"{s}_norm_mbox" if n else f"{s}_mbox": lv for lv, (s, _, n, _) in enumerate(LEVELS)}
    for st in det.steps:
        name = st.name
        if name in ("prep", "select"):
            continue
        kind = "head" if name in head_src else "conv" if st.layer else "pool" if name.endswith("_pool") else "l2norm"
        xin = _images(ctx, det.view(st.src), imgs)
        got = _images(ctx, det.view(st.dst), imgs)
        assert torch.isfinite(got).all(), name
        if kind == "pool":
            assert torch.equal(got, F.max_pool2d(xin, 2, 2)), name
            continue
        if kind == "l2norm":
            src = name[:-5]
            wv = sd[src + "_norm.weight"].to("cuda", torch.float64)
            ref = R.l2norm(xin, wv)
            C = xin.shape[1]
            bound = SAFETY * ((C / 2 + 8) * V32 * ref.abs() + U16 * ref.abs() + SUB16)
        elif kind == "conv":
            e = next(t for t in R.TRUNK if t != "pool" and t[0] == name)
            w = sd[name + ".weight"].to("cuda", torch.float64)
            if name == "conv1_1":
                xin = xin[:, :3]
            w16 = w.half().double()
            ref, bound = conv_bound(xin, w16, sd[name + ".bias"].to("cuda", torch.float64), e[4], e[5], True)
        else:
            lv = head_src[name]
            pre = name[:-5]
            w = torch.cat([sd[pre + "_mbox_conf.weight"], sd[pre + "_mbox_loc.weight"]]).to("cuda", torch.float64).half().double()
            b = torch.cat([sd[pre + "_mbox_conf.bias"], sd[pre + "_mbox_loc.bias"]]).to("cuda", torch.float64)
            ref, bound = conv_bound(xin, w, b, 1, 1, False)
            assert torch.all(got[:, w.shape[0]:] == 0), f"{name}: padded head channels not zero"
            got = got[:, :w.shape[0]]
        ratio = ((got - ref).abs() / bound).max().item()
        amax = got.abs().max().item()
        report.append((name, kind, variants.get(name), ratio, amax))
        if ratio > 1.0:
            bad.append((name, ratio))
        assert amax < 2.0 ** 14, f"{name}: largest activation {amax} leaves less than a 4x margin to the fp16 range"
        del xin, got, ref, bound
    for r in report:
        print("  %-22s %-6s %-70s err/bound %.3f  max|act| %.1f" % (r[0], r[1], r[2], r[3], r[4]))
    ran = {name: v["kernel"] for name, v in variants.items()}
    want = {name: HALO if name in halo else GATHER for name in ran}
    assert ran == want, {n: (ran[n], want[n]) for n in ran if ran[n] != want[n]}
    assert not bad, bad
    det.close()
    torch.cuda.empty_cache()


def _select64(heads, N):
    """float64 restatement of s3fd_select on fp16 head maps [N,h,w,16]: (found, box, score, anchor, top-two gap, raw box)."""
    sc, bx = [], []
    for lv, h in enumerate(heads):
        h = h.astype(np.float64)
        n_, fh, fw, _ = h.shape
        if lv == 0:
            bg, fc, loc = h[..., :3].max(-1), h[..., 3], h[..., 4:8]
        else:
            bg, fc, loc = h[..., 0], h[..., 1], h[..., 2:6]
        s = 1.0 / (1.0 + np.exp(bg - fc))
        stride = 2.0 ** (lv + 2)
        ys, xs = np.meshgrid(np.arange(fh), np.arange(fw), indexing="ij")
        cx, cy, size = stride / 2 + xs * stride, stride / 2 + ys * stride, 4 * stride
        bxc, byc = cx + loc[..., 0] * 0.1 * size, cy + loc[..., 1] * 0.1 * size
        bw, bh = size * np.exp(loc[..., 2] * 0.2), size * np.exp(loc[..., 3] * 0.2)
        x1, y1 = bxc - bw / 2, byc - bh / 2
        sc.append(s.reshape(N, -1))
        bx.append(np.stack([x1, y1, x1 + bw, y1 + bh], -1).reshape(N, -1, 4))
    s, b = np.concatenate(sc, 1), np.concatenate(bx, 1)
    a = s.argmax(1)
    n = np.arange(N)
    top2 = np.sort(s, 1)[:, -2:]
    raw = np.clip(b[n, a], 0, None)
    return s[n, a] > 0.5, np.floor(raw).astype(np.int64), s[n, a], a, top2[:, 1] - top2[:, 0], raw, s, b


def _check_select(det, oi, osc):
    heads = [det.ctx.download(h) for h in det.heads]
    found, box, score, anchor, gap, raw, _, _ = _select64(heads, det.N)
    for i in range(det.N):
        if gap[i] <= 1e-5:
            continue
        assert oi[i, 5] == anchor[i], (i, oi[i], anchor[i])
        assert abs(osc[i] - score[i]) <= 1e-6, (i, osc[i], score[i])
        if abs(score[i] - 0.5) > 1e-6:
            assert bool(oi[i, 0]) == bool(found[i]), i
        near = np.abs(raw[i] - np.round(raw[i])) < 1e-3
        diff = np.abs(oi[i, 1:5] - box[i])
        assert np.all(np.where(near, diff <= 1, diff == 0)), (i, oi[i, 1:5], box[i], raw[i])


def _constructed_heads(H, W, N, rng):
    """fp16 head maps [N,h,w,16] with a known arg-max per image: image i wins on level i % 6, at the top-left map corner (i // 6 = 0;
    loc pushes the box to negative x1 / y1, which the clip must zero), the bottom-right corner (1) or inside the map (2).  Background
    anchors score below sigmoid(-3); every level-0 winner takes its background from c1 or c2 (max-out), and every image has a
    level-0 decoy whose c3 is large but whose c2 is larger (score sigmoid(-1.5)).  Winners have face - background = +2.5 (found)
    or -0.5 (not found: still the arg-max)."""
    shapes = R.head_shapes(H, W)
    heads = []
    for lv, (fh, fw) in enumerate(shapes):
        h = np.zeros((N, fh, fw, 16), np.float32)
        nbg = 3 if lv == 0 else 1
        h[..., :nbg] = rng.uniform(-1, 1, (N, fh, fw, nbg))
        h[..., nbg] = h[..., :nbg].max(-1) - rng.uniform(3, 5, (N, fh, fw))
        h[..., nbg + 1:nbg + 5] = rng.uniform(-1, 1, (N, fh, fw, 4))
        heads.append(h)
    want = []
    for i in range(N):
        fh, fw = shapes[0]
        dy, dx = int(rng.integers(0, fh)), int(rng.integers(0, fw))
        heads[0][i, dy, dx, :4] = (-1.0, -1.0, 7.5, 6.0)
        lv, where = i % 6, (i // 6) % 3
        fh, fw = shapes[lv]
        y, x = {0: (0, 0), 1: (fh - 1, fw - 1)}.get(where, (int(rng.integers(1, fh - 1)), int(rng.integers(1, fw - 1))))
        if lv == 0 and (y, x) == (dy, dx):
            heads[0][i, dy, dx, :4] = 0.0
        margin = 2.5 if i % 4 != 3 else -0.5
        px = heads[lv][i, y, x]
        if lv == 0:
            bg = 0.3
            px[:4] = (-2.0, bg, -1.0, bg + margin) if i % 2 else (-2.0, -1.0, bg, bg + margin)
            loc = px[4:8]
        else:
            px[:2] = (0.0, margin)
            loc = px[2:6]
        loc[:] = rng.uniform(-1, 1, 4)
        if where == 0:
            loc[:2] = -rng.uniform(2.0, 4.0, 2)
        want.append(sum(a * b for a, b in shapes[:lv]) + y * fw + x)
    return [h.astype(np.float16) for h in heads], np.array(want)


@pytest.mark.parametrize("H,W", [(720, 1280), (477, 851)])
def test_select_on_constructed_logits(H, W):
    """s3fd_select against the float64 restatement on head maps whose arg-max is placed on each of the six levels."""
    from livetalking_b200.ops import Ctx
    N = 18
    heads, want_anchor = _constructed_heads(H, W, N, np.random.default_rng(H))
    ctx = Ctx()
    d_heads = [ctx.upload(h) for h in heads]
    oi_d, os_d = ctx.alloc((N, 6), np.int32), ctx.alloc((N,), np.float32)
    ctx.s3fd_select(d_heads, N, 0.5, oi_d, os_d)
    oi, osc = ctx.download(oi_d), ctx.download(os_d)
    ctx.close()
    found, box, score, anchor, gap, raw, _, b = _select64(heads, N)
    np.testing.assert_array_equal(anchor, want_anchor)       # the construction put the arg-max where intended
    np.testing.assert_array_equal(oi[:, 5], want_anchor)
    assert np.all(gap > 1e-3)
    np.testing.assert_allclose(osc, score, rtol=0, atol=1e-6)
    np.testing.assert_array_equal(oi[:, 0].astype(bool), found)
    assert found.any() and not found.all()
    unclipped = b[np.arange(N), anchor]
    assert (unclipped[:, :2] < 0).sum() >= 6 and np.all(oi[unclipped[:, 0] < 0, 1] == 0) and np.all(oi[unclipped[:, 1] < 0, 2] == 0)
    near = (np.abs(raw - np.round(raw)) < 1e-3) & (unclipped >= 0)     # clipped corners must be exactly 0
    diff = np.abs(oi[:, 1:5] - box)
    assert np.all(np.where(near, diff <= 1, diff == 0)), (oi[:, 1:5], box, raw)
    assert near.sum() <= 4, near.sum()                       # the comparison is bit-exact nearly everywhere


@pytest.mark.parametrize("N,H,W", [(16, 720, 1280), (3, 477, 851)])
def test_end_to_end_against_oracle(net, sd, N, H, W):
    from livetalking_b200.s3fd import S3FDDetector
    amps = ([0, 10, 35, 50, 40, 0, 45, 5, 60, 35, 10, 40, 0, 50, 35, 45] * 2)[:N]
    side = min(H, W) // 3
    blobs = [((H // 5 + 23 * i) % (H - side), (W // 7 + 61 * i) % (W - side), side) for i in range(N)]
    frames = R.synth_frames(amps, H, W, seed=5, blob=blobs)
    det = S3FDDetector(net, N, H, W)
    oi, osc = det.run_raw(frames)
    _check_select(det, oi, osc)
    assert det.detect(frames) == [tuple(int(v) for v in r[1:5]) if r[0] else None for r in oi]
    g_heads = [det.ctx.download(h).astype(np.float64) for h in det.heads]
    with torch.no_grad():
        ol = R.forward(sd, R.prep(frames, "cuda"))
    s, b = R.scores_and_boxes(ol)
    s, b = s.double().cpu().numpy(), b.double().cpu().numpy()
    delta = 0.0
    for lv, gh in enumerate(g_heads):
        cls = ol[2 * lv].double().cpu().numpy().transpose(0, 2, 3, 1)
        gc = np.concatenate([gh[..., :3].max(-1, keepdims=True), gh[..., 3:4]], -1) if lv == 0 else gh[..., :2]
        delta = max(delta, float(np.abs(gc - cls).max()))
    print(f"  [{N}x{H}x{W}] largest conf-logit difference {delta:.2e}; found {oi[:, 0].tolist()}")
    assert delta < 0.05
    for i in range(N):
        best = s[i].max()
        if abs(best - 0.5) > 2 * delta:
            assert bool(oi[i, 0]) == (best > 0.5), (i, best)
        a = int(oi[i, 5])
        assert s[i, a] >= best - 2 * delta, (i, a, s[i, a], best)
        if oi[i, 0]:
            want = np.clip(b[i, a], 0, None)
            assert np.all(np.abs(oi[i, 1:5] - want) <= 1.0 + 1e-6), (i, oi[i, 1:5], want)
    assert oi[:, 0].any() and not oi[:, 0].all()
    det.close()


def test_generate_avatar_on_the_engine(net, sd, tmp_path, monkeypatch):
    import torch.hub
    import torch.utils.model_zoo

    import sys
    sys.path.insert(0, os.path.dirname(__file__))
    import stubs
    stubs.install()
    from livetalking_b200.plugin import wav2lip_avatar
    from livetalking_b200.plugin import wav2lip_genavatar as G

    def boom(*a, **k):
        raise AssertionError("a download was attempted")
    monkeypatch.setattr(torch.utils.model_zoo, "load_url", boom)
    monkeypatch.setattr(torch.hub, "load_state_dict_from_url", boom)
    wpath = tmp_path / "s3fd.pth"
    torch.save(sd, wpath)
    frames = R.synth_frames([0, 40, 45, 50, 0, 10, 50, 40, 35, 0, 45, 40], 240, 320, seed=9)
    vid = str(tmp_path / "clip.avi")
    R.write_video(vid, frames)
    progress, split = [], {}
    G.generate_avatar(vid, "eng", save_path=str(tmp_path / "data" / "avatars"), img_size=256, face_det_batch_size=8, weights_path=str(wpath),
                      progress_callback=progress.append, timings=split)
    assert progress[:3] == [5, 20, 40] and progress[-1] == 100
    assert {"decode", "full_png", "detect", "face_png", "pack"} == set(split)

    class OracleDetector:
        def __init__(self, N, H, W):
            pass

        def detect(self, fr):
            return R.detect(sd, np.asarray(fr), "cuda")

        def close(self):
            pass
    G.generate_avatar(vid, "ora", save_path=str(tmp_path / "data" / "avatars"), img_size=256, face_det_batch_size=8, make_detector=OracleDetector)
    av = tmp_path / "data" / "avatars"
    with open(av / "eng" / "coords.pkl", "rb") as f1, open(av / "ora" / "coords.pkl", "rb") as f2:
        ce, co = pickle.load(f1), pickle.load(f2)
    assert ce == co
    crc = lambda d: [zlib.crc32((d / f).read_bytes()) for f in sorted(os.listdir(d))]  # noqa: E731
    assert crc(av / "eng" / "face_imgs") == crc(av / "ora" / "face_imgs")
    monkeypatch.chdir(tmp_path)
    packed = wav2lip_avatar.load_avatar("eng")
    os.remove(av / "eng" / "avatar.ltbav")
    from_dir = wav2lip_avatar.load_avatar("eng")
    for p in (packed, from_dir):
        fl, fa, co_ = p[0], p[1], p[2]
        assert len(fl) == len(fa) == len(co_) == 12
        assert [tuple(c) for c in co_] == ce
        assert p.engine_avatar is not None
    for a, b in zip(packed[1], from_dir[1]):
        np.testing.assert_array_equal(a, b)
