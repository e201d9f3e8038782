"""GPU: the BiSeNet face parser (livetalking_b200/bisenet.py, csrc/bisenet.cu) against float64 and the oracle (oracle/bisenet_ref.py,
pinned to the unmodified reference by tests/test_bisenet_oracle.py).  Everything runs through the C ABI.

* bisenet_prep and maxpool3x3s2 bit-exact against numpy.
* chan_gate and chan_scale_add against float64 within derived bounds (fp32 sums of ceil(HW / T) + T terms, FMA chains of the
  mat-vec length, one fp16 rounding for chan_scale_add).
* Every planner conv against float64 on its own fp16 GPU input with the per-element bound of tests/test_gpu_pfld.py (plus the
  residual, and for the fused nearest-2x convs one fp16 rounding of the summed sub-pixel weights).  Padded channels are exactly 0,
  every activation stays below 2^14, and the test asserts which kernel each conv ran.
* bisenet_upsample_argmax on its own fp16 logits: labels equal the float64 arg-max wherever the top-2 margin exceeds twice the fp32
  interpolation bound, otherwise one of the near-tied classes; constructed exact ties go to the lowest class and the padded channels
  are never read.
* End to end at B = 16 and B = 5 against the float64 oracle: labels equal wherever the oracle's top-2 margin exceeds T_LABEL, 4x the
  largest logit error measured end to end; FaceParsing.__call__ equals the reference's post-processing of the GPU labels.
* generate_avatar on a synthetic 720p clip with the replaying landmark stand-in, the GPU parser and a small MuseTalk VAE for the
  latents writes the same coords.pkl and mask_coords.pkl as the oracle-driven path; every frame's labels equal the float64 oracle's
  wherever its margin exceeds T_LABEL, and every mask equals the reference's host path applied to the engine's labels.  The output
  loads through the MuseTalk plugin as PNGs and as .ltbav, and one inference_batch + paste_back_frame runs on it."""
import math
import os
import pickle
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import bisenet_ref as R
from oracle import pfld_ref

pytestmark = pytest.mark.gpu

SAFETY = 1.25
U16 = 2.0 ** -11
SUB16 = 2.0 ** -25
V32 = 2.0 ** -24
ULP32 = 2.0 ** -23
# largest |logit| error of the fp16 network against the float64 oracle, end to end at B = 16 and 5 on the synthetic weights
# (measured on an H100 80GB HBM3: 4.9e-3 at B = 16, 6.2e-3 at B = 5); T_LABEL = 4x that
LOGIT_ERR = 6.5e-3
T_LABEL = 4 * LOGIT_ERR
GATHER, HALO = 0, 1


def _want_kernel(L):
    """conv_halo_supported: the 4x4 stem and the 1x1 stride-2 downsamples run on the gather kernel; every 3x3 (stride 1 and 2), the
    fused nearest-2x convs and the 1x1 stride-1 GEMMs (Cout % 32 == 0, Cin >= 32, M >= 512) on the halo kernel."""
    if L.name == "stem" or (L.w.shape[-1] == 1 and L.stride == 2):
        return GATHER
    return HALO


@pytest.fixture(scope="module")
def sd():
    return R.synth_state_dict(0)


@pytest.fixture(scope="module")
def net(sd):
    from livetalking_b200 import engine
    from livetalking_b200.bisenet import BiSeNetNet
    engine.set_device(0)
    return BiSeNetNet.from_state_dict(sd)


def _crops(n, seed):
    c = pfld_ref.synth_video_frames(n, 512, 512, seed=seed)[..., ::-1]
    c = np.ascontiguousarray(c)
    c[-1] = np.random.default_rng(seed).integers(0, 256, (512, 512, 3), dtype=np.uint8)
    return c


def test_prep_bit_exact():
    from livetalking_b200.ops import Ctx
    ctx = Ctx()
    rgb = np.random.default_rng(3).integers(0, 256, (2, 512, 512, 3), dtype=np.uint8)
    rgb[0, 0, :86] = np.arange(258).reshape(-1, 3)[:86] % 256
    out = ctx.alloc((2, 259, 259, 16))
    ctx.bisenet_prep(ctx.upload(rgb), 2, out)
    got = ctx.download(out)
    ctx.close()
    t = rgb.astype(np.float32) / np.float32(255)
    norm = ((t - np.array(R.MEAN, np.float32)) / np.array(R.STD, np.float32)).astype(np.float16)
    want = R.space_to_depth(torch.from_numpy(norm.astype(np.float32)).permute(0, 3, 1, 2)).permute(0, 2, 3, 1).numpy().astype(np.float16)
    np.testing.assert_array_equal(got.view(np.uint16), want.view(np.uint16))


def test_maxpool_bit_exact():
    from livetalking_b200.ops import Ctx
    ctx = Ctx()
    for H, W in ((256, 256), (15, 9)):
        x = (np.random.default_rng(H).standard_normal((3, H, W, 64)) * 3).astype(np.float16)
        out = ctx.alloc((3, (H - 1) // 2 + 1, (W - 1) // 2 + 1, 64))
        ctx.maxpool3x3s2(ctx.upload(x), 3, H, W, out)
        want = F.max_pool2d(torch.from_numpy(x.astype(np.float32)).permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1).numpy().astype(np.float16)
        np.testing.assert_array_equal(ctx.download(out).view(np.uint16), want.view(np.uint16))
    ctx.close()


def _act(v, a):
    return np.maximum(v, 0) if a == 1 else (1 / (1 + np.exp(-v)) if a == 2 else v)


@pytest.mark.parametrize("C,n1,n2,HW,pitch,off", [(512, 128, 0, 256, 512, 0), (128, 128, 0, 1024, 128, 0), (256, 64, 256, 4096, 256, 0),
                                                   (128, 96, 0, 37, 256, 128)])
def test_chan_gate_against_float64(C, n1, n2, HW, pitch, off):
    from livetalking_b200.ops import Ctx
    ctx = Ctx()
    rng = np.random.default_rng(C + n1 + n2)
    N = 5
    x = np.full((N, HW, pitch), 7e3, np.float16)              # channels outside the slice must not be read
    x[..., off:off + C] = rng.uniform(0, 6, (N, HW, C)).astype(np.float16)
    w1 = (rng.standard_normal((C, n1)) * C ** -0.5).astype(np.float32)
    b1 = (rng.standard_normal(n1) * 0.1).astype(np.float32)
    w2 = (rng.standard_normal((n1, n2)) * n1 ** -0.5).astype(np.float32) if n2 else None
    act1, act2 = (1, 2) if n2 else (2, 0)
    d = ctx.upload(x)
    xv = type(d)(d.ptr, (N, HW, C), pitch=pitch, c_off=off)
    out = ctx.alloc((N, n2 or n1), np.float32)
    ctx.chan_gate(xv, N, ctx.upload(w1), None if n2 else ctx.upload(b1), act1, out, ctx.upload(w2) if n2 else None, None, act2)
    got = ctx.download(out)
    ctx.close()
    xs = x[..., off:off + C].astype(np.float64)
    avg = xs.mean(1)
    T = 512 // (C // 8)
    e_avg = (math.ceil(HW / T) + T + 1) * V32 * np.abs(xs).mean(1)
    bb1 = np.zeros(n1) if n2 else b1.astype(np.float64)
    pre1 = avg @ w1 + bb1
    e1 = e_avg @ np.abs(w1) + (C + 2) * V32 * (np.abs(avg) @ np.abs(w1) + np.abs(bb1))
    h = _act(pre1, act1)
    if n2:
        ref = _act(h @ w2, act2)
        e = (e1 @ np.abs(w2) + (n1 + 2) * V32 * (np.abs(h) @ np.abs(w2))) * 0.25 + 4 * V32
    else:
        ref = h
        e = e1 * 0.25 + 4 * V32
    ratio = np.abs(got - ref) / (SAFETY * e)
    print(f"  chan_gate C={C} n1={n1} n2={n2} err/bound {ratio.max():.3f}")
    assert ratio.max() <= 1.0


@pytest.mark.parametrize("mode", ["vec", "map", "self"])
def test_chan_scale_add_against_float64(mode):
    from livetalking_b200.ops import Ctx, DevTensor
    ctx = Ctx()
    rng = np.random.default_rng(len(mode))
    N, H, W, C = 4, 16, 32, 128
    x = rng.uniform(0, 8, (N, H, W, C)).astype(np.float16)
    g = rng.uniform(0, 1, (N, C)).astype(np.float32)
    yv = rng.uniform(0, 4, (N, C)).astype(np.float32)
    y = rng.uniform(0, 8, (N, H, W, C)).astype(np.float16)
    out = ctx.alloc((N, H, W, 2 * C), zero=True)               # the result goes to channels [C, 2C) of a wider map
    ov = DevTensor(out.ptr, (N, H, W, C), pitch=2 * C, c_off=C)
    kw = {"vec": {"yvec": ctx.upload(yv)}, "map": {"y": ctx.upload(y)}, "self": {}}[mode]
    ctx.chan_scale_add(ctx.upload(x), N, ctx.upload(g), ov, **kw)
    got = ctx.download(out).astype(np.float64)
    ctx.close()
    xg = x.astype(np.float64) * g[:, None, None, :]
    add = {"vec": np.broadcast_to(yv[:, None, None, :], xg.shape), "map": y, "self": x}[mode].astype(np.float64)
    ref = xg + add
    bound = SAFETY * (U16 * np.abs(ref) + 2 * V32 * (np.abs(xg) + np.abs(add)) + SUB16)
    assert np.all(got[..., :C] == 0)
    assert np.all(np.abs(got[..., C:] - ref) <= bound)


def _nchw(a):
    return torch.from_numpy(np.asarray(a, np.float32)).permute(0, 3, 1, 2).to("cuda", torch.float64)


@pytest.mark.parametrize("N", [16, 5])
def test_every_conv_against_float64(net, N):
    from livetalking_b200.bisenet import BiSeNetParser
    p = BiSeNetParser(net, N)
    p.parse(_crops(N, 11 + N))
    variants = p.conv_variants()
    ctx, bad, report = p.ctx, [], []
    imgs = [0, N - 1]
    for L in net.layers:
        xb = ctx.download(p.buf[L.src[0]])[imgs][..., L.src[1]:L.src[1] + L.src[2]]
        yfull = ctx.download(p.buf[L.dst[0]])[imgs]
        assert np.isfinite(yfull).all(), L.name
        got = _nchw(yfull[..., L.dst[1]:L.dst[1] + L.dst[2]])
        x = _nchw(xb)
        if L.up:
            x = F.interpolate(x, scale_factor=2, mode="nearest")
        w = torch.from_numpy(L.w).to("cuda", torch.float64)
        bb = torch.from_numpy(L.b).to("cuda", torch.float64)[None, :, None, None]
        conv = F.conv2d(x, w, stride=L.stride, padding=L.pad)
        A = F.conv2d(x.abs(), w.abs(), stride=L.stride, padding=L.pad)
        pre = conv + bb
        extra = torch.zeros_like(A)
        if L.res is not None:
            # the epilogue may round conv + bias to fp16 before it adds the residual: one more fp16 rounding of that sum
            r = _nchw(ctx.download(p.buf[L.res[0]])[imgs][..., L.res[1]:L.res[1] + L.res[2]])
            extra = r.abs() + (U16 / V32) * pre.abs()
            pre = pre + r
        ref = torch.relu(pre) if L.relu else pre
        K = w.shape[1] * w.shape[2] * w.shape[3]
        acc = 18 * math.ceil(K / 16) * ULP32 * A + (3 + min(32, K // 128)) * V32 * (A + bb.abs() + extra)
        if L.up:
            acc = acc + U16 * A                                    # the summed sub-pixel weights are rounded to fp16 once
        bound = SAFETY * (acc + U16 * ref.abs() + SUB16)
        ratio = ((got - ref).abs() / bound).max().item()
        real = np.abs(L.w).reshape(L.w.shape[0], -1).max(1) > 0
        if (~real).any():
            assert torch.all(got[:, torch.from_numpy(~real).cuda()] == 0), f"{L.name}: a padded channel is not zero"
        amax = got.abs().max().item()
        report.append((L.name, variants[L.name]["kernel"], ratio, amax))
        if ratio > 1.0:
            bad.append((L.name, ratio))
        assert amax < 2.0 ** 14, f"{L.name}: largest activation {amax}"
    for r in report:
        print("  %-32s kernel %d  err/bound %.3f  max|act| %.2f" % r)
    ran = {name: v["kernel"] for name, v in variants.items()}
    want = {L.name: _want_kernel(L) for L in net.layers}
    assert ran == want, {n: (ran[n], want[n]) for n in ran if ran[n] != want[n]}
    assert not bad, bad
    lab = ctx.download(p.labels)
    assert lab.max() < R.N_CLASSES
    p.close()


def _interp64(lg):
    """float64 bilinear align_corners=True of [n, 64, 64, C] -> [n, C, 512, 512] and the fp32 arithmetic's error bound."""
    t = torch.from_numpy(lg.astype(np.float64)).permute(0, 3, 1, 2).cuda()
    v = R.upsample(t)
    bound = 16 * V32 * R.upsample(t.abs()) + 1e-30
    return v, bound


def test_upsample_argmax_against_float64():
    from livetalking_b200.ops import Ctx
    ctx = Ctx()
    rng = np.random.default_rng(5)
    N = 3
    lg = np.zeros((N, 64, 64, 32), np.float16)
    lg[..., :19] = rng.standard_normal((N, 64, 64, 19)) * 2
    lg[..., 19:] = 100                                          # padded classes are never read
    lg[2, ..., :19] = -10                                       # image 2: classes 3 and 7 tie exactly everywhere
    lg[2, ..., 3] = lg[2, ..., 7] = rng.standard_normal((64, 64)) + 20
    out = ctx.alloc((N, 512, 512), np.uint8)
    ctx.bisenet_upsample_argmax(ctx.upload(lg), N, 19, out)
    got = ctx.download(out).astype(np.int64)
    ctx.close()
    v, b = _interp64(lg[..., :19])
    top2 = v.topk(2, 1).values
    margin = (top2[:, 0] - top2[:, 1]).cpu().numpy()
    bmax = b.max(1).values.cpu().numpy()
    want = v.argmax(1).cpu().numpy()
    clear = margin > 2 * bmax
    assert np.all(got[:2][clear[:2]] == want[:2][clear[:2]])
    near = (v >= (top2[:, :1] - 2 * b.max(1, keepdim=True).values)).cpu().numpy()
    n_idx, y_idx, x_idx = np.nonzero(~clear[:2])
    assert np.all(near[n_idx, got[n_idx, y_idx, x_idx], y_idx, x_idx])
    assert np.all(got[2] == 3)


@pytest.mark.parametrize("N", [16, 5])
def test_end_to_end_against_oracle(net, sd, N):
    """Largest |logit| error against float64, measured on an H100 80GB HBM3 with the synthetic weights: 4.9e-3 at B = 16 and
    6.2e-3 at B = 5 (logits up to 3.2); LOGIT_ERR = 6.5e-3 bounds it and T_LABEL = 4 x LOGIT_ERR.  The synthetic skin class is a
    1.05x copy of the background class (oracle/bisenet_ref.py), so near-ties are common: about a third of the pixels have a top-2
    margin above 0.08."""
    from livetalking_b200.bisenet import BiSeNetParser
    from livetalking_b200.plugin import musetalk_face_parsing as mfp
    p = BiSeNetParser(net, N)
    crops = _crops(N, 21 + N)
    lab = p.parse(crops)
    lg = torch.from_numpy(p.ctx.download(p.buf["logits"]).astype(np.float64)).permute(0, 3, 1, 2).cuda()
    lab2 = p.parse(crops[: N - 2])                 # partial batch: the same per-image result
    np.testing.assert_array_equal(lab2, lab[: N - 2])
    fw = R.folded(sd)
    with torch.no_grad():
        lg64 = R.forward(fw, R.prep(crops).double().cuda())
    assert torch.all(lg[:, 19:] == 0)
    err = (lg[:, :19] - lg64).abs().max().item()
    print(f"  [B={N}] largest logit error {err:.3e} (logits up to {lg64.abs().max().item():.2f})")
    assert err <= LOGIT_ERR
    agree = 0
    for i in range(N):
        v = R.upsample(lg64[i:i + 1])[0]
        top2 = v.topk(2, 0).values
        clear = ((top2[0] - top2[1]) > T_LABEL).cpu().numpy()
        want = v.argmax(0).cpu().numpy()
        assert np.all(lab[i][clear] == want[clear]), i
        agree += clear.mean()
    assert agree / N > 0.3
    fp = mfp.FaceParsing(90, 90, make_parser=lambda n: BiSeNetParser(net, n))
    from PIL import Image
    for mode in ("raw", "neck", "jaw"):
        im = Image.fromarray(np.ascontiguousarray(crops[0]))
        got = np.asarray(fp(im, mode=mode))
        np.testing.assert_array_equal(got, R.postprocess(lab[0], mode, 90, 90))
    fp.close()
    p.close()


def test_generate_avatar_on_the_engine(net, sd, tmp_path, monkeypatch):
    sys.path.insert(0, os.path.dirname(__file__))
    import stubs
    stubs.install()
    import cv2
    from PIL import Image
    from transformers import WhisperConfig, WhisperModel
    import registry
    from livetalking_b200.bisenet import BiSeNetParser
    from livetalking_b200.musetalk import encode_avatar_latents
    from livetalking_b200.plugin import musetalk_avatar as MT
    from livetalking_b200.plugin import musetalk_face_parsing as mfp
    from livetalking_b200.plugin import musetalk_genavatar as G
    from oracle import musetalk_ref as M
    from oracle import paste_ref as P
    from oracle import s3fd_ref

    torch.manual_seed(1)
    wm = WhisperModel(WhisperConfig(d_model=384, encoder_layers=4, encoder_attention_heads=6, encoder_ffn_dim=1536, decoder_layers=1,
                                    decoder_attention_heads=6, decoder_ffn_dim=64)).eval()
    model = MT.make_model(M.synth_unet_state_dict(M.UNET_SMALL), M.synth_vae_state_dict(M.VAE_SMALL), wm.state_dict(), M.UNET_SMALL,
                          M.VAE_SMALL)
    n = 20
    frames = pfld_ref.synth_video_frames(n, 720, 1280, seed=9)
    vid = str(tmp_path / "clip.avi")
    s3fd_ref.write_video(vid, frames)
    boxes = [(400 + 9 * i, 200 + 5 * i, 700 + 9 * i, 560 + 3 * i) for i in range(n)]
    lms = [R.synth_landmarks(b, seed=i) for i, b in enumerate(boxes)]
    enc = lambda crops: encode_avatar_latents(model.net, crops)  # noqa: E731
    fw = R.folded(sd)
    clear = []

    class Oracle:
        def parse(self, rgb):
            with torch.no_grad():
                v = R.upsample(R.forward(fw, R.prep(rgb).double().cuda()))
            top2 = v.topk(2, 1).values
            clear.extend(((top2[:, 0] - top2[:, 1]) > T_LABEL).cpu().numpy())
            return v.argmax(1).cpu().numpy().astype(np.uint8)

        def close(self):
            pass

    save = tmp_path / "data" / "avatars"
    split = {}
    eng_labels, ora_labels = [], []

    def recorder(make, store):
        def mk(N):
            inner = make(N)

            class Rec:
                def parse(self, rgb):
                    out = inner.parse(rgb)
                    store.extend(out)
                    return out

                def close(self):
                    inner.close()
            return Rec()
        return mk

    G.generate_avatar(vid, "eng", save_path=str(save), detect=lambda fr: list(boxes), landmarks=R.ReplayLandmarks(lms),
                      face_parsing=mfp.FaceParsing(90, 90, make_parser=recorder(lambda N: BiSeNetParser(net, N), eng_labels)),
                      encode_latents=enc, timings=split)
    assert {"decode", "full_png", "detect", "latents", "masks", "pack"} <= set(split)
    G.generate_avatar(vid, "ora", save_path=str(save), detect=lambda fr: list(boxes), landmarks=R.ReplayLandmarks(lms),
                      face_parsing=mfp.FaceParsing(90, 90, make_parser=recorder(lambda N: Oracle(), ora_labels)), encode_latents=enc)
    assert len(eng_labels) == len(ora_labels) == len(clear) == n
    for name in ("coords.pkl", "mask_coords.pkl"):
        assert (save / "eng" / name).read_bytes() == (save / "ora" / name).read_bytes()
    with open(save / "eng" / "coords.pkl", "rb") as f:
        coords = [[int(v) for v in c] for c in pickle.load(f)]
    with open(save / "eng" / "mask_coords.pkl", "rb") as f:
        crop_boxes = [[int(v) for v in c] for c in pickle.load(f)]
    # the engine's labels equal the float64 oracle's wherever its margin is clear, and every engine mask is the reference's host
    # path (oracle post-processing, then get_image_prepare_material's crop, resize, paste and blur) applied to the engine's labels
    for i in range(n):
        np.testing.assert_array_equal(eng_labels[i][clear[i]], ora_labels[i][clear[i]], err_msg=f"frame {i}")
        frame = cv2.imread(str(save / "eng" / "full_imgs" / f"{i:08d}.png"))
        face_large, crop_box = mfp.crop_for_parsing(frame, coords[i])
        want, box = mfp.finish_material(face_large, Image.fromarray(R.postprocess(eng_labels[i], "jaw", 90, 90)), coords[i], crop_box)
        assert box == crop_boxes[i]
        np.testing.assert_array_equal(cv2.imread(str(save / "eng" / "mask" / f"{i:08d}.png"), cv2.IMREAD_UNCHANGED), want,
                                      err_msg=f"frame {i}")
    print(f"  {n} masks checked, {np.mean([c.mean() for c in clear]):.2f} of the label pixels clear; timings {split}")

    monkeypatch.chdir(tmp_path)
    packed = MT.load_avatar("eng", model)
    os.remove(save / "eng" / "avatar.ltbav")
    from_dir = MT.load_avatar("eng", model)
    for pl in (packed, from_dir):
        assert len(pl[0]) == len(pl[1]) == len(pl[2]) == len(pl[3]) == len(pl[4]) == n
        assert pl.engine_avatar is not None and pl.engine_avatar.lat_hw == 32
    for a, b in zip(packed[1], from_dir[1]):
        np.testing.assert_array_equal(a, b)
    assert [tuple(int(v) for v in c) for c in packed[2]] == [tuple(c) for c in coords]
    lat = torch.load(save / "eng" / "latents.pt")
    assert len(lat) == n and lat[0].shape == (1, 8, 32, 32) and lat[0].dtype == torch.float16
    # one inference_batch + paste_back_frame on the generated avatar
    B = 2
    av = registry.create("avatar", "musetalk", opt=stubs.Opt(batch_size=B), model=model, avatar=from_dir)
    feats = [f.numpy() for f in M.synth_latents_and_audio(B, seed=5)[1]]
    pred = av.inference_batch(3, feats)
    assert pred.shape == (B, 256, 256, 3) and pred.dtype == np.uint8
    for k in range(B):
        out = av.paste_back_frame(pred[k], 3 + k)
        want = P.mt_paste_back(pred[k], from_dir[0][3 + k], from_dir[2][3 + k], from_dir[1][3 + k], from_dir[3][3 + k])
        np.testing.assert_array_equal(out, want)
    av.close()
