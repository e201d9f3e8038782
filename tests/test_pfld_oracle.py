"""CPU: oracle/pfld_ref.py and the host side of the UltraLight avatar generator against the unmodified reference's outputs in
tests/golden/pfld_golden.npz (tests/golden/make_pfld_golden.py), and the padded device layout of livetalking_b200/pfld.py against
the unpadded folded network."""
import io
import os
import pickle
import zlib

import cv2
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import pfld_ref as R

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def g():
    return np.load(os.path.join(GOLDEN, "pfld_golden.npz"))


@pytest.fixture(scope="module")
def sd():
    return R.synth_state_dict(0)


@pytest.fixture(scope="module")
def mean_face():
    return R.read_mean_face(os.path.join(GOLDEN, "pfld_mean_face.txt"))


def test_folded_net_matches_train_time_reference(g, sd):
    """The float64 fold of every MobileOneBlock, run in fp32, against PFLD_GhostOne's six-branch train-time forward."""
    with torch.no_grad():
        out = R.forward(R.folded(sd), R.prep(g["net_crops"])).numpy()
    ref = g["net_out"]
    assert out.shape == ref.shape == (4, 220)
    assert np.abs(out - ref).max() <= 1e-4 * np.abs(ref).max(), np.abs(out - ref).max()
    assert np.abs(ref).max() > 0.02          # landmarks move away from the mean face
    with torch.no_grad():                     # the train-time restatement the benchmark times
        assert np.abs(R.forward_train(sd, R.prep(g["net_crops"])).numpy() - ref).max() <= 1e-6 * np.abs(ref).max()


def test_reparameterised_state_dict_is_accepted(sd):
    fw = R.folded(sd)
    rep = {k: v for k, v in sd.items() if not any(t in k for t in (".rbr_conv.", ".rbr_scale.", ".rbr_skip."))}
    for p, (w, b, *_rest) in fw.items():
        if p not in ("conv8", "conv_out"):
            rep[p + ".reparam_conv.weight"], rep[p + ".reparam_conv.bias"] = w.float(), b.float()
    from livetalking_b200 import pfld
    a, _, _ = pfld.plan(sd)
    b, _, _ = pfld.plan({"pfld_backbone": rep})
    for la, lb in zip(a, b):
        assert la.name == lb.name
        assert np.abs(la.w - lb.w).max() <= 2.0 ** -10 * max(1.0, np.abs(la.w).max()), la.name   # fp32 round trip of the fold
        assert np.allclose(la.b, lb.b, rtol=1e-6, atol=1e-7), la.name


def _run_plan(layers, bufs, taps, x):
    """The padded device plan in float64 on the CPU (NCHW): returns the 256 features of the five taps' real channels."""
    t = {"in": torch.zeros(x.shape[0], 16, 192, 192, dtype=torch.float64)}
    t["in"][:, :3] = x
    for name, (h, w, c) in bufs.items():
        if name != "in":
            t[name] = torch.full((x.shape[0], c, h, w), float("nan"), dtype=torch.float64)
    for L in layers:
        src, c_in, C = L.src
        dst, c_out, Co = L.dst
        wt, b = torch.from_numpy(L.w).double(), torch.from_numpy(L.b).double()
        if L.name == "conv8":
            xin = t[src].permute(0, 2, 3, 1).reshape(x.shape[0], -1, 1, 1)
            y = F.conv2d(xin, wt, b)
        elif L.kind == "dw":
            y = F.conv2d(t[src][:, c_in:c_in + C], wt, b, stride=L.stride, padding=1, groups=C)
        else:
            k = wt.shape[-1]
            y = F.conv2d(t[src][:, c_in:c_in + C], wt, b, stride=L.stride, padding=k // 2)
        t[dst][:, c_out:c_out + Co] = torch.relu(y) if L.relu else y
    feats = [t[name][:, idx].mean((2, 3)) for name, idx in taps]
    return torch.cat(feats, 1), t


def test_padded_layout_computes_the_unpadded_network(sd):
    """The padded half-channels hold exact zeros and the zero-padded consumer weights see only the real channels: the device plan
    in float64 equals the folded network (with the same fp16 weights and fp32 biases) in float64."""
    from livetalking_b200 import pfld
    layers, bufs, taps = pfld.plan(sd)
    fw = R.folded(sd)
    h16 = lambda w: torch.from_numpy(w.numpy().astype(np.float16)).double()      # noqa: E731  (one rounding, as numpy does it)
    fw16 = {k: ((h16(w) if k != "conv_out" else w), None if b is None else b.float().double(), *r) for k, (w, b, *r) in fw.items()}
    x = R.prep(R.synth_video_frames(2, 192, 192, seed=5)).double()
    keep = {}
    with torch.no_grad():
        R.forward(fw16, x, keep)
        feat, t = _run_plan(layers, bufs, taps, x)
    want = keep["multi_scale"].reshape(2, -1)
    assert feat.shape == (2, 256)
    assert torch.allclose(feat, want, rtol=1e-12, atol=1e-12), (feat - want).abs().max()
    for L in layers:                                    # every padded channel is an exact zero
        dst, c_out, Co = L.dst
        assert torch.isfinite(t[dst]).all(), dst
    for name, idx in taps[1:4]:
        pad = sorted(set(range(t[name].shape[1])) - set(idx))
        assert pad and torch.all(t[name][:, pad] == 0), name
    # alignment the kernels need: Cin, Cout of every planner conv % 16, every depthwise C / c_off % 8
    for L in layers:
        if L.kind == "conv":
            assert L.w.shape[0] % 16 == 0 and L.w.shape[1] % 16 == 0, L.name
        else:
            assert L.src[1] % 8 == 0 and L.dst[1] % 8 == 0 and L.src[2] % 8 == 0, L.name


def test_fp16_range_is_checked(sd):
    from livetalking_b200 import pfld
    bad = dict(sd)
    bad["conv7.rbr_conv.0.conv.weight"] = sd["conv7.rbr_conv.0.conv.weight"] * 1e5
    with pytest.raises(ValueError, match="fp16 range"):
        pfld.plan(bad)


def test_flop_count_matches_oracle():
    from livetalking_b200 import pfld
    assert abs(pfld.gflop_per_frame() - R.gflop_per_frame()) < 1e-12
    assert [b[1:] for b in pfld._blocks()] == [b[1:] for b in R.mobileone_blocks()]
    assert [b[0] for b in pfld._blocks()] == [b[0] for b in R.mobileone_blocks()]


def _decoded(g, tmp_path):
    vid = tmp_path / "clip.avi"
    vid.write_bytes(g["ga_video"].tobytes())
    cap = cv2.VideoCapture(str(vid))
    frames = []
    while True:
        ok, f = cap.read()
        if not ok:
            break
        frames.append(f)
    return str(vid), frames


def test_face_det_and_landmarks_match_reference(g, sd, mean_face, tmp_path):
    """face_det (boxes, border shift, crop size) bit-exact; the oracle's landmarks equal Landmark.detect's wherever the value is not
    within 1e-3 px of an integer."""
    from livetalking_b200.plugin import ultralight_genavatar as G
    _, frames = _decoded(g, tmp_path)
    det = R.ReplayDetector(R.face_records(g["ga_boxes"].tolist()))
    fw = R.folded(sd)
    for i, img in enumerate(frames):
        cropped, x1, y1 = G.face_det(img, det, i)
        assert (int(x1), int(y1)) == tuple(g["ga_x1y1"][i]), i
        assert (cropped.shape[1], cropped.shape[0]) == tuple(g["ga_crop_wh"][i]), i
        ref_c, ref_box = R.face_det(img, R.ReplayDetector(R.face_records([g["ga_boxes"][i].tolist()])))
        assert np.array_equal(cropped, ref_c) and ref_box[:2] == [x1, y1]
        with torch.no_grad():
            raw = R.forward(fw, R.prep(cv2.resize(cropped, (192, 192))[None])).numpy()[0]
        lms = R.landmarks(raw, mean_face, cropped.shape[1], cropped.shape[0])
        exact = (raw.astype(np.float32) + mean_face).reshape(-1, 2) * np.array([cropped.shape[1], cropped.shape[0]], np.float32)
        near = np.abs(exact - np.round(exact)) < 1e-3
        assert np.all((lms == g["ga_lms"][i]) | near), i
    assert (g["ga_x1y1"] < 0).any()           # the border case is in the golden
    with pytest.raises(ValueError, match="frame 4: no face"):
        G.face_det(frames[0], R.ReplayDetector([(np.zeros((0, 4)), np.zeros(0, np.int32), np.zeros((0, 5, 2)))]), 4)


def test_generate_avatar_host_path_bit_exact(g, tmp_path):
    """generate_avatar with the reference's landmarks injected: full and face PNG bytes and coords.pkl bytes equal the reference's."""
    from livetalking_b200.plugin import ultralight_genavatar as G
    vid, _ = _decoded(g, tmp_path)
    lms = g["ga_lms"]

    class Replay:
        def __init__(self, N):
            self.i = 0

        def run(self, crops, wh):
            n = len(crops)
            assert crops.shape[1:] == (192, 192, 3) and wh.shape == (n, 2)
            np.testing.assert_array_equal(wh, g["ga_crop_wh"][self.i:self.i + n])
            out = lms[self.i:self.i + n]
            self.i += n
            return out.astype(np.float32), out

        def close(self):
            pass
    ckpt = tmp_path / "ul.pth"
    ckpt.write_bytes(b"unet")
    progress, split = [], {}
    det = R.ReplayDetector(R.face_records(g["ga_boxes"].tolist()))
    G.generate_avatar(vid, "ga", save_path=str(tmp_path / "av"), checkpoint=str(ckpt), detector=det, make_landmarker=Replay,
                      progress_callback=progress.append, timings=split)
    av = tmp_path / "av" / "ga"
    crc = lambda d: np.array([zlib.crc32((av / d / f).read_bytes()) for f in sorted(os.listdir(av / d))], np.uint32)  # noqa: E731
    np.testing.assert_array_equal(crc("full_imgs"), g["ga_full_crc"])
    np.testing.assert_array_equal(crc("face_imgs"), g["ga_face_crc"])
    assert (av / "coords.pkl").read_bytes() == g["ga_coords_pkl"].tobytes()
    assert (av / "ultralight.pth").read_bytes() == b"unet"
    assert (av / "avatar.ltbav").exists()
    coords = pickle.load(io.BytesIO(g["ga_coords_pkl"].tobytes()))
    assert coords[7][2] == 320 and coords[7][2] - coords[7][0] < coords[7][3] - coords[7][1] + 5     # sliced at the right edge
    assert progress[0] == 5 and progress[-1] == 100 and progress == sorted(progress)
    assert {"decode", "full_png", "detect", "landmarks", "face_png", "pack"} == set(split)


def test_mouth_crop_slicing_and_interpolation():
    """numpy slicing of the reference (a negative start counts from the end), w / h of the sliced crop in the coords, INTER_LINEAR
    (cv2.resize's third positional argument is dst), and a clear error where the reference's cv2.resize fails."""
    from livetalking_b200.plugin import ultralight_genavatar as G
    img = np.random.default_rng(0).integers(0, 256, (100, 120, 3), dtype=np.uint8)
    lms = np.zeros((110, 2), np.int32)
    lms[1], lms[31], lms[52] = (10, 0), (50, 0), (0, 30)
    lms[1], lms[31] = (5, 0), (25, 0)
    crop, box = G.mouth_crop(img, lms, np.int32(-30), np.int32(60), 24)           # xmin -25, xmax -5: wraps to columns 95..115
    np.testing.assert_array_equal(crop, cv2.resize(img[90:100, -25:-5], (24, 24), interpolation=cv2.INTER_LINEAR))
    assert box == (-25, 90, -25 + 20, 90 + 10)
    lms[1], lms[31], lms[52] = (100, 0), (140, 0), (0, 70)                         # past the right and bottom edges
    crop, box = G.mouth_crop(img, lms, 0, 0, 16)
    assert box == (100, 70, 120, 100)
    assert not np.array_equal(crop, cv2.resize(img[70:110, 100:140], (16, 16), interpolation=cv2.INTER_AREA))
    with pytest.raises(ValueError, match="frame 9: the mouth box"):
        lms[1], lms[31], lms[52] = (10, 0), (50, 0), (0, 10)
        G.mouth_crop(img, lms, 0, -20, 16, 9)                                      # ymin -10 -> img[-10:30] is empty


def test_cli_matches_reference(g):
    from livetalking_b200.plugin import ultralight_genavatar as G
    ours = [f"{a.dest}|{a.default}|{getattr(a.type, '__name__', None)}" for a in G.parser()._actions if a.dest != "help"]
    assert ours == g["ga_args"].tolist()


def test_missing_weights_raise(tmp_path, monkeypatch):
    from livetalking_b200.plugin import ultralight_genavatar as G
    monkeypatch.chdir(tmp_path)
    with pytest.raises(FileNotFoundError, match="PFLD checkpoint"):
        G.generate_avatar("none.mp4", "x", save_path=str(tmp_path))
    assert not (tmp_path / "x").exists()
