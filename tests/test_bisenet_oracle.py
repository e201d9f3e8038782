"""CPU: the BiSeNet oracle (oracle/bisenet_ref.py) and the engine's host-side plan (livetalking_b200/bisenet.py) against the golden
file made by running the unmodified reference (tests/golden/make_bisenet_golden.py)."""
import os
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import bisenet_ref as R
from oracle import pfld_ref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bisenet_golden.npz")


@pytest.fixture(scope="module")
def g():
    return np.load(GOLDEN)


def test_oracle_matches_the_reference_network(g):
    rgb = np.ascontiguousarray(pfld_ref.synth_video_frames(2, 512, 512, seed=3)[..., ::-1])
    assert zlib.crc32(rgb.tobytes()) == int(g["net_rgb_crc"])
    with torch.no_grad():
        out = R.upsample(R.forward(R.folded(R.synth_state_dict(0)), R.prep(rgb).double())).numpy()
    ref = g["net_logits_s8"].astype(np.float64)
    assert np.abs(out[:, :, ::8, ::8] - ref).max() <= 1e-4 * np.abs(ref).max()
    top2 = np.sort(out, 1)[:, -2:]
    clear = (top2[:, 1] - top2[:, 0]) > 1e-4 * np.abs(ref).max()
    assert clear.mean() > 0.99
    np.testing.assert_array_equal(out.argmax(1)[clear], g["net_labels"][clear])


def test_s2d_stem_equals_the_7x7_stride2_conv():
    from livetalking_b200.bisenet import s2d_stem
    rng = np.random.default_rng(0)
    w7 = rng.standard_normal((64, 3, 7, 7))
    x = torch.from_numpy(rng.standard_normal((2, 3, 512, 512)))
    ref = F.conv2d(x, torch.from_numpy(w7), stride=2, padding=3)
    got = F.conv2d(R.space_to_depth(x), torch.from_numpy(s2d_stem(w7)))
    assert got.shape == ref.shape
    assert (got - ref).abs().max().item() <= 1e-12 * ref.abs().max().item()


@pytest.mark.parametrize("mode", ["raw", "neck", "jaw"])
def test_mode_postprocessing_bit_exact(g, mode):
    from livetalking_b200.plugin import musetalk_face_parsing as mfp
    lab = g["fp_labels"]
    np.testing.assert_array_equal(R.postprocess(lab, mode, 90, 90), g["fp_" + mode])
    fp = mfp.FaceParsing(90, 90, make_parser=lambda n: _Replay([lab]))
    np.testing.assert_array_equal(mfp.labels_to_mask(lab, mode, fp.kernel, fp.cheek_kernel, fp.cheek_mask), g["fp_" + mode])


class _Replay:
    """A parser that hands back recorded label maps in order (and records the crops it was given)."""

    def __init__(self, labels):
        self.labels, self.i, self.seen = list(labels), 0, []

    def parse(self, rgb):
        self.seen += [zlib.crc32(np.ascontiguousarray(r).tobytes()) for r in rgb]
        out = np.stack(self.labels[self.i:self.i + len(rgb)])
        self.i += len(rgb)
        return out

    def close(self):
        pass


def test_face_parsing_call_matches_the_reference(g):
    from PIL import Image
    from livetalking_b200.plugin import musetalk_face_parsing as mfp
    img = Image.fromarray(np.ascontiguousarray(pfld_ref.synth_video_frames(1, 280, 300, seed=5)[0][..., ::-1]))
    assert zlib.crc32(np.asarray(img).tobytes()) == int(g["fp_img_crc"])
    rep = _Replay([g["fp_labels"]] * 3)
    fp = mfp.FaceParsing(90, 90, make_parser=lambda n: rep)
    for mode in ("raw", "neck", "jaw"):
        got = fp(img, mode=mode)
        assert got.mode == "L"
        np.testing.assert_array_equal(np.asarray(got), g["fp_" + mode])


def test_plan_layout_and_range_checks():
    from livetalking_b200 import bisenet as B
    sd = R.synth_state_dict(0)
    layers, gates, bufs = B.plan(sd)
    assert len(layers) == 27 and set(gates) == {"avg", "att32", "att16", "attffm"}
    assert abs(B.gflop_per_frame() - 26.77) < 0.01
    cls = [L for L in layers if L.name == "classes"][0]
    assert cls.w.shape == (32, 256, 1, 1) and np.all(cls.w[19:] == 0) and np.all(cls.b == 0)
    stem = layers[0]
    assert stem.w.shape == (64, 16, 4, 4) and np.all(stem.w[:, 12:] == 0)
    bad = dict(sd)
    bad["cp.resnet.layer3.0.bn1.weight"] = sd["cp.resnet.layer3.0.bn1.weight"] * 1e6
    with pytest.raises(ValueError, match="fp16"):
        B.plan(bad)
