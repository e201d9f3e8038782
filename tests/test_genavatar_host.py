"""CPU: the host side of livetalking_b200/plugin/wav2lip_genavatar.generate_avatar, with a fake detector that returns the
unmodified reference's per-frame detections (tests/golden/s3fd_golden.npz): the None branch, pads and clamps, the int64 smoothing,
the coords.pkl order, the face PNG bytes, the progress sequence, the batch halving, avatar.ltbav, and the no-download rule."""
import os
import pickle
import zlib

import numpy as np
import pytest
import torch.hub
import torch.utils.model_zoo

from livetalking_b200 import avatar_pack
from livetalking_b200.plugin import wav2lip_genavatar as G

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "s3fd_golden.npz")


@pytest.fixture(autouse=True)
def no_download(monkeypatch):
    def boom(*a, **k):
        raise AssertionError("a download was attempted")
    monkeypatch.setattr(torch.utils.model_zoo, "load_url", boom)
    monkeypatch.setattr(torch.hub, "load_state_dict_from_url", boom)


@pytest.fixture(scope="module")
def g():
    return np.load(GOLDEN)


class FakeDetector:
    """Replays the reference's detections in frame order; fails allocation above max_batch like a too-large engine graph."""

    def __init__(self, dets, N, max_batch):
        if N > max_batch:
            raise RuntimeError("device allocation failed")
        self.dets, self.N, self.pos = dets, N, 0

    def detect(self, frames):
        assert 1 <= len(frames) <= self.N
        out = self.dets[self.pos:self.pos + len(frames)]
        self.pos += len(frames)
        return out

    def close(self):
        pass


def _dets(g):
    return [tuple(int(v) for v in b) if f else None for f, b in zip(g["ga_det_found"], g["ga_det_box"])]


def _run(tmp_path, g, max_batch=16, batch=4):
    vid = tmp_path / "clip.avi"
    vid.write_bytes(g["ga_video"].tobytes())
    dets, log, progress = _dets(g), [], []

    def make(N, H, W):
        det = FakeDetector(dets, N, max_batch)
        log.append(N)
        return det
    G.generate_avatar(str(vid), "ga", save_path=str(tmp_path / "avatars"), face_det_batch_size=batch, progress_callback=progress.append,
                      make_detector=make)
    return tmp_path / "avatars" / "ga", progress, log


def test_generate_avatar_bit_exact_with_reference(tmp_path, g):
    av, progress, log = _run(tmp_path, g)
    assert log == [4]
    assert progress == list(g["ga_progress"])
    with open(av / "coords.pkl", "rb") as fh:
        coords = pickle.load(fh)
    assert all(type(v) is int for c in coords for v in c)
    np.testing.assert_array_equal(np.array(coords), g["ga_coords"])
    crc = lambda d: [zlib.crc32((av / d / f).read_bytes()) for f in sorted(os.listdir(av / d))]  # noqa: E731
    assert crc("face_imgs") == list(g["ga_face_crc"])
    assert crc("full_imgs") == list(g["ga_full_crc"])
    assert not g["ga_det_found"].all() and g["ga_det_found"].any()       # the None branch (full-frame box) is exercised


def test_packed_avatar_round_trips(tmp_path, g):
    av, _, _ = _run(tmp_path, g)
    frames, faces, coords = avatar_pack.read_wav2lip_dir(str(av))
    pf, pfa, pc = avatar_pack.load_packed(str(av / "avatar.ltbav")).wav2lip_lists()
    assert len(pf) == len(frames) == len(pfa) == len(faces)
    for a, b in zip(pf, frames):
        np.testing.assert_array_equal(a, b)
    for a, b in zip(pfa, faces):
        np.testing.assert_array_equal(a, b)
    np.testing.assert_array_equal(np.asarray(pc), np.asarray(coords))


def test_allocation_failure_halves_the_batch(tmp_path, g):
    av, progress, log = _run(tmp_path, g, max_batch=2, batch=8)
    assert log == [2]                                           # 8 -> 4 -> 2 (the factories that raised never returned)
    with open(av / "coords.pkl", "rb") as fh:
        np.testing.assert_array_equal(np.array(pickle.load(fh)), g["ga_coords"])
    with pytest.raises(RuntimeError, match="Image too big"):
        _run(tmp_path, g, max_batch=0, batch=2)


def test_missing_weights_raise_and_never_download(tmp_path, g, monkeypatch):
    monkeypatch.chdir(tmp_path)
    vid = tmp_path / "clip.avi"
    vid.write_bytes(g["ga_video"].tobytes())
    with pytest.raises(FileNotFoundError, match="s3fd.pth"):
        G.generate_avatar(str(vid), "x", save_path=str(tmp_path / "avatars"))
    with pytest.raises(FileNotFoundError):
        G.generate_avatar(str(vid), "x", save_path=str(tmp_path / "avatars"), weights_path=str(tmp_path / "nope.pth"))
    assert not (tmp_path / "avatars").exists()


def test_smoothing_is_the_reference_int_rule():
    b = np.array([[0, 0, 10, 10], [1, 1, 11, 11], [3, 2, 13, 12], [7, 3, 17, 13], [9, 9, 19, 19], [2, 2, 3, 3]])
    want = b.copy()
    for i in range(len(want)):                         # restated: in place, truncating int64 means
        w = want[len(want) - 5:] if i + 5 > len(want) else want[i:i + 5]
        want[i] = np.mean(w, axis=0)
    got = G.get_smoothened_boxes(b.copy(), T=5)
    assert got.dtype == np.int64
    np.testing.assert_array_equal(got, want)
