"""CPU: the host steps of the MuseTalk avatar generator (plugin/musetalk_genavatar.py, plugin/musetalk_face_parsing.py) bit for bit
against the unmodified reference's generate_avatar run recorded in tests/golden/bisenet_golden.npz, with the detector, landmarks,
parser and latents replaced by replaying fakes."""
import json
import os
import pickle
import zlib

import numpy as np
import pytest
import torch

from oracle import bisenet_ref as R

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bisenet_golden.npz")


class _Replay:
    def __init__(self, labels):
        self.labels, self.i, self.seen = list(labels), 0, []

    def parse(self, rgb):
        self.seen += [zlib.crc32(np.ascontiguousarray(r).tobytes()) for r in rgb]
        out = np.stack(self.labels[self.i:self.i + len(rgb)])
        self.i += len(rgb)
        return out

    def close(self):
        pass


@pytest.fixture(scope="module")
def g():
    return np.load(GOLDEN)


def _run(g, tmp_path, boxes=None, batch_size=3):
    from livetalking_b200.plugin import musetalk_face_parsing as mfp
    from livetalking_b200.plugin import musetalk_genavatar as G
    vid = tmp_path / "clip.avi"
    vid.write_bytes(g["ga_video"].tobytes())
    rep = _Replay(g["ga_labels"])
    crops, progress = [], []

    def enc(c):
        crops.extend(zlib.crc32(np.ascontiguousarray(x).tobytes()) for x in c)
        return np.stack([np.full((8, 32, 32), float(x.mean()) / 255, np.float32) for x in c])
    boxes = [tuple(int(v) for v in b) for b in g["ga_boxes"]] if boxes is None else boxes
    lms = R.ReplayLandmarks([R.synth_landmarks(tuple(int(v) for v in b), seed=i) for i, b in enumerate(g["ga_lm_boxes"])])
    G.generate_avatar(str(vid), "ga", save_path=str(tmp_path / "av"), progress_callback=progress.append, detect=lambda fr: list(boxes),
                      landmarks=lms, face_parsing=mfp.FaceParsing(90, 90, make_parser=lambda n: rep, batch_size=batch_size),
                      encode_latents=enc, batch_size=batch_size)
    return tmp_path / "av" / "ga", rep, crops, progress, str(vid)


def test_generate_avatar_bit_exact(g, tmp_path):
    av, rep, crops, progress, vid = _run(g, tmp_path)
    crc = lambda d: [zlib.crc32((av / d / f).read_bytes()) for f in sorted(os.listdir(av / d))]  # noqa: E731
    assert rep.seen == [int(v) for v in g["ga_rgb_crc"]]                  # the PIL crops and resizes the parser saw
    assert crops == [int(v) for v in g["ga_latent_crc"]]                  # the LANCZOS4 crops handed to the VAE
    assert crc("full_imgs") == [int(v) for v in g["ga_full_crc"]]
    assert crc("mask") == [int(v) for v in g["ga_mask_crc"]]
    assert (av / "coords.pkl").read_bytes() == g["ga_coords_pkl"].tobytes()
    assert (av / "mask_coords.pkl").read_bytes() == g["ga_mask_coords_pkl"].tobytes()
    info, ref = json.loads((av / "avator_info.json").read_text()), json.loads(g["ga_info"].tobytes())
    assert list(info) == list(ref) and info["video_path"] == vid and {k: info[k] for k in info if k != "video_path"} == \
        {k: ref[k] for k in ref if k != "video_path"}
    assert progress == [int(v) for v in g["ga_progress"]]
    with open(av / "mask_coords.pkl", "rb") as f:
        assert min(pickle.load(f)[2][:2]) < 0                            # frame 2's crop box leaves the frame at the top-left
    lat = torch.load(av / "latents.pt")
    assert len(lat) == 8 and all(t.shape == (1, 8, 32, 32) and t.dtype == torch.float16 for t in lat)
    from livetalking_b200 import avatar_pack
    fr, masks, co, mc, la = avatar_pack.read_musetalk_dir(str(av))
    assert len(fr) == len(masks) == len(co) == len(mc) == len(la) == 8
    packed = avatar_pack.load_packed(str(av / "avatar.ltbav")).musetalk_lists()
    for a, b in zip(packed[1], masks):
        np.testing.assert_array_equal(a, b)


def test_frame_without_a_face_raises(g, tmp_path):
    boxes = [tuple(int(v) for v in b) for b in g["ga_boxes"]]
    boxes[3] = None
    with pytest.raises(ValueError, match="frame 3"):
        _run(g, tmp_path, boxes=boxes)


def test_missing_weights_raise(tmp_path, monkeypatch):
    from livetalking_b200.plugin import musetalk_face_parsing as mfp
    from livetalking_b200.plugin import musetalk_genavatar as G
    monkeypatch.chdir(tmp_path)
    monkeypatch.setattr(torch.hub, "load_state_dict_from_url", lambda *a, **k: pytest.fail("tried to download"))
    with pytest.raises(FileNotFoundError, match="79999_iter.pth"):
        mfp.FaceParsing()
    with pytest.raises(FileNotFoundError, match="s3fd.pth"):
        G.generate_avatar(str(tmp_path / "clip.mp4"), "x", face_parsing=object())
    assert not (tmp_path / "data").exists()


def test_cli_options_match(g):
    import argparse
    from livetalking_b200.plugin import musetalk_genavatar as G
    src = open(G.__file__).read()
    ns = {}
    exec(src[src.index("    parser = argparse.ArgumentParser()"):src.index("    args = parser.parse_args()")].replace("\n    ", "\n").strip(),
         {"argparse": argparse}, ns)
    got = [f"{a.dest}|{a.default}|{getattr(a.type, '__name__', None)}" for a in ns["parser"]._actions if a.dest != "help"]
    assert got == [str(v) for v in g["ga_args"]]


def test_run_app_alias():
    import inspect
    from livetalking_b200 import run_app
    assert '"avatars.musetalk.genavatar"' in inspect.getsource(run_app.install_aliases)


def test_no_face_in_any_frame_raises_before_the_adjust_range(g, tmp_path):
    with pytest.raises(ValueError, match="frame 0 .* and 7 more"):
        _run(g, tmp_path, boxes=[None] * 8)


def test_engine_detection_groups_frames_by_size(tmp_path, monkeypatch):
    """A folder of PNGs may mix frame sizes: each size gets its own detector and the boxes come back in frame order."""
    from livetalking_b200 import s3fd
    from livetalking_b200.plugin import musetalk_genavatar as G
    from livetalking_b200.plugin import wav2lip_genavatar as W
    made = []

    class FakeDetector:
        def __init__(self, net, N, H, W_):
            self.N, self.hw = N, (H, W_)
            made.append((N, H, W_))

        def detect(self, frames):
            assert frames.shape[1:3] == self.hw
            return [(int(f[0, 0, 0]), 0, 1, 1) for f in frames]

        def close(self):
            pass
    monkeypatch.setattr(s3fd, "S3FDDetector", FakeDetector)
    monkeypatch.setattr(W, "load_net", lambda path: None)
    monkeypatch.chdir(tmp_path)
    weights = tmp_path / G.S3FD_REL
    weights.parent.mkdir(parents=True)
    weights.write_bytes(b"")
    sizes = [(40, 60), (50, 30), (40, 60), (50, 30), (40, 60)]
    frames = [np.full((h, w, 3), i, np.uint8) for i, (h, w) in enumerate(sizes)]
    boxes = G._engine_detect(2)(frames)
    assert [b[0] for b in boxes] == list(range(5))
    assert sorted({m[1:] for m in made}) == [(40, 60), (50, 30)]


def test_dense_only_ops_reject_channel_slices():
    from livetalking_b200.ops import Ctx, DevTensor
    sl = DevTensor(0, (1, 8, 8, 16), pitch=32, c_off=16)
    dense = DevTensor(0, (1, 4, 4, 16))
    with pytest.raises(ValueError, match="channel slice"):
        Ctx.maxpool3x3s2(None, sl, 1, 8, 8, dense)
    with pytest.raises(ValueError, match="channel 0"):
        Ctx.bisenet_upsample_argmax(None, sl, 1, 19, DevTensor(0, (1, 64, 64), np.uint8))
