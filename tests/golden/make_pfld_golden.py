"""Writes tests/golden/pfld_golden.npz (and pfld_mean_face.txt, the reference's data file) by running the unmodified LiveTalking
PFLD_GhostOne, Landmark.detect and the UltraLight genavatar script on the CPU:

    python tests/golden/make_pfld_golden.py /path/to/LiveTalking

Weights: oracle.pfld_ref.synth_state_dict(0) in train-time form (six conv branches, scale and skip BatchNorms per MobileOneBlock),
loaded into PFLD_GhostOne() and run in eval mode; the weights are regenerated from the seed by the tests, only inputs and outputs are
stored.  Landmark() reads the synthetic checkpoint from ./models/checkpoint_epoch_335.pth.tar of a temporary working directory,
.cuda() is a no-op, and SCRFD is replaced by oracle.pfld_ref.ReplayDetector over recorded boxes.

Contents:
  net_crops / net_out      u8 BGR 192 x 192 crops and PFLD_GhostOne's output [n, 220] (fp32)
  ga_video                 bytes of the MJPG clip genavatar.py ran on (GA_N frames of GA_H x GA_W)
  ga_boxes                 the replayed SCRFD boxes (x, y, w, h) per frame; frame 3 touches the top-left border (negative x1 and
                           y1 after face_det's shift), frame 7's mouth box runs past the right edge
  ga_lms / ga_x1y1 / ga_crop_wh   Landmark.detect per frame: int32 landmarks, (x1, y1), and the width / height of the bordered crop
  ga_coords_pkl            bytes of coords.pkl;  ga_face_crc / ga_full_crc: zlib.crc32 of the PNG files
  ga_args                  genavatar.py's argparse options as "dest|default|type" strings"""
import os
import pickle
import runpy
import shutil
import sys
import tempfile
import zlib

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import pfld_ref as R  # noqa: E402
from oracle import s3fd_ref  # noqa: E402

GA_N, GA_H, GA_W = 10, 240, 320
GA_BOXES = [(60.4, 50.8, 110.0, 120.5), (62.9, 52.1, 108.3, 119.0), (70.0, 40.5, 100.2, 130.7), (2.6, -20.2, 120.0, 130.0),
            (100.5, 80.25, 90.0, 95.0), (99.1, 60.9, 104.6, 100.1), (150.3, 70.7, 80.0, 90.0), (230.4, 60.6, 100.0, 110.0),
            (120.0, 100.0, 96.0, 96.0), (40.8, 30.3, 150.9, 160.4)]


def main(ref_root):
    sys.path.insert(0, ref_root)
    from avatars.ultralight.face_detect_utils import get_landmark
    from avatars.ultralight.face_detect_utils.pfld_mobileone import PFLD_GhostOne

    sd = R.synth_state_dict(0)
    net = PFLD_GhostOne()
    net.load_state_dict(sd)                  # strict: the synthetic keys are exactly the module's
    net.eval()
    out = {}
    crops = R.synth_video_frames(4, 192, 192, seed=3)
    crops[3] = np.random.default_rng(4).integers(0, 256, (192, 192, 3), dtype=np.uint8)
    with torch.no_grad():
        out["net_out"] = net(R.prep(crops)).numpy()
    out["net_crops"] = crops

    tmp = tempfile.mkdtemp(prefix="pfld_golden_")
    os.makedirs(os.path.join(tmp, "avatars", "ultralight", "face_detect_utils"))
    os.makedirs(os.path.join(tmp, "models"))
    mean_src = os.path.join(ref_root, "avatars", "ultralight", "face_detect_utils", "mean_face.txt")
    shutil.copy(mean_src, os.path.join(tmp, "avatars", "ultralight", "face_detect_utils", "mean_face.txt"))
    shutil.copy(mean_src, os.path.join(ROOT, "tests", "golden", "pfld_mean_face.txt"))
    torch.save({"pfld_backbone": sd}, os.path.join(tmp, "models", "checkpoint_epoch_335.pth.tar"))
    unet = os.path.join(tmp, "ul.pth")
    torch.save({"w": torch.zeros(3)}, unet)
    vid = os.path.join(tmp, "clip.avi")
    s3fd_ref.write_video(vid, R.synth_video_frames(GA_N, GA_H, GA_W, seed=7))

    torch.nn.Module.cuda = lambda self, *a, **k: self
    torch.Tensor.cuda = lambda self, *a, **k: self
    get_landmark.SCRFD = lambda *a, **k: R.ReplayDetector(R.face_records(GA_BOXES))
    seen = []
    detect = get_landmark.Landmark.detect

    def recording_detect(self, img_path):
        r = detect(self, img_path)
        img = __import__("cv2").imread(img_path)
        cropped, _ = R.face_det(img, R.ReplayDetector(R.face_records([GA_BOXES[len(seen)]])))
        seen.append((r, cropped.shape[1], cropped.shape[0]))
        return r
    get_landmark.Landmark.detect = recording_detect

    cwd = os.getcwd()
    os.chdir(tmp)
    argv = sys.argv
    sys.argv = ["genavatar.py", "--video_path", vid, "--checkpoint", unet, "--avatar_id", "ga"]
    try:
        g = runpy.run_path(os.path.join(ref_root, "avatars", "ultralight", "genavatar.py"), run_name="__main__")
    finally:
        sys.argv = argv
        os.chdir(cwd)
    av = os.path.join(tmp, "data", "avatars", "ga")
    crc = lambda d: np.array([zlib.crc32(open(os.path.join(av, d, f), "rb").read()) for f in sorted(os.listdir(os.path.join(av, d)))],  # noqa: E731
                             np.uint32)
    out["ga_video"] = np.frombuffer(open(vid, "rb").read(), np.uint8)
    out["ga_boxes"] = np.array(GA_BOXES, np.float32)
    out["ga_lms"] = np.stack([s[0][0] for s in seen])
    out["ga_x1y1"] = np.array([(int(s[0][1]), int(s[0][2])) for s in seen], np.int64)
    out["ga_crop_wh"] = np.array([(s[1], s[2]) for s in seen], np.int64)
    out["ga_coords_pkl"] = np.frombuffer(open(os.path.join(av, "coords.pkl"), "rb").read(), np.uint8)
    out["ga_face_crc"] = crc("face_imgs")
    out["ga_full_crc"] = crc("full_imgs")
    out["ga_args"] = np.array([f"{a.dest}|{a.default}|{getattr(a.type, '__name__', None)}" for a in g["parser"]._actions if a.dest != "help"])
    with open(os.path.join(av, "coords.pkl"), "rb") as fh:
        print("coords", pickle.load(fh))
    print("x1y1", out["ga_x1y1"].tolist(), "crop wh", out["ga_crop_wh"].tolist(), "args", out["ga_args"].tolist())
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "pfld_golden.npz"), **out)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "/path/to/LiveTalking")
