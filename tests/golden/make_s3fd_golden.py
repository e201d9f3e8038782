"""Writes tests/golden/s3fd_golden.npz by running the unmodified LiveTalking S3FD code and generate_avatar on the CPU:

    python tests/golden/make_s3fd_golden.py /path/to/LiveTalking

Weights: oracle.s3fd_ref.synth_state_dict(0), saved to a temporary s3fd.pth that SFDDetector is pointed at (its default
path_to_detector); the model-zoo download functions are replaced by ones that raise, so nothing is fetched.

Contents, per detection case ("even": 6 frames of 128 x 224, "odd": 3 frames of 239 x 427):
  <case>_frames         u8 BGR inputs
  <case>_head<k>        the 12 outputs of s3fd.forward (fp32)
  <case>_found / _box   get_detections_for_batch: found flag, (x1, y1, x2, y2) (zeros where None)
generate_avatar on a 10-frame MJPG video at batch 4:
  ga_video (bytes of the .avi), ga_det_found / ga_det_box (per-frame detections), ga_coords (coords.pkl, (y1, y2, x1, x2)),
  ga_face_crc / ga_full_crc (zlib.crc32 of the PNG files), ga_progress (progress_callback values)."""
import os
import pickle
import sys
import tempfile
import zlib

import numpy as np
import torch
import torch.hub
import torch.utils.model_zoo

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import s3fd_ref as R  # noqa: E402

CASES = {"even": ([0, 10, 35, 50, 5, 40], 128, 224), "odd": ([35, 0, 10], 239, 427)}
GA_AMPS = [0, 40, 45, 40, 0, 10, 50, 40, 35, 0]
GA_H, GA_W, GA_BATCH = 120, 200, 4


def _no_download(*a, **k):
    raise RuntimeError("golden generation must not download anything")


def main(ref_root):
    sys.path.insert(0, ref_root)
    torch.utils.model_zoo.load_url = _no_download
    torch.hub.load_state_dict_from_url = _no_download
    from avatars.wav2lip.face_detection.detection.sfd import sfd_detector
    from avatars.wav2lip.face_detection.detection.sfd.net_s3fd import s3fd
    sfd_detector.load_url = _no_download
    from avatars.wav2lip import face_detection, genavatar

    tmp = tempfile.mkdtemp(prefix="s3fd_golden_")
    sd = R.synth_state_dict(0)
    wpath = os.path.join(tmp, "s3fd.pth")
    torch.save(sd, wpath)
    sfd_detector.SFDDetector.__init__.__defaults__ = (wpath, False)

    out = {}
    net = s3fd()
    net.load_state_dict(sd)
    net.eval()
    fa = face_detection.FaceAlignment(face_detection.LandmarksType._2D, flip_input=False, device="cpu")
    for case, (amps, H, W) in CASES.items():
        frames = R.synth_frames(amps, H, W, seed=len(case))
        x = torch.from_numpy((frames[..., ::-1] - np.array([104, 117, 123])).transpose(0, 3, 1, 2).copy()).float()
        with torch.no_grad():
            ol = net(x)
        dets = fa.get_detections_for_batch(frames)
        out[f"{case}_frames"] = frames
        for k, o in enumerate(ol):
            out[f"{case}_head{k}"] = o.numpy()
        out[f"{case}_found"] = np.array([d is not None for d in dets])
        out[f"{case}_box"] = np.array([d if d is not None else (0, 0, 0, 0) for d in dets], np.int64)
        print(case, dets)

    # generate_avatar end to end
    frames = R.synth_frames(GA_AMPS, GA_H, GA_W, seed=7)
    vid = os.path.join(tmp, "clip.avi")
    R.write_video(vid, frames)
    import cv2
    cap = cv2.VideoCapture(vid)
    decoded = []
    while True:
        ok, f = cap.read()
        if not ok:
            break
        cv2.putText(f, "LiveTalking", (10, 20), cv2.FONT_HERSHEY_SIMPLEX, 0.3, (128, 128, 128), 1)
        decoded.append(f)
    dets = []
    for i in range(0, len(decoded), GA_BATCH):
        dets += fa.get_detections_for_batch(np.array(decoded[i:i + GA_BATCH]))
    progress = []
    save = os.path.join(tmp, "avatars")
    genavatar.generate_avatar(vid, "ga", save_path=save, face_det_batch_size=GA_BATCH, progress_callback=progress.append)
    av = os.path.join(save, "ga")
    with open(os.path.join(av, "coords.pkl"), "rb") as fh:
        coords = pickle.load(fh)
    crc = lambda d: np.array([zlib.crc32(open(os.path.join(av, d, f), "rb").read()) for f in sorted(os.listdir(os.path.join(av, d)))],  # noqa: E731
                             np.uint32)
    out["ga_video"] = np.frombuffer(open(vid, "rb").read(), np.uint8)
    out["ga_det_found"] = np.array([d is not None for d in dets])
    out["ga_det_box"] = np.array([d if d is not None else (0, 0, 0, 0) for d in dets], np.int64)
    out["ga_coords"] = np.array(coords, np.int64)
    out["ga_face_crc"] = crc("face_imgs")
    out["ga_full_crc"] = crc("full_imgs")
    out["ga_progress"] = np.array(progress, np.int64)
    print("generate_avatar", dets, coords, progress)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "s3fd_golden.npz"), **out)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "/path/to/LiveTalking")
