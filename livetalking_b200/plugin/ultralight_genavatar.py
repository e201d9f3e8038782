"""UltraLight avatar generation with the landmark network on the engine (avatars/ultralight/genavatar.py; same command line):

    python -m livetalking_b200.plugin.ultralight_genavatar --video_path clip.mp4 --img_size 168 --checkpoint ul.pth --avatar_id ul1

Same on-disk result under ``./data/avatars/<avatar_id>``: ``full_imgs/%08d.png`` (the decoded frames; this script, unlike the wav2lip
one, draws no watermark), ``face_imgs/%08d.png`` (img_size mouth crops), ``coords.pkl`` ((xmin, ymin, xmin + w, ymin + h) with the
sliced crop's w / h) and ``ultralight.pth`` (a copy of --checkpoint), plus ``avatar.ltbav`` (livetalking_b200/avatar_pack.py), which
the UltraLight plugin prefers when it loads the avatar.

What runs where.  PFLD_GhostOne (Landmark.detect's network, + mean_face, the crop scaling and the int32 truncation) runs on the
device as one graph per batch (livetalking_b200/pfld.py).  Face detection is the reference's own SCRFD class (cv2.dnn on the CPU,
face_detect_utils/detect_face.py, over ./models/scrfd_2.5g_kps.onnx): its network exists only inside that ONNX file.  Decoding,
face_det's crop and zero border, cv2.resize, the mouth box and the PNG writes are the reference's OpenCV / numpy operations, and
SCRFD + crops of batch k + 1 run on the host while the device computes the landmarks of batch k.

Where the reference would crash (no face in a frame: cropped_imgs[0]; an empty mouth slice: cv2.resize) this raises a ValueError
naming the frame.  PFLD weights come from ./models/checkpoint_epoch_335.pth.tar and mean_face.txt from
./avatars/ultralight/face_detect_utils/ under the working directory (a LiveTalking checkout); a missing file raises
FileNotFoundError, nothing is downloaded.  ``run_app.install_aliases`` registers this module as ``avatars.ultralight.genavatar``."""
from __future__ import annotations

import argparse
import glob
import logging
import os
import pickle
import shutil
import threading
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from .. import avatar_pack

logger = logging.getLogger(__name__)

PFLD_REL = os.path.join("models", "checkpoint_epoch_335.pth.tar")
MEAN_FACE_REL = os.path.join("avatars", "ultralight", "face_detect_utils", "mean_face.txt")
SCRFD_REL = os.path.join("models", "scrfd_2.5g_kps.onnx")
BATCH = 16
_NETS = {}
_NETS_LOCK = threading.Lock()


def osmakedirs(path_list):
    for path in path_list:
        os.makedirs(path) if not os.path.exists(path) else None


def parser() -> argparse.ArgumentParser:
    """genavatar.py's options, with the same names, types and defaults."""
    p = argparse.ArgumentParser(description='Create an UltraLight avatar (face landmarks on the GPU)',
                                formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    p.add_argument('--video_path', default='', type=str)
    p.add_argument('--img_size', default=168, type=int)
    p.add_argument('--checkpoint', type=str, default="")
    p.add_argument('--avatar_id', default='ultralight_avatar1', type=str)
    return p


def video2imgs(vid_path, save_path, timings=None):
    """genavatar.video2imgs (cv2.VideoCapture -> PNG per frame); additionally returns the frames and the file names."""
    import cv2
    cap = cv2.VideoCapture(vid_path)
    frames, names = [], []
    t_dec = t_png = 0.0
    while True:
        t0 = time.perf_counter()
        ret, frame = cap.read()
        t1 = time.perf_counter()
        t_dec += t1 - t0
        if not ret:
            break
        name = f"{save_path}/{len(frames):08d}.png"
        cv2.imwrite(name, frame)
        t_png += time.perf_counter() - t1
        frames.append(frame)
        names.append(name)
    cap.release()
    if timings is not None:
        timings["decode"] = t_dec
        timings["full_png"] = t_png
    return frames, names


def face_det(img, detector, idx=None):
    """get_landmark.face_det for its first NMS index -> (cropped image with the zero border, x1, y1).  x1 / y1 are shifted by the
    border and may be negative.  Raises ValueError when the detector finds no face (the reference fails on cropped_imgs[0])."""
    import cv2
    bboxes, indices, kps = detector.detect(img)
    for i in indices:
        x1, y1, x2, y2 = int(bboxes[i, 0]), int(bboxes[i, 1]), int(bboxes[i, 0] + bboxes[i, 2]), int(bboxes[i, 1] + bboxes[i, 3])
        w = x2 - x1
        h = y2 - y1
        cx = (x2 + x1) // 2
        cy = (y2 + y1) // 2
        boxsize = int(np.max(np.asarray([w, h])) * 1.05)
        size = boxsize
        xy = np.asarray((cx - size // 2, cy - size // 2), dtype=np.int32)
        x1, y1 = xy
        x2, y2 = xy + size
        height, width, _ = img.shape
        dx = max(0, -x1)
        dy = max(0, -y1)
        x1 = max(0, x1)
        y1 = max(0, y1)
        edx = max(0, x2 - width)
        edy = max(0, y2 - height)
        x2 = min(width, x2)
        y2 = min(height, y2)
        cropped = img[y1:y2, x1:x2]
        if dx > 0 or dy > 0 or edx > 0 or edy > 0:
            cropped = cv2.copyMakeBorder(cropped, dy, edy, dx, edx, cv2.BORDER_CONSTANT, 0)
            y1 = y1 - dy
            x1 = x1 - dx
        return cropped, x1, y1
    raise ValueError(f"frame {idx}: no face detected (the reference fails on this frame as well)")


def mouth_crop(img, lms, x1, y1, target_size, idx=None):
    """The genavatar loop body after Landmark.detect -> (face crop of target_size, (xmin, ymin, xmin + w, ymin + h)).
    img[ymin:ymax, xmin:xmax] keeps numpy's slicing semantics (a negative start counts from the end, as in the reference), and
    cv2.resize's third positional argument is dst, so the interpolation is the default INTER_LINEAR."""
    import cv2
    xmin = lms[1][0] + x1
    ymin = lms[52][1] + y1
    xmax = lms[31][0] + x1
    width = xmax - xmin
    ymax = ymin + width
    crop_img = img[ymin:ymax, xmin:xmax]
    h, w = crop_img.shape[:2]
    if h == 0 or w == 0:
        raise ValueError(f"frame {idx}: the mouth box img[{ymin}:{ymax}, {xmin}:{xmax}] is empty (the reference fails in cv2.resize)")
    crop_img = cv2.resize(crop_img, (target_size, target_size), cv2.INTER_AREA)
    return crop_img, (xmin, ymin, xmin + w, ymin + h)


def _need(path: str, what: str) -> str:
    if not os.path.isfile(path):
        raise FileNotFoundError(f"{what} not found at {path} (it is never downloaded)")
    return path


def load_net(root=None):
    """PFLDNet over <root>/models/checkpoint_epoch_335.pth.tar and mean_face.txt (root: the working directory), loaded once."""
    root = os.path.abspath(root or os.getcwd())
    ckpt = _need(os.path.join(root, PFLD_REL), "PFLD checkpoint")
    mean = _need(os.path.join(root, MEAN_FACE_REL), "mean_face.txt")
    with _NETS_LOCK:
        if root not in _NETS:
            import torch
            from ..pfld import PFLDNet
            with open(mean, "r") as f:
                mean_face = np.asarray(f.read().split(' '), dtype=np.float32)
            _NETS[root] = PFLDNet.from_state_dict(torch.load(ckpt, map_location="cpu", weights_only=True), mean_face)
        return _NETS[root]


def _scrfd():
    _need(os.path.join(os.getcwd(), SCRFD_REL), "SCRFD model")
    from avatars.ultralight.face_detect_utils.detect_face import SCRFD     # the reference's own detector (LiveTalking checkout)
    return SCRFD('./' + SCRFD_REL.replace(os.sep, '/'), confThreshold=0.1, nmsThreshold=0.5)


def _engine_landmarker(N):
    from ..pfld import PFLDLandmarker
    return PFLDLandmarker(load_net(), N)


def generate_avatar(video_path, avatar_id, save_path='./data/avatars', img_size=168, checkpoint='', detector=None, progress_callback=None,
                    timings=None, make_landmarker=None):
    """genavatar.py's __main__ as a function.  detector: object with detect(img) -> (bboxes, indices, kpss) (default: the reference's
    SCRFD); make_landmarker(N) -> object with run(crops, crop_wh) and close() (default: PFLDLandmarker over the checkpoint).
    timings: optional dict filled with the seconds spent in decode, full_png, detect (SCRFD + crops, host), landmarks (waiting for
    the device), face_png (mouth crops + writes) and pack."""
    import cv2
    timings = {} if timings is None else timings
    avatar_path = os.path.join(save_path, avatar_id)
    full_imgs_path = f"{avatar_path}/full_imgs"
    face_imgs_path = f"{avatar_path}/face_imgs"
    coords_path = f"{avatar_path}/coords.pkl"
    pth_path = f"{avatar_path}/ultralight.pth"
    if make_landmarker is None:
        load_net()                      # fail before any work when the weights are missing
        make_landmarker = _engine_landmarker
    if detector is None:
        detector = _scrfd()
    osmakedirs([avatar_path, full_imgs_path, face_imgs_path])
    if progress_callback: progress_callback(5)

    frames, names = video2imgs(video_path, full_imgs_path, timings=timings)
    input_img_list = sorted(glob.glob(os.path.join(full_imgs_path, '*.[jpJP][pnPN]*[gG]')))
    if [os.path.normpath(p) for p in input_img_list] != [os.path.normpath(p) for p in names]:
        frames = [cv2.imread(p) for p in input_img_list]        # the folder held other images: read it as the reference does
    if progress_callback: progress_callback(20)

    def host_batch(lo, hi):
        crops, wh, xy = [], [], []
        for i in range(lo, hi):
            cropped, x1, y1 = face_det(frames[i], detector, i)
            h, w = cropped.shape[:2]
            crops.append(cv2.resize(cropped, (192, 192)))
            wh.append((w, h))
            xy.append((x1, y1))
        return np.stack(crops), np.array(wh, np.int32), xy

    t_det = t_lm = 0.0
    batch = BATCH
    n = len(frames)
    while True:
        lms, xys = [], []
        lm = None
        try:
            lm = make_landmarker(min(batch, max(n, 1)))
            with ThreadPoolExecutor(1) as pool:
                pending = None
                for lo in range(0, n + batch, batch):
                    t0 = time.perf_counter()
                    nxt = host_batch(lo, min(n, lo + batch)) if lo < n else None
                    t_det += time.perf_counter() - t0
                    if pending is not None:             # the device ran batch k while the host detected batch k + 1
                        t0 = time.perf_counter()
                        lms.append(pending.result()[1])
                        t_lm += time.perf_counter() - t0
                        if progress_callback: progress_callback(20 + int(min(lo, n) / max(n, 1) * 60))
                    pending = pool.submit(lm.run, nxt[0], nxt[1]) if nxt is not None else None
                    if nxt is not None:
                        xys += nxt[2]
        except RuntimeError:
            if batch == 1:
                raise
            batch //= 2
            logger.warning("recovering from a device allocation failure; new batch size: %d", batch)
            continue
        finally:
            if lm is not None:
                lm.close()
        break
    timings["detect"] = t_det
    timings["landmarks"] = t_lm
    lms = np.concatenate(lms) if lms else np.zeros((0, 110, 2), np.int32)

    t0 = time.perf_counter()
    coord_list = []
    faces = []
    for idx in range(n):
        x1, y1 = xys[idx]
        crop_img, box = mouth_crop(frames[idx], lms[idx], x1, y1, img_size, idx)
        cv2.imwrite(f"{face_imgs_path}/{idx:08d}.png", crop_img)
        faces.append(crop_img)
        coord_list.append(box)
    timings["face_png"] = time.perf_counter() - t0
    if progress_callback: progress_callback(90)

    with open(coords_path, 'wb') as f:
        pickle.dump(coord_list, f)
    if checkpoint:
        shutil.copyfile(checkpoint, pth_path)
    t0 = time.perf_counter()
    avatar_pack.pack_wav2lip_lists(frames, faces, coord_list, os.path.join(avatar_path, "avatar.ltbav"))
    timings["pack"] = time.perf_counter() - t0
    if progress_callback: progress_callback(100)
    logger.info("avatar %s written to %s (%d faces)", avatar_id, avatar_path, n)


if __name__ == "__main__":
    args = parser().parse_args()
    print(args)
    generate_avatar(args.video_path, args.avatar_id, save_path="./data/avatars", img_size=args.img_size, checkpoint=args.checkpoint)
