"""wav2lip avatar generation with the face detector on the engine (avatars/wav2lip/genavatar.py, the function the server's avatar
task route calls: server/avatar_routes.py -> server/task_manager.py -> generate_avatar).

Same signature, same on-disk result: ``full_imgs/%08d.png`` (the watermarked frames), ``face_imgs/%08d.png`` (img_size crops) and
``coords.pkl`` ((y1, y2, x1, x2) per frame), plus ``avatar.ltbav`` (livetalking_b200/avatar_pack.py), which the wav2lip plugin
prefers when it loads the avatar.  Decoding, the watermark, smoothing, crop + resize and the PNG writes are the reference's own
OpenCV / numpy operations; only S3FD runs on the device (livetalking_b200/s3fd.py) instead of the reference's fp32 eager model.
The frames detection sees are the decoded, watermarked frames kept in memory: PNG is lossless, so they are the arrays the
reference reads back from full_imgs/.

Weights come from the reference's location (``avatars/wav2lip/face_detection/detection/sfd/s3fd.pth`` under the working directory)
or an explicit ``weights_path``.  A missing file raises FileNotFoundError: nothing is ever downloaded.  ``run_app.install_aliases``
registers this module as ``avatars.wav2lip.genavatar``."""
from __future__ import annotations

import glob
import logging
import os
import pickle
import threading
import time

import numpy as np

from .. import avatar_pack

logger = logging.getLogger(__name__)

WEIGHTS_REL = os.path.join("avatars", "wav2lip", "face_detection", "detection", "sfd", "s3fd.pth")
_NETS = {}
_NETS_LOCK = threading.Lock()


def osmakedirs(path_list):
    for path in path_list:
        os.makedirs(path) if not os.path.exists(path) else None


def video2imgs(vid_path, save_path, ext=".png", cut_frame=10000000, timings=None):
    """genavatar.video2imgs; additionally returns the written frames and the file names."""
    import cv2
    cap = cv2.VideoCapture(vid_path)
    frames, names = [], []
    t_dec = t_png = 0.0
    count = 0
    while True:
        if count > cut_frame:
            break
        t0 = time.perf_counter()
        ret, frame = cap.read()
        if ret:
            cv2.putText(frame, "LiveTalking", (10, 20), cv2.FONT_HERSHEY_SIMPLEX, 0.3, (128, 128, 128), 1)
            t1 = time.perf_counter()
            name = f"{save_path}/{count:08d}.png"
            cv2.imwrite(name, frame)
            t_dec += t1 - t0
            t_png += time.perf_counter() - t1
            frames.append(frame)
            names.append(name)
            count += 1
        else:
            t_dec += time.perf_counter() - t0
            break
    cap.release()
    if timings is not None:
        timings["decode"] = t_dec
        timings["full_png"] = t_png
    return frames, names


def get_smoothened_boxes(boxes, T):
    """genavatar.get_smoothened_boxes: in place on an int64 array (each mean truncated; the tail windows read smoothed boxes)."""
    for i in range(len(boxes)):
        if i + T > len(boxes):
            window = boxes[len(boxes) - T:]
        else:
            window = boxes[i: i + T]
        boxes[i] = np.mean(window, axis=0)
    return boxes


def weights_file(weights_path=None) -> str:
    path = weights_path or os.path.join(os.getcwd(), WEIGHTS_REL)
    if not os.path.isfile(path):
        raise FileNotFoundError(f"S3FD weights not found at {path}: place the reference's s3fd.pth there or pass weights_path "
                                "(they are never downloaded)")
    return path


def load_net(weights_path=None):
    """S3FDNet for the weights file, loaded once per path."""
    path = os.path.abspath(weights_file(weights_path))
    with _NETS_LOCK:
        if path not in _NETS:
            import torch
            from ..s3fd import S3FDNet
            _NETS[path] = S3FDNet.from_state_dict(torch.load(path, map_location="cpu", weights_only=True))
        return _NETS[path]


def _engine_detector(weights_path):
    def make(N, H, W):
        from ..s3fd import S3FDDetector
        return S3FDDetector(load_net(weights_path), N, H, W)
    return make


def generate_avatar(video_path, avatar_id, save_path='./data/avatars', img_size=96, pads=[0, 10, 0, 0], nosmooth=False,
                    face_det_batch_size=16, progress_callback=None, weights_path=None, make_detector=None, timings=None):
    """genavatar.generate_avatar on the engine.  make_detector(N, H, W) -> object with detect(frames) and close(): the detector
    factory (default: S3FDDetector over the weights file).  timings: optional dict the call fills with the seconds it spent in
    decode (+ watermark), full_png, detect, face_png (crops + writes) and pack."""
    import cv2
    timings = {} if timings is None else timings
    avatar_path = os.path.join(save_path, avatar_id)
    full_imgs_path = os.path.join(avatar_path, "full_imgs")
    face_imgs_path = os.path.join(avatar_path, "face_imgs")
    coords_path = os.path.join(avatar_path, "coords.pkl")
    if make_detector is None:
        weights_file(weights_path)          # fail before any work when the weights are missing
        make_detector = _engine_detector(weights_path)

    osmakedirs([avatar_path, full_imgs_path, face_imgs_path])
    if progress_callback: progress_callback(5)

    logger.info("processing video %s", video_path)
    frames, names = video2imgs(video_path, full_imgs_path, ext='png', timings=timings)
    if progress_callback: progress_callback(20)

    input_img_list = sorted(glob.glob(os.path.join(full_imgs_path, '*.[jpJP][pnPN]*[gG]')))
    if [os.path.normpath(p) for p in input_img_list] != [os.path.normpath(p) for p in names]:
        frames = [cv2.imread(p) for p in input_img_list]        # the folder held other images: read it as the reference does
    if progress_callback: progress_callback(40)

    logger.info("detecting faces")
    t0 = time.perf_counter()
    batch_size = face_det_batch_size
    predictions = []
    while frames:
        predictions = []
        det = None
        try:
            H, W = frames[0].shape[:2]
            det = make_detector(min(batch_size, len(frames)), H, W)
            for i in range(0, len(frames), batch_size):
                predictions.extend(det.detect(np.array(frames[i:i + batch_size])))
                if progress_callback:
                    progress = 40 + int((i + batch_size) / len(frames) * 40)
                    progress_callback(min(progress, 80))
        except RuntimeError:
            if batch_size == 1:
                raise RuntimeError('Image too big to run face detection on GPU.')
            batch_size //= 2
            logger.warning("recovering from a device allocation failure; new batch size: %d", batch_size)
            continue
        finally:
            if det is not None:
                det.close()
        break
    timings["detect"] = time.perf_counter() - t0

    results = []
    pady1, pady2, padx1, padx2 = pads
    for rect, image in zip(predictions, frames):
        if rect is None:
            rect = [0, 0, image.shape[1], image.shape[0]]
        y1 = max(0, rect[1] - pady1)
        y2 = min(image.shape[0], rect[3] + pady2)
        x1 = max(0, rect[0] - padx1)
        x2 = min(image.shape[1], rect[2] + padx2)
        results.append([x1, y1, x2, y2])

    boxes = np.array(results)
    if not nosmooth:
        boxes = get_smoothened_boxes(boxes, T=5)
    if progress_callback: progress_callback(85)

    t0 = time.perf_counter()
    coord_list, faces = [], []
    for idx, (rect, frame) in enumerate(zip(boxes, frames)):
        face_frame = frame[int(rect[1]):int(rect[3]), int(rect[0]):int(rect[2])]
        resized_crop_frame = cv2.resize(face_frame, (img_size, img_size))
        cv2.imwrite(f"{face_imgs_path}/{idx:08d}.png", resized_crop_frame)
        faces.append(resized_crop_frame)
        coord_list.append((int(rect[1]), int(rect[3]), int(rect[0]), int(rect[2])))
        if progress_callback:
            progress = 85 + int((idx + 1) / len(boxes) * 15)
            progress_callback(progress)
    timings["face_png"] = time.perf_counter() - t0

    with open(coords_path, 'wb') as f:
        pickle.dump(coord_list, f)
    t0 = time.perf_counter()
    avatar_pack.pack_wav2lip_lists(frames, faces, coord_list, os.path.join(avatar_path, "avatar.ltbav"))
    timings["pack"] = time.perf_counter() - t0
    if progress_callback: progress_callback(100)
    logger.info("avatar %s written to %s", avatar_id, avatar_path)


if __name__ == '__main__':
    import argparse
    parser = argparse.ArgumentParser(description='Create a wav2lip avatar (face detection on the GPU)')
    parser.add_argument('--img_size', default=96, type=int)
    parser.add_argument('--avatar_id', default='wav2lip_avatar1', type=str)
    parser.add_argument('--save_path', default='data/avatars', type=str)
    parser.add_argument('--video_path', default='', type=str)
    parser.add_argument('--nosmooth', default=False, action='store_true',
                        help='Prevent smoothing face detections over a short temporal window')
    parser.add_argument('--pads', nargs='+', type=int, default=[0, 10, 0, 0],
                        help='Padding (top, bottom, left, right). Please adjust to include chin at least')
    parser.add_argument('--face_det_batch_size', type=int, help='Batch size for face detection', default=16)
    parser.add_argument('--weights_path', default=None, type=str, help='s3fd.pth (default: the reference location under the cwd)')
    args = parser.parse_args()
    generate_avatar(video_path=args.video_path, avatar_id=args.avatar_id, save_path=args.save_path, img_size=args.img_size,
                    pads=args.pads, nosmooth=args.nosmooth, face_det_batch_size=args.face_det_batch_size, weights_path=args.weights_path)
