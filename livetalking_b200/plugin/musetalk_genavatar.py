"""MuseTalk avatar generation with the face parser on the engine (avatars/musetalk/genavatar.py, the function the server's avatar task
route calls).

Same signature, same command line, same on-disk result: ``full_imgs/%08d.png`` (the watermarked frames), ``mask/%08d.png`` (the
blurred blend masks), ``coords.pkl`` (face boxes), ``mask_coords.pkl`` (crop boxes), ``latents.pt`` (a list of (1, 8, h, w) fp16 CPU
tensors) and ``avator_info.json``, plus ``avatar.ltbav`` (livetalking_b200/avatar_pack.py), which the MuseTalk plugin prefers.

* Landmarks: ``face_recognition.face_landmarks`` (dlib, CPU) stays the reference's own call: dlib's models are not part of the
  reference tree, so they cannot be restated here.  It is imported when first needed.
* Face boxes: S3FD on the engine (livetalking_b200/s3fd.py) with MuseTalk's weights file, then get_landmark_and_bbox's rule
  restated (bbox_shift, the half-face upper bound, the detector-box fallback and the printed adjust range).
* Latents: the LANCZOS4 256 x 256 crops go through ``musetalk.encode_avatar_latents``, which takes ``latent_dist.mode()``.  The
  reference draws an unseeded ``latent_dist.sample()``, whose noise cannot be reproduced.
* Masks: BiSeNet on the engine (plugin/musetalk_face_parsing.py); PIL crops and resizes of batch k + 1 run on the host while the
  device parses batch k.
* A frame without a face raises ValueError naming it (the reference writes a placeholder box and then fails on a zero-size crop).
  Crop boxes that leave the frame are written as the reference writes them, with a warning listing those frames: the engine's
  MuseTalkAvatar refuses such avatars.

``run_app.install_aliases`` registers this module as ``avatars.musetalk.genavatar``."""
from __future__ import annotations

import glob
import json
import logging
import os
import pickle
import shutil
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from .. import avatar_pack
from . import musetalk_face_parsing as mfp
from .wav2lip_genavatar import video2imgs

logger = logging.getLogger(__name__)

S3FD_REL = os.path.join("avatars", "musetalk", "utils", "face_detection", "detection", "sfd", "s3fd.pth")
coord_placeholder = (0.0, 0.0, 0.0, 0.0)


def is_video_file(file_path):
    video_exts = ['.mp4', '.mkv', '.flv', '.avi', '.mov']
    return os.path.splitext(file_path)[1].lower() in video_exts


def create_dir(dir_path):
    if not os.path.exists(dir_path):
        os.makedirs(dir_path)


def face_landmarks(img_rgb):
    """face_recognition.face_landmarks, imported on first use."""
    try:
        import face_recognition
    except ImportError as e:
        raise ImportError("MuseTalk avatar creation needs the `face_recognition` package (dlib landmarks), as the reference does") from e
    return face_recognition.face_landmarks(img_rgb)


def _engine_detect(batch_size):
    from ..s3fd import S3FDDetector
    from .wav2lip_genavatar import load_net
    path = os.path.join(os.getcwd(), S3FD_REL)
    if not os.path.isfile(path):
        raise FileNotFoundError(f"S3FD weights not found at {path}: place the reference's s3fd.pth there (they are never downloaded)")

    def detect_same_size(frames):
        out, bs, i = [], batch_size, 0
        det = None
        try:
            while i < len(frames):
                n = min(bs, len(frames) - i)
                if det is None or det.N < n:
                    if det is not None:
                        det.close()
                        det = None
                    try:
                        det = S3FDDetector(load_net(path), n, *frames[0].shape[:2])
                    except RuntimeError:
                        if bs == 1:
                            raise
                        bs //= 2
                        logger.warning("recovering from a device allocation failure; detection batch size: %d", bs)
                        continue
                out.extend(det.detect(np.array(frames[i:i + n])))
                i += n
        finally:
            if det is not None:
                det.close()
        return out

    def detect(frames):
        """One detector per frame size: a folder of PNGs may mix sizes, which the reference handles frame by frame."""
        out = [None] * len(frames)
        for shape in dict.fromkeys(np.asarray(f).shape for f in frames):
            idx = [i for i, f in enumerate(frames) if np.asarray(f).shape == shape]
            for i, box in zip(idx, detect_same_size([frames[i] for i in idx])):
                out[i] = box
        return out
    return detect


def get_landmark_and_bbox(frames, upperbondrange=0, detect=None, landmarks=face_landmarks, names=None):
    """preprocessing.get_landmark_and_bbox over decoded frames: detect(frames) -> per frame (x1, y1, x2, y2) or None.  A frame
    without a face raises ValueError naming it (names: the frames' files), before the adjust range is printed: the reference writes
    a placeholder box for it and fails later on a zero-size crop, or divides by zero here when no frame has a face."""
    import cv2
    coords_list = []
    if upperbondrange != 0:
        print('get key_landmark and face bounding boxes with the bbox_shift:', upperbondrange)
    else:
        print('get key_landmark and face bounding boxes with the default value')
    average_range_minus = []
    average_range_plus = []
    boxes = detect(frames)
    for frame, f in zip(frames, boxes):
        img_rgb = cv2.cvtColor(np.asarray(frame), cv2.COLOR_BGR2RGB)
        landmarks_list = landmarks(img_rgb)
        if landmarks_list:
            lm = landmarks_list[0]
            face_land_mark = np.array(lm['chin'] + lm['left_eyebrow'] + lm['right_eyebrow'] + lm['nose_bridge'] + lm['nose_tip'] +
                                      lm['left_eye'] + lm['right_eye'] + lm['top_lip'] + lm['bottom_lip']).astype(np.int32)
        else:
            face_land_mark = np.zeros((68, 2), dtype=np.int32)
        if f is None:
            coords_list += [coord_placeholder]
            continue
        half_face_coord = face_land_mark[29]
        range_minus = (face_land_mark[30] - face_land_mark[29])[1]
        range_plus = (face_land_mark[29] - face_land_mark[28])[1]
        average_range_minus.append(range_minus)
        average_range_plus.append(range_plus)
        if upperbondrange != 0:
            half_face_coord[1] = upperbondrange + half_face_coord[1]
        half_face_dist = np.max(face_land_mark[:, 1]) - half_face_coord[1]
        upper_bond = max(0, half_face_coord[1] - half_face_dist)
        f_landmark = (np.min(face_land_mark[:, 0]), int(upper_bond), np.max(face_land_mark[:, 0]), np.max(face_land_mark[:, 1]))
        x1, y1, x2, y2 = f_landmark
        if y2 - y1 <= 0 or x2 - x1 <= 0 or x1 < 0:
            coords_list += [f]
            print("error bbox:", f)
        else:
            coords_list += [f_landmark]
    missing = [i for i, b in enumerate(coords_list) if b == coord_placeholder]
    if missing:
        where = f" ({names[missing[0]]})" if names is not None else ""
        raise ValueError(f"no face found in frame {missing[0]}{where}" + (f" and {len(missing) - 1} more" if len(missing) > 1 else "")
                         + ": every frame of a MuseTalk avatar needs one")
    print("********************************************bbox_shift parameter adjustment**********************************************************")
    print(f"Total frame:「{len(frames)}」 Manually adjust range : [ -{int(sum(average_range_minus) / len(average_range_minus))}~{int(sum(average_range_plus) / len(average_range_plus))} ] , the current value: {upperbondrange}")
    print("*************************************************************************************************************************************")
    return coords_list


def _default_encoder():
    from ..musetalk import encode_avatar_latents
    from .musetalk_avatar import load_model
    model = load_model()
    return lambda crops: encode_avatar_latents(model.net, crops)


def generate_avatar(video_path, avatar_id, save_path='./data/avatars', bbox_shift=0, extra_margin=10, parsing_mode='jaw', version='v15',
                    progress_callback=None, *, detect=None, landmarks=face_landmarks, face_parsing=None, encode_latents=None,
                    batch_size=16, timings=None):
    """genavatar.generate_avatar on the engine.  Injectable steps (defaults: the engine and the reference's model files under the
    working directory): detect(frames) -> boxes or None per frame; landmarks(rgb) -> face_recognition.face_landmarks' result;
    face_parsing: a musetalk_face_parsing.FaceParsing; encode_latents(crops u8 [n, 256, 256, 3]) -> [n, 8, h, w].  timings: optional
    dict filled with the seconds spent in decode, full_png, detect, latents, masks (parsing + mask PNGs) and pack."""
    import cv2
    import torch
    timings = {} if timings is None else timings
    avatar_save_path = os.path.join(save_path, avatar_id)
    save_full_path = os.path.join(avatar_save_path, 'full_imgs')
    mask_out_path = os.path.join(avatar_save_path, 'mask')
    if detect is None:
        detect = _engine_detect(batch_size)             # fails before any work when the weights are missing
    if face_parsing is None:
        face_parsing = mfp.FaceParsing(left_cheek_width=90, right_cheek_width=90) if version == "v15" else mfp.FaceParsing()
    create_dir(avatar_save_path)
    create_dir(save_full_path)
    create_dir(mask_out_path)
    if progress_callback: progress_callback(5)

    with open(os.path.join(avatar_save_path, 'avator_info.json'), "w") as f:
        json.dump({"avatar_id": avatar_id, "video_path": video_path, "bbox_shift": bbox_shift}, f)

    frames, names = [], []
    if os.path.isfile(video_path):
        if is_video_file(video_path):
            frames, names = video2imgs(video_path, save_full_path, ext='png', timings=timings)
        else:
            shutil.copyfile(video_path, f"{save_full_path}/{os.path.basename(video_path)}")
    else:
        files = sorted(os.listdir(video_path))
        for filename in [file for file in files if file.split(".")[-1] == "png"]:
            shutil.copyfile(f"{video_path}/{filename}", f"{save_full_path}/{filename}")
    if progress_callback: progress_callback(20)

    input_img_list = sorted(glob.glob(os.path.join(save_full_path, '*.[jpJP][pnPN]*[gG]')))
    if [os.path.normpath(p) for p in input_img_list] != [os.path.normpath(p) for p in names]:
        frames = [cv2.imread(p) for p in input_img_list]        # the folder holds other images: read it as the reference does
    print("extracting landmarks...")
    t0 = time.perf_counter()
    coord_list = get_landmark_and_bbox(frames, bbox_shift, detect=detect, landmarks=landmarks, names=input_img_list)
    timings["detect"] = time.perf_counter() - t0
    if progress_callback: progress_callback(50)

    t0 = time.perf_counter()
    if encode_latents is None:
        encode_latents = _default_encoder()
    input_latent_list = []
    for start in range(0, len(frames), batch_size):
        crops = []
        for idx in range(start, min(start + batch_size, len(frames))):
            x1, y1, x2, y2 = coord_list[idx]
            if version == "v15":
                y2 = y2 + extra_margin
                y2 = min(y2, frames[idx].shape[0])
                coord_list[idx] = [x1, y1, x2, y2]
            crops.append(cv2.resize(frames[idx][y1:y2, x1:x2], (256, 256), interpolation=cv2.INTER_LANCZOS4))
        lat = np.asarray(encode_latents(np.stack(crops)))
        input_latent_list += [torch.from_numpy(np.ascontiguousarray(l[None], np.float16)) for l in lat]
        if progress_callback:
            for idx in range(start, min(start + batch_size, len(frames))):
                progress_callback(50 + int((idx + 1) / len(frames) * 25))
    timings["latents"] = time.perf_counter() - t0

    t0 = time.perf_counter()
    mode = parsing_mode if version == "v15" else "raw"
    written = {os.path.normpath(p) for p in names}
    mask_coords_list_cycle, mask_list_cycle = [], []
    batches = [range(s, min(s + batch_size, len(frames))) for s in range(0, len(frames), batch_size)]

    def crops_of(rng):
        return [mfp.crop_for_parsing(frames[i], list(coord_list[i])) for i in rng]

    with ThreadPoolExecutor(1) as pool:
        crops = crops_of(batches[0]) if batches else []
        for k, rng in enumerate(batches):
            segs = pool.submit(face_parsing.parse_many, [c[0] for c in crops], mode)
            nxt = crops_of(batches[k + 1]) if k + 1 < len(batches) else []
            for i, (face_large, crop_box), seg in zip(rng, crops, segs.result()):
                full = os.path.normpath(f"{save_full_path}/{str(i).zfill(8)}.png")
                if full not in written:
                    cv2.imwrite(full, frames[i])
                mask, crop_box = mfp.finish_material(face_large, seg, list(coord_list[i]), crop_box)
                cv2.imwrite(f"{mask_out_path}/{str(i).zfill(8)}.png", mask)
                mask_coords_list_cycle += [crop_box]
                mask_list_cycle.append(mask)
                if progress_callback:
                    progress_callback(75 + int((i + 1) / len(frames) * 20))
            crops = nxt
    timings["masks"] = time.perf_counter() - t0
    H, W = frames[0].shape[:2]
    outside = [i for i, (xs, ys, xe, ye) in enumerate(mask_coords_list_cycle) if xs < 0 or ys < 0 or xe > W or ye > H]
    if outside:
        logger.warning("avatar %s: the crop boxes of frames %s leave the frame; the files are written as the reference writes them, "
                       "but the engine's MuseTalk avatar loader refuses such frames", avatar_id, outside)

    with open(os.path.join(avatar_save_path, 'mask_coords.pkl'), 'wb') as f:
        pickle.dump(mask_coords_list_cycle, f)
    with open(os.path.join(avatar_save_path, 'coords.pkl'), 'wb') as f:
        pickle.dump(coord_list, f)
    torch.save(input_latent_list, os.path.join(avatar_save_path, 'latents.pt'))
    t0 = time.perf_counter()
    if len({fr.shape for fr in frames}) == 1:
        avatar_pack.pack_musetalk_lists(frames, [cv2.cvtColor(m, cv2.COLOR_GRAY2BGR) for m in mask_list_cycle], coord_list,
                                        mask_coords_list_cycle, input_latent_list, os.path.join(avatar_save_path, "avatar.ltbav"))
    timings["pack"] = time.perf_counter() - t0
    if progress_callback: progress_callback(100)
    print("Avatar 生成完成！")


if __name__ == '__main__':
    import argparse
    parser = argparse.ArgumentParser()
    parser.add_argument("--file", type=str, default=r'D:\ok\00000000.png')
    parser.add_argument("--avatar_id", type=str, default='musetalk_avatar1')
    parser.add_argument('--save_path', default='data/avatars', type=str)
    parser.add_argument("--version", type=str, default="v15", choices=["v1", "v15"], help="Version of MuseTalk: v1 or v15")
    parser.add_argument("--gpu_id", type=int, default=0, help="GPU ID to use")
    parser.add_argument("--left_cheek_width", type=int, default=90, help="Width of left cheek region")
    parser.add_argument("--right_cheek_width", type=int, default=90, help="Width of right cheek region")
    parser.add_argument("--bbox_shift", type=int, default=0, help="Bounding box shift value")
    parser.add_argument("--extra_margin", type=int, default=10, help="Extra margin for face cropping")
    parser.add_argument("--parsing_mode", default='jaw', help="Face blending parsing mode")
    args = parser.parse_args()
    generate_avatar(video_path=args.file, avatar_id=args.avatar_id, save_path=args.save_path, bbox_shift=args.bbox_shift,
                    extra_margin=args.extra_margin, parsing_mode=args.parsing_mode, version=args.version)
