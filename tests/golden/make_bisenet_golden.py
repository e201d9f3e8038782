"""Writes tests/golden/bisenet_golden.npz by running the unmodified LiveTalking BiSeNet, FaceParsing, get_image_prepare_material and
MuseTalk genavatar.generate_avatar on the CPU:

    python tests/golden/make_bisenet_golden.py /path/to/LiveTalking

Weights: oracle.bisenet_ref.synth_state_dict(0), written to ./models/face-parse-bisent/{79999_iter,resnet18-5c106cde}.pth of a
temporary working directory (Resnet18.init_weight torch.loads the second).  preprocessing.py builds FaceAlignment and imports
face_recognition at import time and genavatar imports load_all_model (diffusers): replaying stand-ins are injected through
sys.modules for all three.  The stand-in VAE returns a constant (1, 8, 32, 32) latent per crop and records the crops.

Contents:
  net_rgb_crc / net_logits_s8 / net_labels   crc32 of the two 512 x 512 RGB inputs (synth_video_frames(2, 512, 512, seed=3),
                                         RGB order), BiSeNet(x)[0] at every 8th pixel, out.argmax(0)
  fp_img_crc / fp_raw / fp_neck / fp_jaw crc32 of a 300 x 280 crop (synth_video_frames(1, 280, 300, seed=5), RGB order) and
                                         FaceParsing(90, 90)(crop, mode) for the three modes
  fp_labels                              the labels behind them (the arg-max of the net on the resized crop)
  ga_video                               bytes of the MJPG clip generate_avatar ran on (GA_N frames of GA_H x GA_W)
  ga_boxes                               the replayed detector boxes; frame 2's crop box runs past the top-left of the frame
  ga_lm_boxes                            the boxes the replayed landmarks were drawn in; frame 4's lies partly left of the frame, so
                                         its landmark box falls back to the detector box
  ga_rgb_crc / ga_labels                 crc32 of every face_seg input after the 512 resize, and the labels the net gave it
  ga_latent_crc                          zlib.crc32 of each LANCZOS4 crop handed to get_latents_for_unet
  ga_full_crc / ga_mask_crc              zlib.crc32 of the PNG files
  ga_coords_pkl / ga_mask_coords_pkl / ga_info   the bytes of coords.pkl, mask_coords.pkl and avator_info.json
  ga_progress                            the progress_callback sequence
  ga_args                                genavatar.py's argparse options as "dest|default|type" strings"""
import os
import runpy
import sys
import tempfile
import types
import zlib

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import bisenet_ref as R  # noqa: E402
from oracle import pfld_ref, s3fd_ref  # noqa: E402

GA_N, GA_H, GA_W = 8, 240, 320
GA_BOXES = [(100, 60, 190, 170), (104, 62, 192, 168), (2, 3, 90, 110), (150, 80, 230, 190), (60, 40, 160, 150), (120, 70, 200, 180),
            (130, 50, 220, 160), (90, 66, 180, 175)]
GA_LM_BOXES = [(105, 70, 185, 165), (108, 70, 188, 166), (6, 10, 86, 105), (155, 88, 225, 185), (-30, 50, 150, 140),
               (125, 78, 195, 176), (135, 60, 215, 158), (95, 72, 175, 170)]


def _install_stand_ins(seen_crops):
    fd = types.ModuleType("face_detection")

    class FaceAlignment:
        def __init__(self, *a, **k):
            self.i = 0

        def get_detections_for_batch(self, images):
            out = []
            for _ in images:
                out.append(GA_BOXES[self.i])
                self.i += 1
            return out
    fd.FaceAlignment = FaceAlignment
    fd.LandmarksType = types.SimpleNamespace(_2D=1)
    sys.modules["face_detection"] = fd
    fr = types.ModuleType("face_recognition")
    fr.face_landmarks = R.ReplayLandmarks([R.synth_landmarks(b, seed=i) for i, b in enumerate(GA_LM_BOXES)])
    sys.modules["face_recognition"] = fr
    ut = types.ModuleType("avatars.musetalk.utils.utils")

    class VAE:
        def __init__(self):
            self.vae = types.SimpleNamespace(half=lambda: types.SimpleNamespace(to=lambda d: None))

        def get_latents_for_unet(self, img):
            seen_crops.append(zlib.crc32(np.ascontiguousarray(img).tobytes()))
            return torch.full((1, 8, 32, 32), float(img.mean()) / 255)
    ut.load_all_model = lambda device=None: (VAE(), None, None)
    sys.modules["avatars.musetalk.utils.utils"] = ut


def main(ref_root):
    sys.path.insert(0, ref_root)
    seen_crops = []
    _install_stand_ins(seen_crops)
    from PIL import Image
    from avatars.musetalk.utils.face_parsing import FaceParsing
    from avatars.musetalk.utils.face_parsing.model import BiSeNet

    sd = R.synth_state_dict(0)
    tmp = tempfile.mkdtemp(prefix="bisenet_golden_")
    mdir = os.path.join(tmp, "models", "face-parse-bisent")
    os.makedirs(mdir)
    torch.save(sd, os.path.join(mdir, "79999_iter.pth"))
    torch.save({k[len("cp.resnet."):]: v for k, v in sd.items() if k.startswith("cp.resnet.")}, os.path.join(mdir, "resnet18-5c106cde.pth"))
    out = {}
    rgb = np.ascontiguousarray(pfld_ref.synth_video_frames(2, 512, 512, seed=3)[..., ::-1])
    net = BiSeNet(os.path.join(mdir, "resnet18-5c106cde.pth"))
    net.load_state_dict(sd)
    net.eval()
    with torch.no_grad():
        o = net(R.prep(rgb))[0]
    out["net_rgb_crc"], out["net_logits_s8"], out["net_labels"] = zlib.crc32(rgb.tobytes()), o[:, :, ::8, ::8].numpy(), o.numpy().argmax(1).astype(np.uint8)

    cwd = os.getcwd()
    os.chdir(tmp)
    try:
        fp = FaceParsing(left_cheek_width=90, right_cheek_width=90)
        calls = []
        fwd = fp.net.forward

        def recording_forward(x):
            r = fwd(x)
            calls.append(((x[0].permute(1, 2, 0) * torch.tensor(R.STD) + torch.tensor(R.MEAN)) * 255, r[0][0].numpy().argmax(0)))
            return r
        fp.net.forward = recording_forward
        img = Image.fromarray(np.ascontiguousarray(pfld_ref.synth_video_frames(1, 280, 300, seed=5)[0][..., ::-1]))
        out["fp_img_crc"] = zlib.crc32(np.asarray(img).tobytes())
        for mode in ("raw", "neck", "jaw"):
            out["fp_" + mode] = np.asarray(fp(img, mode=mode))
        out["fp_labels"] = calls[0][1].astype(np.uint8)
        calls.clear()

        import avatars.musetalk.utils.face_parsing as fpmod
        orig_init = fpmod.FaceParsing.__init__

        def recording_init(self, *a, **k):
            orig_init(self, *a, **k)
            f = self.net.forward

            def rec(x):
                r = f(x)
                calls.append((np.round(((x[0].permute(1, 2, 0) * torch.tensor(R.STD) + torch.tensor(R.MEAN)) * 255).numpy()).astype(np.uint8),
                              r[0][0].numpy().argmax(0).astype(np.uint8)))
                return r
            self.net.forward = rec
        fpmod.FaceParsing.__init__ = recording_init
        vid = os.path.join(tmp, "clip.avi")
        s3fd_ref.write_video(vid, pfld_ref.synth_video_frames(GA_N, GA_H, GA_W, seed=7))
        progress = []
        argv = sys.argv
        sys.argv = ["genavatar.py"]
        try:
            g = runpy.run_path(os.path.join(ref_root, "avatars", "musetalk", "genavatar.py"), run_name="genavatar")
        finally:
            sys.argv = argv
        g["generate_avatar"](vid, "ga", save_path=os.path.join(tmp, "data", "avatars"), progress_callback=progress.append)
    finally:
        os.chdir(cwd)
    av = os.path.join(tmp, "data", "avatars", "ga")
    crc = lambda d: np.array([zlib.crc32(open(os.path.join(av, d, f), "rb").read()) for f in sorted(os.listdir(os.path.join(av, d)))],  # noqa: E731
                             np.uint32)
    out["ga_video"] = np.frombuffer(open(vid, "rb").read(), np.uint8)
    out["ga_boxes"] = np.array(GA_BOXES, np.int64)
    out["ga_lm_boxes"] = np.array(GA_LM_BOXES, np.int64)
    out["ga_rgb_crc"] = np.array([zlib.crc32(c[0].tobytes()) for c in calls], np.uint32)
    out["ga_labels"] = np.stack([c[1] for c in calls])
    out["ga_latent_crc"] = np.array(seen_crops, np.uint32)
    out["ga_full_crc"] = crc("full_imgs")
    out["ga_mask_crc"] = crc("mask")
    for name, key in (("coords.pkl", "ga_coords_pkl"), ("mask_coords.pkl", "ga_mask_coords_pkl"), ("avator_info.json", "ga_info")):
        out[key] = np.frombuffer(open(os.path.join(av, name), "rb").read(), np.uint8)
    out["ga_progress"] = np.array(progress, np.int64)
    src = open(os.path.join(ref_root, "avatars", "musetalk", "genavatar.py")).read()
    ns = {}
    exec(src[src.index("    parser = argparse.ArgumentParser()"):src.index("    args = parser.parse_args()")].replace("\n    ", "\n").strip(),
         {"argparse": __import__("argparse")}, ns)
    out["ga_args"] = np.array([f"{a.dest}|{a.default}|{getattr(a.type, '__name__', None)}" for a in ns["parser"]._actions if a.dest != "help"])
    print("progress", progress, "args", out["ga_args"].tolist())
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "bisenet_golden.npz"), **out)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "/path/to/LiveTalking")
