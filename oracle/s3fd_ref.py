"""Functional fp32 restatement of the S3FD face detector the wav2lip avatar generator runs (avatars/wav2lip/genavatar.py ->
face_detection/api.py FaceAlignment.get_detections_for_batch -> detection/sfd: net_s3fd.s3fd, detect.batch_detect, bbox.nms).

Selection.  The reference keeps, per image, the first box of nms(candidates, 0.3) whose score is above 0.5, where the candidates
are the anchors at which *any* image of the batch scores above 0.05.  NMS keeps the highest-scoring candidate first, and an anchor
where an image scores above 0.5 is always a candidate, so the result per image is the decoded box of its arg-max anchor over all six
levels when that score is above 0.5, and None otherwise.  Ties of exactly equal scores (implementation-defined in the reference:
numpy argsort) go to the lowest anchor number: levels in order, rows, then columns.

Also the seeded synthetic weights the tests use (no checkpoint is ever downloaded)."""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

MEAN_RGB = (104.0, 117.0, 123.0)
# (name, Cin, Cout, kernel, stride, padding); a "pool" entry is F.max_pool2d(h, 2, 2)
TRUNK = [("conv1_1", 3, 64, 3, 1, 1), ("conv1_2", 64, 64, 3, 1, 1), "pool",
         ("conv2_1", 64, 128, 3, 1, 1), ("conv2_2", 128, 128, 3, 1, 1), "pool",
         ("conv3_1", 128, 256, 3, 1, 1), ("conv3_2", 256, 256, 3, 1, 1), ("conv3_3", 256, 256, 3, 1, 1), "pool",
         ("conv4_1", 256, 512, 3, 1, 1), ("conv4_2", 512, 512, 3, 1, 1), ("conv4_3", 512, 512, 3, 1, 1), "pool",
         ("conv5_1", 512, 512, 3, 1, 1), ("conv5_2", 512, 512, 3, 1, 1), ("conv5_3", 512, 512, 3, 1, 1), "pool",
         ("fc6", 512, 1024, 3, 1, 3), ("fc7", 1024, 1024, 1, 1, 0),
         ("conv6_1", 1024, 256, 1, 1, 0), ("conv6_2", 256, 512, 3, 2, 1),
         ("conv7_1", 512, 128, 1, 1, 0), ("conv7_2", 128, 256, 3, 2, 1)]
# detection levels: (feature layer, channels, L2Norm scale or None); head names are <source>_mbox_conf / _mbox_loc
LEVELS = [("conv3_3", 256, 10.0), ("conv4_3", 512, 8.0), ("conv5_3", 512, 5.0), ("fc7", 1024, None), ("conv6_2", 512, None),
          ("conv7_2", 256, None)]
L2_EPS = 1e-10
CANDIDATE, THRESH = 0.05, 0.5


def head_prefix(level: int) -> str:
    src, _, scale = LEVELS[level]
    return f"{src}_norm" if scale is not None else src


def level_strides():
    return [2 ** (i + 2) for i in range(6)]


def head_shapes(H: int, W: int):
    """(h, w) of the six head maps for an H x W frame."""
    def pool(a):
        return a // 2
    h, w = H, W
    out = []
    for _ in range(2):
        h, w = pool(h), pool(w)
    out.append((h, w))                       # conv3_3
    h, w = pool(h), pool(w)
    out.append((h, w))                       # conv4_3
    h, w = pool(h), pool(w)
    out.append((h, w))                       # conv5_3
    h, w = pool(h) + 4, pool(w) + 4          # fc6: 3x3 with padding 3
    out.append((h, w))                       # fc7
    h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    out.append((h, w))                       # conv6_2
    h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    out.append((h, w))                       # conv7_2
    return out


def gmac_per_frame(H: int, W: int) -> float:
    """Multiply-accumulates of one H x W frame through the trunk and the twelve heads (max-pool and L2Norm not counted)."""
    h, w = H, W
    mac = 0
    shapes = {}
    for e in TRUNK:
        if e == "pool":
            h, w = h // 2, w // 2
            continue
        name, cin, cout, k, s, p = e
        h, w = (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1
        mac += h * w * cout * cin * k * k
        shapes[name] = (h, w)
    for (src, cin, _), hw in zip(LEVELS, head_shapes(H, W)):
        conf = 4 if src == "conv3_3" else 2
        mac += hw[0] * hw[1] * (conf + 4) * cin * 9
    return mac / 1e9


# ---------------------------------------------------------------------------------------------------------------- weights
def synth_state_dict(seed: int = 0, face_gain: float = 1.5e-4, face_bias: float = -3.0) -> dict:
    """Seeded conditioned weights in the reference's key scheme (conv1_1.weight ... conv7_2_mbox_loc.bias).

    Trunk: He-normal weights and zero biases, so the trunk is positively homogeneous: a frame at the channel means
    (BGR 123, 117, 104) gives all-zero features, and the features scale with the amplitude of the content around the means.
    Heads: small random loc weights (boxes near the anchor); on the three L2-normalised levels random conf weights with a
    background bias of +5 (scores stay below 0.05 .. 0.2: candidates, never detections); on fc7 a face logit of
    face_gain * sum_c fc7_c at the centre tap + face_bias with a zero background, so textured regions of enough amplitude are
    faces and flat frames are not; the two coarsest levels score ~0.0025 everywhere."""
    rng = np.random.default_rng(seed)
    sd = {}

    def put(name, w, b):
        sd[name + ".weight"] = torch.from_numpy(np.ascontiguousarray(w, np.float32))
        sd[name + ".bias"] = torch.from_numpy(np.ascontiguousarray(b, np.float32))

    for e in TRUNK:
        if e == "pool":
            continue
        name, cin, cout, k, _, _ = e
        put(name, rng.standard_normal((cout, cin, k, k)) * np.sqrt(2.0 / (cin * k * k)), np.zeros(cout))
    for src, c, scale in LEVELS:
        if scale is not None:
            sd[f"{src}_norm.weight"] = torch.full((c,), scale, dtype=torch.float32)
    for lv, (src, cin, scale) in enumerate(LEVELS):
        pre = head_prefix(lv)
        nconf = 4 if lv == 0 else 2
        put(pre + "_mbox_loc", rng.standard_normal((4, cin, 3, 3)) * (0.5 / np.sqrt(cin * 9 * (100.0 if scale else 1.0e4))),
            rng.standard_normal(4) * 0.1)
        if scale is not None:
            w = rng.standard_normal((nconf, cin, 3, 3)) * (0.6 / (scale * 3.0))
            b = np.zeros(nconf)
            b[:nconf - 1] = 5.0
        elif src == "fc7":
            w = np.zeros((2, cin, 3, 3))
            w[1, :, 1, 1] = face_gain
            b = np.array([0.0, face_bias])
        else:
            w = rng.standard_normal((2, cin, 3, 3)) * 1e-6
            b = np.array([3.0, -3.0])
        put(pre + "_mbox_conf", w, b)
    return sd


# ---------------------------------------------------------------------------------------------------------------- forward
def prep(frames_u8: np.ndarray, device="cpu") -> torch.Tensor:
    """u8 BGR [N,H,W,3] -> fp32 NCHW RGB minus the means (images[..., ::-1] then batch_detect's subtraction)."""
    x = torch.from_numpy(np.ascontiguousarray(frames_u8[..., ::-1])).to(device).float()
    x = x - torch.tensor(MEAN_RGB, device=device)
    return x.permute(0, 3, 1, 2).contiguous()


def _conv(sd, name, h, stride=1, padding=1, relu=True):
    y = F.conv2d(h, sd[name + ".weight"].to(h), sd[name + ".bias"].to(h), stride=stride, padding=padding)
    return F.relu(y) if relu else y


def l2norm(x, w):
    norm = x.pow(2).sum(dim=1, keepdim=True).sqrt() + L2_EPS
    return x / norm * w.to(x).view(1, -1, 1, 1)


def trunk(sd, x, keep=None):
    """Trunk of s3fd.forward; returns the six (un-normalised) level features.  keep: dict filled with every layer output."""
    h = x
    feats = {}
    for e in TRUNK:
        if e == "pool":
            h = F.max_pool2d(h, 2, 2)
            continue
        name, _, _, k, s, p = e
        h = _conv(sd, name, h, stride=s, padding=p)
        if keep is not None:
            keep[name] = h
        feats[name] = h
    return [feats[src] for src, _, _ in LEVELS]


def forward(sd, x, keep=None):
    """s3fd.forward: [cls1, reg1, ..., cls6, reg6] with the max-out background of level 0 (cls1 has 2 channels)."""
    feats = trunk(sd, x, keep)
    out = []
    for lv, (f, (src, _, scale)) in enumerate(zip(feats, LEVELS)):
        if scale is not None:
            f = l2norm(f, sd[f"{src}_norm.weight"])
            if keep is not None:
                keep[f"{src}_norm"] = f
        pre = head_prefix(lv)
        cls = _conv(sd, pre + "_mbox_conf", f, relu=False)
        reg = _conv(sd, pre + "_mbox_loc", f, relu=False)
        if lv == 0:
            c = torch.chunk(cls, 4, 1)
            cls = torch.cat([torch.max(torch.max(c[0], c[1]), c[2]), c[3]], dim=1)
        out += [cls, reg]
    return out


# ---------------------------------------------------------------------------------------------------------------- selection
def scores_and_boxes(olist):
    """Per level: softmax face score [N, h*w] and batch_decode boxes [N, h*w, 4] (fp32, the reference's arithmetic order)."""
    sc, bx = [], []
    for i in range(len(olist) // 2):
        cls, reg = olist[2 * i].float(), olist[2 * i + 1].float()
        N, _, fh, fw = cls.shape
        stride = 2 ** (i + 2)
        s = F.softmax(cls, dim=1)[:, 1].reshape(N, -1)
        ys, xs = torch.meshgrid(torch.arange(fh, device=cls.device), torch.arange(fw, device=cls.device), indexing="ij")
        cx = (stride / 2 + xs.reshape(-1) * stride).float()
        cy = (stride / 2 + ys.reshape(-1) * stride).float()
        size = torch.full_like(cx, stride * 4.0)
        loc = reg.reshape(N, 4, -1).permute(0, 2, 1)                            # [N, hw, 4]
        bxy = torch.stack([cx, cy], 1)[None] + loc[..., :2] * 0.1 * torch.stack([size, size], 1)[None]
        bwh = torch.stack([size, size], 1)[None] * torch.exp(loc[..., 2:] * 0.2)
        b1 = bxy - bwh / 2
        b2 = bwh + b1
        sc.append(s)
        bx.append(torch.cat([b1, b2], -1))
    return torch.cat(sc, 1), torch.cat(bx, 1)


def select(olist, thresh: float = THRESH):
    """-> (found bool [N], boxes int64 [N,4] (clipped at 0, truncated), score float32 [N], anchor int64 [N]) by arg-max."""
    s, b = scores_and_boxes(olist)
    s, b = s.cpu().numpy(), b.cpu().numpy()
    anchor = s.argmax(1)                               # numpy argmax: first (lowest) index among equal maxima
    n = np.arange(s.shape[0])
    score = s[n, anchor]
    box = np.clip(b[n, anchor], 0, None).astype(np.float32)
    return score > thresh, np.trunc(box).astype(np.int64), score, anchor


def detections(olist, thresh: float = THRESH):
    """The get_detections_for_batch contract: list of (x1, y1, x2, y2) or None."""
    found, box, _, _ = select(olist, thresh)
    return [tuple(int(v) for v in box[i]) if found[i] else None for i in range(len(found))]


def detect(sd, frames_u8: np.ndarray, device="cpu"):
    with torch.no_grad():
        return detections(forward(sd, prep(frames_u8, device)))


# ---------------------------------------------------------------------------------------------------------------- test inputs
BG_BGR = (123, 117, 104)          # the channel means in BGR order: prepares to exactly zero


def synth_frames(amps, H: int, W: int, seed: int = 0, blob=None) -> np.ndarray:
    """u8 BGR frames at the channel means with one textured square per frame: frame i has noise of amplitude amps[i] (0: flat,
    never a face; ~10: scores between 0.05 and 0.5, candidates only; >= 35: a face) at blob[i] = (y, x, side)."""
    rng = np.random.default_rng(seed)
    out = np.empty((len(amps), H, W, 3), np.uint8)
    out[:] = BG_BGR
    for i, a in enumerate(amps):
        side = max(16, min(H, W) // 3)
        y, x = (H // 4 + 7 * i) % max(1, H - side), (W // 3 + 11 * i) % max(1, W - side)
        if blob is not None:
            y, x, side = blob[i]
        tex = np.asarray(BG_BGR, np.float64) + a * rng.standard_normal((side, side, 3))
        out[i, y:y + side, x:x + side] = np.clip(np.round(tex), 0, 255).astype(np.uint8)
    return out


def write_video(path: str, frames: np.ndarray, fps: int = 25) -> None:
    """MJPG .avi of the frames (cv2.VideoWriter)."""
    import cv2
    H, W = frames.shape[1:3]
    vw = cv2.VideoWriter(path, cv2.VideoWriter_fourcc(*"MJPG"), fps, (W, H))
    for f in frames:
        vw.write(np.ascontiguousarray(f))
    vw.release()
