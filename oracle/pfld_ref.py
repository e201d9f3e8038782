"""Functional restatement of the landmark step of the UltraLight avatar generator (avatars/ultralight/genavatar.py ->
face_detect_utils/get_landmark.py Landmark.detect -> pfld_mobileone.PFLD_GhostOne(width_factor=0.5, input_size=192)).

* The network in its re-parameterised form: every MobileOneBlock (base_module.py) folded into one conv with bias, in float64, by
  the arithmetic of MobileOneBlock._get_kernel_bias (BN-fold each branch, pad the 1x1 scale branch to k x k, identity kernel for the
  skip BatchNorm), then run in fp32 (or float64) with F.conv2d.
* The host steps of face_det, Landmark.detect and the genavatar loop, restated operation for operation.
* Seeded synthetic train-time weights in the reference's key scheme, and a stand-in for the SCRFD detector that replays recorded
  (bboxes, indices, kpss) (the real one needs ./models/scrfd_2.5g_kps.onnx)."""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

INPUT = 192
LANDMARKS = 110
BRANCHES = 6                 # PFLD_GhostOne.num_conv_branches
BN_EPS = 1e-5                # nn.BatchNorm2d default
W = 0.5                      # width_factor


def _c(x):
    return int(x * W)


# GhostOneBottleneck(in, hidden, out, stride), pfld_mobileone.py:59-72
BOTTLENECKS = [("conv3_1", _c(64), _c(96), _c(80), 2), ("conv3_2", _c(80), _c(120), _c(80), 1), ("conv3_3", _c(80), _c(120), _c(80), 1),
               ("conv4_1", _c(80), _c(200), _c(96), 2), ("conv4_2", _c(96), _c(240), _c(96), 1), ("conv4_3", _c(96), _c(240), _c(96), 1),
               ("conv5_1", _c(96), _c(336), _c(144), 2), ("conv5_2", _c(144), _c(504), _c(144), 1),
               ("conv5_3", _c(144), _c(504), _c(144), 1), ("conv5_4", _c(144), _c(504), _c(144), 1),
               ("conv6", _c(144), _c(216), _c(16), 1)]
TAP_AFTER = {"conv2": 0, "conv3_3": 1, "conv4_3": 2, "conv5_4": 3}   # x1..x4: AvgPool2d over the whole map


def ghost_blocks(name, cin, cout, relu):
    """The two MobileOneBlocks of a GhostOneModule: primary 1x1 cin -> ceil(cout/2), cheap depthwise 3x3; output = their concat."""
    h = math.ceil(cout / 2)
    return [(name + ".primary_conv", cin, h, 1, 1, 1, relu), (name + ".cheap_operation", h, h, 3, 1, h, relu)]


def mobileone_blocks():
    """Every MobileOneBlock in forward order: (prefix, cin, cout, kernel, stride, groups, relu)."""
    out = [("conv1", 3, _c(64), 3, 2, 1, True), ("conv2", _c(64), _c(64), 3, 1, _c(64), True)]
    for name, cin, hid, cout, s in BOTTLENECKS:
        out += ghost_blocks(name + ".ghost_conv.0", cin, hid, True)
        if s == 2:
            out.append((name + ".ghost_conv.1", hid, hid, 3, 2, hid, False))
        out += ghost_blocks(name + ".ghost_conv.2", hid, cout, False)
    out.append(("conv7", _c(16), _c(32), 3, 1, 1, True))
    return out


def has_skip(cin, cout, stride):
    return cin == cout and stride == 1


def gflop_per_frame() -> float:
    """2 x the multiply-accumulates of the folded convs, conv8 and conv_out for one 192 x 192 crop."""
    mac, h = 0, INPUT
    for _, cin, cout, k, s, g, _ in mobileone_blocks():
        h = (h + 2 * (k // 2) - k) // s + 1
        mac += h * h * cout * (cin // g) * k * k
    mac += _c(128) * _c(32) * (INPUT // 16) ** 2 + 2 * LANDMARKS * _c(512)
    return 2.0 * mac / 1e9


# ---------------------------------------------------------------------------------------------------------------- weights
def _bn(rng, sd, p, c, gain=(0.6, 1.4)):
    sd[p + ".weight"] = rng.uniform(*gain, c)
    sd[p + ".bias"] = rng.normal(0, 0.05, c)
    sd[p + ".running_mean"] = rng.normal(0, 0.05, c)
    sd[p + ".running_var"] = rng.uniform(0.5, 1.5, c)
    sd[p + ".num_batches_tracked"] = np.array(0, np.int64)


def synth_state_dict(seed: int = 0, out_scale: float = 0.02) -> dict:
    """Seeded train-time weights in the reference's key scheme (conv1.rbr_conv.0.conv.weight ... conv_out.bias, and the unused
    localization branch).  Each branch is He-normal over sqrt(branches) so the folded blocks keep the activation scale; BN
    statistics are non-trivial; linear blocks get half the gain of ReLU blocks.  conv_out is scaled so the landmark offsets from
    the mean face are of order out_scale."""
    rng = np.random.default_rng(seed)
    sd = {}
    for p, cin, cout, k, s, g, relu in mobileone_blocks():
        nb = BRANCHES + (k > 1) + has_skip(cin, cout, s)
        gain = 1.6 if relu else 0.8
        std = math.sqrt(gain / ((cin // g) * k * k) / nb)
        for i in range(BRANCHES):
            sd[f"{p}.rbr_conv.{i}.conv.weight"] = rng.normal(0, std, (cout, cin // g, k, k))
            _bn(rng, sd, f"{p}.rbr_conv.{i}.bn", cout)
        if k > 1:
            sd[f"{p}.rbr_scale.conv.weight"] = rng.normal(0, math.sqrt(gain / (cin // g) / nb), (cout, cin // g, 1, 1))
            _bn(rng, sd, f"{p}.rbr_scale.bn", cout)
        if has_skip(cin, cout, s):
            _bn(rng, sd, f"{p}.rbr_skip", cin, gain=(0.2, 0.6))
    k8 = INPUT // 16
    sd["conv8.0.weight"] = rng.normal(0, math.sqrt(2.0 / (_c(32) * k8 * k8)), (_c(128), _c(32), k8, k8))
    sd["conv_out.weight"] = rng.normal(0, out_scale / math.sqrt(_c(512)), (2 * LANDMARKS, _c(512), 1, 1))
    sd["conv_out.bias"] = rng.normal(0, out_scale, 2 * LANDMARKS)
    sd["localization.0.weight"] = rng.normal(0, 0.1, (8, 1, 7, 7))
    sd["localization.0.bias"] = rng.normal(0, 0.1, 8)
    sd["localization.3.weight"] = rng.normal(0, 0.1, (10, 8, 5, 5))
    sd["localization.3.bias"] = rng.normal(0, 0.1, 10)
    return {k: torch.from_numpy(np.asarray(v, np.int64 if k.endswith("num_batches_tracked") else np.float32)) for k, v in sd.items()}


def _f64(t):
    return t.detach().cpu().double() if torch.is_tensor(t) else torch.as_tensor(np.asarray(t), dtype=torch.float64)


def fold_block(sd, p, cin, cout, k, stride, groups):
    """MobileOneBlock._get_kernel_bias in float64 -> (kernel [cout, cin/groups, k, k], bias [cout]).  A re-parameterised state dict
    (p.reparam_conv.weight / .bias) is taken as it is."""
    if p + ".reparam_conv.weight" in sd:
        return _f64(sd[p + ".reparam_conv.weight"]), _f64(sd[p + ".reparam_conv.bias"])

    def fuse(kernel, bn):
        std = (_f64(sd[bn + ".running_var"]) + BN_EPS).sqrt()
        g = _f64(sd[bn + ".weight"])
        t = (g / std).reshape(-1, 1, 1, 1)
        return kernel * t, _f64(sd[bn + ".bias"]) - _f64(sd[bn + ".running_mean"]) * g / std

    kern = torch.zeros(cout, cin // groups, k, k, dtype=torch.float64)
    bias = torch.zeros(cout, dtype=torch.float64)
    if k > 1:
        ks, bs = fuse(_f64(sd[p + ".rbr_scale.conv.weight"]), p + ".rbr_scale.bn")
        kern, bias = kern + F.pad(ks, [k // 2] * 4), bias + bs
    if p + ".rbr_skip.weight" in sd:
        idk = torch.zeros(cin, cin // groups, k, k, dtype=torch.float64)
        for i in range(cin):
            idk[i, i % (cin // groups), k // 2, k // 2] = 1
        ki, bi = fuse(idk, p + ".rbr_skip")
        kern, bias = kern + ki, bias + bi
    for i in range(BRANCHES):
        kc, bc = fuse(_f64(sd[f"{p}.rbr_conv.{i}.conv.weight"]), f"{p}.rbr_conv.{i}.bn")
        kern, bias = kern + kc, bias + bc
    return kern, bias


def backbone(sd):
    """The checkpoint's 'pfld_backbone' state dict, or sd itself."""
    return sd["pfld_backbone"] if "pfld_backbone" in sd else sd


def folded(sd) -> dict:
    """prefix -> (kernel, bias, stride, padding, groups, relu) float64 for every MobileOneBlock, plus conv8 and conv_out."""
    sd = backbone(sd)
    out = {}
    for p, cin, cout, k, s, g, relu in mobileone_blocks():
        w, b = fold_block(sd, p, cin, cout, k, s, g)
        out[p] = (w, b, s, k // 2, g, relu)
    out["conv8"] = (_f64(sd["conv8.0.weight"]), None, 1, 0, 1, True)
    out["conv_out"] = (_f64(sd["conv_out.weight"]), _f64(sd["conv_out.bias"]), 1, 0, 1, False)
    return out


# ---------------------------------------------------------------------------------------------------------------- forward
def _conv(fw, name, x):
    w, b, s, p, g, relu = fw[name]
    y = F.conv2d(x, w.to(x), None if b is None else b.to(x), stride=s, padding=p, groups=g)
    return F.relu(y) if relu else y


def forward(fw, x, keep=None, conv=None):
    """PFLD_GhostOne.forward on the folded weights fw (folded()); x [N,3,192,192] in x's dtype -> landmarks [N,220] (before
    mean_face).  keep: dict filled with every block output and the multi-scale features.  conv(name, h): how a block runs
    (default: the folded conv; forward_train passes the train-time branches)."""
    conv = conv or (lambda name, h: _conv(fw, name, h))
    taps = []

    def run(name, h):
        h = conv(name, h)
        if keep is not None:
            keep[name] = h
        return h

    h = run("conv2", run("conv1", x))
    taps.append(F.avg_pool2d(h, INPUT // 2))
    for name, cin, hid, cout, s in BOTTLENECKS:
        a = run(name + ".ghost_conv.0.primary_conv", h)
        h = torch.cat([a, run(name + ".ghost_conv.0.cheap_operation", a)], 1)
        if s == 2:
            h = run(name + ".ghost_conv.1", h)
        a = run(name + ".ghost_conv.2.primary_conv", h)
        h = torch.cat([a, run(name + ".ghost_conv.2.cheap_operation", a)], 1)
        if keep is not None:
            keep[name] = h
        if name in TAP_AFTER:
            taps.append(F.avg_pool2d(h, h.shape[-1]))
    h = run("conv7", h)
    taps.append(run("conv8", h))
    ms = torch.cat(taps, 1)
    if keep is not None:
        keep["multi_scale"] = ms
    return run("conv_out", ms).reshape(x.shape[0], -1)


def forward_train(sd, x):
    """PFLD_GhostOne.forward in its train-time form, eval mode: every MobileOneBlock evaluates its six conv + BN branches, the
    scale branch and the skip BatchNorm (base_module.py MobileOneBlock.forward); weights of sd moved to x's device and dtype."""
    sd = backbone(sd)
    blocks = {b[0]: b for b in mobileone_blocks()}

    def bn(h, p):
        return F.batch_norm(h, sd[p + ".running_mean"], sd[p + ".running_var"], sd[p + ".weight"], sd[p + ".bias"], False, 0.0, BN_EPS)

    def conv(name, h):
        if name == "conv8":
            return F.relu(F.conv2d(h, sd["conv8.0.weight"]))
        if name == "conv_out":
            return F.conv2d(h, sd["conv_out.weight"], sd["conv_out.bias"])
        _, cin, cout, k, s, g, relu = blocks[name]
        out = 0
        if k > 1:
            out = bn(F.conv2d(h, sd[name + ".rbr_scale.conv.weight"], stride=s, groups=g), name + ".rbr_scale.bn")
        if has_skip(cin, cout, s):
            out = out + bn(h, name + ".rbr_skip")
        for i in range(BRANCHES):
            out = out + bn(F.conv2d(h, sd[f"{name}.rbr_conv.{i}.conv.weight"], stride=s, padding=k // 2, groups=g), f"{name}.rbr_conv.{i}.bn")
        return F.relu(out) if relu else out
    return forward(None, x, conv=conv)


def prep(crops_u8: np.ndarray) -> torch.Tensor:
    """Landmark.detect's input: the 192 x 192 BGR crops as fp32 v / 255, NCHW (no channel swap)."""
    x = np.asarray(crops_u8, dtype=np.float32) / 255.0
    return torch.from_numpy(np.ascontiguousarray(x.transpose(0, 3, 1, 2)))


def landmarks(raw: np.ndarray, mean_face: np.ndarray, w: int, h: int) -> np.ndarray:
    """Landmark.detect after the network: + mean_face, x *= w, y *= h (fp32), astype(int32)."""
    p = np.asarray(raw, np.float32) + mean_face
    p = p.reshape(-1, 2)
    p[:, 0] *= w
    p[:, 1] *= h
    return p.astype(np.int32)


def read_mean_face(path: str) -> np.ndarray:
    with open(path, "r") as f:
        return np.asarray(f.read().split(" "), dtype=np.float32)


# ---------------------------------------------------------------------------------------------------------------- host steps
def face_det(img, detector):
    """get_landmark.face_det for the first NMS index: (cropped image with zero border, [x1, y1, x2, y2]) or None without a face."""
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
        return cropped, [x1, y1, x2, y2]
    return None


def mouth_crop(img, lms, x1, y1, target_size):
    """The genavatar loop body after Landmark.detect: (face crop resized to target_size, coords tuple) or None when the slice is
    empty.  img[ymin:ymax, xmin:xmax] keeps numpy's slicing (a negative start counts from the end); cv2.resize's third positional
    argument is dst, so the interpolation is the default INTER_LINEAR."""
    import cv2
    xmin = lms[1][0] + x1
    ymin = lms[52][1] + y1
    xmax = lms[31][0] + x1
    width = xmax - xmin
    ymax = ymin + width
    crop_img = img[ymin:ymax, xmin:xmax]
    h, w = crop_img.shape[:2]
    if h == 0 or w == 0:
        return None
    crop_img = cv2.resize(crop_img, (target_size, target_size), cv2.INTER_AREA)
    return crop_img, (xmin, ymin, xmin + w, ymin + h)


class ReplayDetector:
    """Stands in for SCRFD: detect(img) returns the next recorded (bboxes [k, 4] as x, y, w, h; indices; kpss [k, 5, 2])."""

    def __init__(self, records):
        self.records, self.i = list(records), 0

    def detect(self, img):
        r = self.records[self.i % len(self.records)]
        self.i += 1
        return r


def face_records(boxes):
    """(x, y, w, h) per frame -> SCRFD-style detect() results with one face, index 0 first, and a decoy box after it."""
    out = []
    for x, y, w, h in boxes:
        b = np.array([[x, y, w, h], [x + 5.5, y + 3.25, w * 0.5, h * 0.5]], np.float32)
        kps = np.zeros((2, 5, 2), np.float32)
        kps[0, 0], kps[0, 1] = (x + 0.3 * w, y + 0.4 * h), (x + 0.7 * w, y + 0.42 * h)
        out.append((b, np.array([0, 1], np.int32), kps))
    return out


def synth_video_frames(n: int, H: int, W: int, seed: int = 0) -> np.ndarray:
    """Textured u8 BGR frames (smooth gradients plus noise), so the 192 x 192 crops carry varied content."""
    rng = np.random.default_rng(seed)
    yy, xx = np.meshgrid(np.linspace(0, 1, H), np.linspace(0, 1, W), indexing="ij")
    out = np.empty((n, H, W, 3), np.uint8)
    for i in range(n):
        base = np.stack([128 + 100 * np.sin(6 * xx + i * 0.3 + c) * np.cos(4 * yy - c) for c in range(3)], -1)
        out[i] = np.clip(base + rng.normal(0, 12, (H, W, 3)), 0, 255).astype(np.uint8)
    return out
