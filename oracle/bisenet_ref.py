"""Functional restatement of the MuseTalk face parser (avatars/musetalk/utils/face_parsing: BiSeNet over ResNet-18, FaceParsing's
ToTensor + Normalize, the arg-max and the per-mode class mapping) in float64 / fp32 torch, with every BatchNorm folded in float64.

    fw = folded(sd)                          # sd: the reference's BiSeNet state dict (79999_iter.pth key scheme)
    logits = forward(fw, prep(rgb512_u8))    # [n, 19, 64, 64] before the bilinear resize
    labels = parse(fw, rgb512_u8)            # [n, 512, 512] int64: out.argmax(0) of FaceParsing
    mask = postprocess(labels[0], "jaw", 90, 90)

Only output [0] of BiSeNet is computed (FaceParsing reads nothing else): conv_out16 / conv_out32 are dead code.  The golden file
tests/golden/bisenet_golden.npz, made by running the unmodified reference, pins this module (tests/test_bisenet_oracle.py)."""
from __future__ import annotations

from typing import Dict, Tuple

import numpy as np
import torch
import torch.nn.functional as F

BN_EPS = 1e-5
N_CLASSES = 19
MEAN = (0.485, 0.456, 0.406)
STD = (0.229, 0.224, 0.225)
# (layer, blocks, cin, cout, stride) of Resnet18
LAYERS = [("layer1", 2, 64, 64, 1), ("layer2", 2, 64, 128, 2), ("layer3", 2, 128, 256, 2), ("layer4", 2, 256, 512, 2)]


def _conv_bn_keys():
    """(conv weight key, BN prefix or None, kernel, cin, cout) of every conv of the reference's BiSeNet, dead heads included."""
    out = [("cp.resnet.conv1.weight", "cp.resnet.bn1", 7, 3, 64)]
    for name, nb, cin, cout, s in LAYERS:
        for b in range(nb):
            p = f"cp.resnet.{name}.{b}"
            ci = cin if b == 0 else cout
            out += [(p + ".conv1.weight", p + ".bn1", 3, ci, cout), (p + ".conv2.weight", p + ".bn2", 3, cout, cout)]
            if b == 0 and (cin != cout or s != 1):
                out.append((p + ".downsample.0.weight", p + ".downsample.1", 1, cin, cout))
    for arm, cin in (("cp.arm16", 256), ("cp.arm32", 512)):
        out += [(arm + ".conv.conv.weight", arm + ".conv.bn", 3, cin, 128), (arm + ".conv_atten.weight", arm + ".bn_atten", 1, 128, 128)]
    out += [("cp.conv_head32.conv.weight", "cp.conv_head32.bn", 3, 128, 128), ("cp.conv_head16.conv.weight", "cp.conv_head16.bn", 3, 128, 128),
            ("cp.conv_avg.conv.weight", "cp.conv_avg.bn", 1, 512, 128),
            ("ffm.convblk.conv.weight", "ffm.convblk.bn", 1, 256, 256), ("ffm.conv1.weight", None, 1, 256, 64), ("ffm.conv2.weight", None, 1, 64, 256),
            ("conv_out.conv.conv.weight", "conv_out.conv.bn", 3, 256, 256), ("conv_out.conv_out.weight", None, 1, 256, N_CLASSES)]
    for head in ("conv_out16", "conv_out32"):
        out += [(head + ".conv.conv.weight", head + ".conv.bn", 3, 128, 64), (head + ".conv_out.weight", None, 1, 64, N_CLASSES)]
    return out


def synth_state_dict(seed: int = 0) -> Dict[str, torch.Tensor]:
    """A BiSeNet state dict with the reference's keys (running statistics included), conditioned so that every activation of the
    fp16 engine stays well below 2^14: He-scaled conv weights times 0.7, BN scales in [0.5, 1], small shifts and means."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for wk, bn, k, cin, cout in _conv_bn_keys():
        scale = 0.7 * (2.0 / (cin * k * k)) ** 0.5
        sd[wk] = torch.randn(cout, cin, k, k, generator=g) * scale
        if bn is not None:
            sd[bn + ".weight"] = 0.5 + 0.5 * torch.rand(cout, generator=g)
            sd[bn + ".bias"] = 0.1 * torch.randn(cout, generator=g)
            sd[bn + ".running_mean"] = 0.1 * torch.randn(cout, generator=g)
            sd[bn + ".running_var"] = 0.5 + torch.rand(cout, generator=g)
            sd[bn + ".num_batches_tracked"] = torch.tensor(0)
    # class logits: conv_out's features are post-ReLU (positive means), so a class whose weights have the largest sum would win
    # almost everywhere; zero-mean rows over the input channels let every class win somewhere, and the scale spreads the margins
    w = sd["conv_out.conv_out.weight"]
    w = w - w.mean(1, keepdim=True)
    w[1] = 1.05 * w[0]                # the skin class (1, which the masks keep) takes part of the background class's region
    sd["conv_out.conv_out.weight"] = 4.0 * w
    return sd


def _f64(t) -> np.ndarray:
    return t.detach().cpu().double().numpy() if hasattr(t, "detach") else np.asarray(t, np.float64)


def fold(sd, wk: str, bn) -> Tuple[np.ndarray, np.ndarray]:
    """conv (no bias) + BatchNorm in float64 -> (weight [cout, cin, k, k], bias [cout]); bias 0 without a BN."""
    w = _f64(sd[wk])
    if bn is None:
        return w, np.zeros(w.shape[0])
    s = _f64(sd[bn + ".weight"]) / np.sqrt(_f64(sd[bn + ".running_var"]) + BN_EPS)
    return w * s[:, None, None, None], _f64(sd[bn + ".bias"]) - _f64(sd[bn + ".running_mean"]) * s


def folded(sd) -> Dict[str, Tuple[np.ndarray, np.ndarray]]:
    """Every live conv folded with its BN, keyed by the conv weight's prefix (the key without '.weight')."""
    return {wk[: -len(".weight")]: fold(sd, wk, bn) for wk, bn, *_ in _conv_bn_keys() if not wk.startswith(("conv_out16", "conv_out32"))}


def space_to_depth(x: torch.Tensor) -> torch.Tensor:
    """[n, 3, 512, 512] -> [n, 16, 259, 259], the layout of csrc/bisenet.cu's prep: s2d pixel (j, i), channel (2 by + bx) * 3 + c
    holds input pixel (2 (j - 2) + by, 2 (i - 2) + bx); zero border (2 pixels before, 1 after) and zero channels 12-15."""
    n = x.shape[0]
    p = F.pad(x, (4, 2, 4, 2))                                                # 518 = 2 * 259
    p = p.reshape(n, 3, 259, 2, 259, 2).permute(0, 3, 5, 1, 2, 4).reshape(n, 12, 259, 259)
    return F.pad(p, (0, 0, 0, 0, 0, 4))


def prep(rgb_u8: np.ndarray) -> torch.Tensor:
    """u8 RGB [n, 512, 512, 3] (the PIL resize output) -> fp32 [n, 3, 512, 512]: torchvision ToTensor + Normalize, in their order."""
    t = torch.from_numpy(np.ascontiguousarray(rgb_u8)).permute(0, 3, 1, 2).float().div(255)
    mean = torch.as_tensor(MEAN, dtype=torch.float32)[None, :, None, None]
    std = torch.as_tensor(STD, dtype=torch.float32)[None, :, None, None]
    return (t - mean) / std


def _t(fw, name, like):
    w, b = fw[name]
    return torch.from_numpy(w).to(like), torch.from_numpy(b).to(like)


def _cbr(fw, name, x, stride=1, relu=True):
    w, b = _t(fw, name, x)
    y = F.conv2d(x, w, b, stride=stride, padding=w.shape[-1] // 2)
    return torch.relu(y) if relu else y


def forward(fw, x: torch.Tensor) -> torch.Tensor:
    """BiSeNet(x)[0] before its bilinear resize: x [n, 3, H, W] normalised -> logits [n, 19, H/8, W/8], in x's dtype / device."""
    y = torch.relu(F.conv2d(x, *_t(fw, "cp.resnet.conv1", x), stride=2, padding=3))
    y = F.max_pool2d(y, 3, 2, 1)
    feats = []
    for name, nb, cin, cout, s in LAYERS:
        for b in range(nb):
            p = f"cp.resnet.{name}.{b}"
            st = s if b == 0 else 1
            r = _cbr(fw, p + ".conv1", y, st)
            r = _cbr(fw, p + ".conv2", r, relu=False)
            sc = _cbr(fw, p + ".downsample.0", y, st, relu=False) if p + ".downsample.0" in fw else y
            y = torch.relu(sc + r)
        feats.append(y)
    feat8, feat16, feat32 = feats[1:]

    def gate(name, f, act):
        w, b = _t(fw, name, f)
        return act(F.conv2d(f.mean((2, 3), keepdim=True), w, b))

    avg = gate("cp.conv_avg.conv", feat32, torch.relu)
    a32 = _cbr(fw, "cp.arm32.conv.conv", feat32)
    s32 = a32 * gate("cp.arm32.conv_atten", a32, torch.sigmoid) + avg
    up32 = _cbr(fw, "cp.conv_head32.conv", F.interpolate(s32, scale_factor=2, mode="nearest"))
    a16 = _cbr(fw, "cp.arm16.conv.conv", feat16)
    s16 = a16 * gate("cp.arm16.conv_atten", a16, torch.sigmoid) + up32
    up16 = _cbr(fw, "cp.conv_head16.conv", F.interpolate(s16, scale_factor=2, mode="nearest"))
    feat = _cbr(fw, "ffm.convblk.conv", torch.cat([feat8, up16], 1))
    w1, _ = _t(fw, "ffm.conv1", feat)
    w2, _ = _t(fw, "ffm.conv2", feat)
    att = torch.sigmoid(F.conv2d(torch.relu(F.conv2d(feat.mean((2, 3), keepdim=True), w1)), w2))
    fuse = feat * att + feat
    h = _cbr(fw, "conv_out.conv.conv", fuse)
    return F.conv2d(h, _t(fw, "conv_out.conv_out", h)[0])


def upsample(logits: torch.Tensor, size: int = 512) -> torch.Tensor:
    return F.interpolate(logits, (size, size), mode="bilinear", align_corners=True)


def parse(fw, rgb_u8: np.ndarray, dtype=torch.float64, device="cpu") -> np.ndarray:
    """FaceParsing's labels: out.argmax(0) per crop (numpy: exact ties to the lowest class) -> int64 [n, 512, 512]."""
    with torch.no_grad():
        out = upsample(forward(fw, prep(rgb_u8).to(device, dtype)))
    return out.cpu().numpy().argmax(1)


# ------------------------------------------------------------------------------------------------ FaceParsing's host steps
def cone_kernel() -> np.ndarray:
    """FaceParsing.__init__'s 33 x 33 dilation kernel: a cone of 21 rows (from row 10 on) and a 12-row tail of the base width."""
    cone_h, tail_h = 21, 12
    total = cone_h + tail_h
    k = np.zeros((total, total), np.uint8)
    cx = total // 2
    for row in range(cone_h // 2, cone_h):
        w = 2 * (row - cone_h // 2) + 1
        k[row, cx - w // 2: cx + w // 2 + 1] = 1
    base = int(k[cone_h - 1].sum())
    k[cone_h:, max(0, cx - base // 2): min(total, cx + base // 2 + 1)] = 1
    return k


def cheek_mask(left: int, right: int) -> np.ndarray:
    m = np.zeros((512, 512), np.uint8)
    m[:, : 256 - left + 1] = 255
    m[:, 256 + right:] = 255
    return m


def postprocess(parsing: np.ndarray, mode: str, left: int = 80, right: int = 80) -> np.ndarray:
    """FaceParsing.__call__'s class mapping on one label map -> u8 [512, 512] of 0 / 255."""
    import cv2
    p = np.asarray(parsing).astype(np.int64)
    if mode == "neck":
        keep = np.isin(p, [1, 11, 12, 13, 14])
    elif mode == "jaw":
        face = (p == 1).astype(np.uint8) * 255
        dil = cv2.dilate(face, cone_kernel(), iterations=1)
        ero = cv2.erode(dil, cv2.getStructuringElement(cv2.MORPH_ELLIPSE, (35, 3)), iterations=2)
        cm = cheek_mask(left, right)
        region = (ero & cm) | (dil & ~cm)
        keep = ((region == 255) & (p != 10)) | np.isin(p, [11, 12, 13])
    else:
        keep = np.isin(p, [1, 11, 12, 13])
    return np.where(keep, 255, 0).astype(np.uint8)


# ------------------------------------------------------------------------------------------------ replaying stand-ins
LANDMARK_PARTS = (("chin", 17), ("left_eyebrow", 5), ("right_eyebrow", 5), ("nose_bridge", 4), ("nose_tip", 5), ("left_eye", 6),
                  ("right_eye", 6), ("top_lip", 12), ("bottom_lip", 12))


def synth_landmarks(box, seed: int = 0) -> list:
    """face_recognition.face_landmarks' result for one face inside box (x1, y1, x2, y2): 72 integer points in its part order
    (chin along the lower half, nose bridge down the middle), as a one-element list."""
    x1, y1, x2, y2 = box
    rng = np.random.default_rng(seed)
    w, h = x2 - x1, y2 - y1
    pts = {}
    pts["chin"] = [(int(x1 + w * t), int(y1 + h * (0.5 + 0.5 * np.sin(np.pi * t)))) for t in np.linspace(0, 1, 17)]
    pts["nose_bridge"] = [(int(x1 + w / 2), int(y1 + h * (0.3 + 0.07 * k))) for k in range(4)]
    for name, n in LANDMARK_PARTS:
        if name not in pts:
            pts[name] = [(int(x1 + w * rng.uniform(0.15, 0.85)), int(y1 + h * rng.uniform(0.25, 0.85))) for _ in range(n)]
    return [pts]


class ReplayLandmarks:
    """face_recognition.face_landmarks stand-in: returns the recorded results in call order."""

    def __init__(self, results):
        self.results, self.i = list(results), 0

    def __call__(self, img_rgb, *a, **k):
        r = self.results[self.i]
        self.i += 1
        return r
