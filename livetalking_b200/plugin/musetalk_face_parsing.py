"""MuseTalk face parsing with BiSeNet on the engine: a drop-in for avatars/musetalk/utils/face_parsing.FaceParsing and the blend-mask
step of avatars/musetalk/utils/blending.py (get_image_prepare_material).

``FaceParsing`` keeps the reference's constructor arguments, model paths (under the working directory) and ``__call__`` returning a
PIL ``L`` image; ``parse_many`` runs many crops through one captured graph (livetalking_b200/bisenet.py) per batch.  The PIL resize
to 512 x 512 stays on the host (the reference's own call; the crops differ in size frame to frame), and so does the per-mode class
mapping, restated with the same cv2 / numpy operations: the jaw mode's cone-kernel dilation, cheek-ellipse erosion and cheek mask.

Weights: ``./models/face-parse-bisent/79999_iter.pth`` holds every BiSeNet parameter; the ResNet-18 file the reference loads first is
overwritten by it, so it is not read.  A missing file raises FileNotFoundError; nothing is downloaded."""
from __future__ import annotations

import logging
import os
import threading
from typing import Callable, List, Optional, Sequence

import numpy as np

logger = logging.getLogger(__name__)

MODEL_PTH = "./models/face-parse-bisent/79999_iter.pth"
_NETS = {}
_NETS_LOCK = threading.Lock()


def load_net(model_pth: str = MODEL_PTH):
    """BiSeNetNet for the weights file, loaded once per path."""
    path = os.path.abspath(model_pth)
    if not os.path.isfile(path):
        raise FileNotFoundError(f"BiSeNet weights not found at {path}: place the reference's 79999_iter.pth there (they are never "
                                "downloaded)")
    with _NETS_LOCK:
        if path not in _NETS:
            import torch
            from ..bisenet import BiSeNetNet
            _NETS[path] = BiSeNetNet.from_state_dict(torch.load(path, map_location="cpu", weights_only=True))
        return _NETS[path]


def cone_kernel() -> np.ndarray:
    """FaceParsing.__init__'s dilation kernel, built as the reference builds it."""
    cone_height, tail_height = 21, 12
    total_size = cone_height + tail_height
    kernel = np.zeros((total_size, total_size), dtype=np.uint8)
    center_x = total_size // 2
    for row in range(cone_height):
        if row < cone_height // 2:
            continue
        width = int(2 * (row - cone_height // 2) + 1)
        start = int(center_x - (width // 2))
        end = int(center_x + (width // 2) + 1)
        kernel[row, start:end] = 1
    base_width = int(kernel[cone_height - 1].sum()) if cone_height > 0 else 1
    for row in range(cone_height, total_size):
        start = max(0, int(center_x - (base_width // 2)))
        end = min(total_size, int(center_x + (base_width // 2) + 1))
        kernel[row, start:end] = 1
    return kernel


def create_cheek_mask(left_cheek_width=80, right_cheek_width=80) -> np.ndarray:
    import cv2
    mask = np.zeros((512, 512), dtype=np.uint8)
    center = 512 // 2
    cv2.rectangle(mask, (0, 0), (center - left_cheek_width, 512), 255, -1)
    cv2.rectangle(mask, (center + right_cheek_width, 0), (512, 512), 255, -1)
    return mask


def labels_to_mask(parsing: np.ndarray, mode: str, kernel: np.ndarray, cheek_kernel: np.ndarray, cheek_mask: np.ndarray) -> np.ndarray:
    """FaceParsing.__call__'s class mapping of one [512, 512] label map -> u8 0 / 255 (modes 'neck', 'jaw', anything else = 'raw')."""
    import cv2
    parsing = np.asarray(parsing).astype(np.int64)
    if mode == "neck":
        parsing[np.isin(parsing, [1, 11, 12, 13, 14])] = 255
        parsing[np.where(parsing != 255)] = 0
    elif mode == "jaw":
        face_region = np.isin(parsing, [1]) * 255
        face_region = face_region.astype(np.uint8)
        original_dilated = cv2.dilate(face_region, kernel, iterations=1)
        eroded = cv2.erode(original_dilated, cheek_kernel, iterations=2)
        face_region = cv2.bitwise_and(eroded, cheek_mask)
        face_region = cv2.bitwise_or(face_region, cv2.bitwise_and(original_dilated, ~cheek_mask))
        parsing[(face_region == 255) & (~np.isin(parsing, [10]))] = 255
        parsing[np.isin(parsing, [11, 12, 13])] = 255
        parsing[np.where(parsing != 255)] = 0
    else:
        parsing[np.isin(parsing, [1, 11, 12, 13])] = 255
        parsing[np.where(parsing != 255)] = 0
    return parsing.astype(np.uint8)


class FaceParsing:
    """face_parsing.FaceParsing on the engine.  make_parser(N) -> an object with parse(rgb_u8 [n <= N, 512, 512, 3]) -> u8 labels
    and close() (default: BiSeNetParser over the weights at MODEL_PTH); batch_size: crops per graph replay."""

    def __init__(self, left_cheek_width=80, right_cheek_width=80, make_parser: Optional[Callable] = None, batch_size: int = 16):
        if make_parser is None:
            self.net = self.model_init()
            make_parser = self._engine_parser
        self._make_parser, self.batch_size = make_parser, int(batch_size)
        self._parser, self._parser_n = None, 0
        self.kernel = cone_kernel()
        import cv2
        self.cheek_kernel = cv2.getStructuringElement(cv2.MORPH_ELLIPSE, (35, 3))
        self.cheek_mask = create_cheek_mask(left_cheek_width=left_cheek_width, right_cheek_width=right_cheek_width)

    def model_init(self, resnet_path='./models/face-parse-bisent/resnet18-5c106cde.pth', model_pth=MODEL_PTH):
        return load_net(model_pth)

    def _engine_parser(self, N):
        from ..bisenet import BiSeNetParser
        return BiSeNetParser(self.net, N)

    def labels(self, rgb512: np.ndarray) -> np.ndarray:
        """u8 RGB [n, 512, 512, 3] -> u8 labels [n, 512, 512], batch_size crops per replay; the batch is halved when the device
        cannot allocate a parser of that size."""
        out = []
        i = 0
        while i < len(rgb512):
            n = min(self.batch_size, len(rgb512) - i)
            if self._parser is None or self._parser_n < n:
                self.close()
                try:
                    self._parser = self._make_parser(n)
                    self._parser_n = n
                except RuntimeError:
                    if self.batch_size == 1:
                        raise
                    self.batch_size //= 2
                    logger.warning("recovering from a device allocation failure; face parsing batch size: %d", self.batch_size)
                    continue
            out.append(self._parser.parse(rgb512[i:i + n]))
            i += n
        return np.concatenate(out, 0) if out else np.zeros((0, 512, 512), np.uint8)

    def parse_many(self, images: Sequence, mode: str = "raw", size=(512, 512)) -> List:
        """__call__ over a list of PIL images (or paths), parsed in batches."""
        from PIL import Image
        imgs = [Image.open(im) if isinstance(im, str) else im for im in images]
        rgb = np.stack([np.asarray(im.resize(size, Image.BILINEAR).convert("RGB")) for im in imgs]) if imgs else np.zeros((0, 512, 512, 3), np.uint8)
        if rgb.shape[1:3] != (512, 512):
            raise ValueError(f"BiSeNet on the engine parses 512 x 512 crops, not {size}")
        return [Image.fromarray(labels_to_mask(lab, mode, self.kernel, self.cheek_kernel, self.cheek_mask)) for lab in self.labels(rgb)]

    def __call__(self, image, size=(512, 512), mode="raw"):
        return self.parse_many([image], mode=mode, size=size)[0]

    def close(self):
        if self._parser is not None:
            self._parser.close()
            self._parser, self._parser_n = None, 0


# ------------------------------------------------------------------------------------------------ blending.py
def get_crop_box(box, expand):
    x, y, x1, y1 = box
    x_c, y_c = (x + x1) // 2, (y + y1) // 2
    w, h = x1 - x, y1 - y
    s = int(max(w, h) // 2 * expand)
    crop_box = [x_c - s, y_c - s, x_c + s, y_c + s]
    return crop_box, s


def crop_for_parsing(image, face_box, expand=1.5):
    """First half of get_image_prepare_material: (face_large PIL crop of the body, crop_box)."""
    from PIL import Image
    body = Image.fromarray(image[:, :, ::-1])
    crop_box, _ = get_crop_box(face_box, expand)
    return body.crop(crop_box), crop_box


def finish_material(face_large, seg_image, face_box, crop_box, upper_boundary_ratio=0.5):
    """Second half of get_image_prepare_material, from the parser's mask of face_large: (blurred mask u8 [h, w], crop_box)."""
    import cv2
    from PIL import Image
    x, y, x1, y1 = face_box
    x_s, y_s, x_e, y_e = crop_box
    ori_shape = face_large.size
    mask_image = seg_image.resize(face_large.size)
    mask_small = mask_image.crop((x - x_s, y - y_s, x1 - x_s, y1 - y_s))
    mask_image = Image.new('L', ori_shape, 0)
    mask_image.paste(mask_small, (x - x_s, y - y_s, x1 - x_s, y1 - y_s))
    width, height = mask_image.size
    top_boundary = int(height * upper_boundary_ratio)
    modified_mask_image = Image.new('L', ori_shape, 0)
    modified_mask_image.paste(mask_image.crop((0, top_boundary, width, height)), (0, top_boundary))
    blur_kernel_size = int(0.1 * ori_shape[0] // 2 * 2) + 1
    mask_array = cv2.GaussianBlur(np.array(modified_mask_image), (blur_kernel_size, blur_kernel_size), 0)
    return mask_array, crop_box


def get_image_prepare_material(image, face_box, upper_boundary_ratio=0.5, expand=1.5, fp=None, mode="raw"):
    """blending.get_image_prepare_material, operation for operation."""
    face_large, crop_box = crop_for_parsing(image, face_box, expand)
    return finish_material(face_large, fp(face_large, mode=mode), face_box, crop_box, upper_boundary_ratio)


def prepare_materials(images, face_boxes, fp: FaceParsing, mode="raw", upper_boundary_ratio=0.5, expand=1.5):
    """get_image_prepare_material over many frames with one parse_many call: [(mask, crop_box)] in frame order."""
    crops = [crop_for_parsing(im, box, expand) for im, box in zip(images, face_boxes)]
    segs = fp.parse_many([c[0] for c in crops], mode=mode)
    return [finish_material(c[0], s, box, c[1], upper_boundary_ratio) for c, s, box in zip(crops, segs, face_boxes)]
