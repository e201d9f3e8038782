"""Pack a reference wav2lip256 checkpoint ``state_dict`` into the engine's weight blob.

Input: the key scheme of the reference checkpoint (loaded at avatars/wav2lip_avatar.py:59-70):
``<block>.conv_block.0.{weight,bias}`` + ``<block>.conv_block.1.{weight,bias,running_mean,running_var}``
for the 54 Conv/ConvT+BN blocks, plus ``output_block.1.{weight,bias}``.

What happens here (once, at load time):
  * eval-mode BatchNorm (conv.py:8-11,36-39; eps 1e-5) is folded into the conv:  w' = w * g/sqrt(v+eps),
    b' = (b - mean) * g/sqrt(v+eps) + beta;
  * weights become fp16 K-major rows ``[Cout][tap][Cin]`` (the B operand of the implicit GEMM);
  * ConvTranspose2d(k3,s2,p1,op1) is rewritten as 4 sub-pixel phases (1+2+2+4 taps);
  * the 7x7 stem becomes 7 row-taps of 8 pixels x 8 channels (6 real + 2 zero);
  * ConvTranspose2d(1024,512,k4) on the 1x1 bottleneck becomes a 1x1 conv with 16*512 outputs.

Blob layout: 16-byte header ("LTBW2L1\\0", n_entries, header_bytes), n_entries x 64-byte records
(name[40], dtype u32 (0=f16, 1=f32), pad u32, offset u64, nbytes u64), then 256-byte aligned payloads.
"""
from __future__ import annotations

import struct
from typing import Dict, List, Tuple

import numpy as np

BN_EPS = 1e-5

# (prefix, kind, cin, cout, k) in execution order — wav2lip_v2.py:12-91
_AUDIO = [(1, 32, 3), (32, 32, 3), (32, 32, 3), (32, 64, 3), (64, 64, 3), (64, 64, 3), (64, 128, 3), (128, 128, 3),
          (128, 128, 3), (128, 256, 3), (256, 256, 3), (256, 512, 3), (512, 512, 1)]
_FACE_ENC = [[(6, 16, 7)], [(16, 32, 3), (32, 32, 3), (32, 32, 3)], [(32, 64, 3), (64, 64, 3), (64, 64, 3), (64, 64, 3)],
             [(64, 128, 3), (128, 128, 3), (128, 128, 3)], [(128, 256, 3), (256, 256, 3), (256, 256, 3)],
             [(256, 512, 3), (512, 512, 3)], [(512, 512, 3), (512, 512, 3)], [(512, 512, 4), (512, 512, 1)]]
_FACE_DEC = [[("c", 512, 512, 1)], [("t", 1024, 512, 4), ("c", 512, 512, 3)], [("t", 1024, 512, 3), ("c", 512, 512, 3)],
             [("t", 1024, 512, 3), ("c", 512, 512, 3), ("c", 512, 512, 3)],
             [("t", 768, 384, 3), ("c", 384, 384, 3), ("c", 384, 384, 3)],
             [("t", 512, 256, 3), ("c", 256, 256, 3), ("c", 256, 256, 3)],
             [("t", 320, 128, 3), ("c", 128, 128, 3), ("c", 128, 128, 3)],
             [("t", 160, 64, 3), ("c", 64, 64, 3), ("c", 64, 64, 3)]]

STEM_LAYER = 13
CONVT4_LAYER = 34


def layer_table() -> List[Tuple[str, str, int, int, int]]:
    out = []
    for i, (ci, co, k) in enumerate(_AUDIO):
        out.append((f"audio_encoder.{i}", "c", ci, co, k))
    for b, blk in enumerate(_FACE_ENC):
        for j, (ci, co, k) in enumerate(blk):
            out.append((f"face_encoder_blocks.{b}.{j}", "c", ci, co, k))
    for b, blk in enumerate(_FACE_DEC):
        for j, (kind, ci, co, k) in enumerate(blk):
            out.append((f"face_decoder_blocks.{b}.{j}", kind, ci, co, k))
    out.append(("output_block.0", "c", 80, 32, 3))
    assert len(out) == 54
    return out


def _np(t) -> np.ndarray:
    if hasattr(t, "detach"):
        t = t.detach().cpu().numpy()
    return np.asarray(t, dtype=np.float64)


# sub-pixel phase taps of ConvTranspose2d(k=3,s=2,p=1,op=1): out[2g+a] = sum over (d, k):
#   a=0: (d=0,k=1)       a=1: (d=0,k=2), (d=+1,k=0)      (must match kTd / kTk in csrc/conv_plan.cu)
_T_TAPS = {0: [(0, 1)], 1: [(0, 2), (1, 0)]}


def pack_conv(w: np.ndarray) -> np.ndarray:
    """[Cout,Cin,KH,KW] -> [Cout, KH*KW*Cin] (tap-major, channel-minor)."""
    co, ci, kh, kw = w.shape
    return np.ascontiguousarray(w.transpose(0, 2, 3, 1)).reshape(co, kh * kw * ci)


def pack_convT_s2(w: np.ndarray) -> np.ndarray:
    """ConvTranspose2d weight [Cin,Cout,3,3] -> [Cout, 9*Cin] in phase order (0,0),(0,1),(1,0),(1,1)."""
    ci, co, _, _ = w.shape
    cols = []
    for a in (0, 1):
        for b in (0, 1):
            for (_, kh) in _T_TAPS[a]:
                for (_, kw) in _T_TAPS[b]:
                    cols.append(w[:, :, kh, kw].T)  # [Cout, Cin]
    return np.ascontiguousarray(np.concatenate(cols, axis=1))


def pack_stem(w: np.ndarray) -> np.ndarray:
    """[16,6,7,7] -> [16, 7*64]: K index = kh*64 + kw*8 + c (kw<7, c<6), zeros elsewhere."""
    co = w.shape[0]
    out = np.zeros((co, 7, 8, 8), dtype=w.dtype)
    out[:, :, :7, :6] = w.transpose(0, 2, 3, 1)
    return out.reshape(co, 7 * 64)


def pack_convT4(w: np.ndarray) -> np.ndarray:
    """ConvTranspose2d(1024,512,k4,s1,p0) on a 1x1 map: [Cin,Cout,4,4] -> [(oy*4+ox)*512+co, Cin]."""
    ci, co, kh, kw = w.shape
    return np.ascontiguousarray(w.transpose(2, 3, 1, 0)).reshape(kh * kw * co, ci)


def fold_bn(sd: Dict, prefix: str, kind: str) -> Tuple[np.ndarray, np.ndarray]:
    w = _np(sd[f"{prefix}.conv_block.0.weight"])
    b = _np(sd[f"{prefix}.conv_block.0.bias"])
    g = _np(sd[f"{prefix}.conv_block.1.weight"])
    beta = _np(sd[f"{prefix}.conv_block.1.bias"])
    mean = _np(sd[f"{prefix}.conv_block.1.running_mean"])
    var = _np(sd[f"{prefix}.conv_block.1.running_var"])
    scale = g / np.sqrt(var + BN_EPS)
    if kind == "c":
        w = w * scale[:, None, None, None]
    else:  # ConvTranspose2d weight is [Cin, Cout, kh, kw]
        w = w * scale[None, :, None, None]
    return w, (b - mean) * scale + beta


def pack_state_dict(sd: Dict) -> bytes:
    """Reference state_dict (torch tensors or arrays; optional 'module.' prefixes) -> weight blob bytes."""
    sd = {k.replace("module.", ""): v for k, v in sd.items()}
    entries: List[Tuple[str, int, np.ndarray]] = []
    for i, (prefix, kind, ci, co, k) in enumerate(layer_table()):
        w, b = fold_bn(sd, prefix, kind)
        expect = (co, ci, k, k) if kind == "c" else (ci, co, k, k)
        if tuple(w.shape) != expect:
            raise ValueError(f"{prefix}: weight shape {tuple(w.shape)} != {expect}")
        if i == 0:
            entries.append((f"L{i:02d}.w", 1, w.reshape(32, 9).astype(np.float32)))
        elif i == STEM_LAYER:
            entries.append((f"L{i:02d}.w", 0, pack_stem(w).astype(np.float16)))
        elif i == CONVT4_LAYER:
            entries.append((f"L{i:02d}.w", 0, pack_convT4(w).astype(np.float16)))
            b = np.tile(b, 16)
        elif kind == "t":
            entries.append((f"L{i:02d}.w", 0, pack_convT_s2(w).astype(np.float16)))
        else:
            entries.append((f"L{i:02d}.w", 0, pack_conv(w).astype(np.float16)))
        entries.append((f"L{i:02d}.b", 1, b.astype(np.float32)))
    entries.append(("head.w", 1, _np(sd["output_block.1.weight"]).reshape(3, 32).astype(np.float32)))
    entries.append(("head.b", 1, _np(sd["output_block.1.bias"]).astype(np.float32)))

    header_bytes = 16 + 64 * len(entries)
    off = (header_bytes + 255) // 256 * 256
    recs = []
    payload = []
    for name, dtype, arr in entries:
        raw = np.ascontiguousarray(arr).tobytes()
        recs.append(struct.pack("<40sIIQQ", name.encode(), dtype, 0, off, len(raw)))
        payload.append((off, raw))
        off = (off + len(raw) + 255) // 256 * 256
    blob = bytearray(off)
    blob[0:16] = struct.pack("<8sII", b"LTBW2L1\0", len(entries), header_bytes)
    blob[16:16 + 64 * len(entries)] = b"".join(recs)
    for o, raw in payload:
        blob[o:o + len(raw)] = raw
    return bytes(blob)
