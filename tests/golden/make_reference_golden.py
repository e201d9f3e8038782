"""Record what the reference's own classes produce on the event sequences of tests/test_plugin_host.py and
tests/test_oracle_paste.py -> tests/golden/reference_host_golden.json.  Needs a LiveTalking checkout:

    LTB_REFERENCE=/path/to/LiveTalking python tests/golden/make_reference_golden.py

Audio frames are stored as the index of the seeded input chunk they equal (-1: all zeros, i.e. synthesised silence);
composited frames as the SHA-256 of their bytes (the tests compare bit-exactly)."""
import hashlib
import importlib.util
import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import stubs  # noqa: E402

stubs.install()
REF = os.environ.get("LTB_REFERENCE", "")


def load(name, rel):
    spec = importlib.util.spec_from_file_location(name, os.path.join(REF, rel))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def feed(asr, n, seed):
    rng = np.random.default_rng(seed)
    chunks = [rng.standard_normal(320).astype(np.float32) for _ in range(n)]
    for i, c in enumerate(chunks):
        asr.put_audio_frame(c, {"i": i})
    return chunks


def index(a, chunks):
    a = np.asarray(a, np.float32)
    if not a.any():
        return -1
    return next(i for i, c in enumerate(chunks) if np.array_equal(a, c))


def pcm_indices(pcm, chunks):
    return [index(p, chunks) for p in np.asarray(pcm, np.float32).reshape(-1, 320)]


def drain(q, chunks):
    return [[int(f.type), index(f.data, chunks)] for f in (q.get() for _ in range(q.qsize()))]


def base_asr():
    ref = load("ref_base_asr", "avatars/audio_features/base_asr.py")
    asr = ref.BaseASR(stubs.Opt(batch_size=3))
    chunks = feed(asr, 23, 5)
    asr.warm_up()
    frames = [asr.get_audio_frame() for _ in range(8)]
    return {"get_audio_frame": [[int(f.type), index(f.data, chunks), f.userdata.get("i") if f.userdata else None] for f in frames],
            "output_queue_size": asr.output_queue.qsize(), "frames": [index(f, chunks) for f in asr.frames]}


def ref_base_as_package():
    base = load("ref_base_asr_pkg", "avatars/audio_features/base_asr.py")
    af = types.ModuleType("avatars.audio_features")
    af.__path__ = []
    sys.modules["avatars.audio_features"] = af
    sys.modules["avatars.audio_features.base_asr"] = base


def whisper_asr():
    a2f = types.ModuleType("avatars.musetalk.whisper.audio2feature")
    a2f.Audio2Feature = object
    for name in ("avatars.musetalk", "avatars.musetalk.whisper"):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.modules["avatars.musetalk.whisper.audio2feature"] = a2f
    ref_base_as_package()
    ref = load("ref_whisper_asr", "avatars/audio_features/whisper.py")

    class Recorder:
        calls = []

        def audio2feat(self, pcm):
            self.calls.append(np.asarray(pcm).copy())
            return np.zeros((1500, 5, 384), np.float32)

    B, rec = 3, Recorder()
    asr = ref.WhisperASR(stubs.Opt(batch_size=B), None, rec)
    chunks = feed(asr, 20 + 2 * B + 2, 2)
    asr.warm_up()
    asr.run_step()
    feats = asr.feat_queue.get()
    return {"feat_shapes": [list(np.asarray(f).shape) for f in feats], "calls": [pcm_indices(c, chunks) for c in rec.calls],
            "frames": [index(f, chunks) for f in asr.frames], "output_queue": drain(asr.output_queue, chunks)}


def hubert_asr():
    a2f = types.ModuleType("avatars.ultralight.audio2feature")
    a2f.Audio2Feature = object
    sys.modules.setdefault("avatars.ultralight", types.ModuleType("avatars.ultralight"))
    sys.modules["avatars.ultralight.audio2feature"] = a2f
    ref_base_as_package()
    ref = load("ref_hubert_asr", "avatars/audio_features/hubert.py")

    class Recorder:
        calls = []

        def get_hubert_from_16k_speech(self, pcm):
            self.calls.append(np.asarray(pcm).copy())
            return np.ones(((len(pcm) - 80) // 320, 1024), np.float32)

    B, rec = 3, Recorder()
    asr = ref.HubertASR(stubs.Opt(batch_size=B), None, rec, audio_feat_length=[4, 4])
    chunks = feed(asr, 20 + 2 * B, 4)
    asr.warm_up()
    shapes = []
    for _ in range(3):
        asr.run_step()
        shapes.append([list(np.asarray(f).shape) for f in asr.feat_queue.get()])
    return {"feat_shapes": shapes, "calls": [pcm_indices(c, chunks) for c in rec.calls], "last_is_silence": bool(asr.last_is_silence),
            "frames": [index(f, chunks) for f in asr.frames], "output_queue": drain(asr.output_queue, chunks)}


def musetalk_blend():
    import cv2
    sys.path.insert(0, os.path.dirname(HERE))
    from test_oracle_paste import blend_case
    ref = load("ref_myutil", "avatars/musetalk/myutil.py")
    frame, pred, bbox, crop, masks = blend_case(cv2)
    x1, y1, x2, y2 = bbox
    out = [ref.get_image_blending(frame.copy(), cv2.resize(pred, (x2 - x1, y2 - y1)), bbox, m, crop) for m in masks]
    return [hashlib.sha256(np.ascontiguousarray(o).tobytes()).hexdigest() for o in out]


if __name__ == "__main__":
    if not os.path.isfile(os.path.join(REF, "avatars", "base_avatar.py")):
        sys.exit("set LTB_REFERENCE to a LiveTalking checkout")
    golden = {"base_asr": base_asr(), "whisper_asr": whisper_asr(), "hubert_asr": hubert_asr(), "musetalk_blend_sha256": musetalk_blend()}
    with open(os.path.join(HERE, "reference_host_golden.json"), "w") as fh:
        json.dump(golden, fh, indent=1)
        fh.write("\n")
