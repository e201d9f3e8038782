"""WhisperASR on the B200 engine — drop-in for avatars/audio_features/whisper.py:30-76.

Same bookkeeping as the reference's ``run_step`` (2*B chunks forwarded to ``output_queue``, one list of B (50, 384) feature
arrays queued, l+r chunks of context kept); ``audio2feat`` + ``_feature2chunks`` are one CUDA-graph launch
(livetalking_b200/whisper.py)."""
from __future__ import annotations

import numpy as np

from .base_asr import BaseASR, fixed_chunk


class WhisperASR(BaseASR):
    def __init__(self, opt, parent, audio_processor):
        super().__init__(opt, parent)
        self.audio_processor = audio_processor          # whisper.WhisperFeatures, or batcher.SharedFeatures in cross-session mode
        if audio_processor is None:
            raise RuntimeError("WhisperASR needs an engine WhisperFeatures object (no CPU fallback)")

    def run_step(self):
        for _ in range(self.batch_size * 2):
            audio_frame = self.get_audio_frame()
            audio_frame.data = fixed_chunk(audio_frame.data, self.chunk)    # short tail chunk of a custom-action clip
            self.frames.append(audio_frame.data)
            self.output_queue.put(audio_frame)
        if len(self.frames) <= self.stride_left_size + self.stride_right_size:
            return
        inputs = np.concatenate(self.frames)
        n_expected = (self.stride_left_size + self.stride_right_size + 2 * self.batch_size) * self.chunk
        if inputs.size != n_expected:                  # run_step before warm_up(): no features yet, as the early return above
            return
        feats = self.audio_processor.run(inputs.astype(np.float32, copy=False))       # (B, 50, 384) float16
        self.feat_queue.put([feats[i] for i in range(self.batch_size)])
        self.frames = self.frames[-(self.stride_left_size + self.stride_right_size):]
