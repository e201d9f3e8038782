"""livetalking_b200 — H100-native (sm_90a) lip-sync engine behind LiveTalking's avatar plugin surface.

Host code is Python over a thin C ABI (``include/ltb200.h`` -> ``lib/libltb200.so``); the hot path
(mel, wav2lip256 forward, paste-back) is hand-written CUDA.  There is no CPU fallback: importing the
binding without the built library raises.
"""
__version__ = "0.1.0"
