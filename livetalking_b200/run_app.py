"""Run the reference's app.py UNCHANGED on the B200 engine:

    cd /path/to/LiveTalking && PYTHONPATH=/path/to/this/repo python -m livetalking_b200.run_app --model wav2lip ...

app.py picks the avatar module by a hard-coded map (app.py:128-134: 'avatars.wav2lip_avatar', ...).  We pre-import the
reference's host-side modules and then alias our plugin modules under those names, so `importlib.import_module` in
app.py resolves to the engine-backed implementations and `@register("avatar","wav2lip")` registers our class."""
import importlib
import os
import runpy
import sys


def install_aliases():
    import avatars.base_avatar  # noqa: F401  (reference runtime must be importable: we are inside LiveTalking)
    for ours, theirs in (("livetalking_b200.plugin.wav2lip_avatar", "avatars.wav2lip_avatar"),
                         ("livetalking_b200.plugin.mel_asr", "avatars.audio_features.mel"),
                         ("livetalking_b200.plugin.musetalk_avatar", "avatars.musetalk_avatar"),
                         ("livetalking_b200.plugin.whisper_asr", "avatars.audio_features.whisper"),
                         ("livetalking_b200.plugin.ultralight_avatar", "avatars.ultralight_avatar"),
                         ("livetalking_b200.plugin.hubert_asr", "avatars.audio_features.hubert"),
                         ("livetalking_b200.plugin.wav2lip_genavatar", "avatars.wav2lip.genavatar"),
                         ("livetalking_b200.plugin.ultralight_genavatar", "avatars.ultralight.genavatar"),
                         ("livetalking_b200.plugin.musetalk_genavatar", "avatars.musetalk.genavatar")):
        sys.modules[theirs] = importlib.import_module(ours)


def main():
    sys.path.insert(0, os.getcwd())
    install_aliases()
    sys.argv = ["app.py"] + sys.argv[1:]
    runpy.run_path(os.path.join(os.getcwd(), "app.py"), run_name="__main__")


if __name__ == "__main__":
    main()
