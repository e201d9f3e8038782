"""Host-side mirror of the reference's avatar plugin surface (avatars/base_avatar.py) for the H100 engine.

    plugin.base_asr        <-> avatars/audio_features/base_asr.py   (queues, silence synthesis, warm-up)
    plugin.mel_asr         <-> avatars/audio_features/mel.py        (MelASR.run_step, features from the GPU mel kernels)
    plugin.wav2lip_avatar  <-> avatars/wav2lip_avatar.py            (load_model / load_avatar / warm_up / LipReal)
    plugin.whisper_asr     <-> avatars/audio_features/whisper.py    (WhisperASR.run_step)
    plugin.musetalk_avatar <-> avatars/musetalk_avatar.py           (load_model / load_avatar / warm_up / MuseReal)
    plugin.hubert_asr      <-> avatars/audio_features/hubert.py     (HubertASR.run_step)
    plugin.ultralight_avatar <-> avatars/ultralight_avatar.py       (load_model / load_avatar / warm_up / LightReal)
    plugin.batcher         — cross-session batching scheduler shared by the avatar classes (SURVEY 8 f1)

`python -m livetalking_b200.run_app <app.py args>` aliases these modules over the reference's and runs the
reference's app.py unchanged (see INTEGRATION.md)."""
