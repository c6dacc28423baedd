"""Patch the H100-native classes into an importable KAN-TTS checkout so that its unchanged
``kantts/bin/train_hifigan.py`` / ``kantts.train.trainer.GAN_Trainer`` run on them
(see INTEGRATION.md).  ``model_builder`` looks classes up by name in ``kantts.models``' globals
(kantts/models/__init__.py:38,51) and ``criterion_builder`` in ``loss_dict`` (loss.py:512-544)."""


def install(kantts_models=None, kantts_loss=None, kantts_audio=None):
    from . import audio, hifigan, loss
    if kantts_models is None:
        import kantts.models as kantts_models
    if kantts_loss is None:
        import kantts.train.loss as kantts_loss
    if kantts_audio is None:
        import kantts.utils.audio_torch as kantts_audio
    for name in ("Generator", "MultiPeriodDiscriminator", "MultiScaleDiscriminator"):
        setattr(kantts_models, name, getattr(hifigan, name))
        if hasattr(kantts_models, "hifigan") and hasattr(kantts_models.hifigan, "hifigan"):
            setattr(kantts_models.hifigan.hifigan, name, getattr(hifigan, name))
    for key, cls in loss.loss_dict.items():
        kantts_loss.loss_dict[key] = cls
        setattr(kantts_loss, cls.__name__, cls)
    kantts_audio.MelSpectrogram = audio.MelSpectrogram
    kantts_audio.stft = audio.stft
    return kantts_models
