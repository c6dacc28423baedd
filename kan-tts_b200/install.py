"""Patch the H100-native classes into an importable KAN-TTS checkout so that its unchanged
``kantts/bin/train_hifigan.py`` / ``kantts.train.trainer.GAN_Trainer`` run on them
(see INTEGRATION.md).  ``model_builder`` looks classes up by name in ``kantts.models``' globals
(kantts/models/__init__.py:38,51,131) and ``criterion_builder`` in ``loss_dict`` (loss.py:512-544): the syBERT builder
finds ``KanTtsTextsyBERT`` there and its SeqCELoss arrives through ``loss_dict``.  The speaker-embedding
processor (kantts/preprocess/se_processor/se_processor.py) builds its model as ``DTDNN()`` from its module globals, so
replacing that name runs the unchanged ``SpeakerEmbeddingProcessor`` on speaker.DTDNN."""
import sys


def _with_precision(cls, precision):
    """-> a subclass of HiFi-GAN module class ``cls`` whose instances are built in tensor-core ``precision``
    (hifigan.set_precision), under the same name: the reference's model builder constructs it unchanged."""
    from .hifigan import set_precision

    def __init__(self, *args, **kwargs):
        cls.__init__(self, *args, **kwargs)
        set_precision(self, precision)
    return type(cls.__name__, (cls,), {"__init__": __init__, "__module__": cls.__module__, "__qualname__": cls.__qualname__})


def install(kantts_models=None, kantts_loss=None, kantts_audio=None, kantts_se=None, kantts_dataset=None, precision=None):
    """``precision`` ("bf16" or "bf16x3"; None: the default bf16x3): the tensor-core precision of every HiFi-GAN model and
    PQMF the patched checkout builds, so that its unchanged GAN_Trainer trains in single-pass bf16 with "bf16".

    ``kantts_se``: the speaker-embedding processor module to patch; by default
    kantts.preprocess.se_processor.se_processor when it is already imported.  It is never imported here: it needs
    torchaudio and configures logging at import, which the HiFi-GAN and SAM-BERT flows do not want.

    ``kantts_dataset``: the dataset module (kantts.datasets.dataset) whose ``beta_binomial_prior_distribution`` becomes
    ``data.attn_prior_placeholder``, for a MAS run whose batches go through ``data.AttnPriors`` on the device.  Patched
    only when passed: without that transform the placeholder's NaN prior would reach the model."""
    from . import audio, data, hifigan, loss, pqmf, sambert, speaker
    if precision is not None and precision not in hifigan.PRECISIONS:
        raise ValueError(f"install: precision must be one of {sorted(hifigan.PRECISIONS)}, got {precision!r}")
    wrap = (lambda cls: cls) if precision is None else (lambda cls: _with_precision(cls, precision))
    if kantts_models is None:
        import kantts.models as kantts_models
    if kantts_loss is None:
        import kantts.train.loss as kantts_loss
    if kantts_audio is None:
        import kantts.utils.audio_torch as kantts_audio
    for name in ("Generator", "MultiPeriodDiscriminator", "MultiScaleDiscriminator", "SpecDiscriminator",
                 "MultiSpecDiscriminator"):
        cls = wrap(getattr(hifigan, name))
        setattr(kantts_models, name, cls)
        if hasattr(kantts_models, "hifigan") and hasattr(kantts_models.hifigan, "hifigan"):
            setattr(kantts_models.hifigan.hifigan, name, cls)
    kantts_models.KanTtsTextsyBERT = sambert.KanTtsTextsyBERT
    pqmf_cls = wrap(pqmf.PQMF)
    kantts_models.PQMF = pqmf_cls                            # hifigan_model_builder (kantts/models/__init__.py:65-67)
    if hasattr(kantts_models, "pqmf"):                       # infer_hifigan.py:50-52 imports it from there
        kantts_models.pqmf.PQMF = pqmf_cls
    for key, cls in loss.loss_dict.items():
        kantts_loss.loss_dict[key] = cls
        setattr(kantts_loss, cls.__name__, cls)
    kantts_audio.MelSpectrogram = audio.MelSpectrogram
    kantts_audio.stft = audio.stft
    if kantts_se is None:
        kantts_se = sys.modules.get("kantts.preprocess.se_processor.se_processor")
    if kantts_se is not None:
        kantts_se.DTDNN = speaker.DTDNN
    if kantts_dataset is not None:
        kantts_dataset.beta_binomial_prior_distribution = data.attn_prior_placeholder
    return kantts_models
