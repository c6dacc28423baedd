"""kantts_b200 -- H100-native (sm_90a) implementation of KAN-TTS's HiFi-GAN hot path.

Public surface = the reference's own module API for this path:
  hifigan.Generator / MultiPeriodDiscriminator / MultiScaleDiscriminator   (kantts.models)
  audio.MelSpectrogram / stft                                             (kantts.utils.audio_torch)
  loss.* + criterion_builder                                              (kantts.train.loss)
  train.GanStep (GAN_Trainer.train_step + the data-parallel gradient exchange)
  sambert.KanTtsSAMBERT + MelReconLoss / ProsodyReconLoss                  (kantts.models.sambert, kantts.train.loss)
  train.SambertStep (Sambert_Trainer.train_step)
  infer.synthesize (symbols -> SAM-BERT free-running decode -> HiFi-GAN -> waveforms, no .npy hand-off)
  install.install() patches these into an importable KAN-TTS checkout.
All tensor math runs in libkantts_b200.so (C ABI: include/kantts_b200.h); there is no fallback.
"""
from . import _lib  # noqa: F401
from ._lib import build_library  # noqa: F401
from . import ops, hifigan, audio, loss, sambert_ops, sambert, train, infer, install as _install  # noqa: F401
from .sambert import KanTtsSAMBERT, MelReconLoss, ProsodyReconLoss  # noqa: F401
from .hifigan import Generator, MultiPeriodDiscriminator, MultiScaleDiscriminator  # noqa: F401
from .audio import MelSpectrogram, stft  # noqa: F401
from .loss import (MelSpectrogramLoss, MultiResolutionSTFTLoss, GeneratorAdversarialLoss,  # noqa: F401
                   DiscriminatorAdversarialLoss, FeatureMatchLoss, criterion_builder)
from .train import GanStep, SambertStep, hifigan_model_builder, sambert_model_builder  # noqa: F401
from .infer import synthesize  # noqa: F401



def sambert_24k_config():
    """``Model.KanTtsSAMBERT.params`` of kantts/configs/sambert_24k.yaml plus the linguistic-unit table sizes the
    trainer injects for the PinYin / F7 setup (bin/train_sambert.py:144-146; SURVEY.md section 8d config C4)."""
    return dict(
        max_len=800, embedding_dim=512, encoder_num_layers=8, encoder_num_heads=8, encoder_num_units=128,
        encoder_ffn_inner_dim=1024, encoder_dropout=0.1, encoder_attention_dropout=0.1, encoder_relu_dropout=0.1,
        encoder_projection_units=32, speaker_units=32, emotion_units=32, predictor_filter_size=41,
        predictor_fsmn_num_layers=3, predictor_num_memory_units=128, predictor_ffn_inner_dim=256,
        predictor_dropout=0.1, predictor_shift=0, predictor_lstm_units=128, dur_pred_prenet_units=[128, 128],
        dur_pred_lstm_units=128, decoder_prenet_units=[256, 256], decoder_num_layers=12, decoder_num_heads=8,
        decoder_num_units=128, decoder_ffn_inner_dim=1024, decoder_dropout=0.1, decoder_attention_dropout=0.1,
        decoder_relu_dropout=0.1, outputs_per_step=3, num_mels=80, postnet_filter_size=41,
        postnet_fsmn_num_layers=4, postnet_num_memory_units=256, postnet_ffn_inner_dim=512, postnet_dropout=0.1,
        postnet_shift=17, postnet_lstm_units=128, MAS=False,
        sy=147, tone=10, syllable_flag=8, word_segment=8, emotion=36, speaker=4)


install = _install.install
__version__ = "0.1.0"
