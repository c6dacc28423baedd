"""kantts_b200 -- H100-native (sm_90a) implementation of KAN-TTS's HiFi-GAN hot path.

Public surface = the reference's own module API for this path:
  hifigan.Generator / MultiPeriodDiscriminator / MultiScaleDiscriminator   (kantts.models)
    / SpecDiscriminator / MultiSpecDiscriminator
  pqmf.PQMF (the multi-band generator's filter bank)                      (kantts.models.pqmf)
  audio.MelSpectrogram / stft                                             (kantts.utils.audio_torch)
  loss.* + criterion_builder                                              (kantts.train.loss)
  train.GanStep (GAN_Trainer.train_step + the data-parallel gradient exchange)
  sambert.KanTtsSAMBERT + MelReconLoss / ProsodyReconLoss                  (kantts.models.sambert, kantts.train.loss)
  train.SambertStep (Sambert_Trainer.train_step); data.AttnPriors (the MAS data path's alignment prior)
  sambert.KanTtsTextsyBERT + SeqCELoss, train.SybertStep, data.BertMasker (sybert.yaml: masked-symbol pretraining)
  infer.synthesize (symbols -> SAM-BERT free-running decode -> HiFi-GAN -> waveforms, no .npy hand-off)
  infer.stream_synthesize (the same waveforms chunk by chunk while the decoder runs; non-causal generators with
    allow_lookahead=True)
  infer.TtsServer (continuous batching: requests join and leave the slots of one running stream)
  speaker.DTDNN / kaldi_fbank / speaker_embedding (kantts.preprocess.se_processor: the SE flow's speaker embeddings)
  install.install() patches these into an importable KAN-TTS checkout.
All tensor math runs in libkantts_b200.so (C ABI: include/kantts_b200.h); there is no fallback.
"""
from . import _lib  # noqa: F401
from ._lib import build_library  # noqa: F401
from . import ops, hifigan, pqmf, audio, loss, sambert_ops, sambert, train, infer, speaker, install as _install  # noqa: F401
from .sambert import (KanTtsSAMBERT, MelReconLoss, ProsodyReconLoss, FpCELoss, AttentionCTCLoss,  # noqa: F401
                      AttentionBinarizationLoss, ConvAttention, KanTtsTextsyBERT, SeqCELoss)
from .hifigan import (Generator, MultiPeriodDiscriminator, MultiScaleDiscriminator, SpecDiscriminator,  # noqa: F401
                      MultiSpecDiscriminator, set_precision)
from .pqmf import PQMF  # noqa: F401
from .audio import MelSpectrogram, stft  # noqa: F401
from .loss import (MelSpectrogramLoss, MultiResolutionSTFTLoss, GeneratorAdversarialLoss,  # noqa: F401
                   DiscriminatorAdversarialLoss, FeatureMatchLoss, criterion_builder)
from .train import (GanStep, SambertStep, SybertStep, hifigan_model_builder, sambert_model_builder,  # noqa: F401
                    sybert_model_builder)
from .data import AttnPriors, BertMasker  # noqa: F401
from .infer import synthesize, stream_synthesize, TtsServer, slot_schedule  # noqa: F401
from .speaker import DTDNN, kaldi_fbank, speaker_embedding  # noqa: F401



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


def sambert_fp_8k_config():
    """``Model.KanTtsSAMBERT.params`` of kantts/configs/sambert_fp_8k.yaml: the sambert_24k.yaml network with the
    filled-pause predictor (``FP: True``) and the yaml's six speakers."""
    return dict(sambert_24k_config(), FP=True, speaker=6)


def sambert_16k_mas_config():
    """``Model.KanTtsSAMBERT.params`` of kantts/configs/sambert_16k_MAS.yaml: the sambert_24k.yaml network that learns its
    phone durations by monotonic alignment search (``MAS: True``), with the same linguistic units."""
    return dict(sambert_24k_config(), MAS=True)


def sambert_16k_mas_byte_config():
    """``Model.KanTtsSAMBERT.params`` of kantts/configs/sambert_16k_MAS_byte.yaml: the MAS network on byte inputs
    (``using_byte: True``, lfeat_type_list byte_index,emo_category,speaker_category): ``byte_index`` = 259 embeddings, the
    256 byte values plus padding, end-of-sentence and mask, in place of the PinYin tables."""
    cfg = {k: v for k, v in sambert_16k_mas_config().items() if k not in ("sy", "tone", "syllable_flag", "word_segment")}
    return dict(cfg, using_byte=True, byte_index=259)


def sambert_se_nsf_global_16k_config():
    """``Model.KanTtsSAMBERT.params`` of kantts/configs/sambert_se_nsf_global_16k.yaml: the sambert_24k.yaml network driven
    by a 192-d speaker embedding per symbol (``SE: True``, no speaker table) with NSF outputs (80 mels + f0 + voiced flag,
    f0 normalised globally to [30, 730] Hz), and the PinYin unit sizes."""
    cfg = {k: v for k, v in sambert_24k_config().items() if k != "speaker"}
    return dict(cfg, speaker_units=192, num_mels=82, NSF=True, nsf_norm_type="global", nsf_f0_global_minimum=30.0,
                nsf_f0_global_maximum=730.0, SE=True)


def sybert_config():
    """``Model.KanTtsTextsyBERT.params`` of kantts/configs/sybert.yaml plus the PinYin unit sizes the trainer injects
    (bin/train_sybert.py:129-131), as sambert_24k_config.  The sy table ends with pad, eos and the mask symbol, so the mask
    id is ``sy - 1``."""
    return dict(
        max_len=800, embedding_dim=512, encoder_num_layers=8, encoder_num_heads=8, encoder_num_units=128,
        encoder_ffn_inner_dim=1024, encoder_dropout=0.1, encoder_attention_dropout=0.1, encoder_relu_dropout=0.1,
        encoder_projection_units=32, mask_ratio=0.3, sy=147, tone=10, syllable_flag=8, word_segment=8)


install = _install.install
__version__ = "0.1.0"
