"""Writes tests/golden/se_dtdnn.npz and tests/golden/se_dtdnn_init_checksums.json from the unmodified reference speaker
encoder (kantts/preprocess/se_processor) and torchaudio:
  - three seeded 16 kHz wavs of 8000, 32160 and 52800 samples: 48, 199 and 328 fbank frames, so 24 (shorter than one
    100-row gating segment), 100 (exactly one) and 164 (a partial last segment) rows after the stride-2 TDNN;
  - their torchaudio.compliance.kaldi.fbank(wav, num_mel_bins=80) features (fbank_i) and the processor's mean-normalised
    features (feat_i, se_processor.py:65-67);
  - the embeddings of the reference DTDNN built after torch.manual_seed(0), with its BatchNorm statistics and affines set
    by oracle.dtdnn.seed_bn_stats(seed=7), in eval mode, one wav at a time as the processor runs it (emb [3, 192]).
The extractor has 6.8 M parameters, so its seeded init is stored as checksums only (as make_golden_disc_init.py does):
DTDNN() after torch.manual_seed(0).  Needs an importable KAN-TTS checkout (KANTTS_REFERENCE) and torchaudio.
python tests/golden/make_golden_se.py"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)

from make_golden_disc_init import checksums  # noqa: E402
from oracle.dtdnn import seed_bn_stats  # noqa: E402
from oracle.ref_shims import REF_ROOT, reference_available  # noqa: E402

LENGTHS = (8000, 32160, 52800)


def seeded_wavs(seed=11):
    """Noise plus two seeded sinusoids with a slow envelope, peak about 0.3."""
    g = np.random.default_rng(seed)
    out = []
    for n in LENGTHS:
        t = np.arange(n) / 16000.0
        f1, f2 = g.uniform(100, 300), g.uniform(800, 3000)
        env = 0.5 + 0.5 * np.sin(2 * np.pi * g.uniform(1, 4) * t)
        w = 0.1 * env * np.sin(2 * np.pi * f1 * t) + 0.05 * np.sin(2 * np.pi * f2 * t) + 0.02 * g.standard_normal(n)
        out.append(w.astype(np.float32))
    return out


def main():
    if not reference_available():
        raise RuntimeError(f"reference checkout not found at {REF_ROOT}")
    sys.path.insert(0, REF_ROOT)
    import torchaudio.compliance.kaldi as Kaldi
    from kantts.preprocess.se_processor.D_TDNN import DTDNN

    torch.manual_seed(0)
    init = DTDNN().state_dict()
    with open(os.path.join(HERE, "se_dtdnn_init_checksums.json"), "w") as f:
        json.dump({"DTDNN": checksums(init)}, f)

    torch.manual_seed(0)
    model = DTDNN()
    seed_bn_stats(model, seed=7)
    model.eval()
    arrays = {}
    embs = []
    for i, w in enumerate(seeded_wavs()):
        fb = Kaldi.fbank(torch.from_numpy(w)[None], num_mel_bins=80)
        feat = fb - fb.mean(dim=0, keepdim=True)
        with torch.no_grad():
            embs.append(model(feat.unsqueeze(0)).squeeze(0).numpy())
        arrays[f"wav_{i}"] = w
        arrays[f"fbank_{i}"] = fb.numpy()
        arrays[f"feat_{i}"] = feat.numpy()
    arrays["emb"] = np.stack(embs)
    cfg = dict(lengths=list(LENGTHS), init_seed=0, bn_seed=7, wav_seed=11)
    np.savez_compressed(os.path.join(HERE, "se_dtdnn.npz"), cfg=np.frombuffer(json.dumps(cfg).encode(), dtype=np.uint8),
                        **arrays)


if __name__ == "__main__":
    main()
