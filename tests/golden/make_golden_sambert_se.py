"""Generate the speaker-embedding (SE) SAM-BERT golden by running the UNMODIFIED reference KanTtsSAMBERT (/root/reference,
imported through oracle/ref_shims.py) on CPU.  Build container only:

    python tests/golden/make_golden_sambert_se.py

* sambert_se_small.npz: SMALL_CFG with SE=True (no speaker table) and NSF outputs (num_mels = 8 mels + f0 + voiced flag,
  as sambert_se_nsf_global_16k.yaml), in eval(), a ragged teacher-forcing batch of 3 whose inputs_speaker is each
  utterance's seeded speaker embedding repeated over its symbols, as the reference collate builds it
  (datasets/dataset.py:760-765); forward, the five losses, one backward of their sum.
* se_init_checksums.json: state_dict layout and checksums of KanTtsSAMBERT(SE_CFG) after torch.manual_seed(5) (the
  seeded init without a speaker table).
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)

from oracle.ref_shims import import_reference  # noqa: E402
from make_batch import make_sambert_batch  # noqa: E402
from make_golden_disc_init import checksums  # noqa: E402
from make_golden_sambert import SMALL_CFG  # noqa: E402

import_reference()
from kantts.models.sambert.kantts_sambert import KanTtsSAMBERT  # noqa: E402
from kantts.train.loss import MelReconLoss, ProsodyReconLoss  # noqa: E402

SE_CFG = dict({k: v for k, v in SMALL_CFG.items() if k != "speaker"}, SE=True, num_mels=10, NSF=True,
              nsf_norm_type="global", nsf_f0_global_minimum=30.0, nsf_f0_global_maximum=730.0)


def se_batch(cfg, gen):
    """make_sambert_batch with inputs_speaker = one seeded (speaker_units,) embedding per utterance, repeated per symbol."""
    b = make_sambert_batch(cfg | {"speaker": 1}, B=3, L=10, gen=gen)
    B, L = b["inputs_emotion"].shape
    se = torch.randn(B, 1, cfg["speaker_units"], generator=gen)
    b["inputs_speaker"] = se.expand(B, L, cfg["speaker_units"]).contiguous()
    return b


def main():
    torch.manual_seed(5)
    with open(os.path.join(HERE, "se_init_checksums.json"), "w") as f:
        json.dump({"KanTtsSAMBERT": checksums(KanTtsSAMBERT(SE_CFG).state_dict())}, f)

    torch.manual_seed(1234)
    gen = torch.Generator().manual_seed(1243)
    cfg = SE_CFG
    model = KanTtsSAMBERT(cfg).eval()
    assert not hasattr(model, "spk_tokenizer")
    with torch.no_grad():
        for n, p in model.named_parameters():
            if p.requires_grad and (n.endswith("bias") or "layer_norm" in n or n.endswith("ln.weight")):
                p.add_(0.1 * torch.randn(p.shape, generator=gen))
    batch = se_batch(cfg, gen)
    res = model(batch["inputs_ling"], batch["inputs_emotion"], batch["inputs_speaker"], batch["input_lengths"],
                output_lengths=batch["output_lengths"], mel_targets=batch["mel_targets"],
                duration_targets=batch["duration_targets"], pitch_targets=batch["pitch_targets"],
                energy_targets=batch["energy_targets"])
    l0, l1 = MelReconLoss()(batch["output_lengths"], batch["mel_targets"], res["dec_outputs"], res["postnet_outputs"])
    dl, pl, el = ProsodyReconLoss()(res["valid_inter_lengths"], res["duration_targets"], res["pitch_targets"],
                                    res["energy_targets"], res["log_duration_predictions"], res["pitch_predictions"],
                                    res["energy_predictions"])
    total = l0 + l1 + dl + pl + el
    total.backward()
    arrays = {"sd/" + k: v.detach().numpy().copy() for k, v in model.state_dict().items()}
    arrays.update({"in/" + k: v.numpy() for k, v in batch.items()})
    for k in ("dec_outputs", "postnet_outputs", "log_duration_predictions", "pitch_predictions", "energy_predictions",
              "LR_text_outputs", "LR_emo_outputs", "LR_spk_outputs", "LR_length_rounded"):
        arrays["out/" + k] = res[k].detach().numpy()
    arrays["out/losses"] = np.asarray([float(v) for v in (l0, l1, dl, pl, el, total)], dtype=np.float64)
    for n, p in model.named_parameters():
        if p.grad is not None:
            arrays["grad/" + n] = p.grad.numpy().copy()
    path = os.path.join(HERE, "sambert_se_small.npz")
    np.savez_compressed(path, cfg=np.frombuffer(json.dumps(cfg).encode(), dtype=np.uint8), **arrays)
    print(f"sambert_se_small: {os.path.getsize(path) / 1e6:.2f} MB, {len(arrays)} arrays, losses {arrays['out/losses']}")


if __name__ == "__main__":
    main()
