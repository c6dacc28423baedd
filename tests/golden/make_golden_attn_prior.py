"""Generate tests/golden/attn_prior.npz from the UNMODIFIED reference's ``beta_binomial_prior_distribution``
(kantts/datasets/dataset.py:20-31, one scipy.stats.betabinom per mel frame; /root/reference, imported through
oracle/ref_shims.py).  Build container only:

    python tests/golden/make_golden_attn_prior.py

* ``pair/{P}_{M}``: the (M, P) float64 prior of P symbols over M frames for the pairs of PAIRS: one symbol, one frame,
  fewer frames than symbols, and sizes of real utterances.
* ``batch/*``: a ragged batch of 4 as AM_Dataset.collate_fn builds its ``attn_priors`` (dataset.py:781-793, 816-827,
  outputs_per_step r = 3): valid_input_lengths one short of the symbol count (the trailing eos), the frames rounded up to r
  by the reference's Padder, each utterance's float64 prior copied into a zero float32 (B, T_mel, L) tensor.
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from oracle.ref_shims import import_reference  # noqa: E402

import_reference()
from kantts.datasets.dataset import Padder, beta_binomial_prior_distribution  # noqa: E402

PAIRS = [(1, 1), (1, 5), (2, 1), (3, 7), (7, 3), (13, 47), (60, 300), (121, 600)]
R = 3
SYMBOLS = [23, 9, 31, 12]            # len(ling_data[0]), the eos included
FRAMES = [95, 40, 121, 7]            # mel frames; the last utterance has fewer frames than symbols


def main():
    arrays = {}
    for P, M in PAIRS:
        p = beta_binomial_prior_distribution(P, M)
        assert p.dtype == torch.float64 and p.shape == (M, P)
        arrays[f"pair/{P}_{M}"] = p.numpy()
    valid_in = torch.as_tensor([n - 1 for n in SYMBOLS], dtype=torch.long)
    valid_out = torch.as_tensor(FRAMES, dtype=torch.long)
    t_mel = Padder()._round_up(int(valid_out.max()), R)
    priors = torch.zeros(len(SYMBOLS), t_mel, max(SYMBOLS))
    for i, (P, M) in enumerate(zip(SYMBOLS, FRAMES)):
        p = beta_binomial_prior_distribution(P, M)
        priors[i, : p.shape[0], : p.shape[1]] = p
    arrays["batch/valid_input_lengths"] = valid_in.numpy()
    arrays["batch/valid_output_lengths"] = valid_out.numpy()
    arrays["batch/attn_priors"] = priors.numpy()
    path = os.path.join(HERE, "attn_prior.npz")
    cfg = {"pairs": PAIRS, "outputs_per_step": R}
    np.savez_compressed(path, cfg=np.frombuffer(json.dumps(cfg).encode(), dtype=np.uint8), **arrays)
    print(f"attn_prior: {os.path.getsize(path) / 1e3:.0f} KB, {len(arrays)} arrays, batch {tuple(priors.shape)}")


if __name__ == "__main__":
    main()
