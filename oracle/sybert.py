"""CPU restatement of the masked-symbol pretraining model of sybert.yaml (TEST INFRASTRUCTURE).

* ``sybert_forward``: KanTtsTextsyBERT (kantts/models/sambert/kantts_sambert.py:1047-1068), oracle/sambert.py's
  ``text_encoder`` without the output projection, then the vocabulary Linear.  Pinned against tests/golden/sybert_small.npz.
* ``seq_ce_loss``: SeqCELoss (kantts/train/loss.py:444-460).
* ``masking_counts`` / ``input_bert_masking``: the count rule of MaskingActor._input_bert_masking
  (kantts/datasets/dataset.py:890-920) for a given selection vector, shuffle permutation and replacement id; pinned against
  the reference's own outputs in the same fixture.
* ``bert_mask``: kt_bert_mask's Philox draw (include/kantts_b200.h) in NumPy, bit for bit.

Nothing in the product package imports this file.
"""
import math
import random

import numpy as np
import torch
import torch.nn.functional as F

from . import sambert as S
from .nsf import _MASK, _seed_words, philox4x32_10

P_MASK, P_RAND = 0.8, 0.1
_UTTERANCE_DRAW = 0xFFFFFFFF


def sybert_forward(sd, cfg, inputs_ling, input_lengths):
    """-> {"logits": (B, L, sy), "enc_slf_attn_lst": [...]}.  The encoder is oracle/sambert.text_encoder with its ling_proj
    replaced by the identity matrix, which F.linear applies exactly (each output is one input times 1 plus zeros)."""
    mask = S.length_mask(input_lengths, inputs_ling.shape[1])
    d_model = cfg["encoder_num_units"]
    p = dict(sd)
    p["text_encoder.ling_proj.weight"] = torch.eye(d_model, dtype=sd["fc.weight"].dtype)
    hid, attns, _ = S.text_encoder(inputs_ling, mask, S._SD(p, "text_encoder."), cfg)
    return {"logits": F.linear(hid, sd["fc.weight"], sd["fc.bias"]), "enc_slf_attn_lst": attns}


def seq_ce_loss(logits, targets, masks):
    """-> (masked mean cross-entropy, masked argmax error rate); 0 / 0 (no masked position) is NaN."""
    v = logits.shape[-1]
    ce = F.cross_entropy(logits.reshape(-1, v), targets.reshape(-1), reduction="none")
    m = masks.reshape(-1).to(ce.dtype)
    preds = torch.argmax(logits, dim=-1).reshape(-1)
    return (ce * m).sum() / m.sum(), ((preds != targets.reshape(-1)) * m).sum() / m.sum()


def masking_counts(n):
    """(floor(n * 0.8), floor(n * 0.1)) in float64, as math.floor in the reference."""
    return int(math.floor(n * P_MASK)), int(math.floor(n * P_RAND))


def input_bert_masking(seq, mask, perm, rand_id, mask_id):
    """MaskingActor._input_bert_masking with its shuffle ``perm`` (of arange(n)) and its randint ``rand_id`` given: the
    selected positions taken in the order ``perm``, the first floor(0.8 n) -> mask_id, the next floor(0.1 n) -> rand_id."""
    out = np.array(seq, copy=True)
    sel = np.where(np.asarray(mask) == 1)[0]
    n_mask, n_rand = masking_counts(len(sel))
    perm = np.asarray(perm, dtype=np.int64)
    out[sel[perm[:n_mask]]] = mask_id
    out[sel[perm[n_mask: n_mask + n_rand]]] = rand_id
    return out


def bert_mask(lings, valid_lengths, seed, call_index, mask_ratio, n_sy, mask_id):
    """kt_bert_mask: lings (B, L, n_feat) int64, valid_lengths (B,) -> (masked lings, targets (B, L) int64, bert_masks
    (B, L) float32).  Position i of utterance b draws (w0..w3) = Philox4x32-10((i, b, call low, call high), seed words):
    selected when i < valid_lengths[b] and w0 < ceil(mask_ratio 2^32); ranked by (w1 2^32 + w2, i); the replacement id is
    (w0' n_sy) >> 32 of counter (0xFFFFFFFF, b, call low, call high)."""
    lings = np.asarray(lings, dtype=np.int64)
    B, L, _ = lings.shape
    key = _seed_words(seed)
    c = int(call_index) & 0xFFFFFFFFFFFFFFFF
    c2, c3 = c & _MASK, c >> 32
    threshold = math.ceil(float(mask_ratio) * 2.0 ** 32)
    out = lings.copy()
    targets = lings[:, :, 0].copy()
    masks = np.zeros((B, L), dtype=np.float32)
    pos = np.arange(L, dtype=np.uint64)
    for b in range(B):
        w = philox4x32_10((pos, b, c2, c3), key)
        valid = min(max(int(valid_lengths[b]), 0), L)
        sel = (np.arange(L) < valid) & (w[0] < np.uint64(threshold))
        keys = (w[1] << np.uint64(32)) | w[2]
        idx = np.nonzero(sel)[0]
        perm = np.lexsort((idx, keys[idx]))              # ascending key, ties by position
        rand_id = (int(philox4x32_10((_UTTERANCE_DRAW, b, c2, c3), key)[0]) * int(n_sy)) >> 32
        out[b, :, 0] = input_bert_masking(lings[b, :, 0], sel.astype(np.int64), perm, rand_id, mask_id)
        masks[b, sel] = 1.0
    return out, targets, masks


def reference_bert_masking(seq, mask_ratio, n_sy, mask_id):
    """BERT_Text_Dataset.bert_masking of one utterance as the reference runs it on the host (dataset.py:876-920, 1022-1040):
    numpy's uniform draw thresholded by a per-symbol Python loop, the trailing eos cleared, np.random.shuffle and one
    random.randint.  -> (selection vector, masked symbols)."""
    mask = np.random.uniform(0, 1, len(seq))
    index = 0
    while index < len(mask):
        mask[index] = 1 if mask[index] < mask_ratio else 0
        index += 1
    mask[-1] = 0
    sel = np.where(mask == 1)[0]
    perm = np.arange(len(sel))
    np.random.shuffle(perm)
    n_mask, n_rand = masking_counts(len(sel))
    rand_id = random.randint(0, n_sy - 1) if n_rand > 0 else 0
    return mask, input_bert_masking(seq, mask, perm, rand_id, mask_id)
