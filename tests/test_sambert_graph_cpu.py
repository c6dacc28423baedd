"""CPU: the pieces of SambertStep(cuda_graph=True) that need no GPU -- the collate padding helper (data.pad_sambert_batch),
and the refusal of filled-pause and alignment-search models."""
import pytest
import torch

import kantts_b200 as K
from kantts_b200 import data, sambert
from golden.make_batch import make_c4_batch


def _collate_batch():
    """Three items of 5, 7 and 4 symbols (the trailing '~' included), padded like AM_Dataset.collate_fn: lings with the
    pad ids (1, 2, 3, 4), durations summing to the padded frame count, the padding frames on the symbol after each item's
    last."""
    g = torch.Generator().manual_seed(5)
    B, L, r = 3, 7, 3
    vil = torch.tensor([4, 6, 3])
    lings = torch.stack([torch.randint(5, 9, (B, L), generator=g) for _ in range(4)], -1)
    pad = torch.arange(L)[None, :] > vil[:, None]
    lings = torch.where(pad[:, :, None], torch.tensor([1, 2, 3, 4]), lings)
    dur = torch.randint(1, 4, (B, L), generator=g).masked_fill(pad, 0)
    out_len = dur.sum(1)
    T = -(-int(out_len.max()) // r) * r
    dur = dur.scatter_add(1, (vil + 1).clamp_max(L - 1)[:, None], (T - out_len)[:, None])
    return dict(input_lings=lings, input_emotions=torch.where(pad, 7, 0), input_speakers=torch.where(pad, 9, 1),
                valid_input_lengths=vil, valid_output_lengths=out_len, mel_targets=torch.randn(B, T, 5, generator=g),
                durations=dur, pitch_contours=torch.randn(B, L, generator=g).masked_fill(pad, 0.0),
                energy_contours=torch.randn(B, L, generator=g).masked_fill(pad, 0.0)), r


def test_pad_sambert_batch_pads_with_the_collate_values():
    b, r = _collate_batch()
    B, L = b["input_lings"].shape[:2]
    T = b["mel_targets"].shape[1]
    out = data.pad_sambert_batch(b, 8, 12, r, ling_pad=(1, 2, 3, 4), emotion_pad=7, speaker_pad=9)
    L2, T2 = 8, -(-T // 12) * 12
    assert out["input_lings"].shape == (B, L2, 4) and out["mel_targets"].shape == (B, T2, 5)
    assert torch.equal(out["input_lings"][:, :L], b["input_lings"])
    assert torch.equal(out["input_lings"][:, L:], torch.tensor([1, 2, 3, 4]).expand(B, L2 - L, 4))
    assert torch.equal(out["input_emotions"][:, L:], torch.full((B, L2 - L), 7))
    assert torch.equal(out["input_speakers"][:, L:], torch.full((B, L2 - L), 9))
    assert torch.equal(out["mel_targets"][:, :T], b["mel_targets"]) and not out["mel_targets"][:, T:].any()
    for k in ("pitch_contours", "energy_contours"):
        assert torch.equal(out[k][:, :L], b[k]) and not out[k][:, L:].any()
    for k in ("valid_input_lengths", "valid_output_lengths"):
        assert torch.equal(out[k], b[k])
    # the durations still sum to the padded frame count, the new frames on the symbol after each item's last
    assert torch.equal(out["durations"].sum(1), torch.full((B,), T2))
    want = torch.nn.functional.pad(b["durations"], (0, L2 - L))
    want[torch.arange(B), b["valid_input_lengths"] + 1] += T2 - T
    assert torch.equal(out["durations"], want)
    # already a multiple: nothing changes
    same = data.pad_sambert_batch(b, 7, T, r, ling_pad=(1, 2, 3, 4), emotion_pad=7, speaker_pad=9)
    for k, v in b.items():
        assert torch.equal(same[k], v), k


def test_pad_sambert_batch_speaker_embeddings_and_c4_shape():
    cfg = K.sambert_24k_config()
    b = make_c4_batch(cfg, torch.Generator().manual_seed(2), B=2, L=10, dur=3)
    b["input_speakers"] = torch.randn(2, 10, 6)                 # an SE batch: per-symbol float embeddings
    out = data.pad_sambert_batch(b, 16, 48, cfg["outputs_per_step"], (0, 0, 0, 0), 0, 5)
    assert out["input_speakers"].shape == (2, 16, 6) and not out["input_speakers"][:, 10:].any()
    assert out["mel_targets"].shape[1] == 48
    # valid_input_lengths = L - 1: the new frames go to the first new symbol
    assert torch.equal(out["durations"][:, 10], torch.full((2,), 48 - 30))


def test_pad_sambert_batch_rejects_bad_multiples():
    b, r = _collate_batch()
    with pytest.raises(ValueError, match="multiple of r"):
        data.pad_sambert_batch(b, 8, 10, r, (1, 2, 3, 4), 7, 9)
    with pytest.raises(ValueError, match="without durations"):
        data.pad_sambert_batch(dict(b, durations=None), 8, 12, r, (1, 2, 3, 4), 7, 9)


@pytest.mark.parametrize("variant,match", [("fp", "fp_insert_plan"), ("mas", "align's length validation")])
def test_graph_step_refuses_fp_and_mas_models(variant, match):
    cfg = K.sambert_fp_8k_config() if variant == "fp" else K.sambert_16k_mas_config()
    torch.manual_seed(0)
    model = sambert.KanTtsSAMBERT(cfg)
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    sch = K.train.NoamLR(opt, warmup_steps=10)
    with pytest.raises(ValueError, match=match):
        K.SambertStep(model, opt, sch, {}, cuda_graph=True)
    K.SambertStep(model, opt, sch, {})                          # the eager step is built as before

