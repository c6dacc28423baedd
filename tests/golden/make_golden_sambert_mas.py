"""Generate the monotonic-alignment-search (MAS) SAM-BERT goldens by running the UNMODIFIED reference KanTtsSAMBERT,
mas_width1 (numba, as shipped) and the attention losses (/root/reference, imported through oracle/ref_shims.py) on CPU.
Build container only:

    python tests/golden/make_golden_sambert_mas.py

* sambert_mas_small.npz / sambert_mas_byte_small.npz: SMALL_CFG + MAS=True (the byte twin with using_byte=True) in
  eval(), a ragged batch of 3 with the reference's beta-binomial priors; teacher-forced forward with the alignment
  outputs, the five reference losses + AttentionCTCLoss + AttentionBinarizationLoss at epoch 37 (warm-up ratio 0.37),
  one backward of their sum.  The generator asserts a decision margin of the alignment search: on the chosen path no
  comparison lies within 1e-3 of a tie.
* mas_patterns.npz: b_mas on hand-made maps: exact ties, zero probabilities, T_mel == T_text, one symbol, one frame,
  in_len == T_text, a ragged batch, out_len < in_len.
* attn_ctc.npz: AttentionCTCLoss and its autograd gradient, including an utterance with out_len < in_len (infinite loss,
  zeroed by zero_infinity).
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
from oracle.sambert_mas import mas_margin  # noqa: E402
from make_golden_sambert import SMALL_CFG  # noqa: E402

import_reference()
from kantts.datasets.dataset import beta_binomial_prior_distribution  # noqa: E402
from kantts.models.sambert.alignment import b_mas  # noqa: E402
from kantts.models.sambert.kantts_sambert import KanTtsSAMBERT  # noqa: E402
from kantts.train.loss import (AttentionBinarizationLoss, AttentionCTCLoss, MelReconLoss,  # noqa: E402
                               ProsodyReconLoss)

torch.set_num_threads(8)
EPOCH = 37
CFG = dict(SMALL_CFG, MAS=True)
BYTE_CFG = dict({k: v for k, v in CFG.items() if k not in ("sy", "tone", "syllable_flag", "word_segment")},
                using_byte=True, byte_index=23)


def _save(name, cfg, arrays):
    path = os.path.join(HERE, name + ".npz")
    np.savez_compressed(path, cfg=np.frombuffer(json.dumps(cfg).encode(), dtype=np.uint8), **arrays)
    print(f"{name}: {os.path.getsize(path) / 1e3:.0f} KB, {len(arrays)} arrays")


def make_batch(cfg, gen):
    """Ragged teacher-forcing batch as the MAS collate builds it (datasets/dataset.py:770-826): valid_input_lengths one
    short of the symbol count (the trailing '~'), mel frames rounded up to r, frame-level pitch / energy with unvoiced
    (zero) frames, priors beta_binomial(len + 1, frames) in a zero (B, T_mel, L) tensor."""
    B, L, r = 3, 10, cfg["outputs_per_step"]
    if cfg.get("using_byte"):
        ling = torch.randint(0, cfg["byte_index"], (B, L, 1), generator=gen)
    else:
        ling = torch.stack([torch.randint(0, cfg[k], (B, L), generator=gen)
                            for k in ("sy", "tone", "syllable_flag", "word_segment")], -1)
    in_len = torch.tensor([9, 6, 8])
    out_len = torch.tensor([40, 25, 31])
    Tm = -(-int(out_len.max()) // r) * r
    valid = torch.arange(Tm)[None, :] < out_len[:, None]
    mel = torch.randn(B, Tm, cfg["num_mels"], generator=gen) * valid[:, :, None]
    pitch = torch.randn(B, Tm, generator=gen).abs() * (torch.rand(B, Tm, generator=gen) > 0.3) * valid
    energy = torch.randn(B, Tm, generator=gen).abs() * valid
    prior = torch.zeros(B, Tm, L)
    for b in range(B):
        p = beta_binomial_prior_distribution(int(in_len[b]) + 1, int(out_len[b]))
        prior[b, : p.shape[0], : p.shape[1]] = p
    return dict(inputs_ling=ling, inputs_emotion=torch.randint(0, cfg["emotion"], (B, L), generator=gen),
                inputs_speaker=torch.randint(0, cfg["speaker"], (B, L), generator=gen), input_lengths=in_len,
                output_lengths=out_len, mel_targets=mel, pitch_targets=pitch.float(), energy_targets=energy.float(),
                attn_priors=prior)


def make_model_golden(name, cfg, seed):
    torch.manual_seed(1234)
    gen = torch.Generator().manual_seed(seed)
    model = KanTtsSAMBERT(cfg).eval()
    with torch.no_grad():
        for n, p in model.named_parameters():
            if p.requires_grad and (n.endswith("bias") or "layer_norm" in n or n.endswith("ln.weight")):
                p.add_(0.1 * torch.randn(p.shape, generator=gen))
    batch = make_batch(cfg, gen)
    get_device = torch.Tensor.get_device
    # binarize_attention_parallel returns the hard alignment .to(attn.get_device()), which is -1 for a CPU tensor
    torch.Tensor.get_device = lambda self: get_device(self) if self.is_cuda else "cpu"
    try:
        res = model(batch["inputs_ling"], batch["inputs_emotion"], batch["inputs_speaker"], batch["input_lengths"],
                    output_lengths=batch["output_lengths"], mel_targets=batch["mel_targets"], duration_targets=None,
                    pitch_targets=batch["pitch_targets"], energy_targets=batch["energy_targets"],
                    attn_priors=batch["attn_priors"])
    finally:
        torch.Tensor.get_device = get_device
    soft = res["attn_soft"].detach().numpy()
    margin = min(mas_margin(soft[b, 0, : int(batch["output_lengths"][b]), : int(batch["input_lengths"][b])])
                 for b in range(soft.shape[0]))
    assert margin > 1e-3, f"an alignment decision is {margin} from a tie: change the seed"
    assert torch.equal(res["duration_targets"].sum(1), torch.full((3,), float(batch["mel_targets"].shape[1])))
    l0, l1 = MelReconLoss()(batch["output_lengths"], batch["mel_targets"], res["dec_outputs"], res["postnet_outputs"])
    dl, pl, el = ProsodyReconLoss()(res["valid_inter_lengths"], res["duration_targets"], res["pitch_targets"],
                                    res["energy_targets"], res["log_duration_predictions"], res["pitch_predictions"],
                                    res["energy_predictions"])
    ctc = AttentionCTCLoss()(res["attn_logprob"], batch["input_lengths"], batch["output_lengths"])
    kl = AttentionBinarizationLoss(0, 100)(EPOCH, res["attn_hard"], res["attn_soft"])
    total = l0 + l1 + dl + pl + el + ctc + kl
    total.backward()
    arrays = {"sd/" + k: v.detach().numpy().copy() for k, v in model.state_dict().items()}
    arrays.update({"in/" + k: v.numpy() for k, v in batch.items()})
    for k in ("dec_outputs", "postnet_outputs", "log_duration_predictions", "pitch_predictions", "energy_predictions",
              "LR_text_outputs", "LR_emo_outputs", "LR_spk_outputs", "LR_length_rounded", "duration_targets",
              "pitch_targets", "energy_targets", "attn_soft", "attn_hard", "attn_logprob"):
        arrays["out/" + k] = res[k].detach().numpy()
    for k in ("enc_slf_attn_lst", "pnca_x_attn_lst", "pnca_h_attn_lst"):
        for i, a in enumerate(res[k]):
            arrays[f"out/{k}.{i}"] = a.detach().numpy()
    arrays["out/band_width"] = np.asarray([res["x_band_width"], res["h_band_width"]])
    arrays["out/losses"] = np.asarray([float(v) for v in (l0, l1, dl, pl, el, ctc, kl, total)], dtype=np.float64)
    arrays["out/epoch"] = np.asarray(EPOCH)
    for n, p in model.named_parameters():
        if p.grad is not None:
            arrays["grad/" + n] = p.grad.numpy().copy()
    _save(name, cfg, arrays)
    print(f"  margin {margin:.4f}, durations {res['duration_targets'].tolist()}, losses {arrays['out/losses']}")


def _patterns(gen):
    pats = []

    def add(maps, in_lens, out_lens):
        pats.append((np.asarray(maps, dtype=np.float32), np.asarray(in_lens), np.asarray(out_lens)))

    add(np.full((1, 1, 6, 4), 0.25), [4], [6])                                    # exact ties everywhere
    add(np.full((2, 1, 9, 5), 0.2), [5, 3], [9, 7])                               # ties, ragged
    m = torch.rand(1, 1, 8, 5, generator=gen).numpy()
    m[0, 0, 2:5, 1] = 0.0                                                         # a zero stretch (-inf cells)
    m[0, 0, 0, 0] = 0.0                                                           # row 0 itself -inf
    add(m, [5], [8])
    m = torch.rand(1, 1, 6, 4, generator=gen).numpy()
    m[0, 0, :, 2] = 0.0                                                           # a zero column: every path -inf
    add(m, [4], [6])
    add(torch.rand(1, 1, 7, 7, generator=gen).numpy(), [7], [7])                  # T_mel == T_text
    add(torch.rand(1, 1, 7, 1, generator=gen).numpy(), [1], [7])                  # one symbol
    add(torch.rand(1, 1, 1, 3, generator=gen).numpy(), [3], [1])                  # one frame: the extra row-0 write
    add(torch.rand(1, 1, 5, 1, generator=gen).numpy()[:, :, :1], [1], [1])        # one frame, one symbol
    add(torch.softmax(torch.randn(3, 1, 12, 6, generator=gen) * 3, -1).numpy(), [6, 4, 5], [12, 8, 10])  # ragged, in_len == T_text
    add(torch.rand(2, 1, 3, 6, generator=gen).numpy(), [6, 5], [3, 2])            # out_len < in_len
    add(torch.softmax(torch.randn(2, 1, 40, 13, generator=gen) * 2, -1).numpy(), [13, 9], [40, 31])
    m = torch.softmax(torch.randn(1, 1, 10, 6, generator=gen), -1).numpy()
    m[0, 0, 3] = m[0, 0, 3, :1]                                                   # a uniform row mid-way
    add(m, [6], [10])
    return pats


def make_patterns(gen):
    arrays = {}
    for i, (maps, in_lens, out_lens) in enumerate(_patterns(gen)):
        hard = b_mas(maps, in_lens, out_lens, width=1)
        arrays[f"{i}/soft"] = maps
        arrays[f"{i}/in_len"] = in_lens.astype(np.int64)
        arrays[f"{i}/out_len"] = out_lens.astype(np.int64)
        arrays[f"{i}/hard"] = hard
        arrays[f"{i}/dur"] = hard.sum(2)[:, 0, :]
    _save("mas_patterns", {"patterns": len(arrays) // 5}, arrays)


def make_ctc(gen):
    arrays = {}
    cases = [((3, 20, 7), [7, 5, 6], [20, 14, 4]),          # utterance 2: out_len < in_len (zero_infinity)
             ((2, 31, 9), [9, 4], [31, 9]),
             ((1, 5, 5), [5], [5])]                         # T == N: a single path
    for i, (shape, in_lens, out_lens) in enumerate(cases):
        lp = (torch.randn(shape[0], 1, shape[1], shape[2], generator=gen) * 2).requires_grad_(True)
        loss = AttentionCTCLoss()(lp, torch.tensor(in_lens), torch.tensor(out_lens))
        loss.backward()
        arrays[f"{i}/logprob"] = lp.detach().numpy()
        arrays[f"{i}/in_len"] = np.asarray(in_lens)
        arrays[f"{i}/out_len"] = np.asarray(out_lens)
        arrays[f"{i}/loss"] = np.asarray(float(loss))
        arrays[f"{i}/grad"] = lp.grad.numpy()
        print(f"  ctc case {i}: loss {float(loss):.6f}")
    _save("attn_ctc", {"cases": len(cases)}, arrays)


def main():
    make_model_golden("sambert_mas_small", CFG, 1237)
    make_model_golden("sambert_mas_byte_small", BYTE_CFG, 1241)
    gen = torch.Generator().manual_seed(1239)
    make_patterns(gen)
    make_ctc(gen)


if __name__ == "__main__":
    main()
