"""Generate the filled-pause (FP) SAM-BERT goldens by running the UNMODIFIED reference KanTtsSAMBERT
(/root/reference, imported through oracle/ref_shims.py) on CPU.  Build container only:

    python tests/golden/make_golden_sambert_fp.py

* sambert_fp_small.npz: SMALL_CFG + FP=True in eval(), a fixed fp_dict of random linguistic ids, a ragged batch of 3
  with labels at position 0, consecutive labels, a label on the EOS position (j = input length), an utterance
  without labels and a short utterance whose 3 n_b exceeds max(inter) - max(input_lengths); teacher-forced forward,
  the five reference losses + FpCELoss, one backward of their sum.
* sambert_fp_small_infer.npz: batch-1 free-running inference of the same model with the duration and FP biases
  raised so that several positions insert; the generator asserts an argmax margin of the FP probabilities and a
  rounding margin of the durations.
* fp_insert_maps.npz: the reference insert_fp on label / prediction patterns, with text_hid[b, j, :] = 10000 b + j and
  the rows of filled pause k set to -(1 + 3 (k-1) + m): the output is the index map itself.
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
from make_golden_sambert import SMALL_CFG  # noqa: E402

import_reference()
from kantts.models.sambert.kantts_sambert import KanTtsSAMBERT  # noqa: E402
from kantts.train.loss import FpCELoss, MelReconLoss, ProsodyReconLoss  # noqa: E402

torch.set_num_threads(8)
CFG = dict(SMALL_CFG, FP=True)


def _fp_dict(cfg, gen):
    return {k: torch.stack([torch.randint(0, cfg[n], (1, 3), generator=gen)
                            for n in ("sy", "tone", "syllable_flag", "word_segment")], -1) for k in (1, 2, 3)}


def _save(name, cfg, arrays):
    path = os.path.join(HERE, name + ".npz")
    np.savez_compressed(path, cfg=np.frombuffer(json.dumps(cfg).encode(), dtype=np.uint8), **arrays)
    print(f"{name}: {os.path.getsize(path) / 1e3:.0f} KB, {len(arrays)} arrays")


def _fp_loss_fn():
    cuda = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self          # the reference constructor moves its weight to CUDA
    try:
        return FpCELoss(loss_type="ce", weight=[1, 4, 4, 8])
    finally:
        torch.Tensor.cuda = cuda


def make_train(model, fp_dict, gen):
    B, L, r = 3, 10, CFG["outputs_per_step"]
    ling = torch.stack([torch.randint(0, CFG[k], (B, L), generator=gen)
                        for k in ("sy", "tone", "syllable_flag", "word_segment")], -1)
    emo = torch.randint(0, CFG["emotion"], (B, L), generator=gen)
    spk = torch.randint(0, CFG["speaker"], (B, L), generator=gen)
    in_len = torch.tensor([10, 7, 10])
    lab = torch.zeros(B, L, dtype=torch.long)
    lab[0, 0], lab[0, 4] = 1, 3                              # position 0; a pause in the middle
    lab[1, 2], lab[1, 3], lab[1, 5], lab[1, 7] = 2, 2, 1, 3  # consecutive; EOS position j = 7 = input length
    inter = in_len + 3 * (lab > 0).sum(1)
    T = L + int(inter.max() - in_len.max())
    assert 3 * int((lab[1] > 0).sum()) > int(inter.max() - in_len.max())   # the short utterance's stream overflows T
    dur = torch.randint(1, 4, (B, T), generator=gen) * (torch.arange(T)[None] < inter[:, None])
    i0 = int(dur.sum(1).argmax())
    dur[i0, 0] += (-int(dur[i0].sum())) % r
    out_len = dur.sum(1)
    Tm = int(out_len.max())
    batch = dict(inputs_ling=ling, inputs_emotion=emo, inputs_speaker=spk, input_lengths=in_len, output_lengths=out_len,
                 mel_targets=torch.randn(B, Tm, CFG["num_mels"], generator=gen), duration_targets=dur,
                 pitch_targets=torch.randn(B, T, generator=gen), energy_targets=torch.randn(B, T, generator=gen),
                 fp_label=lab)
    res = model(ling, emo, spk, in_len, output_lengths=out_len, mel_targets=batch["mel_targets"], duration_targets=dur,
                pitch_targets=batch["pitch_targets"], energy_targets=batch["energy_targets"], fp_label=lab)
    l0, l1 = MelReconLoss()(out_len, batch["mel_targets"], res["dec_outputs"], res["postnet_outputs"])
    dl, pl, el = ProsodyReconLoss()(res["valid_inter_lengths"], res["duration_targets"], res["pitch_targets"],
                                    res["energy_targets"], res["log_duration_predictions"], res["pitch_predictions"],
                                    res["energy_predictions"])
    fl = _fp_loss_fn()(in_len, res["fp_predictions"], lab)
    total = l0 + l1 + dl + pl + el + fl
    total.backward()
    arrays = {"sd/" + k: v.detach().numpy().copy() for k, v in model.state_dict().items()}
    arrays.update({"in/" + k: v.numpy() for k, v in batch.items()})
    arrays.update({f"fp_dict/{k}": v.numpy() for k, v in fp_dict.items()})
    for k in ("dec_outputs", "postnet_outputs", "log_duration_predictions", "pitch_predictions", "energy_predictions",
              "LR_text_outputs", "LR_emo_outputs", "LR_spk_outputs", "LR_length_rounded", "fp_predictions",
              "valid_inter_lengths"):
        arrays["out/" + k] = res[k].detach().numpy()
    for k in ("enc_slf_attn_lst", "pnca_x_attn_lst", "pnca_h_attn_lst"):
        for i, a in enumerate(res[k]):
            arrays[f"out/{k}.{i}"] = a.detach().numpy()
    arrays["out/band_width"] = np.asarray([res["x_band_width"], res["h_band_width"]])
    arrays["out/losses"] = np.asarray([float(v) for v in (l0, l1, dl, pl, el, fl, total)], dtype=np.float64)
    for n, p in model.named_parameters():
        if p.grad is not None:
            arrays["grad/" + n] = p.grad.numpy().copy()
    _save("sambert_fp_small", CFG, arrays)
    print("  inter", res["valid_inter_lengths"].tolist(), "T", T, "losses", arrays["out/losses"])
    return batch


def make_infer(model, fp_dict, batch):
    with torch.no_grad():
        model.variance_adaptor.duration_predictor.fc.bias.fill_(1.25)
        model.FP_predictor.fc.bias.copy_(torch.tensor([0.0, 1.5, 1.0, 0.5]))
        inputs = {k: batch[k][:1] for k in ("inputs_ling", "inputs_emotion", "inputs_speaker", "input_lengths")}
        res = model(inputs["inputs_ling"], inputs["inputs_emotion"], inputs["inputs_speaker"], inputs["input_lengths"])
    fp = res["fp_predictions"][0, : int(inputs["input_lengths"][0])]
    top2 = fp.topk(2, dim=-1).values
    fp_margin = float((top2[:, 0] - top2[:, 1]).min())
    assert fp_margin > 1e-3, f"two filled-pause classes are within {fp_margin} of each other: change the bias"
    n_ins = int((fp.argmax(-1) > 0).sum())
    assert n_ins >= 3, f"only {n_ins} positions insert a filled pause: change the bias"
    dur = torch.exp(res["log_duration_predictions"]) - 1
    frac = (dur + 0.5) - torch.floor(dur + 0.5)
    margin = float(torch.minimum(frac, 1 - frac)[dur > 0].min())
    assert margin > 5e-3, f"a predicted duration sits {margin} from a rounding boundary: change the bias"
    arrays = {"sd/" + k: v.numpy().copy() for k, v in model.state_dict().items()}
    arrays.update({"in/" + k: v.numpy() for k, v in inputs.items()})
    arrays.update({f"fp_dict/{k}": v.numpy() for k, v in fp_dict.items()})
    for k in ("dec_outputs", "postnet_outputs", "log_duration_predictions", "pitch_predictions", "energy_predictions",
              "LR_text_outputs", "LR_emo_outputs", "LR_spk_outputs", "LR_length_rounded", "fp_predictions",
              "valid_inter_lengths"):
        arrays["out/" + k] = res[k].numpy()
    for k in ("pnca_x_attn_lst", "pnca_h_attn_lst"):
        for i, a in enumerate(res[k]):
            arrays[f"out/{k}.{i}"] = a.numpy()
    arrays["out/band_width"] = np.asarray([res["x_band_width"], res["h_band_width"]])
    _save("sambert_fp_small_infer", CFG, arrays)
    print(f"  inserted {n_ins}, inter {res['valid_inter_lengths'].tolist()}, fp margin {fp_margin:.4f}, "
          f"rounding margin {margin:.3f}, frames {res['LR_length_rounded'].tolist()}")


class _IdEncoder:
    """Stands in for text_encoder in insert_fp: filled pause k encodes to rows -(1 + 3 (k-1) + m)."""

    def __call__(self, seq, return_attns=True):
        k = int(seq[0, 0, 0])
        rows = torch.tensor([-(1 + 3 * (k - 1) + m) for m in range(3)], dtype=torch.float32)
        return rows[None, :, None].expand(1, 3, 2).clone(), None, None


def _map_patterns(gen):
    pats = []

    def lab(B, L, in_len, fill):
        x = torch.zeros(B, L, dtype=torch.long)
        for (b, j), v in fill.items():
            x[b, j] = v
        return dict(L=L, in_len=torch.tensor(in_len), fp_label=x)

    pats.append(lab(2, 6, [6, 4], {}))                                        # no insertions at all
    pats.append(lab(1, 5, [5], {(0, 0): 1}))                                  # B = 1, position 0
    pats.append(lab(1, 5, [5], {(0, 4): 3}))                                  # last position
    pats.append(lab(1, 3, [3], {(0, 0): 1, (0, 1): 2, (0, 2): 3}))            # every position, delta 9 > L (repeat)
    pats.append(lab(2, 4, [4, 2], {(1, 0): 2, (1, 1): 2, (1, 2): 1, (1, 3): 3}))  # padding-position labels, short row
    pats.append(lab(3, 8, [8, 5, 8], {(0, 3): 1, (1, 5): 2, (2, 1): 3, (2, 2): 3}))  # EOS position label (1, 5)
    pats.append(lab(2, 2, [2, 1], {(0, 0): 1, (0, 1): 1, (1, 0): 3, (1, 1): 2}))   # delta 6 > L = 2
    pats.append(lab(2, 7, [7, 7], {(0, 6): 2, (1, 0): 4}))                    # label 4 counts but inserts nothing
    for i in range(8):                                                        # random ~25 % labelled
        B, L = 1 + i % 4, 4 + 3 * i
        in_len = [L - (b * 2) % max(1, L // 2) for b in range(B)]
        x = torch.randint(1, 4, (B, L), generator=gen) * (torch.rand(B, L, generator=gen) < 0.25)
        pats.append(dict(L=L, in_len=torch.tensor(in_len), fp_label=x.long()))
    # inference: softmax outputs with exact ties (flags counted per class, one insertion per position)
    p = torch.full((2, 5, 4), 0.1)
    p[:, :, 0] = 0.7                                                          # no pause by default
    p[0, 0] = torch.tensor([0.1, 0.7, 0.1, 0.1])                              # class 1
    p[0, 1] = torch.tensor([0.1, 0.4, 0.4, 0.1])                              # tie 1 / 2: inserts 1, counts 2
    p[0, 2] = torch.tensor([0.25, 0.25, 0.25, 0.25])                          # four-way tie: inserts 1, counts 3
    p[0, 3] = torch.tensor([0.1, 0.1, 0.4, 0.4])                              # tie 2 / 3: inserts 2, counts 2
    p[1, 0] = torch.tensor([0.4, 0.1, 0.1, 0.4])                              # tie 0 / 3: inserts 3, counts 1
    p[1, 4] = torch.tensor([0.1, 0.1, 0.1, 0.7])                              # padding position: ignored
    pats.append(dict(L=5, in_len=torch.tensor([5, 4]), fp_p=p))
    q = torch.full((1, 4, 4), 0.25)                                           # every position a four-way tie
    pats.append(dict(L=4, in_len=torch.tensor([4]), fp_p=q))
    r = torch.softmax(torch.randn(3, 9, 4, generator=gen) * 2, -1)
    pats.append(dict(L=9, in_len=torch.tensor([9, 6, 3]), fp_p=r))
    return pats


def make_maps(gen):
    fake = type("FakeModel", (), {})()
    fake.text_encoder = _IdEncoder()
    fp_dict = {k: torch.full((1, 3, 4), k, dtype=torch.long) for k in (1, 2, 3)}
    arrays = {}
    for i, pt in enumerate(_map_patterns(gen)):
        L, in_len = pt["L"], pt["in_len"]
        B = in_len.shape[0]
        text = (10000 * torch.arange(B)[:, None] + torch.arange(L)[None, :]).float()[:, :, None].expand(B, L, 2).clone()
        lab, fpp = pt.get("fp_label"), pt.get("fp_p")
        if fpp is None:
            fpp = torch.zeros(B, L, 4)
        masks = torch.arange(L)[None, :] >= in_len[:, None]
        emo = torch.arange(L)[None, :].expand(B, L).clone()
        out, emo_out, _, inter = KanTtsSAMBERT.insert_fp(fake, text, fpp, lab, fp_dict, emo, emo.clone(), in_len, masks)
        ids = out[:, :, 0]
        assert torch.equal(out[:, :, 0], out[:, :, 1])
        code = torch.where(ids >= 0, ids - 10000 * torch.arange(B)[:, None], ids).long()
        arrays[f"{i}/in_len"] = in_len.numpy()
        if lab is not None:
            arrays[f"{i}/fp_label"] = lab.numpy()
        else:
            arrays[f"{i}/fp_p"] = pt["fp_p"].numpy()
        arrays[f"{i}/map"] = code.numpy()
        arrays[f"{i}/inter"] = inter.numpy()
        arrays[f"{i}/ext"] = emo_out.numpy()
    _save("fp_insert_maps", {"patterns": len(arrays) // 5}, arrays)


def main():
    torch.manual_seed(1234)
    gen = torch.Generator().manual_seed(1236)
    model = KanTtsSAMBERT(CFG).eval()
    with torch.no_grad():
        for n, p in model.named_parameters():
            if p.requires_grad and (n.endswith("bias") or "layer_norm" in n or n.endswith("ln.weight")):
                p.add_(0.1 * torch.randn(p.shape, generator=gen))
    fp_dict = _fp_dict(CFG, gen)
    model.fp_dict = fp_dict
    batch = make_train(model, fp_dict, gen)
    make_infer(model, fp_dict, batch)
    make_maps(gen)


if __name__ == "__main__":
    main()
