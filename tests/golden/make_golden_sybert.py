"""Generate the syBERT goldens by running the UNMODIFIED reference KanTtsTextsyBERT, SeqCELoss and MaskingActor
(/root/reference, imported through oracle/ref_shims.py) on CPU.  Build container only:

    python tests/golden/make_golden_sybert.py

* sybert_small.npz: the encoder fields of SMALL_CFG with mask_ratio 0.3, in eval(), on a ragged batch of 3 masked by the
  reference's MaskingActor and padded as BERT_Text_Dataset.collate_fn pads it; logits, the attention maps, SeqCELoss's
  (loss, err) and the gradients of loss / V, as Textsy_BERT_Trainer.train_step divides.  The reference's forward unpacks two
  of TextFftEncoder's three results and raises, so its text_encoder and fc run here one after the other, which is what that
  forward evidently means.  At two [MASK] positions the original symbol is chosen as the model's argmax (the logits there
  do not depend on it), so that the error rate lies strictly between 0 and 1.  Also MaskingActor._input_bert_masking on
  fixed selection vectors under seeded shuffles ("mask/<i>/..."), with the permutation and the replacement id those seeds
  give, to pin the count rule.
* sybert_init_checksums.json: the state_dict layout and checksums of KanTtsTextsyBERT after torch.manual_seed(5), for the
  small config and for sybert.yaml's params with the PinYin unit sizes, and the yaml's params themselves.
"""
import json
import os
import random
import sys

import numpy as np
import torch
import yaml

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)

from oracle.ref_shims import REF_ROOT, import_reference  # noqa: E402
from make_golden_disc_init import checksums  # noqa: E402
from make_golden_sambert import SMALL_CFG  # noqa: E402

import_reference()
from kantts.datasets.dataset import MaskingActor  # noqa: E402
from kantts.models.sambert.kantts_sambert import KanTtsTextsyBERT  # noqa: E402
from kantts.models.utils import get_mask_from_lengths  # noqa: E402
from kantts.train.loss import SeqCELoss  # noqa: E402

ENCODER_KEYS = ("max_len", "embedding_dim", "encoder_num_layers", "encoder_num_heads", "encoder_num_units",
                "encoder_ffn_inner_dim", "encoder_dropout", "encoder_attention_dropout", "encoder_relu_dropout",
                "encoder_projection_units", "sy", "tone", "syllable_flag", "word_segment")
CFG = dict({k: SMALL_CFG[k] for k in ENCODER_KEYS}, mask_ratio=0.3)
UNITS = dict(sy=147, tone=10, syllable_flag=8, word_segment=8)


def _save(name, cfg, arrays):
    path = os.path.join(HERE, name + ".npz")
    np.savez_compressed(path, cfg=np.frombuffer(json.dumps(cfg).encode(), dtype=np.uint8), **arrays)
    print(f"{name}: {os.path.getsize(path) / 1e3:.0f} KB, {len(arrays)} arrays")


def masked_batch(cfg, gen):
    """Three utterances of 10, 7 and 9 symbols (the last one the eos '~' = sy - 2), valid_input_lengths one short of that
    (collate_fn), each masked by MaskingActor as BERT_Text_Dataset.bert_masking does, padded to 10 with the sy pad id
    (sy - 3) and zeros for the other units, bert_masks padded with 0."""
    sy = cfg["sy"]
    lens = [10, 7, 9]
    L = max(lens)
    actor = MaskingActor(cfg["mask_ratio"])
    ling = torch.zeros(3, L, 4, dtype=torch.long)
    ling[:, :, 0] = sy - 3
    masked = ling.clone()
    bert_masks = torch.zeros(3, L)
    np.random.seed(11)
    random.seed(11)
    for b, n in enumerate(lens):
        seq = torch.randint(0, sy - 3, (n,), generator=gen)
        seq[-1] = sy - 2
        ling[b, :n, 0] = seq
        for f, k in ((1, "tone"), (2, "syllable_flag"), (3, "word_segment")):
            ling[b, :n, f] = torch.randint(0, cfg[k], (n,), generator=gen)
        mask = actor._get_random_mask(n, p1=actor.mask_ratio)
        mask[-1] = 0
        out = actor._input_bert_masking(seq.numpy(), sy, sy - 1, mask)
        masked[b, :n] = ling[b, :n]
        masked[b, :n, 0] = torch.from_numpy(out)
        bert_masks[b, :n] = torch.from_numpy(mask).float()
    assert bert_masks.sum() >= 4 and (masked[:, :, 0] == sy - 1).any()
    return dict(input_lings=masked, valid_input_lengths=torch.tensor([n - 1 for n in lens]), targets=ling[:, :, 0].clone(),
                bert_masks=bert_masks)


def masking_cases():
    """Selection vectors of 0..40 selected positions; per case the permutation np.random.shuffle and the id
    random.randint give under the case's seeds, and the reference's output under the same seeds."""
    actor = MaskingActor(0.3)
    arrays = {}
    rng = np.random.RandomState(5)
    sizes = [0, 1, 2, 4, 5, 9, 10, 11, 19, 20, 21, 29, 30, 39, 40]
    for i, n_sel in enumerate(sizes):
        length = n_sel + 7
        mask = np.zeros(length)
        mask[np.sort(rng.choice(length - 1, n_sel, replace=False))] = 1
        seq = rng.randint(0, 144, length).astype(np.int64)
        np.random.seed(100 + i)
        perm = np.arange(n_sel)
        np.random.shuffle(perm)
        random.seed(200 + i)
        rand_id = random.randint(0, 147 - 1)
        np.random.seed(100 + i)
        random.seed(200 + i)
        out = actor._input_bert_masking(seq, 147, 146, mask)
        for k, v in (("seq", seq), ("mask", mask), ("perm", perm), ("rand_id", np.asarray(rand_id)), ("out", out)):
            arrays[f"mask/{i}/{k}"] = np.asarray(v)
    return arrays, len(sizes)


def main():
    with open(os.path.join(REF_ROOT, "kantts", "configs", "sybert.yaml")) as f:
        params = yaml.safe_load(f)["Model"]["KanTtsTextsyBERT"]["params"]
    init = {"yaml_params": params}
    for name, cfg in (("small", CFG), ("sybert.yaml", dict(params, **UNITS))):
        torch.manual_seed(5)
        init[name] = checksums(KanTtsTextsyBERT(cfg).state_dict())
    with open(os.path.join(HERE, "sybert_init_checksums.json"), "w") as f:
        json.dump(init, f)

    torch.manual_seed(1234)
    gen = torch.Generator().manual_seed(1245)
    model = KanTtsTextsyBERT(CFG).eval()
    with torch.no_grad():
        for n, p in model.named_parameters():
            if n.endswith("bias") or "layer_norm" in n or n.endswith("ln.weight"):
                p.add_(0.1 * torch.randn(p.shape, generator=gen))
    batch = masked_batch(CFG, gen)
    masks = get_mask_from_lengths(batch["valid_input_lengths"], max_len=batch["input_lings"].size(1))
    # A [MASK] position's logits do not depend on its original symbol: make that symbol the argmax at two such positions,
    # so that the error rate is neither 0 nor 1.
    with torch.no_grad():
        preds = model.fc(model.text_encoder(batch["input_lings"].clone(), masks)[0]).argmax(-1)
    hits = [(b, i) for b, i in zip(*torch.nonzero(batch["input_lings"][:, :, 0] == CFG["sy"] - 1, as_tuple=True))
            if int(preds[b, i]) < CFG["sy"] - 3][:2]
    assert len(hits) == 2, hits
    for b, i in hits:
        batch["targets"][b, i] = preds[b, i]
    text_hid, attns, _ = model.text_encoder(batch["input_lings"], masks, return_attns=True)
    logits = model.fc(text_hid)
    loss, err = SeqCELoss()(logits, batch["targets"], batch["bert_masks"])
    (loss / logits.size(-1)).backward()
    arrays = {"sd/" + k: v.detach().numpy().copy() for k, v in model.state_dict().items()}
    arrays.update({"in/" + k: v.numpy() for k, v in batch.items()})
    arrays["out/logits"] = logits.detach().numpy()
    for i, a in enumerate(attns):
        arrays[f"out/enc_slf_attn_lst.{i}"] = a.detach().numpy()
    arrays["out/loss_err"] = np.asarray([float(loss), float(err)], dtype=np.float64)
    for n, p in model.named_parameters():
        if p.grad is not None:
            arrays["grad/" + n] = p.grad.numpy().copy()
    cases, n_cases = masking_cases()
    arrays.update(cases)
    _save("sybert_small", dict(CFG, masking_cases=n_cases), arrays)
    print(f"  loss {float(loss):.6f}, err {float(err):.4f}, masked {int(batch['bert_masks'].sum())} positions")


if __name__ == "__main__":
    main()
