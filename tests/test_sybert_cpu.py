"""CPU: the masked-symbol pretraining model of sybert.yaml.  The oracle restatement (oracle/sybert.py) against the goldens of
the unmodified reference (tests/golden/make_golden_sybert.py), the masking count rule, the config, the module's state_dict
contract and seeded init, and the install patch."""
import json
import math
import os

import numpy as np
import pytest
import torch

import kantts_b200 as K
from conftest import GOLDEN, rel_l2
from oracle import sybert as osy


def _init():
    with open(os.path.join(GOLDEN, "sybert_init_checksums.json")) as f:
        return json.load(f)


def test_sybert_oracle_forward_loss_and_grads_match_reference(golden):
    g = golden("sybert_small")
    sd = g.group("sd/")
    for k, v in sd.items():
        if v.dtype.is_floating_point and "position_enc" not in k:
            v.requires_grad_(True)
    b = g.group("in/")
    res = osy.sybert_forward(sd, g.cfg, b["input_lings"], b["valid_input_lengths"])
    assert res["logits"].shape == g.t("out/logits").shape == (3, 10, g.cfg["sy"])
    assert rel_l2(res["logits"].detach(), g.t("out/logits")) < 2e-6
    assert len(res["enc_slf_attn_lst"]) == g.cfg["encoder_num_layers"]
    for i, a in enumerate(res["enc_slf_attn_lst"]):
        assert a.shape == g.t(f"out/enc_slf_attn_lst.{i}").shape
        assert rel_l2(a.detach(), g.t(f"out/enc_slf_attn_lst.{i}")) < 2e-6, i
    loss, err = osy.seq_ce_loss(res["logits"], b["targets"], b["bert_masks"])
    want_loss, want_err = g.t("out/loss_err").tolist()
    assert abs(float(loss.detach()) - want_loss) < 2e-6 * want_loss and float(err) == pytest.approx(want_err, abs=1e-7)
    assert 0.0 < want_err < 1.0
    (loss / res["logits"].shape[-1]).backward()
    grads = g.group("grad/")
    assert "fc.weight" in grads and "text_encoder.sy_emb.weight" in grads
    for k, w in grads.items():
        got = sd[k].grad
        assert got is not None, k
        assert rel_l2(got, w) < 2e-6 or float((got - w).abs().max()) < 1e-8, (k, rel_l2(got, w))


def test_oracle_masking_reproduces_reference_count_rule(golden):
    g = golden("sybert_small")
    n = g.cfg["masking_cases"]
    assert n >= 10
    sizes = set()
    for i in range(n):
        a = {k: g.arrays[f"mask/{i}/{k}"] for k in ("seq", "mask", "perm", "rand_id", "out")}
        got = osy.input_bert_masking(a["seq"], a["mask"], a["perm"], int(a["rand_id"]), 146)
        assert np.array_equal(got, a["out"]), i
        sel = int(a["mask"].sum())
        sizes.add(sel)
        n_mask, n_rand = osy.masking_counts(sel)
        assert int((a["out"] == 146).sum() - (a["seq"] == 146).sum()) <= n_mask
        assert int(((a["out"] != a["seq"]) & (a["mask"] == 0)).sum()) == 0
    assert {0, 1, 9, 10, 40} <= sizes


def test_masking_counts_floor_like_python():
    for n in range(801):
        assert osy.masking_counts(n) == (math.floor(n * 0.8), math.floor(n * 0.1)), n
        # up to max_len the float64 products never round across an integer: the counts are the exact floors
        assert osy.masking_counts(n) == (4 * n // 5, n // 10), n


def test_oracle_bert_mask_invariants():
    gen = torch.Generator().manual_seed(3)
    B, L = 6, 40
    lens = [39, 12, 25, 1, 0, 30]
    lings = torch.stack([torch.randint(0, 144, (B, L), generator=gen)] + [torch.randint(0, 8, (B, L), generator=gen)
                                                                          for _ in range(3)], -1).numpy()
    out, targets, masks = osy.bert_mask(lings, lens, 99, 4, 0.3, 147, 146)
    assert np.array_equal(targets, lings[:, :, 0]) and np.array_equal(out[:, :, 1:], lings[:, :, 1:])
    for b in range(B):
        sel = masks[b] == 1
        assert not sel[lens[b]:].any()
        n_mask, n_rand = osy.masking_counts(int(sel.sum()))
        changed = out[b, :, 0] != lings[b, :, 0]
        assert not changed[~sel].any()
        assert int((out[b, sel, 0] == 146).sum()) >= n_mask
    again = osy.bert_mask(lings, lens, 99, 4, 0.3, 147, 146)
    assert all(np.array_equal(x, y) for x, y in zip((out, targets, masks), again))
    other = osy.bert_mask(lings, lens, 99, 5, 0.3, 147, 146)
    assert not np.array_equal(other[2], masks)


def test_sybert_model_state_dict_and_seeded_init_match_reference(golden):
    from golden.make_golden_disc_init import checksums
    want = _init()
    for name, cfg in (("small", golden("sybert_small").cfg), ("sybert.yaml", K.sybert_config())):
        torch.manual_seed(5)
        m = K.KanTtsTextsyBERT(cfg)
        sd = m.state_dict()
        assert not any("ling_proj" in k for k in sd)
        assert list(sd)[-2:] == ["fc.weight", "fc.bias"] and all(k.startswith("text_encoder.") for k in list(sd)[:-2])
        got = checksums(sd)
        assert got[0] == want[name][0], name
        assert got[1] == pytest.approx(want[name][1], rel=1e-12) and got[2] == pytest.approx(want[name][2], rel=1e-12)
    m = K.KanTtsTextsyBERT(golden("sybert_small").cfg)
    m.load_state_dict(golden("sybert_small").group("sd/"), strict=True)


def test_sybert_config_is_the_yaml_plus_unit_sizes():
    cfg = K.sybert_config()
    params = _init()["yaml_params"]
    assert cfg == dict(params, sy=147, tone=10, syllable_flag=8, word_segment=8)
    assert cfg["mask_ratio"] == 0.3


def test_byte_sybert_is_not_built():
    cfg = dict(K.sybert_config(), using_byte=True, byte_index=259)
    with pytest.raises(NotImplementedError, match="byte"):
        K.KanTtsTextsyBERT(cfg)


def test_seq_ce_loss_is_built_and_install_patches_the_model():
    crit = K.criterion_builder({"Loss": {"SeqCELoss": {"enable": True, "params": {"loss_type": "ce"}}}})
    assert isinstance(crit["SeqCELoss"], K.SeqCELoss) and crit["SeqCELoss"].loss_type == "ce"
    fake_loss = type("FakeLossModule", (), {"loss_dict": {}})()
    fake_models = type("M", (), {})()
    K.install(kantts_models=fake_models, kantts_loss=fake_loss, kantts_audio=type("A", (), {})())
    assert fake_models.KanTtsTextsyBERT is K.KanTtsTextsyBERT
    assert fake_loss.loss_dict["SeqCELoss"] is K.SeqCELoss and fake_loss.SeqCELoss is K.SeqCELoss


def test_bert_masker_call_counter():
    m = K.BertMasker(0.3, 147, seed=7)
    assert m.mask_id == 146 and m.call_index == 0
    m.call_index = 41
    assert m.call_index == 41
    assert K.BertMasker(0.3, 147, seed=7, mask_id=5).mask_id == 5


def test_sybert_builder_shares_the_sambert_optimizer_and_noam_schedule():
    config = {"Model": {"KanTtsTextsyBERT": {"params": dict(K.sybert_config(), encoder_num_layers=1),
                                             "optimizer": {"type": "Adam", "params": {"lr": 1e-4, "betas": [0.9, 0.98],
                                                                                      "eps": 1e-9, "weight_decay": 0.0}},
                                             "scheduler": {"type": "NoamLR", "params": {"warmup_steps": 10000}}}}}
    model, opt, sch = K.sybert_model_builder(config, "cpu")
    assert isinstance(model, K.KanTtsTextsyBERT) and isinstance(opt, torch.optim.Adam)
    assert isinstance(sch, K.train.NoamLR) and sch.warmup_steps == 10000
    assert opt.param_groups[0]["betas"] == (0.9, 0.98)
