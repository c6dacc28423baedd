"""CPU: the monotonic-alignment-search (MAS) SAM-BERT variant.  The oracle restatement (oracle/sambert_mas.py) against the
goldens of the unmodified reference (tests/golden/make_golden_sambert_mas.py), the configs, the loss registration, the
module's state_dict contract and seeded init."""
import numpy as np
import pytest
import torch

import kantts_b200 as K
from conftest import rel_l2
from oracle import sambert_mas as om

OUT_KEYS = ("dec_outputs", "postnet_outputs", "log_duration_predictions", "pitch_predictions", "energy_predictions",
            "LR_text_outputs", "LR_emo_outputs", "LR_spk_outputs", "pitch_targets", "energy_targets", "attn_soft",
            "attn_logprob")
GOLDENS = ("sambert_mas_small", "sambert_mas_byte_small")


@pytest.mark.parametrize("name", GOLDENS)
def test_mas_oracle_forward_losses_grads_match_reference(golden, name):
    g = golden(name)
    sd = g.group("sd/")
    for k, v in sd.items():
        if v.dtype.is_floating_point and "position_enc" not in k and "inv_timescales" not in k:
            v.requires_grad_(True)
    b = g.group("in/")
    res = om.sambert_forward(sd, g.cfg, b["inputs_ling"], b["inputs_emotion"], b["inputs_speaker"], b["input_lengths"],
                             b["output_lengths"], b["mel_targets"], b["pitch_targets"], b["energy_targets"],
                             b["attn_priors"])
    assert torch.equal(res["attn_hard"], g.t("out/attn_hard"))
    assert torch.equal(res["duration_targets"], g.t("out/duration_targets"))
    assert torch.equal(res["LR_length_rounded"], g.t("out/LR_length_rounded"))
    assert [res["x_band_width"], res["h_band_width"]] == g.t("out/band_width").tolist()
    for k in OUT_KEYS:
        assert res[k].shape == g.t("out/" + k).shape, k
        assert rel_l2(res[k].detach(), g.t("out/" + k)) < 2e-6, (k, rel_l2(res[k].detach(), g.t("out/" + k)))
    total, parts = om.total_loss(res, b, int(g.t("out/epoch")))
    for got, w in zip(list(parts) + [total], g.t("out/losses")):
        assert abs(float(got) - float(w)) < 2e-6 * max(1.0, abs(float(w))), (float(got), float(w))
    total.backward()
    grads = g.group("grad/")
    assert any(k.startswith("align_attention.key_proj") for k in grads)
    assert not any(k.startswith("align_attention.attn_proj") for k in grads)      # never used: no gradient
    for k, w in grads.items():
        got = sd[k].grad
        assert got is not None, k
        assert rel_l2(got, w) < 2e-6 or float((got - w).abs().max()) < 1e-7, (k, rel_l2(got, w))


def test_mas_oracle_reproduces_every_reference_pattern(golden):
    g = golden("mas_patterns")
    n = g.cfg["patterns"]
    assert n >= 10
    for i in range(n):
        hard = om.b_mas(g.arrays[f"{i}/soft"], g.arrays[f"{i}/in_len"], g.arrays[f"{i}/out_len"])
        assert np.array_equal(hard, g.arrays[f"{i}/hard"]), i
        assert np.array_equal(hard.sum(2)[:, 0, :], g.arrays[f"{i}/dur"]), i
    # the one-frame and out_len < in_len patterns end with the extra hard[0][0] = 1 of the reference
    assert any(float(g.arrays[f"{i}/dur"].sum()) > float(g.arrays[f"{i}/out_len"].sum()) for i in range(n))


def test_forward_sum_loss_oracle_matches_reference(golden):
    g = golden("attn_ctc")
    for i in range(g.cfg["cases"]):
        lp = g.t(f"{i}/logprob").requires_grad_(True)
        loss = om.forward_sum_loss(lp, g.t(f"{i}/in_len"), g.t(f"{i}/out_len"))
        loss.backward()
        assert abs(float(loss) - float(g.t(f"{i}/loss"))) < 1e-6 * max(1.0, float(g.t(f"{i}/loss"))), i
        assert rel_l2(lp.grad, g.t(f"{i}/grad")) < 1e-6, i


@pytest.mark.parametrize("name", GOLDENS)
def test_binarization_loss_and_frame_average_match_oracle(golden, name):
    g = golden(name)
    hard, soft = g.t("out/attn_hard"), g.t("out/attn_soft")
    for epoch in (0, 37, 250):
        got = K.AttentionBinarizationLoss(0, 100)(epoch, hard, soft)
        want = om.binarization_loss(epoch, hard, soft)
        assert abs(float(got) - float(want)) < 1e-6 * max(1.0, abs(float(want))), epoch
    assert float(K.AttentionBinarizationLoss(50, 100)(37, hard, soft)) == 0.0
    from kantts_b200 import sambert_ops
    b = g.group("in/")
    dur = hard.sum(2)[:, 0, :]
    for k in ("pitch_targets", "energy_targets"):
        got = sambert_ops.average_frame_feat(b[k], dur)
        assert torch.equal(got, om.average_frame_feat(b[k], dur))
        assert rel_l2(got, g.t("out/" + k)) < 1e-6


def test_mas_configs_match_yamls():
    cfg = K.sambert_16k_mas_config()
    assert cfg["MAS"] is True and "FP" not in cfg
    assert {k: v for k, v in cfg.items() if k != "MAS"} == {k: v for k, v in K.sambert_24k_config().items() if k != "MAS"}
    byte = K.sambert_16k_mas_byte_config()
    assert byte["using_byte"] is True and byte["byte_index"] == 259 and byte["MAS"] is True
    assert not {"sy", "tone", "syllable_flag", "word_segment"} & set(byte)
    assert {k: v for k, v in byte.items() if k not in ("using_byte", "byte_index")} == \
        {k: v for k, v in cfg.items() if k not in ("sy", "tone", "syllable_flag", "word_segment")}


def test_mas_losses_are_built_and_registered():
    # the attention entries of the Loss sections of sambert_16k_MAS.yaml and sambert_16k_MAS_byte.yaml
    loss_cfg = {"Loss": {"AttentionCTCLoss": {"enable": True},
                         "AttentionBinarizationLoss": {"enable": True, "params": {"start_epoch": 0, "warmup_epoch": 100}}}}
    crit = K.criterion_builder(loss_cfg)
    assert isinstance(crit["AttentionCTCLoss"], K.AttentionCTCLoss) and crit["AttentionCTCLoss"].blank_logprob == -1
    kl = crit["AttentionBinarizationLoss"]
    assert isinstance(kl, K.AttentionBinarizationLoss) and (kl.start_epoch, kl.warmup_epoch) == (0, 100)
    fake = type("FakeLossModule", (), {"loss_dict": {}})()
    K.install(kantts_models=type("M", (), {})(), kantts_loss=fake, kantts_audio=type("A", (), {})())
    for name in ("AttentionCTCLoss", "AttentionBinarizationLoss"):
        assert fake.loss_dict[name] is getattr(K, name) and getattr(fake, name) is getattr(K, name)


@pytest.mark.parametrize("name", GOLDENS)
def test_mas_model_state_dict_and_seeded_init_match_reference(golden, name):
    """Same keys, order and shapes as the reference's MAS model; the weights the golden generator did not perturb (every
    one but the biases and LayerNorm parameters) equal the reference's seeded init bit for bit, ConvAttention's xavier
    re-init included."""
    g = golden(name)
    ref = g.group("sd/")
    torch.manual_seed(1234)
    m = K.KanTtsSAMBERT(g.cfg)
    sd = m.state_dict()
    assert list(sd) == list(ref)
    assert [k for k in sd if k.startswith("align_attention.")] == [
        "align_attention.attn_proj.weight", "align_attention.attn_proj.bias"] + [
        f"align_attention.{s}.{i}.conv.{p}" for s, idx in (("key_proj", (0, 2)), ("query_proj", (0, 2, 4)))
        for i in idx for p in ("weight", "bias")]
    for k in sd:
        assert sd[k].shape == ref[k].shape, k
        if not (k.endswith("bias") or "layer_norm" in k or k.endswith("ln.weight")):
            assert torch.equal(sd[k], ref[k]), k
    m.load_state_dict(ref, strict=True)


def test_mas_with_fp_and_se_stay_unbuilt():
    cfg = K.sambert_16k_mas_config()
    for extra in ({"FP": True}, {"SE": True}):
        with pytest.raises(NotImplementedError):
            K.KanTtsSAMBERT(dict(cfg, **extra))
