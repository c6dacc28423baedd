"""CPU: the filled-pause (FP) SAM-BERT variant.  The oracle restatement (oracle/sambert_fp.py) against the goldens of
the unmodified reference (tests/golden/make_golden_sambert_fp.py), the module's state_dict contract and seeded init,
and the loss registration."""
import torch

import kantts_b200 as K
from conftest import rel_l2
from oracle import sambert_fp as ofp

OUT_KEYS = ("dec_outputs", "postnet_outputs", "log_duration_predictions", "pitch_predictions", "energy_predictions",
            "LR_text_outputs", "LR_emo_outputs", "LR_spk_outputs", "fp_predictions")


def _fp_dict(g):
    return {int(k): v for k, v in g.group("fp_dict/").items()}


def _forward(g, sd):
    b = g.group("in/")
    res = ofp.sambert_forward(sd, g.cfg, b["inputs_ling"], b["inputs_emotion"], b["inputs_speaker"], b["input_lengths"],
                              b["output_lengths"], b["mel_targets"], b["duration_targets"], b["pitch_targets"],
                              b["energy_targets"], b["fp_label"], _fp_dict(g))
    return b, res


def test_fp_oracle_forward_losses_grads_match_reference(golden):
    g = golden("sambert_fp_small")
    sd = g.group("sd/")
    for k, v in sd.items():
        if v.dtype.is_floating_point and "position_enc" not in k and "inv_timescales" not in k:
            v.requires_grad_(True)
    b, res = _forward(g, sd)
    for k in OUT_KEYS:
        assert res[k].shape == g.t("out/" + k).shape, k
        assert rel_l2(res[k].detach(), g.t("out/" + k)) < 2e-6, (k, rel_l2(res[k].detach(), g.t("out/" + k)))
    assert torch.equal(res["valid_inter_lengths"], g.t("out/valid_inter_lengths"))
    assert torch.equal(res["LR_length_rounded"], g.t("out/LR_length_rounded"))
    assert [res["x_band_width"], res["h_band_width"]] == g.t("out/band_width").tolist()
    for k in ("enc_slf_attn_lst", "pnca_x_attn_lst", "pnca_h_attn_lst"):
        for i, a in enumerate(res[k]):
            assert rel_l2(a.detach(), g.t(f"out/{k}.{i}")) < 2e-6, (k, i)
    total, parts = ofp.total_loss(res, b)
    for got, w in zip(list(parts) + [total], g.t("out/losses")):
        assert abs(float(got) - float(w)) < 2e-6 * max(1.0, abs(float(w)))
    total.backward()
    grads = g.group("grad/")
    assert any(k.startswith("FP_predictor.") for k in grads)
    for k, w in grads.items():
        got = sd[k].grad
        assert got is not None, k
        assert rel_l2(got, w) < 2e-6 or float((got - w).abs().max()) < 1e-7, (k, rel_l2(got, w))


def test_fp_oracle_free_running_inference_matches_reference(golden):
    g = golden("sambert_fp_small_infer")
    b = g.group("in/")
    with torch.no_grad():
        res = ofp.sambert_infer(g.group("sd/"), g.cfg, b["inputs_ling"], b["inputs_emotion"], b["inputs_speaker"],
                                b["input_lengths"], _fp_dict(g))
    assert torch.equal(res["valid_inter_lengths"], g.t("out/valid_inter_lengths"))
    assert torch.equal(res["LR_length_rounded"], g.t("out/LR_length_rounded"))
    for k in OUT_KEYS:
        assert res[k].shape == g.t("out/" + k).shape, (k, res[k].shape)
        assert rel_l2(res[k], g.t("out/" + k)) < 5e-6, (k, rel_l2(res[k], g.t("out/" + k)))


def test_fp_oracle_reproduces_every_index_map(golden):
    g = golden("fp_insert_maps")
    n = g.cfg["patterns"]
    assert n >= 19
    n_ties = 0
    for i in range(n):
        in_len = g.t(f"{i}/in_len")
        lab = g.t(f"{i}/fp_label") if f"{i}/fp_label" in g.arrays else None
        fpp = g.t(f"{i}/fp_p") if lab is None else None
        want = g.t(f"{i}/map")
        B, L = in_len.shape[0], (lab if lab is not None else fpp).shape[1]
        text = torch.arange(L, dtype=torch.float32)[None, :, None].expand(B, L, 1)
        enc = -(1 + torch.arange(9, dtype=torch.float32)).reshape(3, 3, 1)
        out, inter, ext = ofp.fp_insert(text, enc, in_len, fp_label=lab, fp_p=fpp)
        assert torch.equal(out[:, :, 0].long(), want), i
        assert torch.equal(inter, g.t(f"{i}/inter")), i
        assert torch.equal(ext.expand(B, -1), g.t(f"{i}/ext")), i
        n_ties += lab is None
    assert n_ties >= 3


def test_fp_model_state_dict_and_seeded_init_match_reference(golden):
    """Same keys, order and shapes as the reference's FP model; the weights the golden generator did not perturb (every
    one but the biases and LayerNorm parameters) equal the reference's seeded init bit for bit."""
    g = golden("sambert_fp_small")
    ref = g.group("sd/")
    torch.manual_seed(1234)
    m = K.KanTtsSAMBERT(g.cfg)
    sd = m.state_dict()
    assert list(sd) == list(ref)
    assert [k for k in sd if k.startswith("FP_predictor.")] == [
        f"FP_predictor.{n}.{p}" for n in ("w_1", "w_2", "layer_norm1", "layer_norm2", "fc") for p in ("weight", "bias")]
    for k in sd:
        assert sd[k].shape == ref[k].shape, k
        if not (k.endswith("bias") or "layer_norm" in k or k.endswith("ln.weight")):
            assert torch.equal(sd[k], ref[k]), k
    m.load_state_dict(ref, strict=True)


def test_fp_loss_matches_oracle_and_is_registered(golden):
    g = golden("sambert_fp_small")
    b = g.group("in/")
    fp_pd = g.t("out/fp_predictions")
    crit = K.FpCELoss(loss_type="ce", weight=[1, 4, 4, 8])
    got = crit(b["input_lengths"], fp_pd, b["fp_label"])
    want = ofp.fp_ce_loss(b["input_lengths"], fp_pd, b["fp_label"])
    assert abs(float(got) - float(want)) < 1e-6
    assert abs(float(got) - float(g.t("out/losses")[5])) < 2e-6
    assert [n for n, _ in crit.named_buffers()] == ["weight"]
    crit = K.criterion_builder({"Loss": {"FpCELoss": {"enable": True, "params": {"loss_type": "ce",
                                                                                 "weight": [1, 4, 4, 8]}}}})
    assert isinstance(crit["FpCELoss"], K.FpCELoss)
    fake = type("FakeLossModule", (), {"loss_dict": {}})()
    K.install(kantts_models=type("M", (), {})(), kantts_loss=fake, kantts_audio=type("A", (), {})())
    assert fake.loss_dict["FpCELoss"] is K.FpCELoss and fake.FpCELoss is K.FpCELoss


def test_fp_config_and_variants():
    cfg = K.sambert_fp_8k_config()
    assert cfg["FP"] is True and cfg["speaker"] == 6
    assert {k: v for k, v in cfg.items() if k not in ("FP", "speaker")} == \
        {k: v for k, v in K.sambert_24k_config().items() if k != "speaker"}
    for flag in ("SE", "MAS"):
        try:
            K.KanTtsSAMBERT(dict(cfg, **{flag: True}))
        except NotImplementedError:
            continue
        raise AssertionError(f"{flag}=True must stay unbuilt")
