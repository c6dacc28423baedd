"""GPU: the alignment prior of the MAS data path (kt_attn_prior through data.AttnPriors).  Against the unmodified
reference's beta_binomial_prior_distribution (tests/golden/attn_prior.npz) pair by pair and as a collate batch, against
the float64 oracle at sambert_16k_MAS.yaml batch sizes and past the pad, repeatability, no host synchronisation, and the
MAS train step on the device prior against the same step on the reference's prior."""
import numpy as np
import pytest
import torch

import kantts_b200 as K
from oracle import attn_prior as oap
from test_gpu_sambert_mas import make_mas_batch

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _ulps(got, want):
    """|got - float32(want)| in units in the last place of float32(want) (the smallest subnormal at 0): got float32,
    want float64, either as tensors."""
    w = want.detach().cpu().numpy().astype(np.float32)
    g = got.detach().cpu().numpy()
    assert g.dtype == np.float32
    return np.abs(g.astype(np.float64) - w.astype(np.float64)) / np.spacing(np.abs(w)).astype(np.float64)


def _priors(il, ol, t_mel, t_text):
    batch = dict(valid_input_lengths=il.to(DEV), valid_output_lengths=ol.to(DEV),
                 mel_targets=torch.zeros(len(il), t_mel, 1, device=DEV),
                 input_lings=torch.zeros(len(il), t_text, 4, dtype=torch.long, device=DEV))
    out = K.AttnPriors()(batch)
    assert set(out) == set(batch) | {"attn_priors"}
    return out["attn_priors"]


def test_golden_pairs_as_one_batch(golden):
    g = golden("attn_prior")
    pairs = g.cfg["pairs"]
    il = torch.tensor([P - 1 for P, _ in pairs])
    ol = torch.tensor([M for _, M in pairs])
    T, L = int(ol.max()), int(il.max()) + 1
    got = _priors(il, ol, T, L)
    assert got.shape == (len(pairs), T, L) and got.dtype == torch.float32
    for b, (P, M) in enumerate(pairs):
        u = _ulps(got[b, :M, :P], g.t(f"pair/{P}_{M}"))
        assert u.max() <= 1.0, (P, M, float(u.max()))
        assert not got[b, M:].any() and not got[b, :, P:].any(), (P, M)


def test_golden_collate_batch(golden):
    g = golden("attn_prior")
    want = g.t("batch/attn_priors")
    B, T, L = want.shape
    got = _priors(g.t("batch/valid_input_lengths"), g.t("batch/valid_output_lengths"), T, L)
    assert got.shape == want.shape and got.dtype == want.dtype
    assert _ulps(got, want.double()).max() <= 1.0


def test_training_sized_batch_matches_oracle_and_repeats_bit_for_bit():
    batch = make_mas_batch(K.sambert_16k_mas_config(), torch.Generator().manual_seed(1234))
    il, ol = batch["valid_input_lengths"], batch["valid_output_lengths"]
    T, L = batch["mel_targets"].shape[1], batch["input_lings"].shape[1]
    assert (len(il), T, L) == (16, 1002, 200)
    dev = {k: v.to(DEV) for k, v in batch.items() if v is not None}
    first = K.AttnPriors()(dev)["attn_priors"]
    again = K.AttnPriors()(dev)["attn_priors"]
    assert torch.equal(first, again)
    assert not torch.equal(first, dev["attn_priors"])           # the batch's own prior is replaced, not read
    assert _ulps(first, oap.attn_priors(il, ol, T, L)).max() <= 1.0


@pytest.mark.parametrize("il,ol,t_mel,t_text", [
    ([29, 4], [70, 3], 50, 12),           # M > T and P > L: clipped, values from the true lengths
    ([0, 6], [1, 130], 131, 9),           # one symbol (the eos alone), one frame
    ([300], [2000], 2048, 301),           # more symbols than one pass over the columns, many row tiles
])
def test_past_the_pad_and_edge_lengths_match_oracle(il, ol, t_mel, t_text):
    il, ol = torch.tensor(il), torch.tensor(ol)
    got = _priors(il, ol, t_mel, t_text)
    assert _ulps(got, oap.attn_priors(il, ol, t_mel, t_text)).max() <= 1.0


def test_no_host_synchronisation():
    batch = {k: v.to(DEV) for k, v in make_mas_batch(K.sambert_16k_mas_config(), torch.Generator().manual_seed(3),
                                                     B=4, L=60, T=300).items() if v is not None}
    K.AttnPriors()(batch)                                        # loads the library
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = K.AttnPriors()(batch)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert out["attn_priors"].shape == batch["attn_priors"].shape


def _mas_step_on(g, batch):
    """One SambertStep of the golden model (train mode, fixed dropout seed) -> (step outputs, the hard durations)."""
    from kantts_b200 import sambert
    config = {"Model": {"KanTtsSAMBERT": {"params": g.cfg, "optimizer": {"type": "Adam", "params": {
        "lr": 1e-3, "betas": [0.9, 0.98], "eps": 1e-9, "weight_decay": 0.0}},
        "scheduler": {"type": "NoamLR", "params": {"warmup_steps": 40}}}}}
    model, opt, sch = K.sambert_model_builder(config, DEV)
    model.load_state_dict(g.group("sd/"), strict=True)
    model.train()
    crit = {"MelReconLoss": sambert.MelReconLoss(), "ProsodyReconLoss": sambert.ProsodyReconLoss(),
            "AttentionCTCLoss": sambert.AttentionCTCLoss(), "AttentionBinarizationLoss": sambert.AttentionBinarizationLoss(0, 100)}
    step = K.SambertStep(model, opt, sch, crit)
    step.epoch = int(g.t("out/epoch"))
    durations = []
    model.register_forward_hook(lambda m, i, res: durations.append(res["duration_targets"].detach().clone()))
    torch.manual_seed(77)
    out = step.step(batch)
    return out, durations[0]


def test_mas_step_on_device_priors_equals_reference_priors(golden):
    g = golden("sambert_mas_small")
    b = g.group("in/", DEV)
    batch = dict(input_lings=b["inputs_ling"], input_emotions=b["inputs_emotion"], input_speakers=b["inputs_speaker"],
                 valid_input_lengths=b["input_lengths"], valid_output_lengths=b["output_lengths"],
                 mel_targets=b["mel_targets"], durations=None, pitch_contours=b["pitch_targets"],
                 energy_contours=b["energy_targets"], attn_priors=b["attn_priors"])
    device_batch = K.AttnPriors()(batch)
    assert _ulps(device_batch["attn_priors"], b["attn_priors"].double()).max() <= 1.0
    ref_out, ref_dur = _mas_step_on(g, batch)
    out, dur = _mas_step_on(g, device_batch)
    assert torch.equal(dur, ref_dur)
    assert set(out) == set(ref_out) and "attn_ctc_loss" in out
    for k, v in ref_out.items():
        if torch.is_tensor(v):
            assert abs(float(out[k]) - float(v)) <= 1e-6 * abs(float(v)), (k, float(out[k]), float(v))
        else:
            assert out[k] == v, k
