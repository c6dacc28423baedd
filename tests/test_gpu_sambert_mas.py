"""GPU: the monotonic-alignment-search (MAS) SAM-BERT variant.  kt_mas against the reference's own maps and the oracle
DP, the alignment attention and the forward-sum loss against the oracle and torch autograd, the model against the goldens
of the unmodified reference on both compute paths, the train step at sambert_16k_MAS.yaml sizes and inference."""
import math

import numpy as np
import pytest
import torch

from conftest import rel_l2

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _sops():
    from kantts_b200 import sambert_ops
    return sambert_ops


def test_mas_kernel_reproduces_reference_patterns(golden):
    g = golden("mas_patterns")
    for i in range(g.cfg["patterns"]):
        soft = g.t(f"{i}/soft", DEV)
        hard, dur = _sops().mas(soft, g.t(f"{i}/in_len", DEV), g.t(f"{i}/out_len", DEV))
        assert torch.equal(hard.cpu(), g.t(f"{i}/hard")), i
        assert torch.equal(dur.cpu(), g.t(f"{i}/dur")), i


def _random_maps(B, T, N, gen, sharp=8.0):
    """Peaked soft maps (softmax of a monotone-ish score plus noise) with ragged lengths."""
    i = torch.arange(T, dtype=torch.float64)[:, None] / T
    j = torch.arange(N, dtype=torch.float64)[None, :] / N
    logits = -sharp * N * (i - j).abs() + torch.randn(B, T, N, generator=gen, dtype=torch.float64)
    soft = torch.softmax(logits, -1).float()
    in_len = torch.tensor([N - (b * 7) % max(1, N // 3) for b in range(B)])
    out_len = torch.tensor([T - (b * 13) % max(1, T // 4) for b in range(B)])
    for b in range(B):
        soft[b, :, in_len[b]:] = 0.0
        soft[b, :, : in_len[b]] /= soft[b, :, : in_len[b]].sum(-1, keepdim=True)
    return soft[:, None], in_len, out_len


@pytest.mark.parametrize("B,T,N", [(3, 50, 17), (16, 1000, 200), (4, 333, 97), (2, 3000, 300)])
def test_mas_kernel_matches_oracle_dp_on_random_maps(B, T, N):
    from oracle import sambert_mas as om
    from kantts_b200 import _lib
    soft, in_len, out_len = _random_maps(B, T, N, torch.Generator().manual_seed(B * T + N))
    for b in range(B):
        margin = om.mas_margin(soft[b, 0, : int(out_len[b]), : int(in_len[b])].numpy())
        assert margin > 1e-3, (b, margin)
    if (B, T, N) == (2, 3000, 300):
        assert _lib.load().kt_mas_workspace_bytes(B, T, N) > 0           # the bits go to the global workspace
    want = om.b_mas(soft.numpy(), in_len.numpy(), out_len.numpy())
    runs = [_sops().mas(soft.to(DEV), in_len.to(DEV), out_len.to(DEV)) for _ in range(2)]
    assert torch.equal(runs[0][0].cpu(), torch.from_numpy(want))
    assert torch.equal(runs[0][1].cpu(), torch.from_numpy(want.sum(2)[:, 0, :]))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])


def _attn_inputs(B, Tq, Tk, C, gen, prior):
    q = torch.randn(B, Tq, C, generator=gen) * 3
    k = torch.randn(B, Tk, C, generator=gen) * 3
    kl = torch.tensor([Tk - (3 * b) % max(1, Tk // 2) for b in range(B)])
    pr = torch.rand(B, Tq, Tk, generator=gen) if prior else None
    if pr is not None:
        pr[0, :, -1] = 0.0                                   # zero prior cells: log(1e-8)
    return q, k, kl, pr


@pytest.mark.parametrize("prior", [False, True])
@pytest.mark.parametrize("B,Tq,Tk,C", [(3, 37, 11, 8), (2, 130, 45, 80), (1, 64, 33, 128)])
def test_align_attention_matches_oracle_and_autograd(B, Tq, Tk, C, prior):
    from oracle import sambert_mas as om
    gen = torch.Generator().manual_seed(B * 100 + Tq + Tk + C + prior)
    q, k, kl, pr = _attn_inputs(B, Tq, Tk, C, gen, prior)
    mask = torch.arange(Tk)[None, :] >= kl[:, None]
    ds = torch.randn(B, 1, Tq, Tk, generator=gen)
    dl = torch.randn(B, 1, Tq, Tk, generator=gen)
    qd, kd = q.double().requires_grad_(True), k.double().requires_grad_(True)
    soft_o, lp_o = om.distance_attention(qd, kd, mask, None if pr is None else pr.double())
    for which in ("soft", "logprob", "both"):
        gs = ds if which in ("soft", "both") else None
        gl = dl if which in ("logprob", "both") else None
        outs = []
        for _ in range(2):
            qg, kg = q.to(DEV).requires_grad_(True), k.to(DEV).requires_grad_(True)
            soft, lp = _sops().AlignAttnFn.apply(qg, kg, None if pr is None else pr.to(DEV), kl.to(DEV))
            torch.autograd.backward([t for t, gr in ((soft, gs), (lp, gl)) if gr is not None],
                                    [gr.to(DEV) for gr in (gs, gl) if gr is not None])
            outs.append((soft.detach(), lp.detach(), qg.grad, kg.grad))
        for a, b in zip(outs[0], outs[1]):
            assert torch.equal(a, b)                             # bit-identical runs
        soft, lp, dq, dk = (t.cpu() for t in outs[0])
        assert rel_l2(soft, soft_o.detach()) < 1e-6 and rel_l2(lp, lp_o.detach()) < 1e-6
        qd.grad = kd.grad = None
        torch.autograd.backward([t for t, gr in ((soft_o, gs), (lp_o, gl)) if gr is not None],
                                [gr.double() for gr in (gs, gl) if gr is not None], retain_graph=True)
        assert rel_l2(dq, qd.grad) < 1e-5, (which, rel_l2(dq, qd.grad))
        assert rel_l2(dk, kd.grad) < 1e-5, (which, rel_l2(dk, kd.grad))


def test_attn_ctc_matches_reference_golden_and_float64_ctc(golden):
    from oracle import sambert_mas as om
    g = golden("attn_ctc")
    for i in range(g.cfg["cases"]):
        lp, il, ol = g.t(f"{i}/logprob"), g.t(f"{i}/in_len"), g.t(f"{i}/out_len")
        res = []
        for _ in range(2):
            x = lp.to(DEV).requires_grad_(True)
            loss = _sops().AttnCtcFn.apply(x, il.to(DEV), ol.to(DEV), -1.0)
            loss.backward()
            res.append((loss.detach(), x.grad))
        assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1])   # deterministic
        loss, grad = float(res[0][0]), res[0][1].cpu()
        want = float(g.t(f"{i}/loss"))
        assert abs(loss - want) <= 1e-5 * max(1.0, abs(want)), (i, loss, want)
        assert rel_l2(grad, g.t(f"{i}/grad")) <= 1e-5, (i, rel_l2(grad, g.t(f"{i}/grad")))
        x64 = lp.double().requires_grad_(True)
        l64 = om.forward_sum_loss(x64, il, ol)
        l64.backward()
        assert abs(loss - float(l64)) <= 1e-5 * max(1.0, abs(float(l64)))
        assert rel_l2(grad, x64.grad) <= 1e-5, (i, rel_l2(grad, x64.grad))
        if i == 0:
            assert float(grad[2].abs().max()) == 0.0             # out_len < in_len: zero_infinity


def _run_model(cfg, sd, batch, epoch, force_ffma):
    from kantts_b200 import ops, sambert
    model = sambert.KanTtsSAMBERT(cfg)
    model.load_state_dict(sd, strict=True)
    model = model.to(DEV).eval()
    b = {k: v.to(DEV) for k, v in batch.items()}
    ops.set_force_ffma(force_ffma)
    try:
        with torch.backends.cudnn.flags(enabled=False):      # cuDNN refuses LSTM backward in eval mode
            res = model(b["inputs_ling"], b["inputs_emotion"], b["inputs_speaker"], b["input_lengths"],
                        output_lengths=b["output_lengths"], mel_targets=b["mel_targets"],
                        pitch_targets=b["pitch_targets"], energy_targets=b["energy_targets"],
                        attn_priors=b["attn_priors"])
            l0, l1 = sambert.MelReconLoss()(b["output_lengths"], b["mel_targets"], res["dec_outputs"],
                                            res["postnet_outputs"])
            dl, pl, el = sambert.ProsodyReconLoss()(res["valid_inter_lengths"], res["duration_targets"],
                                                    res["pitch_targets"], res["energy_targets"],
                                                    res["log_duration_predictions"], res["pitch_predictions"],
                                                    res["energy_predictions"])
            ctc = sambert.AttentionCTCLoss()(res["attn_logprob"], b["input_lengths"], b["output_lengths"])
            kl = sambert.AttentionBinarizationLoss(0, 100)(epoch, res["attn_hard"], res["attn_soft"])
            total = l0 + l1 + dl + pl + el + ctc + kl
            total.backward()
    finally:
        ops.set_force_ffma(False)
    return model, res, [float(v) for v in (l0, l1, dl, pl, el, ctc, kl, total)]


OUT_KEYS = ("dec_outputs", "postnet_outputs", "log_duration_predictions", "pitch_predictions", "energy_predictions",
            "LR_text_outputs", "LR_emo_outputs", "LR_spk_outputs", "pitch_targets", "energy_targets", "attn_soft",
            "attn_logprob")


@pytest.mark.parametrize("name", ["sambert_mas_small", "sambert_mas_byte_small"])
@pytest.mark.parametrize("path", ["ffma", "tcgen05"])
def test_sambert_mas_small_matches_reference_golden(golden, name, path):
    g = golden(name)
    ffma = path == "ffma"
    tol_o, tol_g = (1e-5, 2e-4) if ffma else (1e-4, 1e-3)
    model, res, losses = _run_model(g.cfg, g.group("sd/"), g.group("in/"), int(g.t("out/epoch")), ffma)
    assert torch.equal(res["attn_hard"].cpu(), g.t("out/attn_hard"))
    assert torch.equal(res["duration_targets"].cpu(), g.t("out/duration_targets"))
    assert torch.equal(res["LR_length_rounded"].cpu(), g.t("out/LR_length_rounded"))
    assert [res["x_band_width"], res["h_band_width"]] == g.t("out/band_width").tolist()
    for k in OUT_KEYS:
        assert rel_l2(res[k].detach().cpu(), g.t("out/" + k)) < tol_o, (k, rel_l2(res[k].detach().cpu(), g.t("out/" + k)))
    for got, w in zip(losses, g.t("out/losses").tolist()):
        assert abs(got - w) < 1e-4 * max(1.0, abs(w)), (losses, g.t("out/losses").tolist())
    named = dict(model.named_parameters())
    checked = set()
    for k, w in g.group("grad/").items():
        got = named[k].grad
        assert got is not None, k
        if float(w.abs().max()) > 1e-6:
            assert rel_l2(got.cpu(), w) < tol_g, (k, rel_l2(got.cpu(), w))
            checked.add(k)
    assert {"align_attention.key_proj.0.conv.weight", "align_attention.query_proj.4.conv.weight"} <= checked
    assert named["align_attention.attn_proj.weight"].grad is None


def make_mas_batch(cfg, gen, B=16, L=200, T=1000):
    """sambert_16k_MAS.yaml-sized teacher-forcing batch without durations: ragged symbol and frame counts, priors like the
    collate's (a diagonal band standing in for the beta-binomial), frame-level pitch / energy."""
    r = cfg["outputs_per_step"]
    in_len = torch.tensor([L - 1 - (17 * b) % (L // 2) for b in range(B)])
    out_len = torch.tensor([T - (37 * b) % (T // 3) for b in range(B)])
    Tm = -(-int(out_len.max()) // r) * r
    if cfg.get("using_byte"):
        ling = torch.randint(0, cfg["byte_index"], (B, L, 1), generator=gen)
    else:
        ling = torch.stack([torch.randint(0, cfg[k], (B, L), generator=gen)
                            for k in ("sy", "tone", "syllable_flag", "word_segment")], -1)
    valid = torch.arange(Tm)[None, :] < out_len[:, None]
    prior = torch.zeros(B, Tm, L)
    for b in range(B):
        n, t = int(in_len[b]) + 1, int(out_len[b])
        i = torch.arange(t, dtype=torch.float64)[:, None] * n / t
        p = torch.exp(-0.5 * (torch.arange(n, dtype=torch.float64)[None, :] - i) ** 2)
        prior[b, :t, :n] = (p / p.sum(1, keepdim=True)).float()
    return dict(input_lings=ling, input_emotions=torch.randint(0, cfg["emotion"], (B, L), generator=gen),
                input_speakers=torch.randint(0, cfg["speaker"], (B, L), generator=gen), valid_input_lengths=in_len,
                valid_output_lengths=out_len, mel_targets=torch.randn(B, Tm, cfg["num_mels"], generator=gen) * valid[..., None],
                durations=None, pitch_contours=torch.rand(B, Tm, generator=gen) * valid,
                energy_contours=torch.rand(B, Tm, generator=gen) * valid, attn_priors=prior)


def _mas_step(cfg, batch, steps, epoch=10):
    import kantts_b200
    from kantts_b200 import sambert
    torch.manual_seed(1234)
    config = {"Model": {"KanTtsSAMBERT": {"params": cfg, "optimizer": {"type": "Adam", "params": {
        "lr": 1e-3, "betas": [0.9, 0.98], "eps": 1e-9, "weight_decay": 0.0}},
        "scheduler": {"type": "NoamLR", "params": {"warmup_steps": 40}}}}}
    model, opt, sch = kantts_b200.sambert_model_builder(config, DEV)
    model.train()
    crit = {"MelReconLoss": sambert.MelReconLoss(), "ProsodyReconLoss": sambert.ProsodyReconLoss(),
            "AttentionCTCLoss": sambert.AttentionCTCLoss(), "AttentionBinarizationLoss": sambert.AttentionBinarizationLoss(0, 100)}
    step = kantts_b200.SambertStep(model, opt, sch, crit)
    step.epoch = epoch
    proj = model.align_attention.attn_proj.weight.detach().clone()
    outs = []
    for _ in range(steps):
        torch.manual_seed(77)                                  # the same dropout masks in both runs
        outs.append(step.step(batch))
    assert torch.equal(proj, model.align_attention.attn_proj.weight.detach())
    return model, outs


def test_sambert_16k_mas_train_step_is_finite_deterministic_and_aligns():
    import kantts_b200
    cfg = kantts_b200.sambert_16k_mas_config()
    batch = {k: (v.to(DEV) if v is not None else None) for k, v in make_mas_batch(cfg, torch.Generator().manual_seed(5)).items()}
    m1, o1 = _mas_step(cfg, batch, 1)
    m2, o2 = _mas_step(cfg, batch, 1)
    for out in o1:
        for k in ("TotalLoss", "attn_ctc_loss", "attn_kl_loss", "dur_loss"):
            assert math.isfinite(float(out[k])), (k, out)
        assert float(out["attn_kl_loss"]) > 0.0
    for k, v in o1[0].items():
        assert (torch.equal(v, o2[0][k]) if torch.is_tensor(v) else v == o2[0][k]), k
    # The embedding tables are updated by torch's embedding backward, which sums the rows of repeated ids in no fixed
    # order; every other parameter, the alignment path's included, comes out of one step bit for bit the same.
    tables = ("text_encoder.sy_emb.", "text_encoder.tone_emb.", "text_encoder.syllable_flag_emb.", "text_encoder.ws_emb.",
              "spk_tokenizer.", "emo_tokenizer.")
    compared = 0
    for (n, p1), p2 in zip(m1.named_parameters(), m2.parameters()):
        if not n.startswith(tables):
            assert torch.equal(p1, p2), n
            compared += 1
    assert compared > 100
    with torch.no_grad(), torch.backends.cudnn.flags(enabled=False):
        m1.eval()
        res = m1(batch["input_lings"], batch["input_emotions"], batch["input_speakers"], batch["valid_input_lengths"],
                 output_lengths=batch["valid_output_lengths"], mel_targets=batch["mel_targets"],
                 pitch_targets=batch["pitch_contours"], energy_targets=batch["energy_contours"],
                 attn_priors=batch["attn_priors"])
    T = batch["mel_targets"].shape[1]
    assert torch.equal(res["duration_targets"].sum(1).cpu(), torch.full((16,), float(T)))
    hard = res["attn_hard"][:, 0]
    assert torch.equal(hard.sum(2).cpu(), (torch.arange(T)[None, :] < batch["valid_output_lengths"].cpu()[:, None]).float())


def test_sambert_16k_mas_byte_train_step_runs():
    import kantts_b200
    cfg = kantts_b200.sambert_16k_mas_byte_config()
    batch = {k: (v.to(DEV) if v is not None else None)
             for k, v in make_mas_batch(cfg, torch.Generator().manual_seed(6), B=4, L=120, T=500).items()}
    model, outs = _mas_step(cfg, batch, 1)
    assert all(math.isfinite(float(v)) for k, v in outs[0].items() if torch.is_tensor(v))
    assert model.text_encoder.byte_index_emb.weight.grad.abs().sum() > 0


def test_mas_rejects_lengths_without_a_padding_symbol(golden):
    from kantts_b200 import sambert
    g = golden("sambert_mas_small")
    model = sambert.KanTtsSAMBERT(g.cfg).to(DEV).eval()
    b = g.group("in/", DEV)
    bad = b["input_lengths"].clone()
    bad[1] = b["inputs_ling"].shape[1]
    with pytest.raises(ValueError, match="input_lengths"), torch.no_grad():
        model(b["inputs_ling"], b["inputs_emotion"], b["inputs_speaker"], bad, output_lengths=b["output_lengths"],
              mel_targets=b["mel_targets"], pitch_targets=b["pitch_targets"], energy_targets=b["energy_targets"],
              attn_priors=b["attn_priors"])


def test_mas_model_inference_equals_plain_model(golden):
    """Inference (no mel targets) does not run the alignment: synthesize on a MAS model equals the MAS-off model loaded
    with the same weights minus align_attention.*."""
    import kantts_b200 as K
    from kantts_b200 import sambert
    g = golden("sambert_mas_small")
    sd = g.group("sd/")
    mas = sambert.KanTtsSAMBERT(g.cfg).eval()
    mas.load_state_dict(sd, strict=True)
    plain = sambert.KanTtsSAMBERT(dict(g.cfg, MAS=False)).eval()
    plain.load_state_dict({k: v for k, v in sd.items() if not k.startswith("align_attention.")}, strict=True)
    with torch.no_grad():                      # durations long enough for a few frames per symbol, in both models
        for m in (mas, plain):
            m.variance_adaptor.duration_predictor.fc.bias.fill_(1.25)
    torch.manual_seed(3)
    gen = K.Generator(in_channels=g.cfg["num_mels"], channels=32).to(DEV).eval()
    b = g.group("in/", DEV)
    inputs = [b[k][:2] for k in ("inputs_ling", "inputs_emotion", "inputs_speaker", "input_lengths")]
    outs = []
    for m in (mas.to(DEV), plain.to(DEV)):
        with torch.no_grad(), torch.backends.cudnn.flags(enabled=False):
            wavs, res = K.synthesize(m, gen, *inputs)
        assert "attn_hard" not in res
        outs.append((wavs, res))
    for k in ("dec_outputs", "postnet_outputs", "log_duration_predictions"):
        assert torch.equal(outs[0][1][k], outs[1][1][k]), k
    for w0, w1 in zip(outs[0][0], outs[1][0]):
        assert torch.equal(w0, w1)
