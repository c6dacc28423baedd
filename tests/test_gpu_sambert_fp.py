"""GPU: the filled-pause (FP) SAM-BERT variant.  The insertion kernels against the reference's own index maps and torch
autograd, the model against the goldens of the unmodified reference and the CPU oracle on both compute paths, and
the training step at sambert_fp_8k.yaml sizes."""
import math

import pytest
import torch

from conftest import rel_l2

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _sops():
    from kantts_b200 import sambert_ops
    return sambert_ops


def _fp_dict(g, device="cpu"):
    return {int(k): v.to(device) for k, v in g.group("fp_dict/").items()}


def _insert(text, enc, in_len, lab=None, fpp=None):
    sops = _sops()
    codes, rows, inter, t_ins = sops.fp_insert_plan(in_len, text.shape[1], fp_label=lab, fp_p=fpp)
    return sops.FpInsertFn.apply(text, enc, codes, rows, t_ins), inter, codes, rows


@pytest.mark.parametrize("C", [2, 4])
def test_fp_insert_reproduces_reference_index_maps(golden, C):
    g = golden("fp_insert_maps")
    for i in range(g.cfg["patterns"]):
        in_len = g.t(f"{i}/in_len", DEV)
        lab = g.t(f"{i}/fp_label", DEV) if f"{i}/fp_label" in g.arrays else None
        fpp = g.t(f"{i}/fp_p", DEV).float() if lab is None else None
        B, L = in_len.shape[0], (lab if lab is not None else fpp).shape[1]
        text = torch.arange(L, device=DEV, dtype=torch.float32)[None, :, None].expand(B, L, C).contiguous()
        enc = -(1 + torch.arange(9, device=DEV, dtype=torch.float32)).reshape(3, 3, 1).expand(3, 3, C).contiguous()
        for lab_i in ((lab, lab.int()) if lab is not None else (None,)):
            out, inter, _, _ = _insert(text, enc, in_len, lab_i, fpp)
            want = g.t(f"{i}/map")
            assert out.shape == (B, want.shape[1], C), (i, out.shape)
            assert torch.equal(out.cpu().long(), want[:, :, None].expand(-1, -1, C)), i
            assert torch.equal(inter.cpu(), g.t(f"{i}/inter")), i


def _gather_reference(text, enc, codes, t_ins):
    """The same copy as an index_select over [text rows; filled-pause rows], differentiated by torch autograd."""
    B, L, C = text.shape
    c = codes[:, :t_ins].long()
    idx = torch.where(c >= 0, c + L * torch.arange(B, device=c.device)[:, None], B * L - c - 1)
    table = torch.cat([text.reshape(B * L, C), enc.reshape(9, C)], 0)
    return table.index_select(0, idx.reshape(-1)).reshape(B, t_ins, C)


@pytest.mark.parametrize("B,L,C,frac", [(3, 10, 8, 0.3), (1, 3, 5, 1.0), (4, 40, 32, 0.1), (32, 256, 32, 0.1)])
def test_fp_insert_backward_matches_autograd_and_is_deterministic(B, L, C, frac):
    g = torch.Generator().manual_seed(B * 1000 + L)
    lab = (torch.randint(1, 4, (B, L), generator=g) * (torch.rand(B, L, generator=g) < frac)).to(DEV)
    in_len = torch.tensor([L - (3 * b) % max(1, L // 2) for b in range(B)], device=DEV)
    text = torch.randn(B, L, C, generator=g).to(DEV)
    enc = torch.randn(3, 3, C, generator=g).to(DEV)
    grads = []
    for _ in range(2):
        t, e = text.clone().requires_grad_(True), enc.clone().requires_grad_(True)
        out, _, codes, _ = _insert(t, e, in_len, lab)
        dout = torch.randn(out.shape, generator=g.manual_seed(7)).to(DEV)
        (out * dout).sum().backward()
        grads.append((t.grad.clone(), e.grad.clone()))
    tr, er = text.clone().requires_grad_(True), enc.clone().requires_grad_(True)
    ref = _gather_reference(tr, er, codes, out.shape[1])
    (ref * dout).sum().backward()
    assert torch.equal(out.detach(), ref.detach())
    assert rel_l2(grads[0][0].cpu(), tr.grad.cpu()) <= 1e-6
    assert rel_l2(grads[0][1].cpu(), er.grad.cpu()) <= 1e-6
    assert torch.equal(grads[0][0], grads[1][0]) and torch.equal(grads[0][1], grads[1][1])


def _run_model(cfg, sd, batch, fp_dict, force_ffma):
    from kantts_b200 import ops, sambert
    model = sambert.KanTtsSAMBERT(cfg)
    model.load_state_dict(sd, strict=True)
    model = model.to(DEV).eval()
    model.fp_dict = fp_dict
    b = {k: v.to(DEV) for k, v in batch.items()}
    ops.set_force_ffma(force_ffma)
    try:
        with torch.backends.cudnn.flags(enabled=False):      # cuDNN refuses LSTM backward in eval mode
            res = model(b["inputs_ling"], b["inputs_emotion"], b["inputs_speaker"], b["input_lengths"],
                        output_lengths=b["output_lengths"], mel_targets=b["mel_targets"],
                        duration_targets=b["duration_targets"], pitch_targets=b["pitch_targets"],
                        energy_targets=b["energy_targets"], fp_label=b["fp_label"])
            l0, l1 = sambert.MelReconLoss()(b["output_lengths"], b["mel_targets"], res["dec_outputs"],
                                            res["postnet_outputs"])
            dl, pl, el = sambert.ProsodyReconLoss()(res["valid_inter_lengths"], res["duration_targets"],
                                                    res["pitch_targets"], res["energy_targets"],
                                                    res["log_duration_predictions"], res["pitch_predictions"],
                                                    res["energy_predictions"])
            fl = sambert.FpCELoss().to(DEV)(b["input_lengths"], res["fp_predictions"], b["fp_label"])
            total = l0 + l1 + dl + pl + el + fl
            total.backward()
    finally:
        ops.set_force_ffma(False)
    return model, res, [float(v) for v in (l0, l1, dl, pl, el, fl, total)]


OUT_KEYS = ("dec_outputs", "postnet_outputs", "log_duration_predictions", "pitch_predictions", "energy_predictions",
            "LR_text_outputs", "LR_emo_outputs", "LR_spk_outputs", "fp_predictions")


@pytest.mark.parametrize("path", ["ffma", "tcgen05"])
def test_sambert_fp_small_matches_reference_golden(golden, path):
    g = golden("sambert_fp_small")
    ffma = path == "ffma"
    tol_o, tol_g = (1e-5, 2e-4) if ffma else (1e-4, 1e-3)
    model, res, losses = _run_model(g.cfg, g.group("sd/"), g.group("in/"), _fp_dict(g, DEV), ffma)
    for k in OUT_KEYS:
        assert rel_l2(res[k].detach().cpu(), g.t("out/" + k)) < tol_o, (k, rel_l2(res[k].detach().cpu(), g.t("out/" + k)))
    assert torch.equal(res["valid_inter_lengths"].cpu(), g.t("out/valid_inter_lengths"))
    assert torch.equal(res["LR_length_rounded"].cpu(), g.t("out/LR_length_rounded"))
    assert [res["x_band_width"], res["h_band_width"]] == g.t("out/band_width").tolist()
    for k in ("enc_slf_attn_lst", "pnca_x_attn_lst", "pnca_h_attn_lst"):
        for i, a in enumerate(res[k]):
            assert rel_l2(a.cpu(), g.t(f"out/{k}.{i}")) < tol_o, (k, i)
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
    assert {"FP_predictor.fc.weight", "FP_predictor.w_1.weight", "text_encoder.sy_emb.weight"} <= checked


def _infer(cfg, sd, inputs, fp_dict, ffma):
    from kantts_b200 import ops, sambert
    ops.set_force_ffma(ffma)
    try:
        model = sambert.KanTtsSAMBERT(cfg)
        model.load_state_dict(sd, strict=True)
        model = model.to(DEV).eval()
        model.fp_dict = fp_dict
        with torch.no_grad(), torch.backends.cudnn.flags(enabled=False):
            res = model(*(inputs[k].to(DEV) for k in ("inputs_ling", "inputs_emotion", "inputs_speaker", "input_lengths")))
        torch.cuda.synchronize()
    finally:
        ops.set_force_ffma(False)
    return res


INFER_KEYS = ("fp_predictions", "log_duration_predictions", "pitch_predictions", "energy_predictions", "LR_text_outputs",
              "LR_emo_outputs", "LR_spk_outputs", "dec_outputs", "postnet_outputs")


@pytest.mark.parametrize("path", ["ffma", "tcgen05"])
def test_sambert_fp_free_running_inference_matches_reference_golden(golden, path):
    g = golden("sambert_fp_small_infer")
    res = _infer(g.cfg, g.group("sd/"), g.group("in/"), _fp_dict(g, DEV), path == "ffma")
    tol = 2e-5 if path == "ffma" else 2e-4
    assert torch.equal(res["valid_inter_lengths"].cpu(), g.t("out/valid_inter_lengths"))
    assert torch.equal(res["LR_length_rounded"].cpu(), g.t("out/LR_length_rounded"))
    for k in INFER_KEYS:
        assert res[k].shape == g.t("out/" + k).shape, (k, res[k].shape)
        assert rel_l2(res[k].cpu(), g.t("out/" + k)) < tol, (k, rel_l2(res[k].cpu(), g.t("out/" + k)))


def test_sambert_fp_free_running_inference_batch_matches_oracle(golden):
    from oracle import sambert_fp as ofp
    from golden.make_batch import make_sambert_batch
    g = golden("sambert_fp_small_infer")
    batch = make_sambert_batch(g.cfg, B=3, L=9, gen=torch.Generator().manual_seed(31), short=3)
    inputs = {k: batch[k] for k in ("inputs_ling", "inputs_emotion", "inputs_speaker", "input_lengths")}
    with torch.no_grad():
        want = ofp.sambert_infer(g.group("sd/"), g.cfg, *inputs.values(), _fp_dict(g))
    fp = want["fp_predictions"]
    top2 = fp.topk(2, dim=-1).values
    valid = torch.arange(9)[None, :] < inputs["input_lengths"][:, None]
    assert float((top2[..., 0] - top2[..., 1])[valid].min()) > 1e-3          # no filled-pause class near a tie
    assert int(want["valid_inter_lengths"].max()) > 9
    dur = torch.exp(want["log_duration_predictions"]) - 1
    frac = (dur + 0.5) - torch.floor(dur + 0.5)
    assert float(torch.minimum(frac, 1 - frac)[dur > 0].min()) > 2e-3
    res = _infer(g.cfg, g.group("sd/"), inputs, _fp_dict(g, DEV), True)
    assert torch.equal(res["valid_inter_lengths"].cpu(), want["valid_inter_lengths"])
    assert torch.equal(res["LR_length_rounded"].cpu(), want["LR_length_rounded"])
    for k in INFER_KEYS:
        assert res[k].shape == want[k].shape, (k, res[k].shape, want[k].shape)
        assert rel_l2(res[k].cpu(), want[k]) < 2e-5, (k, rel_l2(res[k].cpu(), want[k]))


def test_sambert_fp_forward_without_fp_dict_raises(golden):
    from kantts_b200 import sambert
    g = golden("sambert_fp_small_infer")
    model = sambert.KanTtsSAMBERT(g.cfg).to(DEV).eval()
    b = g.group("in/", DEV)
    with pytest.raises(RuntimeError, match="fp_dict"), torch.no_grad():
        model(b["inputs_ling"], b["inputs_emotion"], b["inputs_speaker"], b["input_lengths"])


def make_fp_batch(cfg, gen, B=16, L=256, dur=3, frac=0.1):
    """sambert_fp_8k.yaml-sized teacher-forcing batch: about ``frac`` of the symbols carry a filled-pause label, and the
    durations / pitch / energy contours are padded to the inserted length (every symbol and pause lasts ``dur``
    frames)."""
    ling = torch.stack([torch.randint(0, cfg[k], (B, L), generator=gen)
                        for k in ("sy", "tone", "syllable_flag", "word_segment")], -1)
    in_len = torch.full((B,), L - 1, dtype=torch.long)
    lab = torch.randint(1, 4, (B, L), generator=gen) * (torch.rand(B, L, generator=gen) < frac)
    lab[:, L - 1] = 0
    inter = in_len + 3 * (lab > 0).sum(1)
    T = L + int(inter.max() - in_len.max())
    durs = dur * (torch.arange(T)[None, :] < inter[:, None]).long()
    out_len = durs.sum(1)
    Tm = int(out_len.max())
    return dict(input_lings=ling, input_emotions=torch.randint(0, cfg["emotion"], (B, L), generator=gen),
                input_speakers=torch.randint(0, cfg["speaker"], (B, L), generator=gen), valid_input_lengths=in_len,
                valid_output_lengths=out_len, mel_targets=torch.randn(B, Tm, cfg["num_mels"], generator=gen),
                durations=durs, pitch_contours=torch.randn(B, T, generator=gen),
                energy_contours=torch.randn(B, T, generator=gen), fp_label=lab)


def test_sambert_fp_8k_train_step_runs_and_learns():
    import kantts_b200
    from kantts_b200 import sambert
    cfg = kantts_b200.sambert_fp_8k_config()
    gen = torch.Generator().manual_seed(1234)
    fp_dict = {k: torch.stack([torch.randint(0, cfg[n], (1, 3), generator=gen)
                               for n in ("sy", "tone", "syllable_flag", "word_segment")], -1) for k in (1, 2, 3)}
    torch.manual_seed(1234)
    config = {"Model": {"KanTtsSAMBERT": {"params": cfg, "optimizer": {"type": "Adam", "params": {
        "lr": 1e-3, "betas": [0.9, 0.98], "eps": 1e-9}}, "scheduler": {"type": "NoamLR", "params": {"warmup_steps": 40}}}}}
    model, opt, sch = kantts_b200.sambert_model_builder(config, DEV, fp_dict=fp_dict)
    model.train()
    crit = {"MelReconLoss": sambert.MelReconLoss(), "ProsodyReconLoss": sambert.ProsodyReconLoss(),
            "FpCELoss": sambert.FpCELoss().to(DEV)}
    step = kantts_b200.SambertStep(model, opt, sch, crit)
    batch = {k: v.to(DEV) for k, v in make_fp_batch(cfg, gen).items()}
    before = model.FP_predictor.fc.weight.detach().clone()
    hist, fp_hist = [], []
    for _ in range(8):
        out = step.step(batch)
        hist.append(float(out["TotalLoss"]))
        fp_hist.append(float(out["fp_loss"]))
    assert all(math.isfinite(v) for v in hist + fp_hist), (hist, fp_hist)
    assert hist[-1] < hist[0], hist
    assert not torch.equal(before, model.FP_predictor.fc.weight.detach())
