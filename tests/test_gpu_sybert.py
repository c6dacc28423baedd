"""GPU: the masked-symbol pretraining model of sybert.yaml.  SeqCELoss's kernels against a float64 torch composite, the model
against the golden of the unmodified reference on both compute paths, kt_bert_mask bit for bit against its oracle
restatement and statistically against the reference's rule, and the train step at sybert.yaml sizes."""
import math

import numpy as np
import pytest
import torch

from conftest import rel_l2

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _composite(logits, targets, masks):
    from oracle import sybert as osy
    return osy.seq_ce_loss(logits, targets, masks)


def _ce_inputs(B, L, V, gen):
    logits = torch.randn(B, L, V, generator=gen) * 3
    targets = torch.randint(0, V, (B, L), generator=gen)
    lens = torch.tensor([L - (7 * b) % max(1, L // 2) for b in range(B)])
    masks = ((torch.rand(B, L, generator=gen) < 0.4) & (torch.arange(L)[None, :] < lens[:, None])).float()
    masks[0, 0] = 1.0
    if V > 1:                                      # exact ties of the row maximum: torch.argmax takes the first index
        top = logits.amax(-1) + 1.0
        for b in range(B):
            for i in range(0, L, 3):
                j1, j2 = sorted(torch.randperm(V, generator=gen)[:2].tolist())
                logits[b, i, j1] = logits[b, i, j2] = top[b, i]
                targets[b, i] = j1 if (i // 3) % 2 else j2
                masks[b, i] = 1.0
    return logits, targets, masks


@pytest.mark.parametrize("V", [1, 5, 147, 2000])
def test_seq_ce_matches_float64_composite_and_is_deterministic(V):
    from kantts_b200 import sambert
    gen = torch.Generator().manual_seed(V)
    logits, targets, masks = _ce_inputs(4, 37, V, gen)
    runs = []
    for _ in range(2):
        x = logits.to(DEV).requires_grad_(True)
        loss, err = sambert.SeqCELoss()(x, targets.to(DEV), masks.to(DEV))
        assert loss.shape == () and err.shape == () and not err.requires_grad
        (loss * 0.37).backward()
        runs.append((loss.detach(), err, x.grad))
    for a, b in zip(runs[0], runs[1]):
        assert torch.equal(a, b)                           # bit-identical calls
    x64 = logits.double().requires_grad_(True)
    l64, e64 = _composite(x64, targets, masks.double())
    (l64 * 0.37).backward()
    loss, err, grad = (t.cpu() for t in runs[0])
    want = float(l64.detach())
    assert abs(float(loss) - want) <= 2e-6 * abs(want) + 1e-7, (float(loss), want)
    assert float(err) == pytest.approx(float(e64), abs=1e-7)
    assert rel_l2(grad, x64.grad) < 1e-5 if V > 1 else float(grad.abs().max()) < 1e-7
    if V == 1:
        assert float(loss) == 0.0 and float(err) == 0.0
    else:
        assert 0.0 < float(err) < 1.0


def test_seq_ce_argmax_ties_take_the_first_index():
    from kantts_b200 import sambert
    logits = torch.zeros(1, 4, 6)
    logits[0, :, 2] = logits[0, :, 4] = 5.0
    targets = torch.tensor([[2, 4, 2, 4]])
    masks = torch.tensor([[1.0, 1.0, 0.0, 1.0]])
    _, err = sambert.SeqCELoss()(logits.to(DEV), targets.to(DEV), masks.to(DEV))
    assert float(err) == pytest.approx(2.0 / 3.0, abs=1e-7)      # the rows whose target is the second maximum are wrong


def test_seq_ce_masks_of_any_dtype_and_an_empty_mask():
    from kantts_b200 import sambert
    gen = torch.Generator().manual_seed(9)
    logits, targets, masks = _ce_inputs(2, 11, 7, gen)
    want = sambert.SeqCELoss()(logits.to(DEV), targets.to(DEV), masks.to(DEV))
    for m in (masks.bool(), masks.long(), masks.to(torch.int32)):
        got = sambert.SeqCELoss()(logits.to(DEV), targets.to(DEV), m.to(DEV))
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
    x = logits.to(DEV).requires_grad_(True)
    loss, err = sambert.SeqCELoss()(x, targets.to(DEV), torch.zeros_like(masks).to(DEV))
    assert math.isnan(float(loss.detach())) and math.isnan(float(err))
    rl, re = _composite(logits, targets, torch.zeros_like(masks))
    assert math.isnan(float(rl)) and math.isnan(float(re))


def test_seq_ce_and_bert_masker_do_not_synchronise():
    import kantts_b200 as K
    gen = torch.Generator().manual_seed(4)
    logits, targets, masks = _ce_inputs(3, 50, 147, gen)
    x = logits.to(DEV).requires_grad_(True)
    t, m = targets.to(DEV), masks.to(DEV)
    lings = torch.randint(0, 144, (3, 50, 4), generator=gen).to(DEV)
    lens = torch.tensor([49, 20, 33]).to(DEV)
    masker = K.BertMasker(0.3, 147, seed=1)
    crit = K.SeqCELoss()
    crit(x, t, m)                                          # library loaded, workspace sizes known
    masker({"input_lings": lings, "valid_input_lengths": lens})
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss, err = crit(x, t, m)
        loss.backward()
        masker({"input_lings": lings, "valid_input_lengths": lens})
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


def _run_model(cfg, sd, batch, force_ffma):
    from kantts_b200 import ops, sambert
    model = sambert.KanTtsTextsyBERT(cfg)
    model.load_state_dict(sd, strict=True)
    model = model.to(DEV).eval()
    b = {k: v.to(DEV) for k, v in batch.items()}
    ops.set_force_ffma(force_ffma)
    try:
        res = model(b["input_lings"], b["valid_input_lengths"])
        loss, err = sambert.SeqCELoss()(res["logits"], b["targets"], b["bert_masks"])
        (loss / res["logits"].size(-1)).backward()
    finally:
        ops.set_force_ffma(False)
    return model, res, float(loss), float(err)


@pytest.mark.parametrize("path", ["ffma", "tcgen05"])
def test_sybert_small_matches_reference_golden(golden, path):
    g = golden("sybert_small")
    ffma = path == "ffma"
    tol_o, tol_g = (1e-5, 2e-4) if ffma else (1e-4, 1e-3)
    model, res, loss, err = _run_model(g.cfg, g.group("sd/"), g.group("in/"), ffma)
    assert rel_l2(res["logits"].detach().cpu(), g.t("out/logits")) < tol_o
    assert len(res["enc_slf_attn_lst"]) == g.cfg["encoder_num_layers"]
    for i, a in enumerate(res["enc_slf_attn_lst"]):
        want = g.t(f"out/enc_slf_attn_lst.{i}")
        assert a.shape == want.shape, (a.shape, want.shape)
        assert rel_l2(a.detach().cpu(), want) < tol_o, i
    want_loss, want_err = g.t("out/loss_err").tolist()
    assert abs(loss - want_loss) < 1e-4 * want_loss and err == pytest.approx(want_err, abs=1e-7)
    named = dict(model.named_parameters())
    checked = set()
    for k, w in g.group("grad/").items():
        got = named[k].grad
        assert got is not None, k
        if float(w.abs().max()) > 1e-6:
            assert rel_l2(got.cpu(), w) < tol_g, (k, rel_l2(got.cpu(), w))
            checked.add(k)
    assert {"fc.weight", "fc.bias", "text_encoder.sy_emb.weight", "text_encoder.ling_enc.fft.0.slf_attn.w_qkv.weight"} <= checked


def _lings(B, L, lens, gen, n_sy=147):
    """(B, L, 4) int64: symbols in [0, n_sy - 3), eos n_sy - 2 at position lens[b], the sy pad id n_sy - 3 after it."""
    x = torch.stack([torch.randint(0, n_sy - 3, (B, L), generator=gen)] +
                    [torch.randint(0, 8, (B, L), generator=gen) for _ in range(3)], -1)
    for b, n in enumerate(lens):
        if n < L:
            x[b, n, 0] = n_sy - 2
            x[b, n + 1:, 0] = n_sy - 3
    return x


@pytest.mark.parametrize("seed,call", [(0, 0), (1234, 7), (2 ** 63 + 12345, 2 ** 32 + 3), (99, 2 ** 64 - 1)])
def test_bert_masker_equals_oracle_bit_for_bit(seed, call):
    import kantts_b200 as K
    from oracle import sybert as osy
    gen = torch.Generator().manual_seed(seed % 1000 + call % 1000)
    B, L = 9, 300
    lens = [299, 64, 1, 0, 150, 256, 200, 17, 298]
    lings = _lings(B, L, lens, gen)
    masker = K.BertMasker(0.3, 147, seed=seed)
    masker.call_index = call
    out = masker({"input_lings": lings.to(DEV), "valid_input_lengths": torch.tensor(lens).to(DEV), "extra": 5})
    assert masker.call_index == call + 1 and out["extra"] == 5
    want = osy.bert_mask(lings.numpy(), lens, seed, call, 0.3, 147, 146)
    assert np.array_equal(out["input_lings"].cpu().numpy(), want[0])
    assert np.array_equal(out["targets"].cpu().numpy(), want[1])
    assert np.array_equal(out["bert_masks"].cpu().numpy(), want[2])
    assert out["bert_masks"].dtype == torch.float32 and out["targets"].dtype == torch.int64


def test_bert_masker_invariants():
    import kantts_b200 as K
    from oracle import sybert as osy
    gen = torch.Generator().manual_seed(21)
    B, L = 16, 260
    lens = [64 + (37 * b) % 190 for b in range(B)]
    lings = _lings(B, L, lens, gen)
    masker = K.BertMasker(0.3, 147, seed=5)
    for _ in range(4):
        out = masker({"input_lings": lings.to(DEV), "valid_input_lengths": torch.tensor(lens).to(DEV)})
        x, t, m = (out[k].cpu() for k in ("input_lings", "targets", "bert_masks"))
        assert torch.equal(t, lings[:, :, 0]) and torch.equal(x[:, :, 1:], lings[:, :, 1:])
        assert set(m.unique().tolist()) <= {0.0, 1.0}
        for b, n_valid in enumerate(lens):
            sel = m[b] == 1
            assert not sel[n_valid:].any()                             # eos and padding are never selected
            assert torch.equal(x[b, ~sel, 0], lings[b, ~sel, 0])
            n = int(sel.sum())
            n_mask, n_rand = osy.masking_counts(n)
            xs, os_ = x[b, sel, 0], lings[b, sel, 0]
            replaced = xs[(xs != 146) & (xs != os_)]
            assert replaced.unique().numel() <= 1                     # one replacement id per utterance
            assert replaced.numel() <= n_rand
            k = int((xs == 146).sum())
            assert k == n_mask or k == n_mask + n_rand, (k, n_mask, n_rand)
            assert int((xs == os_).sum()) >= n - n_mask - n_rand


def test_bert_masker_selection_rate_and_uniform_choice():
    """Selected with probability mask_ratio; given n selected, each position is equally likely to be a mask, a replacement
    or a kept symbol.  Symbols 500.. and mask id 1000 lie outside the replacement range [0, 147), so the three outcomes are
    told apart exactly.  Fixed seed: the statistics are deterministic."""
    import kantts_b200 as K
    from scipy.stats import chi2
    from oracle import sybert as osy
    B, L, calls = 64, 256, 16
    lings = torch.zeros(B, L, 4, dtype=torch.long)
    lings[:, :, 0] = 500 + torch.arange(L)[None, :]
    lens = torch.full((B,), L - 1)
    masker = K.BertMasker(0.3, 147, seed=2024, mask_id=1000)
    counts = np.zeros((L - 1, 3))
    expect = np.zeros((L - 1, 3))
    selected = 0
    for _ in range(calls):
        out = masker({"input_lings": lings.to(DEV), "valid_input_lengths": lens.to(DEV)})
        x, m = out["input_lings"][:, : L - 1, 0].cpu().numpy(), out["bert_masks"][:, : L - 1].cpu().numpy() == 1
        assert not out["bert_masks"][:, L - 1].any()
        selected += int(m.sum())
        counts[:, 0] += ((x == 1000) & m).sum(0)
        counts[:, 1] += ((x < 147) & m).sum(0)
        counts[:, 2] += ((x >= 500) & (x != 1000) & m).sum(0)
        for b in range(B):
            n = int(m[b].sum())
            n_mask, n_rand = osy.masking_counts(n)
            expect[m[b]] += np.array([n_mask, n_rand, n - n_mask - n_rand]) / n
    positions = B * (L - 1) * calls
    assert positions >= 100_000
    sigma = math.sqrt(0.3 * 0.7 / positions)
    assert abs(selected / positions - 0.3) < 5 * sigma, (selected / positions, sigma)
    assert np.allclose(counts.sum(1), expect.sum(1))
    stat = float(((counts - expect) ** 2 / expect).sum())
    dof = 2 * (L - 2)
    assert stat < chi2.isf(1e-6, dof), (stat, dof)


def make_sybert_batch(cfg, gen, B=32, lo=64, hi=256):
    """32 utterances of 64-256 symbols (the last the eos), padded as the collate pads them."""
    n_sy = cfg["sy"]
    lens = torch.randint(lo, hi + 1, (B,), generator=gen)
    L = int(lens.max())
    x = torch.stack([torch.randint(0, n_sy - 3, (B, L), generator=gen)] +
                    [torch.randint(0, cfg[k], (B, L), generator=gen) for k in ("tone", "syllable_flag", "word_segment")], -1)
    for b in range(B):
        n = int(lens[b])
        x[b, n - 1, 0] = n_sy - 2
        x[b, n:, 0] = n_sy - 3
        x[b, n:, 1:] = 0
    return {"input_lings": x, "valid_input_lengths": lens - 1}


def test_sybert_train_step_learns_one_batch():
    import kantts_b200 as K
    cfg = K.sybert_config()
    torch.manual_seed(1234)
    config = {"Model": {"KanTtsTextsyBERT": {"params": cfg, "optimizer": {"type": "Adam", "params": {
        "lr": 1e-3, "betas": [0.9, 0.98], "eps": 1e-9, "weight_decay": 0.0}},
        "scheduler": {"type": "NoamLR", "params": {"warmup_steps": 4}}}}}
    model, opt, sch = K.sybert_model_builder(config, DEV)
    model.train()
    crit = K.criterion_builder({"Loss": {"SeqCELoss": {"enable": True, "params": {"loss_type": "ce"}}}}, DEV)
    step = K.SybertStep(model, opt, sch, crit)
    batch = {k: v.to(DEV) for k, v in make_sybert_batch(cfg, torch.Generator().manual_seed(8)).items()}
    batch = K.BertMasker(cfg["mask_ratio"], cfg["sy"], seed=3)(batch)
    fc0 = model.fc.weight.detach().clone()
    emb0 = model.text_encoder.sy_emb.weight.detach().clone()
    losses = []
    for _ in range(8):
        out = step.step(batch)
        assert set(out) == {"TotalLoss", "Error"}
        losses.append((float(out["TotalLoss"]), float(out["Error"])))
    assert all(math.isfinite(l) and 0.0 <= e <= 1.0 for l, e in losses), losses
    assert losses[-1][0] < losses[0][0], losses
    assert step.steps == 8
    assert not torch.equal(fc0, model.fc.weight.detach())
    assert not torch.equal(emb0, model.text_encoder.sy_emb.weight.detach())
