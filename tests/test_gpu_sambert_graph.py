"""GPU: SAM-BERT training as a replayed CUDA graph.  The LSTM training kernels (kt_lstm_train_fwd / _bwd through
sambert_ops.lstm_layer) against a float64 LSTM recurrence and against each item run alone; SambertStep(cuda_graph=True)
against the eager step, bit for bit, over two alternating batch shapes; graph-mode training with the yaml's dropouts; the
refusal of FP and MAS models."""
import math

import pytest
import torch
import torch.nn as nn

import kantts_b200 as K
from conftest import rel_l2

pytestmark = pytest.mark.gpu

DEV = "cuda"


# ---- kernels -------------------------------------------------------------------------------------------------------------
def _lens(T, B):
    return torch.tensor([T, 1, T // 2 + 1, max(1, T - 3)][:B], dtype=torch.int32)


@pytest.mark.parametrize("bidir,C,H,T,ragged", [
    (True, 128, 128, 64, True), (True, 20, 37, 50, True), (False, 20, 37, 45, True), (False, 256, 128, 800, False),
    (False, 64, 256, 40, False), (True, 32, 128, 770, True)])
def test_lstm_layer_matches_float64(bidir, C, H, T, ragged):
    """h and the gradients of x, W_ih, W_hh and both biases of one layer (exact path) against the oracle's float64
    recurrence, with pack_padded_sequence semantics when ragged."""
    from kantts_b200 import ops
    from kantts_b200 import sambert_ops as sops
    from oracle import sambert as osb
    torch.manual_seed(C * 1000 + H + T)
    B, D = 4, 2 if bidir else 1
    lstm = nn.LSTM(C, H, batch_first=True, bidirectional=bidir)
    x = torch.randn(B, T, C)
    r = torch.randn(B, T, D * H)
    lens = _lens(T, B) if ragged else None
    sd = {"l." + k: v.detach().double().requires_grad_(True) for k, v in lstm.state_dict().items()}
    xr = x.double().requires_grad_(True)
    want = osb.lstm(xr, osb._SD(sd), "l", 1, bidir, None if lens is None else lens.long())
    (want * r.double()).sum().backward()
    m = lstm.to(DEV)
    xg = x.to(DEV).requires_grad_(True)
    ops.set_force_ffma(True)
    try:
        h, _ = sops.lstm_layer(xg, m, 0, None if lens is None else lens.to(DEV))
        (h * r.to(DEV)).sum().backward()
    finally:
        ops.set_force_ffma(False)
    assert rel_l2(h.detach().cpu(), want.detach().float()) < 1e-5
    assert rel_l2(xg.grad.cpu(), xr.grad.float()) < 1e-5
    for k, p in m.named_parameters():
        e = rel_l2(p.grad.cpu(), sd["l." + k].grad.float())
        assert e < 1e-5, (k, e)


@pytest.mark.parametrize("dirs,H,T,ragged", [(2, 128, 64, True), (1, 37, 50, True), (1, 128, 780, False),
                                             (2, 37, 33, False)])
def test_lstm_recurrence_rows_equal_each_item_alone(dirs, H, T, ragged):
    """LstmFn: each item's h rows and gx gradient rows equal that item run alone on its own rows, bit for bit."""
    from kantts_b200 import sambert_ops as sops
    torch.manual_seed(H + T)
    B = 4
    gx = torch.randn(B, T, dirs * 4 * H, device=DEV)
    whh = (torch.randn(dirs * 4 * H, H, device=DEV) / math.sqrt(H))
    r = torch.randn(B, T, dirs * H, device=DEV)
    lens = _lens(T, B).to(DEV) if ragged else None

    def run(g, rr, ln):
        g = g.clone().requires_grad_(True)
        w = whh.clone().requires_grad_(True)
        h, c = sops.LstmFn.apply(g, w, ln, dirs, None, None, True)
        (h * rr).sum().backward()
        return h.detach(), c.detach(), g.grad, w.grad

    h, c, dg, dw = run(gx, r, lens)
    n = lens.tolist() if ragged else [T] * B
    for b in range(B):
        hb, cb, dgb, _ = run(gx[b:b + 1, :n[b]], r[b:b + 1, :n[b]], None if lens is None else lens[b:b + 1])
        assert torch.equal(h[b:b + 1, :n[b]], hb) and torch.equal(c[b:b + 1, :n[b]], cb), b
        assert torch.equal(dg[b:b + 1, :n[b]], dgb), b
        assert not h[b, n[b]:].any() and not c[b, n[b]:].any() and not dg[b, n[b]:].any(), b
    assert torch.isfinite(dw).all()


def _ar_reference(pred, inputs, cond, state):
    """VarRnnARPredictor.forward in float64 on the CPU: prenet, nn.LSTM from ``state``, fc + ReLU."""
    import copy
    import torch.nn.functional as F
    fcs = [m for m in pred.prenet.fcs if isinstance(m, nn.Linear)]
    x = inputs
    for fc in fcs:
        x = F.relu(F.linear(x, fc.weight.double().cpu(), fc.bias.double().cpu()))
    lstm = copy.deepcopy(pred.lstm).cpu().double()
    y, (hn, cn) = lstm(torch.cat([x, cond], -1), state)
    return F.relu(F.linear(y, pred.fc.weight.double().cpu(), pred.fc.bias.double().cpu())).squeeze(-1), hn, cn


def test_ar_predictor_forward_from_an_initial_state():
    """VarRnnARPredictor.forward(h=(h_0, c_0)): outputs, (h_n, c_n) and the gradients of the inputs and of the initial state
    against nn.LSTM in float64; and two halves chained through h_new equal the whole sequence, as the reference's
    step-by-step infer chains it."""
    from kantts_b200 import ops, sambert
    torch.manual_seed(3)
    B, L, C, H = 3, 20, 24, 128
    pred = sambert.VarRnnARPredictor(C, [32, 32], H).to(DEV).eval()           # the prenet dropout off
    inputs, cond = torch.rand(B, L, 1), torch.randn(B, L, C)
    h0, c0 = torch.randn(2, B, H) * 0.5, torch.randn(2, B, H) * 0.5
    r, rh, rc = torch.randn(B, L), torch.randn(2, B, H), torch.randn(2, B, H)
    ref64 = [t.double().requires_grad_(True) for t in (inputs, cond, h0, c0)]
    y, hn, cn = _ar_reference(pred, ref64[0], ref64[1], (ref64[2], ref64[3]))
    ((y * r.double()).sum() + (hn * rh.double()).sum() + (cn * rc.double()).sum()).backward()
    got = [t.to(DEV).requires_grad_(True) for t in (inputs, cond, h0, c0)]
    ops.set_force_ffma(True)
    try:
        yg, (hng, cng) = pred(got[0], got[1], h=(got[2], got[3]))
        ((yg * r.to(DEV)).sum() + (hng * rh.to(DEV)).sum() + (cng * rc.to(DEV)).sum()).backward()
        with torch.no_grad():
            y1, s1 = pred(got[0][:, :9], got[1][:, :9], h=(got[2], got[3]))
            y2, s2 = pred(got[0][:, 9:], got[1][:, 9:], h=s1)
    finally:
        ops.set_force_ffma(False)
    for a, w in ((yg, y), (hng, hn), (cng, cn)):
        assert rel_l2(a.detach().cpu(), w.detach().float()) < 1e-5
    for a, w in zip(got, ref64):
        assert rel_l2(a.grad.cpu(), w.grad.float()) < 1e-5
    assert torch.equal(torch.cat([y1, y2], 1), yg.detach())
    assert torch.equal(s2[0], hng.detach()) and torch.equal(s2[1], cng.detach())


# ---- the train step ------------------------------------------------------------------------------------------------------
def _nsf_config():
    return dict(K.sambert_24k_config(), num_mels=82, NSF=True, nsf_norm_type="global", nsf_f0_global_minimum=30.0,
                nsf_f0_global_maximum=730.0)


CONFIGS = {"24k": K.sambert_24k_config, "nsf": _nsf_config, "se": K.sambert_se_nsf_global_16k_config}


def _batch(cfg, B, L, seed, pad=None):
    """A seeded collate-style batch of B items of up to L symbols; ``pad`` = (symbol multiple, frame multiple): right-padded
    with data.pad_sambert_batch, so that batches of different contents share one shape."""
    from golden.make_batch import make_sambert_batch
    from kantts_b200 import data
    gen = torch.Generator().manual_seed(seed)
    se = cfg.get("SE", False)
    b = make_sambert_batch(dict(cfg, speaker=1) if se else cfg, B=B, L=L, gen=gen, short=3)
    spk = torch.randn(B, 1, cfg["speaker_units"], generator=gen).expand(B, L, -1).contiguous() if se else b["inputs_speaker"]
    out = dict(input_lings=b["inputs_ling"], input_emotions=b["inputs_emotion"], input_speakers=spk,
               valid_input_lengths=b["input_lengths"], valid_output_lengths=b["output_lengths"],
               mel_targets=b["mel_targets"], durations=b["duration_targets"], pitch_contours=b["pitch_targets"],
               energy_contours=b["energy_targets"])
    out = {k: v.to(DEV) for k, v in out.items()}
    return out if pad is None else data.pad_sambert_batch(out, pad[0], pad[1], cfg["outputs_per_step"], (0, 0, 0, 0), 0, 0)


def _step(cfg, cuda_graph, graph_warmup=1):
    from kantts_b200 import sambert
    torch.manual_seed(1234)
    config = {"Model": {"KanTtsSAMBERT": {"params": cfg, "optimizer": {"type": "Adam", "params": {
        "lr": 1e-3, "betas": [0.9, 0.98], "eps": 1e-9, "weight_decay": 0.0}},
        "scheduler": {"type": "NoamLR", "params": {"warmup_steps": 40}}}}}
    model, opt, sch = K.sambert_model_builder(config, DEV)
    crit = {"MelReconLoss": sambert.MelReconLoss(), "ProsodyReconLoss": sambert.ProsodyReconLoss()}
    return model, K.SambertStep(model, opt, sch, crit, cuda_graph=cuda_graph, graph_warmup=graph_warmup)


@pytest.mark.parametrize("name", list(CONFIGS))
def test_graph_step_equals_eager_step_over_two_shapes(name):
    """Dropout off (eval mode): eight steps over two batch shapes, fresh contents every step -- one eager warm-up step per
    shape, then each shape's graph is captured and replayed from refreshed static inputs, also out of capture order.  Every
    loss, the band width and every parameter equal the eager step's bit for bit, the returned values read only after all
    steps (a step's results outlive later replays of either graph)."""
    cfg = CONFIGS[name]()
    m_e, eager = _step(cfg, False)
    m_g, graph = _step(cfg, True)
    m_e.eval()
    m_g.eval()
    results = []
    for i, s in enumerate((0, 1, 0, 1, 1, 0, 0, 1)):
        L, pad = ((12, (16, 60)), (17, (24, 90)))[s]
        batch = _batch(cfg, 3, L, 100 + i, pad)
        results.append((eager.step(batch), graph.step(batch)))
    for i, (a, b) in enumerate(results):
        if i >= 2:
            assert torch.is_tensor(b["x_band_width"]) and b["x_band_width"].is_cuda
        for k, v in a.items():
            if torch.is_tensor(v):
                assert torch.equal(v, b[k]), (i, k, float(v), float(b[k]))
            else:
                assert v == int(b[k]), (i, k)
    assert len(graph._graphs) == 2
    for (n, p), (_, q) in zip(m_e.named_parameters(), m_g.named_parameters()):
        assert torch.equal(p, q), n


def test_graph_step_trains_with_dropout():
    """The yaml's dropouts on: graph mode's losses are finite and the mel loss falls over a few dozen steps on one batch."""
    cfg = K.sambert_24k_config()
    model, step = _step(cfg, True, graph_warmup=3)
    model.train()
    batch = _batch(cfg, 4, 24, 7)
    mel = []
    for _ in range(30):
        out = step.step(batch)
        assert all(torch.isfinite(v).all() for v in out.values() if torch.is_tensor(v)), out
        mel.append(float(out["mel_loss"]))
    assert len(step._graphs) == 1
    assert sum(mel[-5:]) < sum(mel[:5]), mel


@pytest.mark.parametrize("variant,match", [("fp", "fp_insert_plan"), ("mas", "align's length validation")])
def test_graph_step_refuses_fp_and_mas(variant, match):
    cfg = K.sambert_fp_8k_config() if variant == "fp" else K.sambert_16k_mas_config()
    with pytest.raises(ValueError, match=match):
        _step(cfg, True)
