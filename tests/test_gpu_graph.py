"""CUDA-graph replay of the train step must reproduce the eager step exactly (same kernels, same order)."""
import copy

import pytest
import torch

import kantts_b200 as K
from test_gpu_parity import _small_config, DEV

import os

pytestmark = [pytest.mark.gpu]


def _build(g, cfg, graph):
    torch.manual_seed(0)
    model, opt, sched = K.hifigan_model_builder(cfg, DEV)
    model["generator"].load_state_dict(g.group("before/g/"))
    model["discriminator"]["MultiScaleDiscriminator"].load_state_dict(g.group("before/msd/"))
    model["discriminator"]["MultiPeriodDiscriminator"].load_state_dict(g.group("before/mpd/"))
    crit = K.criterion_builder(cfg, DEV)
    return K.GanStep(model, opt, sched, crit, cfg, cuda_graph=graph, graph_warmup=2), model


def test_cuda_graph_step_matches_eager(golden):
    g = golden("trainstep_small")
    cfg = _small_config(g)
    y, x = g.t("y").to(DEV), g.t("x").to(DEV)
    batches = [(y, x), (y.flip(0), x.flip(0)), ((y * 0.5).contiguous(), x), (y, (x * 0.9).contiguous()),
               (y.roll(7, -1), x), (y, x)]
    eager, m_e = _build(g, cfg, False)
    traj_e = [K.train.losses_to_float(eager.step(b)) for b in batches]
    torch.cuda.synchronize()
    graph, m_g = _build(g, cfg, True)
    traj_g = [K.train.losses_to_float(graph.step(b)) for b in batches]   # steps 0-1 eager warm-up, 2 capture, 3+ replay
    for i, (le, lg) in enumerate(zip(traj_e, traj_g)):
        for k in le:
            # replay bugs (stale weight / input buffers) show up as O(1e-1) differences that keep growing; the bit-for-bit
            # check of two runs is test_train_steps_are_deterministic
            tol = (3e-3 if i <= 3 else 3e-2) * (5.0 if k == "feature_matching_loss" else 1.0)
            assert abs(le[k] - lg[k]) <= tol * max(1.0, abs(le[k])), (i, k, le[k], lg[k])
    assert graph._graphs is not None
    for k, v in m_e["generator"].state_dict().items():
        w = m_g["generator"].state_dict()[k]
        assert float((v - w).abs().max()) <= 5e-3 * max(1.0, float(v.abs().max())), k


@pytest.mark.parametrize("ffma", [False, True])
def test_train_steps_are_deterministic(golden, ffma):
    """Two runs of the same eager train steps from the same weights and inputs agree bit for bit -- losses and every
    parameter: no reduction of the step (weight / bias gradients, the mel loss backward, the loss sums) depends on the
    order in which CTAs or side streams happen to run.  ffma: every conv on the exact-fp32 kernels."""
    from kantts_b200 import ops
    prev = ops._FORCE_FFMA
    ops.set_force_ffma(ffma)
    try:
        _check_deterministic(golden)
    finally:
        ops.set_force_ffma(prev)


def _check_deterministic(golden):
    g = golden("trainstep_small")
    cfg = _small_config(g)
    y, x = g.t("y").to(DEV), g.t("x").to(DEV)
    batches = [(y, x), (y.flip(0), x.flip(0)), (y, x)]
    runs = []
    for _ in range(2):
        step, m = _build(g, cfg, False)
        traj = [K.train.losses_to_float(step.step(b)) for b in batches]
        torch.cuda.synchronize()
        params = {f"g.{k}": v.detach().clone() for k, v in m["generator"].state_dict().items()}
        for name, d in m["discriminator"].items():
            params.update({f"{name}.{k}": v.detach().clone() for k, v in d.state_dict().items()})
        runs.append((traj, params))
    assert runs[0][0] == runs[1][0]
    for k, v in runs[0][1].items():
        assert torch.equal(v, runs[1][1][k]), k
