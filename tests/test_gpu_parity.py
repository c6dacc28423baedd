"""GPU parity tests (``pytest -m gpu``).  Every check goes through the C ABI
(ctypes -> libkantts_b200.so) and compares against the CPU oracle / golden vectors from the
unmodified reference.  Tolerances (north_star): waveform RMS <= 1e-3, mel-L1 <= 1e-4; we hold the
exact-fp32 (FFMA) kernels to ~1e-5 relative and the tensor-core (wgmma) bf16x3 kernels to 1e-4 relative."""
import math
import os
import zlib

import pytest
import torch
import torch.nn.functional as F

import kantts_b200 as K
from kantts_b200 import ops
from kantts_b200._lib import KT_ACT_LRELU, KT_ACT_TANH
from conftest import rel_l2
from oracle import convref
from oracle import hifigan as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _to_rows(x):           # (B, C, T) -> (B, T, C) ; (B, C, H, P) -> (B, H, P, C)
    return x.permute(0, 2, 1).contiguous() if x.dim() == 3 else x.permute(0, 2, 3, 1).contiguous()


def _from_rows(x):
    return x.permute(0, 2, 1) if x.dim() == 3 else x.permute(0, 3, 1, 2)


CASES = {
    # name: (spec kwargs, B, T, period, use_resid, weight_norm)
    "causal_dilated_resid": (dict(c_in=64, c_out=64, kernel=7, dilation=3, pad_left=18, act_in=0.1), 2, 300, 0, True, True),
    "noncausal_k3": (dict(c_in=32, c_out=32, kernel=3, pad_left=1, pad_right=1, act_in=0.1), 2, 257, 0, True, True),
    "msd_grouped_strided": (dict(c_in=32, c_out=64, kernel=41, stride=4, pad_left=20, pad_right=20, groups=4, act_out=0.1), 2, 512, 0, False, True),
    "msd_grouped16": (dict(c_in=128, c_out=256, kernel=41, stride=4, pad_left=20, pad_right=20, groups=16, act_out=0.1), 2, 300, 0, False, True),
    "msd_tiny_groups_a": (dict(c_in=16, c_out=16, kernel=41, stride=4, pad_left=20, pad_right=20, groups=4, act_out=0.1), 2, 2048, 0, False, True),
    "msd_tiny_groups_b": (dict(c_in=16, c_out=32, kernel=41, stride=4, pad_left=20, pad_right=20, groups=16, act_out=0.1), 2, 512, 0, False, True),
    "msd_tiny_groups_c": (dict(c_in=64, c_out=64, kernel=41, stride=1, pad_left=20, pad_right=20, groups=16, act_out=0.1), 2, 40, 0, False, False),
    "cin1_k15": (dict(c_in=1, c_out=16, kernel=15, pad_left=7, pad_right=7, act_out=0.1), 3, 1000, 0, False, True),
    "cout1_tanh": (dict(c_in=32, c_out=1, kernel=7, pad_left=6, act_in=0.01, act_out="tanh"), 2, 500, 0, False, True),
    "cin2_cout1_aux": (dict(c_in=2, c_out=1, kernel=15, pad_left=7, pad_right=7, act_out=0.1), 2, 700, 0, False, True),
    "deconv_causal": (dict(c_in=64, c_out=32, kernel=16, stride=8, transposed=True, crop=8, act_in=0.1), 2, 40, 0, True, True),
    "deconv_odd_noncausal": (dict(c_in=32, c_out=16, kernel=11, stride=5, pad_left=3, transposed=True, act_in=0.1), 2, 33, 0, True, True),
    "deconv_k4s2": (dict(c_in=128, c_out=64, kernel=4, stride=2, transposed=True, crop=2, act_in=0.1), 2, 150, 0, True, True),
    "upsample_conv": (dict(c_in=64, c_out=32, kernel=7, pad_left=6, upsample=8, act_in=0.1), 2, 37, 0, False, True),
    "upsample3_noncausal": (dict(c_in=16, c_out=8, kernel=7, pad_left=3, pad_right=3, upsample=3, act_in=0.1), 2, 50, 0, False, True),
    "period_strided": (dict(c_in=4, c_out=8, kernel=5, stride=3, pad_left=2, pad_right=2, act_out=0.1), 2, 100, 3, False, True),
    "period_cin1": (dict(c_in=1, c_out=32, kernel=5, stride=3, pad_left=2, pad_right=2, act_out=0.1), 2, 200, 7, False, True),
    "period_post_plain": (dict(c_in=32, c_out=1, kernel=2, pad_left=1, pad_right=1), 2, 52, 5, False, False),
    "period_stride1_tc": (dict(c_in=64, c_out=64, kernel=5, pad_left=2, pad_right=2, act_out=0.1), 2, 51, 5, False, True),
    "tc_128_k11_d5": (dict(c_in=128, c_out=128, kernel=11, dilation=5, pad_left=50, act_in=0.1), 2, 1000, 0, True, True),
    "tc_256_k3": (dict(c_in=256, c_out=256, kernel=3, pad_left=2, act_in=0.1), 2, 256, 0, True, True),
    "tc_64_to_192": (dict(c_in=64, c_out=192, kernel=7, dilation=1, pad_left=3, pad_right=3), 1, 200, 0, False, True),
    "tc_512_to_1024_k5": (dict(c_in=512, c_out=1024, kernel=5, pad_left=2, pad_right=2, act_out=0.1), 1, 140, 0, False, True),
    "tc_period_s3": (dict(c_in=128, c_out=256, kernel=5, stride=3, pad_left=2, pad_right=2, act_out=0.1), 2, 100, 3, False, True),
    "tc_period_s3_p11": (dict(c_in=64, c_out=128, kernel=5, stride=3, pad_left=2, pad_right=2, act_out=0.1), 2, 83, 11, False, True),
    "tc_strided_s4_k9": (dict(c_in=64, c_out=64, kernel=9, stride=4, pad_left=4, pad_right=4, act_out=0.1), 2, 500, 0, False, True),
    "tc_upsample_conv": (dict(c_in=128, c_out=64, kernel=7, pad_left=6, upsample=2, act_in=0.1), 2, 300, 0, False, True),
    "tc_deconv_128_64_k4s2": (dict(c_in=128, c_out=64, kernel=4, stride=2, transposed=True, crop=2, act_in=0.1), 2, 300, 0, True, True),
    "tc_deconv_256_128": (dict(c_in=256, c_out=128, kernel=16, stride=8, transposed=True, crop=8, act_in=0.1), 2, 32, 0, True, True),
    # SAM-BERT nn.Linear shapes whose widths are not multiples of 64 (dec_out_proj 128->240, postnet 80->512, dec_in_proj 288->128)
    "lin_128_240": (dict(c_in=128, c_out=240, kernel=1), 3, 70, 0, False, False),
    "lin_80_512": (dict(c_in=80, c_out=512, kernel=1), 3, 70, 0, False, False),
    "lin_288_128": (dict(c_in=288, c_out=128, kernel=1), 3, 70, 0, False, False),
    "lin_512_80_k3": (dict(c_in=512, c_out=80, kernel=3, pad_left=1, pad_right=1), 3, 70, 0, False, False),
}


def _run_case(name, force_ffma):
    kw, B, T, period, use_resid, wn = CASES[name]
    kw = dict(kw)
    act_in = kw.pop("act_in", None)
    act_out = kw.pop("act_out", None)
    spec = ops.ConvSpec(**kw)
    if act_in is not None:
        spec.act_in, spec.act_in_slope = KT_ACT_LRELU, act_in
    if act_out == "tanh":
        spec.act_out = KT_ACT_TANH
    elif act_out is not None:
        spec.act_out, spec.act_out_slope = KT_ACT_LRELU, act_out
    g = torch.Generator().manual_seed(zlib.crc32(name.encode()) % 10000)   # deterministic across processes
    wshape = (spec.c_in, spec.c_out, spec.kernel) if spec.transposed else (spec.c_out, spec.c_in // spec.groups, spec.kernel)
    v = torch.randn(wshape, generator=g) * 0.3
    gg = (v.norm(2, dim=(1, 2), keepdim=True) * (1 + 0.2 * torch.randn(wshape[0], 1, 1, generator=g))) if wn else None
    bias = 0.1 * torch.randn(spec.c_out, generator=g)
    xs = (B, spec.c_in, T, period) if period else (B, spec.c_in, T)
    x = torch.randn(xs, generator=g)
    t_out = spec.t_out(T)
    ys = (B, spec.c_out, t_out, period) if period else (B, spec.c_out, t_out)
    resid = torch.randn(ys, generator=g) if use_resid else None
    r = torch.randn(ys, generator=g)

    # oracle (CPU)
    xo, vo, bo = x.clone().requires_grad_(True), v.clone().requires_grad_(True), bias.clone().requires_grad_(True)
    go = gg.clone().requires_grad_(True) if wn else None
    ro = resid.clone().requires_grad_(True) if use_resid else None
    w = O.weight_norm_weight(go, vo) if wn else vo
    yo = convref.conv_layer(xo, w, bo, ro, stride=spec.stride, dilation=spec.dilation, pad_left=spec.pad_left,
                            pad_right=spec.pad_right, groups=spec.groups, transposed=spec.transposed,
                            upsample=spec.upsample, crop=spec.crop, act_in=act_in, act_out=act_out)
    assert tuple(yo.shape) == ys, (yo.shape, ys)

    # product (GPU, through the C ABI)
    ops.set_force_ffma(force_ffma)
    try:
        xg = _to_rows(x).to(DEV).requires_grad_(True)
        vg, bg = v.to(DEV).requires_grad_(True), bias.to(DEV).requires_grad_(True)
        g2 = gg.to(DEV).requires_grad_(True) if wn else None
        rg = _to_rows(resid).to(DEV).requires_grad_(True) if use_resid else None
        tc0 = ops.tc_launch_count()
        y = ops.conv(xg, spec, ops.PreparedWeight(), vg, g2, bg, rg)
        # A fused output LeakyReLU makes the backward mask depend on sign(pre-activation).  The handful of
        # outputs whose sign differs between the two forwards (|y| below the forward error) would change the
        # gradient discontinuously: exclude exactly those outputs from the scalar both sides differentiate.
        if act_out is not None and act_out != "tanh":
            res_o = ro.detach() if use_resid else 0.0
            res_g = _from_rows(rg.detach()).cpu() if use_resid else 0.0
            flip = torch.sign(yo.detach() - res_o) != torch.sign(_from_rows(y.detach()).cpu() - res_g)
            assert float(flip.float().mean()) < 1e-3
            r = r * (~flip)
        (yo * r).sum().backward()
        (y * _to_rows(r).to(DEV)).sum().backward()
        used_tc = ops.tc_launch_count() > tc0
    finally:
        ops.set_force_ffma(False)
    tol = 1e-4 if used_tc else 2e-5
    assert rel_l2(_from_rows(y).cpu(), yo) < tol, ("y", rel_l2(_from_rows(y).cpu(), yo))
    assert rel_l2(_from_rows(xg.grad).cpu(), xo.grad) < tol, ("dx", rel_l2(_from_rows(xg.grad).cpu(), xo.grad))
    tol_w = 3e-4 if used_tc else 5e-5
    if spec.c_out == 1:
        tol_w = max(tol_w, 2e-4)       # a single-channel dg / dbias is ONE float summed with fp32 atomics (5.8e-5 seen)
    assert rel_l2(vg.grad.cpu(), vo.grad) < tol_w, ("dv", rel_l2(vg.grad.cpu(), vo.grad))
    assert rel_l2(bg.grad.cpu(), bo.grad) < tol_w, "dbias"
    if wn:
        assert rel_l2(g2.grad.cpu(), go.grad) < tol_w, "dg"
    if use_resid:
        assert rel_l2(_from_rows(rg.grad).cpu(), ro.grad) < 1e-6, "dresid"
    return used_tc


@pytest.mark.parametrize("name", list(CASES))
def test_conv_layer_ffma_vs_oracle(name):
    _run_case(name, force_ffma=True)


@pytest.mark.parametrize("name", list(CASES))
def test_conv_layer_tcgen05_vs_oracle(name):
    """default dispatch: every layer shape (thin, grouped, strided, period, transposed, upsampled) runs on
    the tensor-core kernels (channels zero-padded to 64-wide K chunks / 16-wide N tiles)."""
    assert _run_case(name, force_ffma=False), "expected the tensor-core path to be taken"


def _check_param_grads(m, refg, exact, tol=(5e-4, 1e-3, 1e-2)):
    """Parameter gradients vs the reference's.  Exact-fp32 kernels: every tensor <= 1e-4 relative.  bf16x3
    tensor-core kernels: a weight gradient is a sum over (batch x time) of products carried to ~2^-17, so
    gradients that are small residuals of large cancelling sums lose relative accuracy; the typical tensor
    must still agree to 5e-4, the whole gradient vector to 1e-3, the worst single (thin) tensor to 1e-2 (round 2: measured
    worst 5.4e-3 over the four module fixtures, scripts/grad_err_report.py)."""
    errs = sorted((rel_l2(p.grad.cpu(), refg[k]), k) for k, p in m.named_parameters())
    if exact:
        assert errs[-1][0] < 1e-4, errs[-1]
        return
    num = sum(float(((p.grad.cpu() - refg[k]).double() ** 2).sum()) for k, p in m.named_parameters())
    den = sum(float((refg[k].double() ** 2).sum()) for k, p in m.named_parameters())
    print("param-grad rel err: median %.2e global %.2e worst %s" % (errs[len(errs) // 2][0], (num / den) ** 0.5, errs[-3:]))
    assert errs[len(errs) // 2][0] < tol[0], ("median", errs[len(errs) // 2])
    assert (num / den) ** 0.5 < tol[1], ("global", (num / den) ** 0.5)
    assert errs[-1][0] < tol[2], ("worst", errs[-1], errs[-5:])


def _load(module, sd):
    module.load_state_dict(sd, strict=True)
    return module.to(DEV)


@pytest.mark.parametrize("name", ["gen_small_causal", "gen_small_noncausal"])
@pytest.mark.parametrize("force_ffma", [True, False])
def test_generator_matches_reference_golden(golden, name, force_ffma):
    g = golden(name)
    ops.set_force_ffma(force_ffma)
    try:
        m = _load(K.Generator(**g.cfg), g.group("sd/"))
        x = g.t("x").to(DEV).requires_grad_(True)
        y = m(x)
        ref = g.t("y")
        assert y.shape == ref.shape
        rms = float((y.detach().cpu() - ref).pow(2).mean().sqrt())
        assert rms < (1e-5 if force_ffma else 1e-4), rms
        (y * g.t("r").to(DEV)).sum().backward()
    finally:
        ops.set_force_ffma(False)
    tol = 1e-4 if force_ffma else 5e-4
    assert rel_l2(x.grad.cpu(), g.t("grad_x")) < tol
    refg = g.group("grad/")
    _check_param_grads(m, refg, exact=force_ffma)


@pytest.mark.parametrize("name,cls", [("mpd_small", "MultiPeriodDiscriminator"), ("msd_small", "MultiScaleDiscriminator")])
def test_discriminators_match_reference_golden(golden, name, cls):
    g = golden(name)
    m = _load(getattr(K, cls)(**g.cfg), g.group("sd/"))
    m.train()
    y = g.t("y").to(DEV).requires_grad_(True)
    outs, fmaps = m(y)
    loss = 0.0
    for i, o in enumerate(outs):
        assert o.shape == g.t(f"out{i}").shape
        assert float((o.detach().cpu() - g.t(f"out{i}")).abs().max()) < 2e-5
        for l, f in enumerate(fmaps[i]):
            assert f.shape == g.t(f"fmap{i}_{l}").shape
            assert rel_l2(f.detach().cpu(), g.t(f"fmap{i}_{l}")) < 2e-5
        loss = loss + (o * g.t(f"r{i}").to(DEV)).sum()
    loss.backward()
    assert rel_l2(y.grad.cpu(), g.t("grad_y")) < 1e-4
    refg = g.group("grad/")
    _check_param_grads(m, refg, exact=False)
    sd = m.state_dict()
    for k, v in g.group("after/").items():
        assert rel_l2(sd[k].cpu(), v) < 1e-5, k


def test_mel_and_stft_losses_match_reference_golden(golden):
    g = golden("mel_stft")
    y = g.t("y").to(DEV)
    cfgs = {"default": {}, "yaml24k": dict(fs=24000, fft_size=1024, hop_size=240, win_length=1024, fmin=0, fmax=8000, log_base=None),
            "c2": dict(fs=22050, fft_size=1024, hop_size=256, win_length=1024, fmin=0, fmax=8000)}
    for tag, cfg in cfgs.items():
        mel = K.MelSpectrogram(**cfg).to(DEV)(y)
        ref = g.t(f"mel_{tag}")
        assert mel.shape == ref.shape
        assert float((mel.cpu() - ref).abs().mean()) < 1e-4          # mel-L1 tolerance of the north star
        y_hat = g.t("y_hat").to(DEV).requires_grad_(True)
        loss = K.MelSpectrogramLoss(**cfg).to(DEV)(y_hat, y)
        assert abs(float(loss) - float(g.t(f"loss_{tag}"))) < 1e-4
        loss.backward()
        assert rel_l2(y_hat.grad.cpu(), g.t(f"grad_{tag}")) < 5e-3
    y_hat = g.t("y_hat").to(DEV).requires_grad_(True)
    sc, mag = K.MultiResolutionSTFTLoss().to(DEV)(y_hat, y)
    assert abs(float(sc) - float(g.t("stft_sc"))) < 1e-4
    assert abs(float(mag) - float(g.t("stft_mag"))) < 1e-4
    (sc + mag).backward()
    assert rel_l2(y_hat.grad.cpu(), g.t("stft_grad")) < 5e-3


def _small_config(g):
    adam = {"type": "Adam", "params": {"lr": 2e-4, "betas": [0.5, 0.9], "weight_decay": 0.0}}
    sched = {"type": "MultiStepLR", "params": {"gamma": 0.5, "milestones": [200000]}}
    return {"Model": {"Generator": {"params": g.cfg["generator"], "optimizer": adam, "scheduler": sched},
                      "MultiScaleDiscriminator": {"params": g.cfg["msd"], "optimizer": adam, "scheduler": sched},
                      "MultiPeriodDiscriminator": {"params": g.cfg["mpd"], "optimizer": adam, "scheduler": sched}},
            "Loss": g.cfg["loss"], "generator_train_start_steps": 1, "discriminator_train_start_steps": 0,
            "generator_grad_norm": -1, "discriminator_grad_norm": -1}


@pytest.mark.parametrize("pair", [True, False])
@pytest.mark.parametrize("force_ffma", [True, False])
def test_gan_train_step_matches_reference_trainer(golden, force_ffma, pair):
    """One full GAN step (both phases, Adam) vs the unmodified GAN_Trainer.train_step.  ``pair``: the
    discriminators run once per phase on the (generated, real) pair as one batch (GanStep default)."""
    g = golden("trainstep_small")
    cfg = _small_config(g)
    ops.set_force_ffma(force_ffma)
    try:
        torch.manual_seed(0)
        model, opt, sched = K.hifigan_model_builder(cfg, DEV)
        model["generator"].load_state_dict(g.group("before/g/"))
        model["discriminator"]["MultiScaleDiscriminator"].load_state_dict(g.group("before/msd/"))
        model["discriminator"]["MultiPeriodDiscriminator"].load_state_dict(g.group("before/mpd/"))
        crit = K.criterion_builder(cfg, DEV)
        step = K.GanStep(model, opt, sched, crit, cfg, pair_discriminators=pair)
        log = K.train.losses_to_float(step.step((g.t("y").to(DEV), g.t("x").to(DEV))))
    finally:
        ops.set_force_ffma(False)
    for k in ("mel_loss", "feature_matching_loss", "generator_loss", "real_loss", "fake_loss", "discriminator_loss"):
        ref = float(g.arrays["loss/" + k])
        assert abs(log[k] - ref) <= 2e-4 * max(1.0, abs(ref)), (k, log[k], ref)
    for tag, m in (("g", model["generator"]), ("msd", model["discriminator"]["MultiScaleDiscriminator"]),
                   ("mpd", model["discriminator"]["MultiPeriodDiscriminator"])):
        after, before = g.group(f"after/{tag}/"), g.group(f"before/{tag}/")
        sd = m.state_dict()
        num = den = 0.0
        for k, v in after.items():
            num += float(((sd[k].cpu() - v).double() ** 2).sum())
            den += float(((before[k] - v).double() ** 2).sum())
        assert num <= 2e-2 * den, (tag, num, den)      # Adam's first step is lr*sign-like: loose on purpose


def test_real_half_reuse_matches_full_recompute(golden):
    """GanStep(reuse_real_half=True): the discriminator phase computes only the re-generated half of every pair batch and
    takes the real half from the generator phase's buffers.  Same kernels on the same data per item: losses and parameters
    must agree with the plain step to rounding (the two steps order the pair batch differently, [fake | real] vs
    [real | fake], which only permutes the batch-summation order of the weight gradients)."""
    g = golden("trainstep_small")
    cfg = _small_config(g)
    res = {}
    for reuse in (False, True):
        torch.manual_seed(0)
        model, opt, sched = K.hifigan_model_builder(cfg, DEV)
        model["generator"].load_state_dict(g.group("before/g/"))
        model["discriminator"]["MultiScaleDiscriminator"].load_state_dict(g.group("before/msd/"))
        model["discriminator"]["MultiPeriodDiscriminator"].load_state_dict(g.group("before/mpd/"))
        crit = K.criterion_builder(cfg, DEV)
        step = K.GanStep(model, opt, sched, crit, cfg, reuse_real_half=reuse)
        y, x = g.t("y").to(DEV), g.t("x").to(DEV)
        logs = [K.train.losses_to_float(step.step((y, x))), K.train.losses_to_float(step.step((y.flip(0), x.flip(0))))]
        mods = {"g": model["generator"], **model["discriminator"]}
        res[reuse] = (logs, {f"{tag}.{k}": v.detach().clone() for tag, m in mods.items() for k, v in m.state_dict().items()})
    for la, lb in zip(res[False][0], res[True][0]):
        for k in la:
            assert abs(la[k] - lb[k]) <= 1e-4 * max(1.0, abs(la[k])), (k, la[k], lb[k])
    for k, v in res[False][1].items():
        w = res[True][1][k]
        # (Adam turns a sign flip of a ~0 gradient into a 2 * lr difference: loose on purpose, the second step's losses are the check)
        assert float((v - w).abs().max()) <= 5e-3 * max(1.0, float(v.abs().max())), k


@pytest.mark.parametrize("name,cls", [("mpd_small", "MultiPeriodDiscriminator"), ("msd_small", "MultiScaleDiscriminator")])
def test_forward_pair_equals_two_calls(golden, name, cls):
    """forward_pair(ya, yb) == (d(ya), d(yb)) incl. the spectral-norm power-iteration state, and with
    ops.grad_items the input gradient of the first half equals the un-batched one."""
    g = golden(name)
    torch.manual_seed(5)
    T = g.t("y").shape[-1]
    ya = (0.3 * torch.randn(3, 1, T)).to(DEV).requires_grad_(True)
    yb = (0.3 * torch.randn(3, 1, T)).to(DEV)
    res = {}
    for mode in ("two", "pair", "two_frozen", "pair_frozen"):
        d = getattr(K, cls)(**g.cfg).to(DEV)
        d.load_state_dict(g.group("sd/"))
        d.train()
        if mode.endswith("frozen"):
            # GanStep's generator phase freezes D (skip_unused_d_grads): the recomputed spectral-norm weight is then a
            # LEAF temporary; it must still get fresh prepared buffers per forward (the first half's backward is pending
            # while the second half's forward re-runs the power iteration) -- ADVICE r1, ops.prepare_weight
            for q in d.parameters():
                q.requires_grad_(False)
        ya.grad = None
        if mode.startswith("two"):
            oa, fa = d(ya)
            with torch.no_grad():
                ob, fb = d(yb)
        else:
            with ops.grad_items(3):
                (oa, fa), (ob, fb) = d.forward_pair(ya, yb, detach_b=True)
            assert not any(o.requires_grad for o in ob)
        sum((o * o).sum() for o in oa).backward()
        K.hifigan.join_side_streams(torch.device(DEV))
        torch.cuda.synchronize()
        res[mode] = ([o.detach().clone() for o in oa], [o.detach().clone() for o in ob],
                     [f.detach().clone() for fm in fa for f in fm], [f.detach().clone() for fm in fb for f in fm],
                     ya.grad.clone(), {k: v.clone() for k, v in d.state_dict().items() if k.endswith(("weight_u", "weight_v"))},
                     {k: q.grad.clone() for k, q in d.named_parameters() if q.grad is not None})
    for mode in ("pair", "two_frozen", "pair_frozen"):
        for i in range(4):
            for a, b in zip(res["two"][i], res[mode][i]):
                assert a.shape == b.shape and rel_l2(b, a) < 1e-4, (mode, i, rel_l2(b, a))
        assert rel_l2(res[mode][4], res["two"][4]) < 1e-4, (mode, rel_l2(res[mode][4], res["two"][4]))
        for k, v in res["two"][5].items():
            assert rel_l2(res[mode][5][k], v) < 1e-5, (mode, k)
        for k, v in res["two"][6].items():                       # parameter gradients (only the un-frozen runs have any)
            if k in res[mode][6]:
                assert rel_l2(res[mode][6][k], v) < 1e-4, (mode, k, rel_l2(res[mode][6][k], v))


def test_direct_grad_accumulation_matches_autograd(golden):
    """FlatGrads marks parameters for in-kernel accumulation (kt_weight_grad_accum): two backward passes must
    leave the same .grad as autograd's AccumulateGrad path."""
    g = golden("gen_small_causal")
    x = g.t("x").to(DEV)
    grads = {}
    for direct in (False, True):
        m = K.Generator(**g.cfg).to(DEV)
        m.load_state_dict(g.group("sd/"))
        fg = K.train.FlatGrads(m, direct=direct)
        fg.zero()
        for scale in (1.0, -0.5):
            (m(x * scale) ** 2).sum().backward()
        K.hifigan.join_side_streams(x.device)
        torch.cuda.synchronize()
        grads[direct] = fg.flat.clone()
    assert rel_l2(grads[True], grads[False]) < 1e-5, rel_l2(grads[True], grads[False])


def test_c1_full_generator_matches_reference(golden):
    """BASELINE config 1: class-default Generator (seed 1234) forward, (1,80,32) -> (1,1,8192)."""
    g = golden("c1_generator")
    torch.manual_seed(1234)
    m = K.Generator().to(DEV).eval()
    x = g.t("x").to(DEV)
    ref = g.t("y")
    for force in (True, False):
        ops.set_force_ffma(force)
        try:
            with torch.no_grad():
                y = m(x).cpu()
        finally:
            ops.set_force_ffma(False)
        rms = float((y - ref).pow(2).mean().sqrt())
        assert rms < 1e-3, (force, rms)                               # waveform RMS tolerance
        mel_l1 = float((O.mel_spectrogram(y) - O.mel_spectrogram(ref)).abs().mean())
        assert mel_l1 < 1e-4, (force, mel_l1)                         # mel-L1 tolerance


def test_full_size_properties():
    """Size-independent properties at the C2 shapes (B=16, 8192 samples)."""
    torch.manual_seed(3)
    B, T = 16, 8192
    # DWT: orthonormal analysis -> energy preserved; adjoint test <Ax, y> = <x, A^T y>
    x = torch.randn(B, T, device=DEV, requires_grad=True)
    y = ops.DwtFn.apply(x)
    assert y.shape == (B, (T + 5) // 2, 2)
    assert abs(float(y.pow(2).sum() / x.pow(2).sum()) - 1) < 1e-5
    r = torch.randn_like(y)
    (y * r).sum().backward()
    x2 = torch.randn(B, T, device=DEV)
    assert abs(float((ops.DwtFn.apply(x2) * r).sum()) - float((x2 * x.grad).sum())) < 1e-2 * float(r.norm() * x2.norm()) * 1e-3 + 1e-2
    # conv linearity + adjointness on the heaviest resblock shape (C=128, T=2048, k=11, d=5), tensor-core path
    spec = ops.ConvSpec(c_in=128, c_out=128, kernel=11, dilation=5, pad_left=50)
    v = torch.randn(128, 128, 11, device=DEV) * 0.05
    cache = ops.PreparedWeight()
    a = torch.randn(B, 2048, 128, device=DEV, requires_grad=True)
    b = torch.randn(B, 2048, 128, device=DEV)
    ya, yb, yab = ops.conv(a, spec, cache, v), ops.conv(b, spec, cache, v), ops.conv(a + 2 * b, spec, cache, v)
    assert rel_l2(yab, ya + 2 * yb) < 1e-4
    rr = torch.randn_like(ya)
    (ya * rr).sum().backward()
    lhs = float((ops.conv(b, spec, cache, v) * rr).sum())
    rhs = float((b * a.grad).sum())
    assert abs(lhs - rhs) < 2e-4 * float(rr.norm() * yb.norm())
    # mel of a full batch: bounded to [-4, 4], silence maps to the floor
    mel = K.MelSpectrogram().to(DEV)
    out = mel(torch.zeros(B, 1, T, device=DEV))
    assert out.shape == (B, 80, 33) and float(out.max()) == -4.0


@pytest.mark.parametrize("force_ffma", [False, True])
def test_full_size_c2_train_step_matches_oracle(force_ffma):
    """BASELINE configs[1] at FULL size (B = 16 x 8192 samples, class-default generator, yaml MSD + MPD -- the very
    workload bench.py times): one GanStep (eager launches, default bf16x3 tensor-core path) against
    oracle.OracleGAN.train_step on the host, same reference-constructed weights and the same synthetic batch: the
    seven logged losses, every parameter-gradient tensor of both phases, and the parameters after the three Adam
    steps (VERDICT r1: 'configs never compared with the oracle on GPU')."""
    import bench
    from oracle import hifigan as O
    torch.manual_seed(1234)
    model, opt, sched = K.hifigan_model_builder(bench.CONFIG, torch.device(DEV))
    crit = K.criterion_builder(bench.CONFIG, torch.device(DEV))
    G, D = model["generator"], model["discriminator"]
    before = {"g": {k: v.detach().cpu().clone() for k, v in G.state_dict().items()},
              **{n: {k: v.detach().cpu().clone() for k, v in m.state_dict().items()} for n, m in D.items()}}
    gan = O.OracleGAN(before["g"], {n: before[n] for n in D}, bench.G_PARAMS,
                      {"MultiScaleDiscriminator": bench.MSD_PARAMS, "MultiPeriodDiscriminator": bench.MPD_PARAMS}, bench.LOSS)
    y, x = bench.synth_batch(bench.B_PER_GPU, 1234)
    step = K.GanStep(model, opt, sched, crit, bench.CONFIG)
    ops.set_force_ffma(force_ffma)      # True: the exact-fp32 kernels -- separates split-precision effects from logic errors
    try:
        log = K.train.losses_to_float(step.step((y.to(DEV), x.to(DEV))))
        torch.cuda.synchronize()
    finally:
        ops.set_force_ffma(False)
    torch.set_num_threads(min(os.cpu_count() or 1, 32))
    ref = gan.train_step(y, x)
    for k in ("mel_loss", "adversarial_loss", "feature_matching_loss", "generator_loss", "real_loss", "fake_loss", "discriminator_loss"):
        assert abs(log[k] - ref[k]) <= 2e-4 * max(1.0, abs(ref[k])), (k, log[k], ref[k])
    failures = []
    for tag, m, od in (("g", G, gan.g), ("msd", D["MultiScaleDiscriminator"], gan.d["MultiScaleDiscriminator"]),
                       ("mpd", D["MultiPeriodDiscriminator"], gan.d["MultiPeriodDiscriminator"])):
        refg = {k: od[k].grad for k, _ in m.named_parameters()}
        # full size: 131 072 output rows per weight gradient and ~100 LeakyReLUs upstream of every tensor -- the ~1e-5
        # forward difference flips the derivative mask of the pre-activations nearest zero (a discontinuous function of
        # the forward), which dominates the per-tensor figure (measured: -s output of this test)
        try:
            _check_param_grads(m, refg, exact=False, tol=(5e-4, 5e-4, 1e-2) if force_ffma else (5e-3, 5e-3, 1e-1))
        except AssertionError as e:
            failures.append((tag, str(e)[:300]))
        sd = m.state_dict()
        num = den = 0.0
        for k, v in od.items():
            if not v.is_floating_point():
                continue
            b = before["g" if tag == "g" else {"msd": "MultiScaleDiscriminator", "mpd": "MultiPeriodDiscriminator"}[tag]][k]
            num += float(((sd[k].cpu() - v.detach()).double() ** 2).sum())
            den += float(((b - v.detach()).double() ** 2).sum())
        assert num <= 2e-2 * den, (tag, num, den)
    assert not failures, failures


RB_CASES = {
    # name: (channels, kernel, dilation, causal, B, T)
    "rb64_k3_d1_causal": (64, 3, 1, True, 2, 300),
    "rb64_k7_d3_causal": (64, 7, 3, True, 2, 515),
    "rb64_k11_d5_noncausal": (64, 11, 5, False, 2, 999),
    "rb32_k3_d1_noncausal": (32, 3, 1, False, 2, 300),
    "rb32_k7_d5_causal": (32, 7, 5, True, 3, 1000),
    "rb32_k11_d5_causal": (32, 11, 5, True, 2, 777),
    "rb32_k11_d3_short": (32, 11, 3, True, 2, 64),          # T shorter than one tile / than the receptive field
}


@pytest.mark.parametrize("name", sorted(RB_CASES))
def test_fused_resblock_unit_vs_oracle(name):
    """kt_resblock_fwd / kt_resblock_bwd (SURVEY 8 row G4 / VERDICT row K1: one (convs1[i], convs2[i]) pair of
    layers.py:213-220 in ONE launch) against the layer oracle: y, and every gradient (x, both weights_v / weight_g, both
    biases), with weight norm on, ragged tile counts, causal and centred padding."""
    C, k, d, causal, B, T = RB_CASES[name]
    p1 = (k - 1) * d if causal else (k - 1) * d // 2
    p2 = (k - 1) if causal else (k - 1) // 2
    s1 = ops.ConvSpec(c_in=C, c_out=C, kernel=k, dilation=d, pad_left=p1, pad_right=(k - 1) * d - p1, act_in=KT_ACT_LRELU, act_in_slope=0.1)
    s2 = ops.ConvSpec(c_in=C, c_out=C, kernel=k, dilation=1, pad_left=p2, pad_right=(k - 1) - p2, act_in=KT_ACT_LRELU, act_in_slope=0.1)
    gen = torch.Generator().manual_seed(zlib.crc32(name.encode()))
    prm = []
    for _ in range(2):
        v = torch.randn(C, C, k, generator=gen) / math.sqrt(C * k)
        g = v.norm(2, dim=(1, 2), keepdim=True) * (1 + 0.2 * torch.randn(C, 1, 1, generator=gen))
        b = 0.1 * torch.randn(C, generator=gen)
        prm += [v, g, b]
    x = torch.randn(B, C, T, generator=gen)
    r = torch.randn(B, C, T, generator=gen)
    # ---- oracle (CPU, channels-first).  LeakyReLU is written as x * where(m > 0, 1, slope) with the mask source m given
    # separately: m = the oracle's own value is the plain function; m = the PRODUCT's value of the same tensor gives the
    # derivative on the product's side of every kink -- the two differ only where a pre-activation's sign differs, i.e. on
    # the ~1e-5 fraction of elements whose magnitude is below the forward error (see the tolerances below)
    def run_oracle(h_mask):
        ref_in = [t.clone().requires_grad_(True) for t in [x] + prm]
        xo, v1, g1, b1, v2, g2, b2 = ref_in
        w1 = g1 * v1 / v1.norm(2, dim=(1, 2), keepdim=True)
        w2 = g2 * v2 / v2.norm(2, dim=(1, 2), keepdim=True)
        lre = lambda t, msk: t * torch.where(msk > 0, torch.ones(()), torch.full((), 0.1))
        ho = convref.conv_layer(lre(xo, xo.detach()), w1, b1, dilation=d, pad_left=p1, pad_right=(k - 1) * d - p1)
        yo = convref.conv_layer(lre(ho, ho.detach() if h_mask is None else h_mask), w2, b2, resid=xo, dilation=1, pad_left=p2,
                                pad_right=(k - 1) - p2)
        (yo * r).sum().backward()
        return ref_in, ho.detach(), yo.detach()
    ref_in, ho, yo = run_oracle(None)
    xo = ref_in[0]
    # ---- product: the fused unit on channels-last rows
    dev_in = [torch.nn.Parameter(t.clone().to(DEV)) for t in prm]
    xg = x.permute(0, 2, 1).contiguous().to(DEV).requires_grad_(True)
    rd = ops.resblock_desc(s1, s2, B, T)
    assert rd is not None, "the fused kernel must support this shape"
    n0 = ops.tc_launch_count()
    y = ops.resblock(xg, s1, ops.PreparedWeight(), dev_in[0], dev_in[1], dev_in[2], s2, ops.PreparedWeight(), dev_in[3], dev_in[4],
                     dev_in[5], rd)
    assert ops.tc_launch_count() == n0 + 1                                  # ONE launch for the pair
    assert rel_l2(y.detach().cpu().permute(0, 2, 1), yo) < 1e-4
    (y * r.permute(0, 2, 1).contiguous().to(DEV)).sum().backward()
    K.hifigan.join_side_streams(torch.device(DEV))
    torch.cuda.synchronize()
    # the product's own intermediate (bit-identical to the fused kernel's, scripts/rb_test.py) as the mask source
    with torch.no_grad():
        h_dev = ops.conv(xg.detach(), s1, ops.PreparedWeight(), dev_in[0], dev_in[1], dev_in[2]).cpu().permute(0, 2, 1)
    flipped = float(((h_dev > 0) != (ho > 0)).float().mean())
    ref_m, _, _ = run_oracle(h_dev)
    # (a) same side of every LeakyReLU kink: arithmetic parity of the gradient kernels
    assert rel_l2(xg.grad.cpu().permute(0, 2, 1), ref_m[0].grad) < 2e-4, ("dx, product masks", flipped)
    for got, want, nm in zip(dev_in, ref_m[1:], ("v1", "g1", "b1", "v2", "g2", "b2")):
        assert rel_l2(got.grad.cpu(), want.grad) < 5e-4, (nm, rel_l2(got.grad.cpu(), want.grad))
    # (b) against the plain oracle: each flipped element changes its gradient by the factor 1 / slope, so the
    # relative difference is ~ sqrt(fraction flipped) -- 3e-3 for a 1e-5 fraction -- whatever the arithmetic precision
    bound = 5e-4 + 3.0 * flipped ** 0.5
    assert rel_l2(xg.grad.cpu().permute(0, 2, 1), xo.grad) < bound, (flipped, bound)
    for got, want, nm in zip(dev_in, ref_in[1:], ("v1", "g1", "b1", "v2", "g2", "b2")):
        assert rel_l2(got.grad.cpu(), want.grad) < 2e-3 + 3.0 * flipped ** 0.5, (nm, rel_l2(got.grad.cpu(), want.grad))


def test_msd_avgpool_variant_matches_oracle():
    """MultiScaleDiscriminator(downsample_pooling="AvgPool1d") (hifigan.py:456-458,466: the class-default pooling, not used
    by the shipped yamls) -- outputs, feature maps, input and parameter gradients vs the oracle."""
    from oracle import hifigan as O
    cfg = dict(scales=3, downsample_pooling="AvgPool1d", downsample_pooling_params={"kernel_size": 4, "stride": 2, "padding": 2},
               discriminator_params=dict(in_channels=1, out_channels=1, kernel_sizes=[15, 41, 5, 3], channels=16,
                                         max_downsample_channels=64, max_groups=4, bias=True, downsample_scales=[2, 2, 4, 4, 1],
                                         nonlinear_activation="LeakyReLU", nonlinear_activation_params={"negative_slope": 0.1}),
               follow_official_norm=False)
    torch.manual_seed(11)
    m = K.MultiScaleDiscriminator(**cfg)
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    y = 0.3 * torch.randn(2, 1, 4096)
    yo = y.clone().requires_grad_(True)
    leaf = {k: (v.clone().requires_grad_(True) if v.is_floating_point() else v) for k, v in sd.items()}
    outs_o, fm_o = O.msd_forward(leaf, yo, True, **cfg)
    sum((o * o).sum() for o in outs_o).backward()
    m = m.to(DEV).train()
    yg = y.to(DEV).requires_grad_(True)
    outs, fm = m(yg)
    sum((o * o).sum() for o in outs).backward()
    K.hifigan.join_side_streams(torch.device(DEV))
    torch.cuda.synchronize()
    for a, b in zip(outs, outs_o):
        assert a.shape == b.shape and rel_l2(a.detach().cpu(), b.detach()) < 1e-4
    for fa, fb in zip(fm, fm_o):
        for a, b in zip(fa, fb):
            assert a.shape == b.shape and rel_l2(a.detach().cpu(), b.detach()) < 1e-4
    assert rel_l2(yg.grad.cpu(), yo.grad) < 5e-4
    for k, p in m.named_parameters():
        assert rel_l2(p.grad.cpu(), leaf[k].grad) < 2e-3, k
