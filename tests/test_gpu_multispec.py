"""MultiSpecDiscriminator on the GPU: the module against the unmodified reference's golden vectors on both conv paths
(outputs, feature maps with their column classes, parameter gradients, the spectral-norm power iteration), the column kernels
against a float64 expand / sum, forward_pair and real-half reuse, the generator's missing gradient, GanStep against
GAN_Trainer.train_step (paired and unpaired, eager and CUDA graph) and the reference trainer's flow on the install()-patched
names."""
import types

import pytest
import torch

import kantts_b200 as K
from kantts_b200 import ops
from conftest import rel_l2
from test_multispec_cpu import case_cfg, expand_columns, fill_params, probe

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


class _path:
    """set_force_ffma(flag) for the duration of a block."""

    def __init__(self, ffma):
        self.ffma = ffma

    def __enter__(self):
        ops.set_force_ffma(self.ffma)

    def __exit__(self, *exc):
        ops.set_force_ffma(False)
        return False


def _module(g, tag):
    """The golden's module of case ``tag``: a spectral one with its stored state_dict, the others with fill_params."""
    if tag == "spectral":
        m = K.MultiSpecDiscriminator(**g.cfg["spectral"])
        m.load_state_dict(g.group("spectral/sd_before/"), strict=True)
    else:
        m = K.MultiSpecDiscriminator(**case_cfg(g.cfg["cases"][tag]))
        fill_params(m)
    return m.to(DEV)


def _lengths(g, tag):
    return [g.t("spectral/wav").shape[-1]] * 2 if tag == "spectral" else g.cfg["cases"][tag]["lengths"]


def _check_param_grads(m, refg, exact):
    """Parameter gradients against a reference, with the bounds of test_gpu_parity._check_param_grads: every tensor within
    1e-4 relative on the exact path.  On the bf16x3 tensor cores a gradient that is a small residual of large cancelling
    sums (a weight-norm gain, above all) loses relative accuracy: the median tensor within 5e-4, the whole gradient vector
    within 1e-3, the worst tensor within 1e-2."""
    errs = sorted((rel_l2(p.grad.cpu(), refg[k]), k) for k, p in m.named_parameters())
    num = sum(float(((p.grad.cpu() - refg[k]).double() ** 2).sum()) for k, p in m.named_parameters())
    den = sum(float((refg[k].double() ** 2).sum()) for k, p in m.named_parameters())
    print(f"exact={exact}: median {errs[len(errs) // 2][0]:.2e} global {(num / den) ** 0.5:.2e} worst {errs[-3:]}")
    if exact:
        assert errs[-1][0] < 1e-4, errs[-3:]
        return
    assert errs[len(errs) // 2][0] < 5e-4 and (num / den) ** 0.5 < 1e-3 and errs[-1][0] < 1e-2, errs[-3:]


@pytest.mark.parametrize("force_ffma", [True, False])
@pytest.mark.parametrize("tag", ["defaults", "spec"])
def test_module_matches_reference_golden(golden, tag, force_ffma):
    """Outputs and every feature map (columns of all classes included) for both waveform lengths; then the parameter
    gradients of sum(out * r) + sum(fmap * r).  1e-5 relative L2 on the exact path, 1e-4 on the tensor cores."""
    g = golden("multispec_small")
    tol = 1e-5 if force_ffma else 1e-4
    with _path(force_ffma):
        m = _module(g, tag)
        for n in _lengths(g, tag):
            with torch.no_grad():
                outs, fmaps = m(g.t(f"{tag}/wav_{n}").to(DEV))
            for i, (o, fm) in enumerate(zip(outs, fmaps)):
                want = g.t(f"{tag}/out_{n}_{i}")
                assert o.shape == want.shape and rel_l2(o.cpu(), want) < tol, (n, i, rel_l2(o.cpu(), want))
                assert len(fm) == 6
                for l, f in enumerate(fm):
                    want = g.t(f"{tag}/fmap_{n}_{i}_{l}")
                    assert f.shape == want.shape and rel_l2(f.cpu(), want) < tol, (n, i, l, rel_l2(f.cpu(), want))
        outs, fmaps = m(g.t(f"{tag}/wav_{_lengths(g, tag)[-1]}").to(DEV))
        total = 0.0
        for i, (o, fm) in enumerate(zip(outs, fmaps)):
            total = total + (o * probe(o.shape, 100 * i + 99).to(DEV)).sum()
            for l, f in enumerate(fm):
                total = total + (f * probe(f.shape, 100 * i + l).to(DEV)).sum()
        total.backward()
        K.hifigan.join_side_streams(torch.device(DEV))
    _check_param_grads(m, g.group(f"{tag}/grad/"), force_ffma)


REFERENCE_RESOLUTIONS = dict(fft_sizes=[1024, 2048, 512], hop_sizes=[120, 240, 50], win_lengths=[600, 1200, 240])


def _mrd_float64(m, params, wav):
    """float64 restatement of the reference's forward (hifigan.py:481-617 on audio_torch.stft) with ``params`` (name ->
    tensor) in place of m's parameters: torch.stft and weight-normed F.conv2d with the int padding of the width-1 axis."""
    import torch.nn.functional as F

    def conv(prefix, x, stride, pad):
        v, g, b = params[prefix + "weight_v"], params[prefix + "weight_g"], params[prefix + "bias"]
        return F.conv2d(x, v * (g / v.norm(2, dim=(1, 2, 3), keepdim=True)), b, stride=stride, padding=pad)

    outs, fmaps = [], []
    for i, d in enumerate(m.discriminators):
        s = torch.stft(wav.squeeze(1), d.fft_size, d.shift_size, d.win_length,
                       torch.hann_window(d.win_length, dtype=torch.float64), return_complex=True)
        x = torch.sqrt(torch.clamp(s.real ** 2 + s.imag ** 2, min=1e-7)).unsqueeze(-1)
        fm = []
        for l, seq in enumerate(d.convs):
            k, stride = seq[0].spec.kernel, seq[0].spec.stride
            x = F.leaky_relu(conv(f"discriminators.{i}.convs.{l}.0.", x, (stride, 1), (k - 1) // 2), 0.1)
            fm.append(x)
        x = conv(f"discriminators.{i}.conv_post.", x, 1, (1, 0))
        fm.append(x)
        outs.append(x)
        fmaps.append(fm)
    return outs, fmaps


@pytest.mark.parametrize("force_ffma", [True, False])
@pytest.mark.parametrize("params", [{"channels": 15, "init_kernel": 1, "kernel_size": 11},
                                    {"channels": 4, "init_kernel": 15, "kernel_size": 11}], ids=["defaults", "spec"])
def test_reference_resolutions_match_float64(params, force_ffma):
    """The reference's resolutions (first layers of 513 / 1025 / 257 input channels, odd row pitches) against a float64
    restatement: outputs, feature maps and parameter gradients."""
    m = K.MultiSpecDiscriminator(**REFERENCE_RESOLUTIONS, discriminator_params=dict(params, stride=2)).to(DEV)
    fill_params(m)
    wav = (0.2 * torch.randn(2, 1, 4801, generator=torch.Generator().manual_seed(11))).clamp(-1, 1)
    p64 = {k: v.detach().cpu().double().requires_grad_(True) for k, v in m.named_parameters()}
    want_o, want_f = _mrd_float64(m, p64, wav.double())
    with _path(force_ffma):
        got_o, got_f = m(wav.to(DEV))
        total, total64 = 0.0, 0.0
        for i in range(len(want_o)):
            for l, (a, b) in enumerate(zip(got_f[i], want_f[i])):
                assert a.shape == b.shape and rel_l2(a.detach().cpu(), b) < (1e-5 if force_ffma else 1e-4), (i, l)
                r = probe(a.shape, 100 * i + l)
                total, total64 = total + (a * r.to(DEV)).sum(), total64 + (b * r.double()).sum()
            assert torch.equal(got_o[i].detach(), got_f[i][-1].detach())
        total.backward()
        K.hifigan.join_side_streams(torch.device(DEV))
    total64.backward()
    _check_param_grads(m, {k: v.grad for k, v in p64.items()}, force_ffma)


def test_spectral_norm_power_iteration_matches_reference(golden):
    """Two train-mode forwards of a spectral-normed MRD: weight_u / weight_v move as the reference's hook moves them, and
    the second forward uses the twice-iterated sigma."""
    g = golden("multispec_small")
    m = _module(g, "spectral")
    m.train()
    wav = g.t("spectral/wav").to(DEV)
    with torch.no_grad():
        m(wav)
        outs, fmaps = m(wav)
    sd = m.state_dict()
    for k, v in g.group("spectral/sd_after/").items():
        assert rel_l2(sd[k].cpu(), v) < 1e-5, k
    for i, (o, fm) in enumerate(zip(outs, fmaps)):
        assert rel_l2(o.cpu(), g.t(f"spectral/out_{i}")) < 1e-4, i
        for l, f in enumerate(fm):
            assert rel_l2(f.cpu(), g.t(f"spectral/fmap_{i}_{l}")) < 1e-4, (i, l)


@pytest.mark.parametrize("batch,t,c,reach", [(3, 7, 5, (5,)), (4, 13, 15, (5, 10, 15, 17)), (2, 9, 1, (7, 12, 17, 22, 24)),
                                             (5, 3, 32, ()), (1, 40, 6, (1, 2, 3))])
def test_column_kernels_match_float64(batch, t, c, reach):
    """kt_spec_columns_fwd is a gather (bit-exact); kt_spec_columns_bwd sums each class over its columns and the items (float64
    reference, and the same bits on a second run)."""
    gen = torch.Generator().manual_seed(batch * 100 + t)
    rows = torch.randn(batch + len(reach), t, c, generator=gen, dtype=torch.float64)
    x = rows.float().to(DEV).requires_grad_(True)
    y = ops.SpecColumnsFn.apply(x, batch, reach)
    want = expand_columns(rows, batch, reach)
    assert y.shape == want.shape and torch.equal(y.cpu(), want.float())
    dout = torch.randn(want.shape, generator=gen, dtype=torch.float64)
    want_grad = torch.autograd.grad((expand_columns(rows.requires_grad_(True), batch, reach) * dout).sum(), rows)[0]
    grads = [torch.autograd.grad((y * dout.float().to(DEV)).sum(), x, retain_graph=True)[0].cpu() for _ in range(2)]
    assert torch.equal(grads[0], grads[1])
    err = float((grads[0].double() - want_grad).abs().max() / want_grad.abs().max())
    assert err < 1e-6, err


@pytest.mark.parametrize("spectral", [False, True])
def test_forward_pair_equals_two_calls(golden, spectral):
    """forward_pair(ya, yb) == (d(ya), d(yb)) with the class rows after the 2B signal items, under grad_items(B); for a
    spectral-normed MRD also the power-iteration state."""
    g = golden("multispec_small")
    tag = "spectral" if spectral else "defaults"
    T = _lengths(g, tag)[-1]
    torch.manual_seed(5)
    ya = (0.3 * torch.randn(3, 1, T)).to(DEV)
    yb = (0.3 * torch.randn(3, 1, T)).to(DEV)
    res = {}
    for mode in ("two", "pair"):
        d = _module(g, tag)
        d.train()
        if mode == "two":
            oa, fa = d(ya)
            with torch.no_grad():
                ob, fb = d(yb)
        else:
            with ops.grad_items(3):
                (oa, fa), (ob, fb) = d.forward_pair(ya, yb, detach_b=True)
            assert not any(o.requires_grad for o in ob)
        K.hifigan.join_side_streams(torch.device(DEV))
        res[mode] = ([o.detach().clone() for o in oa + ob] + [f.detach().clone() for fm in fa + fb for f in fm],
                     {k: v.clone() for k, v in d.state_dict().items() if k.endswith(("weight_u", "weight_v"))})
    for a, b in zip(res["two"][0], res["pair"][0]):
        assert a.shape == b.shape and rel_l2(b, a) < 1e-5, rel_l2(b, a)
    for k, v in res["two"][1].items():
        assert rel_l2(res["pair"][1][k], v) < 1e-6, k


def test_real_half_and_class_rows_reuse_matches_recompute(golden):
    """pair_state("record") then pair_state("reuse", B): only the first B items are recomputed, the real half and the class
    rows come from the record.  The results equal a plain pair forward of the same batch."""
    g = golden("multispec_small")
    d = _module(g, "defaults")
    gen = torch.Generator().manual_seed(3)
    y0, y, y1 = [(0.3 * torch.randn(2, 1, _lengths(g, "defaults")[0], generator=gen)).to(DEV) for _ in range(3)]
    with torch.no_grad():
        with ops.pair_state("record"):
            d.forward_pair(y0, y)
        with ops.pair_state("reuse", 2):
            got = d.forward_pair(y1, y)
        want = d.forward_pair(y1, y)
    flat = lambda r: [o for o in r[0]] + [f for fm in r[1] for f in fm]  # noqa: E731
    for a, b in zip(flat(want[0]), flat(got[0])):             # recomputed on a batch of 2
        assert rel_l2(b, a) < 1e-5, rel_l2(b, a)
    for a, b in zip(flat(want[1]), flat(got[1])):             # recorded
        assert torch.equal(a, b)


def test_waveform_gets_no_gradient_from_the_mrd(golden):
    g = golden("multispec_small")
    d = _module(g, "defaults")
    wav = g.t(f"defaults/wav_{_lengths(g, 'defaults')[-1]}").to(DEV).requires_grad_(True)
    outs, fmaps = d(wav)
    assert all(o.requires_grad for o in outs)
    sum(o.sum() for o in outs).backward()
    assert wav.grad is None


def _config(g, mrd=True):
    adam = {"type": "Adam", "params": {"lr": 2e-4, "betas": [0.5, 0.9], "weight_decay": 0.0}}
    sched = {"type": "MultiStepLR", "params": {"gamma": 0.5, "milestones": [200000]}}
    model = {"Generator": {"params": g.cfg["generator"], "optimizer": adam, "scheduler": sched},
             "MultiScaleDiscriminator": {"params": g.cfg["msd"], "optimizer": adam, "scheduler": sched},
             "MultiPeriodDiscriminator": {"params": g.cfg["mpd"], "optimizer": adam, "scheduler": sched}}
    if mrd:
        model["MultiSpecDiscriminator"] = {"params": g.cfg["mrd"], "optimizer": adam, "scheduler": sched}
    return {"Model": model, "Loss": g.cfg["loss"], "generator_train_start_steps": 1, "discriminator_train_start_steps": 0,
            "generator_grad_norm": -1, "discriminator_grad_norm": -1}


_TAGS = {"MultiScaleDiscriminator": "msd", "MultiPeriodDiscriminator": "mpd", "MultiSpecDiscriminator": "mrd"}


def _build(g, cfg, **kw):
    torch.manual_seed(0)
    model, opt, sched = K.hifigan_model_builder(cfg, DEV)
    model["generator"].load_state_dict(g.group("before/g/"))
    for name, m in model["discriminator"].items():
        m.load_state_dict(g.group(f"before/{_TAGS[name]}/"))
    crit = K.criterion_builder(cfg, DEV)
    return K.GanStep(model, opt, sched, crit, cfg, **kw), model


def _check_against_trainer(g, log, mods):
    for k in ("mel_loss", "feature_matching_loss", "generator_loss", "real_loss", "fake_loss", "discriminator_loss"):
        ref = float(g.arrays["loss/" + k])
        assert abs(log[k] - ref) <= 2e-4 * max(1.0, abs(ref)), (k, log[k], ref)
    for tag, m in mods.items():
        after, before = g.group(f"after/{tag}/"), g.group(f"before/{tag}/")
        sd = m.state_dict()
        num = den = 0.0
        for k, v in after.items():
            num += float(((sd[k].cpu() - v).double() ** 2).sum())
            den += float(((before[k] - v).double() ** 2).sum())
        assert num <= 2e-2 * den, (tag, num, den)      # as test_gan_train_step_matches_reference_trainer


def _mods(model):
    return {"g": model["generator"], **{_TAGS[k]: m for k, m in model["discriminator"].items()}}


@pytest.mark.parametrize("pair", [True, False])
@pytest.mark.parametrize("force_ffma", [True, False])
def test_gan_step_with_mrd_matches_reference_trainer(golden, force_ffma, pair):
    g = golden("trainstep_multispec_small")
    cfg = _config(g)
    with _path(force_ffma):
        step, model = _build(g, cfg, pair_discriminators=pair)
        assert step._can_pair() == pair        # an MRD in the model keeps pairing on for every discriminator
        log = K.train.losses_to_float(step.step((g.t("y").to(DEV), g.t("x").to(DEV))))
    _check_against_trainer(g, log, _mods(model))


def test_mrd_leaves_the_generator_gradients_bit_identical(golden):
    """The MRD passes no gradient to the generator: a step on {MSD, MPD, MRD} gives the generator exactly the gradients and
    the parameters of a step on {MSD, MPD} with the same weights.  Only the logged loss values differ."""
    g = golden("trainstep_multispec_small")
    y, x = g.t("y").to(DEV), g.t("x").to(DEV)
    res = {}
    for mrd in (False, True):
        step, model = _build(g, _config(g, mrd))
        log = K.train.losses_to_float(step.step((y, x)))
        torch.cuda.synchronize()
        res[mrd] = (step.g_grads.flat.clone(), {k: v.clone() for k, v in model["generator"].state_dict().items()}, log)
    assert torch.equal(res[False][0], res[True][0])
    for k, v in res[False][1].items():
        assert torch.equal(v, res[True][1][k]), k
    assert res[False][2]["mel_loss"] == res[True][2]["mel_loss"]
    assert res[False][2]["generator_loss"] != res[True][2]["generator_loss"]


def test_cuda_graph_step_with_mrd_matches_eager(golden):
    g = golden("trainstep_multispec_small")
    cfg = _config(g)
    y, x = g.t("y").to(DEV), g.t("x").to(DEV)
    batches = [(y, x), (y.flip(0), x.flip(0)), ((y * 0.5).contiguous(), x), (y, (x * 0.9).contiguous()),
               (y.roll(7, -1), x), (y, x)]
    eager, m_e = _build(g, cfg)
    traj_e = [K.train.losses_to_float(eager.step(b)) for b in batches]
    torch.cuda.synchronize()
    graph, m_g = _build(g, cfg, cuda_graph=True, graph_warmup=2)
    traj_g = [K.train.losses_to_float(graph.step(b)) for b in batches]   # steps 0-1 eager warm-up, 2 capture, 3+ replay
    assert graph._graphs is not None
    for i, (le, lg) in enumerate(zip(traj_e, traj_g)):
        assert set(le) == set(lg)
        for k in le:
            tol = (3e-3 if i <= 3 else 3e-2) * (5.0 if k == "feature_matching_loss" else 1.0)   # as test_gpu_graph
            assert abs(le[k] - lg[k]) <= tol * max(1.0, abs(le[k])), (i, k, le[k], lg[k])
    for tag, m in _mods(m_e).items():
        sd_g = _mods(m_g)[tag].state_dict()
        for k, v in m.state_dict().items():
            assert float((v - sd_g[k]).abs().max()) <= 5e-3 * max(1.0, float(v.abs().max())), (tag, k)


def test_install_runs_the_trainers_flow_with_mrd(golden):
    """install() on a stub ``kantts`` namespace; the statements of GAN_Trainer.train_step (trainer.py:469-589) drive the
    patched classes, MultiSpecDiscriminator included, through autograd and torch's Adam.  The result must be the unmodified
    trainer's step (trainstep_multispec_small)."""
    g = golden("trainstep_multispec_small")
    models = types.SimpleNamespace(hifigan=types.SimpleNamespace(hifigan=types.SimpleNamespace()))
    loss_mod = types.SimpleNamespace(loss_dict={})
    K.install(kantts_models=models, kantts_loss=loss_mod, kantts_audio=types.SimpleNamespace())
    assert models.MultiSpecDiscriminator is K.MultiSpecDiscriminator
    torch.manual_seed(0)
    G = models.Generator(**g.cfg["generator"]).to(DEV)
    D = {name: getattr(models, name)(**g.cfg[tag]).to(DEV) for name, tag in _TAGS.items()}
    G.load_state_dict(g.group("before/g/"))
    for name, m in D.items():
        m.load_state_dict(g.group(f"before/{_TAGS[name]}/"))
    crit = {}
    for key, spec in g.cfg["loss"].items():
        if spec.get("enable", False):
            crit[key] = loss_mod.loss_dict[key](**spec.get("params", {})).to(DEV)
            setattr(crit[key], "weights", spec.get("weights", 1.0))
    mk = lambda m: torch.optim.Adam(m.parameters(), lr=2e-4, betas=(0.5, 0.9), weight_decay=0.0)  # noqa: E731
    og, od = mk(G), {k: mk(m) for k, m in D.items()}
    y, x = g.t("y").to(DEV), g.t("x").to(DEV)
    # ---- trainer.py:473-553
    y_ = G(x)
    mel_loss = crit["mel_loss"](y_, y)
    gen_loss = mel_loss * crit["mel_loss"].weights
    adv_loss, fm_, fm = 0.0, [], []
    for k in D:
        p_, fmap_ = D[k](y_)
        fm_.append(fmap_)
        adv_loss = adv_loss + crit["generator_adv_loss"](p_)
    gen_loss = gen_loss + adv_loss * crit["generator_adv_loss"].weights
    for k in D:
        with torch.no_grad():
            fm.append(D[k](y)[1])
    fm_loss = 0.0
    for a, b in zip(fm, fm_):
        fm_loss = fm_loss + crit["feat_match_loss"](a, b)
    gen_loss = gen_loss + fm_loss * crit["feat_match_loss"].weights
    og.zero_grad()
    gen_loss.backward()
    K.hifigan.join_side_streams(torch.device(DEV))
    og.step()
    # ---- trainer.py:556-589
    with torch.no_grad():
        y_ = G(x)
    dis_loss, real_t, fake_t = 0.0, 0.0, 0.0
    for k in D:
        p, _ = D[k](y)
        p_, _ = D[k](y_.detach())
        real_loss, fake_loss = crit["discriminator_adv_loss"](p_, p)
        dis_loss = dis_loss + real_loss + fake_loss
        real_t, fake_t = real_t + real_loss, fake_t + fake_loss
    for o in od.values():
        o.zero_grad()
    dis_loss.backward()
    K.hifigan.join_side_streams(torch.device(DEV))
    for o in od.values():
        o.step()
    log = dict(mel_loss=mel_loss, feature_matching_loss=fm_loss, generator_loss=gen_loss, real_loss=real_t, fake_loss=fake_t,
               discriminator_loss=dis_loss)
    _check_against_trainer(g, K.train.losses_to_float(log), {"g": G, **{_TAGS[k]: m for k, m in D.items()}})
