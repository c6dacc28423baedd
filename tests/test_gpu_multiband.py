"""Multi-band HiFi-GAN on the GPU: the Bluestein route of the fused STFT (any n_fft) against float64 torch.stft / autograd,
the sub-band STFT loss and the multi-band generator against the unmodified reference's golden vectors, the PQMF kernels
against the float64 oracle, the GAN step with a PQMF against GAN_Trainer.train_step, its CUDA-graph replay, the reference
trainer's flow on the install()-patched names, and synthesize() with an attached PQMF."""
import types

import pytest
import torch

import kantts_b200 as K
from kantts_b200 import ops
from conftest import rel_l2
from oracle import hifigan as OH
from oracle import pqmf as OP

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


def _stft64(x, n_fft, hop, win):
    """audio_torch.stft (torch.stft, reflect padding, clamp 1e-7) in float64 on the CPU"""
    s = torch.stft(x, n_fft, hop, win, torch.hann_window(win, dtype=torch.float64), return_complex=True)
    return torch.sqrt(torch.clamp(s.real ** 2 + s.imag ** 2, min=1e-7)).transpose(2, 1)


@pytest.mark.parametrize("n_fft,hop,win", [(171, 15, 60), (384, 35, 150), (683, 75, 300), (1000, 123, 1000),
                                           (4095, 511, 3001), (32, 5, 32)])
def test_stft_any_n_fft_matches_float64(n_fft, hop, win):
    """The Bluestein route (n_fft not a power of two) and a small power of two: magnitude and input gradient.  Signals just
    above the reflect-padding limit n_fft / 2, a multiple of the hop, and longer ones."""
    gen = torch.Generator().manual_seed(n_fft)
    for t in (n_fft // 2 + 1, n_fft // 2 + 7, hop * (n_fft // (2 * hop) + 1), 3 * n_fft + 5):   # (a multiple of hop:
        # an odd n_fft has one frame fewer there)
        x = 0.3 * torch.randn(3, t, generator=gen, dtype=torch.float64)
        want = _stft64(x, n_fft, hop, win)
        r = torch.randn(want.shape, generator=gen, dtype=torch.float64)
        xr = x.clone().requires_grad_(True)
        (_stft64(xr, n_fft, hop, win) * r).sum().backward()
        xg = x.float().to(DEV).requires_grad_(True)
        got = K.stft(xg, n_fft, hop, win, torch.hann_window(win, device=DEV))
        assert got.shape == want.shape, (t, got.shape, want.shape)
        err = rel_l2(got.detach().cpu(), want)
        (got * r.float().to(DEV)).sum().backward()
        gerr = rel_l2(xg.grad.cpu(), xr.grad)
        print(f"n_fft={n_fft} t={t}: |X| rel err {err:.2e}, grad rel err {gerr:.2e}")
        assert err <= 1e-5 and gerr <= 1e-4, (t, err, gerr)


def test_mel_any_n_fft_matches_oracle():
    """The mel variant (zero padding, mel projection and its backward) on the Bluestein route."""
    gen = torch.Generator().manual_seed(3)
    y = (0.1 * torch.randn(2, 4000, generator=gen)).clamp(-1, 1)
    y_hat = (y + 0.05 * torch.randn(2, 4000, generator=gen)).requires_grad_(True)
    cfg = dict(fs=24000, fft_size=1200, hop_size=300, win_length=1200, fmin=0, fmax=8000)
    m = K.MelSpectrogram(**cfg).to(DEV)
    got = m(y.to(DEV))
    want = OH.mel_spectrogram(y.unsqueeze(1), **cfg)
    assert got.shape == want.shape and float((got.cpu() - want).abs().mean()) < 1e-4
    yh = y_hat.detach().to(DEV).requires_grad_(True)
    loss = K.MelSpectrogramLoss(**cfg).to(DEV)(yh, y.to(DEV))
    want_loss = torch.mean(torch.abs(OH.mel_spectrogram(y_hat.unsqueeze(1), **cfg) - want))
    want_loss.backward()
    loss.backward()
    assert abs(float(loss.detach()) - float(want_loss.detach())) < 1e-4
    assert rel_l2(yh.grad.cpu(), y_hat.grad) < 5e-3


def test_subband_stft_loss_matches_reference_golden(golden):
    g = golden("multiband_small")
    cfg = g.cfg["sub_stft"]
    y = g.t("stft/y").to(DEV)
    for n, h, w in zip(cfg["fft_sizes"], cfg["hop_sizes"], cfg["win_lengths"]):
        mag = K.stft(y.reshape(-1, y.shape[-1]), n, h, w, torch.hann_window(w, device=DEV))
        assert rel_l2(mag.cpu(), g.t(f"stft/mag_{n}")) < 1e-5, n
    y_hat = g.t("stft/y_hat").to(DEV).requires_grad_(True)
    sc, mag = K.MultiResolutionSTFTLoss(**cfg).to(DEV)(y_hat, y)
    assert abs(float(sc.detach()) - float(g.t("stft/sc"))) < 1e-4
    assert abs(float(mag.detach()) - float(g.t("stft/mag"))) < 1e-4
    (sc + mag).backward()
    assert rel_l2(y_hat.grad.cpu(), g.t("stft/grad")) < 5e-3


@pytest.mark.parametrize("ffma", [True, False])
@pytest.mark.parametrize("subbands", [4, 2])
def test_pqmf_matches_float64_oracle(subbands, ffma):
    p = K.PQMF(subbands).to(DEV)
    ha, hs = OP.filters(subbands)
    gen = torch.Generator().manual_seed(subbands)
    with _path(ffma):
        for batch, n in ((1, 7), (3, 64), (5, 600), (3, 2400)):
            x = 0.3 * torch.randn(batch, 1, subbands * n, generator=gen, dtype=torch.float64)
            xr = x.clone().requires_grad_(True)
            want = OP.analysis(xr, ha, subbands)
            r = torch.randn(want.shape, generator=gen, dtype=torch.float64)
            (want * r).sum().backward()
            xg = x.float().to(DEV).requires_grad_(True)
            got = p.analysis(xg)
            (got * r.float().to(DEV)).sum().backward()
            e1, e2 = rel_l2(got.detach().cpu(), want.detach()), rel_l2(xg.grad.cpu(), xr.grad)
            xs = torch.randn(batch, subbands, n, generator=gen, dtype=torch.float64)
            xsr = xs.clone().requires_grad_(True)
            want = OP.synthesis(xsr, hs, subbands)
            r = torch.randn(want.shape, generator=gen, dtype=torch.float64)
            (want * r).sum().backward()
            xsg = xs.float().to(DEV).requires_grad_(True)
            got_s = p.synthesis(xsg)
            (got_s * r.float().to(DEV)).sum().backward()
            e3, e4 = rel_l2(got_s.detach().cpu(), want.detach()), rel_l2(xsg.grad.cpu(), xsr.grad)
            print(f"S={subbands} ffma={ffma} B={batch} n={n}: analysis {e1:.2e} / {e2:.2e}, synthesis {e3:.2e} / {e4:.2e}")
            assert got.shape == (batch, subbands, n) and got_s.shape == (batch, 1, subbands * n)
            assert max(e1, e2, e3, e4) <= 1e-5, (batch, n, e1, e2, e3, e4)


@pytest.mark.parametrize("ffma", [True, False])
def test_multiband_generator_matches_reference_golden(golden, ffma):
    g = golden("multiband_small")
    gen = K.Generator(**g.cfg["generator"])
    gen.load_state_dict(g.group("gen/sd/"), strict=True)
    gen = gen.to(DEV).eval()
    p = K.PQMF(4).to(DEV)
    with torch.no_grad(), _path(ffma):
        y_mb = gen(g.t("gen/x").to(DEV))
        y = p.synthesis(y_mb)
    tol = 1e-5 if ffma else 1e-4
    assert y_mb.shape == g.t("gen/y_mb").shape and y.shape == g.t("gen/y").shape
    assert rel_l2(y_mb.cpu(), g.t("gen/y_mb")) < tol
    assert rel_l2(y.cpu(), g.t("gen/y")) < tol


def _mb_config(g):
    adam = {"type": "Adam", "params": {"lr": 2e-4, "betas": [0.5, 0.9], "weight_decay": 0.0}}
    sched = {"type": "MultiStepLR", "params": {"gamma": 0.5, "milestones": [200000]}}
    return {"Model": {"Generator": {"params": g.cfg["generator"], "optimizer": adam, "scheduler": sched},
                      "MultiScaleDiscriminator": {"params": g.cfg["msd"], "optimizer": adam, "scheduler": sched},
                      "MultiPeriodDiscriminator": {"params": g.cfg["mpd"], "optimizer": adam, "scheduler": sched}},
            "Loss": g.cfg["loss"], "generator_train_start_steps": 1, "discriminator_train_start_steps": 0,
            "generator_grad_norm": -1, "discriminator_grad_norm": -1}


def _build(g, cfg, **kw):
    torch.manual_seed(0)
    model, opt, sched = K.hifigan_model_builder(cfg, DEV)
    model["generator"].load_state_dict(g.group("before/g/"))
    model["discriminator"]["MultiScaleDiscriminator"].load_state_dict(g.group("before/msd/"))
    model["discriminator"]["MultiPeriodDiscriminator"].load_state_dict(g.group("before/mpd/"))
    crit = K.criterion_builder(cfg, DEV)
    return K.GanStep(model, opt, sched, crit, cfg, **kw), model


_LOSSES = ("spectral_convergence_loss", "log_stft_magnitude_loss", "sub_spectral_convergence_loss",
           "sub_log_stft_magnitude_loss", "mel_loss", "feature_matching_loss", "generator_loss", "real_loss", "fake_loss",
           "discriminator_loss")


def _check_against_trainer(g, log, mods):
    for k in _LOSSES:
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


@pytest.mark.parametrize("pair", [True, False])
@pytest.mark.parametrize("force_ffma", [True, False])
def test_multiband_gan_step_matches_reference_trainer(golden, force_ffma, pair):
    g = golden("trainstep_multiband_small")
    cfg = _mb_config(g)
    with _path(force_ffma):
        step, model = _build(g, cfg, pair_discriminators=pair)
        assert isinstance(model["pqmf"], K.PQMF)
        log = K.train.losses_to_float(step.step((g.t("y").to(DEV), g.t("x").to(DEV))))
    _check_against_trainer(g, log, {"g": model["generator"], "msd": model["discriminator"]["MultiScaleDiscriminator"],
                                    "mpd": model["discriminator"]["MultiPeriodDiscriminator"]})


def test_multiband_cuda_graph_step_matches_eager(golden):
    g = golden("trainstep_multiband_small")
    cfg = _mb_config(g)
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
        assert set(le) == set(lg) and "sub_spectral_convergence_loss" in le
        for k in le:
            tol = (3e-3 if i <= 3 else 3e-2) * (5.0 if k == "feature_matching_loss" else 1.0)   # as test_gpu_graph
            assert abs(le[k] - lg[k]) <= tol * max(1.0, abs(le[k])), (i, k, le[k], lg[k])
    for k, v in m_e["generator"].state_dict().items():
        w = m_g["generator"].state_dict()[k]
        assert float((v - w).abs().max()) <= 5e-3 * max(1.0, float(v.abs().max())), k


def test_install_runs_the_trainers_multiband_flow(golden):
    """install() on a stub ``kantts`` namespace; the reference's builders look the classes up by name
    (kantts/models/__init__.py:38-67: Generator, the discriminators, PQMF; loss.py:528-544: loss_dict) and the statements
    of GAN_Trainer.train_step with a PQMF (trainer.py:469-589) drive them through autograd and torch's Adam on the device.
    The result must be the unmodified trainer's step (trainstep_multiband_small)."""
    g = golden("trainstep_multiband_small")
    models = types.SimpleNamespace(pqmf=types.SimpleNamespace(), hifigan=types.SimpleNamespace(hifigan=types.SimpleNamespace()))
    loss_mod = types.SimpleNamespace(loss_dict={})
    K.install(kantts_models=models, kantts_loss=loss_mod, kantts_audio=types.SimpleNamespace())
    assert models.pqmf.PQMF is K.PQMF
    torch.manual_seed(0)
    G = models.Generator(**g.cfg["generator"]).to(DEV)
    D = {"MultiScaleDiscriminator": models.MultiScaleDiscriminator(**g.cfg["msd"]).to(DEV),
         "MultiPeriodDiscriminator": models.MultiPeriodDiscriminator(**g.cfg["mpd"]).to(DEV)}
    G.load_state_dict(g.group("before/g/"))
    for k, m in D.items():
        m.load_state_dict(g.group(f"before/{'msd' if k.startswith('MultiScale') else 'mpd'}/"))
    pqmf = models.PQMF(subbands=g.cfg["generator"]["out_channels"]).to(DEV)
    crit = {}
    for key, spec in g.cfg["loss"].items():
        if spec.get("enable", False):
            crit[key] = loss_mod.loss_dict[key](**spec.get("params", {})).to(DEV)
            setattr(crit[key], "weights", spec.get("weights", 1.0))
    crit["sub_stft"] = crit["subband_stft_loss"]
    mk = lambda m: torch.optim.Adam(m.parameters(), lr=2e-4, betas=(0.5, 0.9), weight_decay=0.0)  # noqa: E731
    og, od = mk(G), {k: mk(m) for k, m in D.items()}
    y, x = g.t("y").to(DEV), g.t("x").to(DEV)
    log = {}
    # ---- trainer.py:473-553
    y_mb_ = G(x)
    y_ = pqmf.synthesis(y_mb_)
    sc_loss, mag_loss = crit["stft_loss"](y_, y)
    gen_loss = (sc_loss + mag_loss) * crit["stft_loss"].weights
    gen_loss = gen_loss * 0.5
    y_mb = pqmf.analysis(y)
    sub_sc_loss, sub_mag_loss = crit["sub_stft"](y_mb_, y_mb)
    gen_loss = gen_loss + 0.5 * (sub_sc_loss + sub_mag_loss)
    mel_loss = crit["mel_loss"](y_, y)
    gen_loss = gen_loss + mel_loss * crit["mel_loss"].weights
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
        y_ = pqmf.synthesis(G(x))
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
    log = dict(spectral_convergence_loss=sc_loss, log_stft_magnitude_loss=mag_loss, sub_spectral_convergence_loss=sub_sc_loss,
               sub_log_stft_magnitude_loss=sub_mag_loss, mel_loss=mel_loss, feature_matching_loss=fm_loss,
               generator_loss=gen_loss, real_loss=real_t, fake_loss=fake_t, discriminator_loss=dis_loss)
    _check_against_trainer(g, K.train.losses_to_float(log), {"g": G, "msd": D["MultiScaleDiscriminator"],
                                                            "mpd": D["MultiPeriodDiscriminator"]})


def test_synthesize_multiband_matches_oracle(golden):
    from golden.make_batch import make_sambert_batch
    from oracle import sambert as OS
    g = golden("sambert_small_infer")
    cfg = g.cfg
    batch = make_sambert_batch(cfg, B=3, L=9, gen=torch.Generator().manual_seed(31), short=3)
    inputs = [batch[k] for k in ("inputs_ling", "inputs_emotion", "inputs_speaker", "input_lengths")]
    am = K.KanTtsSAMBERT(cfg)
    am.load_state_dict(g.group("sd/"), strict=True)
    am = am.to(DEV).eval()
    gcfg = dict(in_channels=cfg["num_mels"], out_channels=4, channels=32, upsample_scales=[5, 3, 2, 2],
                upsample_kernal_sizes=[10, 6, 4, 4], resblock_kernel_sizes=[3, 7], resblock_dilations=[[1, 3], [1, 3]])
    torch.manual_seed(7)
    gen = K.Generator(**gcfg).to(DEV).eval()
    dev_inputs = [t.to(DEV) for t in inputs]
    with torch.no_grad(), _path(True):
        with pytest.raises(ValueError, match="pqmf"):
            K.synthesize(am, gen, *dev_inputs)
        gen.pqmf = K.PQMF().to(DEV)                       # infer_hifigan.py:47-53
        wavs, res = K.synthesize(am, gen, *dev_inputs)
        want_o = OS.sambert_infer(g.group("sd/"), cfg, *inputs)
        gsd = {k: v.detach().cpu() for k, v in gen.state_dict().items() if not k.startswith("pqmf.")}
        y_mb = OH.generator_forward(gsd, want_o["postnet_outputs"].transpose(1, 2), **gcfg)
        wav_o = OP.synthesis(y_mb.double(), OP.filters(4)[1], 4)
    frames = res["LR_length_rounded"].cpu()
    for b, w in enumerate(wavs):
        n = int(frames[b]) * 60 * 4
        assert w.shape == (n,), (b, w.shape, n)
        err = rel_l2(w.cpu(), wav_o[b, 0, :n])
        print(f"slot {b}: {n} samples, rel err vs oracle {err:.3e}")
        assert err <= 1e-4
