"""tests/golden/multispec_small.npz, trainstep_multispec_small.npz and multispec_init_checksums.json: the multi-resolution
spectrogram discriminator of the UNMODIFIED reference (kantts/models/hifigan/hifigan.py:481-617, MultiSpecDiscriminator /
SpecDiscriminator) on CPU, imported through oracle/ref_shims.py.

multispec_small.npz, for each parameter set {tag} in CASES:
  cfg["layouts"][{tag}]   the state_dict layout: [key, shape] in order (spectral too)
                          the parameters are test_multispec_cpu.fill_params's fixed values (computed, not stored)
  {tag}/wav_{n}           waveforms (2, 1, n) for the case's two lengths: a multiple of every hop, and of none
  {tag}/out_{n}_{i}       the output of resolution i; {tag}/fmap_{n}_{i}_{l} its feature map l
  {tag}/grad/<param>      parameter gradients of sum(out_i * probe) + sum_l sum(fmap_l * probe) on the second wav, with the
                          fixed weights of test_multispec_cpu.probe (computed, not stored)
spectral/...              a spectral-normed MultiSpecDiscriminator: sd_before, two train-mode forwards on wav,
                          sd_after (weight_u / weight_v moved twice) and the second forward's outputs and feature maps
trainstep_multispec_small.npz
  one GAN_Trainer.train_step with the small generator and MPD of make_golden_multiband's train step (the generator
  full-band), an 8-channel MSD and a small MultiSpecDiscriminator, in the layout of trainstep_multiband_small.npz
  (before/, after/, loss/, y, x).
multispec_init_checksums.json
  make_golden_disc_init.checksums of MultiSpecDiscriminator(discriminator_params=DEFAULTS_FIXED) built after
  torch.manual_seed(5), weight-normed and spectral-normed.

Build container only:  python tests/golden/make_golden_multispec.py [module | trainstep | init]"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from make_golden import LOSS_CFG, randomize, save  # noqa: E402  (imports the reference)
from make_golden_multiband import TRAIN_G_MB, TRAIN_MPD, TRAIN_MSD as TRAIN_MSD_MB  # noqa: E402
from make_golden_disc_init import checksums  # noqa: E402
from kantts.models.hifigan.hifigan import (Generator, MultiPeriodDiscriminator, MultiScaleDiscriminator,  # noqa: E402
                                           MultiSpecDiscriminator)
from kantts.train.loss import criterion_builder  # noqa: E402

sys.path.insert(0, os.path.dirname(HERE))
from test_multispec_cpu import fill_params, probe  # noqa: E402

torch.set_num_threads(8)

# the reference's MultiSpecDiscriminator defaults with the one key its SpecDiscriminator accepts (kernel_size, not
# kernel_sizes)
DEFAULTS_FIXED = {"channels": 15, "init_kernel": 1, "kernel_size": 11, "stride": 2, "use_spectral_norm": False,
                  "window": "hann_window", "nonlinear_activation": "LeakyReLU",
                  "nonlinear_activation_params": {"negative_slope": 0.1}}
# Reduced resolutions (the reference's are FFT 1024 / 2048 / 512): the first layer has fft_size/2 + 1 input channels, and
# the fixture stays small.  Each case has its own waveform lengths, longer than its largest fft_size / 2 (reflect padding):
# the first a multiple of every hop, the second of none.
CASES = {
    "defaults": dict(fft_sizes=[256, 512, 128], hop_sizes=[30, 60, 15], win_lengths=[120, 240, 60],
                     discriminator_params=DEFAULTS_FIXED, lengths=[300, 301]),
    # SpecDiscriminator's own defaults (init_kernel 15, kernel_size 11) with fewer channels
    "spec": dict(fft_sizes=[128, 256, 64], hop_sizes=[15, 30, 8], win_lengths=[60, 120, 30],
                 discriminator_params={"channels": 4, "init_kernel": 15, "kernel_size": 11, "stride": 2},
                 lengths=[240, 241]),
}
SPECTRAL = dict(fft_sizes=[128, 256], hop_sizes=[15, 30], win_lengths=[60, 120],
                discriminator_params={"channels": 4, "init_kernel": 3, "kernel_size": 5, "stride": 2,
                                      "use_spectral_norm": True})
SPECTRAL_LENGTH = 241
# make_golden_multiband's small train-step generator as a full-band one (hop 60) with one resblock kernel, and its MSD
# with 8 channels
TRAIN_G = dict(TRAIN_G_MB, out_channels=1, resblock_kernel_sizes=[3], resblock_dilations=[[1, 3]])
TRAIN_MSD = dict(TRAIN_MSD_MB, discriminator_params=dict(TRAIN_MSD_MB["discriminator_params"], channels=8,
                                                        max_downsample_channels=8, max_groups=8))
TRAIN_MRD = dict(fft_sizes=[128, 256, 64], hop_sizes=[15, 30, 8], win_lengths=[60, 120, 30],
                 discriminator_params={"channels": 4, "init_kernel": 3, "kernel_size": 11, "stride": 2})


def _layout(m):
    return [[k, list(v.shape)] for k, v in m.state_dict().items()]


def module_fixture(seed):
    gen = torch.Generator().manual_seed(seed)
    arrays, layouts = {}, {}
    for tag, case in CASES.items():
        cfg = {k: v for k, v in case.items() if k != "lengths"}
        m = MultiSpecDiscriminator(**cfg)
        layouts[tag] = _layout(m)
        fill_params(m)
        for n in case["lengths"]:
            wav = (0.2 * torch.randn(2, 1, n, generator=gen)).clamp(-1, 1)
            arrays[f"{tag}/wav_{n}"] = wav
            with torch.no_grad():
                outs, fmaps = m(wav)
            for i, (o, fm) in enumerate(zip(outs, fmaps)):
                arrays[f"{tag}/out_{n}_{i}"] = o
                for l, f in enumerate(fm):
                    arrays[f"{tag}/fmap_{n}_{i}_{l}"] = f
        outs, fmaps = m(arrays[f"{tag}/wav_{case['lengths'][-1]}"])
        total = 0.0
        for i, (o, fm) in enumerate(zip(outs, fmaps)):
            total = total + (o * probe(o.shape, 100 * i + 99)).sum()
            for l, f in enumerate(fm):
                total = total + (f * probe(f.shape, 100 * i + l)).sum()
        names = [k for k, _ in m.named_parameters()]
        grads = torch.autograd.grad(total, [p for _, p in m.named_parameters()])
        arrays.update({f"{tag}/grad/{k}": g for k, g in zip(names, grads)})
    torch.manual_seed(seed + 1)
    m = MultiSpecDiscriminator(**SPECTRAL)
    layouts["spectral"] = _layout(m)
    randomize(m, gen)
    m.train()
    arrays.update({f"spectral/sd_before/{k}": v.clone() for k, v in m.state_dict().items()})
    wav = (0.2 * torch.randn(2, 1, SPECTRAL_LENGTH, generator=gen)).clamp(-1, 1)
    arrays["spectral/wav"] = wav
    with torch.no_grad():
        m(wav)
        outs, fmaps = m(wav)
    arrays.update({f"spectral/sd_after/{k}": v.clone() for k, v in m.state_dict().items()})
    for i, (o, fm) in enumerate(zip(outs, fmaps)):
        arrays[f"spectral/out_{i}"] = o
        for l, f in enumerate(fm):
            arrays[f"spectral/fmap_{i}_{l}"] = f
    save("multispec_small", {"cases": CASES, "spectral": SPECTRAL, "layouts": layouts}, **arrays)


def trainstep_fixture(seed):
    """GAN_Trainer.train_step (trainer.py:469-589) with TRAIN_G, TRAIN_MSD, make_golden_multiband's TRAIN_MPD and
    TRAIN_MRD."""
    from kantts.train.trainer import GAN_Trainer

    torch.manual_seed(seed)
    gen = torch.Generator().manual_seed(seed + 1)
    g = Generator(**TRAIN_G)
    msd = MultiScaleDiscriminator(**TRAIN_MSD)
    mpd = MultiPeriodDiscriminator(**TRAIN_MPD)
    mrd = MultiSpecDiscriminator(**TRAIN_MRD)
    models = (("g", g), ("msd", msd), ("mpd", mpd), ("mrd", mrd))
    for _, m in models:
        randomize(m, gen)
    arrays = {}
    for tag, m in models:
        for k, v in m.state_dict().items():
            arrays[f"before/{tag}/{k}"] = v.detach().clone()
    discs = {"MultiScaleDiscriminator": msd, "MultiPeriodDiscriminator": mpd, "MultiSpecDiscriminator": mrd}
    model = {"generator": g, "discriminator": discs}
    adam = dict(lr=2e-4, betas=(0.5, 0.9), weight_decay=0.0)
    optimizer = {"generator": torch.optim.Adam(g.parameters(), **adam),
                 "discriminator": {k: torch.optim.Adam(m.parameters(), **adam) for k, m in discs.items()}}
    sched = lambda o: torch.optim.lr_scheduler.MultiStepLR(o, milestones=[200000], gamma=0.5)  # noqa: E731
    scheduler = {"generator": sched(optimizer["generator"]),
                 "discriminator": {k: sched(v) for k, v in optimizer["discriminator"].items()}}
    config = {"Loss": LOSS_CFG, "generator_train_start_steps": 1, "discriminator_train_start_steps": 0,
              "generator_grad_norm": -1, "discriminator_grad_norm": -1, "log_interval_steps": 1000,
              "train_max_steps": 10, "save_interval_steps": 10 ** 9, "eval_interval_steps": 10 ** 9}
    criterion = criterion_builder(config)
    import tempfile
    tr = GAN_Trainer(config=config, model=model, optimizer=optimizer, scheduler=scheduler,
                     criterion=criterion, device=torch.device("cpu"), sampler={"train": None, "valid": None},
                     train_loader=None, valid_loader=None, max_steps=10, save_dir=tempfile.mkdtemp(),
                     save_interval=10 ** 9, valid_interval=10 ** 9, log_interval=10 ** 9)
    tr.steps = 1
    B, Tm = 2, 32
    y = (0.1 * torch.randn(B, 1, Tm * 60, generator=gen)).clamp(-1, 1)
    x = torch.randn(B, TRAIN_G["in_channels"], Tm, generator=gen)
    tr.train_step((y, x))
    for k, v in tr.total_train_loss.items():
        arrays["loss/" + k.replace("train/", "")] = np.float64(v)
    for tag, m in models:
        for k, v in m.state_dict().items():
            arrays[f"after/{tag}/{k}"] = v.detach().clone()
    arrays["y"], arrays["x"] = y, x
    save("trainstep_multispec_small", {"generator": TRAIN_G, "msd": TRAIN_MSD, "mpd": TRAIN_MPD, "mrd": TRAIN_MRD,
                                       "loss": LOSS_CFG, "adam": {"lr": 2e-4, "betas": [0.5, 0.9]}}, **arrays)


def init_checksums():
    out = {}
    for tag, spectral in (("weight_norm", False), ("spectral_norm", True)):
        torch.manual_seed(5)
        m = MultiSpecDiscriminator(discriminator_params=dict(DEFAULTS_FIXED, use_spectral_norm=spectral))
        out[tag] = checksums(m.state_dict())
    with open(os.path.join(HERE, "multispec_init_checksums.json"), "w") as f:
        json.dump({"discriminator_params": DEFAULTS_FIXED, "checksums": out}, f)


if __name__ == "__main__":
    if sys.argv[1:] in ([], ["module"]):
        module_fixture(1250)
    if sys.argv[1:] in ([], ["trainstep"]):
        trainstep_fixture(1251)
    if sys.argv[1:] in ([], ["init"]):
        init_checksums()
