"""tests/golden/multiband_small.npz and trainstep_multiband_small.npz: the multi-band HiFi-GAN of the UNMODIFIED reference
(kantts/models/pqmf.py, Generator(out_channels=4), the sub-band multi-resolution STFT loss and GAN_Trainer.train_step with a
PQMF) on CPU, imported through oracle/ref_shims.py (which supplies the removed ``scipy.signal.kaiser``).

multiband_small.npz
  pqmf{S}/...     S = 4 and 2: the three buffers, analysis / synthesis outputs of fixed inputs and the input gradients of
                  sum(out * r)
  gen/...         a small Generator(out_channels=4): state_dict, mel x, the sub-band output y_mb and its PQMF synthesis y
  stft/...        torch.stft magnitudes (the reference's audio_torch.stft) for the shipped yamls' sub-band resolutions, and
                  the sub-band MultiResolutionSTFTLoss values and input gradient of (sc + mag)
trainstep_multiband_small.npz
  one GAN_Trainer.train_step with pqmf, stft_loss and subband_stft_loss enabled, in the layout of trainstep_small.npz.  The
  reference criterion_builder leaves out the "sub_stft" key its trainer calls; it is added here as the same object.

Build container only:  python tests/golden/make_golden_multiband.py [multiband | trainstep]"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from make_golden import SMALL_MPD, SMALL_MSD, randomize, save  # noqa: E402  (imports the reference)
from kantts.models.hifigan.hifigan import Generator, MultiPeriodDiscriminator, MultiScaleDiscriminator  # noqa: E402
from kantts.models.pqmf import PQMF  # noqa: E402
from kantts.train.loss import MultiResolutionSTFTLoss, criterion_builder  # noqa: E402
from kantts.utils.audio_torch import stft  # noqa: E402

torch.set_num_threads(8)

SUB_STFT = dict(fft_sizes=[384, 683, 171], hop_sizes=[35, 75, 15], win_lengths=[150, 300, 60], window="hann_window")
SMALL_G_MB = dict(in_channels=80, out_channels=4, channels=32, kernel_size=7, upsample_scales=[5, 3, 2, 2],
                  upsample_kernal_sizes=[10, 6, 4, 4], resblock_kernel_sizes=[3, 7, 11], resblock_dilations=[[1, 3, 5]] * 3,
                  bias=True, causal=True, nonlinear_activation="LeakyReLU",
                  nonlinear_activation_params={"negative_slope": 0.1}, use_weight_norm=True)
# the train step's models, smaller than make_golden's so that the before / after parameters stay a small fixture: 20 input
# channels and two resblock kernels, depthwise grouped MSD layers (max_groups = channels), two-channel MPD stems
TRAIN_G_MB = dict(SMALL_G_MB, in_channels=20, resblock_kernel_sizes=[3, 7], resblock_dilations=[[1, 3], [1, 3]])
TRAIN_MSD = dict(SMALL_MSD, discriminator_params=dict(SMALL_MSD["discriminator_params"], channels=16,
                                                      max_downsample_channels=16, max_groups=16))
TRAIN_MPD = dict(SMALL_MPD, discriminator_params=dict(SMALL_MPD["discriminator_params"], channels=2,
                                                      max_downsample_channels=8))
LOSS_CFG_MB = {
    "generator_adv_loss": {"enable": True, "params": {"average_by_discriminators": False}, "weights": 1.0},
    "discriminator_adv_loss": {"enable": True, "params": {"average_by_discriminators": False}, "weights": 1.0},
    "stft_loss": {"enable": True, "params": {}, "weights": 1.0},
    "mel_loss": {"enable": True, "params": dict(fs=24000, fft_size=1024, hop_size=240, win_length=1024, window="hann",
                                                num_mels=80, fmin=0, fmax=8000, log_base=None),
                 "weights": 45.0},
    "subband_stft_loss": {"enable": True, "params": SUB_STFT},
    "feat_match_loss": {"enable": True, "params": {"average_by_discriminators": False, "average_by_layers": False},
                        "weights": 2.0},
}


def pqmf_arrays(subbands, gen):
    p = PQMF(subbands)
    out = {f"pqmf{subbands}/{k}": v for k, v in p.state_dict().items()}
    x = (0.3 * torch.randn(3, 1, 64 * subbands, generator=gen)).requires_grad_(True)
    a = p.analysis(x)
    ra = torch.randn(a.shape, generator=gen)
    out.update({f"pqmf{subbands}/x": x, f"pqmf{subbands}/analysis": a, f"pqmf{subbands}/r_analysis": ra,
                f"pqmf{subbands}/grad_x": torch.autograd.grad((a * ra).sum(), x)[0]})
    xs = torch.randn(3, subbands, 64, generator=gen).requires_grad_(True)
    s = p.synthesis(xs)
    rs = torch.randn(s.shape, generator=gen)
    out.update({f"pqmf{subbands}/xs": xs, f"pqmf{subbands}/synthesis": s, f"pqmf{subbands}/r_synthesis": rs,
                f"pqmf{subbands}/grad_xs": torch.autograd.grad((s * rs).sum(), xs)[0]})
    return out


def multiband_fixture(seed):
    gen = torch.Generator().manual_seed(seed)
    arrays = {}
    for s in (4, 2):
        arrays.update(pqmf_arrays(s, gen))
    torch.manual_seed(seed)
    g = Generator(**SMALL_G_MB)
    randomize(g, gen)
    g.eval()
    arrays.update({"gen/sd/" + k: v for k, v in g.state_dict().items()})
    x = torch.randn(2, 80, 6, generator=gen)
    with torch.no_grad():
        y_mb = g(x)
        y = PQMF(4).synthesis(y_mb)
    arrays.update({"gen/x": x, "gen/y_mb": y_mb, "gen/y": y})
    # sub-band signals of 4 x 480 samples (a 1920-sample waveform at 4 bands), two items
    y_sb = (0.1 * torch.randn(2, 4, 480, generator=gen)).clamp(-1, 1)
    y_hat = (y_sb + 0.05 * torch.randn(2, 4, 480, generator=gen)).requires_grad_(True)
    arrays.update({"stft/y": y_sb, "stft/y_hat": y_hat})
    for n, h, w in zip(SUB_STFT["fft_sizes"], SUB_STFT["hop_sizes"], SUB_STFT["win_lengths"]):
        arrays[f"stft/mag_{n}"] = stft(y_sb.reshape(-1, 480), n, h, w, torch.hann_window(w))
    sc, mag = MultiResolutionSTFTLoss(**SUB_STFT)(y_hat, y_sb)
    arrays.update({"stft/sc": sc, "stft/mag": mag, "stft/grad": torch.autograd.grad(sc + mag, y_hat)[0]})
    save("multiband_small", {"generator": SMALL_G_MB, "sub_stft": SUB_STFT}, **arrays)


def trainstep_fixture(seed):
    """GAN_Trainer.train_step (trainer.py:469-589) with model["pqmf"], as make_golden.trainstep_fixture, on the TRAIN_*
    models."""
    from kantts.train.trainer import GAN_Trainer

    torch.manual_seed(seed)
    gen = torch.Generator().manual_seed(seed + 1)
    g = Generator(**TRAIN_G_MB)
    msd = MultiScaleDiscriminator(**TRAIN_MSD)
    mpd = MultiPeriodDiscriminator(**TRAIN_MPD)
    for m in (g, msd, mpd):
        randomize(m, gen)
    arrays = {}
    for tag, m in (("g", g), ("msd", msd), ("mpd", mpd)):
        for k, v in m.state_dict().items():
            arrays[f"before/{tag}/{k}"] = v.detach().clone()
    model = {"generator": g, "discriminator": {"MultiScaleDiscriminator": msd, "MultiPeriodDiscriminator": mpd},
             "pqmf": PQMF(4)}
    adam = dict(lr=2e-4, betas=(0.5, 0.9), weight_decay=0.0)
    optimizer = {"generator": torch.optim.Adam(g.parameters(), **adam),
                 "discriminator": {"MultiScaleDiscriminator": torch.optim.Adam(msd.parameters(), **adam),
                                   "MultiPeriodDiscriminator": torch.optim.Adam(mpd.parameters(), **adam)}}
    sched = lambda o: torch.optim.lr_scheduler.MultiStepLR(o, milestones=[200000], gamma=0.5)  # noqa: E731
    scheduler = {"generator": sched(optimizer["generator"]),
                 "discriminator": {k: sched(v) for k, v in optimizer["discriminator"].items()}}
    config = {"Loss": LOSS_CFG_MB, "generator_train_start_steps": 1, "discriminator_train_start_steps": 0,
              "generator_grad_norm": -1, "discriminator_grad_norm": -1, "log_interval_steps": 1000,
              "train_max_steps": 10, "save_interval_steps": 10 ** 9, "eval_interval_steps": 10 ** 9}
    criterion = criterion_builder(config)
    criterion["sub_stft"] = criterion["subband_stft_loss"]
    import tempfile
    tr = GAN_Trainer(config=config, model=model, optimizer=optimizer, scheduler=scheduler,
                     criterion=criterion, device=torch.device("cpu"), sampler={"train": None, "valid": None},
                     train_loader=None, valid_loader=None, max_steps=10, save_dir=tempfile.mkdtemp(),
                     save_interval=10 ** 9, valid_interval=10 ** 9, log_interval=10 ** 9)
    tr.steps = 1
    B, Tm = 2, 8
    y = (0.1 * torch.randn(B, 1, Tm * 240, generator=gen)).clamp(-1, 1)
    x = torch.randn(B, TRAIN_G_MB["in_channels"], Tm, generator=gen)
    tr.train_step((y, x))
    for k, v in tr.total_train_loss.items():
        arrays["loss/" + k.replace("train/", "")] = np.float64(v)
    for tag, m in (("g", g), ("msd", msd), ("mpd", mpd)):
        for k, v in m.state_dict().items():
            arrays[f"after/{tag}/{k}"] = v.detach().clone()
    arrays["y"], arrays["x"] = y, x
    save("trainstep_multiband_small", {"generator": TRAIN_G_MB, "msd": TRAIN_MSD, "mpd": TRAIN_MPD,
                                       "loss": LOSS_CFG_MB, "adam": {"lr": 2e-4, "betas": [0.5, 0.9]}}, **arrays)


if __name__ == "__main__":
    if sys.argv[1:] in ([], ["multiband"]):
        multiband_fixture(1240)
    if sys.argv[1:] in ([], ["trainstep"]):
        trainstep_fixture(1241)
