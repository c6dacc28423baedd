"""Checkpoint format round trip (SURVEY.md 8f-4; kantts/train/trainer.py:591-674): a checkpoint written in the trainer's layout
from the native modules loads -- strict -- into fresh native modules; a checkpoint written by the unmodified reference classes
(stored under tests/golden) loads into the native modules, and a native checkpoint has the reference's layout; optimizer /
scheduler states of the reference's `torch.optim.Adam` / `MultiStepLR` restore onto the native parameters (same order)."""
import os

import torch

import kantts_b200 as K

G_CFG = dict(in_channels=80, out_channels=1, channels=32, kernel_size=7, upsample_scales=[4, 2], upsample_kernal_sizes=[8, 4],
             resblock_kernel_sizes=[3, 7], resblock_dilations=[[1, 3], [1, 3]], causal=True)
MSD_CFG = dict(scales=3, downsample_pooling="DWT", downsample_pooling_params={"kernel_size": 4, "stride": 2, "padding": 2},
               discriminator_params=dict(in_channels=1, out_channels=1, kernel_sizes=[15, 41, 5, 3], channels=16,
                                         max_downsample_channels=64, max_groups=4, bias=True, downsample_scales=[4, 4, 4, 4, 1],
                                         nonlinear_activation="LeakyReLU", nonlinear_activation_params={"negative_slope": 0.1}),
               follow_official_norm=True)
MPD_CFG = dict(periods=[2, 3], discriminator_params=dict(in_channels=1, out_channels=1, kernel_sizes=[5, 3], channels=8,
                                                         downsample_scales=[3, 3, 3, 3, 1], max_downsample_channels=64, bias=True,
                                                         nonlinear_activation="LeakyReLU",
                                                         nonlinear_activation_params={"negative_slope": 0.1}, use_spectral_norm=False))


# smaller still for the stored reference checkpoint (tests/golden/checkpoint_reference.pth, kept under 1 MB)
TINY = (dict(G_CFG, channels=8, resblock_kernel_sizes=[3], resblock_dilations=[[1, 3]]),
        dict(MSD_CFG, discriminator_params=dict(MSD_CFG["discriminator_params"], channels=4, max_downsample_channels=16)),
        dict(MPD_CFG, discriminator_params=dict(MPD_CFG["discriminator_params"], channels=2, max_downsample_channels=16)))


def _build(mod, cfgs=(G_CFG, MSD_CFG, MPD_CFG)):
    torch.manual_seed(3)
    g_cfg, msd_cfg, mpd_cfg = cfgs
    model = {"generator": mod.Generator(**g_cfg),
             "discriminator": {"MultiScaleDiscriminator": mod.MultiScaleDiscriminator(**msd_cfg),
                               "MultiPeriodDiscriminator": mod.MultiPeriodDiscriminator(**mpd_cfg)}}
    mk = lambda m: torch.optim.Adam(m.parameters(), lr=2e-4, betas=(0.5, 0.9))
    opt = {"generator": mk(model["generator"]), "discriminator": {k: mk(m) for k, m in model["discriminator"].items()}}
    sch = {"generator": torch.optim.lr_scheduler.MultiStepLR(opt["generator"], milestones=[10], gamma=0.5),
           "discriminator": {k: torch.optim.lr_scheduler.MultiStepLR(o, milestones=[10], gamma=0.5) for k, o in opt["discriminator"].items()}}
    return model, opt, sch


def _save(model, opt, sch, steps, path):      # GAN_Trainer.save_checkpoint, trainer.py:591-632
    sd = {"optimizer": {"generator": opt["generator"].state_dict(), "discriminator": {k: o.state_dict() for k, o in opt["discriminator"].items()}},
          "scheduler": {"generator": sch["generator"].state_dict(), "discriminator": {k: o.state_dict() for k, o in sch["discriminator"].items()}},
          "steps": steps,
          "model": {"generator": model["generator"].state_dict(),
                    "discriminator": {k: m.state_dict() for k, m in model["discriminator"].items()}}}
    torch.save(sd, path)


def _load(model, opt, sch, path):             # GAN_Trainer.load_checkpoint(restore_training_state=True, strict=True), :634-674
    sd = torch.load(path, map_location="cpu")
    model["generator"].load_state_dict(sd["model"]["generator"], strict=True)
    for k in sd["model"]["discriminator"]:
        model["discriminator"][k].load_state_dict(sd["model"]["discriminator"][k], strict=True)
    opt["generator"].load_state_dict(sd["optimizer"]["generator"])
    for k in sd["optimizer"]["discriminator"]:
        opt["discriminator"][k].load_state_dict(sd["optimizer"]["discriminator"][k])
    for k in sd["scheduler"]["discriminator"]:
        sch["discriminator"][k].load_state_dict(sd["scheduler"]["discriminator"][k])
    sch["generator"].load_state_dict(sd["scheduler"]["generator"])
    return sd["steps"]


def _fake_train(model, opt):
    """give the optimizers a state without any GPU: one Adam step on synthetic gradients"""
    g = torch.Generator().manual_seed(5)
    for m, o in [(model["generator"], opt["generator"])] + [(model["discriminator"][k], opt["discriminator"][k]) for k in model["discriminator"]]:
        for p in m.parameters():
            p.grad = 1e-2 * torch.randn(p.shape, generator=g)
        o.step()


def _same(a, b):
    assert list(a.keys()) == list(b.keys())
    for k in a:
        assert a[k].shape == b[k].shape and torch.equal(a[k], b[k]), k


def test_native_checkpoint_round_trip(tmp_path):
    model, opt, sch = _build(K)
    _fake_train(model, opt)
    path = os.path.join(tmp_path, "ckpt", "checkpoint_7.pth")
    os.makedirs(os.path.dirname(path))
    _save(model, opt, sch, 7, path)
    m2, o2, s2 = _build(K)
    assert _load(m2, o2, s2, path) == 7
    _same(model["generator"].state_dict(), m2["generator"].state_dict())
    for k in model["discriminator"]:
        _same(model["discriminator"][k].state_dict(), m2["discriminator"][k].state_dict())
    a, b = opt["generator"].state_dict()["state"], o2["generator"].state_dict()["state"]
    assert a.keys() == b.keys() and all(torch.equal(a[i]["exp_avg"], b[i]["exp_avg"]) for i in a)


def _layout(sd):
    return [(k, tuple(v.shape)) for k, v in sd.items()]


def test_checkpoints_interchange_with_the_reference_classes(tmp_path):
    """tests/golden/checkpoint_reference.pth was written by the unmodified reference classes (make_golden_checkpoint.py): it
    loads strict into native modules / optimizers / schedulers, and a native checkpoint has exactly its layout."""
    ref = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "checkpoint_reference.pth")
    rsd = torch.load(ref, map_location="cpu")
    m3, o3, s3 = _build(K, TINY)
    assert _load(m3, o3, s3, ref) == 4            # reference checkpoint -> native trainer objects, strict
    _same(rsd["model"]["generator"], m3["generator"].state_dict())
    for k in m3["discriminator"]:
        _same(rsd["model"]["discriminator"][k], m3["discriminator"][k].state_dict())
    a, b = rsd["optimizer"]["generator"]["state"], o3["generator"].state_dict()["state"]
    assert a.keys() == b.keys() and all(torch.equal(a[i]["exp_avg_sq"], b[i]["exp_avg_sq"]) for i in a)
    model, opt, sch = _build(K, TINY)             # and the other way: a native checkpoint in the reference's layout
    _fake_train(model, opt)
    p1 = os.path.join(tmp_path, "native.pth")
    _save(model, opt, sch, 3, p1)
    nsd = torch.load(p1, map_location="cpu")
    assert _layout(nsd["model"]["generator"]) == _layout(rsd["model"]["generator"])
    for k in rsd["model"]["discriminator"]:
        assert _layout(nsd["model"]["discriminator"][k]) == _layout(rsd["model"]["discriminator"][k]), k
    for n, r in [(nsd["optimizer"]["generator"], rsd["optimizer"]["generator"])] + \
            [(nsd["optimizer"]["discriminator"][k], rsd["optimizer"]["discriminator"][k]) for k in rsd["optimizer"]["discriminator"]]:
        assert [g["params"] for g in n["param_groups"]] == [g["params"] for g in r["param_groups"]]
        assert all(n["state"][i]["exp_avg"].shape == r["state"][i]["exp_avg"].shape for i in r["state"])
    assert nsd["scheduler"]["generator"].keys() == rsd["scheduler"]["generator"].keys()
