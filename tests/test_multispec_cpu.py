"""MultiSpecDiscriminator on the CPU: the reference's state_dict contract and seeded init, its constructor errors, the
feature-map shapes from a pure-Python frames / width calculator, the column layout the column kernels implement (a float64 restatement
checked against the reference's padded maps), and the name lookups of install() and hifigan_model_builder."""
import json
import os
import types

import pytest
import torch

import kantts_b200 as K

HERE = os.path.dirname(os.path.abspath(__file__))


def probe(shape, salt):
    """Fixed, non-trivial values computed from a shape and a salt: the golden's parameters (fill_params) and the weights of
    the scalar whose parameter gradients it stores (make_golden_multispec.py), so neither is stored."""
    n = 1
    for d in shape:
        n *= d
    return torch.sin(torch.arange(n, dtype=torch.float64) * 0.61803 + salt).float().reshape(shape)


def fill_params(module):
    """Give every parameter of a (reference or native) MultiSpecDiscriminator the golden's fixed values, in named_parameters
    order (the same in both): biases +-0.05, weight_g in [0.8, 1.2], weights of the conv's fan-in scale."""
    with torch.no_grad():
        for j, (k, p) in enumerate(module.named_parameters()):
            r = probe(p.shape, 7 * j + 1)
            if k.endswith("bias"):
                p.copy_(0.05 * r)
            elif k.endswith("weight_g"):
                p.copy_(1.0 + 0.2 * r)
            else:
                p.copy_(r * (0.5 / p[0].numel() ** 0.5))


def case_cfg(case):
    """A golden case's MultiSpecDiscriminator kwargs (without its waveform lengths)."""
    return {k: v for k, v in case.items() if k != "lengths"}


def test_state_dict_keys_order_and_shapes_match_the_reference(golden):
    g = golden("multispec_small")
    cfgs = {tag: case_cfg(case) for tag, case in g.cfg["cases"].items()}
    cfgs["spectral"] = g.cfg["spectral"]
    for tag, cfg in cfgs.items():
        sd = K.MultiSpecDiscriminator(**cfg).state_dict()
        assert [[k, list(v.shape)] for k, v in sd.items()] == g.cfg["layouts"][tag], tag
    K.MultiSpecDiscriminator(**g.cfg["spectral"]).load_state_dict(g.group("spectral/sd_before/"), strict=True)
    keys = list(K.MultiSpecDiscriminator(**cfgs["defaults"]).state_dict())
    assert keys[:4] == ["discriminators.0.window", "discriminators.0.convs.0.0.bias", "discriminators.0.convs.0.0.weight_g",
                        "discriminators.0.convs.0.0.weight_v"]
    assert "discriminators.0.conv_post.weight_g" in keys
    spectral = list(K.MultiSpecDiscriminator(**cfgs["spectral"]).state_dict())
    assert "discriminators.1.conv_post.weight_orig" in spectral and "discriminators.1.conv_post.weight_u" in spectral


def test_seeded_init_matches_the_reference_checksums():
    from golden.make_golden_disc_init import checksums
    with open(os.path.join(HERE, "golden", "multispec_init_checksums.json")) as f:
        ref = json.load(f)
    for tag, spectral in (("weight_norm", False), ("spectral_norm", True)):
        torch.manual_seed(5)
        m = K.MultiSpecDiscriminator(discriminator_params=dict(ref["discriminator_params"], use_spectral_norm=spectral))
        layout, s, a = checksums(m.state_dict())
        want = ref["checksums"][tag]
        assert layout == want[0], tag
        assert abs(s - want[1]) <= 1e-7 * max(1.0, abs(want[2])), tag
        assert abs(a - want[2]) <= 1e-9 * max(1.0, abs(want[2])), tag


def test_reference_defaults_raise_type_error():
    with pytest.raises(TypeError, match="kernel_sizes"):
        K.MultiSpecDiscriminator()


def test_non_leaky_relu_activation_is_not_implemented():
    with pytest.raises(NotImplementedError):
        K.SpecDiscriminator(channels=4, nonlinear_activation="ReLU", nonlinear_activation_params={})


def layer_shapes(frames, init_kernel=15, kernel_size=11, stride=2):
    """-> [(frames, width)] of a SpecDiscriminator's six feature maps for a magnitude of ``frames`` frames: every conv pads
    frames and width by (k-1)//2 (an int padding), conv_post pads frames only."""
    shapes, width = [], 1
    for k, s, pads_width in [(init_kernel, 1, True)] + [(kernel_size, stride, True)] * 3 + [(5, 1, True), (3, 1, False)]:
        p = (k - 1) // 2
        frames = (frames + 2 * p - k) // s + 1
        width += 2 * p if pads_width else 0
        shapes.append((frames, width))
    return shapes


def test_shape_calculator_agrees_with_the_reference(golden):
    g = golden("multispec_small")
    for tag, cfg in g.cfg["cases"].items():
        p = cfg["discriminator_params"]
        for n in cfg["lengths"]:
            for i, hop in enumerate(cfg["hop_sizes"]):
                want = layer_shapes(n // hop + 1, p.get("init_kernel", 15), p.get("kernel_size", 11), p.get("stride", 2))
                for l, (frames, width) in enumerate(want):
                    f = g.arrays[f"{tag}/fmap_{n}_{i}_{l}"]
                    assert f.shape[0] == 2 and f.shape[2:] == (frames, width), (tag, n, i, l, f.shape, frames, width)
                assert g.arrays[f"{tag}/out_{n}_{i}"].shape == g.arrays[f"{tag}/fmap_{n}_{i}_5"].shape
    assert layer_shapes(9600 // 120 + 1, 1, 11)[-1][1] == 35 and [w for _, w in layer_shapes(81)] == [15, 25, 35, 45, 49, 49]


def expand_columns(rows, batch, reach):
    """float64 restatement of kt_spec_columns_fwd: (batch + classes, T, C) rows -> (batch, T, width, C)."""
    width = 2 * reach[-1] + 1 if reach else 1
    centre = width // 2
    out = rows.new_empty(batch, rows.shape[1], width, rows.shape[2])
    for w in range(width):
        d = abs(w - centre)
        if d == 0:
            out[:, :, w] = rows[:batch]
        else:
            k = next(i for i, r in enumerate(reach) if r >= d)
            out[:, :, w] = rows[batch + k]
    return out


def test_column_classes_reproduce_the_reference_maps(golden):
    """The layout the kernels implement holds in the reference's own maps: every column of a class is the same sequence for
    both items, and expanding the centre and one column per class gives the whole map back."""
    g = golden("multispec_small")
    for tag, cfg in g.cfg["cases"].items():
        p = cfg["discriminator_params"]
        pads = [(p.get("init_kernel", 15) - 1) // 2] + [(p.get("kernel_size", 11) - 1) // 2] * 3 + [2, 0]
        for i in range(len(cfg["hop_sizes"])):
            reach = []
            for l, pad in enumerate(pads):
                if pad:
                    reach.append((reach[-1] if reach else 0) + pad)
                n = cfg["lengths"][-1]
                f = torch.from_numpy(g.arrays[f"{tag}/fmap_{n}_{i}_{l}"]).double().permute(0, 2, 3, 1)   # (B, T, W, C)
                centre = f.shape[2] // 2
                rows = torch.cat([f[:, :, centre]] + [f[:1, :, centre + r] for r in reach])
                assert torch.equal(expand_columns(rows, 2, reach), f), (tag, i, l)


def test_install_patches_both_names():
    models = types.SimpleNamespace(hifigan=types.SimpleNamespace(hifigan=types.SimpleNamespace()))
    K.install(kantts_models=models, kantts_loss=types.SimpleNamespace(loss_dict={}), kantts_audio=types.SimpleNamespace())
    for name in ("SpecDiscriminator", "MultiSpecDiscriminator"):
        assert getattr(models, name) is getattr(K, name) and getattr(models.hifigan.hifigan, name) is getattr(K, name)


def test_model_builder_finds_the_discriminator_by_name(golden):
    g = golden("multispec_small")
    opt = {"type": "Adam", "params": {"lr": 2e-4}}
    sch = {"type": "MultiStepLR", "params": {"milestones": [10]}}
    cfg = {"Model": {"Generator": {"params": dict(channels=16, upsample_scales=[4, 4], upsample_kernal_sizes=[8, 8],
                                                  resblock_kernel_sizes=[3], resblock_dilations=[[1]]),
                                   "optimizer": opt, "scheduler": sch},
                     "MultiSpecDiscriminator": {"params": case_cfg(g.cfg["cases"]["defaults"]), "optimizer": opt, "scheduler": sch}}}
    model, optimizer, _ = K.hifigan_model_builder(cfg, "cpu")
    mrd = model["discriminator"]["MultiSpecDiscriminator"]
    assert isinstance(mrd, K.MultiSpecDiscriminator) and len(mrd.discriminators) == 3
    assert hasattr(mrd, "forward_pair")
    assert optimizer["discriminator"]["MultiSpecDiscriminator"].param_groups[0]["params"][0] is next(mrd.parameters())
