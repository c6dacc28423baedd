"""Multi-band HiFi-GAN without a GPU: the PQMF module's buffers and state_dict against the unmodified reference, the float64
oracle PQMF against the reference's outputs, the multi-band Generator's checkpoint compatibility, and the plumbing that adds
or refuses the PQMF (model builder, criterion alias, install(), streaming, synthesize, GanStep)."""
import types

import pytest
import torch

import kantts_b200 as K
from conftest import rel_l2
from oracle import pqmf as OP


@pytest.mark.parametrize("subbands", [4, 2])
def test_pqmf_buffers_match_reference(golden, subbands):
    g = golden("multiband_small")
    ref = g.group(f"pqmf{subbands}/")
    sd = K.PQMF(subbands).state_dict()
    assert list(sd.keys()) == ["analysis_filter", "synthesis_filter", "updown_filter"]
    for k, v in sd.items():
        assert v.dtype == torch.float32 and v.shape == ref[k].shape, k
        assert torch.equal(v, ref[k]), k


@pytest.mark.parametrize("subbands", [4, 2])
def test_oracle_pqmf_matches_reference(golden, subbands):
    g = golden("multiband_small")
    ref = g.group(f"pqmf{subbands}/")
    ha, hs = OP.filters(subbands)
    assert rel_l2(ha.float(), ref["analysis_filter"]) == 0.0 and rel_l2(hs.float(), ref["synthesis_filter"]) == 0.0
    x = ref["x"].double().requires_grad_(True)
    a = OP.analysis(x, ha, subbands)
    assert a.shape == ref["analysis"].shape and rel_l2(a.detach(), ref["analysis"]) < 1e-6
    (a * ref["r_analysis"].double()).sum().backward()
    assert rel_l2(x.grad, ref["grad_x"]) < 1e-6
    xs = ref["xs"].double().requires_grad_(True)
    s = OP.synthesis(xs, hs, subbands)
    assert s.shape == ref["synthesis"].shape and rel_l2(s.detach(), ref["synthesis"]) < 1e-6
    (s * ref["r_synthesis"].double()).sum().backward()
    assert rel_l2(xs.grad, ref["grad_xs"]) < 1e-6


def test_pqmf_rejects_wrong_shapes():
    p = K.PQMF(4)
    with pytest.raises(ValueError):
        p.analysis(torch.zeros(2, 4, 64))
    with pytest.raises(ValueError):
        p.synthesis(torch.zeros(2, 2, 64))


def test_pqmf_conv_specs_give_the_reference_lengths():
    for s in (2, 3, 4, 8):
        p = K.PQMF(s)
        for t in (s * 7, s * 64 + 1, s * 100 + s - 1):
            assert p.analysis_spec.t_out(t) == t // s, (s, t)
        for n in (1, 5, 64):
            assert p.synthesis_spec.t_out(n) == s * n, (s, n)


def test_multiband_generator_loads_reference_checkpoint(golden):
    g = golden("multiband_small")
    gen = K.Generator(**g.cfg["generator"])
    ref = g.group("gen/sd/")
    assert list(gen.state_dict().keys()) == list(ref.keys())
    gen.load_state_dict(ref, strict=True)
    assert gen.conv_post.conv1d.spec.c_out == 4
    assert not any("pqmf" in k for k in gen.state_dict())


def test_multiband_nsf_generator_stays_out_of_scope():
    with pytest.raises(NotImplementedError):
        K.Generator(out_channels=4, channels=32, nsf_params={"nb_harmonics": 7, "sampling_rate": 24000})


def _small_mb_generator():
    return K.Generator(out_channels=4, channels=32, upsample_scales=[5, 3, 2, 2], upsample_kernal_sizes=[10, 6, 4, 4]).eval()


def test_streaming_rejects_multiband():
    gen = _small_mb_generator()
    with pytest.raises(ValueError, match="multi-band"):
        gen.streamer(batch=1, max_frames=4)
    with pytest.raises(ValueError, match="multi-band"):
        K.hifigan.StreamPlan(gen)
    sambert = types.SimpleNamespace(training=False)
    with pytest.raises(ValueError, match="multi-band"):
        K.stream_synthesize(sambert, gen, None, None, None, None)
    with pytest.raises(ValueError, match="multi-band"):
        K.TtsServer(sambert, gen, slots=1, chunk_steps=1, max_steps=8)


def test_synthesize_needs_the_attached_pqmf():
    with pytest.raises(ValueError, match="pqmf"):
        K.synthesize(types.SimpleNamespace(training=False), _small_mb_generator(), None, None, None, None)


def _builder_config(out_channels):
    adam = {"type": "Adam", "params": {"lr": 2e-4, "betas": [0.5, 0.9]}}
    sched = {"type": "MultiStepLR", "params": {"gamma": 0.5, "milestones": [200000]}}
    gp = dict(out_channels=out_channels, channels=32, upsample_scales=[5, 3, 2, 2], upsample_kernal_sizes=[10, 6, 4, 4])
    return {"Model": {"Generator": {"params": gp, "optimizer": adam, "scheduler": sched}}}


def test_model_builder_adds_pqmf_for_multiband_only():
    model, _, _ = K.hifigan_model_builder(_builder_config(1), "cpu")
    assert "pqmf" not in model
    model, _, _ = K.hifigan_model_builder(_builder_config(4), "cpu")
    assert isinstance(model["pqmf"], K.PQMF) and model["pqmf"].subbands == 4
    cfg = dict(_builder_config(2), pqmf={"taps": 48})
    model, _, _ = K.hifigan_model_builder(cfg, "cpu")
    assert model["pqmf"].subbands == 2 and model["pqmf"].analysis_filter.shape == (2, 1, 49)


def test_criterion_builder_aliases_the_subband_loss():
    sub = {"enable": True, "params": dict(fft_sizes=[384, 683, 171], hop_sizes=[35, 75, 15], win_lengths=[150, 300, 60])}
    crit = K.criterion_builder({"Loss": {"subband_stft_loss": sub}})
    assert crit["sub_stft"] is crit["subband_stft_loss"]
    crit = K.criterion_builder({"Loss": {"subband_stft_loss": {"enable": False}}})
    assert "sub_stft" not in crit


def test_gan_step_needs_pqmf_for_the_subband_loss():
    crit = K.criterion_builder({"Loss": {"subband_stft_loss": {"enable": True, "params": {}}}})
    with pytest.raises(ValueError, match="PQMF"):
        K.GanStep({"generator": None, "discriminator": {}}, None, None, crit, {})


def test_install_patches_both_pqmf_names():
    models = types.SimpleNamespace(pqmf=types.SimpleNamespace(PQMF=None), hifigan=None, PQMF=None)
    loss = types.SimpleNamespace(loss_dict={})
    audio = types.SimpleNamespace()
    K.install(kantts_models=models, kantts_loss=loss, kantts_audio=audio)
    assert models.PQMF is K.PQMF and models.pqmf.PQMF is K.PQMF
