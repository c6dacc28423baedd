"""CPU: the single-pass bf16 tensor-core precision (KT_PATH_BF16, hifigan.set_precision) as planned without a GPU -- every
layer of the shipped vocoder yamls that bf16x3 runs on the tensor cores has a bf16 plan, whose operand planes and weight
images are one bf16 plane per operand (half of bf16x3's two); set_precision reaches every conv of a HiFi-GAN tree, the fused
resblock pairs and the stream plan, and refuses SAM-BERT; the model builder and install() pass the precision on."""
import ctypes
import types
from dataclasses import replace

import pytest
import torch

import kantts_b200 as K
import importlib

from kantts_b200 import _lib, hifigan, ops
from kantts_b200._lib import KT_PATH_AUTO, KT_PATH_BF16, KT_PLAN_STREAM, KtResblockDesc


@pytest.fixture(scope="module")
def lib():
    return _lib.load()


_LRELU = {"nonlinear_activation": "LeakyReLU", "nonlinear_activation_params": {"negative_slope": 0.1}}
# Model.Generator.params of the shipped vocoder yamls (kantts/configs/hifigan_*.yaml; the NSF variants add only the 1x1
# source convs and the source_downs, which the non-NSF builds below share in shape)
GENERATORS = {
    "v1_16k": dict(channels=256, upsample_scales=[10, 5, 2, 2], upsample_kernal_sizes=[20, 10, 4, 4],
                   resblock_dilations=[[1, 3, 5, 7]] * 3, causal=True),
    "noncausal_v1_16k": dict(channels=256, upsample_scales=[10, 5, 2, 2], upsample_kernal_sizes=[20, 11, 4, 4],
                             resblock_dilations=[[1, 3, 5, 7]] * 3, causal=False),
    "noncausal_nsf_v1_16k": dict(channels=256, upsample_scales=[10, 5, 2, 2], upsample_kernal_sizes=[20, 11, 4, 4],
                                 resblock_dilations=[[1, 3, 5, 7]] * 3, causal=False,
                                 nsf_params={"nb_harmonics": 7, "sampling_rate": 16000}),
    "v1_24k": dict(channels=512, upsample_scales=[8, 5, 3, 2], upsample_kernal_sizes=[16, 10, 6, 4],
                   resblock_dilations=[[1, 3, 5]] * 3, causal=True),
    "v1_48k": dict(in_channels=128, channels=512, upsample_scales=[10, 5, 3, 2, 2], upsample_kernal_sizes=[20, 10, 6, 4, 4],
                   resblock_dilations=[[1, 3, 5, 7]] * 3, causal=True),
    "v1_8k": dict(channels=256, upsample_scales=[5, 5, 2, 2], upsample_kernal_sizes=[10, 10, 4, 4],
                  resblock_dilations=[[1, 3, 5, 7]] * 3, causal=True),
}
MSD = dict(scales=3, downsample_pooling="DWT", downsample_pooling_params={"kernel_size": 4, "stride": 2, "padding": 2},
           discriminator_params=dict(in_channels=1, out_channels=1, kernel_sizes=[15, 41, 5, 3], channels=128,
                                     max_downsample_channels=1024, max_groups=16, bias=True, downsample_scales=[4, 4, 4, 4, 1],
                                     **_LRELU), follow_official_norm=True)
MPD = dict(periods=[2, 3, 5, 7, 11], discriminator_params=dict(in_channels=1, out_channels=1, kernel_sizes=[5, 3], channels=32,
                                                               downsample_scales=[3, 3, 3, 3, 1], max_downsample_channels=1024,
                                                               bias=True, use_spectral_norm=False, **_LRELU))


# MultiSpecDiscriminator.params as the MRD tests build it
MRD = dict(fft_sizes=[1024, 2048, 512], hop_sizes=[120, 240, 50], win_lengths=[600, 1200, 240],
           discriminator_params=dict(channels=15, init_kernel=1, kernel_size=11, stride=2, window="hann_window", **_LRELU))


def _generator(name):
    return K.Generator(in_channels=GENERATORS[name].get("in_channels", 80), kernel_size=7, resblock_kernel_sizes=[3, 7, 11],
                       bias=True, use_weight_norm=True, **_LRELU,
                       **{k: v for k, v in GENERATORS[name].items() if k != "in_channels"})


def _specs(module):
    return [v for m in module.modules() for v in vars(m).values() if isinstance(v, ops.ConvSpec)]


def _descs(spec, nsubs):
    """The layer's descriptors at the batch of the yamls (16) over sequence lengths from a streamed chunk to a training
    segment, for every period it may run at."""
    for nsub in nsubs:
        for t in (4, 33, 256, 2048, 9600):
            if spec.t_out(t) > 0:
                yield spec.desc(16, nsub, t)


def _yaml_layers():
    out = []
    for name in GENERATORS:
        out += [(f"{name}/{i}", s, (1,)) for i, s in enumerate(_specs(_generator(name)))]
    out += [(f"msd/{i}", s, (1,)) for i, s in enumerate(_specs(K.MultiScaleDiscriminator(**MSD)))]
    mpd = K.MultiPeriodDiscriminator(**MPD)
    for d, p in zip(mpd.discriminators, MPD["periods"]):
        out += [(f"mpd{p}/{i}", s, (p,)) for i, s in enumerate(_specs(d))]
    return out


def _pf(n, planes):
    """plane_floats (tma.cuh): workspace floats of `planes` bf16 planes of n elements, 256-byte aligned."""
    return ((n * planes + 1) // 2 + 63) & ~63


def test_bf16_plans_cover_every_yaml_layer(lib):
    """Every pass of every layer that bf16x3 runs on the tensor cores has a single-pass bf16 plan of the same N tile (and a
    stream plan where bf16x3 has one); layers without one run the FFMA kernels in both."""
    n = 0
    for name, spec, nsubs in _yaml_layers():
        for d in _descs(spec, nsubs):
            b = replace(spec, path=KT_PATH_BF16).desc(d.batch, d.nsub, d.t_in)
            for direction in (0, 1, KT_PLAN_STREAM):
                nt_x3 = lib.kt_conv1d_tc_plan(ctypes.byref(d), direction)
                nt_b = lib.kt_conv1d_tc_plan(ctypes.byref(b), direction)
                assert nt_b == nt_x3, (name, spec, d.t_in, d.nsub, direction, nt_x3, nt_b)
                n += nt_b > 0
            ws_x3 = lib.kt_conv1d_bwd_weight_tc_workspace(ctypes.byref(d))
            assert (lib.kt_conv1d_bwd_weight_tc_workspace(ctypes.byref(b)) > 0) == (ws_x3 > 0), (name, spec, d.t_in)
    assert n > 1000


def _debug_ws(lib, d, direction):
    """workspace floats of the plan made as on a GPU box (kt_debug_conv_tc_plan; kt_conv1d_tc_workspace answers for this
    machine's driver, which may offer no tensor-map encoding)"""
    out = (ctypes.c_int64 * 9)()
    assert lib.kt_debug_conv_tc_plan(ctypes.byref(d), direction, out) == 0
    return int(out[8])


def test_bf16_conv_workspace_and_image_are_one_plane(lib):
    """The TMA-fed conv's gathered-operand workspace holds one bf16 plane per element (bf16x3: two), and every packed
    weight image is half the bytes of its bf16x3 twin."""
    tma = 0
    for name, spec, nsubs in _yaml_layers():
        for d in _descs(spec, nsubs):
            b = replace(spec, path=KT_PATH_BF16).desc(d.batch, d.nsub, d.t_in)
            for direction in (0, 1):
                if not lib.kt_conv1d_tc_plan(ctypes.byref(d), direction):
                    continue
                img_x3 = lib.kt_conv1d_tc_image_bytes(ctypes.byref(d), direction)
                assert img_x3 > 0 and 2 * lib.kt_conv1d_tc_image_bytes(ctypes.byref(b), direction) == img_x3, (name, spec)
                ws_x3, ws_b = (_debug_ws(lib, x, direction) for x in (d, b))
                if ws_x3:
                    rows, c = (d.t_in, d.c_in) if direction == 0 else (d.t_out, d.c_out)
                    n = d.batch * rows * d.nsub * c
                    assert ws_x3 == _pf(n, 2) and ws_b == _pf(n, 1), (name, spec, direction, ws_x3, ws_b)
                    tma += 1
    assert tma > 50


def test_bf16_resblock_image_is_half(lib):
    for c, k, dil in ((32, 3, 1), (32, 7, 5), (32, 11, 3), (64, 3, 7), (64, 7, 3), (64, 11, 5)):
        kw = dict(batch=16, t=4096, channels=c, kernel=k, dilation=dil, pad_left1=(k - 1) * dil // 2, pad_left2=(k - 1) // 2,
                  slope=0.1)
        x3, b = KtResblockDesc(path=KT_PATH_AUTO, **kw), KtResblockDesc(path=KT_PATH_BF16, **kw)
        assert lib.kt_resblock_plan(ctypes.byref(b)) == lib.kt_resblock_plan(ctypes.byref(x3)) == 1
        assert 2 * lib.kt_resblock_image_bytes(ctypes.byref(b)) == lib.kt_resblock_image_bytes(ctypes.byref(x3)) > 0


def test_set_precision_reaches_every_conv_and_back():
    g = _generator("noncausal_nsf_v1_16k")
    mods = [g, K.MultiScaleDiscriminator(**MSD), K.MultiPeriodDiscriminator(**MPD), K.MultiSpecDiscriminator(**MRD), K.PQMF()]
    for m in mods:
        before = [s.path for s in _specs(m)]
        assert before and set(before) <= {KT_PATH_AUTO, _lib.KT_PATH_FFMA}
        assert K.set_precision(m, "bf16") is m
        assert [s.path for s in _specs(m)] == [KT_PATH_BF16 if p == KT_PATH_AUTO else p for p in before]
        K.set_precision(m, "bf16x3")
        assert [s.path for s in _specs(m)] == before
    pq = K.PQMF()
    K.set_precision(pq, "bf16")
    assert pq.analysis_spec.path == pq.synthesis_spec.path == KT_PATH_BF16
    with pytest.raises(ValueError):
        K.set_precision(g, "fp16")


def test_set_precision_reaches_resblock_pairs_and_stream_plan(lib):
    g = K.set_precision(_generator("noncausal_v1_16k").eval(), "bf16")
    rb = next(b for b in g.conv_blocks if b.convs1[0].conv1d.spec.c_in in (32, 64))
    for c1, c2 in zip(rb.convs1, rb.convs2):
        rd = ops.resblock_desc(c1.conv1d.spec, c2.conv1d.spec, 4, 2000)
        assert rd is not None and rd.path == KT_PATH_BF16
    plan = hifigan.StreamPlan(g)
    convs = [st for st in plan.steps if type(st) is hifigan.ConvStep]
    assert convs and all(st.spec.path == KT_PATH_BF16 for st in convs)
    for st in convs:
        d = st.spec.desc(8, 1, 16 * st.spec.stride if not st.spec.transposed else 16)
        if lib.kt_conv1d_tc_plan(ctypes.byref(d), KT_PLAN_STREAM):
            assert lib.kt_conv1d_tc_image_bytes(ctypes.byref(d), 0) > 0
    K.set_precision(g, "bf16x3")
    rd = ops.resblock_desc(rb.convs1[0].conv1d.spec, rb.convs2[0].conv1d.spec, 4, 2000)
    assert rd.path == KT_PATH_AUTO
    assert all(st.spec.path == KT_PATH_AUTO for st in hifigan.StreamPlan(g).steps if type(st) is hifigan.ConvStep)


def test_set_precision_refuses_sambert_and_speaker_models():
    se = K.DTDNN()
    with pytest.raises(ValueError, match="DTDNN"):
        K.set_precision(se, "bf16")
    wrapper = torch.nn.ModuleDict({"vocoder": K.PQMF(), "se": se})
    with pytest.raises(ValueError):
        K.set_precision(wrapper, "bf16")
    assert all(s.path == KT_PATH_AUTO for s in _specs(wrapper["vocoder"]))   # refused before any change


def _config(out_channels=1):
    opt = {"type": "Adam", "params": {"lr": 2e-4, "betas": [0.5, 0.9]}}
    sch = {"type": "MultiStepLR", "params": {"gamma": 0.5, "milestones": [200000]}}
    gen = dict(GENERATORS["v1_8k"], channels=32, out_channels=out_channels)
    return {"Model": {"Generator": {"params": gen, "optimizer": opt, "scheduler": sch},
                      "MultiScaleDiscriminator": {"params": MSD, "optimizer": opt, "scheduler": sch},
                      "MultiPeriodDiscriminator": {"params": MPD, "optimizer": opt, "scheduler": sch}}}


def test_builder_passes_precision_on():
    model, _, _ = K.hifigan_model_builder(_config(4), "cpu", precision="bf16")
    mods = [model["generator"], model["pqmf"], *model["discriminator"].values()]
    assert all(KT_PATH_AUTO not in {s.path for s in _specs(m)} and KT_PATH_BF16 in {s.path for s in _specs(m)} for m in mods)
    model, _, _ = K.hifigan_model_builder(_config(), "cpu")
    assert all(s.path != KT_PATH_BF16 for m in [model["generator"], *model["discriminator"].values()] for s in _specs(m))


install = importlib.import_module("kantts_b200.install")


def _fake_kantts():
    models = types.SimpleNamespace()
    return models, types.SimpleNamespace(loss_dict={}), types.SimpleNamespace()


def test_install_passes_precision_on():
    models, loss, audio = _fake_kantts()
    install.install(models, loss, audio, precision="bf16")
    for name in ("Generator", "MultiPeriodDiscriminator", "MultiScaleDiscriminator", "MultiSpecDiscriminator", "PQMF"):
        cls = getattr(models, name)
        assert cls.__name__ == name and issubclass(cls, getattr(K, name))
    g = models.Generator(channels=32, upsample_scales=[5, 5, 2, 2], upsample_kernal_sizes=[10, 10, 4, 4])
    assert {s.path for s in _specs(g)} >= {KT_PATH_BF16} and KT_PATH_AUTO not in {s.path for s in _specs(g)}
    assert {s.path for s in _specs(models.PQMF())} == {KT_PATH_BF16}
    # precision not given: the classes themselves, the default precision
    models, loss, audio = _fake_kantts()
    install.install(models, loss, audio)
    assert models.Generator is K.Generator and models.PQMF is K.PQMF
    with pytest.raises(ValueError):
        install.install(*_fake_kantts(), precision="fp8")
