"""CPU-side checks of the drop-in boundary: the C-ABI library builds / loads and exports every
symbol include/kantts_b200.h declares; the nn.Modules keep the reference's state_dict contract and
construction-time RNG stream; the product has no CPU fallback."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

import kantts_b200 as K
from kantts_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    _lib.build_library()
    return _lib.load()


def test_library_exports_every_declared_symbol(lib):
    header = open(os.path.join(ROOT, "include", "kantts_b200.h")).read()
    declared = set(re.findall(r"^(?:int|int64_t|const char\*)\s+(kt_\w+)\s*\(", header, flags=re.M))
    assert len(declared) >= 15
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in kantts_b200.h but not exported"
    assert declared == set(_lib.PROTOTYPES) | {"kt_last_error"}
    assert lib.kt_version() >= 2


_CTYPES = {"int32_t": ctypes.c_int32, "int64_t": ctypes.c_int64, "float": ctypes.c_float}
_RESTYPES = {"int": ctypes.c_int, "int64_t": ctypes.c_int64, "const char*": ctypes.c_char_p}


def _accepted_argtypes(param):
    """The ctypes types that pass one C parameter ("const KtConv1dDesc* d") unchanged."""
    param = " ".join(param.replace("*", "* ").split())
    if "*" not in param:
        return (_CTYPES[param.rsplit(" ", 1)[0]],)
    struct = re.match(r"const (Kt\w+)\*", param)
    if struct:
        return ctypes.POINTER(getattr(_lib, struct.group(1))), ctypes.c_void_p
    return (ctypes.c_void_p,)


def test_every_prototype_matches_header(lib):
    """Each entry point's argtypes (PROTOTYPES) and the restype load() sets agree with its declaration in the header, argument
    by argument: a wrong ctypes type would not raise, it would pass corrupted arguments."""
    header = open(os.path.join(ROOT, "include", "kantts_b200.h")).read()
    decls = re.findall(r"^(int|int64_t|const char\*)\s+(kt_\w+)\s*\(([^)]*)\);", header, flags=re.M)
    assert sorted(name for _, name, _ in decls) == sorted(set(_lib.PROTOTYPES) | {"kt_last_error"})
    for ret, name, params in decls:
        params = [] if params.strip() == "void" else params.split(",")
        fn = getattr(lib, name)
        assert len(fn.argtypes) == len(params), name
        for i, (param, argtype) in enumerate(zip(params, fn.argtypes)):
            assert argtype in _accepted_argtypes(param), (name, i, param, argtype)
        assert fn.restype is _RESTYPES[ret], (name, ret, fn.restype)


def test_descriptor_struct_sizes_match_header():
    assert ctypes.sizeof(_lib.KtConv1dDesc) == 18 * 4
    assert ctypes.sizeof(_lib.KtMelDesc) == 14 * 4


def test_state_dict_contract_matches_golden(golden):
    for name, cls in (("gen_small_causal", K.Generator), ("gen_small_noncausal", K.Generator),
                      ("mpd_small", K.MultiPeriodDiscriminator), ("msd_small", K.MultiScaleDiscriminator)):
        g = golden(name)
        m = cls(**g.cfg)
        ref_sd = g.group("sd/")
        sd = m.state_dict()
        assert list(sd.keys()) == list(ref_sd.keys()), name
        for k in sd:
            assert sd[k].shape == ref_sd[k].shape, (name, k)
        m.load_state_dict(ref_sd, strict=True)


def test_construction_reproduces_reference_rng_stream(golden):
    """Generator() under torch.manual_seed(1234) must equal the reference's init bit for bit
    (checksums from the unmodified reference, tests/golden/c1_generator.npz)."""
    g = golden("c1_generator")
    torch.manual_seed(1234)
    m = K.Generator()
    sd = m.state_dict()
    assert set(sd.keys()) == set(g.cfg["checksums"].keys())
    for k, (s, a) in g.cfg["checksums"].items():
        assert abs(float(sd[k].double().sum()) - s) <= 1e-9 * max(1.0, abs(a)), k
        assert abs(float(sd[k].double().abs().sum()) - a) <= 1e-9 * max(1.0, abs(a)), k


def test_init_matches_reference_when_available():
    """Seeded discriminator init == the reference's: same state_dict layout (keys in order, shapes) and float64 checksums
    of the values as the reference classes (tests/golden/disc_init_checksums.json, make_golden_disc_init.py)."""
    import json
    import os
    from golden.make_golden_disc_init import CASES, checksums
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "disc_init_checksums.json")) as f:
        ref = json.load(f)
    for name, kw in CASES:
        torch.manual_seed(5)
        layout, s, a = checksums(getattr(K, name)(**kw).state_dict())
        assert layout == ref[name][0], name
        assert abs(s - ref[name][1]) <= 1e-9 * max(1.0, abs(ref[name][2])) * 100, name
        assert abs(a - ref[name][2]) <= 1e-9 * max(1.0, abs(ref[name][2])), name


def test_no_cpu_fallback(lib):
    m = K.Generator(channels=32)
    with pytest.raises(RuntimeError):
        m(torch.randn(1, 80, 4))
    mel = K.MelSpectrogram()
    with pytest.raises(RuntimeError):
        mel(torch.randn(1, 2048))


def test_mel_filterbank_matches_golden_melmat(golden):
    g = golden("mel_stft")
    for tag, kw in (("default", {}), ("yaml24k", dict(fs=24000, fft_size=1024, hop_size=240, win_length=1024, fmin=0, fmax=8000)),
                    ("c2", dict(fs=22050, fft_size=1024, hop_size=256, win_length=1024, fmin=0, fmax=8000))):
        m = K.MelSpectrogram(**kw)
        assert float((m.melmat - g.t(f"melmat_{tag}")).abs().max()) < 1e-7


def test_criterion_builder_contract():
    cfg = {"Loss": {"generator_adv_loss": {"enable": True, "params": {"average_by_discriminators": False}, "weights": 1.0},
                    "mel_loss": {"enable": True, "params": {"fs": 22050, "fmin": 0, "fmax": 8000, "log_base": None}, "weights": 45.0},
                    "stft_loss": {"enable": False}}}
    crit = K.criterion_builder(cfg)
    assert set(crit) == {"generator_adv_loss", "mel_loss"} and crit["mel_loss"].weights == 45.0
    with pytest.raises(NotImplementedError):
        K.criterion_builder({"Loss": {"nope": {"enable": True}}})


def test_conv_spec_output_lengths():
    from kantts_b200.ops import ConvSpec
    assert ConvSpec(1, 1, 7, pad_left=6).t_out(100) == 100                                  # causal
    assert ConvSpec(1, 1, 16, stride=8, transposed=True, crop=8).t_out(32) == 256          # causal deconv
    assert ConvSpec(1, 1, 11, stride=5, pad_left=3, transposed=True).t_out(7) == 35        # odd non-causal deconv
    assert ConvSpec(1, 1, 5, stride=3, pad_left=2, pad_right=2).t_out(4096) == 1366        # MPD (hifigan.py:229)
    assert ConvSpec(1, 1, 41, stride=4, pad_left=20, pad_right=20).t_out(8192) == 2048     # MSD
    assert ConvSpec(1, 1, 7, pad_left=6, upsample=8).t_out(32) == 256                      # repeat-upsample conv
