"""CPU: the alignment prior of the MAS data path.  The float64 oracle against the unmodified reference's
beta_binomial_prior_distribution (tests/golden/attn_prior.npz) pair by pair and as a padded collate batch, the C ABI
declaration of kt_attn_prior, the install() patch of the dataset module and the refusal of CPU tensors."""
import math
import os
import sys
import types

import numpy as np
import pytest
import torch

import kantts_b200 as K
from kantts_b200 import _lib
from oracle import attn_prior as oap

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _rtol(P, M):
    """1e-12, or 2e-15 ln Gamma(P + M + 1) where the lgamma terms the formula sums are larger: each is rounded to float64,
    so both evaluations carry an error of a few units in the last place of the largest term.  (At P = 121, M = 600 the
    reference's own scipy evaluation is 1.9e-12 off the exact rational value, the lgamma sum 9.1e-13.)"""
    return max(1e-12, 2e-15 * math.lgamma(P + M + 1))


def test_oracle_matches_reference_pairs(golden):
    g = golden("attn_prior")
    for P, M in g.cfg["pairs"]:
        want = g.t(f"pair/{P}_{M}")
        got = oap.beta_binomial_prior_distribution(P, M)
        assert got.dtype == torch.float64 and got.shape == want.shape == (M, P)
        big = want > 1e-300
        rel = ((got - want).abs()[big] / want[big]).max()
        assert rel <= _rtol(P, M), (P, M, float(rel))


def test_oracle_batch_matches_reference_collate(golden):
    g = golden("attn_prior")
    want = g.t("batch/attn_priors")
    il, ol = g.t("batch/valid_input_lengths"), g.t("batch/valid_output_lengths")
    B, T, L = want.shape
    assert T % g.cfg["outputs_per_step"] == 0 and L == int(il.max()) + 1
    got = oap.attn_priors(il, ol, T, L)
    assert got.dtype == torch.float64 and got.shape == want.shape
    got32 = got.float().numpy()
    ref = want.numpy()
    assert np.all(np.abs(got32 - ref) <= np.spacing(np.abs(ref)))            # within one float32 ulp
    for b in range(B):
        n, m = int(il[b]) + 1, int(ol[b])
        assert not ref[b, m:].any() and not ref[b, :, n:].any()
        assert not got32[b, m:].any() and not got32[b, :, n:].any()


def test_kt_attn_prior_is_declared():
    header = open(os.path.join(ROOT, "include", "kantts_b200.h")).read()
    assert "int kt_attn_prior(const int64_t* valid_input_lengths, const int64_t* valid_output_lengths, float* prior," in header
    assert "kt_attn_prior" in _lib.PROTOTYPES


def _stub_dataset():
    def beta_binomial_prior_distribution(phoneme_count, mel_count, scaling=1.0):
        raise AssertionError("the reference prior should not run")
    return types.SimpleNamespace(beta_binomial_prior_distribution=beta_binomial_prior_distribution)


def _install(**kw):
    K.install(kantts_models=type("M", (), {})(), kantts_loss=type("L", (), {"loss_dict": {}})(),
              kantts_audio=type("A", (), {})(), **kw)


def test_install_replaces_the_dataset_prior_with_a_nan_placeholder():
    ds = _stub_dataset()
    _install(kantts_dataset=ds)
    assert ds.beta_binomial_prior_distribution is K.data.attn_prior_placeholder
    p = ds.beta_binomial_prior_distribution(17, 230)
    assert p.shape == (230, 17) and p.stride() == (0, 0) and p.dtype == torch.float32
    assert torch.isnan(p).all()
    pad = torch.zeros(1, 231, 20)
    pad[0, : p.shape[0], : p.shape[1]] = p                                   # the collate's copy into its pad
    assert torch.isnan(pad[0, :230, :17]).all() and not pad[0, 230:].any() and not pad[0, :, 17:].any()


def test_install_without_the_argument_leaves_the_dataset_alone(monkeypatch):
    ds = _stub_dataset()
    before = ds.beta_binomial_prior_distribution
    monkeypatch.setitem(sys.modules, "kantts.datasets.dataset", ds)         # already imported
    _install()
    assert ds.beta_binomial_prior_distribution is before


def test_attn_priors_refuses_cpu_tensors():
    batch = dict(valid_input_lengths=torch.tensor([4, 2]), valid_output_lengths=torch.tensor([9, 5]),
                 mel_targets=torch.zeros(2, 9, 80), input_lings=torch.zeros(2, 5, 4, dtype=torch.long))
    with pytest.raises(RuntimeError, match="CUDA"):
        K.AttnPriors()(batch)
