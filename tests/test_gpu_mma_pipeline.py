"""GPU parity of the tensor-core main loops at full-size shapes (``pytest -m gpu``): every CTA runs at least three tiles
of a persistent loop, the weight ring wraps around, weights are resident, the weight gradient is split over K, the
consumer paths compiled for N = 16 / 32 / 128 all run, and both fused-resblock widths (whose loops keep an MMA group in
flight while ring slots are released) run many tiles.  The layer checks are those of test_gpu_parity.py, on these
extra shapes."""
import pytest

import test_gpu_parity as P

pytestmark = pytest.mark.gpu

CONV_CASES = {
    # (spec kwargs, B, T, period, use_resid, weight_norm), as test_gpu_parity.CASES
    # N = 128, 22 (chunk, tap) steps through a 6-stage weight ring, 512 tiles (~4 per CTA), split-K weight gradient
    "many_tiles_128_k11_ring": (dict(c_in=128, c_out=128, kernel=11, dilation=3, pad_left=30, act_in=0.1), 16, 4096, 0, True, True),
    # N = 32, resident weights, 1024 tiles (~8 per CTA)
    "many_tiles_32_k7_resident": (dict(c_in=32, c_out=32, kernel=7, pad_left=6, act_in=0.1), 16, 8192, 0, True, True),
    # N = 16 (single output channel): 16 K chunks x 3 taps per tile, 512 tiles
    "many_tiles_1024_to_1_k3": (dict(c_in=1024, c_out=1, kernel=3, pad_left=1, pad_right=1), 16, 4096, 0, False, True),
}

RB_CASES = {
    # (channels, kernel, dilation, causal, B, T), as test_gpu_parity.RB_CASES: 1088 / 560 tiles
    "rb32_k7_d3_many_tiles": (32, 7, 3, True, 16, 8192),
    "rb64_k11_d5_many_tiles": (64, 11, 5, True, 8, 8192),
}


@pytest.mark.parametrize("name", sorted(CONV_CASES))
def test_conv_layer_many_tiles_vs_oracle(name, monkeypatch):
    monkeypatch.setitem(P.CASES, name, CONV_CASES[name])
    assert P._run_case(name, force_ffma=False), "expected the tensor-core path to be taken"


@pytest.mark.parametrize("name", sorted(RB_CASES))
def test_fused_resblock_many_tiles_vs_oracle(name, monkeypatch):
    monkeypatch.setitem(P.RB_CASES, name, RB_CASES[name])
    P.test_fused_resblock_unit_vs_oracle(name)
