"""CPU: which tensor-core conv launches take the shared-memory staged epilogue (kt_debug_conv_tc_epilogue, decided without a
GPU as it would be on one), and that the staging blocks fit next to the operand rings."""
import ctypes

import pytest

from kantts_b200 import _lib
from test_conv_tc_plan_cpu import C2, C4, _desc, _plan, _shape_desc

SMEM_MAX = 227 * 1024


@pytest.fixture(scope="module")
def lib():
    return _lib.load()


def _staged(lib, d, direction):
    return lib.kt_debug_conv_tc_epilogue(ctypes.byref(d), direction)


@pytest.mark.parametrize("shape", C2 + C4)
def test_epilogue_rule_over_the_model_layers(lib, shape):
    d = _shape_desc(shape)
    cin, cout, groups = shape[0], shape[1], shape[5]
    for direction in (0, 1):
        p = _plan(lib, d, direction)
        produced = cout if direction == 0 else cin
        staged = _staged(lib, d, direction)
        if p["nt"] == 0 or produced % 4 != 0:
            assert staged == 0, (shape, direction)
        elif groups == 1:
            assert staged == 1, (shape, direction)   # dense layers with aligned channel counts
        if p["nt"]:
            assert p["smem"] <= SMEM_MAX and p["na"] >= 2 and p["nb"] >= 2, (shape, direction, p)
    assert _staged(lib, d, _lib.KT_PLAN_STREAM) == 0   # stream chunks keep the register epilogue


def test_epilogue_refusals(lib):
    assert _staged(lib, _desc(1024, 1, 3, t_in=32), 0) == 0            # single output channel (MSD / MPD output convs)
    assert _staged(lib, _desc(64, 6, 3, t_in=2048), 0) == 0            # 6 produced channels: no float4 rows
    assert _staged(lib, _desc(6, 64, 3, t_in=2048), 1) == 0            # data gradient producing 6 channels
    assert _staged(lib, _desc(24, 36, 3, groups=3, t_in=2048), 0) == 1  # 12 channels per group in a 16-wide N tile
    assert _staged(lib, _desc(128, 128, 3, t_in=2048), 0) == 1


def test_staging_blocks_are_budgeted(lib):
    """The staged launches carry 8 x 2.5 KB of staging blocks: the plan's shared memory grows by that much (plus 16 bytes of
    alignment slack) for a layer whose rings keep their depth, and never passes the limit."""
    d = _desc(128, 128, 3, t_in=2048)
    p = _plan(lib, d, 0)
    s = _plan(lib, d, _lib.KT_PLAN_STREAM)
    assert (p["na"], p["nb"]) == (s["na"], s["nb"])
    assert p["smem"] - s["smem"] == 16 + 8 * 16 * 40 * 4   # alignment slack + blocks
    assert p["smem"] <= SMEM_MAX
