"""CPU: packed M tiles of the tensor-core conv kernel (kt_debug_conv_tc_pack, planned without a GPU as on one).  A layer whose
items have few output rows puts several items in each 128-row tile, each in a block of its output rows plus the halo its taps
read; the MMA rows the kernel issues and throws away shrink accordingly."""
import ctypes

import pytest

from kantts_b200 import _lib
from kantts_b200._lib import KT_PLAN_STREAM
from test_conv_tc_plan_cpu import C2, C4, _desc, _plan, _shape_desc


@pytest.fixture(scope="module")
def lib():
    return _lib.load()


def _pack(lib, d, direction):
    out = (ctypes.c_int64 * 5)()
    assert lib.kt_debug_conv_tc_pack(ctypes.byref(d), direction, out) == 0
    return dict(zip(("P", "L", "mma", "mma_unpacked", "rows"), list(out)))


@pytest.mark.parametrize("shape", C2 + C4)
def test_packing_of_every_model_layer(lib, shape):
    d = _shape_desc(shape)
    for direction in (0, 1):
        p, k = _plan(lib, d, direction), _pack(lib, d, direction)
        if not p["nt"]:
            assert k["P"] == 1
            continue
        assert 1 <= k["P"] <= d.batch and k["rows"] <= k["mma"] <= k["mma_unpacked"], (shape, direction, k)
        assert k["mma"] == 128 * (-(-d.batch // k["P"])) * (k["mma_unpacked"] // (128 * d.batch)), (shape, direction, k)
        if k["P"] > 1:
            assert not p["tma"], (shape, direction)   # a TMA box holds one item: register-staged route only
        if d.stride == 1 and not d.transposed and d.upsample == 1 and not p["tma"]:
            # one phase of M * nsub rows per item, taps spanning (kernel - 1) * dilation steps: the block holds both, and the
            # last item's output rows end inside the 128-row tile
            m_rows = k["rows"] // d.batch
            if m_rows > 64:
                assert k["P"] == 1, (shape, direction)
            else:
                L = m_rows + (d.kernel - 1) * d.dilation * d.nsub
                assert k["P"] == min(d.batch, (128 - m_rows) // L + 1), (shape, direction, k)
                assert k["P"] == 1 or (k["L"] == L and (k["P"] - 1) * L + m_rows <= 128), (shape, direction, k)
    if d.nsub == 1:
        s = _pack(lib, d, KT_PLAN_STREAM)
        assert s["P"] == 1, shape   # stream chunks: one item (slot window) per tile


def test_items_per_tile_of_the_scale_discriminator(lib):
    # dense k5 (tap span 4): 6 / 10 items at 17 / 9 steps on the register-staged route; from 512 K gathered elements on
    # (32 items at 17 steps and more) the TMA route, one item per tile; grouped k41 (span 40): 2 / 2 / 3
    for t, b, p in ((17, 16, 6), (9, 32, 10)):
        assert _pack(lib, _desc(1024, 1024, 5, batch=b, t_in=t), 0)["P"] == p
    for t in (17, 33):
        d = _desc(1024, 1024, 5, batch=32, t_in=t)
        assert _plan(lib, d, 0)["tma"] and _pack(lib, d, 0)["P"] == 1
    for t, p in ((33, 2), (17, 2), (9, 3)):
        k = _pack(lib, _desc(1024, 1024, 41, groups=16, batch=32, t_in=t), 0)
        assert k["P"] == p and k["L"] == t + 40
    # more than 64 rows per item: one item per tile
    assert _pack(lib, _desc(1024, 1024, 5, batch=32, t_in=65), 0)["P"] == 1
    assert _pack(lib, _desc(1024, 1024, 5, batch=32, nsub=3, t_in=34), 0)["P"] == 1
    # a batch smaller than the packing caps it
    assert _pack(lib, _desc(1024, 1024, 5, batch=4, t_in=9), 0)["P"] == 4


def test_n_split_sees_the_packed_tile_count(lib):
    # 256 -> 256 k3 at 16 steps, 64 items: 64 x 2 tiles unpacked (no split), 10 x 2 packed (7 items per tile): N halves
    d = _desc(256, 256, 3, batch=64, t_in=16)
    assert _pack(lib, d, 0)["P"] == 7 and _plan(lib, d, 0)["nt"] == 64
    assert _plan(lib, _desc(256, 256, 3, batch=64, t_in=80), 0)["nt"] == 128


def test_grouped_tiles_of_an_under_filled_grid(lib):
    # scale discriminator 512 -> 1024 k41 s4 g16 (32 -> 64 channels per group) at 32 output steps: 2 groups per N = 128
    # tile over 16 x 128 M tiles; packed 3 items per tile, 6 x 8 tiles would leave most SMs idle: one group per N = 64 tile
    d = _desc(512, 1024, 41, stride=4, groups=16, batch=16, t_in=128, pad=20)
    assert _pack(lib, d, 0)["P"] == 3 and _plan(lib, d, 0)["nt"] == 64
    assert _plan(lib, _desc(512, 1024, 41, stride=4, groups=16, batch=16, t_in=2048, pad=20), 0)["nt"] == 128
    # 256 -> 512 k41 s4 g16 (16 -> 32 per group) at 128 steps: 4 groups per tile x 16 M tiles -> 2 groups, N = 64
    assert _plan(lib, _desc(256, 512, 41, stride=4, groups=16, batch=16, t_in=512, pad=20), 0)["nt"] == 64
    assert _plan(lib, _desc(256, 512, 41, stride=4, groups=16, batch=32, t_in=512, pad=20), 0)["nt"] == 128
    # 8 produced channels per group: the N tile stays >= 16 (2 groups), so it still tells the two tilings apart
    assert _plan(lib, _desc(64, 128, 5, groups=16, batch=1, t_in=8), 0)["nt"] == 16


def test_padding_removed_over_the_c2_step(lib):
    """MMA rows issued per N tile against output rows produced, over every layer and direction of the C2 list."""
    before = after = rows = 0
    for shape in C2:
        d = _shape_desc(shape)
        for direction in (0, 1):
            if not _plan(lib, d, direction)["nt"]:
                continue
            k = _pack(lib, d, direction)
            before, after, rows = before + k["mma_unpacked"], after + k["mma"], rows + k["rows"]
    padding_before, padding_after = before - rows, after - rows
    print(f"C2 conv layers: {rows} output rows; MMA rows {before} -> {after}, padding {padding_before} -> {padding_after}")
    assert after < before and padding_after < padding_before
