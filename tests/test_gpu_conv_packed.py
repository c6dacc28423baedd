"""GPU: packed M tiles of the tensor-core conv kernel (several batch items per 128-row tile when an item has few output rows).

A tile row's accumulator gets the same MMAs in the same order whichever tile it sits in, so every item of a packed batch must
match, bit for bit, the same item run as a batch of one (one item per tile).  The packed results are also checked against
the exact-fp32 kernels at the tensor-core tolerance."""
import ctypes
import zlib

import pytest
import torch

from kantts_b200 import _lib, ops
from kantts_b200._lib import KT_ACT_LRELU
from conftest import rel_l2

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 1e-4

CASES = {
    # name: (spec kwargs, B, T, period, items per tile expected for (forward, data gradient))
    # the scale discriminator's dense 1024-channel layer at 9 and 17 steps (simple register-staged instance, staged
    # epilogue; the data gradient masks with the pre-activation's derivative), batches that are no multiple of the packing
    "dense_k5_t9": (dict(c_in=1024, c_out=1024, kernel=5, pad_left=2, pad_right=2, act_in=0.1, act_out=0.1), 13, 9, 0, (10, 10)),
    "dense_k5_t17": (dict(c_in=1024, c_out=1024, kernel=5, pad_left=2, pad_right=2, act_in=0.1), 7, 17, 0, (6, 6)),
    # its single-channel output layer: register epilogue forward (1 output channel), generic instance
    "post_k3_t17": (dict(c_in=1024, c_out=1, kernel=3, pad_left=1, pad_right=1, act_in=0.1), 9, 17, 0, (6, 6)),
    # grouped k41: two and three items per tile
    "k41_g16_t17": (dict(c_in=1024, c_out=1024, kernel=41, groups=16, pad_left=20, pad_right=20, act_in=0.1), 5, 17, 0, (2, 2)),
    "k41_g16_t9": (dict(c_in=1024, c_out=1024, kernel=41, groups=16, pad_left=20, pad_right=20, act_in=0.1), 7, 9, 0, (3, 3)),
    # strided grouped k41 s4: four residue images per item block; its data gradient four phases of 8-9 rows per item
    "k41_g16_s4": (dict(c_in=512, c_out=1024, kernel=41, stride=4, groups=16, pad_left=20, pad_right=20, act_in=0.1),
                   5, 33, 0, (5, 5)),
    # the generator's conv_pre (80 input channels: a thin second K chunk)
    "conv_pre": (dict(c_in=80, c_out=512, kernel=7, pad_left=3, pad_right=3), 3, 32, 0, (3, 3)),
    # a linear layer at one time step (the speaker embedding's output layer): blocks of one row, every row its own item
    "linear_t1": (dict(c_in=1024, c_out=192, kernel=1), 5, 1, 0, (5, 5)),
    # grouped s4 layer with 16 -> 32 channels per group: 4 groups per tile at 32 items (128 M tiles), 1 per tile alone (the
    # under-filled grid drops the zero blocks): each output gets its own group's K slices in the same order either way
    "k41_g16_s4_groups": (dict(c_in=256, c_out=512, kernel=41, stride=4, groups=16, pad_left=20, pad_right=20, act_in=0.1),
                          32, 512, 0, (1, 1)),
    # sub-sequences (nsub = 5): rows = flattened (time, sub-sequence) positions
    "period5": (dict(c_in=64, c_out=128, kernel=5, pad_left=2, pad_right=2, act_in=0.1, act_out=0.1), 5, 8, 5, (2, 2)),
}


def _spec(kw):
    kw = dict(kw)
    act_in, act_out = kw.pop("act_in", None), kw.pop("act_out", None)
    spec = ops.ConvSpec(**kw)
    if act_in is not None:
        spec.act_in, spec.act_in_slope = KT_ACT_LRELU, act_in
    if act_out is not None:
        spec.act_out, spec.act_out_slope = KT_ACT_LRELU, act_out
    return spec


def _inputs(name, spec, B, T, period):
    g = torch.Generator().manual_seed(zlib.crc32(name.encode()) % 10000)
    wshape = (spec.c_out, spec.c_in // spec.groups, spec.kernel)
    v = (torch.randn(wshape, generator=g) * 0.3).to(DEV)
    gg = (v.norm(2, dim=(1, 2), keepdim=True) * 1.1).to(DEV)
    bias = (0.1 * torch.randn(spec.c_out, generator=g)).to(DEV)
    xs = (B, T, period, spec.c_in) if period else (B, T, spec.c_in)
    x = torch.randn(xs, generator=g).to(DEV)
    t_out = spec.t_out(T)
    shape = (B, t_out, period, spec.c_out) if period else (B, t_out, spec.c_out)
    return v, gg, bias, x, torch.randn(shape, generator=g).to(DEV), torch.randn(shape, generator=g).to(DEV)


def _pack(spec, B, T, period, direction):
    out = (ctypes.c_int64 * 5)()
    d = spec.plan(B, period or 1, T).d
    assert _lib.load().kt_debug_conv_tc_pack(ctypes.byref(d), direction, out) == 0
    return out[0]


def _run(spec, v, gg, bias, x, r, resid=None, exact=False):
    ops.set_force_ffma(exact)
    try:
        xg = x.clone().requires_grad_(True)
        y = ops.conv(xg, spec, ops.PreparedWeight(), v, gg, bias, resid)
        y.backward(r)
    finally:
        ops.set_force_ffma(False)
    torch.cuda.synchronize()
    return y.detach(), xg.grad


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("with_resid", [False, True])
def test_packed_tiles_match_one_item_per_tile(name, with_resid):
    kw, B, T, period, expect = CASES[name]
    spec = _spec(kw)
    assert (_pack(spec, B, T, period, 0), _pack(spec, B, T, period, 1)) == expect
    assert _pack(spec, 1, T, period, 0) == 1 and _pack(spec, 1, T, period, 1) == 1
    v, gg, bias, x, r, res = _inputs(name, spec, B, T, period)
    res = res if with_resid else None
    y, dx = _run(spec, v, gg, bias, x, r, res)
    for i in range(B):
        yi, dxi = _run(spec, v, gg, bias, x[i:i + 1], r[i:i + 1], None if res is None else res[i:i + 1])
        assert torch.equal(y[i:i + 1], yi), (name, i)
        assert torch.equal(dx[i:i + 1], dxi), (name, i)
    if spec.act_out == KT_ACT_LRELU:
        return   # the exact forward may flip a sign and with it the activation derivative (test_gpu_conv_tma)
    y_ex, dx_ex = _run(spec, v, gg, bias, x, r, res, exact=True)
    assert rel_l2(y.cpu(), y_ex.cpu()) < TOL
    assert rel_l2(dx.cpu(), dx_ex.cpu()) < TOL


class _Owner:
    pass


def test_packed_tiles_of_the_pair_reuse_subset_batch():
    """pair_state("reuse", nb): a batch of nb items in the recorded buffer, packed by nb (7 items: tiles of 3, 3 and 1)."""
    spec = _spec(dict(c_in=1024, c_out=1024, kernel=41, groups=16, pad_left=20, pad_right=20, act_in=0.1))
    B, nb, T = 12, 7, 9
    assert _pack(spec, nb, T, 0, 0) == 3
    v, gg, bias, x, _, _ = _inputs("reuse", spec, B, T, 0)
    owner, cache = _Owner(), ops.PreparedWeight()
    with torch.no_grad():
        with ops.pair_state("record"):
            y_full = ops.pair_conv(owner, x, spec, cache, v, gg, bias).clone()
        x2 = x.clone()
        x2[:nb] = torch.randn_like(x2[:nb])
        with ops.pair_state("reuse", nb):
            y2 = ops.pair_conv(owner, x2, spec, cache, v, gg, bias)
        y_one = [ops.conv(x2[i:i + 1].contiguous(), spec, ops.PreparedWeight(), v, gg, bias) for i in range(nb)]
    assert torch.equal(y2[nb:], y_full[nb:])
    assert torch.equal(y2[:nb], torch.cat(y_one))
