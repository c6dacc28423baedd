"""CPU: the route plan of the tensor-core conv kernel (kt_debug_conv_tc_plan, made without a GPU as it would be made on one):
which layers take the TMA-fed route (operand planes written once per call, image boxes pulled by the TMA unit), its M tiles
of whole time steps, its shared memory and its workspace."""
import ctypes

import pytest

from kantts_b200 import _lib, ops
from kantts_b200._lib import KT_ACT_LRELU, KT_PATH_TC, KtConv1dDesc

SMEM_LIMIT = 227 * 1024


@pytest.fixture(scope="module")
def lib():
    return _lib.load()


def _desc(cin, cout, k, stride=1, dil=1, groups=1, transposed=0, up=1, batch=16, nsub=1, t_in=2048, pad=None, path=0):
    pad = (k - 1) * dil // 2 if pad is None else pad
    if transposed:
        t_out = (t_in - 1) * stride - 2 * pad + dil * (k - 1) + 1
    else:
        t_out = (t_in * up + 2 * pad - dil * (k - 1) - 1) // stride + 1
    return KtConv1dDesc(batch=batch, nsub=nsub, t_in=t_in, t_out=t_out, c_in=cin, c_out=cout, groups=groups, kernel=k,
                        stride=stride, dilation=dil, pad_left=pad, transposed=transposed, upsample=up, act_in=KT_ACT_LRELU,
                        act_in_slope=0.1, act_out=KT_ACT_LRELU, act_out_slope=0.1, path=path)


def _plan(lib, d, direction):
    out = (ctypes.c_int64 * 9)()
    assert lib.kt_debug_conv_tc_plan(ctypes.byref(d), direction, out) == 0
    return dict(zip(("nt", "tma", "tt", "R", "a_box_t", "na", "nb", "smem", "ws"), list(out)))


# (c_in, c_out, kernel, stride, dilation, groups, transposed, upsample, batch, nsub, t_in): every conv layer of the C2 train
# step (HiFi-GAN generator, multi-scale and multi-period discriminators, their pair batches) and the SAM-BERT (C4) linears
# and convs
C2 = [(1, 32, 5, 3, 1, 1, 0, 1, 16, 7, 1171), (1, 128, 15, 1, 1, 1, 0, 1, 16, 1, 8192), (1, 128, 15, 1, 1, 1, 0, 1, 32, 1, 4098),
      (2, 1, 15, 1, 1, 1, 0, 1, 32, 1, 2051), (32, 32, 3, 1, 1, 1, 0, 1, 16, 1, 8192), (32, 32, 7, 1, 3, 1, 0, 1, 16, 1, 8192),
      (32, 32, 11, 1, 5, 1, 0, 1, 16, 1, 8192), (64, 32, 7, 1, 1, 1, 0, 2, 16, 1, 4096), (64, 64, 3, 1, 1, 1, 0, 1, 16, 1, 4096),
      (64, 64, 11, 1, 3, 1, 0, 1, 16, 1, 4096), (128, 64, 7, 1, 1, 1, 0, 2, 16, 1, 2048), (128, 128, 3, 1, 1, 1, 0, 1, 16, 1, 2048),
      (128, 128, 7, 1, 1, 1, 0, 1, 16, 1, 2048), (128, 128, 7, 1, 5, 1, 0, 1, 16, 1, 2048), (128, 128, 11, 1, 1, 1, 0, 1, 16, 1, 2048),
      (128, 128, 11, 1, 5, 1, 0, 1, 16, 1, 2048), (128, 128, 41, 4, 1, 4, 0, 1, 16, 1, 8192), (128, 128, 41, 4, 1, 4, 0, 1, 32, 1, 4098),
      (128, 256, 41, 4, 1, 16, 0, 1, 16, 1, 2048), (256, 128, 7, 1, 1, 1, 0, 8, 16, 1, 256), (256, 128, 16, 8, 1, 1, 1, 1, 16, 1, 256),
      (256, 256, 3, 1, 1, 1, 0, 1, 16, 1, 256), (256, 256, 11, 1, 3, 1, 0, 1, 16, 1, 256), (256, 512, 41, 4, 1, 16, 0, 1, 16, 1, 512),
      (512, 256, 7, 1, 1, 1, 0, 8, 16, 1, 32), (512, 256, 16, 8, 1, 1, 1, 1, 16, 1, 32), (512, 1024, 41, 4, 1, 16, 0, 1, 16, 1, 128),
      (1024, 1, 3, 1, 1, 1, 0, 1, 16, 1, 32), (1024, 1024, 5, 1, 1, 1, 0, 1, 16, 1, 32), (1024, 1024, 5, 1, 1, 1, 0, 1, 32, 1, 9),
      (1024, 1024, 41, 1, 1, 16, 0, 1, 16, 1, 32)]
for p, t1, t2, t3 in ((2, 456, 152, 51), (3, 304, 102, 34), (5, 183, 61, 21), (7, 131, 44, 15), (11, 83, 28, 10)):
    C2 += [(128, 512, 5, 3, 1, 1, 0, 1, 32, p, t1), (512, 1024, 5, 3, 1, 1, 0, 1, 32, p, t2), (512, 1024, 5, 3, 1, 1, 0, 1, 16, p, t2),
           (1024, 1024, 5, 1, 1, 1, 0, 1, 32, p, t3), (1024, 1, 2, 1, 1, 1, 0, 1, 32, p, t3)]
C4 = [(128, 1024, 3, 1, 1, 1, 0, 1, 32, 1, 256), (1024, 128, 1, 1, 1, 1, 0, 1, 32, 1, 256), (128, 240, 1, 1, 1, 1, 0, 1, 32, 1, 256),
      (80, 512, 1, 1, 1, 1, 0, 1, 32, 1, 256), (288, 128, 1, 1, 1, 1, 0, 1, 32, 1, 256), (512, 80, 3, 1, 1, 1, 0, 1, 32, 1, 256),
      (512, 512, 5, 1, 1, 1, 0, 1, 32, 1, 256)]


def _shape_desc(s):
    cin, cout, k, stride, dil, groups, tr, up, B, nsub, t = s
    return _desc(cin, cout, k, stride, dil, groups, tr, up, B, nsub, t)


@pytest.mark.parametrize("shape", C2 + C4)
def test_every_model_layer_has_a_consistent_route(lib, shape):
    d = _shape_desc(shape)
    for direction in (0, 1):
        p = _plan(lib, d, direction)
        assert p["nt"] == lib.kt_conv1d_tc_plan(ctypes.byref(d), direction), (shape, direction)
        if not p["nt"]:
            continue
        assert 0 < p["smem"] <= SMEM_LIMIT, (shape, direction, p)
        assert p["na"] >= 2 and p["nb"] >= 2, (shape, direction, p)
        gathered_c = d.c_in if direction == 0 else d.c_out
        gathered_t = d.t_in if direction == 0 else d.t_out
        if p["tma"]:
            # M tiles of whole time steps, R = tt * nsub <= 128 rows (at most nsub - 1 of the 128 MMA rows unused); one box
            # holds the tile's time steps plus the tap span, at most 256 of them
            assert p["R"] == p["tt"] * d.nsub and 128 - d.nsub < p["R"] <= 128, (shape, direction, p)
            assert p["tt"] <= p["a_box_t"] <= 256, (shape, direction, p)
            assert d.upsample == 1 and gathered_c % 8 == 0, (shape, direction)
            # workspace = hi + lo bf16 planes of the gathered operand: one float per element, padded to 64 floats
            n = d.batch * gathered_t * d.nsub * gathered_c
            assert p["ws"] == (n + 63) // 64 * 64, (shape, direction, p)
        else:
            assert p["R"] == 128 and p["ws"] == 0, (shape, direction, p)


def test_route_of_the_layers_the_split_pass_is_for(lib):
    tma = lambda d, direction: _plan(lib, d, direction)["tma"] == 1
    # period discriminator: 1024-channel stride-1 layers (8 N tiles re-staged each image) and stride-3 layers (1-2 taps per
    # residue image), both directions
    for p in (2, 3, 5, 7, 11):
        assert tma(_desc(1024, 1024, 5, batch=32, nsub=p, t_in=34), 0) and tma(_desc(1024, 1024, 5, batch=32, nsub=p, t_in=34), 1)
        assert tma(_desc(512, 1024, 5, stride=3, nsub=p, t_in=102), 0) and tma(_desc(512, 1024, 5, stride=3, nsub=p, t_in=102), 1)
    # scale discriminator, transposed upsampler (2 taps per polyphase phase), the waveform layer's data gradient
    assert tma(_desc(1024, 1024, 5, t_in=32), 0) and tma(_desc(1024, 1, 3, t_in=32), 0)
    assert tma(_desc(256, 128, 16, stride=8, transposed=1, t_in=256, pad=4), 0)
    assert tma(_desc(1, 32, 5, stride=3, nsub=7, t_in=1171), 1)
    # one N tile over >= 4 M gathered elements stays register-staged (HBM-bound either way: the generator's 128-channel
    # convs at 32 K rows, the period discriminator's 128 -> 512 data gradient) ...
    for k, dil in ((3, 1), (7, 1), (11, 1), (11, 5)):
        assert not tma(_desc(128, 128, k, dil=dil), 0) and not tma(_desc(128, 128, k, dil=dil), 1)
    assert not tma(_desc(128, 512, 5, stride=3, batch=32, nsub=2, t_in=456), 1)
    # ... but the 256-channel ones are staged once per N tile (2 tiles)
    assert tma(_desc(256, 256, 11, t_in=256), 0) and tma(_desc(256, 256, 3, t_in=256), 1)
    # too small for any producer to be the bound: register-staged (batch-1 inference, 1024 channels at 9 time steps)
    assert not tma(_desc(1024, 1024, 5, batch=32, t_in=9), 0) and not tma(_desc(256, 128, 16, stride=8, transposed=1, batch=1, t_in=32), 0)
    # grouped layers stay register-staged
    assert not tma(_desc(128, 128, 41, stride=4, groups=4, t_in=8192), 1)
    assert not tma(_desc(512, 1024, 41, stride=4, groups=16, t_in=128), 1)


def test_route_refusals(lib):
    tma = lambda d, direction: _plan(lib, d, direction)["tma"] == 1
    # nearest-upsampled input: the planes hold the tensor as stored
    d = _desc(256, 128, 3, up=8, t_in=256)
    assert _plan(lib, d, 0)["nt"] > 0 and not tma(d, 0)
    # c_in = 1 (a tensor-core layer by request): a 2-byte row is no 16-byte TMA stride
    d = _desc(1, 32, 5, stride=3, nsub=3, t_in=300, path=KT_PATH_TC)
    assert _plan(lib, d, 0)["nt"] > 0 and not tma(d, 0)
    # channel counts not divisible by 8: gathered width, and the channels of one grouped tile
    d = _desc(36, 64, 3, t_in=1000)
    assert _plan(lib, d, 0)["nt"] > 0 and not tma(d, 0) and tma(d, 1)
    d = _desc(64, 36, 3, t_in=1000)
    assert not tma(d, 1) and tma(d, 0)


def test_conv_plan_allocates_the_workspaces(lib):
    """ConvPlan asks the library for the forward / data-gradient workspaces.  Without a driver (this machine) the TMA route
    is unavailable, so they are 0 here; with one they match kt_debug_conv_tc_plan."""
    spec = ops.ConvSpec(c_in=512, c_out=1024, kernel=5, stride=3, pad_left=2, pad_right=2)
    p = spec.plan(16, 3, 102)
    for ws, direction in ((p.ws_fwd, 0), (p.ws_bwd, 1)):
        assert ws == lib.kt_conv1d_tc_workspace(ctypes.byref(p.d), direction)
        assert ws in (0, _plan(lib, p.d, direction)["ws"])
