"""GPU: the shared-memory staged epilogue of the tensor-core conv kernel (bias, output activation, residual, act' mask of the
data gradient, partial M tiles, grouped tiles narrower than their MMA tile, sub-sequences) against the exact-fp32 kernels at
the bf16x3 tolerance, and against the register epilogue bit for bit."""
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
    # name: (spec kwargs, B, T, period, residual)
    # generator resblock conv: pre-activation, fused residual; T = 1000 leaves a partial last M tile
    "resid_fwd_partial": (dict(c_in=128, c_out=128, kernel=3, pad_left=1, pad_right=1, act_in=0.1), 4, 1000, 0, True),
    # output activation + masked data gradient (act_in's derivative), two N tiles
    "lrelu_two_ntiles": (dict(c_in=256, c_out=256, kernel=7, pad_left=3, pad_right=3, act_in=0.1, act_out=0.1), 4, 300, 0, False),
    # polyphase transposed forward (o_step = 4) and its strided data gradient
    "deconv_k8s4": (dict(c_in=128, c_out=64, kernel=8, stride=4, transposed=True, crop=2, act_in=0.1), 4, 257, 0, False),
    # strided conv (its data gradient is polyphase), period layer (nsub = 3) with a time count that leaves partial tiles
    "period3_stride3": (dict(c_in=64, c_out=128, kernel=5, stride=3, pad_left=2, pad_right=2, act_out=0.1), 4, 100, 3, False),
    "period5": (dict(c_in=32, c_out=64, kernel=5, pad_left=2, pad_right=2, act_in=0.1), 4, 70, 5, False),
    # block-diagonal grouped tile: 12 produced channels per group in a 16-wide MMA tile
    "grouped_nstride12": (dict(c_in=24, c_out=36, kernel=3, groups=3, pad_left=1, pad_right=1, act_in=0.1), 4, 500, 0, True),
    # 64 -> 48: a 48-wide N tile (a partial 32-column chunk)
    "c48": (dict(c_in=64, c_out=48, kernel=3, pad_left=1, pad_right=1), 4, 700, 0, True),
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


def _run(spec, v, gg, bias, x, resid, r, exact):
    ops.set_force_ffma(exact)
    try:
        xg = x.clone().requires_grad_(True)
        y = ops.conv(xg, spec, ops.PreparedWeight(), v, gg, bias, resid=resid)
        y.backward(r)
    finally:
        ops.set_force_ffma(False)
    return y.detach(), xg.grad


@pytest.mark.parametrize("name", list(CASES))
def test_staged_epilogue_matches_the_exact_kernels(name):
    kw, B, T, period, with_resid = CASES[name]
    spec = _spec(kw)
    lib = _lib.load()
    d = spec.plan(B, period or 1, T).d
    assert lib.kt_debug_conv_tc_epilogue(ctypes.byref(d), 0) == 1
    assert lib.kt_debug_conv_tc_epilogue(ctypes.byref(d), 1) == (1 if spec.c_in % 4 == 0 else 0)
    g = torch.Generator().manual_seed(zlib.crc32(name.encode()) % 10000)
    wshape = (spec.c_in, spec.c_out, spec.kernel) if spec.transposed else (spec.c_out, spec.c_in // spec.groups, spec.kernel)
    v = (torch.randn(wshape, generator=g) * 0.3).to(DEV)
    gg = (v.norm(2, dim=(1, 2), keepdim=True) * 1.1).to(DEV)
    bias = (0.1 * torch.randn(spec.c_out, generator=g)).to(DEV)
    x = torch.randn((B, T, period, spec.c_in) if period else (B, T, spec.c_in), generator=g).to(DEV)
    t_out = spec.t_out(T)
    yshape = (B, t_out, period, spec.c_out) if period else (B, t_out, spec.c_out)
    resid = torch.randn(yshape, generator=g).to(DEV) if with_resid else None
    r = torch.randn(yshape, generator=g).to(DEV)
    y_tc, dx_tc = _run(spec, v, gg, bias, x, resid, r, False)
    y_ex, dx_ex = _run(spec, v, gg, bias, x, resid, r, True)
    assert rel_l2(y_tc.cpu(), y_ex.cpu()) < TOL, ("y", rel_l2(y_tc.cpu(), y_ex.cpu()))
    if spec.act_out == KT_ACT_LRELU:
        # outputs whose sign differs between the two forwards switch the activation derivative: recompute without them
        flip = torch.sign(y_tc) != torch.sign(y_ex)
        assert float(flip.float().mean()) < 1e-3
        r = r * (~flip)
        _, dx_tc = _run(spec, v, gg, bias, x, resid, r, False)
        _, dx_ex = _run(spec, v, gg, bias, x, resid, r, True)
    assert rel_l2(dx_tc.cpu(), dx_ex.cpu()) < TOL, ("dx", rel_l2(dx_tc.cpu(), dx_ex.cpu()))


def test_staged_and_register_epilogues_write_the_same_bits():
    """A residual whose storage starts 8 bytes into an allocation is not 16-byte aligned (the register epilogue's float2
    loads still are): that launch takes the register epilogue.  Both epilogues do the same fp32 operations per element, so
    the outputs are bit-identical."""
    spec = _spec(dict(c_in=128, c_out=128, kernel=3, pad_left=1, pad_right=1, act_in=0.1, act_out=0.1))
    B, T = 4, 1000
    g = torch.Generator().manual_seed(7)
    v = (torch.randn((128, 128, 3), generator=g) * 0.3).to(DEV)
    gg = (v.norm(2, dim=(1, 2), keepdim=True) * 1.1).to(DEV)
    bias = (0.1 * torch.randn(128, generator=g)).to(DEV)
    x = torch.randn((B, T, 128), generator=g).to(DEV)
    resid = torch.randn((B, T, 128), generator=g).to(DEV)
    cache = ops.PreparedWeight()
    with torch.no_grad():
        y_aligned = ops.conv(x, spec, cache, v, gg, bias, resid=resid)
        buf = torch.empty(resid.numel() + 2, device=DEV)
        resid_odd = buf[2:].view(resid.shape)
        resid_odd.copy_(resid)
        assert resid_odd.data_ptr() % 16 == 8
        y_odd = ops.conv(x, spec, cache, v, gg, bias, resid=resid_odd)
    assert torch.equal(y_aligned, y_odd)
