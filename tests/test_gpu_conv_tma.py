"""GPU: the TMA-fed route of the tensor-core conv kernel (the gathered operand written once per call as hi / lo bf16 planes,
the images pulled as boxes of whole time steps by the TMA unit) against the exact-fp32 kernels, forward and data gradient,
at the bf16x3 tolerance of the tensor-core path."""
import ctypes
import zlib

import pytest
import torch

from kantts_b200 import _lib, ops
from kantts_b200._lib import KT_ACT_LRELU, check, ptr, stream_ptr
from conftest import rel_l2

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 1e-4
KT_ERR_WORKSPACE = -3

CASES = {
    # name: (spec kwargs, B, T, period, TMA route expected for (forward, data gradient))
    # (the route needs >= 512 K gathered elements)
    # every period, with T not a multiple of the M tile's tt = 128 // period time steps
    **{f"period{p}": (dict(c_in=64, c_out=128, kernel=5, pad_left=2, pad_right=2, act_in=0.1, act_out=0.1), 16, t, p, (True, True))
       for p, t in ((2, 260), (3, 180), (5, 110), (7, 80), (11, 50))},
    # stride-3 residue images (1-2 taps each) with a left pad: negative time coordinates are the TMA unit's zeros
    "period3_stride3": (dict(c_in=128, c_out=256, kernel=5, stride=3, pad_left=2, pad_right=2, act_out=0.1), 16, 150, 3, (True, True)),
    "period11_stride3": (dict(c_in=64, c_out=128, kernel=5, stride=3, pad_left=2, pad_right=2, act_out=0.1), 16, 83, 11, (True, True)),
    # transposed k16 s8 upsampler (8 polyphase phases of 2 taps)
    "deconv_k16s8": (dict(c_in=256, c_out=128, kernel=16, stride=8, transposed=True, crop=8, act_in=0.1), 16, 130, 0, (True, True)),
    # 80 input channels: the second K chunk is 16 real channels and 48 zero-filled ones
    "cin80": (dict(c_in=80, c_out=512, kernel=3, pad_left=1, pad_right=1), 16, 420, 0, (True, True)),
    # 256 channels (two N tiles), fused tanh output
    "c256_tanh": (dict(c_in=256, c_out=256, kernel=3, pad_left=2, act_in=0.1, act_out="tanh"), 8, 300, 0, (True, True)),
}


def _spec(kw):
    kw = dict(kw)
    act_in, act_out = kw.pop("act_in", None), kw.pop("act_out", None)
    spec = ops.ConvSpec(**kw)
    if act_in is not None:
        spec.act_in, spec.act_in_slope = KT_ACT_LRELU, act_in
    if act_out == "tanh":
        spec.act_out = _lib.KT_ACT_TANH
    elif act_out is not None:
        spec.act_out, spec.act_out_slope = KT_ACT_LRELU, act_out
    return spec


def _inputs(name, spec, B, T, period):
    g = torch.Generator().manual_seed(zlib.crc32(name.encode()) % 10000)
    wshape = (spec.c_in, spec.c_out, spec.kernel) if spec.transposed else (spec.c_out, spec.c_in // spec.groups, spec.kernel)
    v = (torch.randn(wshape, generator=g) * 0.3).to(DEV)
    gg = (v.norm(2, dim=(1, 2), keepdim=True) * 1.1).to(DEV)
    bias = (0.1 * torch.randn(spec.c_out, generator=g)).to(DEV)
    xs = (B, T, period, spec.c_in) if period else (B, T, spec.c_in)
    x = torch.randn(xs, generator=g).to(DEV)
    t_out = spec.t_out(T)
    r = torch.randn((B, t_out, period, spec.c_out) if period else (B, t_out, spec.c_out), generator=g).to(DEV)
    return v, gg, bias, x, r


def _forward(spec, v, gg, bias, x, exact):
    ops.set_force_ffma(exact)
    try:
        xg = x.clone().requires_grad_(True)
        y = ops.conv(xg, spec, ops.PreparedWeight(), v, gg, bias)
    finally:
        ops.set_force_ffma(False)
    return xg, y


@pytest.mark.parametrize("name", list(CASES))
def test_tma_route_matches_the_exact_kernels(name):
    kw, B, T, period, expect = CASES[name]
    spec = _spec(kw)
    plan = spec.plan(B, period or 1, T)
    assert (plan.ws_fwd > 0, plan.ws_bwd > 0) == expect, (plan.ws_fwd, plan.ws_bwd)
    v, gg, bias, x, r = _inputs(name, spec, B, T, period)
    x_tc, y_tc = _forward(spec, v, gg, bias, x, False)
    x_ex, y_ex = _forward(spec, v, gg, bias, x, True)
    assert rel_l2(y_tc.detach().cpu(), y_ex.detach().cpu()) < TOL, ("y", rel_l2(y_tc.detach().cpu(), y_ex.detach().cpu()))
    if spec.act_out == KT_ACT_LRELU:
        # outputs whose sign differs between the two forwards switch the activation derivative: left out of the comparison
        flip = torch.sign(y_tc.detach()) != torch.sign(y_ex.detach())
        assert float(flip.float().mean()) < 1e-3
        r = r * (~flip)
    y_tc.backward(r)
    y_ex.backward(r)
    assert rel_l2(x_tc.grad.cpu(), x_ex.grad.cpu()) < TOL, ("dx", rel_l2(x_tc.grad.cpu(), x_ex.grad.cpu()))


def test_tma_route_of_the_upsampled_conv_data_gradient():
    """The nearest-upsampled conv's data gradient runs the plain conv over the up-sampled rows (ConvPlan.up_bwd): that conv
    takes the TMA route."""
    spec = _spec(dict(c_in=128, c_out=64, kernel=3, pad_left=2, upsample=2, act_in=0.1))
    B, T = 8, 600
    plan = spec.plan(B, 1, T)
    assert plan.up_bwd and plan.ws_fwd == 0 and plan.ws_bwd > 0
    v, gg, bias, x, r = _inputs("up_bwd", spec, B, T, 0)
    x_tc, y_tc = _forward(spec, v, gg, bias, x, False)
    x_ex, y_ex = _forward(spec, v, gg, bias, x, True)
    y_tc.backward(r)
    y_ex.backward(r)
    assert rel_l2(x_tc.grad.cpu(), x_ex.grad.cpu()) < TOL


class _Owner:
    pass


def test_tma_route_of_the_pair_reuse_subset_batch():
    """pair_state("reuse", nb): only the first nb items are computed (a batch of nb in the recorded buffer), the rest is kept."""
    spec = _spec(dict(c_in=512, c_out=1024, kernel=5, stride=3, pad_left=2, pad_right=2, act_out=0.1))
    B, nb, T, p = 8, 4, 60, 5
    assert spec.plan(nb, p, T).ws_fwd > 0
    v, gg, bias, x, _ = _inputs("reuse", spec, B, T, p)
    owner, cache = _Owner(), ops.PreparedWeight()
    with torch.no_grad():
        with ops.pair_state("record"):
            y_full = ops.pair_conv(owner, x, spec, cache, v, gg, bias).clone()
        x2 = x.clone()
        x2[:nb] = torch.randn_like(x2[:nb])
        with ops.pair_state("reuse", nb):
            y2 = ops.pair_conv(owner, x2, spec, cache, v, gg, bias)
        _, y_ex = _forward(spec, v, gg, bias, x2[:nb].contiguous(), True)
    assert torch.equal(y2[nb:], y_full[nb:])
    assert rel_l2(y2[:nb].cpu(), y_ex.cpu()) < TOL


def test_too_small_workspace_is_refused():
    spec = _spec(dict(c_in=1024, c_out=1024, kernel=5, pad_left=2, pad_right=2))
    B, T, p = 16, 20, 3
    plan = spec.plan(B, p, T)
    d, nt, ws_floats = plan.d, plan.tile(0), plan.ws_fwd
    assert ws_floats > 0
    v, gg, bias, x, _ = _inputs("ws", spec, B, T, p)
    pw = ops.prepare_weight(ops.PreparedWeight(), spec, v, gg)
    img = pw.image((0, nt), d)
    y = torch.empty((B, d.t_out, p, spec.c_out), device=DEV)
    ws = torch.empty(ws_floats, device=DEV)
    lib = _lib.load()
    for buf, n in ((ws, ws_floats - 1), (None, 0)):
        rc = lib.kt_conv1d_fwd_tc(ctypes.byref(d), ptr(x), ptr(img, True), None, None, ptr(y), ptr(buf), n, stream_ptr())
        assert rc == KT_ERR_WORKSPACE, rc
    check(lib.kt_conv1d_fwd_tc(ctypes.byref(d), ptr(x), ptr(img, True), None, None, ptr(y), ptr(ws), ws_floats, stream_ptr()),
          "kt_conv1d_fwd_tc")
    torch.cuda.synchronize()
    assert torch.isfinite(y).all()
