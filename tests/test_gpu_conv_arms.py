"""Every pass of the training conv layers against a float64 reference of the same operation, instance by instance: the
forward, data gradient, weight and bias gradient on the exact-fp32 kernels (conv_ffma.cu: conv_core_kernel,
conv_wgrad_kernel, split_sum_kernel / split_sum_wide_kernel, colsum_kernel) and on the tensor-core kernels (conv_tc.cu:
conv_tc_kernel<0 | 1 | 2>; wgrad_tc.cu: wgrad_tc_kernel / wgrad_tma_kernel and their split-K reduces), and the weight-norm
kernels (weights.cu), each called through its C entry point.

The backward entry points get the x and y the test chooses as the sources of their activation derivatives, and the
reference uses the same tensors, so every comparison is arithmetic only (no outputs whose activation sign flips).  Each
result is checked per element, |got - ref| <= c * scale with scale the same sums over magnitudes (the bound of any
summation order), so that one wrong row, tap, channel or split cannot hide under a whole-tensor norm; the relative L2 is
bounded at the suite's bounds too.

Each pass is pinned to the kernel instances it is named for: the kernels it launches are read from a CUDA graph captured
around a second call and compared with a mirror of the host dispatch (run_core / run_wgrad / split_sum of conv_ffma.cu,
run_tc's `simple` predicate) and with the plans kt_debug_conv_tc_plan / kt_debug_wgrad_plan make on this device.
test_conv_arms_cpu.py checks, without a GPU, that the cases reach every instance.

The weight-gradient paths promise a fixed summation order (one CTA per element per split slice, slices summed in order,
the SPLITM warp fold in warp order): every weight-gradient pass runs twice and must give the same bits.
"""
import ctypes
import math
import re
import zlib
from dataclasses import dataclass, replace

import pytest
import torch

from conftest import rel_l2
from test_gpu_stream_conv import _launched_kernels, _mangled, conv_phase_rows, core_instance

DEV = "cuda"
F64 = torch.float64
KT_ACT_NONE, KT_ACT_LRELU, KT_ACT_TANH = 0, 1, 2

# Per-element error over the error scale, per route and summation:
#   conv   forward / data gradient: k * c_in / groups products per element (exact fp32: one FMA chain per thread; bf16x3:
#          fp32 MMA accumulation of the hi*hi + hi*lo + lo*hi products, each operand's bits below its 16-bit split dropped)
#   wgrad  weight gradient: B * nsub * t products per element, split into chunks and split-K slices summed in order
#   bias   bias gradient: B * nsub * t_out terms per channel, 8 row lanes per CTA and the CTA slots summed in order
#   weight weight norm and its backward: a row norm over d1 * k squares, one dot product over the row
# Worst over all cases on an H100 80GB HBM3 (700 W power limit): exact fp32 conv 4.61e-7 (c7_4_d2_rm8), wgrad 2.98e-7
# (c4_64_deconv_k16s8), bias 5.91e-8 on both routes (one_step: the fp32 product dy * act'); bf16x3 conv 1.99e-5
# (c2_70_deconv_k4s2_rm8), wgrad 1.58e-5 (one_step_c16); weight norm 1.89e-7 (transposed_tiled, mode 1).  The bounds are
# about 4x those.
ELEM_BOUND = {
    "ffma": {"conv": 1.9e-6, "wgrad": 1.2e-6, "bias": 2.4e-7},
    "tc": {"conv": 8e-5, "wgrad": 6.4e-5, "bias": 2.4e-7},
}
WEIGHT_BOUND = 7.5e-7
# Relative L2: the suite's bounds (forward, gradients) for the two routes (worst measured: exact 5.9e-7, bf16x3 7.6e-6)
L2_BOUND = {"ffma": (2e-5, 5e-5), "tc": (1e-4, 3e-4)}


def _lib():
    from kantts_b200 import _lib
    return _lib.load()


def _call(fn, *args):
    from kantts_b200 import ops
    ops.call(fn, *args)


def _ptr(t, aux=False):
    from kantts_b200._lib import ptr
    return ptr(t, aux)


# ------------------------------------------------------------------------------------------------
# cases
# ------------------------------------------------------------------------------------------------


@dataclass
class Case:
    name: str
    kw: dict                   # ConvSpec fields; act_in: LeakyReLU slope, act_out: slope or "tanh"
    B: int
    T: int
    period: int = 0            # nsub (0: the (B, T, C) layout)
    resid: bool = False

    @property
    def spec(self):
        from kantts_b200.ops import ConvSpec
        kw = dict(self.kw)
        act_in, act_out = kw.pop("act_in", None), kw.pop("act_out", None)
        s = ConvSpec(**kw)
        if act_in is not None:
            s.act_in, s.act_in_slope = KT_ACT_LRELU, act_in
        if act_out == "tanh":
            s.act_out = KT_ACT_TANH
        elif act_out is not None:
            s.act_out, s.act_out_slope = KT_ACT_LRELU, act_out
        return s

    @property
    def nsub(self):
        return self.period or 1

    def desc(self, spec=None, t_in=None):
        return (spec or self.spec).desc(self.B, self.nsub, t_in or self.T)


L = dict(act_in=0.1)
CASES = {c.name: c for c in [
    # 16 items x 19 M tiles of 128 rows: >= 296 CTAs, the exact kernel's 16-row-per-warp tiles (RM 16)
    Case("c3_20_rm16", dict(c_in=3, c_out=20, kernel=3, pad_left=1, pad_right=1, **L), 16, 2400),
    Case("c4_40_s2_rm16", dict(c_in=4, c_out=40, kernel=5, stride=2, pad_left=2, pad_right=2), 16, 4800),
    Case("c3_100_d3_period4_rm16", dict(c_in=3, c_out=100, kernel=3, dilation=3, pad_left=3, pad_right=3,
                                        act_out=0.2), 4, 2400, period=4),
    Case("c80_200_g2_rm16", dict(c_in=80, c_out=200, kernel=3, groups=2, pad_left=1, pad_right=1, **L), 8, 2400,
         resid=True),
    # 16 items x 19 M tiles of 64 rows (RM 8)
    Case("c3_36_tanh_rm8", dict(c_in=3, c_out=36, kernel=3, pad_left=1, pad_right=1, act_out="tanh"), 16, 1200),
    Case("c2_70_deconv_k4s2_rm8", dict(c_in=2, c_out=70, kernel=4, stride=2, pad_left=1, transposed=True, **L), 16, 1200),
    Case("c7_4_d2_rm8", dict(c_in=7, c_out=4, kernel=5, dilation=2, pad_left=4, pad_right=4, act_in=0.2), 16, 1200),
    Case("c40_72_up2_rm8", dict(c_in=40, c_out=72, kernel=3, upsample=2, pad_left=1, pad_right=1, **L), 16, 600),
    # few rows (RM 4), odd lengths
    Case("c3_5_k7_t37", dict(c_in=3, c_out=5, kernel=7, pad_left=3, pad_right=3, act_out=0.1), 2, 37),
    Case("c4_64_deconv_k16s8", dict(c_in=4, c_out=64, kernel=16, stride=8, pad_left=4, transposed=True, crop=8, **L), 2,
         45),
    Case("c2_80_t50", dict(c_in=2, c_out=80, kernel=3, pad_left=2, act_out=0.2), 2, 50, resid=True),
    Case("c40_96_s3_t101", dict(c_in=40, c_out=96, kernel=5, stride=3, pad_left=2, pad_right=2, **L), 3, 101),
    # the weight gradient's remaining (RN, RMA, SPLITM) instances
    Case("c6_48_rm8", dict(c_in=6, c_out=48, kernel=3, pad_left=1, pad_right=1), 16, 1200),
    Case("c8_100_t300", dict(c_in=8, c_out=100, kernel=2, pad_left=1, act_out=0.1), 4, 300),
    Case("c20_30_t257", dict(c_in=20, c_out=30, kernel=3, pad_left=2, **L), 4, 257),
    Case("c24_64_period3", dict(c_in=24, c_out=64, kernel=5, pad_left=2, pad_right=2, **L), 4, 200, period=3),
    Case("c32_128_t600", dict(c_in=32, c_out=128, kernel=3, pad_left=1, pad_right=1, act_out=0.1), 8, 600),
    Case("c64_64_tma", dict(c_in=64, c_out=64, kernel=3, pad_left=1, pad_right=1, **L), 16, 600, resid=True),
    # tensor-core route 1 from a fused tanh alone
    Case("c32_4_tanh", dict(c_in=32, c_out=4, kernel=7, pad_left=3, pad_right=3, act_out="tanh", **L), 4, 300),
    # one output time step, one item: a single weight-gradient split that writes dw directly
    Case("one_step", dict(c_in=5, c_out=12, kernel=3, pad_left=1, pad_right=1, act_out=0.2), 1, 1),
    Case("one_step_c16", dict(c_in=16, c_out=16, kernel=3, pad_left=1, pad_right=1), 1, 1),
    # phases no tap reaches: a transposed conv with stride 4 > kernel 3, and the data gradient of a conv with stride 3 > 2
    Case("deconv_k3s4_empty_phase", dict(c_in=16, c_out=12, kernel=3, stride=4, transposed=True), 2, 40),
    Case("c6_10_k2s3_empty_phase", dict(c_in=6, c_out=10, kernel=2, stride=3, act_out=0.1), 2, 61),
    # weight gradients whose size is not a multiple of 4 (the reduces' scalar branches): few units, then many
    Case("c3_5_k7_reduce", dict(c_in=3, c_out=5, kernel=7, pad_left=3, pad_right=3), 2, 150),
    Case("c2_1_k15_wide", dict(c_in=2, c_out=1, kernel=15, pad_left=7, pad_right=7, act_out="tanh"), 8, 2000),
    Case("c8_16_t200", dict(c_in=8, c_out=16, kernel=3, pad_left=1, pad_right=1), 2, 200),
]}


# ------------------------------------------------------------------------------------------------
# mirrors of the host dispatch
# ------------------------------------------------------------------------------------------------


def _split_sum(n, nsplit):
    """split_sum's kernel for n outputs of nsplit slots (misc.cu)."""
    return "split_sum_wide_kernel" if nsplit >= 64 and n <= 4096 else "split_sum_kernel"


def _colsum(c):
    """colsum_bias over the B * nsub * t_out rows of dy: colsum_kernel, then its ny CTA slots summed by split_sum."""
    s = c.spec
    rows = c.B * c.nsub * s.t_out(c.T)
    ny = min(max(1, rows // 256), 512)
    return {"colsum_kernel", _split_sum(s.c_out, ny)}


def exact_wgrad(c):
    """-> (kernels, nsplit) of kt_conv1d_bwd_weight: run_wgrad's conv_wgrad_kernel instance and launch_wgrad's split count
    (1: atomics straight into dw), the split sum, and the bias gradient's kernels."""
    s = c.spec
    if s.transposed:
        ca_g, cb_g, M = s.c_out, s.c_in, c.T
    else:
        ca_g, cb_g, M = s.c_in // s.groups, s.c_out // s.groups, s.t_out(c.T)
    rn = 4 if cb_g > 64 else (2 if cb_g > 32 else 1)
    rma, splitm = (4, True) if ca_g <= 4 else (8, True) if ca_g <= 8 else (4, False) if ca_g <= 32 else (8, False)
    tca = rma if splitm else 8 * rma
    npass = -(-s.kernel // 3)
    units = c.B * c.nsub * -(-M // 32)
    base = -(-ca_g // tca) * s.groups * -(-cb_g // (32 * rn)) * npass
    nsplit = max(1, 528 // max(1, base))
    nsplit = min(nsplit, max(1, units // 4), 4096)
    g_size = s.w_numel
    nsplit = max(1, min(nsplit, 2 ** 25 // g_size))
    names = {f"conv_wgrad_kernel<{rn}, {rma}, {'true' if splitm else 'false'}>"} | _colsum(c)
    if nsplit > 1:
        names.add(_split_sum(g_size, nsplit))
    return names, nsplit


def exact_conv(c, direction):
    """The conv_core_kernel instances of kt_conv1d_fwd (direction 0) / kt_conv1d_bwd_data (1), one per phase."""
    s = c.spec
    cin_g, cout_g = s.c_in // s.groups, s.c_out // s.groups
    if direction:
        cin_g, cout_g = cout_g, cin_g
    return {core_instance(M, cin_g, cout_g, s.groups, c.B * c.nsub) for M in conv_phase_rows(s, c.T, direction)}


def up_bwd_spec(c):
    """The data gradient of a nearest-upsampled conv on the tensor cores: the same conv over the up-sampled rows (upsample
    1, no pre-activation), folded back by kt_upsample_grad_reduce (ops.ConvPlan.up_bwd)."""
    return replace(c.spec, upsample=1, act_in=KT_ACT_NONE, act_in_slope=0.0)


def tc_conv(c, direction):
    """-> (descriptor, route, causes) of the tensor-core pass (0 forward, 1 data gradient) from kt_debug_conv_tc_plan and
    run_tc's `simple` predicate, None when the pass stays on the exact kernels.  causes: why a register-staged launch is not
    the simple route 0 ("nsub", "upsample", "tanh", "alignment")."""
    s = c.spec
    if direction and s.upsample > 1:
        if s.c_in % 4 or s.transposed:
            return None
        s = up_bwd_spec(c)
        d = c.desc(s, c.T * c.spec.upsample)
    else:
        d = c.desc()
    out = (ctypes.c_int64 * 9)()
    assert _lib().kt_debug_conv_tc_plan(ctypes.byref(d), direction, out) == 0
    if not out[0]:
        return None
    if out[1]:
        return d, 2, ()
    g = s.groups
    kin, pout = (s.c_in, s.c_out) if direction == 0 else (s.c_out, s.c_in)
    kin, pout = kin // g, pout // g
    if g > 1:                                            # layer_plan: groups packed per N tile
        gt = 1
        while gt * 2 <= g and g % (gt * 2) == 0 and kin * gt * 2 <= 64 and pout * gt * 2 <= 128:
            gt *= 2
        kg, n_stride = gt * kin, gt * pout
    else:
        kg, n_stride = kin, int(out[0])
    up = s.upsample if direction == 0 and not s.transposed else 1
    causes = []
    if c.nsub > 1:
        causes.append("nsub")
    if up > 1:
        causes.append("upsample")
    if direction == 0 and s.act_out == KT_ACT_TANH:
        causes.append("tanh")
    if kg % 8 or (kin * g) % 4 or (pout * g) % 4 or n_stride % 4:
        causes.append("alignment")
    return d, (1 if causes else 0), tuple(causes)


def tc_wgrad(c):
    """-> (kernels, nsplit, reduce branch) of kt_conv1d_bwd_weight_tc from kt_debug_wgrad_plan (this device's SM count),
    None when the layer stays on the exact kernels.  The reduce runs its scalar branch when the gradient's size is not a
    multiple of 4."""
    s = c.spec
    d = c.desc()
    out = (ctypes.c_int32 * 12)()
    assert _lib().kt_debug_wgrad_plan(ctypes.byref(d), out) == 0
    if not out[0]:
        return None
    names = {f"wgrad_{'tma' if out[1] else 'tc'}_kernel<{out[8]}>"} | _colsum(c)
    ns = int(out[7])
    branch = "float4" if s.w_numel % 4 == 0 else "scalar"
    if ns >= 16:
        names.add("wgrad_reduce_wide_kernel")
    elif ns > 1:
        names.add("wgrad_reduce_kernel")
    return names, ns, branch


def passes(c):
    """-> {(route, pass): expected kernels} of case c: every pass on the exact route, and on the tensor cores the passes
    the tensor-core kernels take."""
    out = {("ffma", "fwd"): exact_conv(c, 0), ("ffma", "dgrad"): exact_conv(c, 1), ("ffma", "wgrad"): exact_wgrad(c)[0]}
    for direction, p in ((0, "fwd"), (1, "dgrad")):
        t = tc_conv(c, direction)
        if t is not None:
            out[("tc", p)] = {f"conv_tc_kernel<{t[1]}, false, false>"}
    w = tc_wgrad(c)
    if w is not None:
        out[("tc", "wgrad")] = w[0]
    return out


WATCHED = ("conv_core_kernel", "conv_wgrad_kernel", "split_sum_kernel", "split_sum_wide_kernel", "colsum_kernel",
           "conv_tc_kernel", "wgrad_tc_kernel", "wgrad_tma_kernel", "wgrad_reduce_kernel", "wgrad_reduce_wide_kernel",
           "weight_prepare_kernel", "weight_prepare_tiled_kernel", "weight_grad_kernel", "weight_grad_tiled_kernel")


def _instances(mangled):
    """Mangled kernel names -> the set of watched instances among them, e.g. 'conv_core_kernel<1, 16, 4, false, false>'."""
    out = set()
    for n in mangled:
        m = re.match(r"_ZN2kt(\d+)", n)
        if not m:
            continue
        base = n[m.end():m.end() + int(m.group(1))]
        if base not in WATCHED:
            continue
        rest = n[m.end() + len(base):]
        if rest.startswith("I"):
            args = re.findall(r"L([ib])(\d+)E", re.match(r"I((?:L[ib]\d+E)+)E", rest).group(1))
            base += "<" + ", ".join({"0": "false", "1": "true"}[v] if t == "b" else v for t, v in args) + ">"
            assert _mangled(base) in n, (base, n)
        out.add(base)
    return out


# ------------------------------------------------------------------------------------------------
# float64 reference
# ------------------------------------------------------------------------------------------------


def _cf(t, period):
    """kernel layout [B][T][nsub][C] -> the reference's channels-first (B, C, T[, nsub])"""
    return t.permute(0, 3, 1, 2) if period else t.permute(0, 2, 1)


def _cl(t, period):
    return t.permute(0, 2, 3, 1) if period else t.permute(0, 2, 1)


def _lrelu(v, slope):
    return torch.where(v > 0, v, v * slope)


def _dact(v, act, slope):
    """derivative of activation act at its output (or, for the input LeakyReLU, its input) v"""
    if act == KT_ACT_LRELU:
        return torch.where(v > 0, torch.ones((), dtype=v.dtype), torch.full((), slope, dtype=v.dtype))
    if act == KT_ACT_TANH:
        return 1 - v * v
    return torch.ones_like(v)


def kernel_layouts(w, transposed, groups):
    """Reference-layout weight (d0, d1, k) -> (w_fwd, w_bwd) flat, the kernel layouts of kantts_b200.h: a conv
    (c_out, c_in / g, k) -> [k][c_in / g][c_out] and [k][c_out / g][c_in]; a transposed conv (c_in, c_out, k) ->
    [k][c_in][c_out] and [k][c_out][c_in]."""
    if transposed:
        fwd, bwd = w.permute(2, 0, 1), w.permute(2, 1, 0)
    else:
        d0, d1, k = w.shape
        fwd = w.permute(2, 1, 0)
        bwd = w.reshape(groups, d0 // groups, d1, k).permute(3, 1, 0, 2).reshape(k, d0 // groups, groups * d1)
    return fwd.contiguous().flatten(), bwd.contiguous().flatten()


def reference(c, x, w, bias, resid, dy):
    """-> {output: (float64 value, scale)} of case c, plus y_src: the fp32 act_out(pre-activation) the backward kernels get
    as the source of act_out'.  dw in the kernel layout of kt_conv1d_bwd_weight."""
    from oracle import convref
    s, P = c.spec, c.period
    geo = dict(stride=s.stride, dilation=s.dilation, pad_left=s.pad_left, pad_right=s.pad_right, groups=s.groups,
               transposed=s.transposed, upsample=s.upsample, crop=s.crop)
    xd = x.to(F64)
    xa = _lrelu(xd, s.act_in_slope) if s.act_in == KT_ACT_LRELU else xd
    W, b = w.to(F64), bias.to(F64)
    # the linear conv on the values and on their magnitudes; autograd gives its transposes
    a = _cf(xa, P).detach().requires_grad_(True)
    Wv = W.clone().requires_grad_(True)
    z = convref.conv_layer(a, Wv, **geo)
    aa = _cf(xa.abs(), P).detach().requires_grad_(True)
    Wa = W.abs().requires_grad_(True)
    za = convref.conv_layer(aa, Wa, **geo)
    pre = _cl(z.detach(), P) + b
    if s.act_out == KT_ACT_LRELU:
        act = _lrelu(pre, s.act_out_slope)
    elif s.act_out == KT_ACT_TANH:
        act = torch.tanh(pre)
    else:
        act = pre
    r = resid.to(F64) if resid is not None else torch.zeros((), dtype=F64)
    out = {"y": (act + r, _cl(za.detach(), P) + b.abs() + r.abs())}
    y_src = act.float().contiguous()
    dpre = dy.to(F64) * _dact(y_src.to(F64), s.act_out, s.act_out_slope)
    z.backward(_cf(dpre, P))
    za.backward(_cf(dpre.abs(), P))
    din = _dact(xd, s.act_in, s.act_in_slope)
    out["dx"] = (din * _cl(a.grad, P), din.abs() * _cl(aa.grad, P))
    k = int(s.transposed)
    out["dw"] = (kernel_layouts(Wv.grad, s.transposed, s.groups)[k], kernel_layouts(Wa.grad, s.transposed, s.groups)[k])
    rows = tuple(range(dpre.dim() - 1))
    out["db"] = (dpre.sum(rows), dpre.abs().sum(rows))
    return out, y_src


def _inputs(c):
    s = c.spec
    g = torch.Generator().manual_seed(zlib.crc32(c.name.encode()))
    lead = (c.B, c.T, c.period) if c.period else (c.B, c.T)
    t_out = s.t_out(c.T)
    out_lead = (c.B, t_out, c.period) if c.period else (c.B, t_out)
    x = torch.randn(*lead, s.c_in, generator=g)
    w_shape = (s.c_in, s.c_out, s.kernel) if s.transposed else (s.c_out, s.c_in // s.groups, s.kernel)
    w = torch.randn(w_shape, generator=g) / math.sqrt(s.kernel * s.c_in / s.groups)
    bias = 0.3 * torch.randn(s.c_out, generator=g)
    resid = torch.randn(*out_lead, s.c_out, generator=g) if c.resid else None
    dy = torch.randn(*out_lead, s.c_out, generator=g)
    return x, w, bias, resid, dy


# ------------------------------------------------------------------------------------------------
# GPU test of the conv passes
# ------------------------------------------------------------------------------------------------


def _check(where, route, kind, got, want, scale, l2_bound):
    err = (got.cpu().to(F64) - want).abs()
    ratio = err / scale.clamp_min(1e-300)
    worst = int(ratio.flatten().argmax())
    idx = tuple(int(i) for i in torch.unravel_index(torch.tensor(worst), ratio.shape))
    l2 = rel_l2(got.cpu(), want)
    print(f"  {where}: elem {float(ratio.max()):.3e} at {idx} rel_l2 {l2:.3e}")
    bad = err > ELEM_BOUND[route][kind] * scale
    assert not bool(bad.any()), (where, "elements over the bound", int(bad.sum()), "first at",
                                 [tuple(int(v) for v in i) for i in bad.nonzero()[:8]])
    assert l2 <= l2_bound, (where, l2)


def _bits(t):
    return t.view(torch.int32)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_conv_pass_matches_float64(name):
    c = CASES[name]
    s = c.spec
    x, w, bias, resid, dy = _inputs(c)
    ref, y_src = reference(c, x, w, bias, resid, dy)
    w_fwd, w_bwd = (t.to(DEV) for t in kernel_layouts(w, s.transposed, s.groups))
    xd, bd, dyd, ysd = x.to(DEV), bias.to(DEV), dy.to(DEV), y_src.to(DEV)
    rd = None if resid is None else resid.to(DEV)
    d = c.desc()
    lib = _lib()
    t_out = s.t_out(c.T)
    y_shape = (c.B, t_out, c.period, s.c_out) if c.period else (c.B, t_out, s.c_out)

    def image(dd, direction, src):
        img = torch.empty(int(lib.kt_conv1d_tc_image_bytes(ctypes.byref(dd), direction)) // 2, dtype=torch.bfloat16,
                          device=DEV)
        _call("kt_weight_pack_tc", ctypes.byref(dd), direction, _ptr(src), _ptr(img, True))
        return img

    def workspace(n):
        return torch.empty(int(n), device=DEV) if n else None

    # (route, pass) -> (launch, outputs): launch() writes the outputs
    runs = {}
    y, dx = torch.empty(y_shape, device=DEV), torch.empty_like(xd)
    dw, db = torch.empty(s.w_numel, device=DEV), torch.empty(s.c_out, device=DEV)
    runs[("ffma", "fwd")] = (lambda: _call("kt_conv1d_fwd", ctypes.byref(d), _ptr(xd), _ptr(w_fwd), _ptr(bd), _ptr(rd),
                                           _ptr(y)), {"y": y})
    runs[("ffma", "dgrad")] = (lambda: _call("kt_conv1d_bwd_data", ctypes.byref(d), _ptr(dyd), _ptr(ysd), _ptr(w_bwd),
                                             _ptr(xd), _ptr(dx)), {"dx": dx})
    runs[("ffma", "wgrad")] = (lambda: _call("kt_conv1d_bwd_weight", ctypes.byref(d), _ptr(xd), _ptr(dyd), _ptr(ysd),
                                             _ptr(dw), _ptr(db)), {"dw": dw, "db": db})
    expected = passes(c)
    if ("tc", "fwd") in expected:
        img0, ws0, yt = image(d, 0, w_fwd), workspace(lib.kt_conv1d_tc_workspace(ctypes.byref(d), 0)), torch.empty_like(y)
        runs[("tc", "fwd")] = (lambda: _call("kt_conv1d_fwd_tc", ctypes.byref(d), _ptr(xd), _ptr(img0, True), _ptr(bd),
                                             _ptr(rd), _ptr(yt), _ptr(ws0), 0 if ws0 is None else ws0.numel()), {"y": yt})
    if ("tc", "dgrad") in expected:
        d1, _, _ = tc_conv(c, 1)
        img1, ws1, dxt = image(d1, 1, w_bwd), workspace(lib.kt_conv1d_tc_workspace(ctypes.byref(d1), 1)), torch.empty_like(dx)
        nws1 = 0 if ws1 is None else ws1.numel()
        if s.upsample > 1:
            dxu = torch.empty((c.B, c.T * s.upsample, s.c_in), device=DEV)

            def tc_dgrad():
                _call("kt_conv1d_bwd_data_tc", ctypes.byref(d1), _ptr(dyd), _ptr(ysd), _ptr(img1, True), None, _ptr(dxu),
                      _ptr(ws1), nws1)
                _call("kt_upsample_grad_reduce", _ptr(dxu), _ptr(xd), s.act_in, s.act_in_slope, _ptr(dxt), c.B * c.T,
                      s.upsample, s.c_in)
        else:
            def tc_dgrad():
                _call("kt_conv1d_bwd_data_tc", ctypes.byref(d1), _ptr(dyd), _ptr(ysd), _ptr(img1, True), _ptr(xd),
                      _ptr(dxt), _ptr(ws1), nws1)
        runs[("tc", "dgrad")] = (tc_dgrad, {"dx": dxt})
    if ("tc", "wgrad") in expected:
        wsw = workspace(lib.kt_conv1d_bwd_weight_tc_workspace(ctypes.byref(d)))
        dwt, dbt = torch.empty_like(dw), torch.empty_like(db)
        runs[("tc", "wgrad")] = (lambda: _call("kt_conv1d_bwd_weight_tc", ctypes.byref(d), _ptr(xd), _ptr(dyd), _ptr(ysd),
                                               _ptr(dwt), _ptr(dbt), _ptr(wsw), wsw.numel()), {"dw": dwt, "db": dbt})
    assert set(runs) == set(expected), (sorted(runs), sorted(expected))

    for (route, p), (launch, outs) in runs.items():
        for t in outs.values():
            t.fill_(float("nan"))
        launch()
        torch.cuda.synchronize()
        got = {k: t.clone() for k, t in outs.items()}
        launched = _instances(_launched_kernels(launch))
        print(f"conv_arms {name} {route} {p}: {' '.join(sorted(launched))}")
        assert launched == expected[(route, p)], (route, p, sorted(launched), sorted(expected[(route, p)]))
        if p == "wgrad":
            # the same bits again: the weight-gradient paths sum in a fixed order
            for t in outs.values():
                t.fill_(float("nan"))
            launch()
            torch.cuda.synchronize()
            for k, t in outs.items():
                assert torch.equal(_bits(t), _bits(got[k])), (route, k, "differs between two runs")
        for k, t in got.items():
            kind = {"y": "conv", "dx": "conv", "dw": "wgrad", "db": "bias"}[k]
            want, scale = ref[k]
            _check(f"{route} {p} {k}", route, kind, t.view(want.shape), want, scale, L2_BOUND[route][k != "y"])


# ------------------------------------------------------------------------------------------------
# weight norm
# ------------------------------------------------------------------------------------------------

# (d0, d1, k, transposed, groups): the small layers take one CTA per row, those of >= 256 K elements the tiled kernels --
# d0 = 203 / 204 rows (row blocks of 8 with a ragged last one), d1 = 260 (slices of 64: a ragged last slice of 4, and
# rows of 1300 elements, more than one 1024-float tile)
WEIGHT_LAYOUTS = {
    "dense": (37, 19, 7, False, 1),
    "grouped": (24, 5, 3, False, 4),
    "transposed": (13, 22, 4, True, 1),
    "dense_tiled": (203, 260, 5, False, 1),
    "grouped_tiled": (204, 260, 5, False, 4),
    "transposed_tiled": (203, 260, 5, True, 1),
}
INV_SIGMA = 0.37


def weight_tiled(d0, d1, k):
    """weight_tiled_plan: the tiled kernels take layers of >= 256 K elements with rows of >= 256 elements."""
    return d0 * d1 * k >= 262144 and d1 * k >= 256 and k <= 1024


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1], ids=["plain", "weight_norm"])
@pytest.mark.parametrize("layout", list(WEIGHT_LAYOUTS))
def test_weight_norm_matches_float64(layout, mode):
    """kt_weight_prepare (mode 1: w = g v / ||v|| per row; mode 0: w = v * inv_sigma) writes the same fp32 value at the
    two kernel-layout positions of every reference element, within the float64 bound; kt_weight_grad's dv / dg match
    float64; kt_weight_grad_accum adds exactly kt_weight_grad's result (and the bias hand-over) to its buffers."""
    d0, d1, k, tr, groups = WEIGHT_LAYOUTS[layout]
    tiled = weight_tiled(d0, d1, k)
    assert tiled == layout.endswith("_tiled")
    gen = torch.Generator().manual_seed(zlib.crc32(layout.encode()) + mode)
    v = torch.randn(d0, d1, k, generator=gen)
    g = 0.5 + torch.rand(d0, generator=gen)
    dW = torch.randn(d0, d1, k, generator=gen)
    nb = 37
    vd, gd = v.to(DEV), g.to(DEV) if mode else None
    inv = None if mode else torch.tensor([INV_SIGMA], device=DEV)
    n = d0 * d1 * k
    w_fwd, w_bwd, w_ref = (torch.full((n,), float("nan"), device=DEV) for _ in range(3))
    norm = torch.full((d0,), float("nan"), device=DEV) if mode else None

    def prepare():
        _call("kt_weight_prepare", _ptr(vd), _ptr(gd), _ptr(inv), mode, d0, d1, k, int(tr), groups, _ptr(w_fwd),
              _ptr(w_bwd), _ptr(norm), _ptr(w_ref))

    prepare()
    torch.cuda.synchronize()
    assert _instances(_launched_kernels(prepare)) == {"weight_prepare_tiled_kernel" if tiled else "weight_prepare_kernel"}
    wr = w_ref.cpu().view(d0, d1, k)
    lf, lb = kernel_layouts(wr, tr, groups)
    assert torch.equal(_bits(w_fwd.cpu()), _bits(lf)) and torch.equal(_bits(w_bwd.cpu()), _bits(lb)), "layout mapping"
    v64 = v.to(F64)
    nrm = v64.flatten(1).norm(dim=1)[:, None, None]
    if mode:
        want, scale = g.to(F64)[:, None, None] * v64 / nrm, g.to(F64)[:, None, None] * v64.abs() / nrm
        err = ((norm.cpu().to(F64) - nrm.flatten()).abs() / nrm.flatten()).max()
        print(f"weight {layout} norm rel {float(err):.3e}")
        assert float(err) <= WEIGHT_BOUND
    else:
        want = v64 * torch.tensor(INV_SIGMA, dtype=torch.float32).to(F64)
        scale = want.abs()
    ratio = float(((wr.to(F64) - want).abs() / scale.clamp_min(1e-300)).max())
    print(f"weight {layout} mode {mode} prepare elem {ratio:.3e}")
    assert bool(((wr.to(F64) - want).abs() <= WEIGHT_BOUND * scale).all()), ratio

    # backward: dw in the layout kt_conv1d_bwd_weight writes (w_fwd for a conv, w_bwd for a transposed conv)
    dwk = kernel_layouts(dW, tr, groups)[int(tr)].to(DEV)
    dv, dg = torch.full((d0, d1, k), float("nan"), device=DEV), torch.full((d0,), float("nan"), device=DEV)
    dgp = dg if mode else None

    def grad():
        _call("kt_weight_grad", _ptr(dwk), _ptr(vd), _ptr(gd), _ptr(norm), _ptr(inv), mode, d0, d1, k, int(tr), groups,
              _ptr(dv), _ptr(dgp))

    grad()
    torch.cuda.synchronize()
    assert _instances(_launched_kernels(grad)) == {"weight_grad_tiled_kernel" if tiled else "weight_grad_kernel"}
    dW64 = dW.to(F64)
    if mode:
        g64 = g.to(F64)[:, None, None]
        dot = (dW64 * v64).flatten(1).sum(1)[:, None, None]
        adot = (dW64.abs() * v64.abs()).flatten(1).sum(1)[:, None, None]
        want_dv = g64 / nrm * dW64 - g64 * dot / nrm ** 3 * v64
        scale_dv = g64.abs() / nrm * dW64.abs() + g64.abs() * adot / nrm ** 3 * v64.abs()
        rg = float(((dg.cpu().to(F64) - (dot / nrm).flatten()).abs() / (adot / nrm).flatten()).max())
        print(f"weight {layout} dg elem {rg:.3e}")
        assert rg <= WEIGHT_BOUND
    else:
        want_dv = dW64 * torch.tensor(INV_SIGMA, dtype=torch.float32).to(F64)
        scale_dv = want_dv.abs()
    rv = float(((dv.cpu().to(F64) - want_dv).abs() / scale_dv.clamp_min(1e-300)).max())
    print(f"weight {layout} mode {mode} dv elem {rv:.3e}")
    assert bool(((dv.cpu().to(F64) - want_dv).abs() <= WEIGHT_BOUND * scale_dv).all()), rv

    # the accumulating form: exactly the fp32 sums buffer + kt_weight_grad's result, and the bias hand-over
    dv0, dg0 = torch.randn(d0, d1, k, generator=gen).to(DEV), torch.randn(d0, generator=gen).to(DEV)
    bsrc, bdst0 = torch.randn(nb, generator=gen).to(DEV), torch.randn(nb, generator=gen).to(DEV)
    dva, dga, bdst = dv0.clone(), dg0.clone(), bdst0.clone()
    _call("kt_weight_grad_accum", _ptr(dwk), _ptr(vd), _ptr(gd), _ptr(norm), _ptr(inv), mode, d0, d1, k, int(tr), groups,
          _ptr(dva), _ptr(dga if mode else None), _ptr(bsrc), _ptr(bdst), nb)
    torch.cuda.synchronize()
    assert torch.equal(_bits(dva), _bits(dv0 + dv)), "dv += kt_weight_grad"
    if mode:
        assert torch.equal(_bits(dga), _bits(dg0 + dg)), "dg += kt_weight_grad"
    assert torch.equal(_bits(bdst), _bits(bdst0 + bsrc)), "dbias hand-over"
