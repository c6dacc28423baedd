"""Without a GPU: the case table of test_gpu_conv_arms.py reaches every training conv kernel instance and every branch of
its dispatch, by the same mirrors of the host dispatch and the same plan calls (kt_debug_conv_tc_plan /
kt_debug_wgrad_plan plan for an H100 here) the GPU test pins each case with.  A threshold change that moves a case off
its instance fails here; a mirror that drifts from the C++ dispatch fails the GPU test's captured kernel names.  Also
checks the float64 reference of the GPU test against autograd through the whole layer."""
import pytest
import torch

import test_gpu_conv_arms as arms

F64 = torch.float64


def _b(v):
    return "true" if v else "false"


def test_cases_reach_every_conv_instance():
    cases = list(arms.CASES.values())
    assert not any(c.spec.c_in == 1 for c in cases)          # c_in = 1 layers take the thin kernels (thin.cu)
    every = [arms.passes(c) for c in cases]

    # exact route: all 18 conv_core_kernel instances over the forward and data-gradient phases
    core = set().union(*(p[("ffma", "fwd")] | p[("ffma", "dgrad")] for p in every))
    want = {f"conv_core_kernel<{rn}, {rm}, {kc}, false, false>" for rn in (1, 2, 4) for rm in (4, 8, 16) for kc in (4, 16)}
    assert core == want, sorted(want - core)

    # exact route: all 12 conv_wgrad_kernel instances, and the three ways the splits of dw are summed
    wg = {k for p in every for k in p[("ffma", "wgrad")] if k.startswith("conv_wgrad_kernel")}
    want = {f"conv_wgrad_kernel<{rn}, {rma}, {_b(sm)}>" for rn in (1, 2, 4) for rma, sm in ((4, True), (8, True),
                                                                                               (4, False), (8, False))}
    assert wg == want, sorted(want - wg)
    sums = set()
    for c in cases:
        _, ns = arms.exact_wgrad(c)
        sums.add("atomics into dw" if ns == 1 else arms._split_sum(c.spec.w_numel, ns))
    assert sums == {"atomics into dw", "split_sum_kernel", "split_sum_wide_kernel"}, sums

    # the bias gradient's column sums of a plain dy, of dy * LReLU'(y) and of dy * tanh'(y)
    assert {c.spec.act_out for c in cases} == {arms.KT_ACT_NONE, arms.KT_ACT_LRELU, arms.KT_ACT_TANH}
    assert all("colsum_kernel" in p[("ffma", "wgrad")] for p in every)

    # tensor cores, forward and data gradient: all three routes; route 1 from each cause alone
    routes = {k for p in every for r, q in p if r == "tc" and q != "wgrad" for k in p[(r, q)]}
    assert routes == {f"conv_tc_kernel<{r}, false, false>" for r in (0, 1, 2)}, routes
    causes = {t[2] for c in cases for direction in (0, 1) if (t := arms.tc_conv(c, direction)) is not None}
    for cause in ("nsub", "upsample", "tanh", "alignment"):
        assert (cause,) in causes, (cause, causes)

    # tensor cores, weight gradient: both kernels at both N tiles; dw written directly by each, and both branches of
    # each split-K reduce
    kernels, outcomes = set(), set()
    for c in cases:
        w = arms.tc_wgrad(c)
        if w is None:
            continue
        names, ns, branch = w
        kern = next(k for k in names if k.startswith("wgrad_t"))
        kernels.add(kern)
        if ns == 1:
            outcomes.add((kern.split("<")[0], "direct"))
        else:
            outcomes.add(("wgrad_reduce_wide_kernel" if ns >= 16 else "wgrad_reduce_kernel", branch))
    assert kernels == {f"wgrad_{k}_kernel<{nt}>" for k in ("tc", "tma") for nt in (64, 128)}, kernels
    assert outcomes == {("wgrad_tc_kernel", "direct"), ("wgrad_tma_kernel", "direct"),
                        ("wgrad_reduce_kernel", "float4"), ("wgrad_reduce_kernel", "scalar"),
                        ("wgrad_reduce_wide_kernel", "float4"), ("wgrad_reduce_wide_kernel", "scalar")}, outcomes


def test_cases_hold_the_edges():
    cases = list(arms.CASES.values())
    t_outs = [c.spec.t_out(c.T) for c in cases]
    assert any(t % 128 and t % 32 for t in t_outs) and any(c.T % 128 and c.T % 32 for c in cases)
    assert 1 in t_outs
    # phases no tap reaches (scatter_phases' placeholder tap): a transposed forward and a strided data gradient
    def empty_phase(s, direction):
        if (direction == 0) != bool(s.transposed):
            return False
        return any(all((r + s.pad_left - j * s.dilation) % s.stride for j in range(s.kernel)) for r in range(s.stride))
    assert any(empty_phase(c.spec, 0) for c in cases) and any(empty_phase(c.spec, 1) for c in cases)
    chans = {ch for c in cases for ch in (c.spec.c_in, c.spec.c_out)}
    assert any(ch % 2 for ch in chans) and chans & {5, 6, 7, 8}
    assert any(c.spec.groups > 1 for c in cases) and any(c.period for c in cases)
    assert any(c.spec.upsample > 1 for c in cases) and any(c.spec.dilation > 1 for c in cases)


def _tiled_plan(d0, d1, k):
    """weight_tiled_plan: (row blocks, b slices, b per slice)"""
    nblk = -(-d0 // 8)
    nsl = max(1, min(max(1, d1 // 32), -(-296 // nblk)))
    b_slice = (-(-d1 // nsl) + 31) & ~31
    return nblk, -(-d1 // b_slice), b_slice


def test_weight_layouts_reach_both_kernels():
    """Dense, grouped and transposed layouts each on the per-row and the tiled kernels; the tiled ones with a ragged last
    row block and more than one b slice, the last one ragged."""
    seen = set()
    for name, (d0, d1, k, tr, groups) in arms.WEIGHT_LAYOUTS.items():
        tiled = arms.weight_tiled(d0, d1, k)
        seen.add(("transposed" if tr else "grouped" if groups > 1 else "dense", tiled))
        if tiled:
            _, nsl, b_slice = _tiled_plan(d0, d1, k)
            assert d0 % 8 and nsl > 1 and d1 % b_slice, name
            assert d1 * k > 1024, name                       # a row spans more than one shared-memory tile
    assert seen == {(lay, t) for lay in ("dense", "grouped", "transposed") for t in (False, True)}


def test_kernel_layouts_match_the_documented_index_maps():
    d0, d1, k, g = 6, 3, 2, 2
    w = torch.arange(d0 * d1 * k, dtype=F64).view(d0, d1, k)
    fwd, bwd = arms.kernel_layouts(w, False, g)
    cout_g, cin = d0 // g, d1 * g
    for co in range(d0):
        for ci in range(d1):
            for j in range(k):
                assert fwd[(j * d1 + ci) * d0 + co] == w[co, ci, j]
                assert bwd[(j * cout_g + co % cout_g) * cin + (co // cout_g) * d1 + ci] == w[co, ci, j]
    fwd, bwd = arms.kernel_layouts(w, True, 1)                 # (c_in, c_out, k)
    for a in range(d0):
        for b in range(d1):
            for j in range(k):
                assert fwd[(j * d0 + a) * d1 + b] == w[a, b, j] and bwd[(j * d1 + b) * d0 + a] == w[a, b, j]


@pytest.mark.parametrize("name", [n for n, c in arms.CASES.items() if c.B * c.T * c.nsub <= 2000])
def test_reference_matches_autograd_of_the_whole_layer(name):
    """The float64 reference (linear conv + its autograd transposes, activation derivatives applied around them) equals
    autograd through oracle.convref.conv_layer with its activations, bias and residual."""
    from oracle import convref
    c = arms.CASES[name]
    s = c.spec
    x, w, bias, resid, dy = arms._inputs(c)
    ref, y_src = arms.reference(c, x, w, bias, resid, dy)
    P = c.period
    act_out = None if s.act_out == arms.KT_ACT_NONE else ("tanh" if s.act_out == arms.KT_ACT_TANH else s.act_out_slope)
    xd = arms._cf(x.to(F64), P).detach().requires_grad_(True)
    W = w.to(F64).requires_grad_(True)
    b = bias.to(F64).requires_grad_(True)
    y = convref.conv_layer(xd, W, b, None if resid is None else arms._cf(resid.to(F64), P), stride=s.stride,
                           dilation=s.dilation, pad_left=s.pad_left, pad_right=s.pad_right, groups=s.groups,
                           transposed=bool(s.transposed), upsample=s.upsample, crop=s.crop,
                           act_in=s.act_in_slope if s.act_in else None, act_out=act_out)
    y.backward(arms._cf(dy.to(F64), P))
    tol = dict(rtol=1e-6, atol=1e-6)      # act_out' from the fp32 y_src
    assert torch.allclose(ref["y"][0], arms._cl(y.detach(), P), rtol=1e-12, atol=1e-12)
    assert torch.allclose(ref["dx"][0], arms._cl(xd.grad, P), **tol)
    assert torch.allclose(ref["dw"][0], arms.kernel_layouts(W.grad, s.transposed, s.groups)[int(s.transposed)], **tol)
    assert torch.allclose(ref["db"][0], b.grad, **tol)
    for k, (v, sc) in ref.items():
        assert bool((sc >= v.abs() - 1e-9).all()), k
