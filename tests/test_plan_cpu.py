"""CPU: host-side planning logic of the C ABI (no kernel is launched): tensor-core tile plans, packed-weight image sizes,
split-K workspaces and the dispatch rules added for thin / grouped / waveform-input layers."""
import ctypes

import pytest

from kantts_b200 import _lib, ops
from kantts_b200._lib import KT_ACT_LRELU, KT_PATH_AUTO, KT_PATH_FFMA, KT_PATH_TC


@pytest.fixture(scope="module")
def lib():
    return _lib.load()


def _desc(B, t_in, nsub=1, **kw):
    path = kw.pop("path", KT_PATH_AUTO)
    spec = ops.ConvSpec(path=path, **kw)
    return spec, spec.desc(B, nsub, t_in)


def test_dense_layer_tiles(lib):
    # 1024 -> 1024 k5 (period discriminator): N tiles of 128 (register accumulators), 16 K chunks of 64
    _, d = _desc(32, 34, nsub=3, c_in=1024, c_out=1024, kernel=5, pad_left=2, pad_right=2)
    assert lib.kt_conv1d_tc_plan(ctypes.byref(d), 0) == 128 and lib.kt_conv1d_tc_plan(ctypes.byref(d), 1) == 128
    # image = taps x K chunks x N tiles x (hi + lo) x NT x 64 bf16
    assert lib.kt_conv1d_tc_image_bytes(ctypes.byref(d), 0) == 5 * 16 * 8 * 2 * 128 * 64 * 2
    # generator resblock conv: one N tile of the layer's width
    _, d = _desc(16, 8192, c_in=32, c_out=32, kernel=7, pad_left=6)
    assert lib.kt_conv1d_tc_plan(ctypes.byref(d), 0) == 32


def test_thin_groups_share_block_diagonal_tiles(lib):
    # 128 -> 256, 16 groups (8 -> 16 channels per group): 8 groups per tile = K 64 x N 128, 2 N tiles
    _, d = _desc(16, 2048, c_in=128, c_out=256, kernel=41, stride=4, pad_left=20, pad_right=20, groups=16)
    assert lib.kt_conv1d_tc_plan(ctypes.byref(d), 0) == 128
    assert lib.kt_conv1d_tc_image_bytes(ctypes.byref(d), 0) == 41 * 1 * 2 * 2 * 128 * 64 * 2
    # its data gradient contracts 16 channels per group and produces 8: 4 groups per tile = K 64 x N 32
    assert lib.kt_conv1d_tc_plan(ctypes.byref(d), 1) == 32
    # 64-channel groups already fill a K chunk: one group per tile
    _, d = _desc(16, 32, c_in=1024, c_out=1024, kernel=41, pad_left=20, pad_right=20, groups=16)
    assert lib.kt_conv1d_tc_plan(ctypes.byref(d), 0) == 64


def test_waveform_input_layers_leave_the_tensor_path(lib):
    kw = dict(c_in=1, c_out=32, kernel=5, stride=3, pad_left=2, pad_right=2, act_out=1, act_out_slope=0.1)
    _, d = _desc(32, 2731, nsub=3, **kw)
    assert lib.kt_conv1d_tc_plan(ctypes.byref(d), 0) == 0            # forward: FIR kernel (thin.cu)
    assert lib.kt_conv1d_bwd_weight_tc_workspace(ctypes.byref(d)) == 0
    assert lib.kt_conv1d_tc_plan(ctypes.byref(d), 1) > 0             # its data gradient stays on the tensor cores
    _, d = _desc(32, 2731, nsub=3, path=KT_PATH_TC, **kw)            # explicitly requested: still available
    assert lib.kt_conv1d_tc_plan(ctypes.byref(d), 0) > 0 and lib.kt_conv1d_bwd_weight_tc_workspace(ctypes.byref(d)) > 0


def test_upsampled_conv_data_gradient_plan(lib):
    spec, d = _desc(16, 32, c_in=512, c_out=256, kernel=7, pad_left=6, upsample=8, act_in=1, act_in_slope=0.1)
    assert lib.kt_conv1d_tc_plan(ctypes.byref(d), 0) > 0
    assert lib.kt_conv1d_tc_plan(ctypes.byref(d), 1) == 0            # not directly ...
    p = spec.plan(16, 1, 32)
    d2 = p.d_bwd
    assert p.up_bwd and d2.t_in == 32 * 8 and d2.t_out == d.t_out and d2.act_in == 0 and d2.upsample == 1
    assert lib.kt_conv1d_tc_plan(ctypes.byref(d2), 1) == p.nt_bwd > 0   # ... but as the plain conv over the up-sampled rows
    # a layer that insists on the tensor cores gets no detour: its forward runs, its data gradient raises when it runs
    spec = ops.ConvSpec(c_in=512, c_out=256, kernel=7, pad_left=6, upsample=8, act_in=1, act_in_slope=0.1, path=KT_PATH_TC)
    p = spec.plan(16, 1, 32)
    assert p.tile(0) > 0 and not p.up_bwd
    with pytest.raises(RuntimeError, match="cannot run on the tensor-core path"):
        p.tile(1)
    ops.set_force_ffma(True)
    try:
        assert _no_tensor_routes(spec.plan(16, 1, 32))              # set_force_ffma overrides KT_PATH_TC
    finally:
        ops.set_force_ffma(False)


def test_split_k_workspace_is_whole_slices_of_the_gradient(lib):
    for kw, B, T, nsub in ((dict(c_in=1024, c_out=1024, kernel=5, pad_left=2, pad_right=2), 32, 34, 3),
                           (dict(c_in=32, c_out=32, kernel=11, pad_left=10), 16, 8192, 1),
                           (dict(c_in=128, c_out=256, kernel=41, stride=4, pad_left=20, pad_right=20, groups=16), 16, 2048, 1)):
        spec, d = _desc(B, T, nsub=nsub, **kw)
        ws = lib.kt_conv1d_bwd_weight_tc_workspace(ctypes.byref(d))
        # one slice of the weight gradient per split (the bias gradient is the column-sum kernel's)
        out = (ctypes.c_int32 * 12)()
        assert lib.kt_debug_wgrad_plan(ctypes.byref(d), out) == 0
        if out[1] and ws % spec.w_numel:
            # TMA variant (a driver is present): the slices, padded to 64 floats, then the hi / lo bf16 operand planes of
            # both operands (one float per element each, padded to 64 floats)
            r64 = lambda n: (n + 63) & ~63
            planes = r64(d.batch * d.t_in * d.nsub * d.c_in) + r64(d.batch * d.t_out * d.nsub * d.c_out)
            assert ws - planes == r64(out[7] * spec.w_numel), (ws, planes, out[7])
            nsplit = out[7]
        else:
            assert ws > 0 and ws % spec.w_numel == 0
            nsplit = ws // spec.w_numel
        assert 1 <= nsplit <= 296


def _resblock_specs(C, k, d, causal):
    p1 = (k - 1) * d if causal else (k - 1) * d // 2
    p2 = (k - 1) if causal else (k - 1) // 2
    s1 = ops.ConvSpec(c_in=C, c_out=C, kernel=k, dilation=d, pad_left=p1, pad_right=(k - 1) * d - p1, act_in=KT_ACT_LRELU, act_in_slope=0.1)
    s2 = ops.ConvSpec(c_in=C, c_out=C, kernel=k, dilation=1, pad_left=p2, pad_right=(k - 1) - p2, act_in=KT_ACT_LRELU, act_in_slope=0.1)
    return s1, s2


def test_resblock_plan_fuses_the_shipped_pairs_and_rejects_boxes_over_256_rows(lib):
    """kt_resblock_plan (geometry only, no GPU): every pair of the fused-resblock parity tests and of the shipped generator
    stages (C = 32 / 64, k = 3 / 7 / 11, dilation 1 / 3 / 5) runs on the fused kernel.  Its x tile is one TMA box of
    ceil8(128 + (k - 1) * dilation) (+ dilation when C = 32) rows, at most 256: C = 32, k = 15, dilation 11 needs 282, so
    that pair runs as two conv launches."""
    from test_gpu_parity import RB_CASES
    shapes = [(C, k, d, causal, B, T) for C, k, d, causal, B, T in RB_CASES.values()]
    shapes += [(C, k, d, causal, 16, 8192) for C in (32, 64) for k in (3, 7, 11) for d in (1, 3, 5) for causal in (True, False)]
    for C, k, d, causal, B, T in shapes:
        s1, s2 = _resblock_specs(C, k, d, causal)
        rd = ops.resblock_desc(s1, s2, B, T)
        assert rd is not None and lib.kt_resblock_plan(ctypes.byref(rd)) == 1, (C, k, d, causal, B, T)
        assert lib.kt_resblock_image_bytes(ctypes.byref(rd)) > 0
    s1, s2 = _resblock_specs(32, 15, 11, True)
    assert ops.resblock_desc(s1, s2, 2, 1000) is None


def test_grad_items_context_restores_state():
    assert ops._grad_items is None
    with ops.grad_items(4):
        assert ops._grad_items == 4
        with ops.grad_items(2):
            assert ops._grad_items == 2
        assert ops._grad_items == 4
    assert ops._grad_items is None


def _no_tensor_routes(p):
    return p.tile(0) == p.tile(1) == p.wg_ws == 0 and not p.up_bwd and p.d_bwd is p.d


def test_ffma_path_has_no_tensor_plan(lib):
    for kw in (dict(c_in=64, c_out=64, kernel=3, pad_left=2),
               dict(c_in=512, c_out=256, kernel=7, pad_left=6, upsample=8, act_in=1, act_in_slope=0.1)):
        assert _no_tensor_routes(ops.ConvSpec(path=KT_PATH_FFMA, **kw).plan(2, 1, 100)), kw


def test_plan_cache_follows_the_exact_path_flag(lib):
    spec = ops.ConvSpec(c_in=64, c_out=64, kernel=3, pad_left=2)
    p = spec.plan(2, 1, 100)
    assert p.tile(0) > 0 and p.tile(1) > 0 and p.wg_ws > 0
    s1, s2 = _resblock_specs(32, 7, 3, True)
    assert ops.resblock_desc(s1, s2, 16, 8192) is not None
    ops.set_force_ffma(True)
    try:
        assert _no_tensor_routes(spec.plan(2, 1, 100))
        assert ops.resblock_desc(s1, s2, 16, 8192) is None
    finally:
        ops.set_force_ffma(False)
    assert spec.plan(2, 1, 100) is p and ops.resblock_desc(s1, s2, 16, 8192) is not None
    s1, s2 = _resblock_specs(32, 15, 11, True)                       # 282 rows: over the 256-row TMA box
    assert ops.resblock_desc(s1, s2, 2, 1000) is None


def test_tma_weight_gradient_plans_respect_the_hardware_limits():
    """kt_debug_wgrad_plan: the TMA-fed weight-gradient plan (made without a GPU) of the layer shapes of the 24 kHz model and of
    awkward ones (tiny T, long halos, every period): chunk rows = time steps x sub-sequences padded to whole K = 16 slices, TMA
    box extents <= 256, >= 2 ring stages inside the 227 KB of shared memory, a positive split-K factor."""
    import ctypes
    import numpy as np
    from kantts_b200 import _lib
    from kantts_b200._lib import KtConv1dDesc
    lib = _lib.load()

    def desc(cin, cout, k, stride=1, dil=1, groups=1, batch=16, nsub=1, t_in=2048, pad=None, transposed=0, up=1):
        pad = (k - 1) * dil // 2 if pad is None else pad
        t_out = (t_in * up + 2 * pad - dil * (k - 1) - 1) // stride + 1
        return KtConv1dDesc(batch=batch, nsub=nsub, t_in=t_in, t_out=t_out, c_in=cin, c_out=cout, groups=groups, kernel=k,
                            stride=stride, dilation=dil, pad_left=pad, transposed=transposed, upsample=up, act_in=0,
                            act_in_slope=0.0, act_out=1, act_out_slope=0.1, path=0)

    cases = [desc(128, 128, 11), desc(128, 128, 7, dil=3), desc(32, 32, 11, dil=5, t_in=8192), desc(64, 64, 3, t_in=4096),
             desc(256, 256, 11, t_in=256), desc(80, 512, 7, t_in=32), desc(1024, 1024, 5, batch=32, t_in=33), desc(1024, 1024, 5, t_in=9),
             desc(128, 256, 41, stride=4, groups=16), desc(1024, 1024, 41, groups=16, t_in=17), desc(512, 1024, 41, stride=4, groups=16, t_in=128),
             desc(128, 128, 41, stride=4, groups=4, t_in=8192)]
    for p in (2, 3, 5, 7, 11):
        cases += [desc(1024, 1024, 5, nsub=p, batch=32, t_in=max(2, 8192 // p // 81)), desc(512, 1024, 5, stride=3, nsub=p, t_in=8192 // p // 27),
                  desc(128, 512, 5, stride=3, nsub=p, t_in=8192 // p // 9), desc(32, 128, 5, stride=3, nsub=p, t_in=8192 // p // 3)]
    n_tma = 0
    for d in cases:
        out = (ctypes.c_int32 * 12)()
        assert lib.kt_debug_wgrad_plan(ctypes.byref(d), out) == 0
        ok, tma, tt, R, Rp, ns, smem, nsplit, NT, ngroups, a_box_t, rows_a_p = list(out)
        sig = (d.c_in, d.c_out, d.kernel, d.stride, d.groups, d.nsub, d.t_in)
        assert ok == 1, sig
        assert nsplit >= 1 and ngroups >= 1 and NT % 64 == 0 and NT <= 256, sig
        assert smem <= 227 * 1024, (sig, smem)
        if tma:
            n_tma += 1
            assert R == tt * d.nsub and Rp % 16 == 0 and 0 <= Rp - R < 16 and Rp <= 256, (sig, tt, R, Rp)
            assert 2 <= ns <= 4 and NT <= 128, (sig, ns, NT)
            assert a_box_t >= tt and a_box_t <= 256 and d.nsub <= 256, (sig, a_box_t)
            assert rows_a_p % 8 == 0 and rows_a_p >= Rp, (sig, rows_a_p)
            assert nsplit <= d.batch * -(-d.t_out // tt), sig
    assert n_tma >= len(cases) - 2     # every channel count here is a multiple of 8: (almost) all take the TMA variant
