"""CPU: host-side planning logic of the C ABI (no kernel is launched): tensor-core tile plans, packed-weight image sizes,
split-K workspaces and the dispatch rules added for thin / grouped / waveform-input layers."""
import ctypes

import pytest

from kantts_b200 import _lib, ops
from kantts_b200._lib import KT_PATH_AUTO, KT_PATH_FFMA, KT_PATH_TC


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
    s2 = spec.without_upsample()
    d2 = s2.desc(16, 1, 32 * 8)
    assert d2.t_out == d.t_out and s2.act_in == 0 and s2.upsample == 1
    assert lib.kt_conv1d_tc_plan(ctypes.byref(d2), 1) > 0            # ... but as the plain conv over the up-sampled rows


def test_split_k_workspace_is_whole_slices_of_the_gradient(lib):
    for kw, B, T, nsub in ((dict(c_in=1024, c_out=1024, kernel=5, pad_left=2, pad_right=2), 32, 34, 3),
                           (dict(c_in=32, c_out=32, kernel=11, pad_left=10), 16, 8192, 1),
                           (dict(c_in=128, c_out=256, kernel=41, stride=4, pad_left=20, pad_right=20, groups=16), 16, 2048, 1)):
        spec, d = _desc(B, T, nsub=nsub, **kw)
        ws = lib.kt_conv1d_bwd_weight_tc_workspace(ctypes.byref(d))
        # one slice per split: the weight gradient + (when the bias gradient rides along as an all-ones MMA unit) the
        # bias gradient padded to a multiple of 4 floats
        per = spec.w_numel + ((spec.c_out + 3) & ~3)
        out = (ctypes.c_int32 * 12)()
        assert lib.kt_debug_wgrad_plan(ctypes.byref(d), out) == 0
        if out[1] and ws % spec.w_numel and ws % per:
            # TMA variant (a driver is present): the slices, padded to 64 floats, then the hi / lo bf16 operand planes of
            # both operands (one float per element each, padded to 64 floats)
            r64 = lambda n: (n + 63) & ~63
            planes = r64(d.batch * d.t_in * d.nsub * d.c_in) + r64(d.batch * d.t_out * d.nsub * d.c_out)
            assert ws - planes in (r64(out[7] * spec.w_numel), r64(out[7] * per)), (ws, planes, out[7])
            nsplit = out[7]
        else:
            assert ws > 0 and (ws % spec.w_numel == 0 or ws % per == 0)
            nsplit = ws // per if ws % per == 0 else ws // spec.w_numel
        assert 1 <= nsplit <= 296


def test_grad_items_context_restores_state():
    assert ops._grad_items is None
    with ops.grad_items(4):
        assert ops._grad_items == 4
        with ops.grad_items(2):
            assert ops._grad_items == 2
        assert ops._grad_items == 4
    assert ops._grad_items is None


def test_ffma_path_has_no_tensor_plan(lib):
    _, d = _desc(2, 100, c_in=64, c_out=64, kernel=3, pad_left=2, path=KT_PATH_FFMA)
    spec = ops.ConvSpec(c_in=64, c_out=64, kernel=3, pad_left=2, path=KT_PATH_FFMA)
    assert ops._tc_tile(lib, spec, d, 0) == 0 and ops._wgrad_tc_workspace(lib, spec, d) == 0


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
