"""Every dispatch arm of the exact-fp32 CUDA-core kernels, and the fused STFT/mel forward and backward, against plain
float64 references on the CPU.  Several kernels are templates picked by a host switch (attention rows per warp, LayerNorm
columns per lane, FSMN taps per thread, thin-conv kernel size): each arm is a separate compiled kernel, so each is tested
by name, and each case checks with torch.profiler that the arm it is named for is the one that ran -- a later change of a
shared-memory budget or a threshold cannot move a case onto another arm unnoticed.

Tolerances are relative L2 errors against float64; each one's comment gives the fp32 summation it bounds."""
import copy
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F
from torch.profiler import ProfilerActivity, profile

from conftest import rel_l2

pytestmark = pytest.mark.gpu
DEV = "cuda"
F64 = torch.float64


def _sops():
    from kantts_b200 import sambert_ops
    return sambert_ops


def _ops():
    from kantts_b200 import ops
    return ops


def _profiled(fn, kernels, leaves=()):
    """-> fn(), checked by torch.profiler to launch, for each name in `kernels`, a CUDA kernel whose name contains it.
    The profiler can deliver a run's kernel records incompletely (none at all, or without some launches), so a run
    whose records miss one of `kernels` is repeated, up to three runs, with the gradients of `leaves` cleared first.
    The dispatch is deterministic: a kernel that is not the arm which runs is missing from every run and fails."""
    for _ in range(3):
        for t in leaves:
            t.grad = None
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            out = fn()
            torch.cuda.synchronize()
        names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
        if all(any(k in n for n in names) for k in kernels):
            return out
    for k in kernels:
        assert any(k in n for n in names), (k, sorted(n for n in names if k.split("<")[0] in n))


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


# ------------------------------------------------------------------------------------------------
# attention: attn_{fwd,bwd_q}_kernel<D, RW>, attn_bwd_kv_kernel<D>
# ------------------------------------------------------------------------------------------------


def _ref_attention(q, k, v, mask, n_head, keep=None, p_drop=0.0):
    """q (B, Lq, HD), k / v (B, Lk, HD), mask (B, Lk) or (B or 1, Lq, Lk) -> out (B, Lq, HD), probs (H*B, Lq, Lk)."""
    B, Lq, hd = q.shape
    d = hd // n_head

    def split(t):
        return t.view(B, t.shape[1], n_head, d).permute(2, 0, 1, 3).reshape(n_head * B, t.shape[1], d)

    a = torch.bmm(split(q), split(k).transpose(1, 2)) / math.sqrt(d)
    if mask is not None:
        m = mask if mask.dim() == 3 else mask.unsqueeze(1).expand(-1, Lq, -1)
        a = a.masked_fill(m.expand(B, -1, -1).repeat(n_head, 1, 1), float("-inf"))
    a = torch.softmax(a, dim=2)
    if keep is not None:
        a = a * keep.to(a.dtype) / (1.0 - p_drop)
    o = torch.bmm(a, split(v))
    return o.view(n_head, B, Lq, d).permute(1, 2, 0, 3).reshape(B, Lq, hd), a


# (d_head, L, rows per warp): the score buffer [8*RW][Lk] plus one key tile fills 227 KB of shared memory at
# Lk = 1657 (d_head 16) and Lk = 1721 (d_head 8), where RW drops from 4 to 2; one below each switch point stays at 4.
# Every L but 2048 leaves a ragged last query tile (8*RW rows).
ATTN_ARMS = [(8, 1720, 4), (8, 1721, 2), (8, 2048, 2), (16, 1656, 4), (16, 1657, 2), (16, 2048, 2), (32, 1999, 2),
             (32, 2048, 2), (64, 1657, 1), (64, 2048, 1)]


@pytest.mark.parametrize("D,L,rw", ATTN_ARMS)
def test_self_attention_arm_matches_float64(D, L, rw):
    """Fused QKV rows (row stride 3*H*D), key-padding mask, forward / dq / dk / dv."""
    B, H = 2, 2
    hd = H * D
    g = torch.Generator().manual_seed(D * 10000 + L)
    qkv = torch.randn(B, L, 3 * hd, generator=g)
    r = torch.randn(B, L, hd, generator=g)
    mask = torch.arange(L)[None, :] >= torch.tensor([L, L - 37])[:, None]
    qr = qkv.to(F64).requires_grad_(True)
    o_ref, a_ref = _ref_attention(*qr.chunk(3, -1), mask, H)
    (o_ref * r.to(F64)).sum().backward()

    qg = qkv.to(DEV).requires_grad_(True)

    def run():
        o, a = _sops().SelfAttnFn.apply(qg, mask.to(DEV), H)
        (o * r.to(DEV)).sum().backward()
        return o, a

    o, a = _profiled(run, [f"attn_fwd_kernel<{D}, {rw}>", f"attn_bwd_q_kernel<{D}, {rw}>", f"attn_bwd_kv_kernel<{D}>"],
                     [qg])
    # forward: a D-term dot product, a softmax over Lk and an Lk-term P V sum per output
    assert rel_l2(o.cpu(), o_ref) < 5e-6, rel_l2(o.cpu(), o_ref)
    assert rel_l2(a.cpu(), a_ref) < 5e-6, rel_l2(a.cpu(), a_ref)
    # gradients: Lk-term (dq) and Lq-term (dk, dv) sums of products of forward quantities
    for i, name in enumerate(("dq", "dk", "dv")):
        sl = slice(i * hd, (i + 1) * hd)
        e = rel_l2(qg.grad[..., sl].cpu(), qr.grad[..., sl])
        assert e < 2e-5, (name, e)


def test_self_attention_dropout_arm_matches_float64():
    D, L, H, B, p = 8, 1721, 2, 1, 0.1
    hd = H * D
    g = torch.Generator().manual_seed(77)
    qkv = torch.randn(B, L, 3 * hd, generator=g)
    r = torch.randn(B, L, hd, generator=g)
    keep = torch.rand(H * B, L, L, generator=g) >= p
    qr = qkv.to(F64).requires_grad_(True)
    o_ref, a_ref = _ref_attention(*qr.chunk(3, -1), None, H, keep, p)
    (o_ref * r.to(F64)).sum().backward()
    qg = qkv.to(DEV).requires_grad_(True)

    def run():
        o, a = _sops().SelfAttnFn.apply(qg, None, H, p, keep.to(DEV))
        (o * r.to(DEV)).sum().backward()
        return o, a

    o, a = _profiled(run, ["attn_fwd_kernel<8, 2>", "attn_bwd_q_kernel<8, 2>"], [qg])
    assert rel_l2(o.cpu(), o_ref) < 5e-6
    assert rel_l2(a.cpu(), a_ref) < 5e-6
    assert rel_l2(qg.grad.cpu(), qr.grad) < 2e-5, rel_l2(qg.grad.cpu(), qr.grad)


@pytest.mark.parametrize("D,Lh,rw", [(8, 1800, 2), (16, 1700, 2), (32, 2048, 2), (64, 1500, 1)])
def test_pnca_attention_pair_arm_matches_float64(D, Lh, rw):
    """The PNCA pair: the memory part (Lq = 45 decoder rows against Lh memory rows, K / V row stride 2*H*D) adds its dq
    onto the self part's (accum_dq)."""
    B, H, L = 2, 2, 45
    hd = H * D
    g = torch.Generator().manual_seed(D + Lh)
    x_qkv = torch.randn(B, L, 3 * hd, generator=g)
    h_kv = torch.randn(B, Lh, 2 * hd, generator=g)
    rx, rh = torch.randn(B, L, hd, generator=g), torch.randn(B, L, hd, generator=g)
    mx = (torch.arange(L)[None, :] > torch.arange(L)[:, None])[None]                 # causal, shared by the batch
    mh = torch.arange(Lh)[None, :] >= torch.tensor([Lh, Lh - 100])[:, None]           # memory key padding
    xr, hr = x_qkv.to(F64).requires_grad_(True), h_kv.to(F64).requires_grad_(True)
    q, k, v = xr.chunk(3, -1)
    hk, hv = hr.chunk(2, -1)
    ox_ref, ax_ref = _ref_attention(q, k, v, mx, H)
    oh_ref, ah_ref = _ref_attention(q, hk, hv, mh, H)
    ((ox_ref * rx.to(F64)).sum() + (oh_ref * rh.to(F64)).sum()).backward()
    xg, hg = x_qkv.to(DEV).requires_grad_(True), h_kv.to(DEV).requires_grad_(True)

    def run():
        out = _sops().PncaAttnFn.apply(xg, hg, mx.to(DEV), mh.to(DEV), H)
        ((out[0] * rx.to(DEV)).sum() + (out[1] * rh.to(DEV)).sum()).backward()
        return out

    ox, oh, ax, ah = _profiled(run, [f"attn_fwd_kernel<{D}, {rw}>", f"attn_bwd_q_kernel<{D}, {rw}>"], [xg, hg])
    for name, got, want in (("ox", ox, ox_ref), ("oh", oh, oh_ref), ("ax", ax, ax_ref), ("ah", ah, ah_ref)):
        assert rel_l2(got.cpu(), want) < 5e-6, (name, rel_l2(got.cpu(), want))
    for name, got, want in (("dq", xg.grad[..., :hd], xr.grad[..., :hd]), ("dx_kv", xg.grad[..., hd:], xr.grad[..., hd:]),
                            ("dh_kv", hg.grad, hr.grad)):
        assert rel_l2(got.cpu(), want) < 2e-5, (name, rel_l2(got.cpu(), want))


# ------------------------------------------------------------------------------------------------
# LayerNorm: layernorm_{fwd,bwd}_kernel<NC>, C <= 32 * NC
# ------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("rows,c,nc", [(1, 129, 8), (300, 129, 8), (257, 200, 8), (1, 256, 8), (1000, 256, 8),
                                       (50, 20, 1), (50, 50, 2), (50, 100, 4), (50, 300, 16), (1, 777, 32), (70, 777, 32)])
def test_layernorm_arm_matches_float64(rows, c, nc):
    g = torch.Generator().manual_seed(rows * 1000 + c)
    x = torch.randn(rows, c, generator=g) * 2 + 0.5
    w, b = torch.randn(c, generator=g), torch.randn(c, generator=g)
    r = torch.randn(rows, c, generator=g)
    xr, wr, br = (t.to(F64).requires_grad_(True) for t in (x, w, b))
    yr = F.layer_norm(xr, (c,), wr, br, 1e-6)
    (yr * r.to(F64)).sum().backward()
    xg, wg, bg = (t.to(DEV).requires_grad_(True) for t in (x, w, b))

    def run():
        y = _sops().layer_norm(xg.view(1, rows, c), wg, bg, 1e-6)
        (y.view(rows, c) * r.to(DEV)).sum().backward()
        return y

    y = _profiled(run, [f"layernorm_fwd_kernel<{nc}>", f"layernorm_bwd_kernel<{nc}>"], [xg, wg, bg])
    assert rel_l2(y.view(rows, c).cpu(), yr) < 2e-6, rel_l2(y.view(rows, c).cpu(), yr)        # C-term mean / variance
    assert rel_l2(xg.grad.cpu(), xr.grad) < 1e-5, rel_l2(xg.grad.cpu(), xr.grad)
    assert rel_l2(wg.grad.cpu(), wr.grad) < 1e-5, rel_l2(wg.grad.cpu(), wr.grad)              # rows-term column sums
    assert rel_l2(bg.grad.cpu(), br.grad) < 1e-5, rel_l2(bg.grad.cpu(), br.grad)


# ------------------------------------------------------------------------------------------------
# FSMN memory block: fsmn_fir_kernel (forward and data gradient), fsmn_bwd_weight_kernel<TJ>, 4 * TJ >= K
# ------------------------------------------------------------------------------------------------


def _fsmn_ref(x, w, mask, lp):
    K = w.shape[-1]
    xm = x.masked_fill(mask.unsqueeze(-1), 0)
    y = F.conv1d(F.pad(xm, (0, 0, lp, K - 1 - lp)).transpose(1, 2), w, None, groups=x.shape[2]).transpose(1, 2) + xm
    return y.masked_fill(mask.unsqueeze(-1), 0)


# T = 700: two full 256-step weight-gradient chunks and a ragged third; C = 100: a ragged second 64-channel tile
@pytest.mark.parametrize("K,lp,tj", [(17, 0, 8), (17, 16, 8), (32, 0, 8), (32, 31, 8), (49, 0, 16), (49, 48, 16),
                                     (64, 0, 16), (64, 63, 16), (64, 30, 16)])
def test_fsmn_arm_matches_float64(K, lp, tj):
    B, T, C = 2, 700, 100
    g = torch.Generator().manual_seed(K * 100 + lp)
    x = torch.randn(B, T, C, generator=g)
    w = torch.randn(C, 1, K, generator=g) * 0.2
    r = torch.randn(B, T, C, generator=g)
    mask = torch.arange(T)[None, :] >= torch.tensor([T, T - 37])[:, None]
    xr, wr = x.to(F64).requires_grad_(True), w.to(F64).requires_grad_(True)
    (_fsmn_ref(xr, wr, mask, lp) * r.to(F64)).sum().backward()
    yr = _fsmn_ref(x.to(F64), w.to(F64), mask, lp)
    xg, wg = x.to(DEV).requires_grad_(True), w.to(DEV).requires_grad_(True)

    def run():
        y = _sops().FsmnMemoryFn.apply(xg, wg, mask.to(DEV), lp)
        (y * r.to(DEV)).sum().backward()
        return y

    y = _profiled(run, ["fsmn_fir_kernel", f"fsmn_bwd_weight_kernel<{tj}>"], [xg, wg])
    assert rel_l2(y.cpu(), yr) < 2e-6, rel_l2(y.cpu(), yr)                        # K-term FIR
    assert rel_l2(xg.grad.cpu(), xr.grad) < 1e-5, rel_l2(xg.grad.cpu(), xr.grad)
    assert rel_l2(wg.grad.cpu(), wr.grad) < 1e-5, rel_l2(wg.grad.cpu(), wr.grad)  # B*T-term sums


@pytest.mark.parametrize("K,lp", [(65, 32), (256, 0), (256, 255), (201, 77)])
def test_fsmn_long_filter_forward_matches_float64(K, lp):
    B, T, C = 2, 300, 72
    g = torch.Generator().manual_seed(K + lp)
    x = torch.randn(B, T, C, generator=g)
    w = torch.randn(C, 1, K, generator=g) * 0.1
    mask = torch.arange(T)[None, :] >= torch.tensor([T, 211])[:, None]
    y = _sops().FsmnMemoryFn.apply(x.to(DEV), w.to(DEV), mask.to(DEV), lp)
    yr = _fsmn_ref(x.to(F64), w.to(F64), mask, lp)
    assert rel_l2(y.cpu(), yr) < 2e-6, rel_l2(y.cpu(), yr)


# ------------------------------------------------------------------------------------------------
# autoregressive duration predictor (kt_ar_duration_infer)
# ------------------------------------------------------------------------------------------------


def _ar_duration_ref(m, cond):
    """VarRnnARPredictor.infer in float64: prenet -> 2-layer LSTM -> Linear -> ReLU, each output fed back as the next
    step's input (adaptors.py:67-83)."""
    fc1, fc2 = [copy.deepcopy(l).cpu().to(F64) for l in m.prenet.fcs if isinstance(l, torch.nn.Linear)][:2]
    lstm = copy.deepcopy(m.lstm).cpu().to(F64)
    fw, fb = m.fc.weight.detach().cpu().to(F64), m.fc.bias.detach().cpu().to(F64)
    B, L, _ = cond.shape
    x = torch.zeros(B, 1, dtype=F64)
    state, out = None, []
    for i in range(L):
        p = F.relu(F.linear(F.relu(F.linear(x, fc1.weight, fc1.bias)), fc2.weight, fc2.bias))
        h, state = lstm(torch.cat([p, cond[:, i]], -1).unsqueeze(1), state)
        x = F.relu(F.linear(h[:, 0], fw, fb))
        out.append(x)
    return torch.cat(out, 1)


# (cond_units, prenet units, H, B, L): sambert_24k (cond 96, prenet [128, 128], H 128: 512 threads), the kernel's size
# limits (H 256: 1024 threads, P1 = P2 = 1024), H 40 (160 threads: the cell updates end in a partial warp)
@pytest.mark.parametrize("cu,pre,H,B,L", [(96, [128, 128], 128, 2, 60), (96, [128, 128], 128, 3, 256),
                                          (64, [1024, 1024], 256, 2, 40), (24, [8, 8], 40, 3, 50)])
def test_ar_duration_predictor_matches_float64(cu, pre, H, B, L):
    from kantts_b200 import sambert
    torch.manual_seed(H * 7 + L)
    m = sambert.VarRnnARPredictor(cu, pre, H).eval()
    with torch.no_grad():
        m.fc.bias.fill_(0.5)               # durations mostly above the ReLU's kink, as trained models give
    cond = torch.randn(B, L, cu)
    want = _ar_duration_ref(m, cond.to(F64))
    m = m.to(DEV)
    got = _profiled(lambda: m.infer(cond.to(DEV)), ["ar_duration_kernel"])
    assert float(want.abs().max()) > 0.1
    # each step: P1-, P2- and (P2 + H)-term dot products, an error that the recurrence carries through L steps
    assert rel_l2(got.cpu(), want) < 2e-5, rel_l2(got.cpu(), want)


def test_sambert_24k_free_running_inference_batch_matches_oracle():
    """sambert_24k_config at full width, free-running on a ragged batch of 3, against the CPU oracle."""
    import kantts_b200 as K
    from kantts_b200 import sambert
    from oracle import sambert as osb
    from golden.make_batch import make_sambert_batch
    from test_gpu_sambert import INFER_KEYS, _infer_model
    cfg = K.sambert_24k_config()
    torch.manual_seed(5)
    sd = {k: v.detach().clone() for k, v in sambert.KanTtsSAMBERT(cfg).state_dict().items()}
    (dur_bias,) = [k for k in sd if k.endswith("duration_predictor.fc.bias")]
    sd[dur_bias].fill_(1.4)                 # about 3 frames per symbol from the untrained predictor
    batch = make_sambert_batch(cfg, B=3, L=12, gen=torch.Generator().manual_seed(41), short=4)
    inputs = {k: batch[k] for k in ("inputs_ling", "inputs_emotion", "inputs_speaker", "input_lengths")}
    with torch.no_grad():
        want = osb.sambert_infer(sd, cfg, inputs["inputs_ling"], inputs["inputs_emotion"], inputs["inputs_speaker"],
                                 inputs["input_lengths"])
    dur = torch.exp(want["log_duration_predictions"]) - 1
    frac = (dur + 0.5) - torch.floor(dur + 0.5)
    assert float(torch.minimum(frac, 1 - frac)[dur > 0].min()) > 2e-3       # no duration sits on a rounding boundary
    res = _infer_model(cfg, sd, inputs, True)
    assert torch.equal(res["LR_length_rounded"].cpu(), want["LR_length_rounded"])
    for k in INFER_KEYS:
        assert res[k].shape == want[k].shape, (k, res[k].shape, want[k].shape)
        assert rel_l2(res[k].cpu(), want[k]) < 2e-5, (k, rel_l2(res[k].cpu(), want[k]))


# ------------------------------------------------------------------------------------------------
# thin C_in = 1 convs: thin_c128_{fwd,wgrad}_kernel<K>, thin_cin1_{fwd,wgrad}_kernel
# ------------------------------------------------------------------------------------------------


THIN_CASES = {
    # name: (spec kwargs, act_out slope or None, B, T, period, kernels)
    "c128_k3": (dict(c_out=128, kernel=3, pad_left=1, pad_right=1), None, 2, 3000, 0, "thin_c128_{}_kernel<3>"),
    "c128_k3_lrelu": (dict(c_out=128, kernel=3, pad_left=1, pad_right=1), 0.2, 2, 3000, 0, "thin_c128_{}_kernel<3>"),
    "c128_k5": (dict(c_out=128, kernel=5, pad_left=2, pad_right=2), None, 2, 3001, 0, "thin_c128_{}_kernel<5>"),
    "c128_k5_lrelu": (dict(c_out=128, kernel=5, pad_left=2, pad_right=2), 0.1, 2, 3001, 0, "thin_c128_{}_kernel<5>"),
    "c128_k15": (dict(c_out=128, kernel=15, pad_left=7, pad_right=7), None, 3, 2000, 0, "thin_c128_{}_kernel<15>"),
    "c128_k15_lrelu": (dict(c_out=128, kernel=15, pad_left=7, pad_right=7), 0.1, 3, 2000, 0, "thin_c128_{}_kernel<15>"),
    "c64_period_s3": (dict(c_out=64, kernel=5, stride=3, pad_left=2, pad_right=2), 0.1, 2, 600, 5, "thin_cin1_{}_kernel"),
    "c256_d2": (dict(c_out=256, kernel=7, dilation=2, pad_left=6, pad_right=6), None, 2, 1000, 0, "thin_cin1_{}_kernel"),
    "c256_d3_lrelu": (dict(c_out=256, kernel=5, dilation=3, pad_left=6, pad_right=6), 0.1, 2, 999, 0,
                      "thin_cin1_{}_kernel"),
    "c128_period_d2": (dict(c_out=128, kernel=5, dilation=2, pad_left=4, pad_right=4), 0.1, 2, 300, 3,
                       "thin_cin1_{}_kernel"),
}


@pytest.mark.parametrize("name", list(THIN_CASES))
def test_thin_conv_arm_matches_float64(name):
    from kantts_b200._lib import KT_ACT_LRELU
    from oracle import convref
    from oracle import hifigan as O
    ops = _ops()
    kw, slope, B, T, period, kernel = THIN_CASES[name]
    spec = ops.ConvSpec(c_in=1, **kw)
    if slope is not None:
        spec.act_out, spec.act_out_slope = KT_ACT_LRELU, slope
    g = torch.Generator().manual_seed(len(name) * 31 + T)
    v = torch.randn(spec.c_out, 1, spec.kernel, generator=g) * 0.3
    gg = v.norm(2, dim=(1, 2), keepdim=True) * (1 + 0.2 * torch.randn(spec.c_out, 1, 1, generator=g))
    bias = 0.1 * torch.randn(spec.c_out, generator=g)
    x = torch.randn((B, 1, T, period) if period else (B, 1, T), generator=g)
    xo, vo, go, bo = (t.to(F64).requires_grad_(True) for t in (x, v, gg, bias))
    yo = convref.conv_layer(xo, O.weight_norm_weight(go, vo), bo, stride=spec.stride, dilation=spec.dilation,
                            pad_left=spec.pad_left, pad_right=spec.pad_right, act_out=slope)
    rows = lambda t: t.permute(0, 2, 1).contiguous() if t.dim() == 3 else t.permute(0, 2, 3, 1).contiguous()
    unrows = lambda t: t.permute(0, 2, 1) if t.dim() == 3 else t.permute(0, 3, 1, 2)
    r = torch.randn(yo.shape, generator=g)
    xg, vg, g2, bg = x.to(DEV), v.to(DEV).requires_grad_(True), gg.to(DEV).requires_grad_(True), bias.to(DEV).requires_grad_(True)
    xg = rows(xg).requires_grad_(True)

    def fwd():
        return ops.conv(xg, spec, ops.PreparedWeight(), vg, g2, bg)

    y = _profiled(fwd, [kernel.format("fwd")])
    if slope is not None:
        # outputs whose sign differs between fp32 and float64 (|y| below the forward error) would switch the LeakyReLU's
        # slope in the gradient: leave exactly those out of the scalar both sides differentiate
        flip = torch.sign(yo.detach()) != torch.sign(unrows(y.detach()).cpu().to(F64))
        assert float(flip.double().mean()) < 1e-3
        r = r * (~flip)
    (yo * r.to(F64)).sum().backward()
    _profiled(lambda: (y * rows(r).to(DEV)).sum().backward(retain_graph=True), [kernel.format("wgrad")], [xg, vg, g2, bg])
    assert rel_l2(unrows(y).cpu(), yo) < 2e-6, rel_l2(unrows(y).cpu(), yo)          # k-term FIR
    assert rel_l2(unrows(xg.grad).cpu(), xo.grad) < 1e-4, rel_l2(unrows(xg.grad).cpu(), xo.grad)
    # B*T_out*nsub-term sums per tap, then the weight-norm backward
    for nm, got, want in (("dv", vg.grad, vo.grad), ("dg", g2.grad, go.grad), ("dbias", bg.grad, bo.grad)):
        assert rel_l2(got.cpu(), want) < 2e-5, (nm, rel_l2(got.cpu(), want))


# ------------------------------------------------------------------------------------------------
# fused STFT / mel: stft_mel_fwd_kernel, stft_mel_bwd_kernel, ola_gather_kernel
# ------------------------------------------------------------------------------------------------

MEL_NORM = (20.0, -100.0, 8.0, 4.0, -4.0, 4.0)      # ref_db, min_db, scale, shift, lo, hi (MelSpectrogram's defaults)


def _stft_pre(wav, window, n_fft, hop, pad_mode):
    """|STFT|^2, (B, frames, n_fft/2 + 1), float64, centre-padded with zeros (0) or by reflection (1)."""
    z = torch.stft(wav, n_fft, hop, window=window, center=True, pad_mode="reflect" if pad_mode else "constant",
                   return_complex=True)
    return (z.real ** 2 + z.imag ** 2).transpose(1, 2)


def _mel_chain(pw, eps, melmat):
    """-> (output, {threshold name: (pre-clamp value, threshold, relative distance that fp32 rounding can bridge)}) of
    the kernel's amplitude -> mel -> dB chain.  A bin's fp32 power has an absolute error of ~1e-7 of its frame's energy,
    so a power within 10 % of eps can land on either side of the clamp; the mel and dB values are good to ~1e-6."""
    amp = pw.clamp_min(eps).sqrt()
    if melmat is None:
        return amp, {"power": (pw, eps, 0.1)}
    ref_db, min_db, scale, shift, lo, hi = MEL_NORM
    acc = amp @ melmat                                                    # (B, frames, n_mels)
    melc = acc.clamp_min(eps)
    x = melc.clamp_min(1e-5)
    v = scale * ((20 * torch.log10(x) - ref_db - min_db) / (-min_db)) - shift
    return v.clamp(lo, hi).transpose(1, 2), {"mel": (melc.transpose(1, 2), 1e-5, 1e-4),
                                             "lo": (v.transpose(1, 2), lo, 1e-4), "hi": (v.transpose(1, 2), hi, 1e-4)}


def _test_signal(B, T, n_fft, g):
    """Item 0: noise with an exactly silent stretch (whole frames of zeros) and a loud burst that drives the mel to its
    +4 ceiling; item 1: silent throughout; item 2: loud throughout."""
    w = 0.1 * torch.randn(B, T, generator=g)
    if T >= 4 * n_fft:
        w[0, T // 4: T // 4 + 2 * n_fft] = 0
        w[0, -T // 4 - n_fft: -T // 4] *= 1e4
    w[1] = 0
    w[2] *= 1e7
    return w


# (n_fft, hop, win_length, T, pad_mode, mel): every FFT size the kernel takes, both pad modes; the three resolutions of
# the multi-resolution STFT loss (hop not dividing T, win_length < n_fft); reflect at its shortest T = n_fft/2 + 1;
# zero padding with T < n_fft
STFT_CASES = [
    (64, 16, 64, 1000, 0, True), (64, 16, 64, 1001, 1, False), (64, 16, 48, 33, 1, True),
    (512, 128, 512, 5000, 0, True), (512, 128, 512, 5000, 1, False),
    (1024, 256, 1024, 8191, 0, True), (1024, 256, 1024, 8191, 1, True), (1024, 256, 1024, 513, 1, False),
    (1024, 256, 1024, 700, 0, True),
    (2048, 512, 2048, 12000, 0, True), (2048, 512, 2048, 12000, 1, False),
    (4096, 1024, 4096, 20000, 0, True), (4096, 1024, 4096, 20001, 1, False), (4096, 1024, 4096, 3000, 0, False),
    (1024, 120, 600, 8000, 1, False), (2048, 240, 1200, 8000, 1, False), (512, 50, 240, 8000, 1, False),
]


@pytest.mark.parametrize("n_fft,hop,win,T,pad_mode,mel", STFT_CASES)
def test_stft_mel_matches_float64(n_fft, hop, win, T, pad_mode, mel):
    from kantts_b200.audio import _padded_window, slaney_mel_filterbank
    ops = _ops()
    B = 3
    g = torch.Generator().manual_seed(n_fft + hop + T + pad_mode)
    wav = _test_signal(B, T, n_fft, g)
    window = _padded_window(win, n_fft, "cpu")
    melmat = torch.from_numpy(slaney_mel_filterbank(22050, n_fft, 80, 80, 7600).T.copy()) if mel else None
    eps = 1e-10 if mel else 1e-7
    pw = _stft_pre(wav.to(F64), window.to(F64), n_fft, hop, pad_mode)
    want, pre = _mel_chain(pw, eps, None if melmat is None else melmat.to(F64))
    if mel:
        # a mel mixes every bin of its frame, so no bin may sit where rounding decides the power clamp
        assert not bool(((pw > 0.1 * eps) & (pw < 10 * eps)).any())
    # leave out of the comparison only outputs whose float64 pre-clamp value lies within rounding of a clamp threshold
    near = torch.zeros(want.shape, dtype=torch.bool)
    for val, thr, band in pre.values():
        near |= (val - thr).abs() <= band * abs(thr)
    assert float(near.double().mean()) < 1e-3
    r = torch.randn(want.shape, generator=g) * (~near)

    wr = wav.to(F64).requires_grad_(True)
    out_r, _ = _mel_chain(_stft_pre(wr, window.to(F64), n_fft, hop, pad_mode), eps,
                          None if melmat is None else melmat.to(F64))
    (out_r * r.to(F64)).sum().backward()

    wg = wav.to(DEV).requires_grad_(True)

    def run():
        o = ops.StftMelFn.apply(wg, window.to(DEV), None if melmat is None else melmat.to(DEV), n_fft, hop, pad_mode, eps)
        (o * r.to(DEV)).sum().backward()
        return o

    out = _profiled(run, ["stft_mel_fwd_kernel", "stft_mel_bwd_kernel", "ola_gather_kernel"], [wg])
    keep = ~near
    assert rel_l2(out.cpu()[keep], want[keep]) < 1e-5, rel_l2(out.cpu()[keep], want[keep])
    dw = wg.grad.cpu()
    assert rel_l2(dw, wr.grad) < 1e-5, rel_l2(dw, wr.grad)
    # the reflected / zero-padded edges on their own: they are a small share of the whole signal's norm
    edge = min(n_fft, T)
    for part in (slice(0, edge), slice(T - edge, T)):
        assert rel_l2(dw[0, part], wr.grad[0, part]) < 1e-5, (part, rel_l2(dw[0, part], wr.grad[0, part]))
    # a silent item has every bin at the power clamp: its gradient is exactly zero
    assert torch.equal(dw[1], torch.zeros(T))
    if mel:
        # the loud item has every mel at the +4 ceiling (or, for an empty filter, at the floor): exactly zero gradient
        assert bool((pre["hi"][0][2] > MEL_NORM[5] + 1e-3).logical_or(pre["lo"][0][2] < MEL_NORM[4] - 1e-3).all())
        assert torch.equal(dw[2], torch.zeros(T))


# ------------------------------------------------------------------------------------------------
# misc.cu: db3 DWT, upsample_grad_reduce, sinadd, add3_scale, l1_sum (split_sum_kernel / split_sum_wide_kernel)
# ------------------------------------------------------------------------------------------------

# PyWavelets Wavelet('db3').dec_lo; dec_hi is its quadrature mirror hi[j] = (-1)^(j+1) lo[5-j]
DB3_LO = [0.035226291882100656, -0.08544127388224149, -0.13501102001039084, 0.4598775021193313, 0.8068915093133388,
          0.3326705529509569]


def _dwt_ref(x):
    """y[b][n] = (sum_j lo[j] x[2n+1-j], sum_j hi[j] x[2n+1-j]), zero outside [0, T), n < (T + 5) // 2."""
    lo = torch.tensor(DB3_LO, dtype=F64)
    hi = torch.tensor([(-1) ** (j + 1) * DB3_LO[5 - j] for j in range(6)], dtype=F64)
    B, T = x.shape
    t2 = (T + 5) // 2
    xp = F.pad(x, (5, 6))                       # xp[s + 5] = x[s]
    cols = []
    for filt in (lo, hi):
        cols.append(sum(filt[j] * xp[:, 2 * torch.arange(t2) + 1 - j + 5] for j in range(6)))
    return torch.stack(cols, -1)


def test_db3_filter_constants():
    lo = torch.tensor(DB3_LO, dtype=F64)
    # orthonormal to the 1e-11 that PyWavelets' tabulated values carry
    assert abs(float(lo.sum()) - math.sqrt(2)) < 1e-10 and abs(float((lo * lo).sum()) - 1) < 1e-10
    assert abs(float((lo[:-2] * lo[2:]).sum())) < 1e-10 and abs(float((lo[:-4] * lo[4:]).sum())) < 1e-10


@pytest.mark.parametrize("T", [1, 2, 3, 5, 6, 7, 1000, 1001])
def test_dwt_matches_explicit_db3_sum(T):
    g = torch.Generator().manual_seed(T)
    x = torch.randn(3, T, generator=g)
    xr = x.to(F64).requires_grad_(True)
    yr = _dwt_ref(xr)
    r = torch.randn(yr.shape, generator=g)
    (yr * r.to(F64)).sum().backward()
    xg = x.to(DEV).requires_grad_(True)
    y = _ops().DwtFn.apply(xg)
    (y * r.to(DEV)).sum().backward()
    assert y.shape == yr.shape
    assert rel_l2(y.cpu(), yr) < 1e-6, rel_l2(y.cpu(), yr)           # 6-term sums
    assert rel_l2(xg.grad.cpu(), xr.grad) < 1e-6, rel_l2(xg.grad.cpu(), xr.grad)


@pytest.mark.parametrize("up,c,act", [(2, 64, False), (8, 32, True), (3, 12, True), (16, 4, False)])
def test_upsample_grad_reduce_matches_float64(up, c, act):
    from kantts_b200._lib import KT_ACT_LRELU, KT_ACT_NONE
    rows, slope = 2 * 317, 0.1
    g = torch.Generator().manual_seed(up * 100 + c)
    dxu = torch.randn(rows * up, c, generator=g)
    x = torch.randn(rows, c, generator=g)
    want = dxu.to(F64).view(rows, up, c).sum(1)
    if act:
        want = torch.where(x > 0, want, want * slope)
    dxu_g, x_g = dxu.to(DEV), x.to(DEV)
    dx = torch.empty(rows, c, device=DEV)
    _ops().call("kt_upsample_grad_reduce", _ptr(dxu_g), _ptr(x_g) if act else None, KT_ACT_LRELU if act else KT_ACT_NONE,
                slope, _ptr(dx), rows, up, c)
    assert rel_l2(dx.cpu(), want) < 1e-6, rel_l2(dx.cpu(), want)     # up-term sums


def test_upsample_grad_reduce_rejects_misaligned_rows():
    from kantts_b200._lib import KT_ACT_NONE
    buf = torch.randn(2 * 8 * 16 + 1, device=DEV)
    dxu = buf[1:].view(2 * 8, 16)                       # contiguous, 4 bytes past a 16-byte boundary
    dx = torch.empty(2, 16, device=DEV)
    with pytest.raises(RuntimeError, match="aligned"):
        _ops().call("kt_upsample_grad_reduce", _ptr(dxu), None, KT_ACT_NONE, 0.0, _ptr(dx), 2, 8, 16)


def _offset_view(t, offset):
    """t's values in a contiguous view that starts `offset` floats into its storage."""
    buf = torch.empty(t.numel() + offset, device=t.device, dtype=t.dtype)
    v = buf[offset:].view(t.shape)
    v.copy_(t)
    return v


# n % 4 != 0 exercises the scalar tail; 2^22 + 3 wraps the grid-stride loop; offset 1 is a misaligned contiguous view
@pytest.mark.parametrize("n,offset", [(1, 0), (3, 0), (4097, 0), ((1 << 22) + 3, 0), (4097, 1), ((1 << 22) + 3, 3)])
def test_sinadd_matches_float64(n, offset):
    g = torch.Generator().manual_seed(n)
    x = torch.randn(n, generator=g) * 3
    dy = torch.randn(n, generator=g)
    xg = _offset_view(x.to(DEV), offset).requires_grad_(True)
    y = _ops().SinAddFn.apply(xg)
    y.backward(_offset_view(dy.to(DEV), offset))
    x64 = x.to(F64)
    assert rel_l2(y.cpu(), x64 + torch.sin(x64)) < 1e-6, rel_l2(y.cpu(), x64 + torch.sin(x64))
    assert rel_l2(xg.grad.cpu(), dy.to(F64) * (1 + torch.cos(x64))) < 1e-6


@pytest.mark.parametrize("n,offset,nb", [(5, 0, 3), (4099, 0, 1), (4099, 0, 2), ((1 << 22) + 1, 0, 3), (4099, 1, 3),
                                         ((1 << 22) + 1, 2, 2)])
def test_add3_scale_matches_float64(n, offset, nb):
    """nb of the three addends given (b, then c, may be missing)."""
    g = torch.Generator().manual_seed(n + nb)
    ts = [torch.randn(n, generator=g) for _ in range(nb)]
    dy = torch.randn(n, generator=g)
    gs = [_offset_view(t.to(DEV), offset + i).requires_grad_(True) for i, t in enumerate(ts)]
    args = gs + [None] * (3 - nb)
    y = _ops().Mean3Fn.apply(1 / 3, *args)
    y.backward(_offset_view(dy.to(DEV), offset))
    want = sum(t.to(F64) for t in ts) / 3
    assert rel_l2(y.cpu(), want) < 1e-6, rel_l2(y.cpu(), want)
    for t in gs:
        assert rel_l2(t.grad.cpu(), dy.to(F64) / 3) < 1e-6


# blocks = n/4/256 + 1 partial sums: fewer than 64 are summed by split_sum_kernel, 64 or more by split_sum_wide_kernel
@pytest.mark.parametrize("n,offset,kernel", [(1, 0, "split_sum_kernel"), (1001, 1, "split_sum_kernel"),
                                             (64000, 0, "split_sum_kernel"), (65536, 0, "split_sum_wide_kernel"),
                                             (3_000_001, 0, "split_sum_wide_kernel"),
                                             (3_000_001, 1, "split_sum_wide_kernel")])
def test_l1_sum_matches_float64(n, offset, kernel):
    ops = _ops()
    g = torch.Generator().manual_seed(n + offset)
    a, b = torch.randn(n, generator=g), torch.randn(n, generator=g)
    ag, bg = _offset_view(a.to(DEV), offset), _offset_view(b.to(DEV), 2 * offset)
    want = 0.37 * float((a.to(F64) - b.to(F64)).abs().sum())
    got = _profiled(lambda: ops.l1_sum(ag, bg, 0.37), ["l1_sum_kernel", kernel + "("])
    # per-thread running sums of ~n / (blocks * 256) terms, then block and split sums
    assert abs(float(got) - want) <= 1e-6 * want, (float(got), want)
    acc = torch.full((), 2.5, device=DEV)
    _profiled(lambda: (acc.fill_(2.5), ops.l1_sum_acc(acc, ag, bg, 0.37)), [kernel + "("])
    assert abs(float(acc) - (2.5 + want)) <= 1e-6 * (2.5 + want), (float(acc), 2.5 + want)


def test_l1_sum_empty():
    ops = _ops()
    e = torch.empty(0, device=DEV)
    assert float(ops.l1_sum(e, e)) == 0.0
    acc = torch.full((), 1.25, device=DEV)
    ops.l1_sum_acc(acc, e, e, 2.0)
    assert float(acc) == 1.25
