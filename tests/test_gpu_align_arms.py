"""Every alignment-learning kernel of align.cu against a float64 reference of the same operation, at the training shape of
sambert_16k_MAS.yaml (16 utterances, about 200 symbols and 1000 frames, c = 80) and at the edges of each kernel's tiling:
the distance attention (align_attn_fwd_kernel, align_attn_bwd_rows_kernel, align_attn_bwd_keys_kernel), the forward-sum
loss (ctc_fwd_kernel, ctc_bwd_kernel) and the width-1 MAS (mas_kernel), each called through its C entry point, and the
attention -> MAS -> binarization + forward-sum chain of one training batch.

Each result is checked per element, |got - ref| <= c * scale with scale the sum over magnitudes of the terms the element
is computed from, so that one wrong row, key, tile or state cannot hide under a whole-tensor norm.  Every kernel here
promises a fixed order per item: each call runs twice and must give the same bits, and each item's rows must equal that
item run alone.
"""
import math

import numpy as np
import pytest
import torch

from conftest import rel_l2
from test_gpu_sambert_mas import _random_maps, make_mas_batch

pytestmark = pytest.mark.gpu

DEV = "cuda"
F64 = torch.float64

# Per-element error over the error scale (the bound of any summation order of fp32 terms is a few units of 2^-24 times
# the scale).  Worst over all cases on an H100 80GB HBM3 (700 W power limit) in brackets; the bounds are about 4x those.
#   z        logprob without a prior: c squares summed in channel order; scale 0.0005 sum_c (q_c - k_c)^2       [7.8e-7]
#   logprob  with a prior: z - logsumexp_j z + log(prior + 1e-8); scale |z_j| + max_j |z_j| + |lse| + |log prior| [1.8e-7]
#   soft     softmax over the valid keys; scale soft_j (1 + L_j + sum_j' soft_j' L_j'), L the logprob scale    [2.8e-7]
#   dz       softmax and log_softmax backward; scale the magnitudes of their terms (D below)                   [1.4e-7]
#   dq       -0.001 sum_j dz_ij (q_i - k_j) in key order; scale 0.001 sum_j D_ij |q_i - k_j|                     [3.2e-7]
#   dk       0.001 sum_i dz_ij (q_i - k_j) in query order; scale 0.001 sum_i D_ij |q_i - k_j|                     [3.0e-7]
#   ctc      d_logprob = g (softmax_tj - posterior_tj); scale g (softmax_tj (1 + |y_tj| + |lse_t|) + posterior_tj) [2.8e-7]
#   ctc_loss nll_b / N_b over fp32 frame normalisers, and their mean; scale (nll_b + sum_t |lse_t|) / N_b        [1.1e-7]
# The ctc bound holds only with the alpha / beta recursions in float64: with fp32 state the posterior exp(alpha + beta -
# y + nll) cancels values in the thousands, and the same cases measured 2.1e-3 at the training shape (relative L2 3.9e-4)
# and 5.8e-2 at t_k = 3071 (relative L2 2.6e-2).
BOUND = {"z": 3e-6, "logprob": 7e-7, "soft": 1.2e-6, "dz": 6e-7, "dq": 1.3e-6, "dk": 1.2e-6, "ctc": 1.2e-6,
         "ctc_loss": 4e-7}


def _ops():
    from kantts_b200 import _lib, ops, sambert_ops
    return _lib, ops, sambert_ops


def _call(fn, *args):
    _ops()[1].call(fn, *args)


def _ptr(t, aux=False):
    return _ops()[0].ptr(t, aux)


def _i32(t):
    return t.to(DEV, torch.int32).contiguous()


def _check(name, got, ref, scale, case):
    """|got - ref| <= BOUND[name] * scale element by element (exactly equal where the scale is 0); prints the worst
    ratio."""
    got, ref, scale = got.to(DEV, F64), ref.to(DEV, F64), scale.to(DEV, F64)
    assert got.shape == ref.shape == scale.shape, (name, got.shape, ref.shape, scale.shape)
    assert torch.isfinite(got).all(), (name, case, "non-finite")
    err = (got - ref).abs()
    assert torch.equal(err[scale == 0], torch.zeros_like(err[scale == 0])), (name, case, "nonzero where exact")
    ratio = torch.where(scale > 0, err / scale.clamp_min(1e-300), torch.zeros_like(err))
    worst = float(ratio.max()) if ratio.numel() else 0.0
    print(f"align_arms {case} {name}: worst |err| / scale {worst:.3g} (bound {BOUND[name]:.1g})")
    at = np.unravel_index(int(ratio.argmax()), tuple(ratio.shape)) if ratio.numel() else ()
    assert worst <= BOUND[name], (name, case, worst, at, float(got[at]), float(ref[at]), float(scale[at]))


def _same_bits(a, b, what):
    for k in a:
        assert torch.equal(a[k], b[k]), (what, k)


# ------------------------------------------------------------------------------------------------
# distance attention
# ------------------------------------------------------------------------------------------------


def _attn_kernel(q, k, prior, key_len, ds, dl):
    """kt_align_attn_fwd then kt_align_attn_bwd on fp32 device tensors; outputs prefilled with NaN, so that an element
    the kernels leave unwritten fails."""
    B, Tq, C = q.shape
    Tk = k.shape[1]
    nan = lambda *s: torch.full(s, float("nan"), device=DEV)
    lp, soft, dz, dq, dk = nan(B, Tq, Tk), nan(B, Tq, Tk), nan(B, Tq, Tk), nan(B, Tq, C), nan(B, Tk, C)
    lse = nan(B, Tq) if prior is not None else None
    kl = _i32(key_len)
    _call("kt_align_attn_fwd", _ptr(q), _ptr(k), _ptr(prior), _ptr(kl, True), _ptr(lp), _ptr(soft), _ptr(lse), B, Tq, Tk, C)
    _call("kt_align_attn_bwd", _ptr(q), _ptr(k), _ptr(prior), _ptr(soft), _ptr(lse), _ptr(ds), _ptr(dl), _ptr(dz),
          _ptr(dq), _ptr(dk), B, Tq, Tk, C)
    torch.cuda.synchronize()
    return {"logprob": lp, "soft": soft, "dz": dz, "dq": dq, "dk": dk}


def _attn_reference(q, k, prior, key_len, ds, dl, dl_mag=None):
    """float64 on the device: soft, logprob, dq and dk by oracle.sambert_mas.distance_attention and autograd; dz, the
    gradient of z = -0.0005 sum_c (q - k)^2, by autograd through the same formulas from a z leaf (attention.py:122-125
    as the oracle states them), and the error scales of every output.  ds / dl: the upstream gradients (None: absent);
    dl_mag: the magnitude of dl's own error scale where dl is itself a computed gradient (default |dl|)."""
    from oracle import sambert_mas as om
    B, Tq, C = q.shape
    Tk = k.shape[1]
    q64 = q.to(DEV, F64).requires_grad_(True)
    k64 = k.to(DEV, F64).requires_grad_(True)
    n = key_len.to(DEV).long().clamp(1, Tk)                       # the kernels clamp the key length to [1, t_k]
    mask = torch.arange(Tk, device=DEV)[None, :] >= n[:, None]
    pr = None if prior is None else prior.to(DEV, F64)
    soft_o, lp_o = om.distance_attention(q64, k64, mask, pr)
    outs = [(t, g) for t, g in ((soft_o, ds), (lp_o, dl)) if g is not None]
    dq, dk = torch.autograd.grad([t for t, _ in outs], [q64, k64], [g.to(DEV, F64)[:, None] for _, g in outs])
    with torch.no_grad():
        z = -0.0005 * ((q64[:, :, None] - k64[:, None]) ** 2).sum(-1)
    zl = z.clone().requires_grad_(True)
    lse = torch.logsumexp(zl, -1, keepdim=True)
    lp = zl - lse + torch.log(pr + 1e-8) if pr is not None else zl
    soft = torch.softmax(lp.masked_fill(mask[:, None], -math.inf), -1)
    outs = [(t, g) for t, g in ((soft, ds), (lp, dl)) if g is not None]
    (dz,) = torch.autograd.grad([t for t, _ in outs], [zl], [g.to(DEV, F64) for _, g in outs])
    with torch.no_grad():
        assert rel_l2(soft, soft_o[:, 0]) < 1e-12 and rel_l2(lp, lp_o[:, 0]) < 1e-12
        za = z.abs()
        zmax = za.amax(-1, keepdim=True)
        if pr is None:
            lp_scale = za
        else:
            lp_scale = za + zmax + lse.abs() + torch.log(pr + 1e-8).abs()
        s = soft
        s_rel = 1 + lp_scale + (s * lp_scale).sum(-1, keepdim=True)       # soft's relative error scale
        soft_scale = s * s_rel
        g = ds.to(DEV, F64).abs() if ds is not None else torch.zeros_like(z)
        lm = (dl_mag if dl_mag is not None else dl).to(DEV, F64).abs() if dl is not None else torch.zeros_like(z)
        sg = s * s_rel * g
        da_mag = lm + sg + s * s_rel * sg.sum(-1, keepdim=True)
        D = da_mag
        if pr is not None:
            p_rel = 1 + za + zmax + lse.abs()
            D = D + torch.exp(z - lse) * p_rel * da_mag.sum(-1, keepdim=True)
        dq_scale = torch.empty_like(q64)
        dk_scale = torch.empty_like(k64)
        for b in range(B):                                          # 0.001 sum D |q_i - k_j|, one item at a time
            ad = (q64[b, :, None] - k64[b, None]).abs()             # (Tq, Tk, C)
            dq_scale[b] = 0.001 * torch.einsum("ij,ijc->ic", D[b], ad)
            dk_scale[b] = 0.001 * torch.einsum("ij,ijc->jc", D[b], ad)
    ref = {"logprob": lp.detach(), "soft": soft.detach(), "dz": dz, "dq": dq, "dk": dk}
    scale = {"logprob": lp_scale, "soft": soft_scale, "dz": D, "dq": dq_scale, "dk": dk_scale}
    return ref, scale


def _check_attention(q, k, prior, key_len, ds, dl, case):
    """Kernel against the float64 reference per element, twice with the same bits, and every item run by itself equal
    to its rows of the batch."""
    args = [None if t is None else t.to(DEV).contiguous() for t in (q, k, prior)]
    grads = [None if t is None else t.to(DEV).float().contiguous() for t in (ds, dl)]
    got = _attn_kernel(*args, key_len, *grads)
    _same_bits(got, _attn_kernel(*args, key_len, *grads), case + " rerun")
    for b in range(q.shape[0]):
        sl = lambda t: None if t is None else t[b:b + 1].contiguous()
        one = _attn_kernel(*(sl(t) for t in args), key_len[b:b + 1], *(sl(t) for t in grads))
        _same_bits({kk: v for kk, v in one.items()}, {kk: v[b:b + 1] for kk, v in got.items()}, f"{case} item {b} alone")
    ref, scale = _attn_reference(q, k, prior, key_len, ds, dl)
    _check("z" if prior is None else "logprob", got["logprob"], ref["logprob"], scale["logprob"], case)
    _check("soft", got["soft"], ref["soft"], scale["soft"], case)
    for name in ("dz", "dq", "dk"):
        _check(name, got[name], ref[name], scale[name], case)
    return got


def _attn_case(B, Tq, Tk, C, key_len, seed, prior_kind):
    gen = torch.Generator().manual_seed(seed)
    q = torch.randn(B, Tq, C, generator=gen) * 3
    k = torch.randn(B, Tk, C, generator=gen) * 3
    prior = None
    if prior_kind == "rand":
        prior = torch.rand(B, Tq, Tk, generator=gen)
        prior[:, :, -1] = 0.0                                        # prior cells of exactly 0: log(1e-8)
        prior[:, ::3, 0] = 0.0
    ds = torch.randn(B, Tq, Tk, generator=gen)
    dl = torch.randn(B, Tq, Tk, generator=gen)
    return q, k, prior, torch.tensor(key_len), ds, dl


GRADS = {"soft": (True, False), "logprob": (False, True), "both": (True, True)}

# (B, t_q, t_k, c, key lengths): t_q % 8 in {1, 7} and t_q = 1 (ragged last query tile of 8 rows), t_k % 32 in {1, 31}
# (ragged last key tile of 32 keys), c in {1, 31, 33, 97, 128} (partial 32-lane channel blocks of the row kernels, every
# residue of the 8 channel groups of the per-key kernel), key lengths 1, t_k and above t_k (clamped)
ATTN_EDGES = {
    "tq1_tk33_c1": (3, 1, 33, 1, [1, 33, 50]),
    "tq9_tk31_c31": (2, 9, 31, 31, [31, 1]),
    "tq15_tk65_c33": (3, 15, 65, 33, [65, 64, 1000]),
    "tq57_tk95_c97": (2, 57, 95, 97, [40, 95]),
    "tq7_tk1_c128": (2, 7, 1, 128, [1, 5]),
    "tq129_tk63_c128": (2, 129, 63, 128, [63, 17]),
}


@pytest.mark.parametrize("grads", list(GRADS))
@pytest.mark.parametrize("prior_kind", ["none", "rand"])
@pytest.mark.parametrize("case", list(ATTN_EDGES))
def test_align_attention_edges_match_float64(case, prior_kind, grads):
    B, Tq, Tk, C, kl = ATTN_EDGES[case]
    q, k, prior, key_len, ds, dl = _attn_case(B, Tq, Tk, C, kl, Tq * 1000 + Tk * 10 + C, prior_kind)
    want_s, want_l = GRADS[grads]
    _check_attention(q, k, prior, key_len, ds if want_s else None, dl if want_l else None, f"{case}/{prior_kind}/{grads}")


def _mas_batch():
    import kantts_b200
    return make_mas_batch(kantts_b200.sambert_16k_mas_config(), torch.Generator().manual_seed(5))


@pytest.mark.parametrize("grads", list(GRADS))
@pytest.mark.parametrize("prior_kind", ["none", "batch"])
def test_align_attention_training_shape_matches_float64(prior_kind, grads):
    """B = 16, t_q = 1002 frames (ragged utterances padded to a multiple of outputs_per_step), t_k = 200 symbols, c = 80,
    key lengths and prior of make_mas_batch (a diagonal band, exact zeros outside each utterance)."""
    batch = _mas_batch()
    prior = batch["attn_priors"] if prior_kind == "batch" else None
    B, Tq, Tk = batch["attn_priors"].shape
    q, k, _, _, ds, dl = _attn_case(B, Tq, Tk, 80, [0] * B, 17, "none")
    want_s, want_l = GRADS[grads]
    _check_attention(q, k, prior, batch["valid_input_lengths"], ds if want_s else None, dl if want_l else None,
                     f"train/{prior_kind}/{grads}")


# ------------------------------------------------------------------------------------------------
# forward-sum (CTC) loss
# ------------------------------------------------------------------------------------------------


def _ctc_kernel(lp, in_len, out_len, d_loss, blank=-1.0):
    """kt_attn_ctc_fwd then kt_attn_ctc_bwd; d_logprob prefilled with NaN, so that an element left unwritten fails."""
    lib = _ops()[0].load()
    B, Tq, Tk = lp.shape
    n = int(lib.kt_attn_ctc_workspace_bytes(B, Tq, Tk))
    ws = torch.empty(n // 4, device=DEV)
    loss = torch.full((1,), float("nan"), device=DEV)
    grad = torch.full_like(lp, float("nan"))
    il, ol = _i32(in_len), _i32(out_len)
    dloss = torch.tensor([d_loss], device=DEV)
    _call("kt_attn_ctc_fwd", _ptr(lp), _ptr(il, True), _ptr(ol, True), _ptr(loss), _ptr(ws), n, B, Tq, Tk, blank)
    _call("kt_attn_ctc_bwd", _ptr(lp), _ptr(il, True), _ptr(ol, True), _ptr(dloss), _ptr(ws), n, _ptr(grad), B, Tq, Tk,
          blank)
    torch.cuda.synchronize()
    return {"loss": loss, "grad": grad}


def _ctc_reference(lp, in_len, out_len, d_loss, blank=-1.0):
    """float64 on the CPU: oracle.sambert_mas.forward_sum_loss and autograd on the clamped lengths, with the error scales
    of the loss and of every gradient element, and the per-utterance losses nll_b / N_b (0 when infinite)."""
    from oracle import sambert_mas as om
    B, Tq, Tk = lp.shape
    il = in_len.cpu().long().clamp(max=Tk)
    ol = out_len.cpu().long().clamp(max=Tq)
    x = lp.detach().cpu().to(F64).requires_grad_(True)
    loss = om.forward_sum_loss(x[:, None], il, ol, blank)
    (grad,) = torch.autograd.grad(loss * d_loss, [x])
    grad_scale = torch.zeros(B, Tq, Tk, dtype=F64)
    per_item = torch.zeros(B, dtype=F64)
    item_scale = torch.zeros(B, dtype=F64)
    with torch.no_grad():
        for b in range(B):
            T, N = int(ol[b]), int(il[b])
            per_item[b] = om.forward_sum_loss(x[b:b + 1, None], il[b:b + 1], ol[b:b + 1], blank)
            if T < 1 or N < 1 or per_item[b] == 0:
                continue
            padded = torch.cat([torch.full((T, 1), blank, dtype=F64), x[b, :T, :N]], -1)
            lse = torch.logsumexp(padded, -1, keepdim=True)
            y = padded[:, 1:] - lse
            g = d_loss / (B * N)
            sm = torch.exp(y)
            post = sm - grad[b, :T, :N] / g
            grad_scale[b, :T, :N] = g * (sm * (1 + y.abs() + lse.abs()) + post.abs())
            item_scale[b] = (float(per_item[b]) * N + float(lse.abs().sum())) / N
    scale = {"loss": item_scale.mean().reshape(1), "grad": grad_scale, "item_loss": item_scale}
    return {"loss": loss.detach().reshape(1), "grad": grad, "item_loss": per_item}, scale


def _check_ctc(lp, in_len, out_len, case, d_loss=1.75):
    """The kernel pair against float64 per element (the mean loss, each utterance's loss, every gradient element), twice
    with the same bits, and each item run by itself with d_loss / B equal to its rows of the batch (B a power of two:
    d_loss / B is exact, so the item's gradient factor d_loss / (B N) rounds the same)."""
    B = lp.shape[0]
    lp = lp.to(DEV).float().contiguous()
    got = _ctc_kernel(lp, in_len, out_len, d_loss)
    _same_bits(got, _ctc_kernel(lp, in_len, out_len, d_loss), case + " rerun")
    ref, scale = _ctc_reference(lp, in_len, out_len, d_loss)
    _check("ctc_loss", got["loss"], ref["loss"], scale["loss"], case)
    _check("ctc", got["grad"], ref["grad"], scale["grad"], case)
    rl2 = rel_l2(got["grad"].cpu(), ref["grad"]) if float(ref["grad"].abs().max()) > 0 else 0.0
    print(f"align_arms {case} ctc: gradient relative L2 {rl2:.3g}, loss {float(got['loss'][0]):.9g} vs "
          f"{float(ref['loss'][0]):.9g}")
    assert rl2 <= 1e-5, (case, rl2)
    if B & (B - 1) == 0:
        for b in range(B):
            one = _ctc_kernel(lp[b:b + 1].contiguous(), in_len[b:b + 1], out_len[b:b + 1], d_loss / B)
            assert torch.equal(one["grad"][0], got["grad"][b]), (case, b)
            _check("ctc_loss", one["loss"], ref["item_loss"][b:b + 1], scale["item_loss"][b:b + 1], f"{case} item {b}")
    return got


def _ragged_train_lengths(B=16, L=200, T=1000):
    batch_in = torch.tensor([L - 1 - (17 * b) % (L // 2) for b in range(B)])
    batch_out = torch.tensor([T - (37 * b) % (T // 3) for b in range(B)])
    return batch_in, batch_out


def test_attn_ctc_training_shape_flat_rows_matches_float64():
    """B = 16, T ragged up to 1000 frames, N ragged up to 199 symbols: log_softmax(3 randn) rows, as flat as training's
    first steps."""
    il, ol = _ragged_train_lengths()
    gen = torch.Generator().manual_seed(11)
    lp = torch.log_softmax(3 * torch.randn(16, 1002, 200, generator=gen), -1)
    _check_ctc(lp, il, ol, "train_flat")


def test_attn_ctc_training_shape_attention_rows_matches_float64():
    """The same lengths, with the logprob rows the distance attention makes from make_mas_batch's prior."""
    batch = _mas_batch()
    B, Tq, Tk = batch["attn_priors"].shape
    gen = torch.Generator().manual_seed(12)
    q = (torch.randn(B, Tq, 80, generator=gen) * 3).to(DEV)
    k = (torch.randn(B, Tk, 80, generator=gen) * 3).to(DEV)
    _, lp = _ops()[2].AlignAttnFn.apply(q, k, batch["attn_priors"].to(DEV), batch["valid_input_lengths"].to(DEV))
    _check_ctc(lp[:, 0].detach(), batch["valid_input_lengths"], batch["valid_output_lengths"], "train_attn")


# (t_q, t_k, [(T, N)] per utterance): N >= 128 (S = 2N + 1 > 256 states, so threads own two or three), N at the kernel's
# shared-memory limit, N = 1, T = 1, T = N (a single path), T < N (infinite: zero loss and gradient), lengths above t_q /
# t_k (clamped)
CTC_EDGES = {
    "n128_s257": (300, 128, [(300, 128), (257, 128)]),
    "n300_s601": (700, 300, [(700, 300), (650, 299), (301, 300), (500, 150)]),
    "n1_t1": (4, 3, [(1, 1), (4, 1), (1, 3), (3, 3)]),
    "t_eq_n": (40, 40, [(40, 40), (17, 17)]),
    "t_lt_n": (30, 40, [(30, 40), (20, 25), (30, 10), (1, 2)]),
    "clamped": (50, 20, [(80, 45), (50, 20), (60, 7), (9, 300)]),
}


@pytest.mark.parametrize("case", list(CTC_EDGES))
def test_attn_ctc_edges_match_float64(case):
    Tq, Tk, lens = CTC_EDGES[case]
    B = len(lens)
    gen = torch.Generator().manual_seed(Tq * 31 + Tk)
    lp = torch.log_softmax(3 * torch.randn(B, Tq, Tk, generator=gen), -1)
    got = _check_ctc(lp, torch.tensor([n for _, n in lens]), torch.tensor([t for t, _ in lens]), case)
    for b, (T, N) in enumerate(lens):
        if min(T, Tq) < min(N, Tk):
            assert float(got["grad"][b].abs().max()) == 0.0, (case, b)


def test_attn_ctc_at_the_shared_memory_limit_matches_float64():
    """t_k = 3071: the largest key count whose two state rows fit the kernel's 96 KiB of shared memory, one utterance
    using all of it; one more key is refused."""
    lib = _ops()[0].load()
    Tq, Tk = 3200, 3071
    gen = torch.Generator().manual_seed(3071)
    lp = torch.log_softmax(3 * torch.randn(2, Tq, Tk, generator=gen), -1)
    _check_ctc(lp, torch.tensor([Tk, 2000]), torch.tensor([Tq, 2500]), "smem_limit")
    x = torch.zeros(1, 8, Tk + 1, device=DEV)
    n = int(lib.kt_attn_ctc_workspace_bytes(1, 8, Tk + 1))
    ws = torch.empty(n // 4, device=DEV)
    one = _i32(torch.tensor([1]))
    with pytest.raises(RuntimeError, match="shared-memory"):
        _call("kt_attn_ctc_fwd", _ptr(x), _ptr(one, True), _ptr(one, True), _ptr(torch.empty(1, device=DEV)), _ptr(ws), n,
              1, 8, Tk + 1, -1.0)


# ------------------------------------------------------------------------------------------------
# MAS
# ------------------------------------------------------------------------------------------------


def _mas_kernel(soft, in_len, out_len):
    lib = _ops()[0].load()
    B, Tq, Tk = soft.shape
    n = int(lib.kt_mas_workspace_bytes(B, Tq, Tk))
    ws = torch.empty(max(1, n // 4), device=DEV, dtype=torch.int32)
    hard = torch.full((B, Tq, Tk), float("nan"), device=DEV)
    dur = torch.full((B, Tk), float("nan"), device=DEV)
    il, ol = _i32(in_len), _i32(out_len)                  # held until the launch: their memory must not be reused
    _call("kt_mas", _ptr(soft), _ptr(il, True), _ptr(ol, True), _ptr(hard), _ptr(dur), _ptr(ws, True), n, B, Tq, Tk)
    torch.cuda.synchronize()
    return {"hard": hard, "dur": dur}


def _check_mas(soft, in_len, out_len, case):
    """kt_mas against oracle.sambert_mas.b_mas on the clamped lengths, bit for bit; twice; each item alone."""
    from oracle import sambert_mas as om
    B, Tq, Tk = soft.shape
    soft = soft.to(DEV).float().contiguous()
    got = _mas_kernel(soft, in_len, out_len)
    _same_bits(got, _mas_kernel(soft, in_len, out_len), case + " rerun")
    with np.errstate(divide="ignore", invalid="ignore"):
        want = om.b_mas(soft.cpu().numpy()[:, None], in_len.clamp(max=Tk).numpy(), out_len.clamp(max=Tq).numpy())[:, 0]
    assert torch.equal(got["hard"].cpu(), torch.from_numpy(want)), case
    assert torch.equal(got["dur"].cpu(), torch.from_numpy(want.sum(1))), case
    for b in range(B):
        one = _mas_kernel(soft[b:b + 1].contiguous(), in_len[b:b + 1], out_len[b:b + 1])
        assert torch.equal(one["hard"][0], got["hard"][b]) and torch.equal(one["dur"][0], got["dur"][b]), (case, b)
    return got


def test_mas_edges_match_oracle():
    """T = 1, N = 1, N > T, lengths above t_q / t_k (clamped), rows and whole maps of all-zero soft (log 0 = -inf: every
    comparison a tie, resolved towards key j - 1 as in the reference)."""
    gen = torch.Generator().manual_seed(21)
    Tq, Tk = 12, 20
    soft = torch.softmax(2 * torch.randn(8, Tq, Tk, generator=gen), -1)
    lens = [(1, 1), (1, 7), (5, 9), (12, 3), (40, 50), (12, 20), (12, 20), (9, 6)]
    soft[5, 3:6] = 0.0                                                # zero rows inside the path
    soft[6] = 0.0                                                     # an all-zero map
    soft[7, :, 2] = 0.0                                               # a zero key column
    from oracle import sambert_mas as om
    for b, (t, n) in enumerate(lens):                                 # every decision on the path clear of rounding
        assert om.mas_margin(soft[b, : min(t, Tq), : min(n, Tk)].numpy()) > 1e-3, b
    _check_mas(soft, torch.tensor([n for _, n in lens]), torch.tensor([t for t, _ in lens]), "edges")


@pytest.mark.parametrize("t_q", [3072, 3073])
def test_mas_decision_bits_switch_from_shared_memory_to_workspace(t_q):
    """t_k = 256 keys (8 words of decision bits per row): 3072 rows fill exactly 96 KiB of shared memory, 3073 go to the
    global workspace."""
    lib = _ops()[0].load()
    B, Tk = 2, 256
    assert lib.kt_mas_workspace_bytes(B, t_q, Tk) == (0 if t_q == 3072 else B * t_q * 8 * 4)
    soft, in_len, out_len = _random_maps(B, t_q, Tk, torch.Generator().manual_seed(3085))
    from oracle import sambert_mas as om
    for b in range(B):
        assert om.mas_margin(soft[b, 0, : int(out_len[b]), : int(in_len[b])].numpy()) > 1e-3, b
    _check_mas(soft[:, 0], in_len, out_len, f"switch_{t_q}")


# ------------------------------------------------------------------------------------------------
# the composed alignment loss of one training batch
# ------------------------------------------------------------------------------------------------


def test_alignment_loss_chain_at_training_size_matches_float64():
    """make_mas_batch's batch: the distance attention with its prior -> MAS -> the binarization loss (warm-up over) plus
    the forward-sum loss, backward to q and k on the kernels, against the float64 oracle chain on the same hard alignment
    (which must be the oracle's MAS of the kernel's soft map)."""
    from kantts_b200 import sambert
    from oracle import sambert_mas as om
    sops = _ops()[2]
    batch = _mas_batch()
    prior, il, ol = batch["attn_priors"], batch["valid_input_lengths"], batch["valid_output_lengths"]
    B, Tq, Tk = prior.shape
    gen = torch.Generator().manual_seed(23)
    q0 = torch.randn(B, Tq, 80, generator=gen) * 3
    k0 = torch.randn(B, Tk, 80, generator=gen) * 3
    runs = []
    for _ in range(2):
        q, k = q0.to(DEV).requires_grad_(True), k0.to(DEV).requires_grad_(True)
        soft, lp = sops.AlignAttnFn.apply(q, k, prior.to(DEV), il.to(DEV))
        hard, _ = sops.mas(soft, il.to(DEV), ol.to(DEV))
        loss = (sops.AttnCtcFn.apply(lp, il.to(DEV), ol.to(DEV), -1.0)
                + sambert.AttentionBinarizationLoss(0, 100)(100, hard, soft))
        loss.backward()
        runs.append({"loss": loss.detach(), "hard": hard, "dq": q.grad, "dk": k.grad, "soft": soft.detach()})
    _same_bits(runs[0], runs[1], "chain rerun")
    got = runs[0]
    hard = got["hard"][:, 0].cpu()
    with np.errstate(divide="ignore"):
        want = om.b_mas(got["soft"].cpu().numpy(), il.numpy(), ol.numpy())[:, 0]
    assert torch.equal(hard, torch.from_numpy(want))
    # the upstream gradients in float64: the binarization loss through soft, the forward-sum loss through logprob
    ref0, _ = _attn_reference(q0, k0, prior, il, None, torch.zeros(B, Tq, Tk))
    S = ref0["soft"].cpu().requires_grad_(True)
    Lp = ref0["logprob"].cpu().requires_grad_(True)
    loss64 = om.forward_sum_loss(Lp[:, None], il, ol) + om.binarization_loss(100, hard[:, None].to(F64), S[:, None])
    ds, dl = torch.autograd.grad(loss64, [S, Lp])
    _, ctc_scale = _ctc_reference(ref0["logprob"].float(), il, ol, 1.0)
    assert abs(float(got["loss"]) - float(loss64)) <= 1e-5 * abs(float(loss64)), (float(got["loss"]), float(loss64))
    ref, scale = _attn_reference(q0, k0, prior, il, ds, dl, dl_mag=ctc_scale["grad"])
    _check("dq", got["dq"], ref["dq"], scale["dq"], "chain")
    _check("dk", got["dk"], ref["dk"], scale["dk"], "chain")
    for name in ("dq", "dk"):
        r = rel_l2(got[name].cpu(), ref[name].cpu())
        print(f"align_arms chain {name}: relative L2 {r:.3g}")
        assert r <= 1e-5, (name, r)
