"""autograd wrappers of the SAM-BERT entry points of libkantts_b200.so (LayerNorm, multi-head attention,
FSMN memory block, LengthRegulator gather, LSTM recurrence, filled-pause insertion).  Same contract as ops.py: CUDA fp32 tensors only, explicit
stream, RuntimeError on any failure -- no PyTorch / CPU fallback."""
import ctypes
import math

import torch

from . import _lib, ops
from ._lib import KtAttnDesc, ptr
from .ops import call


def _u8(mask):
    """bool mask -> uint8 view for the C ABI (zero-copy)."""
    if mask is None:
        return None
    m = mask.contiguous()
    return m.view(torch.uint8) if m.dtype == torch.bool else m


class LayerNormFn(torch.autograd.Function):
    """nn.LayerNorm over the last dim (kt_layernorm_fwd / kt_layernorm_bwd)."""

    @staticmethod
    def forward(ctx, x, gamma, beta, eps):
        x = x.contiguous()
        c = x.shape[-1]
        rows = x.numel() // c
        y = torch.empty_like(x)
        mean = torch.empty(rows, device=x.device, dtype=torch.float32)
        rstd = torch.empty(rows, device=x.device, dtype=torch.float32)
        call("kt_layernorm_fwd", ptr(x), ptr(gamma.detach()), ptr(beta.detach()), ptr(y), ptr(mean), ptr(rstd), rows, c,
             float(eps))
        ctx.save_for_backward(x, gamma, mean, rstd)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, gamma, mean, rstd = ctx.saved_tensors
        c = x.shape[-1]
        rows = x.numel() // c
        dy = dy.contiguous()
        dx = torch.empty_like(x)
        dgamma = torch.empty_like(gamma)
        dbeta = torch.empty_like(gamma)
        n = int(_lib.load().kt_layernorm_bwd_workspace(rows, c))
        ws = torch.empty(n, device=x.device, dtype=torch.float32)
        call("kt_layernorm_bwd", ptr(dy), ptr(x), ptr(gamma.detach()), ptr(mean), ptr(rstd), ptr(dx), ptr(dgamma), ptr(dbeta),
             ptr(ws), n, rows, c, launches=2)
        return dx, dgamma, dbeta, None


def layer_norm(x, gamma, beta, eps):
    return LayerNormFn.apply(x, gamma, beta, eps)


def _attn_desc(B, H, D, lq, lk, qs, ks, vs, os_, mask, p_drop=0.0):
    d = KtAttnDesc(batch=B, heads=H, d_head=D, lq=lq, lk=lk, q_stride=qs, k_stride=ks, v_stride=vs, o_stride=os_,
                   mask_q_stride=0, mask_b_stride=0, scale=float(D) ** -0.5, keep_scale=1.0 / (1.0 - p_drop))
    if mask is not None:
        if mask.dim() == 2:                      # (B, Lk) key-padding mask, broadcast over the queries
            assert mask.shape == (B, lk), (mask.shape, B, lk)
            d.mask_q_stride, d.mask_b_stride = 0, lk
        else:                                    # (B or 1, Lq, Lk)
            assert mask.shape[1:] == (lq, lk) and mask.shape[0] in (1, B), (mask.shape, B, lq, lk)
            d.mask_q_stride, d.mask_b_stride = lk, (lq * lk if mask.shape[0] == B else 0)
    return d


def _keep_mask(p_drop, shape, device):
    """nn.Dropout(p) on the attention probabilities (sambert/__init__.py:26): Bernoulli keep mask, uint8."""
    if p_drop <= 0.0:
        return None
    return (torch.rand(shape, device=device) >= p_drop).view(torch.uint8)


def _off(t, col):
    """device address of column `col` of the first row of a contiguous row tensor."""
    return ptr(t) + 4 * col


class SelfAttnFn(torch.autograd.Function):
    """softmax(Q K^T / sqrt(d) + mask) V over all heads, straight from the fused QKV projection
    (sambert/__init__.py:80-100).  qkv: (B, L, 3*H*D) -> out (B, L, H*D), probs (H*B, L, L)."""

    @staticmethod
    def forward(ctx, qkv, mask, n_head, p_drop=0.0, keep=None):
        qkv = qkv.contiguous()
        B, L, w = qkv.shape
        hd = w // 3
        D = hd // n_head
        m = _u8(mask)
        d = _attn_desc(B, n_head, D, L, L, w, w, w, hd, m, p_drop)
        out = torch.empty(B, L, hd, device=qkv.device, dtype=torch.float32)
        probs = torch.empty(n_head * B, L, L, device=qkv.device, dtype=torch.float32)
        keep = _u8(keep) if keep is not None else _keep_mask(p_drop, probs.shape, qkv.device)
        dropped = torch.empty_like(probs) if keep is not None else None
        call("kt_attention_fwd", ctypes.byref(d), _off(qkv, 0), _off(qkv, hd), _off(qkv, 2 * hd), ptr(m, True), ptr(keep, True),
             ptr(out), ptr(probs), ptr(dropped))
        ctx.d, ctx.hd = d, hd
        ctx.save_for_backward(qkv, probs, keep)
        attn = probs if dropped is None else dropped
        ctx.mark_non_differentiable(attn)
        return out, attn

    @staticmethod
    def backward(ctx, dout, _dprobs):
        qkv, probs, keep = ctx.saved_tensors
        d, hd = ctx.d, ctx.hd
        dout = dout.contiguous()
        dqkv = torch.empty_like(qkv)
        delta = torch.empty(d.heads * d.batch * d.lq, device=qkv.device, dtype=torch.float32)
        call("kt_attention_bwd", ctypes.byref(d), _off(qkv, 0), _off(qkv, hd), _off(qkv, 2 * hd), ptr(probs), ptr(keep, True),
             ptr(dout), _off(dqkv, 0), _off(dqkv, hd), _off(dqkv, 2 * hd), ptr(delta), 0, launches=2)
        return dqkv, None, None, None, None


class PncaAttnFn(torch.autograd.Function):
    """The two attentions of MultiHeadPNCAAttention (sambert/__init__.py:269-300) sharing their queries:
    x_qkv (B, L, 3HD) self part under the causal band mask, h_kv (B, Lh, 2HD) memory part under the
    look-ahead band mask.  -> out_x, out_h (B, L, HD), probs_x (H*B, L, L), probs_h (H*B, L, Lh)."""

    @staticmethod
    def forward(ctx, x_qkv, h_kv, mask_x, mask_h, n_head, p_drop=0.0, keep_x=None, keep_h=None):
        x_qkv, h_kv = x_qkv.contiguous(), h_kv.contiguous()
        B, L, w = x_qkv.shape
        hd = w // 3
        D = hd // n_head
        Lh = h_kv.shape[1]
        mx, mh = _u8(mask_x), _u8(mask_h)
        dx = _attn_desc(B, n_head, D, L, L, w, w, w, hd, mx, p_drop)
        dh = _attn_desc(B, n_head, D, L, Lh, w, 2 * hd, 2 * hd, hd, mh, p_drop)
        out_x = torch.empty(B, L, hd, device=x_qkv.device, dtype=torch.float32)
        out_h = torch.empty_like(out_x)
        px = torch.empty(n_head * B, L, L, device=x_qkv.device, dtype=torch.float32)
        ph = torch.empty(n_head * B, L, Lh, device=x_qkv.device, dtype=torch.float32)
        kx = _u8(keep_x) if keep_x is not None else _keep_mask(p_drop, px.shape, x_qkv.device)
        kh = _u8(keep_h) if keep_h is not None else _keep_mask(p_drop, ph.shape, x_qkv.device)
        pxd = torch.empty_like(px) if kx is not None else None
        phd = torch.empty_like(ph) if kh is not None else None
        call("kt_attention_fwd", ctypes.byref(dx), _off(x_qkv, 0), _off(x_qkv, hd), _off(x_qkv, 2 * hd), ptr(mx, True),
             ptr(kx, True), ptr(out_x), ptr(px), ptr(pxd))
        call("kt_attention_fwd", ctypes.byref(dh), _off(x_qkv, 0), _off(h_kv, 0), _off(h_kv, hd), ptr(mh, True), ptr(kh, True),
             ptr(out_h), ptr(ph), ptr(phd))
        ctx.dx, ctx.dh, ctx.hd = dx, dh, hd
        ctx.save_for_backward(x_qkv, h_kv, px, ph, kx, kh)
        ax = px if pxd is None else pxd
        ah = ph if phd is None else phd
        ctx.mark_non_differentiable(ax, ah)
        return out_x, out_h, ax, ah

    @staticmethod
    def backward(ctx, dox, doh, _dpx, _dph):
        x_qkv, h_kv, px, ph, kx, kh = ctx.saved_tensors
        dx, dh, hd = ctx.dx, ctx.dh, ctx.hd
        dox, doh = dox.contiguous(), doh.contiguous()
        dqkv = torch.empty_like(x_qkv)
        dhkv = torch.empty_like(h_kv)
        delta = torch.empty(dx.heads * dx.batch * dx.lq, device=x_qkv.device, dtype=torch.float32)
        call("kt_attention_bwd", ctypes.byref(dx), _off(x_qkv, 0), _off(x_qkv, hd), _off(x_qkv, 2 * hd), ptr(px), ptr(kx, True),
             ptr(dox), _off(dqkv, 0), _off(dqkv, hd), _off(dqkv, 2 * hd), ptr(delta), 0, launches=2)
        call("kt_attention_bwd", ctypes.byref(dh), _off(x_qkv, 0), _off(h_kv, 0), _off(h_kv, hd), ptr(ph), ptr(kh, True),
             ptr(doh), _off(dqkv, 0), _off(dhkv, 0), _off(dhkv, hd), ptr(delta), 1, launches=2)
        return dqkv, dhkv, None, None, None, None, None, None


def pnca_step_slots(q_row, x_kv, h_kv, st, n_head):
    """One decoder step of MultiHeadPNCAAttention for every slot of a SlotDecoder at its own step (kt_pnca_step_slots):
    q_row (B, 1, 3HD); x_kv / h_kv (B, max_steps, 2HD), x_kv's row at each active slot's step written here; ``st`` holds
    the device arrays step, mem_len, x_bw, h_bw (int32) and active (uint8).  -> out_x, out_h (B, 1, HD), zero for an
    inactive slot."""
    B, _, w = q_row.shape
    hd = w // 3
    out_x = torch.empty(B, 1, hd, device=q_row.device, dtype=torch.float32)
    out_h = torch.empty_like(out_x)
    call("kt_pnca_step_slots", ptr(q_row), ptr(x_kv), ptr(h_kv), ptr(st.step, True), ptr(st.mem_len, True), ptr(st.x_bw, True),
         ptr(st.h_bw, True), ptr(st.active, True), ptr(out_x), ptr(out_h), B, n_head, hd // n_head, x_kv.shape[1])
    return out_x, out_h


def pnca_attn_step(q_row, x_cache, h_kv, mask_x, mask_h, n_head):
    """One free-running decoder step of MultiHeadPNCAAttention (sambert/__init__.py:212-300), inference only.
    q_row (B, 1, 3HD): this step's fused QKV projection (only its q block is read here; the caller has already written
    the row into ``x_cache``); x_cache (B, Lmax, 3HD): the preallocated K/V state of the self part (rows beyond the
    current step are masked by ``mask_x`` (B or 1, 1, Lmax), so the reference's ``torch.cat`` growth is never needed);
    h_kv (B, Lh, 2HD): the memory keys / values projected once; mask_h (B or 1, 1, Lh).
    -> out_x, out_h (B, 1, HD), probs_x (H*B, 1, Lmax), probs_h (H*B, 1, Lh)."""
    assert q_row.is_contiguous() and x_cache.is_contiguous() and h_kv.is_contiguous()
    B, _, w = q_row.shape
    hd = w // 3
    D = hd // n_head
    lmax, lh = x_cache.shape[1], h_kv.shape[1]
    mx, mh = _u8(mask_x), _u8(mask_h)
    dx = _attn_desc(B, n_head, D, 1, lmax, w, w, w, hd, mx)
    dh = _attn_desc(B, n_head, D, 1, lh, w, 2 * hd, 2 * hd, hd, mh)
    out_x = torch.empty(B, 1, hd, device=q_row.device, dtype=torch.float32)
    out_h = torch.empty_like(out_x)
    px = torch.empty(n_head * B, 1, lmax, device=q_row.device, dtype=torch.float32)
    ph = torch.empty(n_head * B, 1, lh, device=q_row.device, dtype=torch.float32)
    call("kt_attention_fwd", ctypes.byref(dx), _off(q_row, 0), _off(x_cache, hd), _off(x_cache, 2 * hd), ptr(mx, True), None,
         ptr(out_x), ptr(px), None)
    call("kt_attention_fwd", ctypes.byref(dh), _off(q_row, 0), _off(h_kv, 0), _off(h_kv, hd), ptr(mh, True), None, ptr(out_h),
         ptr(ph), None)
    return out_x, out_h, px, ph


class FsmnMemoryFn(torch.autograd.Function):
    """MemoryBlockV2 (fsmn.py:46-77).  x (B, T, C), w (C, 1, K), mask (B, T) bool or None."""

    @staticmethod
    def forward(ctx, x, w, mask, pad_left):
        x = x.contiguous()
        B, T, C = x.shape
        K = w.shape[-1]
        m = _u8(mask)
        y = torch.empty_like(x)
        call("kt_fsmn_fwd", ptr(x), ptr(w.detach().contiguous()), ptr(m, True), ptr(y), B, T, C, K, pad_left)
        ctx.pad_left = pad_left
        ctx.save_for_backward(x, w, m)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, m = ctx.saved_tensors
        B, T, C = x.shape
        K = w.shape[-1]
        dy = dy.contiguous()
        dx = torch.empty_like(x) if ctx.needs_input_grad[0] else None
        dw = ws = None
        n = 0
        if ctx.needs_input_grad[1]:
            dw = torch.empty_like(w)
            n = int(_lib.load().kt_fsmn_bwd_workspace(B, T, C, K))
            ws = torch.empty(n, device=x.device, dtype=torch.float32)
        call("kt_fsmn_bwd", ptr(x), ptr(dy), ptr(w.detach().contiguous()), ptr(m, True), ptr(dx), ptr(dw), ptr(ws), n, B, T, C,
             K, ctx.pad_left, launches=3)
        return dx, dw, None, None


class RowsGatherFn(torch.autograd.Function):
    """LengthRegulator expansion (adaptors.py:15-37) as a gather; idx (B, T_out) int32 (-1 = zero row),
    start / count (B, T_in) int32 = each input row's span of output rows."""

    @staticmethod
    def forward(ctx, x, idx, start, count):
        x = x.contiguous()
        B, T_in, C = x.shape
        T_out = idx.shape[1]
        out = torch.empty(B, T_out, C, device=x.device, dtype=torch.float32)
        call("kt_rows_gather_fwd", ptr(x), ptr(idx, True), ptr(out), B, T_out, T_in, C)
        ctx.save_for_backward(idx, start, count)
        ctx.t_in = T_in
        return out

    @staticmethod
    def backward(ctx, dout):
        idx, start, count = ctx.saved_tensors
        dout = dout.contiguous()
        B, T_out, C = dout.shape
        din = torch.empty(B, ctx.t_in, C, device=dout.device, dtype=torch.float32)
        call("kt_rows_gather_bwd", ptr(dout), ptr(idx, True), ptr(start, True), ptr(count, True), ptr(din), B, T_out, ctx.t_in, C)
        return din, None, None, None


class LstmFn(torch.autograd.Function):
    """The recurrence of one nn.LSTM layer (kt_lstm_train_fwd / _bwd), uni- or bidirectional: gx (B, T, D * 4H), the input
    projection x . W_ih^T + b_ih + b_hh of each direction, and whh (D * 4H, H), each direction's W_hh, -> h and the cell
    states c, (B, T, D * H) each.  ``lengths`` (device int32 (B,) or None): the packed semantics of pack_padded_sequence
    (rows >= lengths[b] of h and c are zero), or every row.  ``h0`` / ``c0`` (B, D, H) or None: the initial state of each
    direction (zeros when None).  ``grad``: whether the caller records autograd (the forward then keeps the cell states and
    gate activations for the backward).  The backward recurrence gives dgx and the initial state's gradient; dW_hh is the
    k = 1 weight gradient of the grouped (one group per direction) conv whose input is each row's recurrent input h_prev."""

    @staticmethod
    def forward(ctx, gx, whh, lengths, dirs, h0, c0, grad):
        gx = gx.contiguous()
        B, T, G = gx.shape
        H = G // (4 * dirs)
        w = whh.detach()
        whh_t = w.view(dirs, 4 * H, H).transpose(1, 2).contiguous()
        init = None if h0 is None else torch.stack([h0.detach(), c0.detach()], 2).contiguous()
        h = torch.empty(B, T, dirs * H, device=gx.device, dtype=torch.float32)
        c = torch.empty_like(h)
        save = grad and any(ctx.needs_input_grad[:2] + ctx.needs_input_grad[4:6])
        acts = torch.empty_like(gx) if save else None
        call("kt_lstm_train_fwd", ptr(gx), ptr(whh_t), ptr(lengths, True), ptr(init), ptr(h), ptr(c), ptr(acts), B, T, dirs, H)
        ctx.dirs = dirs
        # an unused c (the usual case) then reaches the backward as None, and the kernel reads no dc rows
        ctx.set_materialize_grads(False)
        if save:
            ctx.save_for_backward(h, c, acts, whh, lengths, init)
        return h, c

    @staticmethod
    def backward(ctx, dh, dc):
        h, c, acts, whh, lengths, init = ctx.saved_tensors
        B, T, DH = h.shape
        dirs = ctx.dirs
        H = DH // dirs
        dh = torch.zeros_like(h) if dh is None else dh.contiguous()
        dc = None if dc is None else dc.contiguous()
        w = whh.detach().contiguous()
        dgx = torch.empty_like(acts)
        h_prev = torch.empty_like(h)
        dstate = torch.empty_like(init) if init is not None and any(ctx.needs_input_grad[4:6]) else None
        call("kt_lstm_train_bwd", ptr(dh), ptr(dc), ptr(w), ptr(lengths, True), ptr(init), ptr(h), ptr(c), ptr(acts), ptr(dgx),
             ptr(h_prev), ptr(dstate), B, T, dirs, H)
        dwhh = None
        if ctx.needs_input_grad[1]:
            spec = _whh_spec(dirs, H)
            _, dwhh, _ = ops._weight_backward(spec, spec.plan(B, 1, T), h_prev, dgx, None, w, None, (whh, None, None), None,
                                              True, False, False)
            dwhh = dwhh.view_as(whh)
        dh0 = dc0 = None
        if dstate is not None:
            dh0, dc0 = dstate[:, :, 0], dstate[:, :, 1]
        return dgx, dwhh, None, None, dh0, dc0, None


_WHH_SPECS = {}


def _whh_spec(dirs, H):
    """The recurrent term h_prev . W_hh^T of all directions as one grouped k = 1 conv (its weight gradient is dW_hh)."""
    spec = _WHH_SPECS.get((dirs, H))
    if spec is None:
        spec = _WHH_SPECS[(dirs, H)] = ops.ConvSpec(c_in=dirs * H, c_out=dirs * 4 * H, kernel=1, groups=dirs)
    return spec


def lstm_layer(x, lstm, layer, lengths=None, state=None):
    """Layer ``layer`` of the nn.LSTM ``lstm`` (batch_first, its parameters as they are) over x (B, T, C) -> h (B, T, D * H),
    c (B, T, D * H).  The input projection of all directions is one k = 1 conv (ops.conv: dx, dW_ih and the biases' gradient
    come from its backward), the recurrence LstmFn.  ``lengths``: see LstmFn.  ``state``: None (zeros) or nn.LSTM's initial
    (h_0, c_0), each (num_layers * D, B, H)."""
    sfx = [f"_l{layer}"] + ([f"_l{layer}_reverse"] if lstm.bidirectional else [])
    p = lambda name: [getattr(lstm, name + s) for s in sfx]
    H, D = lstm.hidden_size, len(sfx)
    w_ih = torch.cat(p("weight_ih")).unsqueeze(-1)
    bias = torch.cat([bi + bh for bi, bh in zip(p("bias_ih"), p("bias_hh"))])
    specs = lstm.__dict__.setdefault("_kt_specs", {})
    spec = specs.get(layer)
    if spec is None:
        spec = specs[layer] = ops.ConvSpec(c_in=w_ih.shape[1], c_out=D * 4 * H, kernel=1)
    gx = ops.conv(x.contiguous(), spec, ops.PreparedWeight(), w_ih, None, bias)
    h0 = c0 = None
    if state is not None:
        h0, c0 = (t[layer * D:(layer + 1) * D].transpose(0, 1) for t in state)
    return LstmFn.apply(gx, torch.cat(p("weight_hh")), lengths, D, h0, c0, torch.is_grad_enabled())


def fp_insert_plan(input_lengths, length, fp_label=None, fp_p=None):
    """Index plan of KanTtsSAMBERT.insert_fp (kantts_sambert.py:766-860, kt_fp_insert_plan): from ``fp_label`` (B, L)
    integer labels (training) or the (B, L, 4) predictions ``fp_p`` (inference).  -> codes (B, t_cap) int32,
    rows (B, L) int32, inter_lengths (B,) int64, t_ins.  Reading t_ins is the one host synchronisation."""
    B = input_lengths.shape[0]
    lens = input_lengths.to(torch.int32).contiguous()
    if fp_label is not None:
        lab = fp_label if fp_label.dtype in (torch.int32, torch.int64) else fp_label.long()
        lab, nbytes, p, t_cap = lab.contiguous(), lab.element_size(), None, 4 * length
    else:
        lab, nbytes, p, t_cap = None, 0, fp_p.detach().contiguous(), 10 * length
    codes = torch.empty(B, t_cap, device=lens.device, dtype=torch.int32)
    rows = torch.empty(B, length, device=lens.device, dtype=torch.int32)
    inter = torch.empty(B, device=lens.device, dtype=torch.int32)
    call("kt_fp_insert_plan", ptr(lab, True), nbytes, ptr(p), ptr(lens, True), B, length, t_cap, ptr(codes, True),
         ptr(rows, True), ptr(inter, True))
    t_ins = length + int(inter.max() - lens.max())
    return codes, rows, inter.to(input_lengths.dtype), t_ins


class FpInsertFn(torch.autograd.Function):
    """Filled-pause splice of KanTtsSAMBERT.insert_fp as a row gather (kt_fp_insert_fwd / _bwd): text_hid (B, L, C)
    and fp_enc (3, 3, C), the text encoder's output for the three filled-pause symbol sequences, -> (B, t_ins, C)."""

    @staticmethod
    def forward(ctx, text_hid, fp_enc, codes, rows, t_ins):
        text_hid, fp_enc = text_hid.contiguous(), fp_enc.contiguous()
        B, L, C = text_hid.shape
        assert fp_enc.shape == (3, 3, C), fp_enc.shape
        out = torch.empty(B, t_ins, C, device=text_hid.device, dtype=torch.float32)
        call("kt_fp_insert_fwd", ptr(text_hid), ptr(fp_enc), ptr(codes, True), ptr(out), B, L, codes.shape[1], t_ins, C)
        ctx.save_for_backward(codes, rows)
        ctx.shape = (B, L, C)
        return out

    @staticmethod
    def backward(ctx, dout):
        codes, rows = ctx.saved_tensors
        B, L, C = ctx.shape
        dout = dout.contiguous()
        dev = dout.device
        dtext = torch.empty(B, L, C, device=dev, dtype=torch.float32) if ctx.needs_input_grad[0] else None
        dfp = torch.empty(3, 3, C, device=dev, dtype=torch.float32) if ctx.needs_input_grad[1] else None
        part = torch.empty(9 * B * C, device=dev, dtype=torch.float32) if dfp is not None else None
        call("kt_fp_insert_bwd", ptr(dout), ptr(codes, True), ptr(rows, True), ptr(dtext), ptr(dfp), ptr(part),
             0 if part is None else part.numel(), B, L, codes.shape[1], dout.shape[1], C, launches=1 + 2 * (dfp is not None))
        return dtext, dfp, None, None, None


# ------------------------------------------------------------------------------------------------
# alignment learning (MAS: True): kt_align_attn_*, kt_mas, kt_attn_ctc_*, kt_attn_prior
# ------------------------------------------------------------------------------------------------


def _i32(t):
    return t.to(torch.int32).contiguous()


class AlignAttnFn(torch.autograd.Function):
    """The distance attention of ConvAttention.forward (attention.py:100-125) after its two projections: queries q
    (B, T_mel, C) and keys k (B, T_text, C), as rows; the optional prior (B, T_mel, T_text); key_lengths (B,) (the padded
    keys are masked for ``soft`` only).  -> attn_soft, attn_logprob (B, 1, T_mel, T_text).  Both outputs carry gradient:
    the softmax backward through soft (masked keys excluded), then with a prior the log_softmax backward over all keys."""

    @staticmethod
    def forward(ctx, q, k, prior, key_lengths):
        q, k = q.contiguous(), k.contiguous()
        B, Tq, C = q.shape
        Tk = k.shape[1]
        pr = None if prior is None else prior.contiguous()
        if pr is not None:
            assert pr.shape == (B, Tq, Tk), (pr.shape, B, Tq, Tk)
        kl = _i32(key_lengths)
        logprob = torch.empty(B, Tq, Tk, device=q.device, dtype=torch.float32)
        soft = torch.empty_like(logprob)
        lse = torch.empty(B, Tq, device=q.device, dtype=torch.float32) if pr is not None else None
        call("kt_align_attn_fwd", ptr(q), ptr(k), ptr(pr), ptr(kl, True), ptr(logprob), ptr(soft), ptr(lse), B, Tq, Tk, C)
        ctx.save_for_backward(q, k, pr, soft, lse)
        return soft.view(B, 1, Tq, Tk), logprob.view(B, 1, Tq, Tk)

    @staticmethod
    def backward(ctx, d_soft, d_logprob):
        q, k, pr, soft, lse = ctx.saved_tensors
        B, Tq, C = q.shape
        Tk = k.shape[1]
        ds = None if d_soft is None else d_soft.reshape(B, Tq, Tk).contiguous()
        dl = None if d_logprob is None else d_logprob.reshape(B, Tq, Tk).contiguous()
        dq, dk = torch.empty_like(q), torch.empty_like(k)
        if ds is None and dl is None:
            return dq.zero_(), dk.zero_(), None, None
        dz = torch.empty(B, Tq, Tk, device=q.device, dtype=torch.float32)
        call("kt_align_attn_bwd", ptr(q), ptr(k), ptr(pr), ptr(soft), ptr(lse), ptr(ds), ptr(dl), ptr(dz), ptr(dq), ptr(dk),
             B, Tq, Tk, C, launches=2)
        return dq, dk, None, None


def mas(attn_soft, in_lengths, out_lengths):
    """binarize_attention_parallel (kantts_sambert.py:752-764) on the device, no autograd: mas_width1 of every
    attn_soft[b, 0, :out_lengths[b], :in_lengths[b]] (kt_mas).  -> attn_hard (B, 1, T_mel, T_text) and the durations
    attn_hard.sum(2) as (B, T_text) float32."""
    soft = attn_soft.detach().reshape(attn_soft.shape[0], attn_soft.shape[-2], attn_soft.shape[-1]).contiguous()
    B, Tq, Tk = soft.shape
    hard = torch.empty(B, 1, Tq, Tk, device=soft.device, dtype=torch.float32)
    dur = torch.empty(B, Tk, device=soft.device, dtype=torch.float32)
    n = int(_lib.load().kt_mas_workspace_bytes(B, Tq, Tk))
    ws = torch.empty((n + 3) // 4, device=soft.device, dtype=torch.int32) if n else None
    il, ol = _i32(in_lengths), _i32(out_lengths)          # held until the launch: their memory must not be reused
    call("kt_mas", ptr(soft), ptr(il, True), ptr(ol, True), ptr(hard), ptr(dur), ptr(ws, True), n, B, Tq, Tk)
    return hard, dur


class AttnCtcFn(torch.autograd.Function):
    """AttentionCTCLoss.forward (train/loss.py:488-508): attn_logprob (B, 1, T_mel, T_text), in_lengths / out_lengths (B,)
    -> the scalar mean over the batch of each utterance's CTC loss / in_length (0 when infinite).  The per-frame
    log_softmax over [blank, valid keys], the alpha / beta recursions and the gradient run in kt_attn_ctc_*."""

    @staticmethod
    def forward(ctx, attn_logprob, in_lengths, out_lengths, blank_logprob=-1.0):
        lp = attn_logprob.reshape(attn_logprob.shape[0], attn_logprob.shape[-2], attn_logprob.shape[-1]).contiguous()
        B, Tq, Tk = lp.shape
        il, ol = _i32(in_lengths), _i32(out_lengths)
        n = int(_lib.load().kt_attn_ctc_workspace_bytes(B, Tq, Tk))
        ws = torch.empty(n // 4, device=lp.device, dtype=torch.float32)
        loss = torch.empty((), device=lp.device, dtype=torch.float32)
        call("kt_attn_ctc_fwd", ptr(lp), ptr(il, True), ptr(ol, True), ptr(loss), ptr(ws), n, B, Tq, Tk, float(blank_logprob),
             launches=2)
        ctx.save_for_backward(lp, il, ol, ws)
        ctx.shape, ctx.blank = attn_logprob.shape, float(blank_logprob)
        return loss

    @staticmethod
    def backward(ctx, d_loss):
        lp, il, ol, ws = ctx.saved_tensors
        B, Tq, Tk = lp.shape
        d_lp = torch.empty_like(lp)
        d_loss = d_loss.contiguous()
        call("kt_attn_ctc_bwd", ptr(lp), ptr(il, True), ptr(ol, True), ptr(d_loss), ptr(ws), ws.numel() * 4,
             ptr(d_lp), B, Tq, Tk, ctx.blank)
        return d_lp.view(ctx.shape), None, None, None


def attn_prior(valid_input_lengths, valid_output_lengths, t_mel, t_text):
    """The collate's ``attn_priors`` on the device (kt_attn_prior): the beta-binomial prior of P = valid_input_lengths[b] + 1
    symbols over M = valid_output_lengths[b] frames (beta_binomial_prior_distribution, kantts/datasets/dataset.py:20-31),
    zero-padded to (B, t_mel, t_text) float32.  One launch, no host synchronisation."""
    il = valid_input_lengths.to(torch.int64).contiguous()
    ol = valid_output_lengths.to(torch.int64).contiguous()
    prior = torch.empty(il.shape[0], t_mel, t_text, device=il.device, dtype=torch.float32)
    call("kt_attn_prior", ptr(il, True), ptr(ol, True), ptr(prior), il.shape[0], int(t_mel), int(t_text))
    return prior


def average_frame_feat(feat, durs):
    """average_frame_feat (kantts_sambert.py:652-674) as device torch ops: feat (B, T_frames) frame values, durs (B, L)
    -> (B, L) the mean of each symbol's frames over its non-zero frames (0 when it has none), from cumulative-sum
    differences."""
    ends = torch.cumsum(durs, dim=1).long()
    starts = torch.nn.functional.pad(ends[:, :-1], (1, 0))
    nonzero = torch.nn.functional.pad(torch.cumsum(feat != 0.0, dim=1), (1, 0))
    sums = torch.nn.functional.pad(torch.cumsum(feat, dim=1), (1, 0))
    total = (torch.gather(sums, 1, ends) - torch.gather(sums, 1, starts)).float()
    count = (torch.gather(nonzero, 1, ends) - torch.gather(nonzero, 1, starts)).float()
    return torch.where(count == 0.0, count, total / count)


# masked-symbol pretraining (KanTtsTextsyBERT): kt_seq_ce_*, kt_bert_mask
# ------------------------------------------------------------------------------------------------


class SeqCEFn(torch.autograd.Function):
    """SeqCELoss.forward (train/loss.py:444-460): logits (..., V), int64 targets (...) and float masks (...) -> the masked
    mean cross-entropy ``loss`` and the masked argmax error rate ``err``, both 0-d device tensors.  One pass over the logits
    in kt_seq_ce_fwd (log-sum-exp, target logit, argmax with torch's first-index rule, fixed-order masked sums); ``err`` is
    not differentiable.  The backward is kt_seq_ce_bwd, with the incoming gradient and the mask sum read on the device."""

    @staticmethod
    def forward(ctx, logits, targets, masks):
        V = logits.shape[-1]
        x = logits.reshape(-1, V).contiguous()
        rows = x.shape[0]
        t = targets.reshape(-1).to(torch.int64).contiguous()
        m = masks.reshape(-1).to(torch.float32).contiguous()
        assert t.numel() == rows and m.numel() == rows, (logits.shape, targets.shape, masks.shape)
        dev = x.device
        lse = torch.empty(rows, device=dev, dtype=torch.float32)
        loss, err, msum = (torch.empty((), device=dev, dtype=torch.float32) for _ in range(3))
        n = int(_lib.load().kt_seq_ce_workspace_bytes(rows))
        ws = torch.empty(n // 8, device=dev, dtype=torch.float64)
        call("kt_seq_ce_fwd", ptr(x), ptr(t, True), ptr(m), ptr(lse), ptr(loss), ptr(err), ptr(msum), ptr(ws, True), n,
             rows, V, launches=2)
        ctx.save_for_backward(x, t, m, lse, msum)
        ctx.shape = logits.shape
        ctx.mark_non_differentiable(err)
        return loss, err

    @staticmethod
    def backward(ctx, d_loss, _d_err):
        x, t, m, lse, msum = ctx.saved_tensors
        dx = torch.empty_like(x)
        d_loss = d_loss.to(torch.float32).contiguous()
        call("kt_seq_ce_bwd", ptr(x), ptr(t, True), ptr(m), ptr(lse), ptr(msum), ptr(d_loss), ptr(dx),
             x.shape[0], x.shape[1])
        return dx.view(ctx.shape), None, None


def bert_mask(lings, valid_lengths, seed, call_index, mask_ratio, n_sy, mask_id):
    """BERT masking of the symbol column of ``lings`` (B, L, n_feat) int64 on the device (kt_bert_mask), positions
    [0, valid_lengths[b]) eligible.  -> (masked lings, targets = the unmasked symbol column (B, L) int64, bert_masks (B, L)
    float32 with 1 at the selected positions).  ``seed`` and ``call_index`` (host ints) key the draw."""
    x = lings.to(torch.int64).contiguous()
    B, L, F = x.shape
    vl = _i32(valid_lengths)
    out = torch.empty_like(x)
    targets = torch.empty(B, L, device=x.device, dtype=torch.int64)
    masks = torch.empty(B, L, device=x.device, dtype=torch.float32)
    threshold = math.ceil(float(mask_ratio) * 2.0 ** 32)
    call("kt_bert_mask", ptr(x, True), ptr(vl, True), ptr(out, True), ptr(targets, True), ptr(masks), B, L, F,
         _wrap64(seed), _wrap64(call_index), threshold, int(n_sy), int(mask_id))
    return out, targets, masks


def _wrap64(v):
    """A Python int as the int64 whose bits are its low 64 bits (seeds and call counters are unsigned 64-bit words)."""
    v = int(v) & 0xFFFFFFFFFFFFFFFF
    return v - (1 << 64) if v >= 1 << 63 else v
