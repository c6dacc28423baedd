"""H100-native SAM-BERT acoustic model with the reference's module API.

Drop-in for ``kantts.models.sambert.kantts_sambert.KanTtsSAMBERT`` (KAN-TTS
kantts/models/sambert/kantts_sambert.py:652-1044 and the blocks it is built from: sambert/__init__.py,
adaptors.py, fsmn.py, positions.py): same class names, the same single-dict constructor, the same forward
signature and result dict, identical ``state_dict`` keys / shapes / order and identical parameter
initialisation for a given ``torch.manual_seed`` (sub-modules are created in the reference's order from
the same torch initialisers).

Where the arithmetic runs:
  * every Linear / Conv1d (QKV and output projections, conv feed-forward, prenets, FSMN feed-forward,
    pitch / energy embeddings) -> the conv kernels of libkantts_b200.so (tensor-core split-bf16 or exact fp32 FFMA)
    through ops.ConvFn, on the model's native (B, L, C) rows, with bias / ReLU / residual fused;
  * LayerNorm, multi-head attention (both PNCA attentions, probabilities materialised like the reference),
    the FSMN memory block and the LengthRegulator expansion -> the kernels in csrc/sambert.cu;
  * the four LSTMs stay on cuDNN (``nn.LSTM``) -- SURVEY.md section 2c rules them out of scope for custom
    kernels -- and the remaining glue (embedding lookups, concatenations, padding masks, sinusoid tables,
    dropout) is torch elementwise / indexing code, as in the reference.
Not built: MAS alignment (``MAS: True``), the filled-pause predictor (``FP``) and speaker-encoder (``SE``)
variants -- the shipped sambert_24k.yaml disables all three.
"""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import ops
from . import sambert_ops as sops
from ._lib import KT_ACT_LRELU, KT_ACT_NONE


def get_mask_from_lengths(lengths, max_len=None):
    """models/utils.py:13-23; True marks padding."""
    if max_len is None:
        max_len = int(torch.max(lengths).item())
    return torch.arange(max_len, device=lengths.device)[None, :] >= lengths[:, None]


def _drop(x, p, training):
    return F.dropout(x, p, True) if (training and p > 0.0) else x


class Linear(nn.Linear):
    """nn.Linear parameters, computed as a kernel-size-1 convolution over (B, L, C) rows; optional fused ReLU
    and fused residual add."""

    def __init__(self, in_features, out_features, bias=True, relu=False):
        super().__init__(in_features, out_features, bias=bias)
        self.spec = ops.ConvSpec(c_in=in_features, c_out=out_features, kernel=1,
                                 act_out=KT_ACT_LRELU if relu else KT_ACT_NONE, act_out_slope=0.0)
        self._cache = ops.PreparedWeight()

    def forward(self, x, resid=None):
        shape = x.shape
        if x.dim() != 3:
            x = x.reshape(1, -1, shape[-1])
            resid = None if resid is None else resid.reshape(1, -1, self.out_features)
        y = ops.conv(x, self.spec, self._cache, self.weight, None, self.bias, resid)
        return y if len(shape) == 3 else y.reshape(*shape[:-1], self.out_features)


class RowConv1d(nn.Conv1d):
    """nn.Conv1d parameters applied to (B, L, C) rows (the reference transposes to (B, C, L) and back around
    every such conv, e.g. sambert/__init__.py:141-149)."""

    def __init__(self, in_channels, out_channels, kernel_size, padding=0, bias=True, relu=False):
        super().__init__(in_channels, out_channels, kernel_size, padding=padding, bias=bias)
        self.spec = ops.ConvSpec(c_in=in_channels, c_out=out_channels, kernel=kernel_size, pad_left=padding,
                                 pad_right=padding, act_out=KT_ACT_LRELU if relu else KT_ACT_NONE, act_out_slope=0.0)
        self._cache = ops.PreparedWeight()

    def forward(self, x, resid=None):
        return ops.conv(x, self.spec, self._cache, self.weight, None, self.bias, resid)


class LayerNorm(nn.LayerNorm):
    def forward(self, x):
        return sops.layer_norm(x, self.weight, self.bias, self.eps)


class ScaledDotProductAttention(nn.Module):
    """sambert/__init__.py:8-29 -- parameter-free; kept for module-tree parity.  The math (including the
    training-mode dropout on the probabilities) lives in kt_attention_fwd/bwd."""

    def __init__(self, temperature, dropatt=0.0):
        super().__init__()
        self.temperature = temperature
        self.softmax = nn.Softmax(dim=2)
        self.dropatt = nn.Dropout(dropatt)


class Prenet(nn.Module):
    """sambert/__init__.py:32-49 (Linear -> ReLU -> Dropout(0.5) per hidden layer; ReLU fused)."""

    def __init__(self, in_units, prenet_units, out_units=0):
        super().__init__()
        self.fcs = nn.ModuleList()
        for in_dim, out_dim in zip([in_units] + prenet_units[:-1], prenet_units):
            self.fcs.append(Linear(in_dim, out_dim, relu=True))
            self.fcs.append(nn.ReLU())
            self.fcs.append(nn.Dropout(0.5))
        if out_units:
            self.fcs.append(Linear(prenet_units[-1], out_units))

    def forward(self, input):
        out = input
        for layer in self.fcs:
            if isinstance(layer, nn.ReLU):
                continue                       # fused into the preceding Linear
            out = layer(out)
        return out


class MultiHeadSelfAttention(nn.Module):
    """sambert/__init__.py:52-106."""

    def __init__(self, n_head, d_in, d_model, d_head, dropout, dropatt=0.0):
        super().__init__()
        self.n_head, self.d_head, self.d_in, self.d_model = n_head, d_head, d_in, d_model
        self.layer_norm = LayerNorm(d_in, eps=1e-6)
        self.w_qkv = Linear(d_in, 3 * n_head * d_head)
        self.attention = ScaledDotProductAttention(temperature=np.power(d_head, 0.5), dropatt=dropatt)
        self.fc = Linear(n_head * d_head, d_model)
        self.dropout = nn.Dropout(dropout)
        self.dropatt = dropatt

    def forward(self, input, mask=None):
        """mask: (B, L) key-padding mask (the reference expands it over the queries, kantts_sambert.py:72-75)
        or a full (B, L, L) mask."""
        qkv = self.w_qkv(self.layer_norm(input))
        ctx, attn = sops.SelfAttnFn.apply(qkv, mask, self.n_head, self.dropatt if self.training else 0.0)
        drop = self.training and self.dropout.p > 0.0
        same = self.d_model == self.d_in
        out = self.fc(ctx, resid=input if (same and not drop) else None)
        if drop:
            out = self.dropout(out)
            if same:
                out = out + input
        return out, attn


class PositionwiseConvFeedForward(nn.Module):
    """sambert/__init__.py:109-152."""

    def __init__(self, d_in, d_hid, kernel_size=(3, 1), dropout_inner=0.1, dropout=0.1):
        super().__init__()
        self.w_1 = RowConv1d(d_in, d_hid, kernel_size[0], padding=(kernel_size[0] - 1) // 2, relu=True)
        self.w_2 = RowConv1d(d_hid, d_in, kernel_size[1], padding=(kernel_size[1] - 1) // 2)
        self.layer_norm = LayerNorm(d_in, eps=1e-6)
        self.dropout_inner = nn.Dropout(dropout_inner)
        self.dropout = nn.Dropout(dropout)

    def forward(self, x, mask=None):
        h = self.w_1(self.layer_norm(x))
        if mask is not None:
            h = h.masked_fill(mask.unsqueeze(-1), 0)
        h = self.dropout_inner(h)
        if self.training and self.dropout.p > 0.0:
            return self.dropout(self.w_2(h)) + x
        return self.w_2(h, resid=x)


class FFTBlock(nn.Module):
    """sambert/__init__.py:155-184."""

    def __init__(self, d_in, d_model, n_head, d_head, d_inner, kernel_size, dropout, dropout_attn=0.0,
                 dropout_relu=0.0):
        super().__init__()
        self.slf_attn = MultiHeadSelfAttention(n_head, d_in, d_model, d_head, dropout=dropout, dropatt=dropout_attn)
        self.pos_ffn = PositionwiseConvFeedForward(d_model, d_inner, kernel_size, dropout_inner=dropout_relu,
                                                   dropout=dropout)

    def forward(self, input, mask=None, slf_attn_mask=None):
        out, attn = self.slf_attn(input, mask=slf_attn_mask)
        if mask is not None:
            out = out.masked_fill(mask.unsqueeze(-1), 0)
        out = self.pos_ffn(out, mask=mask)
        if mask is not None:
            out = out.masked_fill(mask.unsqueeze(-1), 0)
        return out, attn


class MultiHeadPNCAAttention(nn.Module):
    """sambert/__init__.py:187-307.  Teacher-forced forward from a reset state; the incremental
    (free-running) state machine of update_x_state / update_h_state is `MelPNCADecoder.infer`'s job."""

    def __init__(self, n_head, d_model, d_mem, d_head, dropout, dropatt=0.0):
        super().__init__()
        self.n_head, self.d_head, self.d_model, self.d_mem = n_head, d_head, d_model, d_mem
        self.layer_norm = LayerNorm(d_model, eps=1e-6)
        self.w_x_qkv = Linear(d_model, 3 * n_head * d_head)
        self.fc_x = Linear(n_head * d_head, d_model)
        self.w_h_kv = Linear(d_mem, 2 * n_head * d_head)
        self.fc_h = Linear(n_head * d_head, d_model)
        self.attention = ScaledDotProductAttention(temperature=np.power(d_head, 0.5), dropatt=dropatt)
        self.dropout = nn.Dropout(dropout)
        self.dropatt = dropatt
        self.reset_state()

    def reset_state(self):
        self.h_kv = None
        self.x_kv = None
        self.x_state_size = 0

    def forward_step(self, x, h, step, mask_x, mask_h):
        """Free-running decoding (update_x_state / update_h_state, sambert/__init__.py:212-267): x (B, 1, d_model) is
        step ``step``'s input; the self keys / values of all steps live in ONE preallocated (B, Lmax, 3HD) buffer
        (the reference grows them with torch.cat), the memory keys / values are projected at step 0."""
        if step == 0 or self.h_kv is None:
            self.h_kv = self.w_h_kv(h).contiguous()
            self.x_kv = torch.zeros(x.shape[0], h.shape[1], 3 * self.n_head * self.d_head, device=x.device,
                                    dtype=torch.float32)
            self.x_state_size = 0
        q_row = self.w_x_qkv(self.layer_norm(x)).contiguous()
        self.x_kv[:, step:step + 1] = q_row
        self.x_state_size = step + 1
        ox, oh, attn_x, attn_h = sops.pnca_attn_step(q_row, self.x_kv, self.h_kv, mask_x, mask_h, self.n_head)
        return self.fc_h(oh, resid=self.fc_x(ox, resid=x)), attn_x, attn_h

    def forward(self, x, h, mask_x=None, mask_h=None):
        x_qkv = self.w_x_qkv(self.layer_norm(x))
        h_kv = self.w_h_kv(h)
        ox, oh, attn_x, attn_h = sops.PncaAttnFn.apply(x_qkv, h_kv, mask_x, mask_h, self.n_head,
                                                       self.dropatt if self.training else 0.0)
        if self.training and self.dropout.p > 0.0:
            out = self.dropout(self.fc_x(ox) + self.fc_h(oh)) + x
        else:
            out = self.fc_h(oh, resid=self.fc_x(ox, resid=x))
        return out, attn_x, attn_h


class PNCABlock(nn.Module):
    """sambert/__init__.py:310-348."""

    def __init__(self, d_model, d_mem, n_head, d_head, d_inner, kernel_size, dropout, dropout_attn=0.0,
                 dropout_relu=0.0):
        super().__init__()
        self.pnca_attn = MultiHeadPNCAAttention(n_head, d_model, d_mem, d_head, dropout=dropout, dropatt=dropout_attn)
        self.pos_ffn = PositionwiseConvFeedForward(d_model, d_inner, kernel_size, dropout_inner=dropout_relu,
                                                   dropout=dropout)

    def forward(self, input, memory, mask=None, pnca_x_attn_mask=None, pnca_h_attn_mask=None):
        out, ax, ah = self.pnca_attn(input, memory, pnca_x_attn_mask, pnca_h_attn_mask)
        if mask is not None:
            out = out.masked_fill(mask.unsqueeze(-1), 0)
        out = self.pos_ffn(out, mask=mask)
        if mask is not None:
            out = out.masked_fill(mask.unsqueeze(-1), 0)
        return out, ax, ah

    def forward_step(self, input, memory, step, mask=None, pnca_x_attn_mask=None, pnca_h_attn_mask=None):
        out, ax, ah = self.pnca_attn.forward_step(input, memory, step, pnca_x_attn_mask, pnca_h_attn_mask)
        if mask is not None:
            out = out.masked_fill(mask.unsqueeze(-1), 0)
        out = self.pos_ffn(out, mask=mask)
        if mask is not None:
            out = out.masked_fill(mask.unsqueeze(-1), 0)
        return out, ax, ah

    def reset_state(self):
        self.pnca_attn.reset_state()


# ------------------------------------------------------------------------------------------------
# positions.py
# ------------------------------------------------------------------------------------------------


class SinusoidalPositionEncoder(nn.Module):
    """positions.py:8-58."""

    def __init__(self, max_len, depth):
        super().__init__()
        self.max_len, self.depth = max_len, depth
        self.position_enc = nn.Parameter(self.get_sinusoid_encoding_table(max_len, depth).unsqueeze(0),
                                         requires_grad=False)

    def forward(self, input):
        bz, length, _ = input.size()
        if length > self.max_len:
            self.max_len = length
            self.position_enc.data = self.get_sinusoid_encoding_table(length, self.depth).unsqueeze(0).to(input.device)
        return input + self.position_enc[:, :length, :]

    @staticmethod
    def get_sinusoid_encoding_table(n_position, d_hid, padding_idx=None):
        pos = np.arange(1, n_position + 1, dtype=np.float64)[:, None]
        hid = np.arange(d_hid // 2, dtype=np.float64)[None, :]
        angle = pos / np.power(10000, hid / float(d_hid / 2 - 1))
        table = np.zeros((n_position, d_hid))
        table[:, : d_hid // 2] = np.sin(angle)
        table[:, d_hid // 2:] = np.cos(angle)
        if padding_idx is not None:
            table[padding_idx] = 0.0
        return torch.FloatTensor(table)


def _duration_spans(durations, t_out, masks, r):
    """Shared index arithmetic of LengthRegulator / DurSinusoidalPositionEncoder (adaptors.py:16-25,
    positions.py:77-90): for every output frame the symbol it copies (-1: none) and its 1-based position inside
    that symbol's span.  Integer glue on (B, L)/(B, T) tensors; no host synchronisation when t_out is given."""
    reps = (durations + 0.5).long()
    cums = torch.cumsum(reps, dim=1)
    total = cums[:, -1:]
    if t_out is None:
        t_out = int(total.max().item())
    t = torch.arange(t_out, device=durations.device)[None, :].expand(durations.shape[0], -1).contiguous()
    idx = torch.searchsorted(cums, t, right=True).clamp_max(durations.shape[1] - 1)
    start = cums - reps
    valid = t < total
    pos = (t - torch.gather(start, 1, idx) + 1).float()
    pos = torch.where(valid, pos, t.float() + 1)        # frames past the last span: offsets == 0 in the reference
    if masks is not None:
        valid = valid & ~masks
        pos = pos.masked_fill(masks, 0.0)
    idx = torch.where(valid, idx, torch.full_like(idx, -1))
    pad = r - t_out % r
    if pad < r:
        idx = F.pad(idx, (0, pad), value=-1)
        pos = F.pad(pos, (0, pad), value=0.0)
    return idx.int(), start.int(), reps.int(), pos, reps.sum(dim=1)


class DurSinusoidalPositionEncoder(nn.Module):
    """positions.py:61-103."""

    def __init__(self, depth, outputs_per_step):
        super().__init__()
        self.depth, self.outputs_per_step = depth, outputs_per_step
        inv = [np.power(10000, 2 * (i // 2) / depth) for i in range(depth)]
        self.inv_timescales = nn.Parameter(torch.FloatTensor(inv), requires_grad=False)

    def encode(self, dur_pos):
        pe = dur_pos[:, :, None] / self.inv_timescales[None, None, :]
        out = torch.empty_like(pe)
        out[:, :, 0::2] = torch.sin(pe[:, :, 0::2])
        out[:, :, 1::2] = torch.cos(pe[:, :, 1::2])
        return out

    def forward(self, durations, masks=None):
        t_out = None if masks is None else masks.size(1)
        _, _, _, pos, _ = _duration_spans(durations, t_out, masks, self.outputs_per_step)
        return self.encode(pos)


# ------------------------------------------------------------------------------------------------
# fsmn.py / adaptors.py
# ------------------------------------------------------------------------------------------------


class FeedForwardNet(nn.Module):
    """fsmn.py:8-43."""

    def __init__(self, d_in, d_hid, d_out, kernel_size=[1, 1], dropout=0.1):
        super().__init__()
        self.w_1 = RowConv1d(d_in, d_hid, kernel_size[0], padding=(kernel_size[0] - 1) // 2, relu=True)
        self.w_2 = RowConv1d(d_hid, d_out, kernel_size[1], padding=(kernel_size[1] - 1) // 2, bias=False)
        self.dropout = nn.Dropout(dropout)

    def forward(self, x):
        return self.w_2(self.dropout(self.w_1(x)))


class MemoryBlockV2(nn.Module):
    """fsmn.py:46-77."""

    def __init__(self, d, filter_size, shift, dropout=0.0):
        super().__init__()
        lp = int(round((filter_size - 1) / 2))
        rp = int((filter_size - 1) / 2)
        if shift > 0:
            lp += shift
            rp -= shift
        self.lp, self.rp = lp, rp
        self.conv_dw = nn.Conv1d(d, d, filter_size, 1, 0, groups=d, bias=False)
        self.dropout = nn.Dropout(dropout)

    def forward(self, input, mask=None):
        if self.training and self.dropout.p > 0.0:
            # dropout sits between the skip-sum and the output mask (fsmn.py:71-75): unfused order
            out = sops.FsmnMemoryFn.apply(input, self.conv_dw.weight, mask, self.lp)
            out = self.dropout(out)
            return out if mask is None else out.masked_fill(mask.unsqueeze(-1), 0)
        return sops.FsmnMemoryFn.apply(input, self.conv_dw.weight, mask, self.lp)


class FsmnEncoderV2(nn.Module):
    """fsmn.py:80-127."""

    def __init__(self, filter_size, fsmn_num_layers, input_dim, num_memory_units, ffn_inner_dim, dropout=0.0, shift=0):
        super().__init__()
        self.filter_size, self.fsmn_num_layers = filter_size, fsmn_num_layers
        self.num_memory_units, self.ffn_inner_dim, self.dropout = num_memory_units, ffn_inner_dim, dropout
        self.shift = shift if isinstance(shift, list) else [shift for _ in range(fsmn_num_layers)]
        self.ffn_lst = nn.ModuleList()
        self.ffn_lst.append(FeedForwardNet(input_dim, ffn_inner_dim, num_memory_units, dropout=dropout))
        for _ in range(1, fsmn_num_layers):
            self.ffn_lst.append(FeedForwardNet(num_memory_units, ffn_inner_dim, num_memory_units, dropout=dropout))
        self.memory_block_lst = nn.ModuleList()
        for i in range(fsmn_num_layers):
            self.memory_block_lst.append(MemoryBlockV2(num_memory_units, filter_size, self.shift[i], dropout))

    def forward(self, input, mask=None):
        x = _drop(input, self.dropout, self.training)
        for ffn, memory_block in zip(self.ffn_lst, self.memory_block_lst):
            memory = memory_block(ffn(x), mask)
            memory = _drop(memory, self.dropout, self.training)
            if memory.size(-1) == x.size(-1):
                memory = memory + x
            x = memory
        return x


class LengthRegulator(nn.Module):
    """adaptors.py:9-37, as a gather (kt_rows_gather_*) instead of the (B, T_out, T_in) one-hot matmul."""

    def __init__(self, r=1):
        super().__init__()
        self.r = r

    def forward(self, inputs, durations, masks=None):
        t_out = None if masks is None else masks.size(1)
        idx, start, count, _, out_lens = _duration_spans(durations, t_out, masks, self.r)
        return sops.RowsGatherFn.apply(inputs, idx, start, count), out_lens


class VarRnnARPredictor(nn.Module):
    """adaptors.py:40-83."""

    def __init__(self, cond_units, prenet_units, rnn_units):
        super().__init__()
        self.prenet = Prenet(1, prenet_units)
        self.lstm = nn.LSTM(prenet_units[-1] + cond_units, rnn_units, num_layers=2, batch_first=True,
                            bidirectional=False)
        self.fc = Linear(rnn_units, 1, relu=True)

    def forward(self, inputs, cond, h=None, masks=None):
        x = torch.cat([self.prenet(inputs), cond], dim=-1)
        x, h_new = self.lstm(x, h)
        x = self.fc(x).squeeze(-1)
        if masks is not None:
            x = x.masked_fill(masks, 0.0)
        return x, h_new

    def infer(self, cond, masks=None):
        """adaptors.py:67-83: the per-symbol Python loop of the reference (prenet -> LSTM step -> fc, ~10 launches per symbol)
        is ONE kernel (kt_ar_duration_infer: one CTA per batch item walks the recurrence); the condition's share of the
        layer-0 input projection is one k = 1 conv over all symbols."""
        from ._lib import load, check, ptr, stream_ptr
        lstm, B, L = self.lstm, cond.size(0), cond.size(1)
        H = lstm.hidden_size
        fc1, fc2 = [m for m in self.prenet.fcs if isinstance(m, nn.Linear)][:2]
        P1, P2 = fc1.out_features, fc2.out_features
        if not cond.is_cuda:
            raise RuntimeError("kantts_b200: VarRnnARPredictor.infer needs CUDA tensors (no CPU fallback)")
        with torch.no_grad():
            w_ih0 = lstm.weight_ih_l0
            wc = w_ih0[:, P2:].contiguous().unsqueeze(-1)                       # (4H, cond_units, 1)
            spec = self.__dict__.setdefault("_cond_spec", ops.ConvSpec(c_in=wc.shape[1], c_out=4 * H, kernel=1))
            g0c = ops.conv(cond.contiguous(), spec, ops.PreparedWeight(), wc, None, (lstm.bias_ih_l0 + lstm.bias_hh_l0).contiguous())
            out = torch.empty(B, L, device=cond.device, dtype=torch.float32)
            t = lambda w: w.detach().t().contiguous()
            args = (g0c, fc1.weight.detach()[:, 0].contiguous(), fc1.bias.detach(), t(fc2.weight), fc2.bias.detach(),
                    t(w_ih0[:, :P2]), t(lstm.weight_hh_l0), t(lstm.weight_ih_l1), t(lstm.weight_hh_l1),
                    (lstm.bias_ih_l1 + lstm.bias_hh_l1).detach().contiguous(), self.fc.weight.detach()[0].contiguous())
            check(load().kt_ar_duration_infer(*[ptr(a) for a in args], float(self.fc.bias.detach()[0]), ptr(out), B, L, H, P1, P2,
                                              stream_ptr()), "kt_ar_duration_infer")
            ops._count(2)
        if masks is not None:
            out = out.masked_fill(masks, 0.0)
        return out


class VarFsmnRnnNARPredictor(nn.Module):
    """adaptors.py:86-141."""

    def __init__(self, in_dim, filter_size, fsmn_num_layers, num_memory_units, ffn_inner_dim, dropout, shift,
                 lstm_units):
        super().__init__()
        self.fsmn = FsmnEncoderV2(filter_size, fsmn_num_layers, in_dim, num_memory_units, ffn_inner_dim, dropout,
                                  shift)
        self.blstm = nn.LSTM(num_memory_units, lstm_units, num_layers=1, batch_first=True, bidirectional=True)
        self.fc = Linear(2 * lstm_units, 1)

    def forward(self, inputs, masks=None):
        x = self.fsmn(inputs, masks)
        if masks is not None:
            lengths = torch.sum((~masks).float(), dim=1).long()
            x = nn.utils.rnn.pack_padded_sequence(x, lengths.tolist(), batch_first=True, enforce_sorted=False)
            x, _ = self.blstm(x)
            x, _ = nn.utils.rnn.pad_packed_sequence(x, batch_first=True, total_length=inputs.size(1))
        else:
            x, _ = self.blstm(x)
        x = self.fc(x).squeeze(-1)
        if masks is not None:
            x = x.masked_fill(masks, 0.0)
        return x


# ------------------------------------------------------------------------------------------------
# kantts_sambert.py
# ------------------------------------------------------------------------------------------------


class SelfAttentionEncoder(nn.Module):
    """kantts_sambert.py:22-87."""

    def __init__(self, n_layer, d_in, d_model, n_head, d_head, d_inner, dropout, dropout_att, dropout_relu,
                 position_encoder):
        super().__init__()
        self.d_in, self.d_model, self.dropout = d_in, d_model, dropout
        d_in_lst = [d_in] + [d_model] * (n_layer - 1)
        self.fft = nn.ModuleList([FFTBlock(d, d_model, n_head, d_head, d_inner, (3, 1), dropout, dropout_att,
                                           dropout_relu) for d in d_in_lst])
        self.ln = LayerNorm(d_model, eps=1e-6)
        self.position_enc = position_encoder

    def forward(self, input, mask=None, return_attns=False):
        input *= self.d_model ** 0.5                      # in place, like kantts_sambert.py:62
        if not isinstance(self.position_enc, SinusoidalPositionEncoder):
            raise NotImplementedError
        x = self.position_enc(input)
        x = _drop(x, self.dropout, self.training)
        attns = []
        for layer in self.fft:
            # the (B, L) key-padding mask is broadcast over the queries inside the kernel
            x, attn = layer(x, mask=mask, slf_attn_mask=mask)
            if return_attns:
                attns += [attn]
        return self.ln(x), attns


class HybridAttentionDecoder(nn.Module):
    """kantts_sambert.py:90-253."""

    def __init__(self, d_in, prenet_units, n_layer, d_model, d_mem, n_head, d_head, d_inner, dropout, dropout_att,
                 dropout_relu, d_out):
        super().__init__()
        self.d_model, self.dropout = d_model, dropout
        self.prenet = Prenet(d_in, prenet_units, d_model)
        self.dec_in_proj = Linear(d_model + d_mem, d_model)
        self.pnca = nn.ModuleList([PNCABlock(d_model, d_mem, n_head, d_head, d_inner, (1, 1), dropout, dropout_att,
                                             dropout_relu) for _ in range(n_layer)])
        self.ln = LayerNorm(d_model, eps=1e-6)
        self.dec_out_proj = Linear(d_model, d_out)

    def reset_state(self):
        for layer in self.pnca:
            layer.reset_state()

    def get_pnca_attn_mask(self, device, max_len, x_band_width, h_band_width, mask=None):
        """kantts_sambert.py:137-168.  True = masked.  x: keys [i - x_bw, i]; h: keys [i, i + h_bw]; padded keys are
        masked except on padded QUERY rows, which stay fully open so that their softmax is finite."""
        i = torch.arange(max_len, device=device)[:, None]
        j = torch.arange(max_len, device=device)[None, :]
        mx = ~((j >= (i - x_band_width).clamp_min(0)) & (j <= i))[None]
        mh = ~((j >= i) & (j <= i + h_band_width))[None]
        pnca_attn_mask = None
        if mask is not None:
            pnca_attn_mask = mask.unsqueeze(1).expand(-1, max_len, -1)
            qpad = pnca_attn_mask.transpose(1, 2)
            mx = (mx | pnca_attn_mask).masked_fill(qpad, False)
            mh = (mh | pnca_attn_mask).masked_fill(qpad, False)
        return pnca_attn_mask, mx, mh

    def forward(self, input, memory, x_band_width, h_band_width, mask=None, return_attns=False):
        x = self.dec_in_proj(torch.cat([memory, self.prenet(input)], dim=-1))
        if mask is not None:
            x = x.masked_fill(mask.unsqueeze(-1), 0)
        x = x * self.d_model ** 0.5
        x = _drop(x, self.dropout, self.training)
        _, mx, mh = self.get_pnca_attn_mask(x.device, x.size(1), x_band_width, h_band_width, mask)
        ax_lst, ah_lst = [], []
        for layer in self.pnca:
            x, ax, ah = layer(x, memory, mask=mask, pnca_x_attn_mask=mx, pnca_h_attn_mask=mh)
            if return_attns:
                ax_lst += [ax]
                ah_lst += [ah]
        return self.dec_out_proj(self.ln(x)), ax_lst, ah_lst

    def infer(self, step, input, memory, x_band_width, h_band_width, mask=None, return_attns=False):
        """kantts_sambert.py:207-253: one decoder step; ``reset_state()`` must precede step 0.  The band masks are
        built once per utterance (step 0) and sliced per step; any batch size (the reference's masks lose the batch
        dimension, so it only runs batch 1)."""
        max_len = memory.size(1)
        if step == 0 or getattr(self, "_step_masks", None) is None or self._step_masks[0].shape[-1] != max_len:
            _, mx, mh = self.get_pnca_attn_mask(memory.device, max_len, x_band_width, h_band_width, mask)
            self._step_masks = (mx.contiguous(), mh.contiguous())
        mx, mh = self._step_masks
        x = self.dec_in_proj(torch.cat([memory[:, step:step + 1, :], self.prenet(input)], dim=-1))
        x = x * self.d_model ** 0.5
        x = _drop(x, self.dropout, self.training)
        mask_step = None if mask is None else mask[:, step:step + 1]
        ax_lst, ah_lst = [], []
        for layer in self.pnca:
            # (the self-attention mask row covers the whole preallocated key range: keys after `step` are masked)
            x, ax, ah = layer.forward_step(x, memory, step, mask=mask_step,
                                           pnca_x_attn_mask=mx[:, step:step + 1, :].contiguous(),
                                           pnca_h_attn_mask=mh[:, step:step + 1, :].contiguous())
            if return_attns:
                ax_lst += [ax]
                ah_lst += [ah]
        return self.dec_out_proj(self.ln(x)), ax_lst, ah_lst


class TextFftEncoder(nn.Module):
    """kantts_sambert.py:256-337."""

    def __init__(self, config):
        super().__init__()
        d_emb = config["embedding_dim"]
        self.using_byte = bool(config.get("using_byte", False))
        if self.using_byte:
            self.byte_index_emb = nn.Embedding(config["byte_index"], d_emb)
        else:
            self.sy_emb = nn.Embedding(config["sy"], d_emb)
            self.tone_emb = nn.Embedding(config["tone"], d_emb)
            self.syllable_flag_emb = nn.Embedding(config["syllable_flag"], d_emb)
            self.ws_emb = nn.Embedding(config["word_segment"], d_emb)
        d_model = config["encoder_num_units"]
        nb_heads = config["encoder_num_heads"]
        self.d_model = d_model
        position_enc = SinusoidalPositionEncoder(config["max_len"], d_emb)
        self.ling_enc = SelfAttentionEncoder(
            config["encoder_num_layers"], d_emb, d_model, nb_heads, d_model // nb_heads,
            config["encoder_ffn_inner_dim"], config["encoder_dropout"], config["encoder_attention_dropout"],
            config["encoder_relu_dropout"], position_enc)
        self.ling_proj = Linear(d_model, config["encoder_projection_units"], bias=False)

    def forward(self, inputs_ling, masks=None, return_attns=False):
        if self.using_byte:
            ling_embedding = self.byte_index_emb(inputs_ling[:, :, 0])
        else:
            ling_embedding = (self.sy_emb(inputs_ling[:, :, 0]) + self.tone_emb(inputs_ling[:, :, 1])
                              + self.syllable_flag_emb(inputs_ling[:, :, 2]) + self.ws_emb(inputs_ling[:, :, 3]))
        enc_output, attns = self.ling_enc(ling_embedding, masks, return_attns)
        if hasattr(self, "ling_proj"):
            enc_output = self.ling_proj(enc_output)
        return enc_output, attns, ling_embedding


class VarianceAdaptor(nn.Module):
    """kantts_sambert.py:340-500."""

    def __init__(self, config):
        super().__init__()
        d_proj = config["encoder_projection_units"]
        input_dim = d_proj + config["emotion_units"] + config["speaker_units"]
        pred = (input_dim, config["predictor_filter_size"], config["predictor_fsmn_num_layers"],
                config["predictor_num_memory_units"], config["predictor_ffn_inner_dim"], config["predictor_dropout"],
                config["predictor_shift"], config["predictor_lstm_units"])
        self.pitch_predictor = VarFsmnRnnNARPredictor(*pred)
        self.energy_predictor = VarFsmnRnnNARPredictor(*pred)
        self.duration_predictor = VarRnnARPredictor(input_dim, config["dur_pred_prenet_units"],
                                                    config["dur_pred_lstm_units"])
        self.length_regulator = LengthRegulator(config["outputs_per_step"])
        self.dur_position_encoder = DurSinusoidalPositionEncoder(d_proj, config["outputs_per_step"])
        self.pitch_emb = RowConv1d(1, d_proj, 9, padding=4)
        self.energy_emb = RowConv1d(1, d_proj, 9, padding=4)

    def forward(self, inputs_text_embedding, inputs_emo_embedding, inputs_spk_embedding, masks=None,
                output_masks=None, duration_targets=None, pitch_targets=None, energy_targets=None):
        batch_size = inputs_text_embedding.size(0)
        var_in = torch.cat([inputs_text_embedding, inputs_spk_embedding, inputs_emo_embedding], dim=-1)
        pitch_predictions = self.pitch_predictor(var_in, masks)
        energy_predictions = self.energy_predictor(var_in, masks)
        pitch = pitch_targets if pitch_targets is not None else pitch_predictions
        energy = energy_targets if energy_targets is not None else energy_predictions
        text_aug = self.energy_emb(energy.unsqueeze(-1),
                                   resid=self.pitch_emb(pitch.unsqueeze(-1), resid=inputs_text_embedding))
        cond = torch.cat([text_aug, inputs_spk_embedding, inputs_emo_embedding], dim=-1)
        if duration_targets is not None:
            go = torch.zeros(batch_size, 1, device=inputs_text_embedding.device)
            dur_in = torch.log(torch.cat([go, duration_targets[:, :-1].float()], dim=-1) + 1)
            log_duration_predictions, _ = self.duration_predictor(dur_in.unsqueeze(-1), cond, masks=masks)
            durations = duration_targets
        else:
            log_duration_predictions = self.duration_predictor.infer(cond, masks=masks)
            durations = torch.exp(log_duration_predictions) - 1
        # one index computation serves the three expansions and the duration position encoding
        r = self.length_regulator.r
        t_out = None if output_masks is None else output_masks.size(1)
        idx, start, count, pos, lr_len = _duration_spans(durations, t_out, output_masks, r)
        lr_text = sops.RowsGatherFn.apply(text_aug, idx, start, count) + self.dur_position_encoder.encode(pos)
        lr_emo = sops.RowsGatherFn.apply(inputs_emo_embedding, idx, start, count)
        lr_spk = sops.RowsGatherFn.apply(inputs_spk_embedding, idx, start, count)
        return (lr_text, lr_emo, lr_spk, lr_len, log_duration_predictions, pitch_predictions, energy_predictions)


class MelPNCADecoder(nn.Module):
    """kantts_sambert.py:503-612."""

    def __init__(self, config):
        super().__init__()
        nb_heads = config["decoder_num_heads"]
        d_model = config["decoder_num_units"]
        r = config["outputs_per_step"]
        d_mem = config["encoder_projection_units"] * r + config["emotion_units"] + config["speaker_units"]
        self.d_mel, self.r, self.nb_layers = config["num_mels"], r, config["decoder_num_layers"]
        self.mel_dec = HybridAttentionDecoder(
            self.d_mel, config["decoder_prenet_units"], self.nb_layers, d_model, d_mem, nb_heads, d_model // nb_heads,
            config["decoder_ffn_inner_dim"], config["decoder_dropout"], config["decoder_attention_dropout"],
            config["decoder_relu_dropout"], self.d_mel * r)

    def forward(self, memory, x_band_width, h_band_width, target=None, mask=None, return_attns=False):
        go_frame = torch.zeros((memory.size(0), 1, self.d_mel), device=memory.device)
        self.mel_dec.reset_state()
        if target is None:
            # free-running decoding (kantts_sambert.py:567-612): each step's last d_mel outputs feed the next step.
            # Attention rows come back at the full key length (masked keys are exact zeros), which is what the
            # reference builds by zero-padding every step's row before concatenating.
            outs = []
            ax_steps = [[] for _ in range(self.nb_layers)]
            ah_steps = [[] for _ in range(self.nb_layers)]
            inp = go_frame
            for step in range(memory.size(1)):
                out, ax, ah = self.mel_dec.infer(step, inp, memory, x_band_width, h_band_width, mask=mask,
                                                 return_attns=return_attns)
                inp = out[:, :, -self.d_mel:]
                outs.append(out)
                for i, (a, b) in enumerate(zip(ax, ah)):
                    ax_steps[i].append(a)
                    ah_steps[i].append(b)
            dec = torch.cat(outs, dim=1)
            if not return_attns:
                return dec, [], []
            return dec, [torch.cat(a, dim=1) for a in ax_steps], [torch.cat(a, dim=1) for a in ah_steps]
        inp = torch.cat([go_frame, target[:, self.r - 1:: self.r, :]], dim=1)[:, :-1, :]
        return self.mel_dec(inp, memory, x_band_width, h_band_width, mask=mask, return_attns=return_attns)


class PostNet(nn.Module):
    """kantts_sambert.py:615-649."""

    def __init__(self, config):
        super().__init__()
        self.num_mels = config["num_mels"]
        self.fsmn = FsmnEncoderV2(config["postnet_filter_size"], config["postnet_fsmn_num_layers"], self.num_mels,
                                  config["postnet_num_memory_units"], config["postnet_ffn_inner_dim"],
                                  config["postnet_dropout"], config["postnet_shift"])
        self.lstm = nn.LSTM(config["postnet_num_memory_units"], config["postnet_lstm_units"], num_layers=1,
                            batch_first=True)
        self.fc = Linear(config["postnet_lstm_units"], self.num_mels)

    def forward(self, x, mask=None, resid=None):
        h, _ = self.lstm(self.fsmn(x, mask))
        return self.fc(h, resid=resid)


class KanTtsSAMBERT(nn.Module):
    """kantts_sambert.py:652-1044."""

    def __init__(self, config):
        super().__init__()
        for flag in ("SE", "MAS", "FP"):
            if config.get(flag, False):
                raise NotImplementedError(f"KanTtsSAMBERT variant {flag}=True is not built (see module docstring)")
        self.text_encoder = TextFftEncoder(config)
        self.se_enable = False
        self.spk_tokenizer = nn.Embedding(config["speaker"], config["speaker_units"])
        self.emo_tokenizer = nn.Embedding(config["emotion"], config["emotion_units"])
        self.variance_adaptor = VarianceAdaptor(config)
        self.mel_decoder = MelPNCADecoder(config)
        self.mel_postnet = PostNet(config)
        self.MAS = False
        self.fp_enable = False

    def get_lfr_mask_from_lengths(self, lengths, max_len):
        """kantts_sambert.py:681-695 without the per-item host loop: ceil(len / r) frames are valid."""
        r = self.mel_decoder.r
        return get_mask_from_lengths((lengths + r - 1) // r, max_len=max_len // r)

    def forward(self, inputs_ling, inputs_emotion, inputs_speaker, input_lengths, output_lengths=None,
                mel_targets=None, duration_targets=None, pitch_targets=None, energy_targets=None, attn_priors=None,
                fp_label=None):
        batch_size = inputs_ling.size(0)
        r = self.mel_decoder.r
        input_masks = get_mask_from_lengths(input_lengths, max_len=inputs_ling.size(1))
        text_hid, enc_attns, _ = self.text_encoder(inputs_ling, input_masks, return_attns=True)
        inter_lengths = input_lengths
        emo_hid = self.emo_tokenizer(inputs_emotion)
        spk_hid = self.spk_tokenizer(inputs_speaker)
        inter_masks = get_mask_from_lengths(inter_lengths, max_len=text_hid.size(1))
        output_masks = None
        if output_lengths is not None:
            output_masks = get_mask_from_lengths(output_lengths, max_len=mel_targets.size(1))
        (lr_text, lr_emo, lr_spk, lr_len, log_dur_p, pitch_p, energy_p) = self.variance_adaptor(
            text_hid, emo_hid, spk_hid, masks=inter_masks, output_masks=output_masks,
            duration_targets=duration_targets, pitch_targets=pitch_targets, energy_targets=energy_targets)
        if output_lengths is not None:
            lfr_masks = self.get_lfr_mask_from_lengths(output_lengths, max_len=lr_text.size(1))
        else:
            output_masks = get_mask_from_lengths(lr_len, max_len=lr_text.size(1))
            lfr_masks = None
        # LFR: r consecutive frames side by side (text) / the first of every r frames (speaker, emotion)
        lfr_text = lr_text.contiguous().view(batch_size, -1, r * text_hid.shape[-1])
        lfr_emo = lr_emo.contiguous().view(batch_size, -1, r * emo_hid.shape[-1])[:, :, : emo_hid.shape[-1]]
        lfr_spk = lr_spk.contiguous().view(batch_size, -1, r * spk_hid.shape[-1])[:, :, : spk_hid.shape[-1]]
        memory = torch.cat([lfr_text, lfr_spk, lfr_emo], dim=-1)
        if duration_targets is not None:
            x_band_width = int(duration_targets.float().masked_fill(inter_masks, 0).max() / r + 0.5)
        else:
            x_band_width = int((torch.exp(log_dur_p) - 1).max() / r + 0.5)
        h_band_width = x_band_width
        dec, ax_lst, ah_lst = self.mel_decoder(memory, x_band_width, h_band_width, target=mel_targets,
                                               mask=lfr_masks, return_attns=True)
        dec_outputs = dec.contiguous().view(batch_size, -1, self.mel_decoder.d_mel)
        if output_masks is not None:
            dec_outputs = dec_outputs.masked_fill(output_masks.unsqueeze(-1), 0)
        postnet_outputs = self.mel_postnet(dec_outputs, output_masks, resid=dec_outputs)
        if output_masks is not None:
            postnet_outputs = postnet_outputs.masked_fill(output_masks.unsqueeze(-1), 0)
        return {
            "x_band_width": x_band_width, "h_band_width": h_band_width, "enc_slf_attn_lst": enc_attns,
            "pnca_x_attn_lst": ax_lst, "pnca_h_attn_lst": ah_lst, "dec_outputs": dec_outputs,
            "postnet_outputs": postnet_outputs, "LR_length_rounded": lr_len,
            "log_duration_predictions": log_dur_p, "pitch_predictions": pitch_p, "energy_predictions": energy_p,
            "duration_targets": duration_targets, "pitch_targets": pitch_targets, "energy_targets": energy_targets,
            "fp_predictions": None, "valid_inter_lengths": inter_lengths,
            "LR_text_outputs": lr_text, "LR_emo_outputs": lr_emo, "LR_spk_outputs": lr_spk,
        }


# ------------------------------------------------------------------------------------------------
# train/loss.py:7-85
# ------------------------------------------------------------------------------------------------


class MelReconLoss(nn.Module):
    """train/loss.py:7-40."""

    def __init__(self, loss_type="mae"):
        super().__init__()
        if loss_type not in ("mae", "mse"):
            raise ValueError("Unknown loss type: {}".format(loss_type))
        self.loss_type = loss_type

    def _err(self, a, b):
        return (a - b).abs() if self.loss_type == "mae" else (a - b) ** 2

    def forward(self, output_lengths, mel_targets, dec_outputs, postnet_outputs=None):
        valid = ~get_mask_from_lengths(output_lengths, max_len=mel_targets.size(1))
        denom = valid.sum() * mel_targets.size(-1)
        mel_loss_ = torch.sum(self._err(mel_targets, dec_outputs) * valid.unsqueeze(-1)) / denom
        mel_loss = 0.0
        if postnet_outputs is not None:
            mel_loss = torch.sum(self._err(mel_targets, postnet_outputs) * valid.unsqueeze(-1)) / denom
        return mel_loss_, mel_loss


class ProsodyReconLoss(nn.Module):
    """train/loss.py:43-85."""

    def __init__(self, loss_type="mae"):
        super().__init__()
        if loss_type not in ("mae", "mse"):
            raise ValueError("Unknown loss type: {}".format(loss_type))
        self.loss_type = loss_type

    def _err(self, a, b):
        return (a - b).abs() if self.loss_type == "mae" else (a - b) ** 2

    def forward(self, input_lengths, duration_targets, pitch_targets, energy_targets, log_duration_predictions,
                pitch_predictions, energy_predictions):
        valid = ~get_mask_from_lengths(input_lengths, max_len=duration_targets.size(1))
        n = valid.sum()
        dur_loss = torch.sum(self._err(torch.log(duration_targets.float() + 1), log_duration_predictions) * valid) / n
        pitch_loss = torch.sum(self._err(pitch_targets, pitch_predictions) * valid) / n
        energy_loss = torch.sum(self._err(energy_targets, energy_predictions) * valid) / n
        return dur_loss, pitch_loss, energy_loss
