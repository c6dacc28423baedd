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
  * the four LSTMs (the ``nn.LSTM`` modules hold their parameters) -> in training sambert_ops.lstm_layer: the input
    projection on the conv kernels, the recurrence and its backward in kt_lstm_train_fwd / _bwd, lengths on the device;
    inference runs the duration predictor's in kt_ar_duration_infer, the pitch / energy predictors' BiLSTMs in
    kt_blstm_ragged and the streamed post-net's in kt_lstm_stream_slots -- and the remaining glue (embedding lookups,
    concatenations, padding masks, sinusoid tables, dropout) is torch elementwise / indexing code, as in the reference.
The filled-pause variant (``FP: True``, sambert_fp_8k.yaml) is built: FP_Predictor on the same conv / LayerNorm
kernels, and the splice of the predicted or labelled pauses into the text encoding as an index plan plus one
gather each way (kt_fp_insert_*).  The alignment-learning variant (``MAS: True``, sambert_16k_MAS*.yaml) is built:
ConvAttention's projections on the conv kernels, its distance attention fused in kt_align_attn_* (no (B, C, T_mel,
T_text) difference tensor), monotonic alignment search on the GPU (kt_mas, no host copy) and the forward-sum loss in
kt_attn_ctc_*.  The speaker-embedding variant (``SE: True``, sambert_se_nsf_global_16k.yaml) is built: it has no speaker
table, and ``inputs_speaker`` is the float (B, L, speaker_units) per-symbol embedding (speaker.speaker_embedding) in
place of the ids.  The masked-symbol pretraining model of sybert.yaml (KanTtsTextsyBERT) is built on the same text
encoder, with its loss (SeqCELoss) fused in kt_seq_ce_*.  Not built: MAS together with FP (the reference's two branches
do not compose: its MAS durations have one entry per symbol before the pause splice), and SE together with FP or MAS.
"""
import ctypes
from collections import namedtuple

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import ops
from . import sambert_ops as sops
from ._lib import KT_ACT_LRELU, KT_ACT_NONE, ptr
from .stream import Streamer, WindowTable, own_weight


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

    def forward(self, x, mask=None, per_item=False):
        """``per_item``: w_1 reads the LayerNorm of the padding rows as zeros, the zero padding an item has run alone
        (in a padded batch a padding row's LayerNorm is its bias, which a k > 1 w_1 reads at the item's last rows)."""
        h = self.layer_norm(x)
        if per_item and mask is not None:
            h = h.masked_fill(mask.unsqueeze(-1), 0)
        h = self.w_1(h)
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

    def forward(self, input, mask=None, slf_attn_mask=None, per_item=False):
        out, attn = self.slf_attn(input, mask=slf_attn_mask)
        if mask is not None:
            out = out.masked_fill(mask.unsqueeze(-1), 0)
        out = self.pos_ffn(out, mask=mask, per_item=per_item)
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


def _duration_spans(durations, t_out, masks, r, per_item=False):
    """Shared index arithmetic of LengthRegulator / DurSinusoidalPositionEncoder (adaptors.py:16-25,
    positions.py:77-90): for every output frame the symbol it copies (-1: none) and its 1-based position inside
    that symbol's span.  Integer glue on (B, L)/(B, T) tensors; no host synchronisation when t_out is given.
    ``per_item``: the frames that pad an item's own frame count up to a multiple of r take position 0, as they do when the
    item runs alone, instead of the padded batch's t + 1."""
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
    if per_item:
        pos = pos.masked_fill((t >= total) & (t < (total + r - 1) // r * r), 0.0)
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
        """Over all rows from ``h`` (nn.LSTM's initial (h_0, c_0), or None: zeros), one sambert_ops.lstm_layer per layer
        -> (x, h_new = (h_n, c_n)), (num_layers, B, H) each."""
        x = torch.cat([self.prenet(inputs), cond], dim=-1)
        h_n, c_n = [], []
        for layer in range(self.lstm.num_layers):
            x, c = sops.lstm_layer(x, self.lstm, layer, state=h)
            h_n.append(x[:, -1])
            c_n.append(c[:, -1])
        h_new = (torch.stack(h_n), torch.stack(c_n))
        x = self.fc(x).squeeze(-1)
        if masks is not None:
            x = x.masked_fill(masks, 0.0)
        return x, h_new

    def infer(self, cond, masks=None):
        """adaptors.py:67-83: the per-symbol Python loop of the reference (prenet -> LSTM step -> fc, ~10 launches per symbol)
        is ONE kernel (kt_ar_duration_infer: one CTA per batch item walks the recurrence); the condition's share of the
        layer-0 input projection is one k = 1 conv over all symbols."""
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
            ops.call("kt_ar_duration_infer", *[ptr(a) for a in args], float(self.fc.bias.detach()[0]), ptr(out), B, L, H, P1, P2,
                     launches=2)
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
        if not self.training and not torch.is_grad_enabled():
            x = self.blstm_infer(x, masks)
        else:
            # pack_padded_sequence -> BiLSTM -> pad_packed_sequence, with each item's length on the device
            lengths = None if masks is None else (~masks).sum(1, dtype=torch.int32)
            x, _ = sops.lstm_layer(x, self.blstm, 0, lengths)
        x = self.fc(x).squeeze(-1)
        if masks is not None:
            x = x.masked_fill(masks, 0.0)
        return x

    def blstm_infer(self, x, masks=None):
        """The packed BiLSTM of ``forward`` for inference (no autograd): both directions over each item's own rows
        [0, len_b) in ONE kernel (kt_blstm_ragged), with the lengths taken from ``masks`` on the device (no host read);
        rows >= len_b are zero.  The input projection of both directions is one k = 1 conv over the concatenated [8H]
        weights.  An item's rows do not depend on the other items of the batch or on its padding.  Training runs
        sambert_ops.lstm_layer."""
        lstm, (B, L) = self.blstm, x.shape[:2]
        H = lstm.hidden_size
        if not x.is_cuda:
            raise RuntimeError("kantts_b200: VarFsmnRnnNARPredictor.blstm_infer needs CUDA tensors (no CPU fallback)")
        with torch.no_grad():
            spec, pw, w, bias, whh_t = self._blstm_weights()
            gx = ops.conv(x.contiguous(), spec, pw, w, None, bias)
            if masks is None:
                lengths = torch.full((B,), L, device=x.device, dtype=torch.int32)
            else:
                lengths = (~masks).sum(1, dtype=torch.int32)
            h = torch.empty(B, L, 2 * H, device=x.device, dtype=torch.float32)
            ops.call("kt_blstm_ragged", ptr(gx), ptr(whh_t), ptr(lengths, True), ptr(h), B, L, H)
        return h

    def _blstm_weights(self):
        """-> (spec, PreparedWeight, w, bias, whh_t) of blstm_infer: the input projection of both directions as one
        k = 1 conv (w (8H, C, 1), bias (8H,)) and W_hh^T of both directions (2, H, 4H).  Built once and kept until a
        parameter of the LSTM changes; w is a Parameter so that its prepared (tensor-core) layouts are kept with it."""
        lstm = self.blstm
        params = [lstm.weight_ih_l0, lstm.weight_ih_l0_reverse, lstm.bias_ih_l0, lstm.bias_hh_l0,
                  lstm.bias_ih_l0_reverse, lstm.bias_hh_l0_reverse, lstm.weight_hh_l0, lstm.weight_hh_l0_reverse]
        key = tuple((p.data_ptr(), p._version, getattr(p, "_kt_epoch", 0)) for p in params)
        cache = self.__dict__.get("_blstm_cache")
        if cache is None or cache[0] != key:
            H = lstm.hidden_size
            w = nn.Parameter(torch.cat([lstm.weight_ih_l0, lstm.weight_ih_l0_reverse]).unsqueeze(-1).detach(),
                             requires_grad=False)
            bias = torch.cat([lstm.bias_ih_l0 + lstm.bias_hh_l0, lstm.bias_ih_l0_reverse + lstm.bias_hh_l0_reverse])
            whh_t = torch.stack([lstm.weight_hh_l0.t(), lstm.weight_hh_l0_reverse.t()]).contiguous()
            spec = ops.ConvSpec(c_in=lstm.input_size, c_out=8 * H, kernel=1)
            cache = (key, (spec, ops.PreparedWeight(), w, bias.detach(), whh_t.detach()))
            self.__dict__["_blstm_cache"] = cache
        return cache[1]


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

    def forward(self, input, mask=None, return_attns=False, per_item=False):
        input *= self.d_model ** 0.5                      # in place, like kantts_sambert.py:62
        if not isinstance(self.position_enc, SinusoidalPositionEncoder):
            raise NotImplementedError
        x = self.position_enc(input)
        x = _drop(x, self.dropout, self.training)
        attns = []
        for layer in self.fft:
            # the (B, L) key-padding mask is broadcast over the queries inside the kernel
            x, attn = layer(x, mask=mask, slf_attn_mask=mask, per_item=per_item)
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
        """kantts_sambert.py:137-168.  True = masked.  The band widths are ints or 0-d device tensors.  x: keys [i - x_bw, i]; h: keys [i, i + h_bw]; padded keys are
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

    def forward(self, inputs_ling, masks=None, return_attns=False, per_item=False):
        if self.using_byte:
            ling_embedding = self.byte_index_emb(inputs_ling[:, :, 0])
        else:
            ling_embedding = (self.sy_emb(inputs_ling[:, :, 0]) + self.tone_emb(inputs_ling[:, :, 1])
                              + self.syllable_flag_emb(inputs_ling[:, :, 2]) + self.ws_emb(inputs_ling[:, :, 3]))
        enc_output, attns = self.ling_enc(ling_embedding, masks, return_attns, per_item)
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
                output_masks=None, duration_targets=None, pitch_targets=None, energy_targets=None, per_item=False):
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
        idx, start, count, pos, lr_len = _duration_spans(durations, t_out, output_masks, r, per_item)
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

    def infer_steps(self, memory, x_band_width, h_band_width, mask=None, return_attns=False):
        """Free-running decoding, one step at a time (kantts_sambert.py:567-612): yields (out, attn_x, attn_h) of every LFR
        step, out (B, 1, r * d_mel); each step's last d_mel outputs feed the next step.  Step s depends only on earlier
        steps, so a consumer can use a step's rows as soon as it is yielded."""
        go_frame = torch.zeros((memory.size(0), 1, self.d_mel), device=memory.device)
        self.mel_dec.reset_state()
        inp = go_frame
        for step in range(memory.size(1)):
            out, ax, ah = self.mel_dec.infer(step, inp, memory, x_band_width, h_band_width, mask=mask,
                                             return_attns=return_attns)
            inp = out[:, :, -self.d_mel:]
            yield out, ax, ah

    def forward(self, memory, x_band_width, h_band_width, target=None, mask=None, return_attns=False):
        if target is None:
            # Attention rows come back at the full key length (masked keys are exact zeros), which is what the
            # reference builds by zero-padding every step's row before concatenating.
            outs = []
            ax_steps = [[] for _ in range(self.nb_layers)]
            ah_steps = [[] for _ in range(self.nb_layers)]
            for out, ax, ah in self.infer_steps(memory, x_band_width, h_band_width, mask, return_attns):
                outs.append(out)
                for i, (a, b) in enumerate(zip(ax, ah)):
                    ax_steps[i].append(a)
                    ah_steps[i].append(b)
            dec = torch.cat(outs, dim=1)
            if not return_attns:
                return dec, [], []
            return dec, [torch.cat(a, dim=1) for a in ax_steps], [torch.cat(a, dim=1) for a in ah_steps]
        go_frame = torch.zeros((memory.size(0), 1, self.d_mel), device=memory.device)
        self.mel_dec.reset_state()
        inp = torch.cat([go_frame, target[:, self.r - 1:: self.r, :]], dim=1)[:, :-1, :]
        return self.mel_dec(inp, memory, x_band_width, h_band_width, mask=mask, return_attns=return_attns)

    def slots(self, batch, max_steps):
        """-> a SlotDecoder: free-running decoding of ``batch`` independent utterances of up to ``max_steps`` steps each."""
        return SlotDecoder(self, batch, max_steps)


class SlotDecoder:
    """Free-running decoding (MelPNCADecoder.infer_steps) of one utterance per slot, every slot at its own step
    (MelPNCADecoder.slots).

    Per slot on the device: the memory rows (batch, max_steps, d_mem), each PNCA layer's memory K / V projection and self
    K / V cache, ``step``, ``mem_len`` (decoder steps), ``x_bw`` / ``h_bw`` (band widths) and ``active``.  ``admit`` places an
    utterance in a slot (inactive until ``start``); ``advance()`` runs one decoder step of every active slot and returns the
    (batch, 1, r * d_mel) outputs, zero for the inactive slots.  A slot reads its own memory row at its step and feeds back
    its own previous output (zeros, the go frame, at its step 0); it goes inactive after its last step.  Each
    slot's rows equal ``infer_steps`` of its utterance alone.  No call reads device data on the host."""

    def __init__(self, decoder, batch, max_steps):
        if decoder.training:
            raise ValueError("slot decoding runs a decoder in eval() mode")
        dec = decoder.mel_dec
        self.decoder, self.batch, self.max_steps = decoder, int(batch), int(max_steps)
        if self.batch < 1 or self.max_steps < 1:
            raise ValueError(f"slots: batch ({batch}) and max_steps ({max_steps}) must be >= 1")
        attn = dec.pnca[0].pnca_attn
        self.n_head, hd = attn.n_head, attn.n_head * attn.d_head
        self.device = dev = next(decoder.parameters()).device
        if dev.type != "cuda":
            raise RuntimeError("kantts_b200: the slot decoder runs on a CUDA device (no CPU fallback)")
        B, L = self.batch, self.max_steps
        self.memory = torch.zeros(B, L, attn.d_mem, device=dev)
        self.h_kv = [torch.zeros(B, L, 2 * hd, device=dev) for _ in dec.pnca]
        self.x_kv = [torch.zeros(B, L, 2 * hd, device=dev) for _ in dec.pnca]
        self.step = torch.zeros(B, dtype=torch.int32, device=dev)
        self.mem_len = torch.zeros(B, dtype=torch.int32, device=dev)
        self.x_bw = torch.zeros(B, dtype=torch.int32, device=dev)
        self.h_bw = torch.zeros(B, dtype=torch.int32, device=dev)
        self.active = torch.zeros(B, dtype=torch.uint8, device=dev)
        self._inp = torch.zeros(B, 1, decoder.d_mel, device=dev)

    def admit(self, slot, memory, band_width):
        """Place one utterance in slot ``slot`` (an int): ``memory`` (1, n, d_mem) its decoder memory (n <= max_steps),
        ``band_width`` its band (an int or a device tensor of one element), for both attentions.  Its memory K / V rows are
        projected here; the slot stays inactive until ``start``."""
        b, n = int(slot), memory.shape[1]
        if not 0 <= b < self.batch:
            raise ValueError(f"admit: slot must lie in [0, {self.batch}), got {slot}")
        if memory.dim() != 3 or memory.shape[0] != 1 or memory.shape[2] != self.memory.shape[2]:
            raise ValueError(f"admit: expected a (1, n, {self.memory.shape[2]}) memory, got {tuple(memory.shape)}")
        if not 1 <= n <= self.max_steps:
            raise ValueError(f"admit: an utterance of {n} decoder steps does not fit max_steps = {self.max_steps}")
        with torch.no_grad():
            self.memory[b].zero_()
            self.memory[b, :n].copy_(memory[0])
            for layer, h_kv in zip(self.decoder.mel_dec.pnca, self.h_kv):
                h_kv[b, :n].copy_(layer.pnca_attn.w_h_kv(memory)[0])
            # the go frame: the slot's fed-back input is zero at its step 0 even when its previous utterance ended on the
            # step before (a copy, since the fed-back rows are a view of the last step's returned output)
            self._inp = self._inp.clone()
            self._inp[b].zero_()
            for t, v in ((self.step, 0), (self.mem_len, n), (self.active, 0)):
                t[b] = v
            for t in (self.x_bw, self.h_bw):
                t[b].copy_(band_width.reshape(())) if torch.is_tensor(band_width) else t[b].fill_(int(band_width))

    def start(self, slot):
        """Slot ``slot`` decodes its step 0 in the next ``advance()``."""
        self.active[int(slot)] = 1

    def advance(self):
        """One decoder step of every active slot -> (batch, 1, r * d_mel), zero rows for the inactive slots."""
        dec, B = self.decoder.mel_dec, self.batch
        with torch.no_grad():
            idx = self.step.long().clamp_(max=self.max_steps - 1).view(B, 1, 1).expand(B, 1, self.memory.shape[2])
            x = dec.dec_in_proj(torch.cat([torch.gather(self.memory, 1, idx), dec.prenet(self._inp)], dim=-1))
            x = x * dec.d_model ** 0.5
            for layer, h_kv, x_kv in zip(dec.pnca, self.h_kv, self.x_kv):
                attn = layer.pnca_attn
                q_row = attn.w_x_qkv(attn.layer_norm(x)).contiguous()
                ox, oh = sops.pnca_step_slots(q_row, x_kv, h_kv, self, attn.n_head)
                x = layer.pos_ffn(attn.fc_h(oh, resid=attn.fc_x(ox, resid=x)))
            live = self.active.bool().view(B, 1, 1)
            out = dec.dec_out_proj(dec.ln(x)).masked_fill(~live, 0)
            self._inp = out[:, :, -self.decoder.d_mel:]
            self.step += self.active
            self.active &= (self.step < self.mem_len).to(torch.uint8)
        return out


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
        h, _ = sops.lstm_layer(self.fsmn(x, mask), self.lstm, 0)
        return self.fc(h, resid=resid)

    def streamer(self, batch, max_frames, lengths):
        """-> a PostNetStreamer that runs this (eval-mode) post-net chunk by chunk over ``batch`` utterances of ``lengths``
        (host ints or device tensor (batch,)) frames, at most ``max_frames`` decoder rows per chunk.  Its output trails
        the decoder rows by ``delay`` rows; ``reset(slots, lengths, start_row)`` starts utterances in some slots (see
        PostNetStreamer)."""
        return PostNetStreamer(self, batch, max_frames, lengths)


# One launch of a post-net chunk over named windows.  kind "conv": a k = 1 conv of ``module`` (a Linear, or the nn.LSTM's
# input projection); "fsmn": the memory block ``module`` of FSMN layer ``layer``; "lstm": the nn.LSTM's recurrence.
# ``resid`` (or None) is added to the output from ``res_lag`` rows before the output's chunk rows.
PostNetStep = namedtuple("PostNetStep", "kind module src dst resid res_lag layer", defaults=(None, 0, -1))


class PostNetStreamPlan:
    """What a PostNetStreamer runs per chunk, as data (no device needed).  The post-net is causal except for the right
    padding of its memory blocks: output frame t is final once decoder row t + delay exists.
      layers              per FSMN layer: {lp, rp, kernel, lag}: the memory block's left / right padding and filter size, and
                          how many rows the layer's input lags the decoder rows (the sum of rp over the layers before it)
      delay               D = the sum of rp: the post-net output of a chunk is its decoder rows shifted back by D rows
      windows             one entry per tensor of a chunk: {name, channels, rows_per_frame (1), history}; a memory block's
                          input keeps k - 1 rows, a residual read lagging its tensor by n rows keeps n, the others keep none
      lags                {window: rows it trails the decoder rows} of the masked reads: ctx{i} (lag), "gates", "out" (D)
      steps               PostNetStep records, in launch order
      launches_per_chunk  library calls of a steady chunk: one per step, one window advance and one output mask; the copy of
                          the decoder rows into their window is not counted"""

    def __init__(self, postnet):
        if postnet.training:
            raise ValueError("streaming runs a post-net in eval() mode")
        fsmn = postnet.fsmn
        table = WindowTable()
        self.windows, self.layers, self.steps, self.lags = table.windows, [], [], {}
        x, lag = table.add("dec", postnet.num_mels), 0
        mid = table.add("mid", fsmn.ffn_inner_dim)
        units = fsmn.num_memory_units
        for i, (ffn, mb) in enumerate(zip(fsmn.ffn_lst, fsmn.memory_block_lst)):
            k = mb.conv_dw.kernel_size[0]
            if mb.rp < 0:
                raise ValueError(f"streaming needs rp >= 0 in every memory block: layer {i} has shift > (filter_size - 1) / 2 "
                                 f"(lp {mb.lp}, rp {mb.rp})")
            self.layers.append(dict(lp=mb.lp, rp=mb.rp, kernel=k, lag=lag))
            ctx = table.add(f"ctx{i}", units)
            table.read(ctx, k - 1)
            self.lags[ctx] = lag
            resid = x if ffn.w_1.in_channels == units else None
            if resid is not None:
                table.read(resid, mb.rp)
            out = table.add(f"x{i + 1}", units)
            self.steps += [PostNetStep("conv", ffn.w_1, x, mid), PostNetStep("conv", ffn.w_2, mid, ctx),
                           PostNetStep("fsmn", mb, ctx, out, resid, res_lag=mb.rp, layer=i)]
            x, lag = out, lag + mb.rp
        self.delay = lag
        table.read("dec", self.delay)                      # the output Linear's residual: the decoder rows D rows back
        gates = table.add("gates", 4 * postnet.lstm.hidden_size)
        h = table.add("h", postnet.lstm.hidden_size)
        self.steps += [PostNetStep("conv", postnet.lstm, x, gates), PostNetStep("lstm", postnet.lstm, gates, h),
                       PostNetStep("conv", postnet.fc, h, table.add("out", postnet.num_mels), "dec", res_lag=self.delay)]
        self.lags.update(gates=self.delay, out=self.delay)
        self.launches_per_chunk = table.launches_per_chunk(len(self.steps)) + 1


class PostNetStreamer(Streamer):
    """Chunk-by-chunk PostNet (PostNet.streamer) over decoder rows that arrive step by step.

    ``push(dec_rows)`` takes the next (B, f, num_mels) decoder rows of every slot (de-LFR'd and masked, 1 <= f <=
    max_frames) and returns f rows of the post-net output ``fc(lstm(fsmn(x))) + x``: row t of slot b is frame
    frames_done[b] - delay + t of its utterance (frames_done counts the decoder rows since its frame 0), zero outside
    [0, lengths[b]).  ``finish()`` pushes ``delay`` all-padding rows and returns their output.  The rows returned in
    order from frame 0 on are then the whole-sequence post-net output.  ``reset(slots, lengths, start_row)`` starts new
    utterances in the given slots with frame 0 at row ``start_row`` of the next push; the other slots go on.  A slot's
    new utterance must start after the previous one's last row was returned.  No call reads device data on the host.

    Every chunk runs over all f rows of every slot.  Where each slot is in its utterance lives on the device
    (stream.SlotUtterances, whose frames are the decoder rows).  A tensor a layer reads before the chunk lives in a window
    (stream.py).  The memory blocks (kt_fsmn_fwd_stream_slots) read frames outside [0, lengths[b]) as zeros, the
    whole-sequence padding, and the LSTM (kt_lstm_stream_slots) starts from zeros at frame 0, so starting an utterance
    clears no window history or LSTM state; every other step reads only the frame it writes, and the output is masked
    outside the utterance.  The weights are prepared once, when the streamer is created."""

    out, f_axis = "out", 1

    def __init__(self, postnet, batch, max_frames, lengths):
        plan = PostNetStreamPlan(postnet)
        super().__init__(plan, batch, max_frames, next(postnet.parameters()).device, "post-net streamer", masked=True,
                         in_channels=postnet.num_mels)
        self.hidden = postnet.lstm.hidden_size
        self._state = torch.zeros(self.batch, 2, self.hidden, device=self.device)
        with torch.no_grad(), torch.cuda.device(self.device):
            self._weights = [self._own_weight(st) for st in plan.steps]
            self.reset(range(self.batch), lengths)

    @staticmethod
    def _own_weight(st):
        """-> copies of what step st reads besides its windows: (spec, PreparedWeight, bias), the (C, k) taps or W_hh^T."""
        mod = st.module
        if st.kind == "fsmn":
            return mod.conv_dw.weight.detach().reshape(mod.conv_dw.out_channels, -1).clone()
        if st.kind == "lstm":
            return mod.weight_hh_l0.detach().t().contiguous()
        if isinstance(mod, nn.LSTM):                       # x . W_ih^T + b_ih + b_hh as one k = 1 conv
            spec = ops.ConvSpec(c_in=mod.input_size, c_out=4 * mod.hidden_size, kernel=1)
            return (spec, *own_weight(spec, mod.weight_ih_l0.unsqueeze(-1), None, mod.bias_ih_l0 + mod.bias_hh_l0))
        return (mod.spec, *own_weight(mod.spec, mod.weight, None, mod.bias))

    def _chunk(self, f):
        """Every launch of one chunk of f decoder rows (already in the "dec" window)."""
        b, B, masks = self._win.buf, self.batch, self._masks
        for st, w, place in zip(self.plan.steps, self._weights, self._places):
            src, dst, resid = b[st.src], b[st.dst], None if st.resid is None else b[st.resid]
            if st.kind == "conv":
                spec, pw, bias = w
                ops.stream_conv(spec, pw, bias, src, dst, f, place, resid)
            elif st.kind == "fsmn":
                layer = self.plan.layers[st.layer]
                ops.call("kt_fsmn_fwd_stream_slots", ctypes.byref(place), ctypes.byref(masks[st.src]), ptr(src), ptr(w),
                         ptr(resid), ptr(dst), B, f, src.shape[2], layer["kernel"], layer["lp"])
            else:
                ops.call("kt_lstm_stream_slots", ptr(src), ptr(w), ptr(self._state), ptr(dst), ctypes.byref(masks[st.src]),
                         B, f, self.hidden, src.shape[1], dst.shape[1])
        self._end_chunk(f)

    def push(self, dec_rows):
        """dec_rows: (B, f, num_mels), 1 <= f <= max_frames -> the (B, f, num_mels) post-net rows ``delay`` rows behind
        them."""
        with torch.no_grad(), torch.cuda.device(self.device):
            f = self._win.push("dec", dec_rows, 1, ("{} decoder rows", "rows", "the rows are"))
            self._chunk(f)
            return self._output(f)

    def reset(self, slots, lengths, start_row=0):
        """The given slots (host ints) start new utterances of ``lengths`` frames (host ints or a device tensor, in the
        order of ``slots``), with frame 0 at row ``start_row`` of the next push (0 <= start_row < max_frames); the other
        slots go on.  Clears no window or LSTM state and reads no device data."""
        if not 0 <= int(start_row) < self.max_frames:
            raise ValueError(f"reset: start_row must lie in [0, {self.max_frames}), got {start_row}")
        self._slots.reset(slots, lengths, start_row)


class FP_Predictor(nn.Module):
    """kantts_sambert.py:677-710: filled-pause class probabilities (none / en / a / e) per symbol.  The two ReLUs are
    fused into the convs; the 4-class softmax stays a torch op."""

    def __init__(self, config):
        super().__init__()
        d_proj, d_hid = config["encoder_projection_units"], config["embedding_dim"] // 2
        self.w_1 = RowConv1d(d_proj, d_hid, 3, padding=1, relu=True)
        self.w_2 = RowConv1d(d_hid, d_proj, 1, relu=True)
        self.layer_norm1 = LayerNorm(d_hid, eps=1e-6)
        self.layer_norm2 = LayerNorm(d_proj, eps=1e-6)
        self.dropout_inner = nn.Dropout(0.1)
        self.dropout = nn.Dropout(0.1)
        self.fc = Linear(d_proj, 4)

    def forward(self, x):
        x = self.dropout_inner(self.layer_norm1(self.w_1(x)))
        x = self.dropout(self.layer_norm2(self.w_2(x)))
        return F.softmax(self.fc(x), dim=2)


class ConvNorm(nn.Module):
    """attention.py:6-39: a "same"-padded Conv1d re-initialised with xavier_uniform_ at the gain of ``w_init_gain``,
    applied to (B, L, C) rows; ``relu`` fuses the ReLU that follows it in its Sequential."""

    def __init__(self, in_channels, out_channels, kernel_size=1, bias=True, w_init_gain="linear", relu=False):
        super().__init__()
        assert kernel_size % 2 == 1
        self.conv = RowConv1d(in_channels, out_channels, kernel_size, padding=(kernel_size - 1) // 2, bias=bias, relu=relu)
        nn.init.xavier_uniform_(self.conv.weight, gain=nn.init.calculate_gain(w_init_gain))

    def forward(self, x):
        return self.conv(x)


class ConvAttention(nn.Module):
    """attention.py:42-125: the alignment attention of the MAS variant.  Same constructor, sub-modules, ``state_dict`` and
    seeded init as the reference (``attn_proj`` is kept although the forward never uses it).  Unlike the reference's
    (B, C, T) inputs, ``forward`` takes the model's (B, T, C) rows: queries (B, T_mel, n_mel_channels), keys
    (B, T_text, n_text_channels), ``mask`` the (B, T_text) key-padding mask of a length vector (True = padding), the
    optional ``attn_prior`` (B, T_mel, T_text).  -> attn_soft, attn_logprob (B, 1, T_mel, T_text).  The projections run on
    the conv kernels (ReLUs fused), the distance attention in kt_align_attn_fwd / _bwd."""

    def __init__(self, n_mel_channels=80, n_text_channels=512, n_att_channels=80, temperature=1.0, use_query_proj=True):
        super().__init__()
        self.temperature = temperature
        self.att_scaling_factor = np.sqrt(n_att_channels)
        self.softmax = nn.Softmax(dim=3)
        self.log_softmax = nn.LogSoftmax(dim=3)
        self.attn_proj = nn.Conv2d(n_att_channels, 1, kernel_size=1)
        self.use_query_proj = bool(use_query_proj)
        self.key_proj = nn.Sequential(
            ConvNorm(n_text_channels, n_text_channels * 2, kernel_size=3, bias=True, w_init_gain="relu", relu=True),
            nn.ReLU(),
            ConvNorm(n_text_channels * 2, n_att_channels, kernel_size=1, bias=True))
        self.query_proj = nn.Sequential(
            ConvNorm(n_mel_channels, n_mel_channels * 2, kernel_size=3, bias=True, w_init_gain="relu", relu=True),
            nn.ReLU(),
            ConvNorm(n_mel_channels * 2, n_mel_channels, kernel_size=1, bias=True, relu=True),
            nn.ReLU(),
            ConvNorm(n_mel_channels, n_att_channels, kernel_size=1, bias=True))

    @staticmethod
    def _project(seq, x):
        for layer in seq:
            if not isinstance(layer, nn.ReLU):          # the ReLUs are fused into the preceding convs
                x = layer(x)
        return x

    def forward(self, queries, keys, mask=None, attn_prior=None):
        keys_enc = self._project(self.key_proj, keys)
        queries_enc = self._project(self.query_proj, queries) if self.use_query_proj else queries
        if mask is None:
            key_lengths = torch.full((keys.size(0),), keys.size(1), device=keys.device, dtype=torch.int32)
        else:
            key_lengths = (~mask).sum(1, dtype=torch.int32)
        return sops.AlignAttnFn.apply(queries_enc, keys_enc, attn_prior, key_lengths)


class KanTtsSAMBERT(nn.Module):
    """kantts_sambert.py:652-1044.  With ``FP: True`` the model builder must set ``fp_dict`` ({1: en, 2: a, 3: e},
    each a (1, 3, 4) long tensor of linguistic ids) before the first forward, as kantts/models/__init__.py:99-105
    does."""

    def __init__(self, config):
        super().__init__()
        if config.get("SE", False) and (config.get("FP", False) or config.get("MAS", False)):
            raise NotImplementedError("KanTtsSAMBERT with SE=True together with FP or MAS is not built (see module docstring)")
        if config.get("MAS", False) and config.get("FP", False):
            raise NotImplementedError("KanTtsSAMBERT with both MAS=True and FP=True is not built (see module docstring)")
        self.text_encoder = TextFftEncoder(config)
        self.se_enable = bool(config.get("SE", False))
        if not self.se_enable:
            self.spk_tokenizer = nn.Embedding(config["speaker"], config["speaker_units"])
        self.emo_tokenizer = nn.Embedding(config["emotion"], config["emotion_units"])
        self.variance_adaptor = VarianceAdaptor(config)
        self.mel_decoder = MelPNCADecoder(config)
        self.mel_postnet = PostNet(config)
        self.MAS = bool(config.get("MAS", False))
        if self.MAS:
            self.align_attention = ConvAttention(n_mel_channels=config["num_mels"], n_text_channels=config["embedding_dim"],
                                                 n_att_channels=config["num_mels"])
        self.fp_enable = bool(config.get("FP", False))
        if self.fp_enable:
            self.FP_predictor = FP_Predictor(config)
        self.fp_dict = None

    def insert_fp(self, text_hid, fp_p, fp_label, inputs_emotion, inputs_speaker, input_lengths, per_item=False):
        """kantts_sambert.py:766-860: splice the encodings of the filled pauses (labelled, or predicted when
        ``fp_label`` is None) in front of their symbols.  The three pause sequences go through the text encoder as one
        unmasked batch; the emotion / speaker ids are only extended (row t takes row t mod L, or with ``per_item`` row t mod
        the item's own length, as when it runs alone)."""
        if self.fp_dict is None:
            raise RuntimeError("KanTtsSAMBERT(FP=True) needs model.fp_dict = {1: en, 2: a, 3: e} (each a (1, 3, 4) "
                               "long tensor of linguistic ids) before the forward, as the reference model builder sets")
        seqs = torch.cat([self.fp_dict[k].reshape(1, 3, -1) for k in (1, 2, 3)], 0).to(text_hid.device)
        fp_enc, _, _ = self.text_encoder(seqs)
        L = text_hid.size(1)
        codes, rows, inter_lengths, t_ins = sops.fp_insert_plan(input_lengths, L, fp_label=fp_label, fp_p=fp_p)
        text_hid = sops.FpInsertFn.apply(text_hid, fp_enc, codes, rows, t_ins)
        n = input_lengths.clamp_min(1)[:, None] if per_item else L
        ext = torch.arange(t_ins, device=text_hid.device)[None, :] % n
        items = torch.arange(text_hid.size(0), device=text_hid.device)[:, None]
        return text_hid, inputs_emotion[items, ext], inputs_speaker[items, ext], inter_lengths

    def get_lfr_mask_from_lengths(self, lengths, max_len):
        """kantts_sambert.py:681-695 without the per-item host loop: ceil(len / r) frames are valid."""
        r = self.mel_decoder.r
        return get_mask_from_lengths((lengths + r - 1) // r, max_len=max_len // r)

    def align(self, ling_embedding, mel_targets, input_lengths, output_lengths, input_masks, attn_priors, pitch_targets,
              energy_targets):
        """The monotonic-alignment-search branch of the teacher-forced forward (kantts_sambert.py:901-925): the alignment
        attention of the mel targets over the (scaled) symbol embeddings, MAS durations, the frame-level pitch / energy
        targets averaged per symbol, and the trailing padding symbol input_lengths[b] given the T_mel - output_lengths[b]
        padding frames.  Validates the lengths on the host (the branch's one host read).  -> dict."""
        L, T_mel = ling_embedding.size(1), mel_targets.size(1)
        in_lens, out_lens = torch.stack([input_lengths.long(), output_lengths.long()]).tolist()
        for b, (n, t) in enumerate(zip(in_lens, out_lens)):
            if not 1 <= n < L:
                raise ValueError(f"MAS: input_lengths[{b}] = {n} must lie in [1, {L}): the symbol after the last valid one "
                                 "(the trailing '~') receives the padding frames")
            if not 1 <= t <= T_mel:
                raise ValueError(f"MAS: output_lengths[{b}] = {t} must lie in [1, {T_mel}]")
        attn_soft, attn_logprob = self.align_attention(mel_targets, ling_embedding, input_masks, attn_priors)
        attn_hard, durations = sops.mas(attn_soft, input_lengths, output_lengths)
        pitch = sops.average_frame_feat(pitch_targets, durations)
        energy = sops.average_frame_feat(energy_targets, durations)
        pad = (T_mel - output_lengths).to(durations.dtype).unsqueeze(1)
        durations.scatter_(1, input_lengths.long().unsqueeze(1), pad)
        return dict(attn_soft=attn_soft, attn_hard=attn_hard, attn_logprob=attn_logprob, duration_targets=durations,
                    pitch_targets=pitch, energy_targets=energy)

    def front_half(self, inputs_ling, inputs_emotion, inputs_speaker, input_lengths, output_lengths=None,
                   mel_targets=None, duration_targets=None, pitch_targets=None, energy_targets=None, fp_label=None,
                   attn_priors=None, per_item=False):
        """Everything of ``forward`` before the decoder: text encoder, filled-pause insertion (``FP``), alignment search
        (``MAS``, when ``mel_targets`` is given), variance adaptor, the decoder memory and the band width of its attentions.
        -> dict of the intermediate results ``forward`` and ``infer.stream_synthesize`` continue from.
        ``per_item`` (inference): every item gets what it gets run alone, the reference's batch-1 inference, bit for bit on
        both compute paths: ``memory`` rows [0, ceil(lr_len / r)), ``lr_len``, ``band_width_rows`` and ``log_dur_p`` /
        ``pitch_p`` / ``energy_p`` on its ``inter_lengths`` rows.  The kernels already give an item's rows independently
        of the batch (in inference the BiLSTMs run in kt_blstm_ragged); what the flag changes is the rules by which the
        reference's padded batch differs from one item alone: the k = 3 convs of the encoder's feed-forward blocks and of
        the ``FP`` predictor read an item's padding rows as zeros (in the padded batch a padding row's LayerNorm is its
        bias), the frames that pad an item's last decoder step take position code 0 (t + 1 in the padded batch), and with
        ``FP`` the emotion / speaker rows are extended mod the item's length, not mod the padded length.
        ``x_band_width``, the batch-max band (a 0-d int64 device tensor: ``forward`` makes it the reference's int), is
        batch-dependent by definition."""
        batch_size = inputs_ling.size(0)
        r = self.mel_decoder.r
        input_masks = get_mask_from_lengths(input_lengths, max_len=inputs_ling.size(1))
        text_hid, enc_attns, ling_embedding = self.text_encoder(inputs_ling, input_masks, return_attns=True,
                                                                per_item=per_item)
        inter_lengths = input_lengths
        mas = {}
        if self.MAS and mel_targets is not None:
            mas = self.align(ling_embedding, mel_targets, input_lengths, output_lengths, input_masks, attn_priors,
                             pitch_targets, energy_targets)
            duration_targets, pitch_targets, energy_targets = (mas["duration_targets"], mas["pitch_targets"],
                                                               mas["energy_targets"])
        fp_p = None
        if self.fp_enable:
            # per_item: the predictor's k = 3 w_1 reads zeros past an item's last symbol, as run alone (the encoder's
            # padding rows are its final LayerNorm bias through ling_proj)
            fp_p = self.FP_predictor(text_hid.masked_fill(input_masks.unsqueeze(-1), 0) if per_item else text_hid)
            text_hid, inputs_emotion, inputs_speaker, inter_lengths = self.insert_fp(
                text_hid, fp_p, fp_label, inputs_emotion, inputs_speaker, input_lengths, per_item)
        emo_hid = self.emo_tokenizer(inputs_emotion)
        spk_hid = inputs_speaker if self.se_enable else self.spk_tokenizer(inputs_speaker)
        inter_masks = get_mask_from_lengths(inter_lengths, max_len=text_hid.size(1))
        output_masks = None
        if output_lengths is not None:
            output_masks = get_mask_from_lengths(output_lengths, max_len=mel_targets.size(1))
        (lr_text, lr_emo, lr_spk, lr_len, log_dur_p, pitch_p, energy_p) = self.variance_adaptor(
            text_hid, emo_hid, spk_hid, masks=inter_masks, output_masks=output_masks,
            duration_targets=duration_targets, pitch_targets=pitch_targets, energy_targets=energy_targets, per_item=per_item)
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
            dur = duration_targets.float().masked_fill(inter_masks, 0)
        else:
            dur = torch.exp(log_dur_p) - 1
        # the reference's int(dur.max() / r + 0.5), kept on the device (0-d int64)
        x_band_width = torch.trunc(dur.max() / r + 0.5).long()
        # each utterance's own band (the batch-1 rule), on the device: the max over its symbols only
        band_width_rows = torch.trunc(dur.masked_fill(inter_masks, float("-inf")).amax(1) / r + 0.5).to(torch.int32)
        return dict(enc_attns=enc_attns, fp_p=fp_p, inter_lengths=inter_lengths, output_masks=output_masks,
                    lfr_masks=lfr_masks, lr_text=lr_text, lr_emo=lr_emo, lr_spk=lr_spk, lr_len=lr_len, log_dur_p=log_dur_p,
                    pitch_p=pitch_p, energy_p=energy_p, memory=memory, x_band_width=x_band_width,
                    band_width_rows=band_width_rows, duration_targets=duration_targets, pitch_targets=pitch_targets,
                    energy_targets=energy_targets,
                    **{k: v for k, v in mas.items() if k.startswith("attn_")})

    def forward(self, inputs_ling, inputs_emotion, inputs_speaker, input_lengths, output_lengths=None,
                mel_targets=None, duration_targets=None, pitch_targets=None, energy_targets=None, attn_priors=None,
                fp_label=None):
        batch_size = inputs_ling.size(0)
        f = self.front_half(inputs_ling, inputs_emotion, inputs_speaker, input_lengths, output_lengths, mel_targets,
                            duration_targets, pitch_targets, energy_targets, fp_label, attn_priors)
        output_masks, lr_len, inter_lengths = f["output_masks"], f["lr_len"], f["inter_lengths"]
        # the reference's Python int, read on the host -- except under CUDA-graph capture, where it stays a 0-d device tensor
        x_band_width = f["x_band_width"]
        if not (x_band_width.is_cuda and torch.cuda.is_current_stream_capturing()):
            x_band_width = int(x_band_width)
        h_band_width = x_band_width
        dec, ax_lst, ah_lst = self.mel_decoder(f["memory"], x_band_width, h_band_width, target=mel_targets,
                                               mask=f["lfr_masks"], return_attns=True)
        dec_outputs = dec.contiguous().view(batch_size, -1, self.mel_decoder.d_mel)
        if output_masks is not None:
            dec_outputs = dec_outputs.masked_fill(output_masks.unsqueeze(-1), 0)
        postnet_outputs = self.mel_postnet(dec_outputs, output_masks, resid=dec_outputs)
        if output_masks is not None:
            postnet_outputs = postnet_outputs.masked_fill(output_masks.unsqueeze(-1), 0)
        res = {
            "x_band_width": x_band_width, "h_band_width": h_band_width, "enc_slf_attn_lst": f["enc_attns"],
            "pnca_x_attn_lst": ax_lst, "pnca_h_attn_lst": ah_lst, "dec_outputs": dec_outputs,
            "postnet_outputs": postnet_outputs, "LR_length_rounded": lr_len,
            "log_duration_predictions": f["log_dur_p"], "pitch_predictions": f["pitch_p"],
            "energy_predictions": f["energy_p"],
            "duration_targets": f["duration_targets"], "pitch_targets": f["pitch_targets"],
            "energy_targets": f["energy_targets"],
            "fp_predictions": f["fp_p"], "valid_inter_lengths": inter_lengths,
            "LR_text_outputs": f["lr_text"], "LR_emo_outputs": f["lr_emo"], "LR_spk_outputs": f["lr_spk"],
        }
        if "attn_hard" in f:
            res.update(attn_soft=f["attn_soft"], attn_hard=f["attn_hard"], attn_logprob=f["attn_logprob"])
        return res


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


class FpCELoss(nn.Module):
    """train/loss.py:88-105: class-weighted cross entropy of the filled-pause predictions over the valid symbols.
    ``fp_pd`` is already a softmax output and the cross entropy applies log_softmax to it again, as the reference does.
    The class weights are a buffer, so ``.to(device)`` moves them."""

    def __init__(self, loss_type="ce", weight=[1, 4, 4, 8]):
        super().__init__()
        self.loss_type = loss_type
        self.register_buffer("weight", torch.tensor(weight, dtype=torch.float32))

    def forward(self, input_lengths, fp_pd, fp_label):
        valid = ~get_mask_from_lengths(input_lengths, max_len=fp_label.size(1))
        ce = F.cross_entropy(fp_pd.transpose(2, 1), fp_label, weight=self.weight, reduction="none")
        return torch.sum(ce * valid) / valid.sum()


class AttentionCTCLoss(nn.Module):
    """train/loss.py:481-508: the forward-sum loss of the alignment attention, each utterance's CTC loss of the targets
    1..in_len over its frames' log_softmax([blank_logprob, keys < in_len]), divided by in_len (0 when infinite), averaged
    over the batch -- all utterances in one kt_attn_ctc_fwd / _bwd launch instead of a torch.nn.CTCLoss call each."""

    def __init__(self, blank_logprob=-1):
        super().__init__()
        self.blank_logprob = blank_logprob

    def forward(self, attn_logprob, in_lens, out_lens):
        return sops.AttnCtcFn.apply(attn_logprob, in_lens, out_lens, float(self.blank_logprob))


class AttentionBinarizationLoss(nn.Module):
    """train/loss.py:463-478: -sum log(clamp(soft, eps)) over the cells of the hard alignment / their count, scaled by the
    warm-up ratio min(1, (epoch - start_epoch) / warmup_epoch) (0 before start_epoch).  Written as a masked sum
    (``hard`` is exactly 0 / 1) instead of the reference's boolean indexing, so it never synchronises with the host."""

    def __init__(self, start_epoch=0, warmup_epoch=100):
        super().__init__()
        self.start_epoch = start_epoch
        self.warmup_epoch = warmup_epoch

    def forward(self, epoch, hard_attention, soft_attention, eps=1e-12):
        log_sum = (hard_attention * torch.log(torch.clamp(soft_attention, min=eps))).sum()
        kl_loss = -log_sum / hard_attention.sum()
        if epoch < self.start_epoch:
            warmup_ratio = 0
        else:
            warmup_ratio = min(1.0, (epoch - self.start_epoch) / self.warmup_epoch)
        return kl_loss * warmup_ratio


class KanTtsTextsyBERT(nn.Module):
    """kantts_sambert.py:1047-1068: the masked-symbol pretraining model of sybert.yaml, TextFftEncoder without its output
    projection followed by a Linear onto the ``sy`` vocabulary.  ``ling_proj`` is constructed and then deleted, as the
    reference does: its initialiser consumes the torch RNG, so a seeded init equals the reference's, and the state_dict is
    ``text_encoder.*`` (no ``ling_proj``) then ``fc.*``.  ``fc`` runs on the conv kernels like every other Linear.

    ``forward(inputs_ling, input_lengths)`` -> {"logits": (B, L, sy), "enc_slf_attn_lst": one attention map per encoder
    layer, in the reference's layout}.  The reference's forward unpacks two of TextFftEncoder's three results and raises
    ValueError; this one returns what it evidently means to.  Byte input (``using_byte``) is not built: the reference's
    ``fc`` needs ``config["sy"]``, so it cannot build a byte model either."""

    def __init__(self, config):
        super().__init__()
        if config.get("using_byte", False):
            raise NotImplementedError("KanTtsTextsyBERT: byte input (using_byte) is not built; the output layer is sized by "
                                      "the PinYin 'sy' vocabulary")
        self.text_encoder = TextFftEncoder(config)
        delattr(self.text_encoder, "ling_proj")
        self.fc = Linear(self.text_encoder.d_model, config["sy"])

    def forward(self, inputs_ling, input_lengths):
        input_masks = get_mask_from_lengths(input_lengths, max_len=inputs_ling.size(1))
        text_hid, enc_slf_attn_lst, _ = self.text_encoder(inputs_ling, input_masks, return_attns=True)
        return {"logits": self.fc(text_hid), "enc_slf_attn_lst": enc_slf_attn_lst}


class SeqCELoss(nn.Module):
    """train/loss.py:444-460: ``(loss, err)`` of ``logits`` (..., V), int64 ``targets`` and ``masks`` (float, bool or int):
    the masked mean cross-entropy and the masked argmax error rate.  Both come from one kt_seq_ce_fwd pass over the logits
    (instead of a log-softmax, a gather, an argmax and two masked reductions); the gradient of ``loss`` is kt_seq_ce_bwd and
    ``err`` has none.  An all-zero mask gives NaN, as the reference's 0 / 0 does."""

    def __init__(self, loss_type="ce"):
        super().__init__()
        self.loss_type = loss_type

    def forward(self, logits, targets, masks):
        return sops.SeqCEFn.apply(logits, targets, masks)
