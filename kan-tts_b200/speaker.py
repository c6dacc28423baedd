"""Speaker-embedding extractor of the SE SAM-BERT flow (kantts/preprocess/se_processor): the Kaldi fbank and the D-TDNN,
batched over wavs of different lengths (kernels: csrc/speaker.cu and the conv kernels).

``DTDNN`` has the reference module tree, so its state_dict keys, order and seeded initialisation are the reference's, and a
reference ``se.model`` loads with ``strict=True``.  It is inference only: eval-mode BatchNorm, no backward.  The forward runs
on channels-last rows:
  - the 2-D head: each 3x3 Conv2d (stride (s, 1) on frequency) is one 1-D k=3 conv over the rows of a tap gather
    (B, F_out, T, 3 C), whose channels are the three input frequencies s f + {-1, 0, 1} (kt_se_tap_gather).  A residual
    block's shortcut (identity or strided 1x1) is C more input channels of its second conv, read at the centre time tap,
    so the sum and the ReLU after it run in that conv; every BatchNorm folds into its conv.
  - the dense blocks: one (B, T, C_final) slab per block.  Layer i reads channels [0, c_i) through nonlinear1
    (kt_se_affine_rows), runs linear1 with nonlinear2 folded, and its gated 32 outputs land at channel c_i
    (kt_se_gate_stats + kt_se_gate_apply); no concatenation copies.
  - statistics pooling over each item's valid rows, then the dense layer with its BatchNorm folded.
Item b owns rows [0, lengths[b]) at every stage (half of them, rounded up, after the stride-2 TDNN); every kernel writes
the rows past that as zeros and reduces over the valid rows only, so an item's embedding is that of its wav run alone.
"""
import ctypes
from collections import OrderedDict

import torch
import torch.nn as nn

from . import ops
from ._lib import KT_ACT_LRELU, KT_ACT_NONE, ptr

SAMPLE_RATE = 16000
FRAME_LEN, FRAME_SHIFT = 400, 160
N_MELS = 80
SEG_LEN = 100          # PoolingBlock's segment length (layers.py seg_pooling)


def fbank_frames(n):
    """Frames of a wav of n samples (snip_edges): 1 + (n - 400) // 160, 0 below one frame."""
    return 1 + (n - FRAME_LEN) // FRAME_SHIFT if n >= FRAME_LEN else 0


def _host_lengths(lengths, n_max, what):
    lens = [int(v) for v in (lengths.tolist() if torch.is_tensor(lengths) else lengths)]
    for n in lens:
        if not 1 <= n <= n_max:
            raise ValueError(f"{what}: length {n} outside [1, {n_max}]")
    return lens


def kaldi_fbank(wav, lengths=None):
    """(B, n) wavs at 16 kHz, item b's samples [0, lengths[b]) -> ((B, T, 80) Kaldi fbank with each utterance's mean over
    its frames subtracted, frame counts (list)); frames past an item's last are zeros.  A wav shorter than one 400-sample
    frame raises ValueError."""
    if wav.dim() != 2:
        raise ValueError(f"kaldi_fbank: expected (B, n) wavs, got {tuple(wav.shape)}")
    B, n = wav.shape
    lens = _host_lengths([n] * B if lengths is None else lengths, n, "kaldi_fbank")
    if min(lens) < FRAME_LEN:
        raise ValueError(f"kaldi_fbank: a wav of {min(lens)} samples is shorter than one {FRAME_LEN}-sample frame")
    wav = wav.detach().float().contiguous()
    frames = fbank_frames(n)
    out = torch.empty(B, frames, N_MELS, device=wav.device, dtype=torch.float32)
    lg = torch.tensor(lens, dtype=torch.int32).to(wav.device, non_blocking=True)
    ops.call("kt_kaldi_fbank", ptr(wav), ptr(lg, True), ptr(out), B, n, frames, N_MELS, float(SAMPLE_RATE), 20.0, launches=2)
    return out, [fbank_frames(v) for v in lens]


def speaker_embedding(extractor, wav, lengths=None):
    """(B, n) wavs at 16 kHz -> (B, 192) speaker embeddings: the Kaldi fbank with per-utterance mean normalisation of the
    reference processor (se_processor.py:65-69), then the D-TDNN ``extractor`` over each item's frames."""
    feats, frames = kaldi_fbank(wav, lengths)
    return extractor(feats, frames)


# ---- the reference's module tree (D_TDNN.py, layers.py): names, order and construction order of every parameter --------
def _nonlinear(config_str, channels):
    seq = nn.Sequential()
    for name in config_str.split("-"):
        if name == "relu":
            seq.add_module("relu", nn.ReLU(inplace=True))
        elif name == "batchnorm":
            seq.add_module("batchnorm", nn.BatchNorm1d(channels))
        elif name == "batchnorm_":
            seq.add_module("batchnorm", nn.BatchNorm1d(channels, affine=False))
        else:
            raise ValueError(f"Unexpected module ({name}).")
    return seq


class BasicBlock(nn.Module):
    expansion = 1

    def __init__(self, in_planes, planes, stride=1):
        super().__init__()
        self.stride = stride
        self.conv1 = nn.Conv2d(in_planes, planes, kernel_size=3, stride=(stride, 1), padding=1, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = nn.Conv2d(planes, planes, kernel_size=3, stride=1, padding=1, bias=False)
        self.bn2 = nn.BatchNorm2d(planes)
        self.shortcut = nn.Sequential()
        if stride != 1 or in_planes != planes:
            self.shortcut = nn.Sequential(nn.Conv2d(in_planes, planes, kernel_size=1, stride=(stride, 1), bias=False),
                                          nn.BatchNorm2d(planes))


class CNN_Head(nn.Module):
    def __init__(self, num_blocks=(2, 2), m_channels=32, feat_dim=80):
        super().__init__()
        self.in_planes = m_channels
        self.conv1 = nn.Conv2d(1, m_channels, kernel_size=3, stride=1, padding=1, bias=False)
        self.bn1 = nn.BatchNorm2d(m_channels)
        self.layer1 = self._make_layer(m_channels, num_blocks[0], stride=2)
        self.layer2 = self._make_layer(m_channels, num_blocks[0], stride=2)
        self.conv2 = nn.Conv2d(m_channels, m_channels, kernel_size=3, stride=(2, 1), padding=1, bias=False)
        self.bn2 = nn.BatchNorm2d(m_channels)
        self.out_channels = m_channels * (feat_dim // 8)

    def _make_layer(self, planes, num_blocks, stride):
        layers = []
        for s in [stride] + [1] * (num_blocks - 1):
            layers.append(BasicBlock(self.in_planes, planes, s))
            self.in_planes = planes
        return nn.Sequential(*layers)


class TDNNLayer(nn.Module):
    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, bias=False,
                 config_str="batchnorm-relu"):
        super().__init__()
        if padding < 0:
            padding = (kernel_size - 1) // 2 * dilation
        self.linear = nn.Conv1d(in_channels, out_channels, kernel_size, stride=stride, padding=padding, dilation=dilation,
                                bias=bias)
        self.nonlinear = _nonlinear(config_str, out_channels)


class PoolingBlock(nn.Module):
    def __init__(self, bn_channels, out_channels, kernel_size, stride, padding, dilation, bias, reduction=2):
        super().__init__()
        self.linear_stem = nn.Conv1d(bn_channels, out_channels, kernel_size, stride=stride, padding=padding,
                                     dilation=dilation, bias=bias)
        self.linear1 = nn.Conv1d(bn_channels, bn_channels // reduction, 1)
        self.relu = nn.ReLU(inplace=True)
        self.linear2 = nn.Conv1d(bn_channels // reduction, out_channels, 1)
        self.sigmoid = nn.Sigmoid()


class SEDenseTDNNLayer(nn.Module):
    def __init__(self, in_channels, out_channels, bn_channels, kernel_size, stride=1, dilation=1, bias=False,
                 config_str="batchnorm-relu", memory_efficient=False):
        super().__init__()
        padding = (kernel_size - 1) // 2 * dilation
        self.memory_efficient = memory_efficient
        self.nonlinear1 = _nonlinear(config_str, in_channels)
        self.linear1 = nn.Conv1d(in_channels, bn_channels, 1, bias=False)
        self.nonlinear2 = _nonlinear(config_str, bn_channels)
        self.se = PoolingBlock(bn_channels, out_channels, kernel_size, stride=stride, padding=padding, dilation=dilation,
                               bias=bias)


class SEDenseTDNNBlock(nn.ModuleList):
    def __init__(self, num_layers, in_channels, out_channels, bn_channels, kernel_size, stride=1, dilation=1, bias=False,
                 config_str="batchnorm-relu", memory_efficient=False):
        super().__init__()
        for i in range(num_layers):
            self.add_module("tdnnd%d" % (i + 1), SEDenseTDNNLayer(
                in_channels + i * out_channels, out_channels, bn_channels, kernel_size, stride=stride, dilation=dilation,
                bias=bias, config_str=config_str, memory_efficient=memory_efficient))


class TransitLayer(nn.Module):
    def __init__(self, in_channels, out_channels, bias=True, config_str="batchnorm-relu"):
        super().__init__()
        self.nonlinear = _nonlinear(config_str, in_channels)
        self.linear = nn.Conv1d(in_channels, out_channels, 1, bias=bias)


class DenseLayer(nn.Module):
    def __init__(self, in_channels, out_channels, bias=False, config_str="batchnorm-relu"):
        super().__init__()
        self.linear = nn.Conv1d(in_channels, out_channels, 1, bias=bias)
        self.nonlinear = _nonlinear(config_str, out_channels)


class StatsPool(nn.Module):
    pass


def _bn_affine(bn):
    """eval-mode BatchNorm as y = a x + s (a, s per channel)."""
    a = torch.rsqrt(bn.running_var.detach() + bn.eps)
    if bn.affine:
        a = a * bn.weight.detach()
        s = bn.bias.detach() - bn.running_mean.detach() * a
    else:
        s = -bn.running_mean.detach() * a
    return a, s


def _row_conv(c_in, c_out, k=1, dilation=1, pad=0, stride=1, relu=False):
    return ops.ConvSpec(c_in=c_in, c_out=c_out, kernel=k, stride=stride, dilation=dilation, pad_left=pad, pad_right=pad,
                        act_out=KT_ACT_LRELU if relu else KT_ACT_NONE, act_out_slope=0.0)


class _Layer:
    """One conv as the extractor runs it: its ConvSpec, its folded weight and bias (nn.Parameters refreshed in place, so the
    PreparedWeight cache invalidates exactly when they change) and its PreparedWeight."""

    def __init__(self, spec, w, b):
        self.spec, self.cache = spec, ops.PreparedWeight()
        self.w = nn.Parameter(w.contiguous(), requires_grad=False)
        self.b = None if b is None else nn.Parameter(b.contiguous(), requires_grad=False)

    def update(self, w, b):
        """Copy new folded values in; the in-place copy moves the parameters' versions (``.data`` would not)."""
        with torch.no_grad():
            self.w.copy_(w.reshape(self.w.shape))
            if b is not None:
                self.b.copy_(b)

    def __call__(self, x):
        return ops.conv(x, self.spec, self.cache, self.w, None, self.b)


class DTDNN(nn.Module):
    """kantts.preprocess.se_processor.D_TDNN.DTDNN on the project's kernels; ``forward(feats, lengths=None)`` maps
    (B, T, 80) fbank features, item b's frames [0, lengths[b]), to (B, 192) embeddings.  Inference only."""

    def __init__(self, feat_dim=80, embedding_size=192, growth_rate=32, bn_size=4, init_channels=128,
                 config_str="batchnorm-relu", memory_efficient=True):
        super().__init__()
        self.head = CNN_Head()
        feat_dim = self.head.out_channels
        self.xvector = nn.Sequential(OrderedDict([
            ("tdnn", TDNNLayer(feat_dim, init_channels, 5, stride=2, dilation=1, padding=-1, config_str=config_str))]))
        channels = init_channels
        for i, (num_layers, kernel_size, dilation) in enumerate(zip((12, 24, 16), (3, 3, 3), (1, 2, 3))):
            block = SEDenseTDNNBlock(num_layers, channels, growth_rate, bn_size * growth_rate, kernel_size,
                                     dilation=dilation, config_str=config_str, memory_efficient=memory_efficient)
            self.xvector.add_module("block%d" % (i + 1), block)
            channels = channels + num_layers * growth_rate
            self.xvector.add_module("transit%d" % (i + 1),
                                    TransitLayer(channels, channels // 2, bias=False, config_str=config_str))
            channels //= 2
        self.bn = nn.BatchNorm1d(channels)
        self.relu = nn.ReLU(inplace=True)
        self.xvector.add_module("stats", StatsPool())
        self.xvector.add_module("dense", DenseLayer(channels * 2, embedding_size, config_str="batchnorm_"))
        for m in self.modules():
            if isinstance(m, (nn.Conv1d, nn.Linear)):
                nn.init.kaiming_normal_(m.weight.data)
                if m.bias is not None:
                    nn.init.zeros_(m.bias)
        self.__dict__["_run"] = None     # the folded layers (not module state), see _folded()
        self.__dict__["_run_key"] = None
        # where each parameter and buffer lives: read afresh on every call, so a load_state_dict, an in-place edit or a
        # device move (which replaces the tensors) changes the key
        self.__dict__["_slots"] = [(d, n) for mod in self.modules() for d in (mod._parameters, mod._buffers)
                                   for n, t in d.items() if t is not None]

    # ---- weight folding, once per weight version ---------------------------------------------------------------------
    def _fold(self):
        """-> {name: (ConvSpec, folded weight, folded bias)} and {name: (scale, shift)} of the input affines."""
        convs, affines = {}, {}
        h = self.head

        def taps3(conv, bn):   # W'[o, df * ci + c, dt] = a[o] W[o, c, df, dt]: the 3-frequency gather's channel order
            a, s = _bn_affine(bn)
            w = conv.weight.detach() * a[:, None, None, None]
            co, ci, kf, kt = w.shape
            return w.permute(0, 2, 1, 3).reshape(co, kf * ci, kt), s

        w, s = taps3(h.conv1, h.bn1)
        convs["head.conv1"] = (_row_conv(w.shape[1], w.shape[0], k=3, pad=1, relu=True), w, s)
        for ln in ("layer1", "layer2"):
            for j, blk in enumerate(getattr(h, ln)):
                p = f"head.{ln}.{j}"
                w, s = taps3(blk.conv1, blk.bn1)
                convs[p + ".conv1"] = (_row_conv(w.shape[1], w.shape[0], k=3, pad=1, relu=True), w, s)
                # conv2 and the shortcut as one conv: the shortcut's input (the block input at frequency s f) is 32 more
                # input channels, read at the centre time tap only, so the ReLU after the sum runs in the epilogue
                w2, s2 = taps3(blk.conv2, blk.bn2)
                co = w2.shape[0]
                if len(blk.shortcut):
                    a, s_sc = _bn_affine(blk.shortcut[1])
                    wsc = blk.shortcut[0].weight.detach()[:, :, 0, 0] * a[:, None]
                    s2 = s2 + s_sc
                else:
                    wsc = torch.eye(co, device=w2.device, dtype=w2.dtype)
                extra = torch.zeros(co, wsc.shape[1], 3, device=w2.device, dtype=w2.dtype)
                extra[:, :, 1] = wsc
                w = torch.cat([w2, extra], dim=1)
                convs[p + ".conv2"] = (_row_conv(w.shape[1], co, k=3, pad=1, relu=True), w, s2)
        w, s = taps3(h.conv2, h.bn2)
        convs["head.conv2"] = (_row_conv(w.shape[1], w.shape[0], k=3, pad=1, relu=True), w, s)
        xv = self.xvector
        # TDNN: input channels reordered from the reference's c * 10 + f to the gathered f * 32 + c
        a, s = _bn_affine(xv.tdnn.nonlinear.batchnorm)
        w = xv.tdnn.linear.weight.detach() * a[:, None, None]
        co, ci, k = w.shape
        nf = ci // h.in_planes
        w = w.reshape(co, h.in_planes, nf, k).permute(0, 2, 1, 3).reshape(co, ci, k)
        convs["tdnn"] = (_row_conv(ci, co, k=k, pad=k // 2, stride=2, relu=True), w, s)
        for bi in (1, 2, 3):
            block = getattr(xv, f"block{bi}")
            for name, layer in block.named_children():
                p = f"block{bi}.{name}"
                affines[p] = _bn_affine(layer.nonlinear1.batchnorm)
                a, s = _bn_affine(layer.nonlinear2.batchnorm)
                w = layer.linear1.weight.detach() * a[:, None, None]
                convs[p + ".linear1"] = (_row_conv(w.shape[1], w.shape[0], relu=True), w, s)
                st = layer.se.linear_stem
                convs[p + ".stem"] = (_row_conv(st.in_channels, st.out_channels, k=st.kernel_size[0],
                                                dilation=st.dilation[0], pad=st.padding[0]), st.weight.detach(), None)
            tr = getattr(xv, f"transit{bi}")
            affines[f"transit{bi}"] = _bn_affine(tr.nonlinear.batchnorm)
            w = tr.linear.weight.detach()
            if bi == 3:       # the final BatchNorm + ReLU fold into transit3
                a, s = _bn_affine(self.bn)
                convs["transit3"] = (_row_conv(w.shape[1], w.shape[0], relu=True), w * a[:, None, None], s)
            else:
                convs[f"transit{bi}"] = (_row_conv(w.shape[1], w.shape[0]), w, None)
        a, s = _bn_affine(xv.dense.nonlinear.batchnorm)
        w = xv.dense.linear.weight.detach() * a[:, None, None]
        convs["dense"] = (_row_conv(w.shape[1], w.shape[0]), w, s)
        return convs, affines

    def _folded(self):
        key = tuple((d[n].data_ptr(), d[n]._version) for d, n in self._slots)
        if self._run is not None and self._run_key == key:
            return self._run
        with torch.no_grad():
            convs, affines = self._fold()
            if self._run is None or next(iter(self._run[0].values())).w.device != self.head.conv1.weight.device:
                layers = {n: _Layer(spec, w, b) for n, (spec, w, b) in convs.items()}
                aff = {n: (a.contiguous().clone(), s.contiguous().clone()) for n, (a, s) in affines.items()}
                self.__dict__["_run"] = (layers, aff)
            else:
                layers, aff = self._run
                for n, (_, w, b) in convs.items():
                    layers[n].update(w, b)
                for n, (a, s) in affines.items():
                    aff[n][0].copy_(a)
                    aff[n][1].copy_(s)
        self.__dict__["_run_key"] = key
        return self._run

    # ---- forward ------------------------------------------------------------------------------------------------------
    def forward(self, feats, lengths=None):
        if self.training:
            raise RuntimeError("kantts_b200.DTDNN is inference only (no backward): call .eval() first")
        if feats.dim() != 3 or feats.shape[2] != N_MELS:
            raise ValueError(f"DTDNN: expected (B, T, {N_MELS}) features, got {tuple(feats.shape)}")
        B, T, _ = feats.shape
        lens = _host_lengths([T] * B if lengths is None else lengths, T, "DTDNN")
        with torch.no_grad():
            layers, aff = self._folded()
            x = feats.detach().float().contiguous()
            dev = x.device
            T2 = (T - 1) // 2 + 1
            lens2 = [(n - 1) // 2 + 1 for n in lens]
            lg = torch.tensor(lens + lens2, dtype=torch.int32).to(dev, non_blocking=True)
            lg1, lg2 = lg[:B], lg[B:]
            h = self._head(x, layers, lg1, B, T)                             # (B, T, 320), channels f * 32 + c
            t0 = layers["tdnn"](h)                                           # (B, T2, 128)
            for bi in (1, 2, 3):
                block = getattr(self.xvector, f"block{bi}")
                c0 = t0.shape[2]
                c_final = c0 + sum(l.se.linear_stem.out_channels for l in block)
                slab = torch.empty(B, T2, c_final, device=dev, dtype=torch.float32)
                ops.call("kt_se_affine_rows", ptr(t0), c0, None, None, 0, ptr(lg2, True), ptr(slab), c_final, B, T2, c0)
                c = c0
                for name, layer in block.named_children():
                    c = self._dense_layer(slab, c, c_final, layer, layers, aff, f"block{bi}.{name}", lg2, B, T2)
                a, s = aff[f"transit{bi}"]
                xn = torch.empty(B, T2, c_final, device=dev, dtype=torch.float32)
                ops.call("kt_se_affine_rows", ptr(slab), c_final, ptr(a), ptr(s), 1, ptr(lg2, True), ptr(xn), c_final, B, T2,
                         c_final)
                t0 = layers[f"transit{bi}"](xn)
            c = t0.shape[2]
            stats = torch.empty(B, 1, 2 * c, device=dev, dtype=torch.float32)
            ops.call("kt_se_stats_pool", ptr(t0), ptr(lg2, True), ptr(stats), B, T2, c)
            y = layers["dense"](stats)
        return y.reshape(B, -1)

    def _head(self, x, layers, lg, B, T):
        """(B, T, 80) features -> (B, T, 320) rows of the head's output, channel f * 32 + c, rows past each item zero."""
        F = x.shape[2]

        def gather(src, f_in, c, f_out, taps, stride, pad, y=None, first=0, strides=None):
            """taps frequency rows of src (B, f_in, T, c) per output frequency -> channels [first, first + taps c) of y."""
            if y is None:
                y = torch.empty(B * f_out, T, taps * c, device=x.device, dtype=torch.float32)
            strides = strides or (f_in * T * c, T * c, c)
            ops.call("kt_se_tap_gather", ptr(src), *strides, ptr(lg, True), ctypes.c_void_p(y.data_ptr() + 4 * first),
                     y.shape[2], B, f_in, T, c, f_out, taps, stride, pad)
            return y

        a = layers["head.conv1"](gather(x, F, 1, F, 3, 1, 1, strides=(T * F, 1, F)))     # (B * 80, T, 32)
        f, c = F, a.shape[2]
        for ln in ("layer1", "layer2"):
            for j, blk in enumerate(getattr(self.head, ln)):
                p = f"head.{ln}.{j}"
                s = blk.stride
                fo = (f - 1) // s + 1
                mid = layers[p + ".conv1"](gather(a, f, c, fo, 3, s, 1))
                g2 = torch.empty(B * fo, T, 4 * c, device=x.device, dtype=torch.float32)
                gather(mid, fo, c, fo, 3, 1, 1, y=g2)
                gather(a, f, c, fo, 1, s, 0, y=g2, first=3 * c)                 # the shortcut's input
                a = layers[p + ".conv2"](g2)
                f = fo
        fo = (f - 1) // 2 + 1
        a = layers["head.conv2"](gather(a, f, c, fo, 3, 2, 1))                # (B * 10, T, 32)
        return gather(a, fo, c, 1, fo, 1, 0)                                   # (B, T, 10 * 32)

    def _dense_layer(self, slab, c, c_final, layer, layers, aff, p, lg, B, T):
        """SEDenseTDNNLayer on slab channels [0, c); its outputs land at channel c.  Launches: nonlinear1, linear1, the gate
        statistics, linear_stem, the gate -- five, plus one operand pre-pass for each conv on the tensor cores."""
        dev = slab.device
        a, s = aff[p]
        xn = torch.empty(B, T, c, device=dev, dtype=torch.float32)
        ops.call("kt_se_affine_rows", ptr(slab), c_final, ptr(a), ptr(s), 1, ptr(lg, True), ptr(xn), c, B, T, c)
        hmid = layers[p + ".linear1"](xn)                                    # relu(nonlinear2(linear1(x)))
        cm = hmid.shape[2]
        nseg = (T + SEG_LEN - 1) // SEG_LEN
        stats = torch.empty(B, nseg, 2, cm, device=dev, dtype=torch.float32)
        ops.call("kt_se_gate_stats", ptr(hmid), ptr(lg, True), ptr(stats), B, T, cm, SEG_LEN)
        y = layers[p + ".stem"](hmid)
        se = layer.se
        co = y.shape[2]
        out = ctypes.c_void_p(slab.data_ptr() + 4 * c)
        ops.call("kt_se_gate_apply", ptr(y), ptr(stats), ptr(se.linear1.weight.detach()), ptr(se.linear1.bias.detach()),
                 ptr(se.linear2.weight.detach()), ptr(se.linear2.bias.detach()), ptr(lg, True), out, c_final, B, T, cm,
                 se.linear1.out_channels, co, SEG_LEN)
        return c + co
