"""Restatement of the speaker-embedding extractor of kantts/preprocess/se_processor: the Kaldi fbank the processor takes
from torchaudio (numpy, float64) and the D-TDNN forward (D_TDNN.py, layers.py) in eval mode, as torch functional calls on a
state_dict.  One utterance at a time, like the processor (se_processor.py:54-76); runs on whatever device the state_dict
is on."""
import math

import numpy as np
import torch
import torch.nn.functional as F

FRAME_LEN, FRAME_SHIFT, N_FFT = 400, 160, 512
FLT_EPSILON = float(np.finfo(np.float32).eps)


def _mel(hz):
    return 1127.0 * np.log(1.0 + np.asarray(hz, dtype=np.float64) / 700.0)


def kaldi_mel_banks(n_mels=80, sample_rate=16000, low_hz=20.0):
    """(n_mels, 257) Kaldi triangles on the mel scale 1127 ln(1 + f / 700), low_hz to Nyquist; the Nyquist bin is 0."""
    m_lo, m_hi = _mel(low_hz), _mel(0.5 * sample_rate)
    delta = (m_hi - m_lo) / (n_mels + 1)
    m = np.arange(n_mels, dtype=np.float64)[:, None]
    left, center, right = m_lo + m * delta, m_lo + (m + 1) * delta, m_lo + (m + 2) * delta
    mel = _mel(sample_rate / N_FFT * np.arange(N_FFT // 2))[None, :]
    w = np.maximum(0.0, np.minimum((mel - left) / (center - left), (right - mel) / (right - center)))
    return np.pad(w, ((0, 0), (0, 1)))


def kaldi_fbank(wav, n_mels=80, sample_rate=16000):
    """torchaudio.compliance.kaldi.fbank(wav[None], num_mel_bins=n_mels) at its other defaults, for a 1-D wav: frames of
    400 samples every 160 (snip_edges), DC removal, pre-emphasis 0.97 (the first sample against itself), povey window,
    512-point power spectrum, log(max(e, FLT_EPSILON)).  -> (frames, n_mels) float64."""
    x = np.asarray(wav, dtype=np.float64)
    n = 1 + (len(x) - FRAME_LEN) // FRAME_SHIFT
    if len(x) < FRAME_LEN:
        raise ValueError("shorter than one frame")
    idx = np.arange(n)[:, None] * FRAME_SHIFT + np.arange(FRAME_LEN)[None, :]
    fr = x[idx]
    fr = fr - fr.mean(axis=1, keepdims=True)
    fr = fr - 0.97 * np.concatenate([fr[:, :1], fr[:, :-1]], axis=1)
    win = (0.5 - 0.5 * np.cos(2 * math.pi * np.arange(FRAME_LEN) / (FRAME_LEN - 1))) ** 0.85
    spec = np.abs(np.fft.rfft(fr * win, n=N_FFT)) ** 2
    e = spec @ kaldi_mel_banks(n_mels, sample_rate).T
    return np.log(np.maximum(e, FLT_EPSILON))


def cmn(feat):
    """se_processor.py:67: subtract the mean over the frames."""
    return feat - feat.mean(axis=0, keepdims=True)


# ---- D-TDNN (eval mode) ----------------------------------------------------------------------------------------------
def _bn(sd, p, x):
    return F.batch_norm(x, sd[p + ".running_mean"], sd[p + ".running_var"], sd.get(p + ".weight"), sd.get(p + ".bias"),
                        False, 0.0, 1e-5)


def _basic_block(sd, p, x, stride):
    out = F.relu(_bn(sd, p + ".bn1", F.conv2d(x, sd[p + ".conv1.weight"], stride=(stride, 1), padding=1)))
    out = _bn(sd, p + ".bn2", F.conv2d(out, sd[p + ".conv2.weight"], padding=1))
    if p + ".shortcut.0.weight" in sd:
        x = _bn(sd, p + ".shortcut.1", F.conv2d(x, sd[p + ".shortcut.0.weight"], stride=(stride, 1)))
    return F.relu(out + x)


def _head(sd, x):
    x = x.unsqueeze(1)
    out = F.relu(_bn(sd, "head.bn1", F.conv2d(x, sd["head.conv1.weight"], padding=1)))
    for layer in ("layer1", "layer2"):
        out = _basic_block(sd, f"head.{layer}.0", out, 2)
        out = _basic_block(sd, f"head.{layer}.1", out, 1)
    out = F.relu(_bn(sd, "head.bn2", F.conv2d(out, sd["head.conv2.weight"], stride=(2, 1), padding=1)))
    return out.reshape(out.shape[0], out.shape[1] * out.shape[2], out.shape[3])


def _seg_pooling(x, seg_len=100):
    s = F.max_pool1d(x, kernel_size=seg_len, stride=seg_len, ceil_mode=True)
    return s.unsqueeze(-1).expand(-1, -1, -1, seg_len).reshape(*x.shape[:-1], -1)[:, :, :x.shape[-1]]


def _dense_layer(sd, p, x, dilation):
    h = F.conv1d(F.relu(_bn(sd, p + ".nonlinear1.batchnorm", x)), sd[p + ".linear1.weight"])
    h = F.relu(_bn(sd, p + ".nonlinear2.batchnorm", h))
    y = F.conv1d(h, sd[p + ".se.linear_stem.weight"], padding=dilation, dilation=dilation)
    s = F.conv1d(h.mean(-1, keepdim=True) + _seg_pooling(h), sd[p + ".se.linear1.weight"], sd[p + ".se.linear1.bias"])
    s = torch.sigmoid(F.conv1d(F.relu(s), sd[p + ".se.linear2.weight"], sd[p + ".se.linear2.bias"]))
    return y * s


def dtdnn_forward(sd, feats):
    """(B, T, 80) features (every frame valid) -> (B, 192) embeddings of DTDNN.forward in eval mode."""
    x = _head(sd, feats.permute(0, 2, 1))
    x = F.relu(_bn(sd, "xvector.tdnn.nonlinear.batchnorm", F.conv1d(x, sd["xvector.tdnn.linear.weight"], stride=2,
                                                                      padding=2)))
    for bi, dilation in ((1, 1), (2, 2), (3, 3)):
        i = 1
        while f"xvector.block{bi}.tdnnd{i}.linear1.weight" in sd:
            x = torch.cat([x, _dense_layer(sd, f"xvector.block{bi}.tdnnd{i}", x, dilation)], dim=1)
            i += 1
        p = f"xvector.transit{bi}"
        x = F.conv1d(F.relu(_bn(sd, p + ".nonlinear.batchnorm", x)), sd[p + ".linear.weight"])
    x = F.relu(_bn(sd, "bn", x))
    x = torch.cat([x.mean(dim=-1), x.std(dim=-1, unbiased=True)], dim=-1)
    x = F.conv1d(x.unsqueeze(-1), sd["xvector.dense.linear.weight"]).squeeze(-1)
    return _bn(sd, "xvector.dense.nonlinear.batchnorm", x)


def seed_bn_stats(module_or_sd, seed=7):
    """The documented rule that makes eval-mode BatchNorm no identity in the goldens: for every BatchNorm, in state_dict
    order, from a torch.Generator seeded with `seed`: running_mean = 0.1 N(0, 1), running_var = 0.5 + U(0, 1); with
    affine, weight = 1 + 0.1 N(0, 1), bias = 0.1 N(0, 1).  Applied in place to a state_dict (or a module's)."""
    sd = module_or_sd.state_dict() if hasattr(module_or_sd, "state_dict") else module_or_sd
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for k, v in sd.items():
            if not k.endswith(".running_mean"):
                continue
            p = k[:-len(".running_mean")]
            c = v.numel()
            v.copy_(0.1 * torch.randn(c, generator=g))
            sd[p + ".running_var"].copy_(0.5 + torch.rand(c, generator=g))
            if p + ".weight" in sd:
                sd[p + ".weight"].copy_(1.0 + 0.1 * torch.randn(c, generator=g))
                sd[p + ".bias"].copy_(0.1 * torch.randn(c, generator=g))
    return sd
