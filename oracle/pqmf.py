"""PQMF filter bank: float64 CPU restatement of kantts/models/pqmf.py (TEST INFRASTRUCTURE).

The filters are the reference's design (pqmf.py:13-44 prototype, :62-82 cosine modulation) with ``numpy.kaiser`` for the
removed ``scipy.signal.kaiser``; the two transforms are the reference's two-conv compositions (pqmf.py:107-134), run in
float64 so that they can serve as the reference for the fp32 kernels.  Pinned against tests/golden/multiband_small.npz."""
import numpy as np
import torch
import torch.nn.functional as F


def prototype_filter(taps=62, cutoff_ratio=0.142, beta=9.0):
    """pqmf.py:13-44"""
    omega_c = np.pi * cutoff_ratio
    n = np.arange(taps + 1) - 0.5 * taps
    with np.errstate(invalid="ignore"):
        h_i = np.sin(omega_c * n) / (np.pi * n)
    h_i[taps // 2] = cutoff_ratio
    return h_i * np.kaiser(taps + 1, beta)


def filters(subbands=4, taps=62, cutoff_ratio=0.142, beta=9.0):
    """pqmf.py:62-82 -> (analysis (S, 1, taps + 1), synthesis (1, S, taps + 1)) float64 tensors"""
    h = prototype_filter(taps, cutoff_ratio, beta)
    n = np.arange(taps + 1) - taps / 2
    ha = np.stack([2 * h * np.cos((2 * k + 1) * (np.pi / (2 * subbands)) * n + (-1) ** k * np.pi / 4)
                   for k in range(subbands)])
    hs = np.stack([2 * h * np.cos((2 * k + 1) * (np.pi / (2 * subbands)) * n - (-1) ** k * np.pi / 4)
                   for k in range(subbands)])
    return torch.from_numpy(ha).unsqueeze(1), torch.from_numpy(hs).unsqueeze(0)


def _updown(subbands, dtype):
    """pqmf.py:88-92"""
    u = torch.zeros(subbands, subbands, subbands, dtype=dtype)
    for k in range(subbands):
        u[k, k, 0] = 1.0
    return u


def analysis(x, analysis_filter, subbands, taps=62):
    """pqmf.py:107-118: (B, 1, T) -> (B, S, T // S)"""
    y = F.conv1d(F.pad(x, (taps // 2, taps // 2)), analysis_filter.to(x.dtype))
    return F.conv1d(y, _updown(subbands, x.dtype), stride=subbands)


def synthesis(x, synthesis_filter, subbands, taps=62):
    """pqmf.py:120-134: (B, S, n) -> (B, 1, S * n)"""
    y = F.conv_transpose1d(x, _updown(subbands, x.dtype) * subbands, stride=subbands)
    return F.conv1d(F.pad(y, (taps // 2, taps // 2)), synthesis_filter.to(x.dtype))
