"""``kantts.models.pqmf`` (KAN-TTS kantts/models/pqmf.py:13-134): the pseudo-QMF filter bank of the multi-band HiFi-GAN.

Same constructor, buffers (``analysis_filter``, ``synthesis_filter``, ``updown_filter``) and ``state_dict`` keys as the
reference.  Both transforms are one conv of the library each (ops.conv: forward and data gradient in the sm_90a kernels),
with fixed weights derived from the buffers:
  analysis   conv1d(pad(x, taps/2), analysis_filter) picked at every S-th sample (pqmf.py:107-118) is ONE stride-S conv
             1 -> S over taps + 1 samples, padded by taps/2;
  synthesis  conv_transpose1d(x, S * identity, stride=S) -- S-fold zero stuffing -- then conv1d(pad(., taps/2),
             synthesis_filter) (pqmf.py:120-134) is ONE stride-S transposed conv S -> 1 whose filter is the synthesis filter
             reversed in time and scaled by S.  Its output is S * n samples long, S - 1 beyond the plain transposed length
             (ConvSpec.crop = -(S - 1)); those samples gather only taps that fall on the zero-stuffed tail.
"""
import numpy as np
import torch
import torch.nn as nn

from . import ops


def design_prototype_filter(taps=62, cutoff_ratio=0.142, beta=9.0):
    """pqmf.py:13-44: the Kaiser-windowed sinc prototype (taps + 1,), float64.  ``numpy.kaiser`` is the window of the
    reference's ``scipy.signal.kaiser`` (removed from current scipy)."""
    assert taps % 2 == 0, "The number of taps mush be even number."
    assert 0.0 < cutoff_ratio < 1.0, "Cutoff ratio must be > 0.0 and < 1.0."
    omega_c = np.pi * cutoff_ratio
    n = np.arange(taps + 1) - 0.5 * taps
    with np.errstate(invalid="ignore"):
        h_i = np.sin(omega_c * n) / (np.pi * n)
    h_i[taps // 2] = np.cos(0) * cutoff_ratio
    return h_i * np.kaiser(taps + 1, beta)


def pqmf_filters(subbands=4, taps=62, cutoff_ratio=0.142, beta=9.0):
    """pqmf.py:62-82 -> (analysis (S, taps + 1), synthesis (S, taps + 1)) cosine-modulated filters, float64."""
    h_proto = design_prototype_filter(taps, cutoff_ratio, beta)
    n = np.arange(taps + 1) - taps / 2
    k = np.arange(subbands)[:, None]
    arg = (2 * k + 1) * (np.pi / (2 * subbands)) * n
    phase = (-1.0) ** k * np.pi / 4
    return 2 * h_proto * np.cos(arg + phase), 2 * h_proto * np.cos(arg - phase)


class PQMF(nn.Module):
    def __init__(self, subbands=4, taps=62, cutoff_ratio=0.142, beta=9.0):
        super().__init__()
        h_analysis, h_synthesis = pqmf_filters(subbands, taps, cutoff_ratio, beta)
        self.register_buffer("analysis_filter", torch.from_numpy(h_analysis).float().unsqueeze(1))
        self.register_buffer("synthesis_filter", torch.from_numpy(h_synthesis).float().unsqueeze(0))
        updown_filter = torch.zeros((subbands, subbands, subbands)).float()
        for k in range(subbands):
            updown_filter[k, k, 0] = 1.0
        self.register_buffer("updown_filter", updown_filter)
        self.subbands = subbands
        self.taps = taps
        half = taps // 2
        # pad_right: output length T // S like the reference's stride-S pick, also when S does not divide T
        self.analysis_spec = ops.ConvSpec(c_in=1, c_out=subbands, kernel=taps + 1, stride=subbands, pad_left=half,
                                          pad_right=half - (subbands - 1))
        self.synthesis_spec = ops.ConvSpec(c_in=subbands, c_out=1, kernel=taps + 1, stride=subbands, pad_left=half,
                                           transposed=True, crop=-(subbands - 1))
        self._caches = (ops.PreparedWeight(), ops.PreparedWeight())
        self._w = None

    def _weights(self):
        """-> the (analysis, synthesis) conv weights in the reference conv layouts, rebuilt when a buffer changed (device,
        storage or version).  Frozen nn.Parameters outside the module's registry: ops.prepare_weight keeps their kernel
        layouts across calls and none of them enters ``parameters()`` or the ``state_dict``."""
        a, s = self.analysis_filter, self.synthesis_filter
        key = (a.device, a.data_ptr(), a._version, s.data_ptr(), s._version)
        if self._w is None or self._w[0] != key:
            with torch.no_grad():
                wa = nn.Parameter(a.float().clone().contiguous(), requires_grad=False)                   # (S, 1, k)
                ws = nn.Parameter((s[0].float().flip(-1) * self.subbands).unsqueeze(1).contiguous(),     # (S, 1, k)
                                  requires_grad=False)
            self._w = (key, wa, ws)
        return self._w[1], self._w[2]

    def analysis(self, x):
        """(B, 1, T) -> (B, subbands, T // subbands)"""
        if x.dim() != 3 or x.shape[1] != 1:
            raise ValueError(f"PQMF.analysis expects (B, 1, T), got {tuple(x.shape)}")
        wa, _ = self._weights()
        rows = x.reshape(x.shape[0], x.shape[2], 1)                    # (B, T, 1): the same memory
        return ops.conv(rows, self.analysis_spec, self._caches[0], wa).transpose(1, 2)

    def synthesis(self, x, lengths=None):
        """(B, subbands, n) -> (B, 1, subbands * n).  ``lengths`` (inference only): each item's sub-band samples, a host
        sequence or a device int tensor (B,), 1 <= lengths[b] <= n; item b's output samples [0, subbands * lengths[b]) are
        then ``synthesis(x[b:b+1, :, :lengths[b]])`` and its later samples are zero."""
        if x.dim() != 3 or x.shape[1] != self.subbands:
            raise ValueError(f"PQMF.synthesis expects (B, {self.subbands}, n), got {tuple(x.shape)}")
        _, ws = self._weights()
        rows = x.transpose(1, 2).contiguous()
        if lengths is None:
            y = ops.conv(rows, self.synthesis_spec, self._caches[1], ws)   # (B, S * n, 1)
        else:
            lengths = ops.ragged_lengths(lengths, x.shape[0], x.shape[2], x.device)
            y = ops.conv(rows, self.synthesis_spec, self._caches[1], ws, mask=ops.utterance_mask(lengths, 1))
            ops.rows_mask(y, ops.utterance_mask(lengths, self.subbands))
        return y.reshape(y.shape[0], 1, y.shape[1])
