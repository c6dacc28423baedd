"""Seeded NSF excitation, the definition of kt_nsf_excitation (include/kantts_b200.h) restated in NumPy.

The reference's SourceModule (kantts/models/hifigan/layers.py:229-290) draws its initial phases and noise from torch's global
generator, so two calls never agree.  Here they come from Philox4x32-10 keyed by a per-slot seed and counted by the sample
index, and the harmonic phase is a float64 running sum carried between chunks: a chunk's rows are the matching rows of the
whole utterance's excitation, bit for bit."""
import numpy as np
import torch
import torch.nn.functional as F

from . import hifigan as H

_M0, _M1, _W0, _W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
_MASK = 0xFFFFFFFF
TWO_PI, PI = 2 * np.pi, np.pi


def philox4x32_10(counter, key):
    """Philox4x32-10 (Random123).  counter: 4 arrays (or ints) of uint32 words, key: 2 -> 4 uint64 arrays of the output
    words (values < 2^32), broadcast over the inputs."""
    c = [np.asarray(w, dtype=np.uint64) & _MASK for w in counter]
    k0, k1 = (np.asarray(w, dtype=np.uint64) & _MASK for w in key)
    for r in range(10):
        if r:
            k0, k1 = (k0 + _W0) & _MASK, (k1 + _W1) & _MASK
        p0, p1 = c[0] * np.uint64(_M0), c[2] * np.uint64(_M1)
        hi0, lo0, hi1, lo1 = p0 >> np.uint64(32), p0 & _MASK, p1 >> np.uint64(32), p1 & _MASK
        c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
    return c


def _seed_words(seed):
    s = int(seed) & 0xFFFFFFFFFFFFFFFF
    return s & _MASK, s >> 32


def _frac(x):
    return x - np.floor(x)


def initial_phases(seed, nb_harmonics):
    """phi_h, float32 (H + 1,): phi_0 = 0, phi_h = -pi + 2 pi w0 2^-32 with w0 from counter (0, 0, h, 1)."""
    h = np.arange(nb_harmonics + 1, dtype=np.uint64)
    w0 = philox4x32_10((0, 0, h, 1), _seed_words(seed))[0]
    phi = (-PI + TWO_PI * (w0.astype(np.float64) * 2.0 ** -32)).astype(np.float32)
    phi[0] = 0
    return phi


def normal_noise(seed, n, nb_harmonics):
    """z, float32 (len(n), H + 1): Box-Muller of the first two words of counter (n low, n high, h, 0), in float64."""
    n = np.asarray(n, dtype=np.uint64)[:, None]
    h = np.arange(nb_harmonics + 1, dtype=np.uint64)[None, :]
    w = philox4x32_10((n & _MASK, n >> np.uint64(32), h, 0), _seed_words(seed))
    u1 = (w[0].astype(np.float64) + 0.5) * 2.0 ** -32
    u2 = (w[1].astype(np.float64) + 0.5) * 2.0 ** -32
    return (np.sqrt(-2.0 * np.log(u1)) * np.cos(TWO_PI * u2)).astype(np.float32)


class ExcitationState:
    """One slot's carried state: the seed, phase[H + 1] (float64) and the samples done since the reset."""

    def __init__(self, seed, nb_harmonics):
        self.seed, self.phase, self.samples_done = int(seed), np.zeros(nb_harmonics + 1), 0


def excitation(f0, uv, state, hop, sampling_rate, alpha=0.1, sigma=0.003):
    """One slot's excitation of the frames f0 / uv ((frames,) Hz and voiced flag) -> float32 (frames * hop, H + 1); advances
    ``state``.  A fresh state and the whole utterance's frames give the whole-utterance excitation."""
    nch = state.phase.shape[0]
    f0 = np.asarray(f0, dtype=np.float32).astype(np.float64)
    uv = np.asarray(uv, dtype=np.float32)
    frames = f0.shape[0]
    c = f0[:, None] * np.arange(1, nch + 1, dtype=np.float64)[None, :] / float(sampling_rate)      # (frames, H + 1)
    p = np.empty((frames, nch))
    acc = state.phase.copy()
    for j in range(frames):                                     # the only order-dependent sum
        p[j] = acc
        acc = _frac(acc + float(hop) * c[j])
    i1 = np.arange(1, hop + 1, dtype=np.float64)[None, :, None]
    theta = (TWO_PI * _frac(p[:, None, :] + i1 * c[:, None, :])).astype(np.float32).reshape(frames * hop, nch)
    n = state.samples_done + np.arange(frames * hop, dtype=np.uint64)
    z = normal_noise(state.seed, n, nch - 1)
    phi = initial_phases(state.seed, nch - 1)
    a, s = np.float32(alpha), np.float32(sigma)
    k = np.float32(np.float64(a) / 3.0 / np.float64(s))
    noise = s * z
    voiced = a * np.sin(theta + phi[None, :]) + noise
    unvoiced = k * noise
    uvs = np.repeat(uv, hop)[:, None]
    e = voiced * uvs + unvoiced * (np.float32(1) - uvs)
    state.phase, state.samples_done = acc, state.samples_done + frames * hop
    return e.astype(np.float32)


def batch_excitation(pitch, uv, seeds, hop, sampling_rate, nb_harmonics, alpha=0.1, sigma=0.003):
    """Whole-utterance excitation of a batch: pitch / uv (B, 1, frames) tensors or arrays, one seed per slot -> float32
    (B, H + 1, frames * hop), the layout of the reference's SourceModule before its 1x1 conv."""
    pitch, uv = np.asarray(pitch, dtype=np.float32), np.asarray(uv, dtype=np.float32)
    return np.stack([excitation(pitch[b, 0], uv[b, 0], ExcitationState(s, nb_harmonics), hop, sampling_rate, alpha,
                                sigma).T for b, s in enumerate(seeds)])


def source_ffn(sd, e):
    """The SourceModule's weight-normed 1x1 conv (nb_harmonics+1 -> 1) and tanh over an excitation e (B, H+1, samples)
    (layers.py:283-290)."""
    w = H._resolve_weight(sd, "source_module.ffn.0.")
    return torch.tanh(F.conv1d(e, w, sd["source_module.ffn.0.bias"]))


def generator_forward(sd, x, excitation, **cfg):
    """hifigan.generator_forward of an NSF generator (hifigan.py:145-182) with a GIVEN excitation e (B, nb_harmonics+1,
    samples), e.g. batch_excitation's, in place of the reference's random draw: the same layer functions, the excitation's
    1x1 conv and tanh, then per stage ``source_downs`` (strided convs, kernel 2u / stride u / padding u//2; a 1x1 conv at
    the full rate, :119-143) added to the stage input (:162-166).  x: (B, in_channels + 2, T), the last two channels pitch
    and voiced flag (unused here: the excitation already holds them)."""
    c = dict(H.GENERATOR_DEFAULTS)
    c.update(cfg)
    assert c["repeat_upsample"] and c["nsf_params"] is not None
    causal, ks = c["causal"], c["kernel_size"]
    slope = c["nonlinear_activation_params"]["negative_slope"]
    nk = len(c["resblock_kernel_sizes"])
    x = x[:, :-2, :]
    source = source_ffn(sd, excitation.to(x.dtype))
    scales = list(c["upsample_scales"])
    down_rates = list(np.cumprod([1] + scales[::-1][:-1])[::-1])        # stage i sees the source / down_rates[i]
    x = H.conv1d(sd, "conv_pre.", x, causal, (ks - 1) // 2)
    for i, (s, uk) in enumerate(zip(scales, c["upsample_kernal_sizes"])):
        x = torch.sin(x) + x
        rep = F.leaky_relu(F.interpolate(x, scale_factor=s, mode="nearest"), slope)
        rep = H.conv1d(sd, f"repeat_upsamples.{i}.2.", rep, causal, (ks - 1) // 2)
        up = H.conv_transpose1d(sd, f"transpose_upsamples.{i}.1.", F.leaky_relu(x, slope), causal, s, (uk - s) // 2)
        x = rep + up[:, :, : rep.shape[-1]]
        u = int(down_rates[i])
        if u == 1:
            x = x + H.conv1d(sd, f"source_downs.{i}.", source, False, 0)
        else:
            x = x + H.conv1d(sd, f"source_downs.{i}.", source, causal, u // 2, 1, u)
        xs = None
        for j in range(nk):
            r = H.residual_block(sd, f"conv_blocks.{i * nk + j}.", x, c["resblock_kernel_sizes"][j],
                                 c["resblock_dilations"][j], causal, slope)
            xs = r if xs is None else xs + r
        x = xs / nk
    x = H.conv1d(sd, "conv_post.", F.leaky_relu(x), causal, (ks - 1) // 2)
    return torch.tanh(x)
