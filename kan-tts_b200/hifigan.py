"""H100-native HiFi-GAN modules with the reference's module API.

Drop-in replacements for ``kantts.models.hifigan.hifigan.{Generator, MultiPeriodDiscriminator,
MultiScaleDiscriminator}`` (KAN-TTS kantts/models/hifigan/hifigan.py:22-478, layers.py:15-226):
same class names, constructor kwargs (yaml ``params``), forward signatures / return structure,
``state_dict`` keys and shapes, ``remove_weight_norm()`` and ``nsf_enable``; parameters are plain
leaf ``nn.Parameter``s so ``torch.optim.Adam`` / ``DistributedDataParallel`` work unchanged.

Every tensor op of the forward and backward runs in libkantts_b200.so (hand-written sm_90a
kernels) through ``ops.py``; activations are channels-last rows internally and are converted only
at the module boundary (feature maps are returned as zero-copy permuted views).
The NSF branch (``nsf_params``) is module plumbing over the same kernels and has NOT run on a GPU yet (round 1 ran out
of GPU budget: tests/test_gpu_pipeline.py is opt-in).  Out of scope (SURVEY.md section 8a): MultiSpecDiscriminator, PQMF.
"""
import copy
import math
import os

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import ops
from ._lib import KT_ACT_LRELU, KT_ACT_NONE, KT_ACT_TANH, KT_PATH_AUTO

# --------------------------------------------------------------------------------------------
# parameter holders (names / shapes == the reference's weight_norm / spectral_norm wrapped convs)
# --------------------------------------------------------------------------------------------


_PARALLEL_STREAMS = os.environ.get("KANTTS_B200_STREAMS", "1") != "0"
_SPECTRAL_ON_MAIN = os.environ.get("KANTTS_B200_SPECTRAL_ON_MAIN", "1") != "0"
_STREAMS = {}


def _side_streams(device, n):
    """Per-device pool of side streams for the independent sub-discriminators."""
    key = (device.type, device.index)
    pool = _STREAMS.setdefault(key, [])
    while len(pool) < n:
        pool.append(torch.cuda.Stream(device=device))
    return pool[:n]


def join_side_streams(device=None):
    """Make the current stream wait for everything queued on the side-stream pool.  Needed after a backward
    whose parameter gradients were accumulated inside the kernels (ops.mark_direct_grad): the autograd engine
    only joins the streams its own AccumulateGrad nodes ran on."""
    for (dev_type, dev_index), pool in _STREAMS.items():
        if device is not None and (dev_type, dev_index) != (device.type, device.index):
            continue
        cur = torch.cuda.current_stream(torch.device(dev_type, dev_index))
        for s in pool:
            cur.wait_stream(s)
    ops.join_wgrad_streams(device)


def prefetch_weights(module, streams):
    """Launch the weight preparation of every weight-normed / plain conv of ``module`` on ``streams`` (round-robin,
    one contiguous share of the layers per stream).  The caller forks the streams off the current one before and
    joins them before the module's next forward.  Spectral-normed layers recompute their weight per forward."""
    layers = [m for m in module.modules() if isinstance(m, _NormedConv) and m.norm != "spectral" and m._cache.last is not None]
    n = len(streams)
    for i, s in enumerate(streams):
        share = layers[i::n]
        if not share:
            continue
        with torch.cuda.stream(s):
            for m in share:
                v, g = m.effective_weight()
                ops.prefetch_weight(m._cache, m.spec, v, g)


def _split_pair(outs, fmaps, nb, detach_b):
    """Results of one batched call on cat([ya, yb]) -> ((outs_a, fmaps_a), (outs_b, fmaps_b)); slices of the
    channels-last buffers are contiguous, so downstream fast paths (kt_l1_sum) still apply."""
    det = (lambda t: t.detach()) if detach_b else (lambda t: t)
    a = ([o[:nb] for o in outs], [[f[:nb] for f in fm] for fm in fmaps])
    b = ([det(o[nb:]) for o in outs], [[det(f[nb:]) for f in fm] for fm in fmaps])
    return a, b


def _consume_init_weights_rng(weight):
    """kantts/models/utils.py:7-10 ``init_weights`` runs ``m.weight.data.normal_(0, 0.01)`` AFTER
    weight_norm: it overwrites the derived ``weight`` (recomputed from g, v at the next forward), so
    it only advances the RNG.  Advance it identically to keep seed-for-seed identical inits."""
    torch.empty_like(weight).normal_(0.0, 0.01)


class _NormedConv(nn.Module):
    """Holds the parameters of ``weight_norm(nn.ConvXd)`` / ``spectral_norm(nn.ConvXd)`` / a plain
    conv under the reference's names (``weight_g``/``weight_v`` | ``weight_orig``/``weight_u``/
    ``weight_v`` | ``weight``) and computes the layer through ops.ConvFn."""

    def __init__(self, torch_conv, spec, norm="weight", init_weights=False):
        super().__init__()
        w = torch_conv.weight.detach()
        self.spec = spec
        self.norm = norm
        self._cache = ops.PreparedWeight()
        # registration order matches the reference state_dict key order: weight_norm / spectral_norm
        # re-register the weight AFTER the bias; a plain conv keeps (weight, bias)
        if norm not in ("weight", "spectral"):
            self.weight = nn.Parameter(w.clone())
        if torch_conv.bias is not None:
            self.bias = nn.Parameter(torch_conv.bias.detach().clone())
        else:
            self.register_parameter("bias", None)
        if norm == "weight":
            # torch.nn.utils.weight_norm: g = ||w|| over all dims but 0, v = w
            self.weight_g = nn.Parameter(w.norm(2, dim=tuple(range(1, w.dim())), keepdim=True).clone())
            self.weight_v = nn.Parameter(w.clone())
        elif norm == "spectral":
            # torch.nn.utils.spectral_norm (legacy): u ~ normalize(N(0,1)^h), v ~ normalize(N(0,1)^w)
            h = w.shape[0]
            wd = w.reshape(h, -1).shape[1]
            u = F.normalize(w.new_empty(h).normal_(0, 1), dim=0, eps=1e-12)
            v = F.normalize(w.new_empty(wd).normal_(0, 1), dim=0, eps=1e-12)
            self.weight_orig = nn.Parameter(w.clone())
            self.register_buffer("weight_u", u)
            self.register_buffer("weight_v", v)
        if init_weights:
            _consume_init_weights_rng(w)

    def effective_weight(self):
        """-> (v, g) to hand to the kernel: weight-norm is fused into kt_weight_prepare; the
        spectral-norm power iteration (8 thin layers) runs as torch ops exactly like the reference's
        hook, including the in-place u / v buffer update on every training-mode forward."""
        if self.norm == "weight":
            return self.weight_v, self.weight_g
        if self.norm == "spectral":
            w = self.weight_orig
            wm = w.reshape(w.shape[0], -1)
            u, v = self.weight_u, self.weight_v
            if self.training:
                with torch.no_grad():
                    v_new = F.normalize(torch.mv(wm.t(), u), dim=0, eps=1e-12)
                    u_new = F.normalize(torch.mv(wm, v_new), dim=0, eps=1e-12)
                    v.copy_(v_new)
                    u.copy_(u_new)
                u, v = u.clone(), v.clone()
            sigma = torch.dot(u, torch.mv(wm, v))
            return w / sigma, None
        return self.weight, None

    def run(self, x, resid=None):
        v, g = self.effective_weight()
        if self.norm == "spectral":      # sigma changes with every forward: never part of pair_reuse
            return ops.conv(x, self.spec, self._cache, v, g, self.bias, resid)
        return ops.pair_conv(self, x, self.spec, self._cache, v, g, self.bias, resid)

    def remove_weight_norm(self):
        if self.norm != "weight":
            raise ValueError("weight_norm not applied")
        with torch.no_grad():
            v, g = self.weight_v, self.weight_g
            w = v * (g / v.norm(2, dim=tuple(range(1, v.dim())), keepdim=True))
        del self.weight_g, self.weight_v
        self.weight = nn.Parameter(w)
        self.norm = "none"
        self._cache = ops.PreparedWeight()


def get_padding(kernel_size, dilation=1):
    return int((kernel_size * dilation - dilation) / 2)


class Conv1d(nn.Module):
    """layers.py:15-49 (non-causal, symmetric padding)."""
    causal = False

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1,
                 bias=True, padding_mode="zeros", act_in=None, upsample=1):
        super().__init__()
        ref = nn.Conv1d(in_channels, out_channels, kernel_size, stride, padding=0 if self.causal else padding,
                        dilation=dilation, groups=groups, bias=bias)
        if self.causal:
            pl, pr = (kernel_size - 1) * dilation, 0          # layers.py:66,83-87
        else:
            pl = pr = padding
        spec = ops.ConvSpec(c_in=in_channels, c_out=out_channels, kernel=kernel_size, stride=stride,
                            dilation=dilation, pad_left=pl, pad_right=pr, groups=groups, upsample=upsample)
        if act_in is not None:
            spec.act_in, spec.act_in_slope = KT_ACT_LRELU, float(act_in)
        self.conv1d = _NormedConv(ref, spec, "weight", init_weights=True)

    def forward_rows(self, x, resid=None):
        return self.conv1d.run(x, resid)

    def forward(self, x):
        """(B, C, T) -> (B, C', T'); the reference signature."""
        return self.forward_rows(x.transpose(1, 2).contiguous()).transpose(1, 2)

    def remove_weight_norm(self):
        self.conv1d.remove_weight_norm()


class CausalConv1d(Conv1d):
    """layers.py:49-91"""
    causal = True


class ConvTranspose1d(nn.Module):
    """layers.py:94-124"""
    causal = False

    def __init__(self, in_channels, out_channels, kernel_size, stride, padding=0, output_padding=0, act_in=None):
        super().__init__()
        ref = nn.ConvTranspose1d(in_channels, out_channels, kernel_size, stride, padding=0 if self.causal else padding,
                                 output_padding=0)
        crop = max(kernel_size - stride, 0) if self.causal else 0   # layers.py:151,161
        spec = ops.ConvSpec(c_in=in_channels, c_out=out_channels, kernel=kernel_size, stride=stride,
                            pad_left=0 if self.causal else padding, transposed=True, crop=crop)
        if act_in is not None:
            spec.act_in, spec.act_in_slope = KT_ACT_LRELU, float(act_in)
        self.deconv = _NormedConv(ref, spec, "weight", init_weights=True)
        self.stride = stride
        self.pad = kernel_size - stride

    def forward_rows(self, x, resid=None):
        return self.deconv.run(x, resid)

    def forward(self, x):
        return self.forward_rows(x.transpose(1, 2).contiguous()).transpose(1, 2)

    def remove_weight_norm(self):
        self.deconv.remove_weight_norm()


class CausalConvTranspose1d(ConvTranspose1d):
    """layers.py:127-165"""
    causal = True


class ResidualBlock(nn.Module):
    """layers.py:168-226: for (c1, c2): x = c2(lrelu(c1(lrelu(x)))) + x, the LeakyReLUs fused into the
    conv kernels' operand staging and the residual add into c2's epilogue."""

    def __init__(self, channels, kernel_size=3, dilation=(1, 3, 5), nonlinear_activation="LeakyReLU",
                 nonlinear_activation_params={"negative_slope": 0.1}, causal=False):
        super().__init__()
        assert kernel_size % 2 == 1, "Kernal size must be odd number."
        if nonlinear_activation != "LeakyReLU":
            raise NotImplementedError("kantts_b200: only LeakyReLU is fused into the conv kernels")
        slope = nonlinear_activation_params.get("negative_slope", 0.01)
        conv_cls = CausalConv1d if causal else Conv1d
        self.convs1 = nn.ModuleList([
            conv_cls(channels, channels, kernel_size, 1, dilation=dilation[i],
                     padding=get_padding(kernel_size, dilation[i]), act_in=slope) for i in range(len(dilation))])
        self.convs2 = nn.ModuleList([
            conv_cls(channels, channels, kernel_size, 1, dilation=1, padding=get_padding(kernel_size, 1),
                     act_in=slope) for i in range(len(dilation))])
        self.activation = getattr(nn, nonlinear_activation)(**nonlinear_activation_params)

    def forward_rows(self, x):
        for c1, c2 in zip(self.convs1, self.convs2):
            n1, n2 = c1.conv1d, c2.conv1d
            rd = ops.resblock_desc(n1.spec, n2.spec, x.shape[0], x.shape[1]) \
                if (ops._FUSE_RESBLOCK and not ops._FORCE_FFMA and x.dim() == 3 and n1.norm != "spectral" and n2.norm != "spectral") else None
            if rd is not None:
                # thin stages (32 / 64 channels): the pair is ONE launch, the intermediate stays on the SM (kt_resblock_fwd)
                v1, g1 = n1.effective_weight()
                v2, g2 = n2.effective_weight()
                x = ops.resblock(x, n1.spec, n1._cache, v1, g1, n1.bias, n2.spec, n2._cache, v2, g2, n2.bias, rd)
            else:
                xt = c1.forward_rows(x)
                x = c2.forward_rows(xt, resid=x)
        return x

    def forward(self, x):
        return self.forward_rows(x.transpose(1, 2).contiguous()).transpose(1, 2)

    def remove_weight_norm(self):
        for layer in self.convs1:
            layer.remove_weight_norm()
        for layer in self.convs2:
            layer.remove_weight_norm()


class SourceModule(nn.Module):
    """layers.py:229-290: sine-plus-noise excitation of the neural source filter + a weight-normed 1x1 conv
    (nb_harmonics + 1 -> 1) + tanh (fused into the conv's epilogue).  The excitation itself is O(samples x 8)
    elementwise work under ``no_grad``; like the reference, the random initial phases and the noise are drawn on the
    HOST from torch's global CPU generator (``Uniform`` / ``Normal`` with Python-float parameters sample on the CPU,
    layers.py:266-279) and copied over, which keeps the RNG stream identical to the reference's."""

    def __init__(self, nb_harmonics, upsample_ratio, sampling_rate, alpha=0.1, sigma=0.003):
        super().__init__()
        self.nb_harmonics, self.upsample_ratio, self.sampling_rate = nb_harmonics, int(upsample_ratio), sampling_rate
        self.alpha, self.sigma = alpha, sigma
        ref = nn.Conv1d(nb_harmonics + 1, 1, kernel_size=1, stride=1)
        spec = ops.ConvSpec(c_in=nb_harmonics + 1, c_out=1, kernel=1)
        spec.act_out = KT_ACT_TANH
        self.ffn = nn.Sequential(_NormedConv(ref, spec, "weight"), nn.Tanh())    # keys ffn.0.{bias,weight_g,weight_v}

    def excitation(self, pitch, uv):
        """(B, 1, frames) pitch in Hz and voiced flag -> (B, samples, nb_harmonics + 1) rows (no gradient)."""
        from torch.distributions.normal import Normal
        from torch.distributions.uniform import Uniform
        with torch.no_grad():
            pitch_s = F.interpolate(pitch, scale_factor=self.upsample_ratio, mode="nearest")
            uv_s = F.interpolate(uv, scale_factor=self.upsample_ratio, mode="nearest")
            harm = torch.arange(1, self.nb_harmonics + 2, device=pitch.device, dtype=pitch_s.dtype)[None, :, None]
            theta = 2 * math.pi * (torch.cumsum(pitch_s * harm / self.sampling_rate, dim=-1) % 1)
            phase = Uniform(low=-math.pi, high=math.pi).sample(sample_shape=(pitch.size(0), self.nb_harmonics + 1, 1))
            phase[:, 0, :] = 0
            noise = Normal(loc=0.0, scale=self.sigma).sample(
                sample_shape=(pitch_s.size(0), self.nb_harmonics + 1, pitch_s.size(-1)))
            phase, noise = phase.to(pitch.device), noise.to(pitch.device)
            e_voice = self.alpha * torch.sin(theta + phase) + noise
            e_unvoice = self.alpha / 3 / self.sigma * noise
            e = e_voice * uv_s + e_unvoice * (1 - uv_s)
            return e.transpose(1, 2).contiguous()

    def forward_rows(self, pitch, uv):
        return self.ffn[0].run(self.excitation(pitch, uv))          # (B, samples, 1)

    def forward(self, pitch, uv):
        return self.forward_rows(pitch, uv).transpose(1, 2)

    def remove_weight_norm(self):
        self.ffn[0].remove_weight_norm()


# --------------------------------------------------------------------------------------------
# Generator (hifigan.py:22-198)
# --------------------------------------------------------------------------------------------


class Generator(nn.Module):
    def __init__(self, in_channels=80, out_channels=1, channels=512, kernel_size=7,
                 upsample_scales=(8, 8, 2, 2), upsample_kernal_sizes=(16, 16, 4, 4),
                 resblock_kernel_sizes=(3, 7, 11), resblock_dilations=[(1, 3, 5), (1, 3, 5), (1, 3, 5)],
                 repeat_upsample=True, bias=True, causal=True, nonlinear_activation="LeakyReLU",
                 nonlinear_activation_params={"negative_slope": 0.1}, use_weight_norm=True, nsf_params=None):
        super().__init__()
        assert kernel_size % 2 == 1, "Kernal size must be odd number."
        assert len(upsample_scales) == len(upsample_kernal_sizes)
        assert len(resblock_dilations) == len(resblock_kernel_sizes)
        if not repeat_upsample:
            raise NotImplementedError("kantts_b200: repeat_upsample=False is not used by any shipped config")
        if nonlinear_activation != "LeakyReLU":
            raise NotImplementedError("kantts_b200: only LeakyReLU is fused into the conv kernels")
        if out_channels != 1:
            raise NotImplementedError("kantts_b200: multi-band (PQMF) output is out of scope")
        slope = nonlinear_activation_params.get("negative_slope", 0.01)
        self.upsample_scales = upsample_scales
        self.repeat_upsample = repeat_upsample
        self.num_upsamples = len(upsample_kernal_sizes)
        self.num_kernels = len(resblock_kernel_sizes)
        self.out_channels = out_channels
        self.nsf_enable = nsf_params is not None
        if self.num_kernels > 3:
            raise NotImplementedError("kantts_b200: at most 3 parallel resblocks per stage")

        self.transpose_upsamples = nn.ModuleList()
        self.repeat_upsamples = nn.ModuleList()
        self.conv_blocks = nn.ModuleList()
        conv_cls = CausalConv1d if causal else Conv1d
        deconv_cls = CausalConvTranspose1d if causal else ConvTranspose1d

        self.conv_pre = conv_cls(in_channels, channels, kernel_size, 1, padding=(kernel_size - 1) // 2)
        for i in range(len(upsample_kernal_sizes)):
            cin, cout = channels // (2 ** i), channels // (2 ** (i + 1))
            s, k = upsample_scales[i], upsample_kernal_sizes[i]
            # the LeakyReLU (index 0) is fused into the deconv's operand staging
            self.transpose_upsamples.append(nn.Sequential(
                getattr(nn, nonlinear_activation)(**nonlinear_activation_params),
                deconv_cls(cin, cout, k, s, padding=(k - s) // 2, act_in=slope)))
            # nn.Upsample (index 0) and the LeakyReLU (index 1) are fused into the conv: rows are
            # gathered at t // scale and never materialised
            self.repeat_upsamples.append(nn.Sequential(
                nn.Upsample(mode="nearest", scale_factor=s),
                getattr(nn, nonlinear_activation)(**nonlinear_activation_params),
                conv_cls(cin, cout, kernel_size=kernel_size, stride=1, padding=(kernel_size - 1) // 2,
                         act_in=slope, upsample=s)))
            for j in range(len(resblock_kernel_sizes)):
                self.conv_blocks.append(ResidualBlock(
                    channels=cout, kernel_size=resblock_kernel_sizes[j], dilation=resblock_dilations[j],
                    nonlinear_activation=nonlinear_activation,
                    nonlinear_activation_params=nonlinear_activation_params, causal=causal))
        # F.leaky_relu(x) (default slope 0.01, hifigan.py:178) and tanh (:180) are fused into conv_post
        self.conv_post = conv_cls(channels // (2 ** (i + 1)), out_channels, kernel_size, 1,
                                  padding=(kernel_size - 1) // 2, act_in=0.01)
        self.conv_post.conv1d.spec.act_out = KT_ACT_TANH
        if self.nsf_enable:
            # hifigan.py:119-143: the excitation at the sample rate, brought down to every stage's rate by a strided
            # conv (kernel 2u, stride u, padding u//2; the full-rate stage uses a plain 1x1 conv)
            self.source_module = SourceModule(nb_harmonics=nsf_params["nb_harmonics"],
                                              upsample_ratio=int(np.cumprod(list(upsample_scales))[-1]),
                                              sampling_rate=nsf_params["sampling_rate"])
            self.source_downs = nn.ModuleList()
            self.downsample_rates = [1] + list(upsample_scales)[::-1][:-1]
            self.downsample_cum_rates = np.cumprod(self.downsample_rates)
            for i, u in enumerate(self.downsample_cum_rates[::-1]):
                u = int(u)
                if u == 1:
                    self.source_downs.append(Conv1d(1, channels // (2 ** (i + 1)), 1, 1))
                else:
                    self.source_downs.append(conv_cls(1, channels // (2 ** (i + 1)), u * 2, u, padding=u // 2))

    def forward_rows(self, x, excitation=None):
        x = self.conv_pre.forward_rows(x)
        for i in range(self.num_upsamples):
            x = ops.SinAddFn.apply(x)                                        # hifigan.py:157
            rep = self.repeat_upsamples[i][2].forward_rows(x)                # :158
            if excitation is not None:                                       # :162-166  x = rep + e + up (adds fused)
                rep = self.source_downs[i].forward_rows(excitation, resid=rep)
            x = self.transpose_upsamples[i][1].forward_rows(x, resid=rep)    # :160,168 (crop fused: t_out)
            par = x.is_cuda and _PARALLEL_STREAMS and self.num_kernels > 1
            if par:                                                           # the parallel resblocks are independent
                cur = torch.cuda.current_stream()
                streams = _side_streams(x.device, self.num_kernels)
                rs = []
                for j in range(self.num_kernels):
                    streams[j].wait_stream(cur)
                    with torch.cuda.stream(streams[j]):
                        rs.append(self.conv_blocks[i * self.num_kernels + j].forward_rows(x))
                for s in streams[: self.num_kernels]:
                    cur.wait_stream(s)
            else:
                rs = [self.conv_blocks[i * self.num_kernels + j].forward_rows(x) for j in range(self.num_kernels)]
            rs += [None] * (3 - len(rs))
            x = ops.Mean3Fn.apply(1.0 / self.num_kernels, *rs)               # :170-176
        return self.conv_post.forward_rows(x)                                # :178-180

    def forward(self, x):
        """x: (B, in_channels, T) -> (B, 1, T * prod(scales)); with ``nsf_params`` the last two channels are the
        pitch (Hz) and the voiced flag (hifigan.py:146-150)."""
        excitation = None
        if self.nsf_enable:
            x, pitch, uv = x[:, :-2, :], x[:, -2:-1, :], x[:, -1:, :]
            excitation = self.source_module.forward_rows(pitch, uv)         # (B, samples, 1)
        y = self.forward_rows(x.transpose(1, 2).contiguous(), excitation)   # (B, T', 1)
        return y.transpose(1, 2)

    def remove_weight_norm(self):
        print("Removing weight norm...")
        for layer in self.transpose_upsamples:
            layer[-1].remove_weight_norm()
        for layer in self.repeat_upsamples:
            layer[-1].remove_weight_norm()
        for layer in self.conv_blocks:
            layer.remove_weight_norm()
        self.conv_pre.remove_weight_norm()
        self.conv_post.remove_weight_norm()
        if self.nsf_enable:                                   # (the reference forgets these; harmless either way)
            self.source_module.remove_weight_norm()
            for layer in self.source_downs:
                layer.remove_weight_norm()


# --------------------------------------------------------------------------------------------
# MultiPeriodDiscriminator (hifigan.py:200-302)
# --------------------------------------------------------------------------------------------


class _Conv2dK1(_NormedConv):
    """``norm_f(nn.Conv2d(cin, cout, (k, 1), (s, 1), padding=(p, 0)))`` computed as a Conv1d over
    the ``period`` interleaved sub-sequences of a channels-last (B, H, period, C) tensor."""

    def __init__(self, cin, cout, k, stride, pad, norm, act_out_slope=None):
        ref = nn.Conv2d(cin, cout, (k, 1), (stride, 1), padding=(pad, 0))
        spec = ops.ConvSpec(c_in=cin, c_out=cout, kernel=k, stride=stride, pad_left=pad, pad_right=pad)
        if act_out_slope is not None:
            spec.act_out, spec.act_out_slope = KT_ACT_LRELU, float(act_out_slope)
        super().__init__(ref, spec, norm)


class PeriodDiscriminator(nn.Module):
    def __init__(self, in_channels=1, out_channels=1, period=3, kernel_sizes=[5, 3], channels=32,
                 downsample_scales=[3, 3, 3, 3, 1], max_downsample_channels=1024, bias=True,
                 nonlinear_activation="LeakyReLU", nonlinear_activation_params={"negative_slope": 0.1},
                 use_spectral_norm=False):
        super().__init__()
        if nonlinear_activation != "LeakyReLU":
            raise NotImplementedError("kantts_b200: only LeakyReLU is fused into the conv kernels")
        slope = nonlinear_activation_params.get("negative_slope", 0.01)
        self.period = period
        norm = "spectral" if use_spectral_norm else "weight"
        self.convs = nn.ModuleList()
        in_chs, out_chs = in_channels, channels
        for s in downsample_scales:
            # Sequential(conv, LeakyReLU): the activation (index 1) is fused into the conv epilogue
            self.convs.append(nn.Sequential(
                _Conv2dK1(in_chs, out_chs, kernel_sizes[0], s, (kernel_sizes[0] - 1) // 2, norm, slope),
                getattr(nn, nonlinear_activation)(**nonlinear_activation_params)))
            in_chs = out_chs
            out_chs = min(out_chs * 4, max_downsample_channels)
        self.conv_post = _Conv2dK1(out_chs, out_channels, kernel_sizes[1] - 1, 1, (kernel_sizes[1] - 1) // 2, "none")

    def forward(self, x):
        """x: (B, 1, T) -> (flattened output (B, n), list of (B, C, H, period) feature maps)"""
        fmap = []
        b, c, t = x.shape
        assert c == 1, "PeriodDiscriminator expects a mono waveform (B, 1, T)"
        if t % self.period != 0:
            n_pad = self.period - (t % self.period)
            x = F.pad(x, (0, n_pad), "reflect")
            t = t + n_pad
        # (B, 1, T) -> channels-last (B, H, period, C=1): identical memory
        x = x.reshape(b, t // self.period, self.period, c)
        for layer in self.convs:
            x = layer[0].run(x)
            fmap.append(x.permute(0, 3, 1, 2))
        x = self.conv_post.run(x)
        fmap.append(x.permute(0, 3, 1, 2))
        return torch.flatten(x.permute(0, 3, 1, 2), 1, -1), fmap


class MultiPeriodDiscriminator(nn.Module):
    def __init__(self, periods=[2, 3, 5, 7, 11], discriminator_params={
            "in_channels": 1, "out_channels": 1, "kernel_sizes": [5, 3], "channels": 32,
            "downsample_scales": [3, 3, 3, 3, 1], "max_downsample_channels": 1024, "bias": True,
            "nonlinear_activation": "LeakyReLU", "nonlinear_activation_params": {"negative_slope": 0.1},
            "use_spectral_norm": False}):
        super().__init__()
        self.discriminators = nn.ModuleList()
        for period in periods:
            params = copy.deepcopy(discriminator_params)
            params["period"] = period
            self.discriminators += [PeriodDiscriminator(**params)]

    def forward(self, y):
        # The period discriminators are independent and their late layers are too small to fill 132 SMs:
        # run them on side streams (fork / join around the loop; autograd replays the same streams in
        # backward, and CUDA-graph capture records the branches as parallel graph paths).
        y_d_rs, fmap_rs = [], []
        par = y.is_cuda and _PARALLEL_STREAMS and len(self.discriminators) > 1
        if par:
            cur = torch.cuda.current_stream()
            streams = _side_streams(y.device, len(self.discriminators))
        for i, d in enumerate(self.discriminators):
            if par:
                streams[i].wait_stream(cur)
                with torch.cuda.stream(streams[i]):
                    y_d_r, fmap_r = d(y)
            else:
                y_d_r, fmap_r = d(y)
            y_d_rs.append(y_d_r)
            fmap_rs.append(fmap_r)
        if par:
            for s in streams:
                cur.wait_stream(s)
        return y_d_rs, fmap_rs


    def forward_pair(self, ya, yb, detach_b=False):
        """== (self(ya), self(yb)), evaluated as ONE batch: every layer is launched once on 2B items instead
        of twice on B (the trainer always runs the discriminators on a (generated, real) pair:
        trainer.py:519-531,560-566).  No layer of this discriminator mixes batch items, so the results are
        identical.  ``detach_b``: the second result is returned detached (the reference's no_grad pass)."""
        assert ya.shape == yb.shape
        outs, fmaps = self.forward(torch.cat([ya, yb], 0))
        return _split_pair(outs, fmaps, ya.shape[0], detach_b)


# --------------------------------------------------------------------------------------------
# MultiScaleDiscriminator (hifigan.py:305-478)
# --------------------------------------------------------------------------------------------


class _Conv1dD(_NormedConv):
    def __init__(self, cin, cout, k, stride, pad, groups, bias, norm, act_out_slope=None):
        ref = nn.Conv1d(cin, cout, k, stride=stride, padding=pad, groups=groups, bias=bias)
        spec = ops.ConvSpec(c_in=cin, c_out=cout, kernel=k, stride=stride, pad_left=pad, pad_right=pad, groups=groups)
        if act_out_slope is not None:
            spec.act_out, spec.act_out_slope = KT_ACT_LRELU, float(act_out_slope)
        super().__init__(ref, spec, norm)


class ScaleDiscriminator(nn.Module):
    def __init__(self, in_channels=1, out_channels=1, kernel_sizes=[15, 41, 5, 3], channels=128,
                 max_downsample_channels=1024, max_groups=16, bias=True, downsample_scales=[2, 2, 4, 4, 1],
                 nonlinear_activation="LeakyReLU", nonlinear_activation_params={"negative_slope": 0.1},
                 use_spectral_norm=False):
        super().__init__()
        if nonlinear_activation != "LeakyReLU":
            raise NotImplementedError("kantts_b200: only LeakyReLU is fused into the conv kernels")
        slope = nonlinear_activation_params.get("negative_slope", 0.01)
        norm = "spectral" if use_spectral_norm else "weight"
        assert len(kernel_sizes) == 4
        for ks in kernel_sizes:
            assert ks % 2 == 1
        act = lambda: getattr(nn, nonlinear_activation)(**nonlinear_activation_params)  # noqa: E731
        self.convs = nn.ModuleList()
        self.convs.append(nn.Sequential(
            _Conv1dD(in_channels, channels, kernel_sizes[0], 1, (kernel_sizes[0] - 1) // 2, 1, bias, norm, slope), act()))
        in_chs, out_chs, groups = channels, channels, 4
        for s in downsample_scales:
            self.convs.append(nn.Sequential(
                _Conv1dD(in_chs, out_chs, kernel_sizes[1], s, (kernel_sizes[1] - 1) // 2, groups, bias, norm, slope),
                act()))
            in_chs = out_chs
            out_chs = min(in_chs * 2, max_downsample_channels)
            groups = min(groups * 4, max_groups)
        out_chs = min(in_chs * 2, max_downsample_channels)
        self.convs.append(nn.Sequential(
            _Conv1dD(in_chs, out_chs, kernel_sizes[2], 1, (kernel_sizes[2] - 1) // 2, 1, bias, norm, slope), act()))
        self.conv_post = _Conv1dD(out_chs, out_channels, kernel_sizes[3], 1, (kernel_sizes[3] - 1) // 2, 1, bias, norm)

    def forward_rows(self, x):
        fmap = []
        for layer in self.convs:
            x = layer[0].run(x)
            fmap.append(x.transpose(1, 2))
        x = self.conv_post.run(x)
        fmap.append(x.transpose(1, 2))
        return torch.flatten(x.transpose(1, 2), 1, -1), fmap

    def forward(self, x):
        return self.forward_rows(x.transpose(1, 2).contiguous())


class DWT1DForward(nn.Module):
    """Buffer-compatible stand-in for ``pytorch_wavelets.DWT1DForward(J=1, wave="db3")``
    (hifigan.py:447): keeps the ``h0`` / ``h1`` (1,1,6) buffers in the state_dict; the transform
    itself is the fused kt_dwt_db3 kernel (filters are compile-time constants there)."""
    DEC_LO = [0.035226291882100656, -0.08544127388224149, -0.13501102001039084,
              0.4598775021193313, 0.8068915093133388, 0.3326705529509569]
    DEC_HI = [-0.3326705529509569, 0.8068915093133388, -0.4598775021193313,
              -0.13501102001039084, 0.08544127388224149, 0.035226291882100656]

    def __init__(self, J=1, wave="db3", mode="zero"):
        super().__init__()
        if not (J == 1 and wave == "db3" and mode == "zero"):
            raise NotImplementedError("kantts_b200: only DWT1DForward(J=1, wave='db3', mode='zero')")
        self.register_buffer("h0", torch.tensor(self.DEC_LO[::-1], dtype=torch.float32).view(1, 1, 6))
        self.register_buffer("h1", torch.tensor(self.DEC_HI[::-1], dtype=torch.float32).view(1, 1, 6))

    def forward(self, x):
        """(B, 1, T) -> (yl, [yh]) like the package (each (B, 1, T2))."""
        y = ops.DwtFn.apply(x.reshape(x.shape[0], -1))
        return y[..., 0].unsqueeze(1), [y[..., 1].unsqueeze(1)]


class _AvgPoolRows(nn.Module):
    """nn.AvgPool1d(kernel_size, stride, padding) on the mono waveform (hifigan.py:456-458, count_include_pad=True): a
    1 -> 1 channel FIR with constant taps 1/k on the C_in = 1 kernels (kt_conv1d_fwd / _bwd_data); no parameters, no
    buffers (like the reference's pooling module, it adds nothing to the state_dict)."""

    def __init__(self, kernel_size=4, stride=2, padding=2):
        super().__init__()
        self.spec = ops.ConvSpec(c_in=1, c_out=1, kernel=int(kernel_size), stride=int(stride), pad_left=int(padding),
                                 pad_right=int(padding))
        self._cache = ops.PreparedWeight()
        self._w = None

    def run(self, rows):
        """rows: (B, T, 1) -> (B, T2, 1)"""
        if self._w is None or self._w.device != rows.device:
            self._w = torch.full((1, 1, self.spec.kernel), 1.0 / self.spec.kernel, device=rows.device)
        return ops.conv(rows, self.spec, self._cache, self._w)

    def forward(self, y):
        return self.run(y.transpose(1, 2).contiguous()).transpose(1, 2)


class MultiScaleDiscriminator(nn.Module):
    def __init__(self, scales=3, downsample_pooling="DWT",
                 downsample_pooling_params={"kernel_size": 4, "stride": 2, "padding": 2},
                 discriminator_params={
                     "in_channels": 1, "out_channels": 1, "kernel_sizes": [15, 41, 5, 3], "channels": 128,
                     "max_downsample_channels": 1024, "max_groups": 16, "bias": True,
                     "downsample_scales": [2, 2, 4, 4, 1], "nonlinear_activation": "LeakyReLU",
                     "nonlinear_activation_params": {"negative_slope": 0.1}},
                 follow_official_norm=False):
        super().__init__()
        self.discriminators = nn.ModuleList()
        for i in range(scales):
            params = copy.deepcopy(discriminator_params)
            if follow_official_norm:
                params["use_spectral_norm"] = True if i == 0 else False
            self.discriminators += [ScaleDiscriminator(**params)]
        if downsample_pooling == "DWT":
            self.meanpools = nn.ModuleList([DWT1DForward(wave="db3", J=1), DWT1DForward(wave="db3", J=1)])
            # weight_norm(nn.Conv1d(2, 1, 15, 1, padding=7)) + F.leaky_relu(y, 0.1) (hifigan.py:449-454,471-472)
            self.aux_convs = nn.ModuleList([_Conv1dD(2, 1, 15, 1, 7, 1, True, "weight", 0.1),
                                            _Conv1dD(2, 1, 15, 1, 7, 1, True, "weight", 0.1)])
        else:
            self.meanpools = nn.ModuleList([_AvgPoolRows(**downsample_pooling_params) for _ in range(2)])
            self.aux_convs = None

    def forward(self, y):
        """y: (B, 1, T) -> (list of (B, n_i), list of list of (B, C, T_l) feature maps)"""
        return self._run(y, None)

    def forward_pair(self, ya, yb, detach_b=False):
        """== (self(ya), self(yb)) evaluated as one batch of 2B (see MultiPeriodDiscriminator.forward_pair).
        A spectral-normed scale (follow_official_norm: scale 0) updates its power-iteration vectors on every
        training-mode forward (torch.nn.utils.spectral_norm hook), so its two calls use different sigmas: that
        scale alone still runs twice, on the two halves of the batch, in the reference's order."""
        assert ya.shape == yb.shape
        nb = ya.shape[0]
        outs, fmaps = self._run(torch.cat([ya, yb], 0), nb)
        det = (lambda t: t.detach()) if detach_b else (lambda t: t)
        ra, rb = ([], []), ([], [])
        for o, fm in zip(outs, fmaps):
            if isinstance(o, tuple):                       # a scale that ran per half
                (oa, ob), (fa, fb) = o, fm
                fb = [det(f) for f in fb]
                ob = det(ob)
            else:
                oa, ob = o[:nb], det(o[nb:])
                fa, fb = [f[:nb] for f in fm], [det(f[nb:]) for f in fm]
            ra[0].append(oa); ra[1].append(fa)
            rb[0].append(ob); rb[1].append(fb)
        return ra, rb

    def _run(self, y, pair_nb):
        y_d_rs, fmap_rs = [], []
        rows = y.transpose(1, 2).contiguous()                                 # (B, T, 1)
        inputs = [rows]
        for i in range(1, len(self.discriminators)):                          # the pooling chain is cheap and serial
            if self.aux_convs is None:                                        # nn.AvgPool1d variant (hifigan.py:456-458,466)
                rows = self.meanpools[i - 1].run(rows)
            else:
                cat = ops.DwtFn.apply(rows.reshape(rows.shape[0], -1))        # (B, T2, 2) = cat([yl, yh], 1)
                rows = self.aux_convs[i - 1].run(cat)                          # (B, T2, 1), lrelu fused
            inputs.append(rows)
        par = y.is_cuda and _PARALLEL_STREAMS and len(self.discriminators) > 1
        if par:                                                               # the scales themselves are independent
            cur = torch.cuda.current_stream()
            streams = _side_streams(y.device, len(self.discriminators))

        def run_scale(d, x):
            if pair_nb is not None and any(getattr(l[0], "norm", "") == "spectral" for l in d.convs):
                # the two calls of the reference, in ITS order (the power iteration makes the order observable): the
                # discriminator phase evaluates the real waveforms first (trainer.py:560-561) -- with pair_state("reuse") the
                # batch is [re-generated | real], so the second half goes first
                st = ops._pair_state
                if st is not None and st[0] == "reuse":
                    ob, fb = d.forward_rows(x[pair_nb:])
                    oa, fa = d.forward_rows(x[:pair_nb])
                else:
                    oa, fa = d.forward_rows(x[:pair_nb])
                    ob, fb = d.forward_rows(x[pair_nb:])
                return (oa, ob), (fa, fb)
            return d.forward_rows(x)

        for i, d in enumerate(self.discriminators):
            # a spectral-normed scale stays on the calling stream: its parameters receive their gradients through autograd
            # (w / sigma is recomputed per forward), and with that chain on a side stream the gradient of the first layer's
            # weight_orig was intermittently lost when the scale is used twice in one backward
            side = par and not (_SPECTRAL_ON_MAIN and any(getattr(l[0], "norm", "") == "spectral" for l in d.convs))
            if side:
                streams[i].wait_stream(cur)
                with torch.cuda.stream(streams[i]):
                    y_d_r, fmap_r = run_scale(d, inputs[i])
            else:
                y_d_r, fmap_r = run_scale(d, inputs[i])
            y_d_rs.append(y_d_r)
            fmap_rs.append(fmap_r)
        if par:
            for s in streams:
                cur.wait_stream(s)
        return y_d_rs, fmap_rs
