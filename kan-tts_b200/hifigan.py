"""H100-native HiFi-GAN modules with the reference's module API.

Drop-in replacements for ``kantts.models.hifigan.hifigan.{Generator, MultiPeriodDiscriminator,
MultiScaleDiscriminator, SpecDiscriminator, MultiSpecDiscriminator}`` (KAN-TTS kantts/models/hifigan/hifigan.py:22-617,
layers.py:15-226):
same class names, constructor kwargs (yaml ``params``), forward signatures / return structure,
``state_dict`` keys and shapes, ``remove_weight_norm()`` and ``nsf_enable``; parameters are plain
leaf ``nn.Parameter``s so ``torch.optim.Adam`` / ``DistributedDataParallel`` work unchanged.

Every tensor op of the forward and backward runs in libkantts_b200.so (hand-written sm_90a
kernels) through ``ops.py``; activations are channels-last rows internally and are converted only
at the module boundary (feature maps are returned as zero-copy permuted views).
A multi-band generator (``out_channels`` = S > 1) emits S sub-band signals at 1/S of the sample rate; the PQMF filter bank
(pqmf.py) turns them into the waveform.  Like the reference, the PQMF is not part of the generator: the model builder adds
it next to the generator, and inference attaches it as ``generator.pqmf`` after loading; streaming (GeneratorStreamer)
runs the attached PQMF's synthesis as its last stage.  ``MultiSpecDiscriminator`` (the multi-resolution spectrogram
discriminator, hifigan.py:481-617) trains on the STFT and conv kernels plus kt_spec_columns_fwd / _bwd.  Out of scope
(SURVEY.md section 8a): a multi-band NSF generator.
"""
import copy
import ctypes
import math
from collections import namedtuple
from dataclasses import replace

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import ops
from .audio import stft
from ._lib import KT_ACT_LRELU, KT_ACT_NONE, KT_ACT_TANH, KT_PATH_AUTO, KT_PATH_BF16, KtNsfState, ptr
from .stream import Streamer, WindowTable, check_slots, own_weight, to_device

# --------------------------------------------------------------------------------------------
# parameter holders (names / shapes == the reference's weight_norm / spectral_norm wrapped convs)
# --------------------------------------------------------------------------------------------


_PARALLEL_STREAMS = True   # False: every sub-discriminator on the calling stream (bench.py's per-launch event timings)
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
    """Launch the weight preparation of every weight-normed / plain conv of ``module`` that has run through ConvFn
    (convs that only run inside the fused resblock are left to their forward) on ``streams`` (round-robin,
    one contiguous share of the layers per stream).  The caller forks the streams off the current one before and
    joins them before the module's next forward.  Spectral-normed layers recompute their weight per forward."""
    layers = [m for m in module.modules() if isinstance(m, _NormedConv) and m.norm != "spectral" and m._cache.conv_used]
    n = len(streams)
    for i, s in enumerate(streams):
        share = layers[i::n]
        if not share:
            continue
        with torch.cuda.stream(s):
            for m in share:
                v, g = m.effective_weight()
                ops.prefetch_weight(m._cache, m.spec, v, g)


# tensor-core precisions of set_precision: the compute path of a conv that may take the tensor cores
PRECISIONS = {"bf16x3": KT_PATH_AUTO, "bf16": KT_PATH_BF16}


def set_precision(module, precision):
    """Run every tensor-core conv of a HiFi-GAN ``module`` tree (Generator, discriminators, PQMF) in ``precision``:
    "bf16x3" (the default: split-bf16 operands, three MMAs per product, near-fp32 results) or "bf16" (each operand rounded
    once to bf16, one MMA, fp32 accumulation).  Layers without a tensor-core route keep their exact-fp32 kernels in either.
    The precision is not state: parameters, checkpoints and the optimizer are fp32 in both, and switching back gives the
    bits of a model never switched.  Streamers made afterwards run in the new precision.  SAM-BERT, syBERT and the speaker
    model (DTDNN) have no single-pass bf16 kernels: a tree containing one raises ValueError.  -> ``module``."""
    if precision not in PRECISIONS:
        raise ValueError(f"set_precision: precision must be one of {sorted(PRECISIONS)}, got {precision!r}")
    mods = list(module.modules())
    for m in mods:
        if type(m).__module__.rsplit(".", 1)[-1] in ("sambert", "speaker"):
            raise ValueError(f"set_precision: {type(m).__name__} has no single-pass bf16 kernels (HiFi-GAN models only)")
    new = PRECISIONS[precision]
    for m in mods:
        for spec in vars(m).values():
            if isinstance(spec, ops.ConvSpec) and spec.path in PRECISIONS.values():
                spec.path = new
    return module


def _spectral(d):
    """Is any conv of sub-discriminator ``d`` spectral-normed?"""
    return any(getattr(l[0], "norm", "") == "spectral" for l in d.convs)


def _run_halves(forward, x, pair_nb):
    """A spectral-normed sub-discriminator on a pair batch: the two calls of the reference, in ITS order (the power iteration
    makes the order observable).  The discriminator phase evaluates the real waveforms first (trainer.py:560-561) -- with
    pair_state("reuse") the batch is [re-generated | real], so the second half goes first.  -> ((out_a, out_b), (fmap_a,
    fmap_b)), which _split_runs takes apart."""
    st = ops._pair_state
    if st is not None and st[0] == "reuse":
        ob, fb = forward(x[pair_nb:])
        oa, fa = forward(x[:pair_nb])
    else:
        oa, fa = forward(x[:pair_nb])
        ob, fb = forward(x[pair_nb:])
    return (oa, ob), (fa, fb)


def _split_runs(outs, fmaps, nb, detach_b):
    """Results of one pair-batch run over cat([ya, yb]) whose sub-discriminators either ran on the whole batch or per half
    (_run_halves) -> ((outs_a, fmaps_a), (outs_b, fmaps_b)); ``detach_b``: the second result is returned detached."""
    det = (lambda t: t.detach()) if detach_b else (lambda t: t)
    ra, rb = ([], []), ([], [])
    for o, fm in zip(outs, fmaps):
        if isinstance(o, tuple):                       # a sub-discriminator that ran per half
            (oa, ob), (fa, fb) = o, fm
            fb = [det(f) for f in fb]
            ob = det(ob)
        else:
            oa, ob = o[:nb], det(o[nb:])
            fa, fb = [f[:nb] for f in fm], [det(f[nb:]) for f in fm]
        ra[0].append(oa); ra[1].append(fa)
        rb[0].append(ob); rb[1].append(fb)
    return ra, rb


def _run_parallel(y, jobs):
    """Run the independent sub-discriminator calls ``jobs`` [(fn, may_take_side_stream)] -> ([outputs], [feature maps]).
    On the GPU each call that may runs on a side stream of its own (fork / join around the loop; autograd replays the
    same streams in backward, and CUDA-graph capture records the branches as parallel graph paths).  A spectral-normed
    sub-discriminator stays on the calling stream: its parameters receive their gradients through autograd (w / sigma is
    recomputed per forward), and with that chain on a side stream the gradient of the first layer's weight_orig was
    intermittently lost when the sub-discriminator is used twice in one backward."""
    par = y.is_cuda and _PARALLEL_STREAMS and len(jobs) > 1
    if par:
        cur = torch.cuda.current_stream()
        streams = _side_streams(y.device, len(jobs))
    outs, fmaps, forked = [], [], []
    for i, (fn, side) in enumerate(jobs):
        if par and side:
            streams[i].wait_stream(cur)
            forked.append(streams[i])
            with torch.cuda.stream(streams[i]):
                o, fm = fn()
        else:
            o, fm = fn()
        outs.append(o)
        fmaps.append(fm)
    # join only the streams this call forked: under CUDA-graph capture, waiting on a pool stream whose last work was
    # not captured (a spectral-normed job's slot that nothing else in the graph used) invalidates the capture
    for s in forked:
        cur.wait_stream(s)
    return outs, fmaps


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

    def run(self, x, resid=None, mask=None):
        v, g = self.effective_weight()
        if self.norm == "spectral" or mask is not None:    # sigma changes with every forward: never part of pair_reuse
            return ops.conv(x, self.spec, self._cache, v, g, self.bias, resid, mask=mask)
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

    def forward_rows(self, x, resid=None, mask=None):
        return self.conv1d.run(x, resid, mask)

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

    def forward_rows(self, x, resid=None, mask=None):
        return self.deconv.run(x, resid, mask)

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

    def forward_rows(self, x, mask=None):
        """``mask`` (ops.utterance_mask of x's rows): each item's rows past its utterance read as zeros in both convs of every
        pair (c2 reads the intermediate under the same mask: it has x's rows)."""
        for c1, c2 in zip(self.convs1, self.convs2):
            n1, n2 = c1.conv1d, c2.conv1d
            rd = ops.resblock_desc(n1.spec, n2.spec, x.shape[0], x.shape[1]) \
                if (x.dim() == 3 and n1.norm != "spectral" and n2.norm != "spectral") else None
            if rd is not None:
                # thin stages (32 / 64 channels): the pair is ONE launch, the intermediate stays on the SM (kt_resblock_fwd)
                v1, g1 = n1.effective_weight()
                v2, g2 = n2.effective_weight()
                x = ops.resblock(x, n1.spec, n1._cache, v1, g1, n1.bias, n2.spec, n2._cache, v2, g2, n2.bias, rd, mask)
            else:
                xt = c1.forward_rows(x, mask=mask)
                x = c2.forward_rows(xt, resid=x, mask=mask)
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

    def excitation(self, pitch, uv, seeds=None):
        """(B, 1, frames) pitch in Hz and voiced flag -> (B, samples, nb_harmonics + 1) rows (no gradient).  With ``seeds``
        (one per batch item: a host sequence or a device int64 tensor (B,)) the excitation is kt_nsf_excitation's seeded
        function of (seed, pitch, uv, sample index) instead of the reference's draw from the global CPU generator."""
        if seeds is not None:
            return self._seeded_excitation(pitch, uv, seeds)
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

    def _seeded_excitation(self, pitch, uv, seeds):
        if not pitch.is_cuda:
            raise RuntimeError("kantts_b200: the seeded NSF excitation runs on a CUDA device (no CPU fallback)")
        B, _, frames = pitch.shape
        with torch.no_grad(), torch.cuda.device(pitch.device):
            state = NsfState(self, nsf_seed_tensor(seeds, B, pitch.device))
            f0uv = torch.cat([pitch, uv], 1).transpose(1, 2).float().contiguous()         # (B, frames, 2)
            e = torch.empty(B, frames * self.upsample_ratio, self.nb_harmonics + 1, device=pitch.device)
            self.run_excitation(f0uv, 0, state, e, 0, frames)
            return e

    def run_excitation(self, f0uv, f0uv_first, state, e, e_first, frames):
        """kt_nsf_excitation: rows [f0uv_first, + frames) of the (B, pitch, 2) f0 / uv window -> rows [e_first, + frames * hop)
        of the (B, pitch, nb_harmonics + 1) excitation window; advances ``state`` (an NsfState) on the device."""
        ops.call("kt_nsf_excitation", ptr(f0uv), f0uv.shape[1], f0uv_first, ctypes.byref(state.desc), ptr(e), e.shape[1],
                 e_first, f0uv.shape[0], frames, self.upsample_ratio, self.nb_harmonics, int(self.sampling_rate),
                 float(self.alpha), float(self.sigma), launches=2)

    def forward_rows(self, pitch, uv, seeds=None):
        return self.ffn[0].run(self.excitation(pitch, uv, seeds))   # (B, samples, 1)

    def forward(self, pitch, uv, seeds=None):
        return self.forward_rows(pitch, uv, seeds).transpose(1, 2)

    def remove_weight_norm(self):
        self.ffn[0].remove_weight_norm()


def nsf_seed_tensor(seeds, n, device):
    """-> ``seeds`` (a host sequence of ints or an int64 tensor) as a device int64 tensor (n,); ValueError on a wrong
    count or dtype."""
    if torch.is_tensor(seeds):
        if seeds.dtype != torch.int64:
            raise ValueError(f"NSF seeds must be int64, got {seeds.dtype}")
        s = seeds.reshape(-1)
    else:
        s = torch.as_tensor([int(v) for v in seeds], dtype=torch.int64)
    if s.numel() != n:
        raise ValueError(f"expected {n} NSF seeds (one per slot), got {s.numel()}")
    return s.to(device)


class NsfState:
    """The device state of kt_nsf_excitation for a batch: seeds (B,) int64, phase (B, nb_harmonics + 1) float64 and
    samples_done (B,) int64 (zeros: every slot at the start of its utterance), and the KtNsfState pointing at them."""

    def __init__(self, source, seeds):
        dev = seeds.device
        self.seeds = seeds.contiguous()
        self.phase = torch.zeros(seeds.numel(), source.nb_harmonics + 1, dtype=torch.float64, device=dev)
        self.samples_done = torch.zeros(seeds.numel(), dtype=torch.int64, device=dev)
        self.desc = KtNsfState(seeds=ptr(self.seeds, True), phase=ptr(self.phase, True),
                               samples_done=ptr(self.samples_done, True))

    def reset(self, idx, seeds):
        """Slots ``idx`` (device long tensor) start new utterances with ``seeds`` (device int64, same length)."""
        self.seeds.index_copy_(0, idx, seeds)
        self.phase.index_fill_(0, idx, 0.0)
        self.samples_done.index_fill_(0, idx, 0)


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
        if out_channels > 1 and nsf_params is not None:
            raise NotImplementedError("kantts_b200: a multi-band (PQMF) NSF generator is out of scope")
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

    def forward_rows(self, x, excitation=None, lengths=None):
        """``lengths`` (device int32 (B,), see ``forward``): every conv reads item b's input rows at or past lengths[b] times
        the input's rows per frame as zeros, and the output rows past lengths[b] * hop are zeroed.  The element-wise steps
        (SinAddFn, Mean3Fn, the fused residual adds) run unmasked: only a masked conv reads their rows past an item's end."""
        mask = (lambda rate: None) if lengths is None else (lambda rate: ops.utterance_mask(lengths, rate))
        rate = 1                                                             # x's rows per mel frame
        x = self.conv_pre.forward_rows(x, mask=mask(rate))
        hop = int(np.prod(self.upsample_scales))
        for i in range(self.num_upsamples):
            x = ops.SinAddFn.apply(x)                                        # hifigan.py:157
            m = mask(rate)
            rep = self.repeat_upsamples[i][2].forward_rows(x, mask=m)        # :158
            if excitation is not None:                                       # :162-166  x = rep + e + up (adds fused)
                rep = self.source_downs[i].forward_rows(excitation, resid=rep, mask=mask(hop))
            x = self.transpose_upsamples[i][1].forward_rows(x, resid=rep, mask=m)    # :160,168 (crop fused: t_out)
            rate *= int(self.upsample_scales[i])
            m = mask(rate)
            par = x.is_cuda and _PARALLEL_STREAMS and self.num_kernels > 1
            if par:                                                           # the parallel resblocks are independent
                cur = torch.cuda.current_stream()
                streams = _side_streams(x.device, self.num_kernels)
                rs = []
                for j in range(self.num_kernels):
                    streams[j].wait_stream(cur)
                    with torch.cuda.stream(streams[j]):
                        rs.append(self.conv_blocks[i * self.num_kernels + j].forward_rows(x, m))
                for s in streams[: self.num_kernels]:
                    cur.wait_stream(s)
            else:
                rs = [self.conv_blocks[i * self.num_kernels + j].forward_rows(x, m) for j in range(self.num_kernels)]
            rs += [None] * (3 - len(rs))
            x = ops.Mean3Fn.apply(1.0 / self.num_kernels, *rs)               # :170-176
        y = self.conv_post.forward_rows(x, mask=mask(hop))                   # :178-180
        return y if lengths is None else ops.rows_mask(y, mask(hop))

    def forward(self, x, nsf_seeds=None, lengths=None):
        """x: (B, in_channels, T) -> (B, out_channels, T * prod(scales)); with ``nsf_params`` the last two channels are the
        pitch (Hz) and the voiced flag (hifigan.py:146-150).  ``nsf_seeds`` (NSF only; one per batch item, host sequence
        or device int64 tensor): the excitation is the seeded kt_nsf_excitation instead of the reference's random draw, so
        that the output is a function of (x, seeds) -- the one a streamer with the same seeds computes.
        ``lengths`` (inference only: eval() mode, no autograd): each item's mel frames, a host sequence or a device int
        tensor (B,), 1 <= lengths[b] <= T (a device tensor's values are not read on the host).  Item b's output samples
        [0, lengths[b] * prod(scales)) are then ``self(x[b:b+1, :, :lengths[b]])`` (an NSF generator needs ``nsf_seeds``:
        the same seed) and its later samples are zero."""
        if nsf_seeds is not None and not self.nsf_enable:
            raise ValueError("nsf_seeds: this generator has no NSF source module")
        if lengths is not None:
            if self.training:
                raise RuntimeError("Generator.forward(lengths=...) is inference only: call eval() first")
            if self.nsf_enable and nsf_seeds is None:
                raise ValueError("Generator.forward(lengths=...): an NSF generator needs nsf_seeds for each item's excitation "
                                 "to be its own")
            lengths = ops.ragged_lengths(lengths, x.shape[0], x.shape[2], x.device)
        excitation = None
        if self.nsf_enable:
            x, pitch, uv = x[:, :-2, :], x[:, -2:-1, :], x[:, -1:, :]
            excitation = self.source_module.forward_rows(pitch, uv, nsf_seeds)   # (B, samples, 1)
        y = self.forward_rows(x.transpose(1, 2).contiguous(), excitation, lengths)   # (B, T', 1)
        return y.transpose(1, 2)

    def streamer(self, batch, max_frames, lengths=None, seeds=None):
        """-> a GeneratorStreamer that synthesises ``batch`` independent utterances chunk by chunk (at most ``max_frames``
        mel frames per chunk), giving the waveform of this (eval-mode) generator's forward.  A non-causal generator
        needs each slot's utterance ``lengths`` in frames (host list or device tensor (batch,)); a causal one takes none,
        unless it is multi-band: its attached PQMF's synthesis reads ahead, so that it needs them too.
        An NSF generator needs each slot's excitation ``seeds`` (as ``forward``'s ``nsf_seeds``); others take none."""
        return GeneratorStreamer(self, batch, max_frames, lengths, seeds)

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
# Streaming inference of the generator
# --------------------------------------------------------------------------------------------


def stream_history(spec):
    """Input rows before a chunk that one causal-form layer reads: its left padding for a conv -- (k-1)*d, or less for a
    strided one (stream_spec) -- ceil((k-1)*d / s) for the conv over the nearest-upsampled (by s) input, floor((k-1) / s)
    for the cropped transposed conv with stride s (1 when k = 2s)."""
    if spec.transposed:
        return (spec.kernel - 1) // spec.stride
    return -(-spec.pad_left // spec.upsample)


def stream_spec(spec, in_lag=0):
    """-> the causal form of a non-causal layer whose input trails by ``in_lag`` rows: a conv with all of its padding on
    the left, a transposed conv without padding and cropped by k - s at the end.  It computes the layer's output
    ``stream_lag(spec, in_lag)`` rows late.  A conv with stride s reads, for output t of the chunk, input rows
    t*s + j*d - P: with the lag L of stream_lag, P = L*s + pad_left - in_lag lines those rows up with the non-causal layer's
    (P = (k-1)*d for s = 1), and P + pad_right = (k-1)*d keeps a chunk of n*s input rows at n output rows."""
    if spec.transposed:
        return replace(spec, pad_left=0, crop=max(spec.kernel - spec.stride, 0))
    reach = (spec.kernel - 1) * spec.dilation
    left = stream_lag(spec, in_lag) * spec.stride + spec.pad_left - in_lag * spec.upsample
    assert left >= 0, (spec, in_lag)
    return replace(spec, pad_left=left, pad_right=reach - left)


def stream_lag(spec, in_lag=0):
    """Output rows by which the causal form of a non-causal layer trails its non-causal output when the input trails by
    ``in_lag`` rows.  A transposed conv: in_lag*s + its padding p (its output t reads inputs up to (t + p) / s).  A conv with
    stride s over the input up-sampled by u (s = 1 or u = 1): the input lag in its rows, L_in = in_lag*u, plus the right
    reach (k-1)*d - pad_left, in whole output rows -- the last output of a chunk may read at most its last input row:
    ceil((L_in + (k-1)*d - pad_left - (s-1)) / s), and not below 0.  For s = 1 that is L_in + (k-1)*d - pad_left; for the
    NSF source convs (k = 2s, pad_left = s // 2) from an input of lag 0 it is 1."""
    if spec.transposed:
        return in_lag * spec.stride + spec.pad_left
    assert spec.stride == 1 or spec.upsample == 1, spec
    s = spec.stride
    return max(0, -(-(in_lag * spec.upsample + (spec.kernel - 1) * spec.dilation - spec.pad_left - (s - 1)) // s))


# The steps of a StreamPlan, over windows named by the plan: a conv of ``conv`` (a layer's conv1d or deconv), run as ``spec``
# (the layer's spec, or its causal form), adding the rows of window ``resid`` (or None) that lie ``res_lag`` rows before the
# chunk, on side stream ``side`` of the parallel ResBlocks (None: the current stream); sin(x) + x; a mean of sources read
# ``offsets`` rows before the chunk.
ConvStep = namedtuple("ConvStep", "conv src dst resid side spec res_lag")
SinStep = namedtuple("SinStep", "src dst")
MeanStep = namedtuple("MeanStep", "srcs dst scale offsets")
# the seeded NSF excitation (kt_nsf_excitation) of the chunk's f0 / uv rows in window src into window dst
ExciteStep = namedtuple("ExciteStep", "src dst")


class FixedConv:
    """A conv with fixed weights and no bias that is not a layer of the generator: the PQMF synthesis of a multi-band
    generator (PQMF._weights()), as a ConvStep runs it."""

    def __init__(self, spec, weight):
        self.spec, self.weight, self.bias = spec, weight, None

    def effective_weight(self):
        return self.weight, None


class StreamPlan:
    """What a GeneratorStreamer runs per chunk, as data (no device needed):
      windows             one entry per tensor of the chunk: {name, channels, rows_per_frame, history}; a tensor read by a
                          conv keeps the largest history its consumers need, a residual or a mean source read n rows back
                          keeps n, the others keep none
      layer_history       {layer name (as in named_modules): input rows before the chunk it reads}
      lags                {window name: rows by which its newest row trails the newest pushed mel row}: all 0 for a causal
                          generator.  A non-causal one runs every layer in its causal form (stream_spec), whose output
                          trails the input's lag (times the layer's rate) by stream_lag rows
      delay               the waveform's lag in samples: a chunk returns the samples ``delay`` before the pushed frames' own
      causal              whether the generator is causal
      hop                 waveform samples per mel frame: prod(upsample_scales), times S for a multi-band generator
      launches_per_chunk  library calls of a full chunk: one per conv (one kernel each on the tensor-core path), one per
                          sin-add and per mean, one window advance and, with a delay, one output mask; NSF adds the
                          excitation, its 1x1 ffn conv, one source conv per stage and, where the stage sum cannot be chained
                          in the forward's order, one three-way add per stage; the mel chunk's copy into its window is not
                          counted
      nsf                 whether the generator has the NSF source: the last two input channels (f0, uv) go to window
                          "f0uv", the excitation (kt_nsf_excitation, seeded per slot) to "exc" and its ffn to "source" (rate
                          hop); stage i adds source_downs[i] of "source", in the forward's order up + (e + rep)
      pqmf                the PQMF of a multi-band generator (``out_channels`` = S > 1, attached as ``generator.pqmf`` with
                          ``subbands`` = S), else None.  conv_post writes the S sub-bands to window "sub"
                          (prod(upsample_scales) rows per frame), and one more ConvStep (layer "pqmf") runs the causal form
                          of the synthesis (stream_spec of PQMF.synthesis_spec, weight PQMF._weights()[1]) into "wav".  The
                          synthesis reads taps / 2 samples ahead, so that even a causal multi-band generator streams with a
                          delay: lag("sub") * S + taps / 2 samples, 31 for the default 62 taps
      steps               ConvStep | SinStep | MeanStep | ExciteStep records, in launch order"""

    def __init__(self, gen):
        pqmf = None
        if gen.out_channels > 1:
            pqmf = getattr(gen, "pqmf", None)
            if pqmf is None or pqmf.subbands != gen.out_channels:
                raise ValueError(f"streaming a multi-band (PQMF) generator of {gen.out_channels} sub-bands needs its PQMF "
                                 f"attached as generator.pqmf with as many sub-bands (got "
                                 f"{'none' if pqmf is None else pqmf.subbands}), as synthesize() does")
        if gen.training:
            raise ValueError("streaming runs a generator in eval() mode")
        self.causal = causal = gen.conv_pre.causal
        self.nsf = nsf = gen.nsf_enable
        self.pqmf = pqmf
        synth = None if pqmf is None else FixedConv(pqmf.synthesis_spec, pqmf._weights()[1])
        names = {m: n for n, m in gen.named_modules()}
        if synth is not None:
            names[synth] = "pqmf"
        table = WindowTable()
        self.windows, self.layer_history, self.steps, self.lags = table.windows, {}, [], {}

        def add(name, channels, rate=1):
            self.lags[name] = 0
            return table.add(name, channels, rate)

        def padded(nc):
            """Whether layer nc reads ahead of its output and runs in causal form: every layer of a non-causal generator,
            and the PQMF synthesis"""
            return not causal or nc is synth

        def layer(mod, src):
            nc = mod.conv1d if hasattr(mod, "conv1d") else getattr(mod, "deconv", mod)     # (the NSF ffn is the conv itself)
            return nc, stream_spec(nc.spec, self.lags[src]) if padded(nc) else nc.spec

        def lag_of(mod, src):
            """The lag of mod's output when it reads window src."""
            nc, _ = layer(mod, src)
            return stream_lag(nc.spec, self.lags[src]) if padded(nc) else 0

        def conv(mod, src, dst, resid=None, side=None):
            nc, spec = layer(mod, src)
            h = stream_history(spec)
            self.layer_history[names[mod]] = h
            table.read(src, h)
            self.lags[dst] = lag_of(mod, src)
            res_lag = 0 if resid is None else self.lags[dst] - self.lags[resid]
            if resid is not None:
                assert res_lag >= 0
                table.read(resid, res_lag)
            self.steps.append(ConvStep(nc, src, dst, resid, side, spec, res_lag))

        def mean(srcs, dst, scale):
            """dst = scale * (srcs summed in order), read at dst's lag, the latest of theirs: every source keeps the same
            history, so that they share one pitch"""
            self.lags[dst] = max(self.lags[o] for o in srcs)
            offsets = [self.lags[dst] - self.lags[o] for o in srcs]
            for o in srcs:
                table.read(o, max(offsets))
            self.steps.append(MeanStep(srcs, dst, scale, offsets))

        nk, ch, rate = gen.num_kernels, gen.conv_pre.conv1d.spec.c_out, 1
        hop = int(np.prod(gen.upsample_scales))
        mel = add("mel", gen.conv_pre.conv1d.spec.c_in)
        if nsf:
            sm = gen.source_module
            f0uv, exc = add("f0uv", 2), add("exc", sm.nb_harmonics + 1, hop)
            self.steps.append(ExciteStep(f0uv, exc))
            source = add("source", 1, hop)
            conv(sm.ffn[0], exc, source)
        x = add("x", ch)
        conv(gen.conv_pre, mel, x)
        for i in range(gen.num_upsamples):
            cin, s = ch >> i, gen.upsample_scales[i]
            cout = cin // 2
            sx = add(f"sin{i}", cin, rate)
            self.lags[sx] = self.lags[x]
            self.steps.append(SinStep(x, sx))
            rate *= s
            repm, upm = gen.repeat_upsamples[i][2], gen.transpose_upsamples[i][1]
            rep = add(f"rep{i}", cout, rate)
            up = add(f"up{i}", cout, rate)
            if nsf:
                # up + (e + rep), e = source_downs[i] of the source: the forward's order, kept bit for bit.  When the deconv
                # trails the other two, it is last and adds e + rep, itself formed by the later of the two (float addition
                # commutes); otherwise one three-way add (e + rep) + up at the latest lag
                dm = gen.source_downs[i]
                spec = dm.conv1d.spec
                assert spec.t_out(7 * spec.stride) == 7, f"source_downs[{i}]: {spec} does not bring the source to the stage rate"
                e = add(f"e{i}", cout, rate)
                l_rep, l_up, l_e = lag_of(repm, sx), lag_of(upm, sx), lag_of(dm, source)
                if l_up >= max(l_rep, l_e):
                    first, second = ((repm, sx, rep), (dm, source, e)) if l_e >= l_rep else ((dm, source, e), (repm, sx, rep))
                    conv(*first)
                    conv(*second, resid=first[2])
                    conv(upm, sx, up, resid=second[2])
                    xin0 = up
                else:
                    conv(repm, sx, rep)
                    conv(dm, source, e)
                    conv(upm, sx, up)
                    xin0 = add(f"sum{i}", cout, rate)
                    mean([e, rep, up], xin0, 1.0)
            # up + rep: the later of the two adds the other, read as many rows back as it trails (the deconv, unless its
            # padding is the smaller right reach: k = 4, s = 2 against the k = 7 repeat conv)
            elif lag_of(upm, sx) >= lag_of(repm, sx):
                conv(repm, sx, rep)
                conv(upm, sx, up, resid=rep)
                xin0 = up
            else:
                conv(upm, sx, up)
                conv(repm, sx, rep, resid=up)
                xin0 = rep
            outs = []
            for j in range(nk):
                rb, xin = gen.conv_blocks[i * nk + j], xin0
                side = j if nk > 1 else None
                for p, (c1, c2) in enumerate(zip(rb.convs1, rb.convs2)):
                    h = add(f"rb{i}.{j}.h{p}", cout, rate)
                    conv(c1, xin, h, side=side)
                    xo = add(f"rb{i}.{j}.x{p + 1}", cout, rate)
                    conv(c2, h, xo, resid=xin, side=side)
                    xin = xo
                outs.append(xin)
            # the parallel ResBlocks trail their input by different right reaches: each is read at the mean's lag
            x = add(f"mean{i}", cout, rate)
            mean(outs, x, 1.0 / nk)
        assert rate == hop
        if synth is None:
            conv(gen.conv_post, x, add("wav", 1, rate))
        else:
            sub = add("sub", gen.out_channels, rate)
            conv(gen.conv_post, x, sub)
            rate *= gen.out_channels
            conv(synth, sub, add("wav", 1, rate))
        hist = {w["name"]: w["history"] for w in self.windows}
        for st in self.steps:                  # kt_add3_scale_win reads its sources at one pitch
            assert type(st) is not MeanStep or len({hist[o] for o in st.srcs}) == 1, st
        self.hop = rate
        self.delay = self.lags["wav"]
        self.launches_per_chunk = table.launches_per_chunk(len(self.steps)) + (self.delay > 0)


class GeneratorStreamer(Streamer):
    """Chunk-by-chunk synthesis with a HiFi-GAN generator (Generator.streamer).

    ``push(mel)`` takes the next (B, in_channels, f) mel frames of every batch slot (1 <= f <= max_frames, on the
    generator's GPU) and returns (B, 1, f * hop) waveform samples.  Each batch slot is an independent stream; ``reset(slots)``
    starts new utterances in the given slots.  ``push`` never waits for the device.

    Causal generator: concatenated, the outputs of any split of a mel equal the generator's forward on the whole mel.

    Non-causal generator: a sample depends on mel frames after its own, so the output is delayed.  With p_b the samples of
    the frames pushed to slot b since its reset, a push returns the samples [p_b - delay, p_b - delay + f * hop) of the
    slot's utterance, of ``lengths[b]`` frames; positions outside [0, lengths[b] * hop) are 0, and frames pushed past
    lengths[b] are ignored.  ``finish()`` pushes the ``drain_frames`` frames that bring out an utterance's last sample.
    The chunks of slot b concatenated and cut to [delay, delay + lengths[b] * hop) equal the forward on the slot's mel of
    exactly lengths[b] frames: every layer's zero padding at the utterance's end is applied per slot inside the conv
    kernels (the stream conv's KtStreamMask), from the slots' utterance record (stream.SlotUtterances).  A slot reset
    before its utterance has drained loses the samples not yet returned.

    Multi-band generator (``out_channels`` = S > 1 with its PQMF attached as ``generator.pqmf``): the last stream stage is
    the PQMF synthesis, run in causal form over the S sub-bands, and a push returns the waveform (B, 1, f * hop) with hop =
    prod(upsample_scales) * S.  The synthesis reads taps / 2 samples ahead, so that the stream is delayed as above even for
    a causal generator (delay 31 samples for the default 62 taps, one drain frame), and needs ``lengths``: each slot's
    sub-bands are masked at its utterance end (lengths[b] * hop / S rows), the synthesis's zero padding.  Slot b's chunks,
    cut the same way, equal ``pqmf.synthesis(generator(mel_b[..., :lengths[b]]))``.

    NSF generator: ``push`` takes (B, in_channels + 2, f) -- mel, f0 in Hz and the voiced flag, as ``forward`` -- and each
    slot's excitation is seeded by its ``seeds`` entry (``reset`` takes the new slots' seeds).  The excitation is computed
    per chunk on the device, its phases and sample count carried per slot, so the output equals ``forward(x, nsf_seeds)``
    of the slot's whole utterance with that seed.

    Every tensor a layer reads lives in a window (stream.py) that its producer writes straight into.  A full-size chunk
    replays a CUDA graph; a shorter chunk runs the same kernels eagerly.

    The weights are prepared once, when the streamer is created: a generator whose parameters change later needs a new
    streamer.  Creating one also runs a chunk of zeros through every kernel, so that every kernel is loaded, captures the
    full-size chunk's graph, then clears the state; the capture synchronises the device once."""

    out, f_axis = "wav", 2

    def __init__(self, gen, batch, max_frames, lengths=None, seeds=None):
        plan = StreamPlan(gen)
        self._check_utterances(plan, int(batch), lengths, seeds)         # before any device work
        self.hop, self.in_channels = plan.hop, plan.windows[0]["channels"] + (2 if plan.nsf else 0)
        super().__init__(plan, batch, max_frames, next(gen.parameters()).device, "streamer", masked=plan.delay > 0,
                         in_channels=self.in_channels)
        self._source = gen.source_module if plan.nsf else None
        self._side = [torch.cuda.Stream(device=self.device) for _ in range(gen.num_kernels)] if gen.num_kernels > 1 else []
        with torch.no_grad(), torch.cuda.device(self.device):
            self._weights = {st.conv: self._own_weight(st) for st in plan.steps if type(st) is ConvStep}
            self._nsf = NsfState(self._source, torch.zeros(self.batch, dtype=torch.int64, device=self.device)) \
                if plan.nsf else None
            self._run(self.max_frames)               # warm-up: every kernel and weight image of a full chunk
            self._graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self._graph):
                self._run(self.max_frames)
            self.reset(range(self.batch), lengths, seeds)

    @staticmethod
    def _check_utterances(plan, n, lengths, seeds):
        """-> ``seeds`` as an int64 tensor (n,) where they are (None without NSF), after checking that ``lengths`` are given
        exactly when the stream has a delay and ``seeds`` exactly when the generator is NSF; ValueError otherwise."""
        if plan.nsf and seeds is None:
            raise ValueError("streaming an NSF generator needs per-slot seeds: its excitation is a seeded function of the "
                             "sample index, so that chunks reproduce the whole-utterance forward(x, nsf_seeds)")
        if not plan.nsf and seeds is not None:
            raise ValueError("streamer: seeds are for NSF generators; this one has no NSF source module")
        if not plan.delay and lengths is not None:
            raise ValueError("a causal generator streams without lengths: its output does not depend on where an utterance "
                             "ends")
        if plan.delay and lengths is None:
            raise ValueError(f"streaming a {'multi-band' if plan.causal else 'non-causal'} generator needs per-slot lengths: "
                             f"it reads {plan.delay} samples ahead, so that its output near an utterance's end depends on "
                             "where that end is")
        return None if seeds is None else nsf_seed_tensor(seeds, n, seeds.device if torch.is_tensor(seeds) else "cpu")

    def _own_weight(self, st):
        """The streamer's copy of ConvStep st's weights, on its device (the PQMF synthesis weight lives wherever the PQMF's
        buffers are)."""
        v, g = st.conv.effective_weight()
        return own_weight(st.spec, v.to(self.device), g, st.conv.bias)

    def _run(self, f):
        """Every launch of one chunk of f frames (the mel chunk is in its window), on the current stream."""
        win, masks = self._win, self._masks
        b, B = win.buf, self.batch
        cur = torch.cuda.current_stream()
        forked = False
        for st, place in zip(self.plan.steps, self._places):
            side = st.side if type(st) is ConvStep else None
            if (side is not None) != forked:               # fork the side streams off the current one, or join them
                forked = side is not None
                for s in self._side:
                    s.wait_stream(cur) if forked else cur.wait_stream(s)
            if type(st) is ConvStep:
                pw, bias = self._weights[st.conv]
                with torch.cuda.stream(self._side[side] if side is not None else cur):
                    ops.stream_conv(st.spec, pw, bias, b[st.src], b[st.dst], f * win.rate[st.src], place,
                                    None if st.resid is None else b[st.resid], None if masks is None else masks[st.src])
            elif type(st) is ExciteStep:
                self._source.run_excitation(b[st.src], win.first[st.src], self._nsf, b[st.dst], win.first[st.dst], f)
            elif type(st) is SinStep:
                src, dst = b[st.src], b[st.dst]
                ops.call("kt_sinadd_fwd_win", ptr(src), ptr(dst), B, f * win.rate[st.src], src.shape[2], src.shape[1],
                         dst.shape[1], win.first[st.dst])
            else:
                dst, ch = b[st.dst], b[st.dst].shape[2]
                # source j's chunk starts `offsets[j]` rows before its own chunk row 0 (4-byte rows of ch floats)
                srcs = [ptr(b[s]) + (win.first[s] - o) * ch * 4 for s, o in zip(st.srcs, st.offsets)] + [None] * (3 - len(st.srcs))
                ops.call("kt_add3_scale_win", srcs[0], srcs[1], srcs[2], st.scale, ptr(dst), B, f * win.rate[st.dst], ch,
                         b[st.srcs[0]].shape[1], dst.shape[1], win.first[st.dst])
        self._end_chunk(f)

    def push(self, mel):
        """mel: (B, in_channels, f), 1 <= f <= max_frames, on the streamer's device -> the (B, 1, f * hop) waveform.  NSF:
        the last two of the in_channels are f0 (Hz) and the voiced flag."""
        with torch.no_grad(), torch.cuda.device(self.device):
            if self.plan.nsf:
                if mel.dim() != 3 or mel.shape[1] != self.in_channels:
                    raise ValueError(f"push: expected a (B, {self.in_channels}, f) chunk of mel + f0 + uv, got {tuple(mel.shape)}")
                f = self._win.push("mel", mel[:, :-2], 2, ("a {} mel", "frames", "the mel is"))
                self._win.push("f0uv", mel[:, -2:], 2, ("a {} f0 / uv", "frames", "the f0 / uv is"))
            else:
                f = self._win.push("mel", mel, 2, ("a {} mel", "frames", "the mel is"))
            if f == self.max_frames:
                self._graph.replay()
            else:
                self._run(f)
            return self._output(f)

    def reset(self, slots, lengths=None, seeds=None):
        """The given batch slots start a new utterance: their carried state returns to zeros (one launch).  A generator
        streamed with a delay (non-causal or multi-band) needs the new utterances' ``lengths`` in frames, an NSF one their
        excitation ``seeds``, both in the order of ``slots``.  All of it is checked before the first launch: a rejected
        reset leaves every slot as it was."""
        slots = check_slots(slots, self.batch)
        seeds = self._check_utterances(self.plan, len(slots), lengths, seeds)
        with torch.no_grad(), torch.cuda.device(self.device):
            if lengths is not None:                 # checks the lengths before its first launch
                self._slots.reset(slots, lengths)
            self._win.reset(slots)
            if seeds is not None:                   # excitation phases and sample counts return to zero
                self._nsf.reset(to_device(torch.tensor(slots, dtype=torch.long), self.device), seeds.to(self.device))


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
        return _split_runs(outs, fmaps, nb, detach_b)

    def _run(self, y, pair_nb):
        rows = y.transpose(1, 2).contiguous()                                 # (B, T, 1)
        inputs = [rows]
        for i in range(1, len(self.discriminators)):                          # the pooling chain is cheap and serial
            if self.aux_convs is None:                                        # nn.AvgPool1d variant (hifigan.py:456-458,466)
                rows = self.meanpools[i - 1].run(rows)
            else:
                cat = ops.DwtFn.apply(rows.reshape(rows.shape[0], -1))        # (B, T2, 2) = cat([yl, yh], 1)
                rows = self.aux_convs[i - 1].run(cat)                          # (B, T2, 1), lrelu fused
            inputs.append(rows)

        def run_scale(d, x):
            if pair_nb is not None and _spectral(d):
                return _run_halves(d.forward_rows, x, pair_nb)
            return d.forward_rows(x)

        # the scales themselves are independent
        return _run_parallel(y, [(lambda d=d, x=x: run_scale(d, x), not _spectral(d))
                                 for d, x in zip(self.discriminators, inputs)])


# --------------------------------------------------------------------------------------------
# MultiSpecDiscriminator (hifigan.py:481-617)
# --------------------------------------------------------------------------------------------


class _SpecConv(_NormedConv):
    """``norm_f(nn.Conv2d(cin, cout, (k, 1), (stride, 1), padding))`` of the spectrogram discriminator, computed as a Conv1d
    over frames on channels-last rows.  ``pad_width``: the zero columns the layer adds on each side of the frequency axis
    (the reference passes ``padding=(k-1)//2`` as an int, which pads that width-1 axis too; conv_post pads frames only)."""

    def __init__(self, cin, cout, k, stride, pad_width, norm, act_out_slope=None):
        pad = (k - 1) // 2
        ref = nn.Conv2d(cin, cout, (k, 1), (stride, 1), padding=(pad, pad_width))
        spec = ops.ConvSpec(c_in=cin, c_out=cout, kernel=k, stride=stride, pad_left=pad, pad_right=pad)
        if act_out_slope is not None:
            spec.act_out, spec.act_out_slope = KT_ACT_LRELU, float(act_out_slope)
        super().__init__(ref, spec, norm)
        self.pad_width = pad_width


class SpecDiscriminator(nn.Module):
    """One resolution of the multi-resolution spectrogram discriminator (hifigan.py:481-582).  ``forward(wav)`` takes the
    magnitude spectrogram without gradient (the generator learns nothing from this discriminator; only its own weights do)
    and runs the (k, 1) convs over frames with F = fft_size//2+1 input channels.

    Every conv also pads the width-1 frequency axis, so the maps grow by 2p columns per layer.  All columns born as zeros
    at one layer (a "column class") hold the same sequence for every item: the module computes each class once, as one
    extra batch item after the signal items (a zero item appended to the layer's input becomes lrelu(bias) at its birth),
    and kt_spec_columns_fwd expands the rows into the reference's maps, returned as (B, C, frames, width) views of
    channels-last (B, frames, width, C) buffers."""

    def __init__(self, channels=32, init_kernel=15, kernel_size=11, stride=2, use_spectral_norm=False, fft_size=1024,
                 shift_size=120, win_length=600, window="hann_window", nonlinear_activation="LeakyReLU",
                 nonlinear_activation_params={"negative_slope": 0.1}):
        super().__init__()
        if nonlinear_activation != "LeakyReLU":
            raise NotImplementedError("kantts_b200: only LeakyReLU is fused into the conv kernels")
        slope = nonlinear_activation_params.get("negative_slope", 0.01)
        self.fft_size, self.shift_size, self.win_length = fft_size, shift_size, win_length
        norm = "spectral" if use_spectral_norm else "weight"
        act = lambda: getattr(nn, nonlinear_activation)(**nonlinear_activation_params)  # noqa: E731
        layers = [(fft_size // 2 + 1, init_kernel, 1)] + [(channels, kernel_size, stride)] * 3 + [(channels, 5, 1)]
        self.convs = nn.ModuleList(
            nn.Sequential(_SpecConv(cin, channels, k, s, (k - 1) // 2, norm, slope), act()) for cin, k, s in layers)
        self.conv_post = _SpecConv(channels, 1, 3, 1, 0, norm)
        self.register_buffer("window", getattr(torch, window)(win_length))

    def magnitude(self, wav):
        """(B, 1, T) -> the magnitude rows (B, frames, F) of audio_torch.stft, without gradient (hifigan.py:566-571)."""
        with torch.no_grad():
            return stft(torch.squeeze(wav, 1), self.fft_size, self.shift_size, self.win_length, self.window)

    def forward_rows(self, mag):
        """mag (B, frames, F) -> (output (B, 1, frames', width), [six (B, C, frames_l, width_l) feature maps])"""
        n = mag.shape[0]
        x, reach, fmap = mag, [], []
        for conv in [l[0] for l in self.convs] + [self.conv_post]:
            if conv.pad_width:
                # the columns this layer pads in: their input is zeros at every frame
                x = torch.cat([x, x.new_zeros((1,) + tuple(x.shape[1:]))])
                reach.append((reach[-1] if reach else 0) + conv.pad_width)
            x = conv.run(x)
            fmap.append(ops.SpecColumnsFn.apply(x, n, tuple(reach)).permute(0, 3, 1, 2))
        return fmap[-1].squeeze(-1), fmap

    def forward(self, wav):
        return self.forward_rows(self.magnitude(wav))


class MultiSpecDiscriminator(nn.Module):
    """hifigan.py:585-617: one SpecDiscriminator per (fft size, hop, window length).  The default ``discriminator_params``
    are the reference's, whose ``kernel_sizes`` key SpecDiscriminator does not take: like the reference,
    ``MultiSpecDiscriminator()`` raises TypeError, and a usable config passes ``kernel_size``."""

    def __init__(self, fft_sizes=[1024, 2048, 512], hop_sizes=[120, 240, 50], win_lengths=[600, 1200, 240],
                 discriminator_params={
                     "channels": 15, "init_kernel": 1, "kernel_sizes": 11, "stride": 2, "use_spectral_norm": False,
                     "window": "hann_window", "nonlinear_activation": "LeakyReLU",
                     "nonlinear_activation_params": {"negative_slope": 0.1}}):
        super().__init__()
        self.discriminators = nn.ModuleList()
        for fft_size, hop_size, win_length in zip(fft_sizes, hop_sizes, win_lengths):
            params = copy.deepcopy(discriminator_params)
            params["fft_size"] = fft_size
            params["shift_size"] = hop_size
            params["win_length"] = win_length
            self.discriminators += [SpecDiscriminator(**params)]

    def forward(self, y):
        """y: (B, 1, T) -> (list of (B, 1, frames, width), list of lists of (B, C, frames_l, width_l) feature maps)"""
        return self._run(y, None)

    def forward_pair(self, ya, yb, detach_b=False):
        """== (self(ya), self(yb)) evaluated as one batch of 2B (see MultiPeriodDiscriminator.forward_pair): the column
        classes follow the 2B signal items, so ops.grad_items(B) keeps them out of the gradient of a generator-phase pair
        (nothing there needs it), and pair_state("reuse") reuses them with the real half.  A spectral-normed resolution
        runs per half in the reference's order, as in MultiScaleDiscriminator.forward_pair."""
        assert ya.shape == yb.shape
        nb = ya.shape[0]
        outs, fmaps = self._run(torch.cat([ya, yb], 0), nb)
        return _split_runs(outs, fmaps, nb, detach_b)

    def _run(self, y, pair_nb):
        def run_resolution(d):
            mag = d.magnitude(y)
            if pair_nb is not None and _spectral(d):
                return _run_halves(d.forward_rows, mag, pair_nb)
            return d.forward_rows(mag)

        return _run_parallel(y, [(lambda d=d: run_resolution(d), not _spectral(d)) for d in self.discriminators])
