"""``kantts.train.loss`` surface for the HiFi-GAN path (KAN-TTS kantts/train/loss.py:108-441,
512-544): same class names / kwargs / return values, so ``criterion_builder`` works unchanged.

The mel / STFT spectra come from the fused kernel (audio.py); the scalar reductions over the
(tiny) discriminator outputs and spectra stay torch ops (a few KB each).  The feature-matching
loss is value-only in the reference (its second argument is detached and the trainer passes the
generator's feature maps there, trainer.py:535-538) and uses the streaming kt_l1_sum kernel.
"""
import torch
import torch.nn.functional as F

from . import ops
from .audio import MelSpectrogram, stft
from .sambert import AttentionBinarizationLoss, AttentionCTCLoss, FpCELoss, SeqCELoss


def _as_list(outputs):
    """The trainer hands over one tensor per sub-discriminator (a list / tuple); a bare tensor counts as one."""
    return list(outputs) if isinstance(outputs, (tuple, list)) else [outputs]


def _last(o):
    """A sub-discriminator result may itself be a (feature maps ..., logits) sequence: the logits come last."""
    return o[-1] if isinstance(o, (tuple, list)) else o


def _gan_term(logits, target, loss_type):
    """One sub-discriminator's contribution.  mse: LSGAN distance to ``target`` (1 = real, 0 = fake);
    hinge: mean of min(sign * logits - 1, 0) negated, sign = +1 for the real side, -1 for the fake side."""
    if loss_type == "mse":
        return torch.mean((logits - target) ** 2)
    sign = 1.0 if target > 0.5 else -1.0
    return -torch.mean(torch.clamp(sign * logits - 1.0, max=0.0))


class _AdversarialBase(torch.nn.Module):
    def __init__(self, average_by_discriminators=True, loss_type="mse"):
        super().__init__()
        assert loss_type in ["mse", "hinge"], f"{loss_type} is not supported."
        self.average_by_discriminators = average_by_discriminators
        self.loss_type = loss_type

    def _reduce(self, terms):
        total = sum(terms[1:], terms[0])
        return total / len(terms) if self.average_by_discriminators and len(terms) > 1 else total

    _weights = {}

    def _mse_total(self, outs, target):
        """sum_i mean((o_i - target)^2) [/ n] as ONE chain over the concatenated logits: cat, sub, mul, dot (and their four
        backward kernels) instead of ~10 tiny launches per sub-discriminator -- the loss sits on the critical path between
        the discriminators' forward and backward passes.  Per-element weights 1 / numel_i are cached per shape set."""
        outs = [o.reshape(-1) for o in outs]
        if len(outs) == 1 or not outs[0].is_cuda:
            return self._reduce([torch.mean((o - target) ** 2) for o in outs])
        key = (tuple(o.numel() for o in outs), outs[0].device, bool(self.average_by_discriminators))
        w = self._weights.get(key)
        if w is None:
            scale = 1.0 / len(outs) if self.average_by_discriminators else 1.0
            w = torch.cat([torch.full((o.numel(),), scale / o.numel(), dtype=torch.float32) for o in outs]).to(outs[0].device)
            self._weights[key] = w
        d = torch.cat(outs) - target
        return torch.dot(d * w, d)


class GeneratorAdversarialLoss(_AdversarialBase):
    """kantts/train/loss.py:108-145: the generator wants every sub-discriminator to call its output real
    (mse: distance to 1; hinge: -mean(logits)); summed over the sub-discriminators, optionally averaged."""

    def forward(self, outputs):
        if self.loss_type == "mse":
            return self._mse_total(_as_list(outputs), 1.0)
        terms = [-torch.mean(o) for o in _as_list(outputs)]
        return self._reduce(terms)


class DiscriminatorAdversarialLoss(_AdversarialBase):
    """kantts/train/loss.py:148-214: (real_loss, fake_loss) -- real outputs pushed to 1, generated ones to 0
    (mse) or past the +-1 margins (hinge)."""

    def forward(self, outputs_hat, outputs):
        if self.loss_type == "mse":
            return (self._mse_total([_last(o) for o in _as_list(outputs)], 1.0),
                    self._mse_total([_last(o) for o in _as_list(outputs_hat)], 0.0))
        fake = [_gan_term(_last(o), 0.0, self.loss_type) for o in _as_list(outputs_hat)]
        real = [_gan_term(_last(o), 1.0, self.loss_type) for o in _as_list(outputs)]
        return self._reduce(real), self._reduce(fake)


def _l1_mean(a, b):
    """F.l1_loss(a, b.detach()) for two feature maps.  Channels-last views produced by this package
    share strides, so the permuted-back contiguous buffers are compared directly."""
    if a.requires_grad or not a.is_cuda:
        return F.l1_loss(a, b.detach())
    if a.dim() == 3 and not a.is_contiguous():
        a, b = a.transpose(1, 2), b.transpose(1, 2)
    elif a.dim() == 4 and not a.is_contiguous():
        a, b = a.permute(0, 2, 3, 1), b.permute(0, 2, 3, 1)
    if not (a.is_contiguous() and b.is_contiguous()):
        return F.l1_loss(a, b.detach())
    return ops.l1_sum(a.detach(), b.detach(), 1.0 / a.numel())


def _rows_pair(a, b):
    """-> the contiguous channels-last buffers behind two feature-map views of this package, or None."""
    if a.requires_grad or not a.is_cuda or a.shape != b.shape:
        return None
    if a.dim() == 3 and not a.is_contiguous():
        a, b = a.transpose(1, 2), b.transpose(1, 2)
    elif a.dim() == 4 and not a.is_contiguous():
        a, b = a.permute(0, 2, 3, 1), b.permute(0, 2, 3, 1)
    return (a.detach(), b.detach()) if a.is_contiguous() and b.is_contiguous() else None


class FeatureMatchLoss(torch.nn.Module):
    """kantts/train/loss.py:217-256: sum over sub-discriminators of the (summed or averaged) per-layer L1 distance
    between two feature-map pyramids; the second argument is treated as a constant."""

    def __init__(self, average_by_layers=True, average_by_discriminators=True):
        super().__init__()
        self.average_by_layers = average_by_layers
        self.average_by_discriminators = average_by_discriminators

    def forward(self, feats_hat, feats):
        fast = self._forward_accumulated(feats_hat, feats)
        if fast is not None:
            return fast
        per_disc = []
        for maps_hat, maps in zip(feats_hat, feats):
            layer_terms = [_l1_mean(a, b) for a, b in zip(maps_hat, maps)]
            value = sum(layer_terms[1:], layer_terms[0])
            per_disc.append(value / len(layer_terms) if self.average_by_layers else value)
        total = sum(per_disc[1:], per_disc[0])
        return total / len(per_disc) if self.average_by_discriminators else total


class MelSpectrogramLoss(torch.nn.Module):
    """kantts/train/loss.py:259-311: L1 between the normalised log-mel spectrograms (fused STFT-mel kernel)."""

    def __init__(self, fs=22050, fft_size=1024, hop_size=256, win_length=None, window="hann", num_mels=80,
                 fmin=80, fmax=7600, center=True, normalized=False, onesided=True, eps=1e-10, log_base=10.0):
        super().__init__()
        self.mel_spectrogram = MelSpectrogram(fs=fs, fft_size=fft_size, hop_size=hop_size, win_length=win_length,
                                              window=window, num_mels=num_mels, fmin=fmin, fmax=fmax,
                                              center=center, normalized=normalized, onesided=onesided, eps=eps,
                                              log_base=log_base)

    def forward(self, y_hat, y):
        return torch.mean(torch.abs(self.mel_spectrogram(y_hat) - self.mel_spectrogram(y)))


class SpectralConvergenceLoss(torch.nn.Module):
    """kantts/train/loss.py:314-331: || |Y| - |X| ||_F / || |Y| ||_F."""

    def forward(self, x_mag, y_mag):
        return torch.linalg.vector_norm(y_mag - x_mag) / torch.linalg.vector_norm(y_mag)


class LogSTFTMagnitudeLoss(torch.nn.Module):
    """kantts/train/loss.py:334-350: L1 between the log magnitudes."""

    def forward(self, x_mag, y_mag):
        return torch.mean(torch.abs(torch.log(y_mag) - torch.log(x_mag)))


class STFTLoss(torch.nn.Module):
    """kantts/train/loss.py:353-389: one resolution -> (spectral convergence, log-magnitude L1)."""

    def __init__(self, fft_size=1024, shift_size=120, win_length=600, window="hann_window"):
        super().__init__()
        self.fft_size, self.shift_size, self.win_length = fft_size, shift_size, win_length
        self.spectral_convergence_loss = SpectralConvergenceLoss()
        self.log_stft_magnitude_loss = LogSTFTMagnitudeLoss()
        self.register_buffer("window", getattr(torch, window)(win_length))

    def forward(self, x, y):
        mags = [stft(w, self.fft_size, self.shift_size, self.win_length, self.window) for w in (x, y)]
        return self.spectral_convergence_loss(*mags), self.log_stft_magnitude_loss(*mags)


class MultiResolutionSTFTLoss(torch.nn.Module):
    """kantts/train/loss.py:392-441: mean over the resolutions of both STFT loss terms; (B, bands, T) inputs
    (sub-band signals) are folded into the batch."""

    def __init__(self, fft_sizes=[1024, 2048, 512], hop_sizes=[120, 240, 50], win_lengths=[600, 1200, 240],
                 window="hann_window"):
        super().__init__()
        assert len(fft_sizes) == len(hop_sizes) == len(win_lengths)
        self.stft_losses = torch.nn.ModuleList(
            [STFTLoss(*cfg, window) for cfg in zip(fft_sizes, hop_sizes, win_lengths)])

    def forward(self, x, y):
        if x.dim() == 3:
            x, y = x.reshape(-1, x.size(2)), y.reshape(-1, y.size(2))
        terms = [f(x, y) for f in self.stft_losses]
        n = len(terms)
        return sum(t[0] for t in terms) / n, sum(t[1] for t in terms) / n


def _fm_forward_accumulated(self, feats_hat, feats):
    """Value-only pyramids (the trainer's use, see the module docstring): every layer's weighted L1 sum goes into ONE device
    accumulator -- one launch per feature map instead of memset + kernel + the add / divide chain of the generic path."""
    pairs, scales = [], []
    n_disc = len(feats_hat)
    for maps_hat, maps in zip(feats_hat, feats):
        for a, b in zip(maps_hat, maps):
            rp = _rows_pair(a, b)
            if rp is None:
                return None
            pairs.append(rp)
            s = 1.0 / rp[0].numel()
            if self.average_by_layers:
                s /= len(maps_hat)
            if self.average_by_discriminators:
                s /= n_disc
            scales.append(s)
    if not pairs:
        return None
    out = torch.zeros((), device=pairs[0][0].device, dtype=torch.float32)
    for (a, b), s in zip(pairs, scales):
        ops.l1_sum_acc(out, a, b, s)
    return out


FeatureMatchLoss._forward_accumulated = _fm_forward_accumulated

loss_dict = {
    "generator_adv_loss": GeneratorAdversarialLoss,
    "discriminator_adv_loss": DiscriminatorAdversarialLoss,
    "stft_loss": MultiResolutionSTFTLoss,
    "mel_loss": MelSpectrogramLoss,
    "subband_stft_loss": MultiResolutionSTFTLoss,
    "feat_match_loss": FeatureMatchLoss,
    "FpCELoss": FpCELoss,
    "AttentionCTCLoss": AttentionCTCLoss,
    "AttentionBinarizationLoss": AttentionBinarizationLoss,
    "SeqCELoss": SeqCELoss,
}


def criterion_builder(config, device="cpu"):
    """loss.py:528-544.  An enabled ``subband_stft_loss`` is also stored as ``"sub_stft"``, the key GAN_Trainer calls it
    by (trainer.py:495-498) while it checks for the other: the reference builder leaves that key out, so its trainer
    raises KeyError on the multi-band yamls."""
    criterion = {}
    for key, value in config["Loss"].items():
        if key in loss_dict:
            if value["enable"]:
                criterion[key] = loss_dict[key](**value.get("params", {})).to(device)
                setattr(criterion[key], "weights", value.get("weights", 1.0))
        else:
            raise NotImplementedError("{} is not implemented".format(key))
    if "subband_stft_loss" in criterion:
        criterion["sub_stft"] = criterion["subband_stft_loss"]
    return criterion
