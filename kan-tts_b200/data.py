"""GPU data path of the HiFi-GAN trainer (SURVEY.md 8f-2): ``Voc_Dataset.__getitem__`` length fix-up + ``collate_fn``
random crop / batching (kantts/datasets/dataset.py:225-311) and the OFFLINE mel features the reference reads from
``mel/*.npy`` (kantts/preprocess/audio_processor/core/dsp.py:165-201, mean/std normalisation of
audio_processor.py:363-382) -- here computed on the fly, on the device, for exactly the frames of each crop.

The reference keeps (wav, mel.npy) pairs on disk, crops both on the host in ``collate_fn`` and copies the batch over.
``GpuVocBatcher`` keeps the utterance waveforms resident in HBM (one padded 2-D tensor), draws the crop positions on
the host with numpy's global RNG in the reference's order (``np.random.randint(start_offset, length + end_offset)`` per
item: the same seed gives the same crops), gathers the waveform segments with one indexing kernel and computes the mel
frames of the crop (plus the ``aux_context_window`` frames on either side) with the fused STFT-mel kernel
(``kt_stft_mel_fwd``: framing, hann window, rFFT, magnitude, Slaney mel, dB, normalisation in one launch).  Nothing but
the start frames crosses PCIe per step, and the ``mel/*.npy`` feature format disappears.

A mel frame f of the offline features is centred at sample f * hop of the utterance, reflect-padded by n_fft / 2 at the
utterance ends (librosa.stft).  The crop's frames are therefore computed from the slice of the utterance-level PADDED
waveform that covers their windows, so a cropped-then-computed frame equals the computed-then-cropped frame of the
reference bit for bit in exact arithmetic (fp32 kernel vs float64 numpy: tests/test_gpu_data.py, mel-L1 <= 1e-4)."""
import numpy as np
import torch

from . import ops
from .audio import _padded_window, slaney_mel_filterbank


class GpuVocBatcher:
    def __init__(self, wavs, sampling_rate, hop_length, n_fft=1024, win_length=1024, n_mels=80, fmin=50, fmax=8000,
                 batch_max_steps=8192, aux_context_window=0, max_norm=1.0, min_level_db=-100, ref_level_db=20,
                 symmetric=False, preemphasize=False, mel_mean=None, mel_std=None, device="cuda"):
        """wavs: list of 1-D float arrays (already loaded / resampled / trimmed like librosa.load in __getitem__).
        The keyword names are those of the reference's ``audio_config`` + ``batch_max_steps`` / ``aux_context_window``."""
        if batch_max_steps % hop_length != 0:                      # dataset.py:77-79
            batch_max_steps += -(batch_max_steps % hop_length)
        self.hop, self.n_fft, self.win_length, self.n_mels = int(hop_length), int(n_fft), int(win_length), int(n_mels)
        self.batch_max_steps = int(batch_max_steps)
        self.batch_max_frames = self.batch_max_steps // self.hop
        self.aux = int(aux_context_window)
        self.start_offset = self.aux                               # dataset.py:84-85
        self.end_offset = -(self.batch_max_frames + self.aux)
        self.device = torch.device(device)
        self.preemphasize = bool(preemphasize)
        # frames of one crop: [start - aux, start + batch_max_frames + aux)
        self.n_frames = self.batch_max_frames + 2 * self.aux
        # window start = first frame centre - n_fft/2 - delta, delta making the first wanted frame an INTEGER frame index f0
        # of the slice (the fused kernel frames a signal at multiples of hop from its start, centred)
        half = self.n_fft // 2
        self.delta = (-half) % self.hop
        self.f0 = (half + self.delta) // self.hop
        self.win_samples = (self.n_frames - 1 + 2 * self.f0) * self.hop + 1     # slice length: frames f0 .. f0 + n - 1 are interior
        pad_l = half + self.delta                                   # reflect padding (n_fft / 2) + alignment zeros
        # ---- Voc_Dataset.__getitem__ length fix-up (dataset.py:248-270), then utterance-level reflect padding
        fixed, frames = [], []
        for w in wavs:
            w = np.asarray(w, dtype=np.float32)
            n_mel = len(w) // self.hop + 1                          # frames of the offline mel (centred STFT)
            if n_mel <= self.batch_max_frames:                      # short utterance: zero-extend features and audio
                n_fr = self.batch_max_frames + 1
                w2 = np.zeros(n_fr * self.hop, dtype=np.float32)
                w2[: len(w)] = w
                short = True
            else:
                n_fr = n_mel
                w2 = np.pad(w, (0, self.n_fft), mode="reflect")[: n_fr * self.hop]
                short = False
            fixed.append((w, w2, n_fr, n_mel, short))
            frames.append(n_fr)
        self.frames = np.asarray(frames)
        L = max(len(f[1]) for f in fixed)
        Lp = max(len(f[0]) for f in fixed) + 2 * half + pad_l + self.win_samples + self.hop * (self.batch_max_frames + 2)
        wav_tab = torch.zeros(len(fixed), L, dtype=torch.float32)
        src_tab = torch.zeros(len(fixed), Lp, dtype=torch.float32)  # utterance-level padded signal the mel frames read
        self.valid_mel = []
        for i, (w, w2, n_fr, n_mel, short) in enumerate(fixed):
            wav_tab[i, : len(w2)] = torch.from_numpy(w2)
            y = w.astype(np.float64)
            if self.preemphasize:                                   # dsp.py:53-56 on the ORIGINAL utterance
                y = np.concatenate([y[:1], y[1:] - 0.98 * y[:-1]])
            yp = np.pad(y, half, mode="reflect").astype(np.float32)  # librosa.stft(center=True, pad_mode="reflect")
            src_tab[i, self.delta: self.delta + len(yp)] = torch.from_numpy(yp)
            self.valid_mel.append(n_mel)                            # frames >= n_mel of a short utterance are zero rows
        self.wav_tab = wav_tab.to(self.device)
        self.src_tab = src_tab.to(self.device)
        self.valid_mel_t = torch.tensor(self.valid_mel, device=self.device)
        melmat = slaney_mel_filterbank(sampling_rate, self.n_fft, self.n_mels, fmin, fmax)
        self.melmat = torch.from_numpy(melmat.T.copy()).float().to(self.device).contiguous()
        self.window = _padded_window(self.win_length, self.n_fft, self.device)
        if symmetric:
            self.norm = (float(ref_level_db), float(min_level_db), 2.0 * max_norm, float(max_norm), -float(max_norm), float(max_norm))
        else:
            self.norm = (float(ref_level_db), float(min_level_db), float(max_norm), 0.0, 0.0, float(max_norm))
        self.mel_mean = None if mel_mean is None else torch.as_tensor(mel_mean, dtype=torch.float32, device=self.device).view(1, -1, 1)
        self.mel_std = None if mel_std is None else torch.as_tensor(mel_std, dtype=torch.float32, device=self.device).view(1, -1, 1)
        self._steps = torch.arange(self.batch_max_steps, device=self.device)
        self._win = torch.arange(self.win_samples, device=self.device)

    def __len__(self):
        return self.wav_tab.shape[0]

    def draw_start_frames(self, idx):
        """dataset.py:282-287: one np.random.randint per item, in batch order."""
        return np.array([np.random.randint(self.start_offset, int(self.frames[i]) + self.end_offset) for i in idx])

    def collate(self, idx, start_frames=None):
        """idx: utterance indices of the batch (the sampler's job, unchanged).  -> (wav (B, 1, T), mel (B, n_mels, frames))
        on the device, the reference's ``collate_fn`` return value."""
        idx = np.asarray(idx)
        if start_frames is None:
            start_frames = self.draw_start_frames(idx)
        sf = torch.as_tensor(start_frames, device=self.device, dtype=torch.long)
        ii = torch.as_tensor(idx, device=self.device, dtype=torch.long)
        wav = self.wav_tab[ii[:, None], (sf * self.hop)[:, None] + self._steps[None, :]].unsqueeze(1)
        # slice of the padded utterance whose frame f0 + j is the offline frame (start - aux + j); a frame centre c (utterance
        # samples) sits at src_tab column c + n_fft/2 + delta, the slice's first sample is f0 * hop before the first centre
        first = sf - self.aux
        col0 = first * self.hop + (self.n_fft // 2 + self.delta) - self.f0 * self.hop
        seg = self.src_tab[ii[:, None], col0[:, None] + self._win[None, :]]
        mel = ops.StftMelFn.apply(seg.contiguous(), self.window, self.melmat, self.n_fft, self.hop, 1, 0.0, self.norm)
        mel = mel[:, :, self.f0: self.f0 + self.n_frames]
        # frames past the end of a short (zero-extended) utterance are zero feature rows (dataset.py:249-262)
        fidx = first[:, None] + torch.arange(self.n_frames, device=self.device)[None, :]
        if self.mel_mean is not None:
            mel = (mel - self.mel_mean) / self.mel_std
        mel = torch.where((fidx < self.valid_mel_t[ii][:, None])[:, None, :], mel, torch.zeros((), device=self.device))
        return wav, mel.contiguous()


class BertMasker:
    """The BERT masking of the syBERT data path (``BERT_Text_Dataset.bert_masking`` / ``MaskingActor``,
    kantts/datasets/dataset.py:873-920, and the mask / target columns of its ``collate_fn``, 1022-1100) on the device.

    ``masker(batch)`` takes a batch with the UNMASKED ``input_lings`` (B, L, 4) and ``valid_input_lengths`` (B,) already on
    the device and returns a new dict with the reference collate's keys: ``input_lings`` with the sy column masked,
    ``targets`` (the unmasked sy column, (B, L) int64, padded with whatever pads ``input_lings``: the sy pad id, as the
    collate pads it) and ``bert_masks`` ((B, L) float, 1 at the selected positions), plus the input's other entries.  One
    kt_bert_mask launch per call and no host synchronisation.

    The rule of the reference, kept exactly: each position before ``valid_input_lengths`` (never the trailing eos nor the
    padding) is selected with probability ``mask_ratio``; of the n selected, a uniformly random floor(n * 0.8) become
    ``mask_id``, the next floor(n * 0.1) become ONE id drawn per utterance from [0, n_sy - 1], and the rest keep their
    symbol.  The draws come from Philox4x32-10 keyed by ``seed`` with a counter of (call index, utterance, position), as
    include/kantts_b200.h (kt_bert_mask) defines; they replace numpy's and Python's RNG of the dataset workers, so the masks
    follow the reference's distribution, not its samples.  ``call_index`` advances by one per call and may be set (to
    resume a run where it stopped)."""

    def __init__(self, mask_ratio, n_sy, seed, mask_id=None):
        self.mask_ratio = float(mask_ratio)
        self.n_sy = int(n_sy)
        # the sy table ends with [pad "_", eos "~", mask "@[MASK]"] (kantts/utils/ling_unit/ling_unit.py:130)
        self.mask_id = self.n_sy - 1 if mask_id is None else int(mask_id)
        self.seed = int(seed)
        self.call_index = 0

    def __call__(self, batch):
        from .sambert_ops import bert_mask
        lings, targets, masks = bert_mask(batch["input_lings"], batch["valid_input_lengths"], self.seed, self.call_index,
                                          self.mask_ratio, self.n_sy, self.mask_id)
        self.call_index += 1
        return dict(batch, input_lings=lings, targets=targets, bert_masks=masks)


class AttnPriors:
    """The alignment prior of the MAS data path (``attn_priors`` of ``AM_Dataset``: ``beta_binomial_prior_distribution``
    per utterance in ``__getitem__`` and the zero padding of ``collate_fn``, kantts/datasets/dataset.py:20-31, 497-503,
    816-827) on the device.

    ``priors(batch)`` takes a reference collate batch whose ``valid_input_lengths``, ``valid_output_lengths``,
    ``mel_targets`` and ``input_lings`` are already on the device and returns a new dict with ``attn_priors`` (B, T, L)
    float32, T = ``mel_targets.shape[1]``, L = ``input_lings.shape[1]``, the collate's shape; any ``attn_priors`` the batch
    carries is replaced, never read.  Utterance b holds the beta-binomial pmf of P = valid_input_lengths[b] + 1 symbols
    (the eos included, as the reference's ``len(ling_data[0])``) over its valid_output_lengths[b] frames, zero elsewhere,
    evaluated in float64 and rounded to float32 (include/kantts_b200.h, kt_attn_prior).  One launch and no host
    synchronisation.

    ``install(kantts_dataset=module)`` replaces the dataset's own prior with ``attn_prior_placeholder``, so the workers do
    no per-frame work; the batches then need this transform before the train step."""

    def __call__(self, batch):
        from .sambert_ops import attn_prior
        prior = attn_prior(batch["valid_input_lengths"], batch["valid_output_lengths"], batch["mel_targets"].shape[1],
                           batch["input_lings"].shape[1])
        return dict(batch, attn_priors=prior)


def attn_prior_placeholder(phoneme_count, mel_count):
    """Stand-in for the dataset's ``beta_binomial_prior_distribution`` (see ``install``): an (M, P) float32 view of a single
    NaN with strides (0, 0).  The workers compute and cache nothing per frame, ``collate_fn`` still slices its pad with the
    shape, and a batch that misses ``AttnPriors`` trains on NaN losses instead of silently without a prior (an all-zero
    prior would be a constant under the attention's log-softmax)."""
    return torch.full((), float("nan"), dtype=torch.float32).expand(int(mel_count), int(phoneme_count))


def pad_sambert_batch(batch, symbol_multiple, frame_multiple, r, ling_pad, emotion_pad, speaker_pad):
    """Right-pad a SAM-BERT collate batch (``AM_Dataset.collate_fn``'s keys, tensors on the device) to L' symbols, L' the
    symbol count rounded up to a multiple of ``symbol_multiple``, and T' frames, T' the frame count rounded up to a multiple
    of ``frame_multiple`` (itself a multiple of ``r``), with the collate's pad values: ``ling_pad`` per linguistic column
    and ``emotion_pad`` / ``speaker_pad``, the linguistic unit's "_" ids (``KanTtsLinguisticUnit._sub_unit_pad``; a float
    speaker embedding pads with 0.0 and ignores ``speaker_pad``),
    ``fp_label`` 0, mel / pitch / energy 0.0, durations 0 -- except that the T' - T new frames go to the symbol after each
    item's last one (index valid_input_lengths + 1, or the last column), as the collate gives an item its padding frames.
    Batches with durations only (not MAS).  -> a new dict; the lengths are unchanged.  Device ops only, no host synchronisation.

    Fewer distinct batch shapes mean fewer CUDA graphs (SambertStep(cuda_graph=True) captures one per shape).  Padding is
    not free of consequence: past a batch's own longest item, a padding symbol's encoder row reads as its LayerNorm bias in
    the k = 3 feed-forward convs (see KanTtsSAMBERT.front_half), so the longest item's results change.  Padding is the
    caller's choice; the train step trains on exactly what it is given."""
    import torch.nn.functional as F
    if frame_multiple % r:
        raise ValueError(f"pad_sambert_batch: frame_multiple ({frame_multiple}) must be a multiple of r ({r})")
    if symbol_multiple < 1 or frame_multiple < 1:
        raise ValueError("pad_sambert_batch: the multiples must be >= 1")
    if batch.get("durations") is None:
        raise ValueError("pad_sambert_batch: a batch without durations (MAS: frame-level contours) is not padded here")
    lings = batch["input_lings"]
    L, T = lings.shape[1], batch["mel_targets"].shape[1]
    dl, dt = -L % symbol_multiple, -T % frame_multiple
    out = dict(batch)
    if lings.shape[2] != len(ling_pad):
        raise ValueError(f"pad_sambert_batch: {lings.shape[2]} linguistic columns but {len(ling_pad)} pad ids")
    out["input_lings"] = torch.stack([F.pad(lings[:, :, i], (0, dl), value=int(v)) for i, v in enumerate(ling_pad)], -1)
    out["input_emotions"] = F.pad(batch["input_emotions"], (0, dl), value=int(emotion_pad))
    spk = batch["input_speakers"]
    out["input_speakers"] = F.pad(spk, (0, 0, 0, dl)) if spk.dim() == 3 else F.pad(spk, (0, dl), value=int(speaker_pad))
    if batch.get("fp_label") is not None:
        out["fp_label"] = F.pad(batch["fp_label"], (0, dl), value=0)
    out["mel_targets"] = F.pad(batch["mel_targets"], (0, 0, 0, dt))
    for k in ("pitch_contours", "energy_contours"):
        out[k] = F.pad(batch[k], (0, dl))
    dur = F.pad(batch["durations"], (0, dl))
    if dt:
        at = (batch["valid_input_lengths"].long() + 1).clamp_max(dur.shape[1] - 1).unsqueeze(1)
        dur = dur.scatter_add(1, at, torch.full_like(at, dt, dtype=dur.dtype))
    out["durations"] = dur
    return out
