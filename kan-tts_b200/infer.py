"""End-to-end inference without the reference's ``.npy`` hand-off (SURVEY.md section 8f item 1; BASELINE configs[4]):
symbols -> SAM-BERT free-running decode -> mel stays on the device -> HiFi-GAN generator -> waveforms.

Reference flow: kantts/bin/infer_sambert.py:205-224 writes ``<utt>_mel.npy`` (the post-net mel, one utterance per
forward because its decoder masks only support batch 1), kantts/bin/infer_hifigan.py:112-124 loads it, transposes to
(1, C, T) and runs ``Generator`` with weight norm removed.  Here a whole batch of utterances goes through both models
in one call; every utterance is cut at its own predicted length (frames x product of the up-sampling scales).

``stream_synthesize`` gives the same waveforms chunk by chunk while the decoder runs: decoder steps -> streamed post-net
(PostNet.streamer) -> streamed vocoder (Generator.streamer).  A non-causal vocoder streams with ``allow_lookahead=True``:
its output waits for its look-ahead (``lookahead`` samples, 3424 = 214 ms for the 16 kHz yamls), and each utterance's
audio equals the generator run on exactly that utterance's post-net frames, the reference's hand-off
(infer_sambert.py:136-138 then infer_hifigan.py).  A multi-band vocoder (its PQMF attached as ``generator.pqmf``) streams
its PQMF synthesis as the last stage: the synthesis reads taps/2 samples ahead (31 = 1.3 ms at 24 kHz for the default 62
taps), so that even a causal multi-band vocoder streams late by that look-ahead; being under one frame, it needs no
``allow_lookahead``.

An NSF acoustic model (``num_mels`` = mel + f0 + voiced flag) drives an NSF generator with ``nsf_f0`` and ``nsf_seeds``: the
f0 channel is denormalised and the voiced flag binarised as the reference's hand-off does (kantts/bin/infer_sambert.py:26-56
``denorm_f0``, infer_hifigan.py:57-63 ``binarize``), and the excitation is seeded per utterance (Generator.forward's
``nsf_seeds``), so that the streamed and the whole-utterance waveforms agree."""
import numpy as np
import torch

from .hifigan import StreamPlan


F0_FLOOR, UV_THRESHOLD = 30.0, 0.6          # infer_sambert.py:26 denorm_f0's f0_threshold / uv_threshold


def denorm_f0(rows, nsf_f0):
    """rows (..., num_mels) of an NSF acoustic model -> the same rows with the f0 channel (second to last) denormalised and
    clamped below at 30 Hz and the voiced flag (last) set to 1 where it is >= 0.6, else 0 (infer_sambert.py:26-56).
    ``nsf_f0``: ("mean_std", mean, std) -> f0 * std + mean, or ("global", f0_min, f0_max) -> f0 * (f0_max - f0_min) + f0_min.
    Elementwise torch ops on the rows' device."""
    kind, a, b = nsf_f0
    f0, uv = rows[..., -2:-1], rows[..., -1:]
    if kind == "mean_std":
        f0 = f0 * float(b) + float(a)
    else:
        f0 = f0 * (float(b) - float(a)) + float(a)
    return torch.cat([rows[..., :-2], f0.clamp_min(F0_FLOOR), (uv >= UV_THRESHOLD).to(rows.dtype)], -1)


def _check_nsf(sambert_num_mels, generator, nsf_f0, nsf_seeds, what):
    """-> whether the NSF hand-off runs: both of nsf_f0 / nsf_seeds given (ValueError when only one is, when the generator
    has no NSF, or when the acoustic model's channels are not the generator's mel + f0 + uv)."""
    if nsf_f0 is None and nsf_seeds is None:
        return False
    if nsf_f0 is None or nsf_seeds is None:
        raise ValueError(f"{what}: nsf_f0 and nsf_seeds go together")
    if not generator.nsf_enable:
        raise ValueError(f"{what}: nsf_f0 / nsf_seeds need an NSF generator")
    if len(nsf_f0) != 3 or nsf_f0[0] not in ("mean_std", "global"):
        raise ValueError(f"{what}: nsf_f0 must be ('mean_std', mean, std) or ('global', f0_min, f0_max), got {nsf_f0!r}")
    c_in = generator.conv_pre.conv1d.spec.c_in + 2
    if sambert_num_mels != c_in:
        raise ValueError(f"{what}: the acoustic model makes {sambert_num_mels} mel channels, the NSF generator takes {c_in} "
                         "(mel + f0 + uv)")
    return True


def stream_lookahead(generator, allow_lookahead, what):
    """-> the samples by which ``generator`` streams each sample late (StreamPlan.delay; 0 for a causal full-band generator,
    taps/2 of the PQMF for a causal multi-band one).  ValueError for a generator that does not stream (StreamPlan:
    multi-band without its PQMF attached, training mode), and for a non-causal one unless ``allow_lookahead``: its
    look-ahead adds to every utterance's time to first audio, so the caller opts in.  A causal multi-band generator
    streams without it: its PQMF synthesis reads less than a frame ahead."""
    plan = StreamPlan(generator)
    if not plan.causal and not allow_lookahead:
        raise ValueError(f"{what} needs a causal generator: a non-causal one reads {plan.delay} samples ahead of every "
                         "output sample; allow_lookahead=True accepts that delay")
    return plan.delay


def _check_stream(sambert, generator, chunk_steps, nsf_f0, nsf_seeds, allow_lookahead, what):
    """-> the vocoder's look-ahead (stream_lookahead), after the model checks stream_synthesize and TtsServer share: both
    models in eval() (RuntimeError), and ValueError unless an NSF generator comes with nsf_f0 and nsf_seeds and any other
    with neither, the acoustic model makes the mel channels the generator takes, and chunk_steps >= 1.  TtsServer, whose
    seeds come with each request, passes nsf_seeds = () along with nsf_f0."""
    if sambert.training or generator.training:
        raise RuntimeError(f"{what} expects both models in eval() mode")
    if generator.nsf_enable and (nsf_f0 is None or nsf_seeds is None):
        raise ValueError(f"{what}: an NSF generator streams with nsf_f0 and nsf_seeds: its excitation must be seeded for "
                         "the chunks to reproduce the whole utterance")
    lookahead = stream_lookahead(generator, allow_lookahead, what)
    num_mels = sambert.mel_postnet.num_mels
    if not _check_nsf(num_mels, generator, nsf_f0, nsf_seeds, what) and generator.conv_pre.conv1d.spec.c_in != num_mels:
        raise ValueError(f"{what}: the acoustic model makes {num_mels} mel channels, the generator takes "
                         f"{generator.conv_pre.conv1d.spec.c_in}")
    if int(chunk_steps) < 1:
        raise ValueError(f"{what}: chunk_steps must be >= 1, got {chunk_steps}")
    return lookahead


@torch.no_grad()
def synthesize(sambert, generator, inputs_ling, inputs_emotion, inputs_speaker, input_lengths, nsf_f0=None, nsf_seeds=None,
               per_item=False):
    """sambert: ``KanTtsSAMBERT`` in eval(); generator: ``Generator`` in eval() (``remove_weight_norm()`` optional --
    the prepared weights are cached either way).  A multi-band generator (``out_channels`` > 1) needs its PQMF attached as
    ``generator.pqmf`` (as infer_hifigan.py:47-53 does after loading), whose synthesis makes the waveform.  Tensors as in
    ``KanTtsSAMBERT.forward`` (inference branch).
    ``nsf_f0`` / ``nsf_seeds`` (both or neither): the NSF hand-off, see the module docstring and ``denorm_f0``.
    ``per_item``: the vocoder runs the padded batch with each utterance's ``LR_length_rounded`` frames as its lengths
    (Generator.forward(lengths=), PQMF.synthesis(lengths=)), so each waveform is the generator (and PQMF) on exactly its own
    post-net frames -- the reference's and TtsServer's hand-off.  Without it the vocoder runs the padded batch as is, which
    changes a shorter utterance's last samples when the generator is non-causal or multi-band.
    -> (list of 1-D waveform tensors, dict of the acoustic-model results)."""
    if sambert.training or generator.training:
        raise RuntimeError("synthesize() expects both models in eval() mode")
    pqmf = getattr(generator, "pqmf", None) if generator.out_channels > 1 else None
    if generator.out_channels > 1 and pqmf is None:
        raise ValueError("synthesize(): a multi-band generator needs its PQMF attached as generator.pqmf")
    nsf = _check_nsf(sambert.mel_postnet.num_mels, generator, nsf_f0, nsf_seeds, "synthesize()")
    res = sambert(inputs_ling, inputs_emotion, inputs_speaker, input_lengths)
    mel = res["postnet_outputs"]                                   # (B, T, num_mels), zero beyond each length
    frames = res["LR_length_rounded"]
    # per_item: the frame counts as host ints (read here anyway to cut the waveforms), so the generator checks each one
    # against the post-net's rows
    lengths = [int(n) for n in frames.tolist()] if per_item else None
    if nsf:
        wav = generator(denorm_f0(mel, nsf_f0).transpose(1, 2).contiguous(), nsf_seeds=nsf_seeds, lengths=lengths)
    else:
        wav = generator(mel.transpose(1, 2).contiguous(), lengths=lengths)   # (B, out_channels, T * prod(scales))
    if pqmf is not None:
        scale = int(np.prod(generator.upsample_scales))
        wav = pqmf.synthesis(wav, None if lengths is None else [n * scale for n in lengths])   # (B, 1, T * hop)
    hop = int(np.prod(generator.upsample_scales)) * generator.out_channels
    wavs = [wav[b, 0, : int(frames[b]) * hop] for b in range(wav.shape[0])]
    return wavs, res


def stream_synthesize(sambert, generator, inputs_ling, inputs_emotion, inputs_speaker, input_lengths, chunk_steps=4,
                      nsf_f0=None, nsf_seeds=None, allow_lookahead=False):
    """Streaming ``synthesize``: the encoder, the variance adaptor and the decoder memory run now, then iterating the
    returned TtsStream decodes ``chunk_steps`` decoder steps at a time and yields their audio as soon as the post-net rows
    are final.  An NSF generator needs ``nsf_f0`` and ``nsf_seeds`` (as ``synthesize``), applied to each chunk of post-net
    rows.  For every slot b, the yielded chunks concatenated and cut at ``lengths[b]`` are
    ``synthesize(..., nsf_f0, nsf_seeds)[0][b]`` for a causal generator.
    A non-causal generator is refused unless ``allow_lookahead``: its audio then comes ``TtsStream.lookahead`` samples
    later, and slot b's is the generator run on exactly its ``lengths[b] / hop`` post-net frames (the reference's
    hand-off; ``synthesize`` runs it on the batch's padded mel instead, which changes an utterance's last samples).
    A multi-band generator streams with its PQMF attached, with or without ``allow_lookahead`` when it is causal: slot b's
    audio is ``pqmf.synthesis(generator(mel_b))`` of exactly its frames, later by the synthesis's taps/2 samples (plus the
    generator's own look-ahead when it is non-causal).  Against ``synthesize``, a shorter utterance of the batch differs in
    its last taps/2 samples, where the padded batch's synthesis reads the generator's output past the utterance's end."""
    lookahead = _check_stream(sambert, generator, chunk_steps, nsf_f0, nsf_seeds, allow_lookahead, "stream_synthesize()")
    return TtsStream(sambert, generator, inputs_ling, inputs_emotion, inputs_speaker, input_lengths, int(chunk_steps),
                     lookahead, nsf_f0, nsf_seeds)


class TtsStream:
    """The audio of one batch of utterances, chunk by chunk (made by ``stream_synthesize``).

    ``lengths``: per-slot sample counts, ``LR_length_rounded[b] * hop`` (read on the host once, before decoding).
    ``hop``: the vocoder's samples per frame (GeneratorStreamer.hop: prod(upsample_scales), times S for a multi-band one).
    ``delay`` / ``lookahead``: the post-net's delay in rows and the vocoder's in samples (GeneratorStreamer.delay; 0 for a
    causal full-band one).  The post-net's push of the decoder rows [p, p + f) returns the frames [p - delay, p + f -
    delay), the vocoder's push of the frames [p, p + f) the samples [p·hop - lookahead, (p + f)·hop - lookahead); what
    lies before 0 is dropped, and after the last decoder step each streamer's drain (``finish``) brings out the rest.
    Iterating yields ``(start_sample, wav)``, ``wav`` (B, 1, n) on the device, n > 0, with starts contiguous from 0; slot
    b's audio ends at lengths[b] and is padding after that.  From the first chunk to the last no device data is read on
    the host.  A stream is iterated once."""

    def __init__(self, sambert, generator, inputs_ling, inputs_emotion, inputs_speaker, input_lengths, chunk_steps,
                 lookahead, nsf_f0=None, nsf_seeds=None):
        self.sambert, self.chunk_steps, self.lookahead, self.nsf_f0 = sambert, chunk_steps, lookahead, nsf_f0
        dec = sambert.mel_decoder
        self.r, self.d_mel = dec.r, dec.d_mel
        with torch.no_grad():
            self._front = f = sambert.front_half(inputs_ling, inputs_emotion, inputs_speaker, input_lengths)
        self.batch = B = f["memory"].shape[0]
        frames = f["lr_len"]
        self.max_frames = F = self.r * chunk_steps
        self._post = sambert.mel_postnet.streamer(B, F, frames)
        self.delay = self._post.delay
        # a vocoder with a look-ahead (non-causal, or multi-band: the PQMF synthesis) masks each slot's utterance end on the
        # device, from the lengths the decoder masks by
        self._voc = generator.streamer(batch=B, max_frames=F, lengths=frames if lookahead else None, seeds=nsf_seeds)
        self.hop = self._voc.hop
        self.lengths = [int(n) * self.hop for n in frames.cpu()]
        self._used = False

    @staticmethod
    def _from_zero(x, start, dim):
        """x, a delayed streamer's output whose entries along ``dim`` are the stream's positions from ``start`` on ->
        [(its first position from 0 on, x without the positions before 0)], [] when x holds only those."""
        lo = max(0, -start)
        return [(start + lo, x.narrow(dim, lo, x.shape[dim] - lo))] if lo < x.shape[dim] else []

    def _vocode(self, rows, start):
        """rows (B, n, num_mels) of final post-net output -> [(start sample, wav)] in pieces of at most max_frames frames,
        and the start of the next piece."""
        out = []
        for piece in torch.split(rows, self.max_frames, dim=1):
            out += self._from_zero(self._voc.push(piece.transpose(1, 2)), start, 2)
            start += piece.shape[1] * self.hop
        return out, start

    def __iter__(self):
        if self._used:
            raise RuntimeError("a TtsStream is iterated once")
        self._used = True
        f = self._front
        steps, B, start, row = f["memory"].shape[1], self.batch, -self.lookahead, 0
        outs = []
        with torch.no_grad():
            for s, (out, _, _) in enumerate(self.sambert.mel_decoder.infer_steps(f["memory"], f["x_band_width"],
                                                                                f["x_band_width"])):
                outs.append(out)
                last = s == steps - 1
                if len(outs) < self.chunk_steps and not last:
                    continue
                dec = torch.cat(outs, 1).view(B, -1, self.d_mel)                 # de-LFR: r frames per step
                outs = []
                frames = torch.arange(row, row + dec.shape[1], device=dec.device)
                dec = dec.masked_fill((frames[None, :] >= f["lr_len"][:, None]).unsqueeze(-1), 0)
                rows = self._post.push(dec)
                if last:
                    rows = torch.cat([rows, self._post.finish()], 1)
                for _, mel in self._from_zero(rows, row - self.delay, 1):
                    if self.nsf_f0 is not None:
                        mel = denorm_f0(mel, self.nsf_f0)
                    chunks, start = self._vocode(mel, start)
                    yield from chunks
                row += dec.shape[1]
            if self.lookahead:
                yield from self._from_zero(self._voc.finish(), start, 2)


def slot_schedule(r, chunk_steps, delay, frames, steps, chunk, max_steps, hop=1, lookahead=0):
    """Where an utterance of ``frames`` post-net frames and ``steps`` decoder steps, admitted to a TtsServer slot for chunk
    ``chunk``, runs (decoder rows are counted from row 0 of chunk 0; a chunk holds f = r * chunk_steps rows), into a
    vocoder of ``hop`` samples per frame whose output lags by ``lookahead`` samples (0: a causal vocoder):
      start_step  the step of the admission chunk at which the slot decodes the utterance's step 0: ((-delay) mod f) / r,
                  so that its frame 0, which the post-net returns ``delay`` rows later, is output row 0 of a chunk
      voc_chunk   that chunk: the slot's vocoder is reset just before it.  Chunk voc_chunk + k returns the samples
                  [k·f·hop - lookahead, (k + 1)·f·hop - lookahead) (``chunk_audio``): the first audio is in chunk
                  voc_chunk + lookahead // (f·hop), from its sample lookahead mod (f·hop)
      last_chunk  the chunk that returns the utterance's last sample: voc_chunk + (frames·hop - 1 + lookahead) // (f·hop),
                  with no look-ahead the chunk that returns its last frame
      free_row    the first decoder row after the last frame became final and after the last decoder step
      free_chunk  the first chunk that may admit the slot's next utterance: the chunk holding free_row, or the one after,
                  and late enough that the next utterance's voc_chunk (as far after its admission chunk as this one's) comes
                  after last_chunk: a vocoder reset before the drain would lose the utterance's last samples.  With a
                  look-ahead, free_chunk may come before last_chunk: the next utterance decodes while this one drains
    ValueError when delay is not a multiple of r (frame 0 could not start a chunk) or steps > max_steps."""
    if delay % r:
        raise ValueError(f"serving needs a post-net delay that is a multiple of the decoder's r: delay {delay}, r {r}")
    if steps > max_steps:
        raise ValueError(f"an utterance of {steps} decoder steps does not fit max_steps = {max_steps}")
    f = r * chunk_steps
    p0 = (-delay) % f
    first = chunk * f + p0                                       # decoder row of frame 0
    last_row = first + frames - 1 + delay                        # its arrival makes the last frame final
    free_row = max(last_row, first + steps * r - 1) + 1
    voc_chunk = (first + delay) // f
    # with lookahead 0 this is last_row // f (first + delay is a multiple of f), and the reset bound is below free_row's
    last_chunk = voc_chunk + (frames * hop - 1 + lookahead) // (f * hop)
    return dict(start_step=p0 // r, voc_chunk=voc_chunk, last_chunk=last_chunk, free_row=free_row,
                free_chunk=max(-(-free_row // f), last_chunk + 1 - (voc_chunk - chunk)))


def chunk_audio(voc_chunk, samples, chunk, chunk_samples, lookahead=0):
    """The audio of an utterance of ``samples`` samples in chunk ``chunk``'s vocoder output of ``chunk_samples`` samples,
    the utterance's frame 0 being row 0 of chunk ``voc_chunk`` and the vocoder's output lagging by ``lookahead`` samples
    -> (start, lo, hi): the chunk's samples [lo, hi) are the utterance's [start, start + hi - lo); None when the chunk
    holds none of them."""
    first = (chunk - voc_chunk) * chunk_samples - lookahead
    lo, hi = max(0, -first), min(chunk_samples, samples - first)
    return (first + lo, lo, hi) if lo < hi else None


def pad_requests(inputs):
    """[(ling (1, L_i, 4), emotion (1, L_i), speaker (1, L_i) or (1, L_i, units), length (1,))] of TtsServer requests -> the
    (ling, emotion, speaker, lengths) of ONE ``KanTtsSAMBERT`` batch: each request right-padded with zeros to the longest
    L_i, lengths (k,).  ``front_half(..., per_item=True)`` of the batch gives request i its results alone."""
    L = max(x[0].shape[1] for x in inputs)
    pad = lambda t: torch.cat([t, t.new_zeros(1, L - t.shape[1], *t.shape[2:])], 1)
    return tuple(torch.cat([pad(x[j]) for x in inputs]) for j in range(3)) + (torch.cat([x[3] for x in inputs]),)


class TtsServer:
    """Continuous batching of text-to-speech: requests join and leave the ``slots`` slots of one running stream.

    ``submit(ling, emotion, speaker, length[, nsf_seed])`` queues one utterance (tensors of ``KanTtsSAMBERT.forward``
    without the batch dimension) and returns its request id.  ``step()`` runs one chunk of ``chunk_steps`` decoder steps
    -> (audio, finished): ``audio`` lists ``(request id, start sample, wav)`` for every request with audio in this chunk
    (wav 1-D on the device, cut at the request's end), ``finished`` the ids whose last audio this was.

    Each slot decodes its own utterance (SlotDecoder: its own step, memory length and band), through a per-slot post-net
    streamer into the vocoder streamer.  A request's audio equals ``synthesize`` of that request alone (with its
    ``nsf_seed`` for an NSF generator), whatever the other slots hold.  Admission (at the start of a ``step``, for the queued
    requests that fit free slots) right-pads the round's requests into one batch (``pad_requests``) and runs ``front_half``
    ONCE with ``per_item=True``: each request's memory rows, frame count and band are bit for bit those of the request
    alone, so each slot takes its request's slices.  The round's host reads are that one call's, however many requests it
    admits; between admissions no call reads device data.  The alignment of each slot is ``slot_schedule``.  ``nsf_f0``
    (see ``denorm_f0``) is required for an NSF generator.

    A non-causal generator is refused unless ``allow_lookahead``: each request's audio then comes ``lookahead`` samples
    later (the vocoder's delay; 0 for a causal one) and equals the generator run on exactly that request's post-net
    frames, the reference's hand-off.  A multi-band generator serves with its PQMF attached (``generator.pqmf``); a
    causal one needs no ``allow_lookahead``: its look-ahead is the PQMF synthesis's taps/2 samples, and each request's
    audio is ``pqmf.synthesis(generator(mel))`` of exactly its frames (``synthesize`` of a padded batch differs from it in
    a shorter utterance's last taps/2 samples).  A slot may start decoding its next request while the vocoder still
    drains the previous one's last samples, timed so that its vocoder reset comes after them.  (``delay`` is the
    post-net's delay in rows.)"""

    def __init__(self, sambert, generator, slots, chunk_steps, max_steps, nsf_f0=None, allow_lookahead=False):
        from .sambert import PostNetStreamPlan
        self.lookahead = _check_stream(sambert, generator, chunk_steps, nsf_f0, None if nsf_f0 is None else (),
                                       allow_lookahead, "TtsServer")
        self.nsf = generator.nsf_enable
        self.chunk_steps, self.max_steps, self.batch = int(chunk_steps), int(max_steps), int(slots)
        if self.max_steps < 1 or self.batch < 1:
            raise ValueError(f"TtsServer: slots ({slots}) and max_steps ({max_steps}) must be >= 1")
        dec = sambert.mel_decoder
        self.r, self.d_mel = dec.r, dec.d_mel
        self.delay = PostNetStreamPlan(sambert.mel_postnet).delay
        if self.delay % self.r:
            raise ValueError(f"TtsServer: the post-net delay ({self.delay}) must be a multiple of the decoder's r ({self.r}) "
                             "for an utterance's frame 0 to start a chunk")
        self.sambert, self.nsf_f0 = sambert, nsf_f0
        self.frames_per_chunk = F = self.r * self.chunk_steps
        self.device = next(sambert.parameters()).device
        self._dec = dec.slots(self.batch, self.max_steps)
        with torch.no_grad():
            self._post = sambert.mel_postnet.streamer(self.batch, F, torch.zeros(self.batch, dtype=torch.int32,
                                                                                 device=self.device))
            # every slot is reset, with its request's frame count and seed, before its first audio
            self._voc = generator.streamer(batch=self.batch, max_frames=F, lengths=[1] * self.batch if self.lookahead else None,
                                           seeds=[0] * self.batch if self.nsf else None)
        self.hop = self._voc.hop                        # waveform samples per frame (times S for a multi-band vocoder)
        # _slots: each slot's current request (decoder and post-net); _playing: (slot, request) of every request whose
        # audio has not all come out, which with a vocoder look-ahead can outlast its slot's hold on the decoder
        self._queue, self._slots, self._playing, self._chunk, self._next_id = [], [None] * self.batch, [], 0, 0

    def submit(self, ling, emotion, speaker, length, nsf_seed=None):
        """Queue one utterance: ling (L, 4), emotion (L,) long tensors, speaker (L,) ids, or the (L, speaker_units) float
        embedding rows of a speaker-embedding (SE) model, and its symbol count ``length``; ``nsf_seed`` (an int) for an NSF
        generator.  -> the request id."""
        if self.nsf != (nsf_seed is not None):
            raise ValueError("submit: an NSF generator needs each request's nsf_seed, any other generator none")
        rid, self._next_id = self._next_id, self._next_id + 1
        self._queue.append(dict(id=rid, seed=nsf_seed, inputs=(ling.reshape(1, -1, ling.shape[-1]), emotion.reshape(1, -1),
                                                                speaker.unsqueeze(0), torch.tensor([int(length)]))))
        return rid

    @property
    def idle(self):
        """No request queued, in a slot or with audio still to come."""
        return not self._queue and not self._playing and all(s is None or s["free_chunk"] <= self._chunk
                                                               for s in self._slots)

    def _admit(self, c):
        free = [b for b, s in enumerate(self._slots) if s is None or s["free_chunk"] <= c]
        take = self._queue[:len(free)]
        if not take:
            return
        with torch.no_grad():
            fr = self.sambert.front_half(*(t.to(self.device) for t in pad_requests([req["inputs"] for req in take])),
                                         per_item=True)
        frames = fr["lr_len"].tolist()                                                  # the round's one host read
        sched = []
        for req, n in zip(take, frames):
            try:
                sched.append(slot_schedule(self.r, self.chunk_steps, self.delay, n, -(-n // self.r), c,
                                           self.max_steps, hop=self.hop, lookahead=self.lookahead))
            except ValueError as e:
                self._queue.remove(req)
                raise ValueError(f"request {req['id']}: {e}") from None
        del self._queue[:len(take)]
        for j, (b, req, n, s) in enumerate(zip(free, take, frames, sched)):
            self._dec.admit(b, fr["memory"][j:j + 1, :-(-n // self.r)], fr["band_width_rows"][j])
            self._post.reset([b], [n], start_row=s["start_step"] * self.r)
            seed = None if req["seed"] is None else torch.tensor([int(req["seed"])], dtype=torch.int64).to(self.device)
            self._slots[b] = dict(s, chunk=c, id=req["id"], frames=n, samples=n * self.hop, seed=seed)
            self._playing.append((b, self._slots[b]))

    def step(self):
        """Run one chunk -> (audio, finished), see the class docstring."""
        c, B, F = self._chunk, self.batch, self.frames_per_chunk
        self._admit(c)
        live = [(b, s) for b, s in enumerate(self._slots) if s is not None and s["free_chunk"] > c]
        with torch.no_grad(), torch.cuda.device(self.device):
            rows = []
            for k in range(self.chunk_steps):
                for b, s in live:
                    if s["chunk"] == c and s["start_step"] == k:
                        self._dec.start(b)
                rows.append(self._dec.advance())
            post = self._post.push(torch.cat(rows, 1).view(B, F, self.d_mel))
            if self.nsf_f0 is not None:
                post = denorm_f0(post, self.nsf_f0)
            due = [(b, s) for b, s in live if s["voc_chunk"] == c]
            if due:
                seeds = torch.cat([s["seed"] for _, s in due]) if self.nsf else None
                lengths = [s["frames"] for _, s in due] if self.lookahead else None
                self._voc.reset([b for b, _ in due], lengths, seeds=seeds)
            wav = self._voc.push(post.transpose(1, 2))
        audio, finished = [], []
        for b, s in sorted(self._playing, key=lambda p: p[0]):
            cut = chunk_audio(s["voc_chunk"], s["samples"], c, F * self.hop, self.lookahead)
            if cut is not None:
                start, lo, hi = cut
                audio.append((s["id"], start, wav[b, 0, lo:hi]))
                if c == s["last_chunk"]:
                    finished.append(s["id"])
        self._playing = [(b, s) for b, s in self._playing if s["last_chunk"] > c]
        self._chunk += 1
        return audio, finished
