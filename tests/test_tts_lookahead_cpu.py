"""CPU checks of streaming and serving text-to-speech through a non-causal vocoder (``allow_lookahead``): the slot
schedule with the vocoder's look-ahead covers each utterance's samples exactly once, in order, from the chunks it names;
a slot's vocoder is reset for the next utterance only after the last sample has come out; without a look-ahead the
schedule is the causal one; the flag lets a non-causal generator through and changes nothing for a causal one."""
import pytest
import torch

import kantts_b200 as K
from kantts_b200.hifigan import StreamPlan
from kantts_b200.infer import chunk_audio, slot_schedule, stream_lookahead
from test_stream_cpu import CONFIGS
from test_tts_stream_cpu import _models

R, D = 3, 12                                          # the shipped yamls: outputs_per_step 3, post-net delay 12
# (hop, look-ahead): causal at the 24 kHz hop; a few samples; the small non-causal test generator (90 samples at hop 8,
# more than a chunk of 1 step and less than one of 16); hifigan_noncausal_v1_16k (3424 at hop 200)
LOOKAHEADS = [(240, 0), (8, 5), (8, 90), (200, 3424)]
V1_16K = dict(channels=256, upsample_scales=[10, 5, 2, 2], upsample_kernal_sizes=[20, 11, 4, 4],
              resblock_dilations=[[1, 3, 5, 7]] * 3, causal=False)          # hifigan_noncausal_v1_16k.yaml


def _pieces(s, frames, hop, lookahead, chunk_steps):
    """-> {chunk: (start, lo, hi)} of every chunk from the admission chunk to well past the drain that holds audio."""
    f = R * chunk_steps
    out = {}
    for c in range(s["voc_chunk"] - 3, s["last_chunk"] + 4):
        cut = chunk_audio(s["voc_chunk"], frames * hop, c, f * hop, lookahead)
        if cut is not None:
            out[c] = cut
    return out


@pytest.mark.parametrize("hop,lookahead", LOOKAHEADS)
@pytest.mark.parametrize("chunk_steps", [1, 2, 3, 4, 16])
@pytest.mark.parametrize("chunk", [0, 5])
@pytest.mark.parametrize("frames", [1, 2, 13, 47, 48, 100])
def test_schedule_covers_each_sample_once_and_resets_after_the_drain(chunk_steps, chunk, frames, hop, lookahead):
    f = R * chunk_steps
    steps = -(-frames // R)
    s = slot_schedule(R, chunk_steps, D, frames, steps, chunk, steps, hop=hop, lookahead=lookahead)
    causal = slot_schedule(R, chunk_steps, D, frames, steps, chunk, steps)
    # the decoder and post-net terms are the causal schedule's
    assert {k: s[k] for k in ("start_step", "voc_chunk", "free_row")} == {k: causal[k] for k in ("start_step", "voc_chunk",
                                                                                                  "free_row")}
    # coverage: the chunks' pieces, in chunk order, are [0, frames * hop) once, from a0 at offset lookahead mod (f * hop)
    # to the last chunk
    pieces = _pieces(s, frames, hop, lookahead, chunk_steps)
    a0 = s["voc_chunk"] + lookahead // (f * hop)
    assert min(pieces) == a0 and pieces[a0][1] == lookahead % (f * hop)
    assert max(pieces) == s["last_chunk"] == s["voc_chunk"] + (frames * hop - 1 + lookahead) // (f * hop)
    assert sorted(pieces) == list(range(a0, s["last_chunk"] + 1))
    at = 0
    for c in sorted(pieces):
        start, lo, hi = pieces[c]
        assert start == at and 0 <= lo < hi <= f * hop
        assert start + lookahead == (c - s["voc_chunk"]) * f * hop + lo          # the vocoder's output position
        at += hi - lo
    assert at == frames * hop
    # reset safety: a next utterance admitted at free_chunk has its vocoder reset after the last sample; one chunk earlier
    # would either overlap the decoder / post-net or reset before the drain
    nxt = slot_schedule(R, chunk_steps, D, 5, 2, s["free_chunk"], 2, hop=hop, lookahead=lookahead)
    assert nxt["voc_chunk"] > s["last_chunk"]
    assert s["free_chunk"] >= causal["free_chunk"]
    if s["free_chunk"] > causal["free_chunk"]:
        early = slot_schedule(R, chunk_steps, D, 5, 2, s["free_chunk"] - 1, 2, hop=hop, lookahead=lookahead)
        assert early["voc_chunk"] <= s["last_chunk"]


@pytest.mark.parametrize("hop", [1, 8, 200, 240])
@pytest.mark.parametrize("chunk_steps", [1, 2, 3, 4, 16])
@pytest.mark.parametrize("chunk", [0, 5])
@pytest.mark.parametrize("frames", [1, 2, 13, 47, 48, 100])
def test_schedule_without_lookahead_is_the_causal_schedule(chunk_steps, chunk, frames, hop):
    steps = -(-frames // R)
    s = slot_schedule(R, chunk_steps, D, frames, steps, chunk, steps, hop=hop, lookahead=0)
    assert s == slot_schedule(R, chunk_steps, D, frames, steps, chunk, steps)
    # and its chunk audio is the causal cut: chunk voc_chunk + k holds samples [k * f * hop, ...) from its row 0
    f = R * chunk_steps
    for c, (start, lo, hi) in _pieces(s, frames, hop, 0, chunk_steps).items():
        k = c - s["voc_chunk"]
        assert (start, lo, hi) == (k * f * hop, 0, min(f * hop, frames * hop - k * f * hop))


def test_lookahead_of_the_flag():
    causal = K.Generator(**CONFIGS["small"]).eval()
    assert stream_lookahead(causal, False, "streaming") == stream_lookahead(causal, True, "streaming") == 0
    nc = K.Generator(**V1_16K).eval()
    with pytest.raises(ValueError, match="causal.*allow_lookahead"):
        stream_lookahead(nc, False, "streaming")
    assert stream_lookahead(nc, True, "streaming") == StreamPlan(nc).delay == 3424
    mb = K.Generator(out_channels=4, channels=32, upsample_scales=[5, 3, 2, 2], upsample_kernal_sizes=[10, 6, 4, 4]).eval()
    for allow in (False, True):
        with pytest.raises(ValueError, match="multi-band"):
            stream_lookahead(mb, allow, "streaming")


def test_the_flag_in_stream_synthesize_and_the_server(golden):
    inputs = (torch.zeros(1, 4, 4, dtype=torch.long), torch.zeros(1, 4, dtype=torch.long), torch.zeros(1, 4, dtype=torch.long),
              torch.tensor([4]))
    am, gen = _models(golden)
    # a causal generator meets the same checks either way: here the mel-channel check (80 against the model's 8) ...
    for allow in (False, True):
        with pytest.raises(ValueError, match="mel channels"):
            K.stream_synthesize(am, _models(golden, in_channels=80)[1], *inputs, allow_lookahead=allow)
        # ... and the server's post-net delay check (the small golden SAM-BERT: delay 2, r 3)
        with pytest.raises(ValueError, match="multiple"):
            K.TtsServer(am, gen, slots=2, chunk_steps=2, max_steps=64, allow_lookahead=allow)
    # a non-causal one gets past the causal check to the same later checks only with the flag
    nc80 = _models(golden, in_channels=80, causal=False)[1]
    with pytest.raises(ValueError, match="causal generator"):
        K.stream_synthesize(am, nc80, *inputs)
    with pytest.raises(ValueError, match="mel channels"):
        K.stream_synthesize(am, nc80, *inputs, allow_lookahead=True)
    nc = _models(golden, causal=False)[1]
    with pytest.raises(ValueError, match="causal generator"):
        K.TtsServer(am, nc, slots=2, chunk_steps=2, max_steps=64)
    with pytest.raises(ValueError, match="multiple"):
        K.TtsServer(am, nc, slots=2, chunk_steps=2, max_steps=64, allow_lookahead=True)
    # a multi-band generator stays refused
    mb = _models(golden, out_channels=4)[1]
    with pytest.raises(ValueError, match="multi-band"):
        K.stream_synthesize(am, mb, *inputs, allow_lookahead=True)
    with pytest.raises(ValueError, match="multi-band"):
        K.TtsServer(am, mb, slots=2, chunk_steps=2, max_steps=64, allow_lookahead=True)
