"""CPU checks of continuous-batching text-to-speech (infer.TtsServer): the slot alignment arithmetic (slot_schedule) for chunk
sizes that divide the post-net delay and ones that do not, the exported entry points, and the rejected configurations."""
import pytest
import torch

import kantts_b200 as K
from kantts_b200 import _lib
from kantts_b200.infer import slot_schedule
from test_tts_stream_cpu import _models

R, D = 3, 12                                          # the shipped yamls: outputs_per_step 3, post-net delay 12


@pytest.mark.parametrize("chunk_steps", [1, 2, 4, 3, 16])
@pytest.mark.parametrize("chunk", [0, 5])
@pytest.mark.parametrize("frames", [1, 2, 13, 47, 48, 100])
def test_slot_schedule_aligns_frame_zero_with_a_chunk(chunk_steps, chunk, frames):
    f = R * chunk_steps
    steps = -(-frames // R)
    s = slot_schedule(R, chunk_steps, D, frames, steps, chunk, max_steps=steps)
    assert 0 <= s["start_step"] < chunk_steps
    first = chunk * f + s["start_step"] * R             # decoder row of frame 0
    # frame 0 leaves the post-net D rows later, as output row 0 of the vocoder-reset chunk
    assert (first + D) % f == 0 and (first + D) // f == s["voc_chunk"] > chunk
    # the last frame becomes final with decoder row first + frames - 1 + D; the slot is free from the row after it
    last = first + frames - 1 + D
    assert s["last_chunk"] == last // f and s["free_row"] == last + 1
    assert s["free_chunk"] == -(-(last + 1) // f) and s["free_chunk"] > s["last_chunk"]
    # the decoder's last row (steps * r rows from frame 0's row) lies before the free row
    assert first + steps * R - 1 < s["free_row"]


def test_slot_schedule_values():
    # chunk_steps 1 (f = 3 divides D): start at step 0, frame 0 out four chunks later
    assert slot_schedule(R, 1, D, 10, 4, 0, 100) == dict(start_step=0, voc_chunk=4, last_chunk=7, free_row=22, free_chunk=8)
    # chunk_steps 16 (f = 48 does not): start 12 steps (36 rows) in, frame 0 is row 0 of the next chunk
    assert slot_schedule(R, 16, D, 10, 4, 0, 100) == dict(start_step=12, voc_chunk=1, last_chunk=1, free_row=58, free_chunk=2)
    # chunk_steps 3 (f = 9): (-12) mod 9 = 6 rows = 2 steps in
    assert slot_schedule(R, 3, D, 9, 3, 2, 100)["start_step"] == 2


def test_slot_schedule_rejects():
    with pytest.raises(ValueError, match="multiple"):
        slot_schedule(3, 4, 2, 10, 4, 0, 100)
    with pytest.raises(ValueError, match="max_steps"):
        slot_schedule(R, 4, D, 31, 11, 0, 10)


def test_entry_points_are_exported():
    for name in ("kt_pnca_step_slots", "kt_fsmn_fwd_stream_slots", "kt_lstm_stream_slots"):
        assert name in _lib.PROTOTYPES
    assert K.TtsServer is K.infer.TtsServer and K.slot_schedule is slot_schedule
    assert callable(K.sambert.MelPNCADecoder.slots)


def test_server_rejects_a_delay_that_is_not_a_multiple_of_r(golden):
    am, gen = _models(golden)                          # the small golden SAM-BERT: post-net delay 2, r 3
    with pytest.raises(ValueError, match="multiple"):
        K.TtsServer(am, gen, slots=2, chunk_steps=2, max_steps=64)
    with pytest.raises(RuntimeError, match="eval"):
        K.TtsServer(am, gen.train(), slots=2, chunk_steps=2, max_steps=64)
    with pytest.raises(ValueError, match="causal"):
        K.TtsServer(am, _models(golden, causal=False)[1], slots=2, chunk_steps=2, max_steps=64)
