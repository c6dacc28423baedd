"""The stream window format of the streamed vocoder (hifigan.GeneratorStreamer) and post-net (sambert.PostNetStreamer),
the per-slot utterance record both keep, and the scaffolding both build on (Streamer), DESIGN.md §3.7.  A window is a persistent (B, H + F·rows_per_frame, C)
buffer: rows [0, H) carry the last H rows of the earlier chunks (zeros after a reset: the causal padding), the chunk is
written at row H, and H is the largest history any reader of the tensor needs."""
import ctypes

import torch

from . import ops
from ._lib import KtStreamMask, KtStreamWin, KtWindow, ptr


class WindowTable:
    """Plan-time list of a stream's windows: ``windows`` holds one {name, channels, rows_per_frame, history} dict per
    tensor, in the order they were added."""

    def __init__(self):
        self.windows = []

    def add(self, name, channels, rows_per_frame=1):
        self.windows.append(dict(name=name, channels=channels, rows_per_frame=rows_per_frame, history=0))
        return name

    def read(self, name, history):
        """A reader of ``name`` needs ``history`` rows before the chunk."""
        w = next(w for w in self.windows if w["name"] == name)
        w["history"] = max(w["history"], history)

    def launches_per_chunk(self, steps):
        """``steps`` launches, plus the window advance when any window keeps history."""
        return steps + any(w["history"] for w in self.windows)


class Windows:
    """The buffers of a WindowTable's windows for ``batch`` slots and chunks of 1..max_frames frames, by name: ``buf``
    (B, pitch, C), ``first`` (row H, where the chunk starts) and ``rate`` (rows per frame)."""

    def __init__(self, windows, batch, max_frames, device, what):
        batch, max_frames = int(batch), int(max_frames)
        if batch < 1 or max_frames < 1:
            raise ValueError(f"streamer: batch ({batch}) and max_frames ({max_frames}) must be >= 1")
        if device.type != "cuda":
            raise RuntimeError(f"kantts_b200: the {what} runs on a CUDA device (no CPU fallback)")
        self.batch, self.max_frames, self.device = batch, max_frames, device
        self.buf = {w["name"]: torch.zeros(batch, w["history"] + max_frames * w["rows_per_frame"], w["channels"], device=device)
                    for w in windows}
        self.first = {w["name"]: w["history"] for w in windows}
        self.rate = {w["name"]: w["rows_per_frame"] for w in windows}
        kept = [w for w in windows if w["history"] > 0]
        table = (KtWindow * len(kept))(*[KtWindow(base=self.buf[w["name"]].data_ptr(), pitch=self.buf[w["name"]].shape[1],
                                                  channels=w["channels"], history=w["history"],
                                                  rows_per_frame=w["rows_per_frame"]) for w in kept])
        self._table = torch.frombuffer(bytearray(bytes(table)), dtype=torch.uint8).to(device)
        self._ntable, self._max_c = len(kept), max([w["channels"] for w in kept], default=1)

    def push(self, name, x, f_axis, what):
        """Check the chunk x, (B, C, f) for f_axis 2 or (B, f, C) for f_axis 1, and write it into window ``name`` -> f.
        ``what``: (x's description with {} for the shape, unit of f, "<x> is") for the errors."""
        c = self.buf[name].shape[2]
        if x.dim() != 3 or x.shape[0] != self.batch or x.shape[3 - f_axis] != c:
            shape = (self.batch, c, "f") if f_axis == 2 else (self.batch, "f", c)
            raise ValueError(f"push: expected {what[0].format('(%s, %s, %s)' % shape)}, got {tuple(x.shape)}")
        f = x.shape[f_axis]
        if not 1 <= f <= self.max_frames:
            raise ValueError(f"push: a chunk holds 1 to {self.max_frames} {what[1]}, got {f}")
        if x.device != self.device:
            raise ValueError(f"push: {what[2]} on {x.device}, the streamer on {self.device}")
        h = self.first[name]
        self.buf[name][:, h:h + f].copy_(x if f_axis == 1 else x.transpose(1, 2))
        return f

    def place(self, src, dst, resid=None, res_lag=0):
        """-> the KtStreamWin of a layer reading the chunk of ``src``, writing the chunk of ``dst`` and adding the rows of
        ``resid`` that lie ``res_lag`` rows before its chunk."""
        b, first = self.buf, self.first
        w = KtStreamWin(in_pitch=b[src].shape[1], in_first=first[src], out_pitch=b[dst].shape[1], out_first=first[dst])
        if resid is not None:
            w.res_pitch, w.res_first = b[resid].shape[1], first[resid] - res_lag
        return w

    def advance(self, frames):
        """After a chunk of ``frames`` frames, the last H rows of every window become its history (one launch)."""
        if self._ntable:
            ops.call("kt_stream_advance", ptr(self._table, True), self._ntable, self.batch, frames, self._max_c)

    def reset(self, slots):
        """The history of the given slots returns to zeros in every window (one launch)."""
        mask = torch.zeros(self.batch, dtype=torch.uint8)
        mask[check_slots(slots, self.batch)] = 1
        sel = to_device(mask, self.device)
        if self._ntable:
            ops.call("kt_stream_reset", ptr(self._table, True), self._ntable, self.batch, ptr(sel, True), self._max_c)


class SlotUtterances:
    """Each slot's place in its utterance, on the device: ``lengths`` and ``frames_done`` (frames since frame 0), int32
    (B,).  Chunk row t of a window trailing by ``lag`` rows is frame frames_done[b] + (t - lag) / rows_per_frame."""

    def __init__(self, batch, device):
        self.batch, self.device = batch, device
        self.lengths = torch.zeros(batch, dtype=torch.int32, device=device)
        self.frames_done = torch.zeros(batch, dtype=torch.int32, device=device)

    def reset(self, slots, lengths, start_row=0):
        """``slots`` (host ints) start utterances of ``lengths`` frames (host ints or CUDA tensor) at chunk row
        ``start_row`` of the next push.  All checked before the first launch; none waits."""
        slots = check_slots(slots, self.batch)
        idx = to_device(torch.tensor(slots, dtype=torch.long), self.device)
        if not (torch.is_tensor(lengths) and lengths.is_cuda):
            lengths = torch.as_tensor(lengths, dtype=torch.int32)
            if lengths.numel() and int(lengths.min()) < 1:
                raise ValueError(f"streamer: lengths must be >= 1 frame, got {lengths.tolist()}")
            lengths = to_device(lengths, self.device)
        if lengths.numel() != len(slots):
            raise ValueError(f"streamer: expected {len(slots)} lengths, got {lengths.numel()}")
        self.lengths.index_copy_(0, idx, lengths.to(self.device, torch.int32).reshape(-1))
        self.frames_done.index_fill_(0, idx, -int(start_row))

    def mask(self, rows_per_frame, lag):
        """-> the KtStreamMask of a window of ``rows_per_frame`` rows per frame trailing by ``lag`` rows."""
        return KtStreamMask(ptr(self.lengths, True), ptr(self.frames_done, True), rows_per_frame, lag)

    def mask_advance(self, mask, window_buf, first, rows, frames):
        """One launch: zero the chunk rows [first, first + rows) outside each utterance, then frames_done += frames."""
        ops.call("kt_stream_mask_advance", ctypes.byref(mask), ptr(window_buf), self.batch, rows, window_buf.shape[2],
                 window_buf.shape[1], first, frames)


class Streamer:
    """What a streamer of a plan keeps besides its own steps: the plan's windows, the KtStreamWin of every step record
    with src / dst / resid / res_lag fields (others: None), and when ``masked`` the slots' utterances with one
    KtStreamMask per window of ``plan.lags``.  A subclass names its output window ``out`` and the frame axis ``f_axis``
    of the chunks it takes and returns (2: (B, C, f), 1: (B, f, C)).

    A push of f frames returns f frames' output rows, ``delay`` (the plan's) rows behind the pushed frames; a masked
    stream zeroes the rows outside each slot's utterance, those before its frame 0 included.  ``finish()`` pushes the
    ``drain_frames`` frames of zeros (``in_channels`` wide) that bring out the last ``delay`` rows."""

    out = f_axis = None

    def __init__(self, plan, batch, max_frames, device, what, masked, in_channels):
        self.plan = plan
        self._win = win = Windows(plan.windows, batch, max_frames, device, what)
        self.batch, self.max_frames, self.device, self.delay = win.batch, win.max_frames, win.device, plan.delay
        self.drain_frames = -(-self.delay // win.rate[self.out])
        self._places = [win.place(st.src, st.dst, st.resid, res_lag=st.res_lag) if hasattr(st, "res_lag") else None
                        for st in plan.steps]
        self._slots = self._masks = self._zeros = None
        if masked:
            self._slots = SlotUtterances(self.batch, self.device)
            self._masks = {name: self._slots.mask(win.rate[name], lag) for name, lag in plan.lags.items()}
        if self.drain_frames:
            self._zeros = torch.zeros(self.batch, self.max_frames, in_channels, device=self.device).movedim(1, self.f_axis)

    def _end_chunk(self, f):
        """After the steps of a chunk of f frames: zero the output rows outside each slot's utterance and advance its
        frames_done (masked only), then move every window's history (one launch each)."""
        win, out = self._win, self.out
        if self._slots is not None:
            self._slots.mask_advance(self._masks[out], win.buf[out], win.first[out], f * win.rate[out], f)
        win.advance(f)

    def _output(self, f):
        """-> a copy of the output window's rows of a chunk of f frames, frames on axis f_axis."""
        win, out = self._win, self.out
        rows = win.buf[out][:, win.first[out]:win.first[out] + f * win.rate[out]]
        return rows.movedim(1, self.f_axis).clone(memory_format=torch.contiguous_format)

    def finish(self):
        """Push ``drain_frames`` frames of zeros, at most max_frames at a time -> their output, which ends with the last
        row of every utterance pushed to its end (none without a delay)."""
        outs, left = [], self.drain_frames
        while left > 0:
            f = min(left, self.max_frames)
            outs.append(self.push(self._zeros.narrow(self.f_axis, 0, f)))
            left -= f
        return torch.cat(outs, self.f_axis) if outs else self._output(0)


def check_slots(slots, batch):
    """-> ``slots`` as a list of ints; ValueError unless they are distinct and lie in [0, batch)."""
    slots = [int(s) for s in slots]
    if len(set(slots)) != len(slots) or any(not 0 <= s < batch for s in slots):
        raise ValueError(f"reset: slots must be distinct and lie in [0, {batch}), got {slots}")
    return slots


def to_device(t, device):
    """A small host tensor on ``device`` without waiting for the device: staged in pinned memory and copied asynchronously
    (the pinned block is not reused before the copy has run), so that resetting a slot of a running stream does not
    synchronise the host."""
    return t.pin_memory().to(device, non_blocking=True)


def own_weight(spec, v, g, bias):
    """-> (a fresh PreparedWeight from copies of v and g, a copy of bias): a streamer's own weights, never the module's
    cache.  g and bias may be None."""
    copy = lambda t: None if t is None else t.detach().clone()
    return ops.prepare_weight(ops.PreparedWeight(), spec, copy(v), copy(g)), copy(bias)
