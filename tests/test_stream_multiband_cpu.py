"""CPU checks of streaming a multi-band generator (Generator.streamer with the PQMF attached as generator.pqmf): a float64
chunk-by-chunk restatement of the oracle's PQMF synthesis -- a window of (taps) // S sub-band rows, the output taps/2
samples late, each slot's input zero past its utterance -- equals the whole synthesis for every chunk schedule, alone and
behind the chunk-by-chunk generator restatements of test_stream_cpu / test_stream_noncausal_cpu; the plan's window,
hop, delay and launch count agree with it; and a multi-band generator without its PQMF, or with one of other sub-bands,
is refused by every streaming entry point."""
import types

import pytest
import torch
import torch.nn.functional as F

import kantts_b200 as K
from kantts_b200.hifigan import ConvStep, StreamPlan, stream_spec
from kantts_b200.infer import stream_lookahead
from oracle import hifigan as O
from oracle import pqmf as OP
from test_stream_cpu import CONFIGS, SCHEDULES, T, generator_stream
from test_stream_noncausal_cpu import LENGTHS, generator_stream_nc

# the small generator of test_stream_cpu with S sub-band outputs, and G_MB of scripts/multiband_step.py at reduced width
MB_CONFIGS = {
    "small4": dict(CONFIGS["small"], out_channels=4),
    "small2": dict(CONFIGS["small"], out_channels=2),
    "mb24k": dict(channels=32, out_channels=4, upsample_scales=[5, 3, 2, 2], upsample_kernal_sizes=[10, 6, 4, 4]),
}


def synthesis_stream(chunks, lengths, hs, subbands, taps, lag=0):
    """oracle.pqmf.synthesis restated chunk by chunk: chunks (B, S, rows) of sub-band rows that trail the utterance by ``lag``
    rows.  Each chunk runs over [history | chunk], history the last (taps) // S rows (zeros at the start), its rows outside
    [0, lengths[b]) of the utterance zeroed (the whole synthesis's zero padding, per slot).  Its output sample t is utterance
    sample (pushed - lag) * S - taps/2 + t, zero outside [0, lengths[b] * S).  -> (the concatenated waveform (B, 1, n), its
    lag in samples, the history in rows)."""
    S, H = subbands, taps // subbands
    lens = torch.tensor(lengths)
    up = OP._updown(S, torch.float64) * S
    hist, pushed, outs = None, 0, []
    for x in chunks:
        B, f = x.shape[0], x.shape[-1]
        full = torch.cat([x.new_zeros(B, S, H) if hist is None else hist, x], -1)
        hist = full[..., full.shape[-1] - H:]
        u = pushed - lag - H + torch.arange(H + f)
        full = full * ((u[None] >= 0) & (u[None] < lens[:, None]))[:, None]
        z = F.conv_transpose1d(full, up, stride=S)                     # zero stuffing: sample S * r is row r (times S)
        # output t reads stuffed samples t .. t + taps from the one at taps before the chunk's first sample
        z = F.pad(z, (max(0, taps - H * S), 0))[..., max(0, H * S - taps):]
        y = F.conv1d(z, hs)
        v = (pushed - lag) * S - taps // 2 + torch.arange(S * f)
        outs.append(y * ((v[None] >= 0) & (v[None] < lens[:, None] * S))[:, None])
        pushed += f
    return torch.cat(outs, -1), lag * S + taps // 2, H


def _chunks(x, schedule, rate, drain):
    """x (B, C, frames * rate) split into chunks of schedule[i] * rate rows, and ``drain`` rows of garbage after them"""
    return list(torch.split(x, [f * rate for f in schedule], -1)) + [torch.randn(x.shape[0], x.shape[1], drain,
                                                                                   dtype=x.dtype)]


@pytest.mark.parametrize("schedule", sorted(SCHEDULES))
@pytest.mark.parametrize("subbands,taps", [(4, 62), (4, 48), (2, 62)])
def test_oracle_synthesis_stream_equals_whole_synthesis(subbands, taps, schedule):
    _, hs = OP.filters(subbands, taps)
    rate = 3                                                           # sub-band rows per frame
    x = torch.randn(2, subbands, T * rate, generator=torch.Generator().manual_seed(subbands + taps), dtype=torch.float64)
    lengths = [n * rate for n in LENGTHS]
    drain = -(-(taps // 2) // subbands)
    got, lag, hist = synthesis_stream(_chunks(x, SCHEDULES[schedule], rate, drain), lengths, hs, subbands, taps)
    assert lag == taps // 2 and hist == (taps // subbands)
    for b, n in enumerate(lengths):
        want = OP.synthesis(x[b:b + 1, :, :n], hs, subbands, taps)
        out = got[b:b + 1, :, lag:lag + n * subbands]
        assert out.shape == want.shape
        assert float((out - want).abs().max()) <= 1e-12, (b, schedule)
        assert int(got[b, :, :lag].count_nonzero()) == 0 and int(got[b, :, lag + n * subbands:].count_nonzero()) == 0


def _mb(cfg, seed=3, taps=62):
    torch.manual_seed(seed)
    g = K.Generator(**cfg).eval()
    g.pqmf = K.PQMF(cfg["out_channels"], taps=taps)
    return g


@pytest.mark.parametrize("schedule", sorted(SCHEDULES))
@pytest.mark.parametrize("causal", [True, False], ids=["causal", "noncausal"])
@pytest.mark.parametrize("name", sorted(MB_CONFIGS))
def test_oracle_stream_equals_per_utterance_handoff(name, causal, schedule):
    """generator restatement -> synthesis restatement, chunk by chunk, against pqmf.synthesis(generator(mel_b[..., :n]))
    of the oracle, with the plan's delay and histories."""
    cfg = dict(MB_CONFIGS[name], causal=causal)
    g = _mb(cfg)
    plan = StreamPlan(g)
    S = cfg["out_channels"]
    sd = {k: v.detach().double() for k, v in g.state_dict().items()}
    _, hs = OP.filters(S)
    mel = torch.randn(2, 80, T, generator=torch.Generator().manual_seed(5), dtype=torch.float64)
    chunks = list(torch.split(mel, SCHEDULES[schedule], -1))
    chunks.append(torch.randn(2, 80, -(-plan.delay // plan.hop), dtype=torch.float64))
    gcfg = {k: v for k, v in cfg.items() if k != "out_channels"}
    if causal:
        sub, lag = generator_stream(sd, chunks, **gcfg)[0], 0
    else:
        sub, lag, _ = generator_stream_nc(sd, chunks, LENGTHS, **gcfg)
    rate = plan.hop // S
    assert lag == plan.lags["sub"] and sub.shape[1] == S
    got, delay, hist = synthesis_stream(list(torch.split(sub, [c.shape[-1] * rate for c in chunks], -1)),
                                        [n * rate for n in LENGTHS], hs, S, 62, lag)
    assert delay == plan.delay and hist == plan.layer_history["pqmf"]
    for b, n in enumerate(LENGTHS):
        want = OP.synthesis(O.generator_forward(sd, mel[b:b + 1, :, :n], **gcfg), hs, S)
        out = got[b:b + 1, :, delay:delay + n * plan.hop]
        assert out.shape == want.shape
        assert float((out - want).abs().max()) <= 1e-6, (name, schedule, b)
        assert int(got[b, :, :delay].count_nonzero()) == 0 and int(got[b, :, delay + n * plan.hop:].count_nonzero()) == 0


@pytest.mark.parametrize("subbands,taps,delay,hist", [(4, 62, 31, 15), (4, 48, 24, 12), (2, 62, 31, 31)])
def test_causal_plan(subbands, taps, delay, hist):
    cfg = dict(MB_CONFIGS["mb24k"], out_channels=subbands)
    g = _mb(cfg, taps=taps)
    plan = StreamPlan(g)
    full = StreamPlan(K.Generator(**dict(cfg, out_channels=1)).eval())
    assert plan.causal and plan.pqmf is g.pqmf
    assert plan.delay == delay and plan.hop == 60 * subbands
    assert -(-plan.delay // plan.hop) == 1                             # one drain frame
    win = {w["name"]: w for w in plan.windows}
    assert win["sub"] == dict(name="sub", channels=subbands, rows_per_frame=60, history=hist)
    assert win["wav"] == dict(name="wav", channels=1, rows_per_frame=60 * subbands, history=0)
    assert plan.layer_history["pqmf"] == hist
    # the generator's own layers stream as in the full-band plan: causal, no lags
    assert {k: v for k, v in plan.lags.items() if k not in ("sub", "wav")} == {k: v for k, v in full.lags.items()
                                                                               if k != "wav"}
    assert set(plan.lags.values()) == {0, delay}
    st = plan.steps[-1]
    assert type(st) is ConvStep and (st.src, st.dst, st.resid, st.side, st.res_lag) == ("sub", "wav", None, None, 0)
    assert st.spec == stream_spec(g.pqmf.synthesis_spec) and st.spec.pad_left == 0 and st.spec.crop == taps + 1 - subbands
    assert st.spec.t_out(7) == 7 * subbands
    assert st.conv.bias is None and st.conv.effective_weight()[0] is g.pqmf._weights()[1]
    assert plan.steps[-2].dst == "sub" and plan.steps[-2].spec is g.conv_post.conv1d.spec
    # + the synthesis conv and the output mask
    assert plan.launches_per_chunk == full.launches_per_chunk + 2


def test_noncausal_plan():
    """the small non-causal structure of test_gpu_stream_noncausal (full-band delay 90): 90 * 4 + 31 = 391 samples"""
    cfg = dict(MB_CONFIGS["small4"], causal=False)
    plan = StreamPlan(_mb(cfg))
    full = StreamPlan(K.Generator(**dict(cfg, out_channels=1)).eval())
    assert full.delay == 90 and plan.lags["sub"] == full.delay
    assert plan.delay == 391 and plan.hop == 32 and -(-plan.delay // plan.hop) == 13
    st = plan.steps[-1]
    assert st.spec == stream_spec(plan.pqmf.synthesis_spec, 90)
    assert plan.launches_per_chunk == full.launches_per_chunk + 1      # the output mask was there already


def test_refusals_without_the_matching_pqmf():
    sambert = types.SimpleNamespace(training=False)
    bare = K.Generator(**MB_CONFIGS["mb24k"]).eval()
    other = K.Generator(**MB_CONFIGS["mb24k"]).eval()
    other.pqmf = K.PQMF(2)
    for g in (bare, other):
        for call in (lambda: StreamPlan(g), lambda: g.streamer(batch=1, max_frames=4, lengths=[4]),
                     lambda: stream_lookahead(g, True, "streaming"),
                     lambda: K.stream_synthesize(sambert, g, None, None, None, None, allow_lookahead=True),
                     lambda: K.TtsServer(sambert, g, slots=1, chunk_steps=1, max_steps=8, allow_lookahead=True)):
            with pytest.raises(ValueError, match="multi-band"):
                call()
    with pytest.raises(ValueError, match="2"):
        StreamPlan(other)


def test_causal_multiband_streams_with_lengths_and_without_allow_lookahead():
    g = _mb(MB_CONFIGS["mb24k"])
    assert stream_lookahead(g, False, "streaming") == stream_lookahead(g, True, "streaming") == 31
    with pytest.raises(ValueError, match="multi-band generator needs per-slot lengths"):
        g.streamer(batch=1, max_frames=4)
    with pytest.raises(RuntimeError, match="CUDA"):                     # past the checks: no CPU fallback
        g.streamer(batch=1, max_frames=4, lengths=[4])
    nc = _mb(dict(MB_CONFIGS["mb24k"], causal=False))
    with pytest.raises(ValueError, match="causal.*allow_lookahead"):
        stream_lookahead(nc, False, "streaming")
