"""Streaming multi-band generators on the GPU (Generator.streamer with the PQMF attached as generator.pqmf): the PQMF
synthesis stage's stream conv against a float64 windowed reference; each slot's delayed chunks, cut to
[delay, delay + length * hop), equal the per-utterance hand-off pqmf.synthesis(generator(mel_b[..., :n])) for causal and
non-causal generators of 4 and 2 sub-bands, every chunk schedule and ragged lengths; graph replay equals eager; a reset
after draining touches one slot only; and stream_synthesize and TtsServer with a multi-band vocoder give every request
the hand-off's audio."""
import contextlib
import math

import pytest
import torch

import kantts_b200 as K
from kantts_b200 import ops
from kantts_b200.hifigan import stream_history, stream_spec
from conftest import rel_l2
from test_gpu_stream_conv import DEV, ELEM_BOUND, F64, L2_BOUND, Case, _Run, _mangled, _routes
from test_gpu_stream_noncausal import _schedule
from test_stream_cpu import CONFIGS, SCHEDULES

pytestmark = [pytest.mark.gpu]

# causal and non-causal multi-band generators whose whole forward runs on the GPU (every deconv with k - s even)
MB_CONFIGS = {
    "small4": dict(CONFIGS["small"], out_channels=4),
    "small2": dict(CONFIGS["small"], out_channels=2),
    "small4_nc": dict(CONFIGS["small"], out_channels=4, causal=False),
    "small2_nc": dict(CONFIGS["small"], out_channels=2, causal=False),
}
LENGTHS = [23, 17]


# ---- the synthesis stage's stream conv -----------------------------------------------------------------------------------
def _synthesis_case(subbands, masked, lag):
    spec = stream_spec(K.PQMF(subbands).synthesis_spec)
    rpf = 60                                                           # sub-band rows per frame of the 24 kHz structure
    return Case(f"pqmf{subbands}{'_masked' if masked else ''}", spec, t_in=16 * rpf, hist=stream_history(spec),
                B=8 if masked else 2, masked=masked, rpf=rpf, lag=lag)


@pytest.mark.parametrize("masked,lag", [(False, 0), (True, 0), (True, 45)], ids=["plain", "masked", "masked_lag45"])
@pytest.mark.parametrize("subbands", [4, 2])
def test_synthesis_stream_conv_matches_float64(subbands, masked, lag):
    """The causal form of PQMF.synthesis_spec (taps + 1 = 63 taps, stride S, crop k - s) in one chunk of 16 frames with
    the history it reads, on the exact route and the route the plan picks; masked: every slot in its own utterance state."""
    c = _synthesis_case(subbands, masked, lag)
    assert c.hist == 62 // subbands and c.spec.t_out(c.t_in) == subbands * c.t_in
    run = _Run(c)
    fill = float("nan") if masked else None
    want, scale = run.reference()
    try:
        for route, force, kernels in _routes(c):
            ops.set_force_ffma(force)
            y, untouched = run(fill)
            assert untouched, (route, "wrote outside its output chunk or changed an input")
            convs = [k for k in run(fill, capture=True) if "conv_core_kernelI" in k or "conv_tc_kernelI" in k]
            named = [_mangled(k) for k in kernels]
            assert all(any(w in k for k in convs) for w in named) and all(any(w in k for w in named) for k in convs), \
                (route, kernels, convs)
            if masked:                                     # rows outside the utterances are never read
                y_zero, ok = run(0.0)
                y_plain, ok2 = run(0.0, masked=False)
                assert ok and ok2
                assert torch.equal(y.view(torch.int32), y_zero.view(torch.int32)), route
                assert torch.equal(y.view(torch.int32), y_plain.view(torch.int32)), route
            err = (y.to(F64) - want).abs()
            ratio = float((err / scale.clamp_min(1e-300)).max())
            l2 = rel_l2(y, want)
            print(f"pqmf{subbands} masked={masked} lag={lag} {route} {' '.join(kernels)} elem {ratio:.3e} rel_l2 {l2:.3e}")
            assert bool((err <= ELEM_BOUND[route] * scale).all()), (route, ratio)
            assert l2 <= L2_BOUND[route], (route, l2)
    finally:
        ops.set_force_ffma(False)


# ---- generator + synthesis streams ---------------------------------------------------------------------------------------
def _setup(name, B=2, T=23, seed=3):
    torch.manual_seed(seed)
    cfg = MB_CONFIGS[name]
    g = K.Generator(**cfg).eval()
    g.pqmf = K.PQMF(cfg["out_channels"])
    mel = torch.randn(B, 80, T, generator=torch.Generator().manual_seed(5))
    return g, mel


def _stream(g, mel, schedule, lengths, max_frames=None):
    st = g.streamer(batch=mel.shape[0], max_frames=max_frames or max(schedule), lengths=lengths)
    outs = [st.push(c) for c in torch.split(mel, schedule, -1)] + [st.finish()]
    return torch.cat(outs, -1), st


def _handoff(g, x, lengths):
    return [g.pqmf.synthesis(g(x[b:b + 1, :, :n])) for b, n in enumerate(lengths)]


def _cut(wav, st, lengths):
    return [wav[b:b + 1, :, st.delay:st.delay + n * st.hop] for b, n in enumerate(lengths)]


@pytest.mark.parametrize("schedule", sorted(SCHEDULES))
@pytest.mark.parametrize("name", sorted(MB_CONFIGS))
def test_stream_equals_per_utterance_handoff(name, schedule):
    from oracle import hifigan as O
    from oracle import pqmf as OP
    g, mel = _setup(name)
    S = MB_CONFIGS[name]["out_channels"]
    sched = _schedule(schedule, mel.shape[-1])
    sd = {k: v.detach().double() for k, v in g.state_dict().items()}
    _, hs = OP.filters(S)
    wav_o = [OP.synthesis(O.generator_forward(sd, mel[b:b + 1, :, :n].double(), **MB_CONFIGS[name]), hs, S)
             for b, n in enumerate(LENGTHS)]
    g, x = g.cuda(), mel.cuda()
    g.pqmf = g.pqmf.cuda()
    with torch.no_grad():
        ops.set_force_ffma(True)
        try:
            want = _handoff(g, x, LENGTHS)
            wav, st = _stream(g, x, sched, LENGTHS)
        finally:
            ops.set_force_ffma(False)
        assert st.hop == 8 * S and st.delay == (31 if g.conv_pre.causal else 90 * S + 31)
        got = _cut(wav, st, LENGTHS)
        err = max(float((a - b).abs().max()) for a, b in zip(got, want))
        print(f"{name}/{schedule} exact path: delay {st.delay}, max |stream - hand-off| = {err:.3e} "
              f"(bitwise equal: {err == 0.0})")
        assert all(a.shape == b.shape for a, b in zip(got, want)) and err <= 1e-6
        for b, n in enumerate(LENGTHS):                                 # outside the utterance: zeros
            assert int(wav[b, :, :st.delay].count_nonzero()) == 0
            assert int(wav[b, :, st.delay + n * st.hop:].count_nonzero()) == 0
        want = _handoff(g, x, LENGTHS)
        wav, st = _stream(g, x, sched, torch.tensor(LENGTHS, device="cuda"))
        for a, w, o in zip(_cut(wav, st, LENGTHS), want, wav_o):
            rel, rms = rel_l2(a.cpu(), w.cpu()), float((a.cpu().double() - o).pow(2).mean().sqrt())
            print(f"{name}/{schedule} bf16x3 path: rel L2 {rel:.3e}, RMS against float64 {rms:.3e}")
            assert rel <= 1e-4 and rms <= 1e-3


def test_graph_replay_equals_eager_bitwise():
    g, mel = _setup("small4", T=14)
    g, mel = g.cuda(), mel.cuda()
    g.pqmf = g.pqmf.cuda()
    sched = [4, 4, 4, 2]
    with torch.no_grad():
        graphed, st = _stream(g, mel, sched, [14, 9], max_frames=4)     # replayed full chunks, eager tails
        eager, _ = _stream(g, mel, sched, [14, 9], max_frames=5)        # every chunk eager
    assert graphed.shape == eager.shape and graphed.shape[-1] >= (14 + st.drain_frames) * st.hop
    assert torch.equal(graphed, eager)


@pytest.mark.parametrize("name", ["small4", "small2_nc"])
def test_reset_after_drain_starts_an_exact_utterance_in_one_slot_only(name):
    g, a = _setup(name, B=3, T=12)
    u = torch.randn(1, a.shape[1], 9, generator=torch.Generator().manual_seed(9))
    g, a, u = g.cuda(), a.cuda(), u.cuda()
    g.pqmf = g.pqmf.cuda()
    with torch.no_grad():
        ops.set_force_ffma(True)
        try:
            want_a = _handoff(g, a, [12, 12, 12])
            want_u = g.pqmf.synthesis(g(u))
            st = g.streamer(batch=3, max_frames=4, lengths=[12, 12, 12])
            first = torch.cat([st.push(a[:, :, t:t + 4]) for t in (0, 4, 8)] + [st.finish()], -1)
            st.reset([1], [9])
            pad = torch.zeros(3, a.shape[1], 12, device="cuda")
            pad[1, :, :9] = u[0]
            second = torch.cat([st.push(pad[:, :, t:t + 4]) for t in (0, 4, 8)] + [st.finish()], -1)
        finally:
            ops.set_force_ffma(False)
    L, hop = st.delay, st.hop
    for b in range(3):
        assert float((first[b:b + 1, :, L:L + 12 * hop] - want_a[b]).abs().max()) <= 1e-6
    assert float((second[1:2, :, L:L + 9 * hop] - want_u).abs().max()) <= 1e-6
    for b in (0, 2):                                   # drained slots keep streaming silence past their utterance
        assert int(second[b].count_nonzero()) == 0


# ---- text-to-speech ------------------------------------------------------------------------------------------------------
def _tts_models(golden, causal):
    """The small seeded SAM-BERT of the serving tests (4 frames per symbol) and the small multi-band generator of 4
    sub-bands with its PQMF."""
    from test_gpu_tts_serve import _models as serve_models
    cfg, am, _ = serve_models(golden)
    with torch.no_grad():
        am.variance_adaptor.duration_predictor.fc.bias.fill_(math.log(4 + 1))
    torch.manual_seed(7)
    gen = K.Generator(**dict(CONFIGS["small"], in_channels=cfg["num_mels"], out_channels=4, causal=causal)).to(DEV).eval()
    gen.pqmf = K.PQMF(4).to(DEV)
    return cfg, am, gen


def _tts_handoff(am, gen, inputs):
    """-> [1-D waveform of pqmf.synthesis(generator) on exactly postnet_outputs[b, :LR_length_rounded[b]]]"""
    res = am(*inputs)
    return [gen.pqmf.synthesis(gen(res["postnet_outputs"][b:b + 1, :n].transpose(1, 2).contiguous()))[0, 0]
            for b, n in enumerate(res["LR_length_rounded"].tolist())]


@pytest.mark.parametrize("chunk_steps", [1, 4])
@pytest.mark.parametrize("causal", [True, False], ids=["causal", "noncausal"])
def test_stream_synthesize_equals_the_handoff(golden, causal, chunk_steps):
    from test_gpu_tts_lookahead import _batch, _check, _collect
    from test_gpu_tts_stream import _exact
    cfg, am, gen = _tts_models(golden, causal)
    inputs = _batch(cfg)
    for exact in (True, False):
        with torch.no_grad(), (_exact() if exact else contextlib.nullcontext()):
            want = _tts_handoff(am, gen, inputs)
            # a causal multi-band vocoder streams without allow_lookahead: its look-ahead is the synthesis's 31 samples
            st = K.stream_synthesize(am, gen, *inputs, chunk_steps=chunk_steps, allow_lookahead=not causal)
            got = _collect(st)
        assert st.hop == 32 and st.lookahead == (31 if causal else 391)
        _check(got, want, exact, f"causal={causal} chunk_steps={chunk_steps} exact={exact} slot")


@pytest.mark.parametrize("slots,chunk_steps", [(3, 4), (1, 2)])
@pytest.mark.parametrize("causal", [True, False], ids=["causal", "noncausal"])
def test_server_matches_the_handoff_alone(golden, causal, slots, chunk_steps):
    from test_gpu_tts_lookahead import _check, _serve
    from test_gpu_tts_serve import ARRIVE, _requests
    from test_gpu_tts_stream import _exact
    cfg, am, gen = _tts_models(golden, causal)
    reqs = _requests(cfg)
    for exact in ((True, False) if slots == 3 else (True,)):
        with torch.no_grad(), (_exact() if exact else contextlib.nullcontext()):
            want = []
            for ling, emo, spk, m in reqs:
                one = [ling[None].to(DEV), emo[None].to(DEV), spk[None].to(DEV), torch.tensor([m], device=DEV)]
                want.append(_tts_handoff(am, gen, one)[0])
            server = K.TtsServer(am, gen, slots=slots, chunk_steps=chunk_steps, max_steps=48, allow_lookahead=not causal)
            got, done, last, _ = _serve(server, reqs, ARRIVE)
        assert server.hop == 32 and server.lookahead == (31 if causal else 391)
        _check([got[i] for i in range(len(reqs))], want, exact,
               f"causal={causal} slots={slots} chunk_steps={chunk_steps} exact={exact} request")
        assert done == last
