"""Streamed and served text-to-speech through non-causal vocoders on the GPU (``allow_lookahead=True``): every utterance's
audio equals the reference's hand-off, the generator run on exactly that utterance's post-net frames
(infer_sambert.py:136-138 then infer_hifigan.py; for NSF after denorm_f0, with the utterance's seed), for plain and NSF
generators, ragged batches, every chunk size and a server whose slots take new requests right after a vocoder drain;
starts are contiguous from 0 with no empty chunk, no host synchronisation while streaming, and a speaker-embedding model
streams and serves through the non-causal NSF-global generator it ships with."""
import contextlib
import math

import pytest
import torch

import kantts_b200 as K
from kantts_b200.infer import denorm_f0
from conftest import rel_l2
from test_gpu_sambert_se import _embeddings, _se_models
from test_gpu_tts_serve import ARRIVE, _requests
from test_gpu_tts_stream import _exact
from test_nsf_stream_cpu import STREAM_CONFIGS
from test_stream_cpu import CONFIGS

pytestmark = [pytest.mark.gpu]
DEV = "cuda"
MEAN_STD, GLOBAL = ("mean_std", 180.0, 40.0), ("global", 30.0, 730.0)


def _models(golden, nsf):
    """The small seeded SAM-BERT of the serving tests (post-net delay 3 = r) predicting 4 frames per symbol, so that
    utterances of some symbol counts are not a whole number of decoder steps, and the small non-causal generator (NSF
    with ``nsf``: 80 mel channels + f0 + uv)."""
    from test_gpu_tts_serve import _models as serve_models
    cfg, am, _ = serve_models(golden, num_mels=82 if nsf else None, nsf=nsf)
    with torch.no_grad():
        am.variance_adaptor.duration_predictor.fc.bias.fill_(math.log(4 + 1))
    torch.manual_seed(7)
    gcfg = STREAM_CONFIGS["small_nc"] if nsf else dict(CONFIGS["small"], in_channels=cfg["num_mels"], causal=False)
    return cfg, am, K.Generator(**gcfg).to(DEV).eval()


def _handoff(am, gen, inputs, nsf_f0=None, seeds=None):
    """-> [1-D waveform of the generator on exactly postnet_outputs[b, :LR_length_rounded[b]]] for the batch ``inputs``."""
    res = am(*inputs)
    wavs = []
    for b, n in enumerate(res["LR_length_rounded"].tolist()):
        mel = res["postnet_outputs"][b:b + 1, :n]
        if nsf_f0 is None:
            w = gen(mel.transpose(1, 2).contiguous())
        else:
            w = gen(denorm_f0(mel, nsf_f0).transpose(1, 2).contiguous(), nsf_seeds=seeds[b:b + 1])
        wavs.append(w[0, 0])
    return wavs


def _check(got, want, exact, what):
    """got / want: lists of 1-D waveforms.  The tolerances of test_gpu_stream_noncausal.py."""
    for i, (g, w) in enumerate(zip(got, want)):
        assert g.shape == w.shape, (what, i, g.shape, w.shape)
        g, w = g.cpu(), w.cpu()
        err, rel, rms = float((g - w).abs().max()), rel_l2(g, w), float((g - w).pow(2).mean().sqrt())
        print(f"{what} {i}: {w.shape[0]} samples, max |diff| {err:.3e}, rel L2 {rel:.3e}, RMS {rms:.3e}")
        if exact:
            assert err <= 1e-6, (what, i)
        else:
            assert rel <= 1e-4 and rms <= 1e-3, (what, i)


def _collect(stream):
    """-> [1-D audio of slot b, cut at lengths[b]], after checking the chunks' starts and sizes."""
    wavs, start = [], 0
    for s, w in stream:
        assert s == start and w.shape[:2] == (stream.batch, 1) and w.shape[2] > 0
        wavs.append(w)
        start += w.shape[2]
    wav = torch.cat(wavs, -1)
    assert wav.shape[-1] >= max(stream.lengths)
    return [wav[b, 0, :n] for b, n in enumerate(stream.lengths)]


def _batch(cfg, speakers=None):
    from golden.make_batch import make_sambert_batch
    b = make_sambert_batch(dict(cfg, speaker=1) if speakers is not None else cfg, B=3, L=9,
                           gen=torch.Generator().manual_seed(31))
    spk = b["inputs_speaker"].to(DEV) if speakers is None else speakers[:, None, :].expand(3, 9, speakers.shape[-1]).contiguous()
    return [b["inputs_ling"].to(DEV), b["inputs_emotion"].to(DEV), spk, torch.tensor([9, 7, 5], device=DEV)]   # ragged


# ---- lockstep streaming --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("chunk_steps", [1, 2, 4, 16])
@pytest.mark.parametrize("nsf", [False, True])
def test_stream_equals_the_handoff(golden, nsf, chunk_steps):
    cfg, am, gen = _models(golden, nsf)
    inputs = _batch(cfg)
    kw = dict(nsf_f0=MEAN_STD, nsf_seeds=[11, 12, 13]) if nsf else {}
    for exact in (True, False):
        with torch.no_grad(), (_exact() if exact else contextlib.nullcontext()):
            want = _handoff(am, gen, inputs, kw.get("nsf_f0"), kw.get("nsf_seeds"))
            st = K.stream_synthesize(am, gen, *inputs, chunk_steps=chunk_steps, allow_lookahead=True, **kw)
            got = _collect(st)
        frames = [n // st.hop for n in st.lengths]
        assert st.lookahead == 90 and len(set(frames)) > 1 and any(n % am.mel_decoder.r for n in frames), frames
        _check(got, want, exact, f"nsf={nsf} chunk_steps={chunk_steps} exact={exact} slot")


def test_stream_does_not_synchronise(golden):
    cfg, am, gen = _models(golden, True)
    inputs = _batch(cfg)
    with torch.no_grad():
        it = iter(K.stream_synthesize(am, gen, *inputs, chunk_steps=2, nsf_f0=MEAN_STD, nsf_seeds=[1, 2, 3],
                                      allow_lookahead=True))
        next(it)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            rest = list(it)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert len(rest) > 1


def test_causal_generator_streams_as_without_the_flag(golden):
    from test_gpu_tts_serve import _models as serve_models
    cfg, am, gen = serve_models(golden)
    inputs = _batch(cfg)
    with torch.no_grad(), _exact():
        a = list(K.stream_synthesize(am, gen, *inputs, chunk_steps=2))
        b = list(K.stream_synthesize(am, gen, *inputs, chunk_steps=2, allow_lookahead=True))
    assert [s for s, _ in a] == [s for s, _ in b]
    assert all(torch.equal(x, y) for (_, x), (_, y) in zip(a, b))


# ---- serving -------------------------------------------------------------------------------------------------------------
def _serve(server, reqs, arrive, seeds=None):
    """Submit reqs[i] at chunk arrive[i], step until idle -> ({request index: 1-D audio}, {index: chunk it was reported
    finished}, {index: chunk of its last audio}, {index: (slot, voc_chunk, last_chunk)})."""
    ids, audio, done, last, sched, c = {}, {}, {}, {}, {}, 0
    while len(ids) < len(reqs) or not server.idle:
        for i, (req, a) in enumerate(zip(reqs, arrive)):
            if a == c:
                ids[server.submit(*req, **({} if seeds is None else dict(nsf_seed=seeds[i])))] = i
        pieces, finished = server.step()
        for b, s in enumerate(server._slots):
            if s is not None:
                sched[ids[s["id"]]] = (b, s["voc_chunk"], s["last_chunk"])
        for rid, start, w in pieces:
            got = audio.setdefault(ids[rid], [])
            assert start == sum(x.shape[0] for x in got) and w.shape[0] > 0
            got.append(w)
            last[ids[rid]] = c
        for rid in finished:
            done[ids[rid]] = c
        c += 1
        assert c < 1000
    return {i: torch.cat(w) for i, w in audio.items()}, done, last, sched


def _alone(am, gen, req, nsf_f0=None, seed=None):
    ling, emo, spk, m = req
    inputs = [ling[None].to(DEV), emo[None].to(DEV), spk[None].to(DEV), torch.tensor([m], device=DEV)]
    return _handoff(am, gen, inputs, nsf_f0, None if seed is None else [seed])[0]


@pytest.mark.parametrize("slots,chunk_steps", [(3, 4), (3, 1), (1, 2), (2, 16)])
@pytest.mark.parametrize("nsf", [False, True])
def test_server_matches_the_handoff_alone(golden, nsf, slots, chunk_steps):
    cfg, am, gen = _models(golden, nsf)
    reqs = _requests(cfg)
    nsf_f0, seeds = (MEAN_STD, [101 + i for i in range(len(reqs))]) if nsf else (None, None)
    for exact in ((True, False) if slots == 3 and chunk_steps == 4 else (True,)):
        with torch.no_grad(), (_exact() if exact else contextlib.nullcontext()):
            want = [_alone(am, gen, r, nsf_f0, None if seeds is None else seeds[i]) for i, r in enumerate(reqs)]
            server = K.TtsServer(am, gen, slots=slots, chunk_steps=chunk_steps, max_steps=48, nsf_f0=nsf_f0,
                                 allow_lookahead=True)
            got, done, last, sched = _serve(server, reqs, ARRIVE, seeds)
        assert server.lookahead == 90 and server.delay == 3
        _check([got[i] for i in range(len(reqs))], want, exact,
               f"nsf={nsf} slots={slots} chunk_steps={chunk_steps} exact={exact} request")
        assert done == last                           # finished in the chunk of the last sample
        # a slot's vocoder is reset for its next request only after the previous one's last sample
        by_slot = {}
        for i, (b, v, l) in sorted(sched.items(), key=lambda kv: kv[1][1]):
            by_slot.setdefault(b, []).append((v, l))
        for runs in by_slot.values():
            assert all(v2 > l1 for (_, l1), (v2, _) in zip(runs, runs[1:]))
        if slots == 1:                                # requests queue: each follows the previous drain at once
            assert all(v2 == l1 + 1 for (_, l1), (v2, _) in zip(by_slot[0], by_slot[0][1:])), by_slot[0]
    assert len({w.shape[0] for w in want}) > 3


def test_server_does_not_synchronise_between_admissions(golden):
    cfg, am, gen = _models(golden, True)
    reqs = _requests(cfg, 3)
    server = K.TtsServer(am, gen, slots=3, chunk_steps=2, max_steps=48, nsf_f0=MEAN_STD, allow_lookahead=True)
    for i, r in enumerate(reqs):
        server.submit(*r, nsf_seed=i)
    with torch.no_grad():
        server.step()                                  # admits all three
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            pieces = []
            while not server.idle:
                pieces += server.step()[0]
        finally:
            torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert {rid for rid, _, _ in pieces} == {0, 1, 2}


# ---- speaker embeddings --------------------------------------------------------------------------------------------------
def test_se_model_streams_and_serves_through_the_nsf_global_generator(golden):
    cfg, am, se = _se_models(golden, num_mels=82)
    torch.manual_seed(7)
    gen = K.Generator(**STREAM_CONFIGS["small_nc"]).to(DEV).eval()
    emb = _embeddings(se, 4)
    seeds = [21, 22, 23, 24]
    with torch.no_grad(), _exact():
        inputs = _batch(cfg, emb[:3])
        want = _handoff(am, gen, inputs, GLOBAL, seeds[:3])
        st = K.stream_synthesize(am, gen, *inputs, chunk_steps=4, nsf_f0=GLOBAL, nsf_seeds=seeds[:3], allow_lookahead=True)
        got = _collect(st)
        _check(got, want, True, "SE stream slot")
        from golden.make_batch import make_sambert_batch
        lens, arrive = [9, 4, 7, 5], [0, 0, 1, 3]
        b = make_sambert_batch(dict(cfg, speaker=1), B=4, L=9, gen=torch.Generator().manual_seed(31))
        e = emb.cpu()
        reqs = [(b["inputs_ling"][i, :m], b["inputs_emotion"][i, :m], e[i][None].expand(m, 192).contiguous(), m)
                for i, m in enumerate(lens)]
        want = [_alone(am, gen, r, GLOBAL, s) for r, s in zip(reqs, seeds)]
        server = K.TtsServer(am, gen, slots=2, chunk_steps=4, max_steps=48, nsf_f0=GLOBAL, allow_lookahead=True)
        got, done, last, _ = _serve(server, reqs, arrive, seeds)
    _check([got[i] for i in range(4)], want, True, "SE request")
    assert done == last
