"""Continuous-batching text-to-speech on the GPU: kt_pnca_step_slots equals plain torch attention over each slot's bands;
the slot decoder gives each utterance's batch-1 infer_steps rows with staggered starts; the post-net with staggered slot
resets gives each slot the rows of that utterance streamed alone, bit for bit; TtsServer gives every request
synthesize()'s audio of that request alone, bit for bit whether the other slots are busy or idle, for plain and NSF
generators, without synchronising between admissions."""
import pytest
import torch

import kantts_b200 as K
from kantts_b200.sambert import PostNet
from conftest import rel_l2
from test_gpu_tts_stream import _exact

pytestmark = [pytest.mark.gpu]
DEV = "cuda"


# ---- kt_pnca_step_slots -------------------------------------------------------------------------------------------------
class _State:
    def __init__(self, **kw):
        for k, v in kw.items():
            setattr(self, k, torch.tensor(v, device=DEV, dtype=torch.uint8 if k == "active" else torch.int32))


def _attend(q, k, v):
    p = torch.softmax(q @ k.T / q.shape[-1] ** 0.5, -1)
    return p @ v


@pytest.mark.parametrize("d_head", [8, 16, 32])
def test_pnca_step_slots_matches_torch(d_head):
    B, H, L = 5, 3, 40
    hd = H * d_head
    g = torch.Generator().manual_seed(4)
    q_row = torch.randn(B, 1, 3 * hd, generator=g).to(DEV)
    x_kv = torch.randn(B, L, 2 * hd, generator=g).to(DEV)
    h_kv = torch.randn(B, L, 2 * hd, generator=g).to(DEV)
    # slot 0 at step 0; slot 2's memory band runs past its memory end; slot 3 is inactive; slot 4 has a band wider than 32
    st = _State(step=[0, 7, 17, 5, 39], mem_len=[12, 30, 19, 20, 40], x_bw=[3, 4, 6, 2, 35], h_bw=[3, 4, 6, 2, 37],
                active=[1, 1, 1, 0, 1])
    x0 = x_kv.clone()
    ox, oh = K.sambert_ops.pnca_step_slots(q_row, x_kv, h_kv, st, H)
    torch.cuda.synchronize()
    for b in range(B):
        s, ml, xb, hb = (int(t[b]) for t in (st.step, st.mem_len, st.x_bw, st.h_bw))
        if not st.active[b]:
            assert torch.equal(x_kv[b], x0[b])
            assert torch.equal(ox[b], torch.zeros_like(ox[b])) and torch.equal(oh[b], torch.zeros_like(oh[b]))
            continue
        want_kv = x0[b].clone()
        want_kv[s] = q_row[b, 0, hd:]
        assert torch.equal(x_kv[b], want_kv)                    # the step's K / V row, nothing else
        for h in range(H):
            sl = slice(h * d_head, (h + 1) * d_head)
            q = q_row[b, 0, sl].double()
            lo = max(0, s - xb)
            kx, vx = want_kv[lo:s + 1, sl].double(), want_kv[lo:s + 1, hd + h * d_head: hd + (h + 1) * d_head].double()
            hi = min(s + hb, ml - 1)
            kh, vh = h_kv[b, s:hi + 1, sl].double(), h_kv[b, s:hi + 1, hd + h * d_head: hd + (h + 1) * d_head].double()
            assert rel_l2(ox[b, 0, sl], _attend(q, kx, vx)) <= 1e-6, (b, h)
            assert rel_l2(oh[b, 0, sl], _attend(q, kh, vh)) <= 1e-6, (b, h)


# ---- models ---------------------------------------------------------------------------------------------------------------
def _models(golden, num_mels=None, nsf=False):
    """The small seeded SAM-BERT of the streaming tests with three post-net FSMN layers (delay 3 = r) and ~3.5 frames per
    symbol, and a small causal generator (NSF with ``nsf``)."""
    from test_stream_cpu import CONFIGS
    from test_nsf_stream_cpu import NSF16
    g = golden("sambert_small_infer")
    cfg = dict(g.cfg, postnet_fsmn_num_layers=3)
    if num_mels:
        cfg["num_mels"] = num_mels
    torch.manual_seed(1234)
    am = K.KanTtsSAMBERT(cfg)
    with torch.no_grad():
        am.variance_adaptor.duration_predictor.fc.bias.fill_(1.5)
    am = am.to(DEV).eval()
    torch.manual_seed(7)
    gcfg = dict(CONFIGS["small"], nsf_params=NSF16) if nsf else dict(
        in_channels=cfg["num_mels"], channels=32, upsample_scales=[4, 2], upsample_kernal_sizes=[8, 4],
        resblock_kernel_sizes=[3, 7], resblock_dilations=[[1, 3], [1, 3]])
    return cfg, am, K.Generator(**gcfg).to(DEV).eval()


LENS = [9, 4, 7, 2, 9, 5, 8]
ARRIVE = [0, 0, 1, 1, 3, 6, 6]                       # chunk at which each request is submitted


def _requests(cfg, n=len(LENS)):
    from golden.make_batch import make_sambert_batch
    b = make_sambert_batch(cfg, B=n, L=max(LENS), gen=torch.Generator().manual_seed(31))
    return [(b["inputs_ling"][i, :m], b["inputs_emotion"][i, :m], b["inputs_speaker"][i, :m], m)
            for i, m in enumerate(LENS[:n])]


def _alone(am, gen, req, **kw):
    ling, emo, spk, m = req
    wavs, res = K.synthesize(am, gen, ling[None].to(DEV), emo[None].to(DEV), spk[None].to(DEV), torch.tensor([m], device=DEV),
                             **kw)
    return wavs[0], res


def _serve(server, reqs, arrive, seeds=None):
    """Submit reqs[i] at chunk arrive[i], step until idle -> {request index: 1-D audio}."""
    ids, audio, c = {}, {}, 0
    while len(ids) < len(reqs) or not server.idle:
        for i, (req, a) in enumerate(zip(reqs, arrive)):
            if a == c:
                ids[server.submit(*req, **({} if seeds is None else dict(nsf_seed=seeds[i])))] = i
        pieces, _ = server.step()
        for rid, start, w in pieces:
            got = audio.setdefault(ids[rid], [])
            assert start == sum(x.shape[0] for x in got)
            got.append(w)
        c += 1
        assert c < 500
    return {i: torch.cat(w) for i, w in audio.items()}


# ---- slot decoder --------------------------------------------------------------------------------------------------------
def test_slot_decoder_matches_batch1_infer_steps(golden):
    cfg, am, _ = _models(golden)
    reqs = _requests(cfg, 4)
    dec = am.mel_decoder
    with torch.no_grad(), _exact():
        fronts = [am.front_half(r[0][None].to(DEV), r[1][None].to(DEV), r[2][None].to(DEV), torch.tensor([r[3]], device=DEV))
                  for r in reqs]
        for f in fronts:
            assert int(f["band_width_rows"][0]) == f["x_band_width"]
        # the seeded model predicts about the same duration for every symbol: give the utterances different bands
        bands = [f["x_band_width"] + k for f, k in zip(fronts, (0, 2, 5, 1))]
        want = [torch.cat([o for o, _, _ in dec.infer_steps(f["memory"], w, w)], 1) for f, w in zip(fronts, bands)]
        assert len({w.shape[1] for w in want}) > 1
        sd = dec.slots(3, 40)
        start = [0, 3, 5]                              # staggered; request 3 follows request 1 in slot 1 at once
        got = {i: [] for i in range(4)}
        holder = {}
        for t in range(60):
            for i, s in enumerate(start):
                if s == t:
                    sd.admit(i, fronts[i]["memory"], fronts[i]["band_width_rows"] + (bands[i] - fronts[i]["x_band_width"]))
                    sd.start(i)
                    holder[i] = (i, t)
            if t == start[1] + want[1].shape[1]:       # the step after request 1's last: its go frame must be zeros
                sd.admit(1, fronts[3]["memory"], bands[3])
                sd.start(1)
                holder[1] = (3, t)
            out = sd.advance()
            for b, (i, t0) in holder.items():
                if t - t0 < want[i].shape[1]:
                    got[i].append(out[b:b + 1])
                elif t - t0 < want[i].shape[1] + 2:
                    assert torch.equal(out[b], torch.zeros_like(out[b]))          # finished: zero rows
    for i in range(4):
        g = torch.cat(got[i], 1)
        err = rel_l2(g.cpu(), want[i].cpu())
        print(f"utterance {i}: {want[i].shape[1]} steps, band {bands[i]}, rel err {err:.3e}")
        assert err <= 1e-5


# ---- post-net slot resets ------------------------------------------------------------------------------------------------
def test_postnet_slot_resets_give_each_utterance_its_rows_alone_bitwise():
    torch.manual_seed(3)
    pn = PostNet(K.sambert_24k_config()).to(DEV).eval()
    lens, starts, T = [30, 7, 22], [0, 5, 13], 30
    g = torch.Generator().manual_seed(5)
    dec = [torch.randn(1, n, 80, generator=g).to(DEV) for n in lens]
    chunks = [4, 7, 1, 9, 12, 3, 12, 12, 12]
    total = sum(chunks)
    with torch.no_grad(), _exact():
        st = pn.streamer(3, max(chunks), torch.zeros(3, dtype=torch.int32, device=DEV))
        rows = torch.zeros(3, total, 80, device=DEV)
        for b in range(3):
            rows[b, starts[b]:starts[b] + lens[b]] = dec[b][0]
        outs, r0 = [], 0
        for f in chunks:
            for b in range(3):
                if r0 <= starts[b] < r0 + f:
                    st.reset([b], [lens[b]], start_row=starts[b] - r0)
            outs.append(st.push(rows[:, r0:r0 + f]))
            r0 += f
        got = torch.cat(outs, 1)
        assert got.shape == (3, total, 80)
        for b in range(3):
            one = pn.streamer(1, 6, torch.tensor([lens[b]], device=DEV))
            want = torch.cat([one.push(c) for c in torch.split(dec[b], 6, 1)] + [one.finish()], 1)
            assert want.shape[1] == one.delay + lens[b]
            assert torch.equal(want[:, :one.delay], torch.zeros_like(want[:, :one.delay]))     # the rows before frame 0
            want = want[:, one.delay:]
            first = starts[b] + st.delay                 # output row of frame 0
            assert torch.equal(got[b, first:first + lens[b]], want[0]), b
            assert torch.equal(got[b, :first], torch.zeros_like(got[b, :first]))
            assert torch.equal(got[b, first + lens[b]:], torch.zeros_like(got[b, first + lens[b]:]))


def test_rejected_postnet_slot_reset_leaves_the_stream_as_it_was():
    torch.manual_seed(3)
    pn = PostNet(K.sambert_24k_config()).to(DEV).eval()
    rows = torch.randn(2, 24, 80, generator=torch.Generator().manual_seed(5)).to(DEV)
    outs = {}
    with torch.no_grad(), _exact():
        for rejected in (False, True):
            st = pn.streamer(2, 8, torch.zeros(2, dtype=torch.int32, device=DEV))
            st.reset([0, 1], [20, 13], start_row=0)
            got = [st.push(rows[:, :8])]
            if rejected:
                with pytest.raises(ValueError, match="distinct"):
                    st.reset([1, 1], [5, 5], start_row=2)
                with pytest.raises(ValueError, match="start_row"):
                    st.reset([1], [5], start_row=8)
            got += [st.push(rows[:, t:t + 8]) for t in (8, 16)]
            outs[rejected] = torch.cat(got, 1)
    assert torch.equal(outs[True], outs[False])


# ---- server --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("chunk_steps", [1, 3, 4])
def test_server_matches_synthesize_alone_and_isolates_slots(golden, chunk_steps):
    cfg, am, gen = _models(golden)
    reqs = _requests(cfg)
    with torch.no_grad(), _exact():
        want = [_alone(am, gen, r)[0] for r in reqs]
        got = _serve(K.TtsServer(am, gen, slots=3, chunk_steps=chunk_steps, max_steps=48), reqs, ARRIVE)
        alone = {i: _serve(K.TtsServer(am, gen, slots=3, chunk_steps=chunk_steps, max_steps=48), [reqs[i]], [0])[0]
                 for i in (0, 3, 6)}
    assert len({w.shape[0] for w in want}) > 3
    for i, w in enumerate(want):
        assert got[i].shape == w.shape, i
        err = rel_l2(got[i].cpu(), w.cpu())
        print(f"chunk_steps {chunk_steps} request {i}: {w.shape[0]} samples, rel err vs synthesize {err:.3e}")
        assert err <= 1e-5
    for i, w in alone.items():
        assert torch.equal(got[i], w), i
    # the tensor-core path, within the tolerance of the streaming tests
    with torch.no_grad():
        want = [_alone(am, gen, r)[0] for r in reqs]
        got = _serve(K.TtsServer(am, gen, slots=3, chunk_steps=chunk_steps, max_steps=48), reqs, ARRIVE)
    for i, w in enumerate(want):
        assert got[i].shape == w.shape and rel_l2(got[i].cpu(), w.cpu()) <= 1e-4, i


def test_server_with_an_nsf_generator_matches_synthesize_alone(golden):
    cfg, am, gen = _models(golden, num_mels=82, nsf=True)
    reqs = _requests(cfg)
    nsf_f0, seeds = ("mean_std", 180.0, 40.0), [101 + i for i in range(len(reqs))]
    with torch.no_grad(), _exact():
        want = [_alone(am, gen, r, nsf_f0=nsf_f0, nsf_seeds=[s])[0] for r, s in zip(reqs, seeds)]
        got = _serve(K.TtsServer(am, gen, slots=3, chunk_steps=4, max_steps=48, nsf_f0=nsf_f0), reqs, ARRIVE, seeds)
    for i, w in enumerate(want):
        err = rel_l2(got[i].cpu(), w.cpu())
        print(f"NSF request {i}: {w.shape[0]} samples, rel err {err:.3e}")
        assert got[i].shape == w.shape and err <= 1e-5


def test_server_rejects_a_request_longer_than_max_steps(golden):
    cfg, am, gen = _models(golden)
    reqs = _requests(cfg, 2)
    server = K.TtsServer(am, gen, slots=2, chunk_steps=2, max_steps=4)
    server.submit(*reqs[0])
    with torch.no_grad(), pytest.raises(ValueError, match="max_steps"):
        server.step()


def test_server_does_not_synchronise_between_admissions(golden):
    cfg, am, gen = _models(golden)
    reqs = _requests(cfg, 3)
    server = K.TtsServer(am, gen, slots=3, chunk_steps=2, max_steps=48)
    for r in reqs:
        server.submit(*r)
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
