"""Streamed text-to-speech on the GPU: the post-net streamer equals PostNet.forward, its two kernels equal their
whole-sequence counterparts, and stream_synthesize gives synthesize()'s waveforms chunk by chunk (bit for bit across chunk
sizes on the exact path) without synchronising the host."""
import ctypes

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import kantts_b200 as K
from kantts_b200 import _lib, ops
from kantts_b200._lib import KtStreamMask, KtStreamWin, check, ptr, stream_ptr
from kantts_b200.sambert import PostNet
from conftest import rel_l2
from test_tts_stream_cpu import LENGTHS, SCHEDULES, T
from oracle import sambert as O

pytestmark = [pytest.mark.gpu]
DEV = "cuda"


class _exact:
    """The exact-fp32 path: every conv on the FFMA kernels, nn.LSTM without cuDNN."""

    def __enter__(self):
        ops.set_force_ffma(True)
        self.cudnn = torch.backends.cudnn.flags(enabled=False)
        self.cudnn.__enter__()

    def __exit__(self, *exc):
        self.cudnn.__exit__(*exc)
        ops.set_force_ffma(False)


def _postnet_case():
    torch.manual_seed(3)
    pn = PostNet(K.sambert_24k_config()).to(DEV).eval()
    lengths = torch.tensor(LENGTHS, device=DEV)
    mask = torch.arange(T, device=DEV)[None, :] >= lengths[:, None]
    dec = torch.randn(len(LENGTHS), T, 80, generator=torch.Generator().manual_seed(5)).to(DEV)
    return pn, dec.masked_fill(mask.unsqueeze(-1), 0), lengths, mask


def _stream_postnet(pn, dec, lengths, schedule):
    """-> the streamed rows from frame 0 on, after checking that every push returns its f rows, the first ``delay`` (before
    frame 0) zero."""
    st = pn.streamer(batch=dec.shape[0], max_frames=max(schedule), lengths=lengths)
    outs = [st.push(c) for c in torch.split(dec, schedule, 1)]
    assert [o.shape[1] for o in outs] == list(schedule)
    got = torch.cat(outs + [st.finish()], 1)
    assert got.shape[1] == T + st.delay
    assert torch.equal(got[:, :st.delay], torch.zeros_like(got[:, :st.delay]))
    return got[:, st.delay:]


@pytest.mark.parametrize("schedule", sorted(SCHEDULES))
def test_postnet_streamer_rows_from_frame_0_match_forward(schedule):
    pn, dec, lengths, mask = _postnet_case()
    with torch.no_grad():
        with _exact():
            want = pn(dec, mask, resid=dec).masked_fill(mask.unsqueeze(-1), 0)
            got = _stream_postnet(pn, dec, lengths, SCHEDULES[schedule])
        assert got.shape == want.shape
        err = rel_l2(got.cpu(), want.cpu())
        print(f"{schedule}: exact path rel err {err:.3e}")
        assert err <= 2e-6
        want = pn(dec, mask, resid=dec).masked_fill(mask.unsqueeze(-1), 0)
        got = _stream_postnet(pn, dec, lengths, SCHEDULES[schedule])
        assert rel_l2(got.cpu(), want.cpu()) <= 1e-4


def test_postnet_streamer_reset_of_every_slot_starts_a_new_batch():
    pn, dec, lengths, mask = _postnet_case()
    other = torch.randn(dec.shape, generator=torch.Generator().manual_seed(8)).to(DEV)
    with torch.no_grad():
        st = pn.streamer(batch=dec.shape[0], max_frames=6, lengths=lengths)
        first = torch.cat([st.push(c) for c in torch.split(dec, 6, 1)] + [st.finish()], 1)
        slots = range(dec.shape[0])
        st.reset(slots, lengths)
        again = torch.cat([st.push(c) for c in torch.split(dec, 6, 1)] + [st.finish()], 1)
        # a batch cut off mid-stream leaves its rows in every window and its LSTM state carried: a reset clears neither
        st.reset(slots, torch.full_like(lengths, T))
        for c in torch.split(other[:, :16], 6, 1):
            st.push(c)
        st.reset(slots, lengths)
        after = torch.cat([st.push(c) for c in torch.split(dec, 6, 1)] + [st.finish()], 1)
    assert torch.equal(first[:, :st.delay], torch.zeros_like(first[:, :st.delay]))      # the rows before frame 0
    assert torch.equal(first, again)
    assert torch.equal(first, after)                  # first: the output of a fresh streamer


def test_fsmn_stream_slots_masked_rows_equal_whole_sequence_rows_bitwise():
    lib = _lib.load()
    B, C, K_, lp = 3, 96, 41, 37
    rp = K_ - 1 - lp
    g = torch.Generator().manual_seed(7)
    x = torch.randn(B, T, C, generator=g).to(DEV)
    w = (0.2 * torch.randn(C, K_, generator=g)).to(DEV)
    resid = torch.randn(B, T, C, generator=g).to(DEV)
    lengths = torch.tensor(LENGTHS, device=DEV, dtype=torch.int32)
    mask = (torch.arange(T, device=DEV)[None, :] >= lengths[:, None]).to(torch.uint8)
    y = torch.empty_like(x)
    done = torch.zeros(B, dtype=torch.int32, device=DEV)
    m = KtStreamMask(lengths=ptr(lengths, True), frames_done=ptr(done, True), rows_per_frame=1, lag=0)
    check(lib.kt_fsmn_fwd(ptr(x), ptr(w), ptr(mask, True), ptr(y), B, T, C, K_, lp, stream_ptr()), "kt_fsmn_fwd")
    # one window holding the whole input after k - 1 history rows (zeros), and rp padding rows at the end; the outputs are
    # frames -rp .. T-1 (the first rp rows are before the utterance)
    xw = torch.cat([x.new_zeros(B, K_ - 1, C), x, x.new_zeros(B, rp, C)], 1)
    rw = torch.cat([x.new_zeros(B, rp, C), resid], 1)
    for res in (None, rw):
        yw = torch.full((B, T + rp, C), float("nan"), device=DEV)
        s = 0
        for f in (7, 1, 12, 3, T + rp - 23):
            win = KtStreamWin(in_pitch=xw.shape[1], in_first=K_ - 1 + s, out_pitch=T + rp, out_first=s, res_pitch=T + rp,
                              res_first=s)
            done.fill_(s)
            check(lib.kt_fsmn_fwd_stream_slots(ctypes.byref(win), ctypes.byref(m), ptr(xw), ptr(w), ptr(res), ptr(yw), B, f,
                                               C, K_, lp, stream_ptr()), "kt_fsmn_fwd_stream_slots")
            s += f
        assert s == T + rp
        want = y if res is None else y + resid
        assert torch.equal(yw[:, rp:], want)
        assert torch.equal(yw[:, :rp], torch.zeros_like(yw[:, :rp]))


@pytest.mark.parametrize("H", [128, 40])
def test_lstm_stream_slots_masked_carries_state_across_uneven_chunks(H):
    lib = _lib.load()
    B, L, D = 3, 37, 64
    torch.manual_seed(11)
    lstm = nn.LSTM(D, H, batch_first=True)
    x = torch.randn(B, L, D, generator=torch.Generator().manual_seed(2))
    sd = {"lstm." + k: v.detach().double() for k, v in lstm.state_dict().items()}
    want = O.lstm(x.double(), O._SD(sd), "lstm")
    gx = F.linear(x.double(), sd["lstm.weight_ih_l0"], sd["lstm.bias_ih_l0"] + sd["lstm.bias_hh_l0"]).float().to(DEV)
    whh_t = lstm.weight_hh_l0.detach().t().contiguous().to(DEV)
    state = torch.zeros(B, 2, H, device=DEV)
    h = torch.empty(B, L, H, device=DEV)
    lengths = torch.full((B,), L, dtype=torch.int32, device=DEV)
    done = torch.zeros(B, dtype=torch.int32, device=DEV)
    m = KtStreamMask(lengths=ptr(lengths, True), frames_done=ptr(done, True), rows_per_frame=1, lag=0)
    t0 = 0
    for f in (5, 1, 13, 2, 16):
        done.fill_(t0)
        check(lib.kt_lstm_stream_slots(ptr(gx) + 4 * t0 * 4 * H, ptr(whh_t), ptr(state), ptr(h) + 4 * t0 * H,
                                       ctypes.byref(m), B, f, H, L, L, stream_ptr()), "kt_lstm_stream_slots")
        t0 += f
    assert t0 == L
    err = rel_l2(h.cpu(), want)
    print(f"H={H}: rel err {err:.3e}")
    assert err <= 2e-6
    assert rel_l2(state[:, 0].cpu(), want[:, -1]) <= 2e-6


# ---- end to end -------------------------------------------------------------------------------------------------------
def _small(golden, fp):
    from golden.make_batch import make_sambert_batch
    g = golden("sambert_fp_small_infer" if fp else "sambert_small_infer")
    cfg = g.cfg
    batch = make_sambert_batch(cfg, B=3, L=9, gen=torch.Generator().manual_seed(31), short=3)
    inputs = [batch[k] for k in ("inputs_ling", "inputs_emotion", "inputs_speaker", "input_lengths")]
    am = K.KanTtsSAMBERT(cfg)
    am.load_state_dict(g.group("sd/"), strict=True)
    am = am.to(DEV).eval()
    fp_dict = {int(k): v for k, v in g.group("fp_dict/").items()} if fp else None
    if fp:
        am.fp_dict = {k: v.to(DEV) for k, v in fp_dict.items()}
    gcfg = dict(in_channels=cfg["num_mels"], channels=32, upsample_scales=[4, 2], upsample_kernal_sizes=[8, 4],
                resblock_kernel_sizes=[3, 7], resblock_dilations=[[1, 3], [1, 3]])
    torch.manual_seed(7)
    gen = K.Generator(**gcfg)
    return g, am, gen.to(DEV).eval(), gcfg, inputs, fp_dict


def _collect(stream):
    """-> the (B, 1, samples) concatenation of the yielded chunks, after checking their start samples."""
    wavs, start = [], 0
    for s, w in stream:
        assert s == start and w.shape[0] == stream.batch and w.shape[1] == 1 and w.shape[2] > 0
        wavs.append(w)
        start += w.shape[2]
    return torch.cat(wavs, -1)


@pytest.mark.parametrize("fp", [False, True])
def test_stream_synthesize_matches_synthesize_and_oracle(golden, fp):
    from oracle import hifigan as OH, sambert_fp as OFP
    g, am, gen, gcfg, inputs, fp_dict = _small(golden, fp)
    dev_inputs = [t.to(DEV) for t in inputs]
    with torch.no_grad(), _exact():
        wavs, res = K.synthesize(am, gen, *dev_inputs)
        steps = res["postnet_outputs"].shape[1] // am.mel_decoder.r
        got = {}
        for cs in sorted({1, 2, 5, steps}):
            st = K.stream_synthesize(am, gen, *dev_inputs, chunk_steps=cs)
            assert st.lengths == [w.shape[0] for w in wavs]
            got[cs] = _collect(st)
        want_o = (OFP.sambert_infer(g.group("sd/"), g.cfg, *inputs, fp_dict) if fp
                  else O.sambert_infer(g.group("sd/"), g.cfg, *inputs))
        gsd = {k: v.detach().cpu() for k, v in gen.state_dict().items()}
        wav_o = OH.generator_forward(gsd, want_o["postnet_outputs"].transpose(1, 2), **gcfg)
    for cs, w in got.items():
        assert torch.equal(w, got[1]), cs
    w = got[1].cpu()
    for b, want in enumerate(wavs):
        n = want.shape[0]
        err = rel_l2(w[b, 0, :n], want.cpu())
        print(f"fp={fp} slot {b}: {n} samples, rel err vs synthesize {err:.3e}")
        assert err <= 1e-5
        assert float((w[b, 0, :n] - wav_o[b, 0, :n]).pow(2).mean().sqrt()) <= 1e-3


def test_full_size_stream_matches_synthesize():
    from golden.make_batch import make_sambert_batch
    cfg = K.sambert_24k_config()
    torch.manual_seed(1234)
    am = K.KanTtsSAMBERT(cfg)
    with torch.no_grad():
        am.variance_adaptor.duration_predictor.fc.bias.fill_(1.5)     # about 3.5 frames per symbol
    am = am.to(DEV).eval()
    gen = K.Generator(upsample_scales=[8, 5, 3, 2], upsample_kernal_sizes=[16, 10, 6, 4]).to(DEV).eval()
    batch = make_sambert_batch(cfg, B=4, L=24, gen=torch.Generator().manual_seed(3))
    batch["input_lengths"] = torch.tensor([24, 17, 9, 20])
    inputs = [batch[k].to(DEV) for k in ("inputs_ling", "inputs_emotion", "inputs_speaker", "input_lengths")]
    with torch.no_grad():
        wavs, res = K.synthesize(am, gen, *inputs)
        st = K.stream_synthesize(am, gen, *inputs, chunk_steps=4)
        w = _collect(st).cpu()
    lens = [x.shape[0] for x in wavs]
    assert st.lengths == lens and len(set(lens)) > 1
    for b, want in enumerate(wavs):
        err = rel_l2(w[b, 0, :lens[b]], want.cpu())
        print(f"slot {b}: {lens[b]} samples, rel err {err:.3e}")
        assert err <= 1e-4


def test_stream_does_not_synchronise(golden):
    _, am, gen, _, inputs, _ = _small(golden, False)
    with torch.no_grad():
        it = iter(K.stream_synthesize(am, gen, *(t.to(DEV) for t in inputs), chunk_steps=2))
        next(it)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            rest = list(it)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert rest
