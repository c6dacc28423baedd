"""Streaming a non-causal generator on the GPU (Generator.streamer with lengths): each slot's delayed chunks, cut to
[delay, delay + length * hop), equal the batch-1 forward on the slot's mel of exactly its length, for any chunk schedule and
ragged lengths; a slot reset after draining starts an exact new utterance without touching the others, and a rejected reset
touches nothing; graph-replayed chunks equal eager ones bit for bit; push and finish never synchronise the host."""
import pytest
import torch

import kantts_b200 as K
from kantts_b200 import ops
from conftest import rel_l2
from test_stream_cpu import CONFIGS, SCHEDULES

pytestmark = [pytest.mark.gpu]

V1_16K = dict(channels=256, upsample_scales=[10, 5, 2, 2], upsample_kernal_sizes=[20, 11, 4, 4],
              resblock_dilations=[[1, 3, 5, 7]] * 3)          # hifigan_noncausal_v1_16k.yaml
# the structures whose non-causal whole-utterance forward runs on the GPU (a deconv with k - s even): the small generator, the
# 16 kHz one at reduced and at full width.  The others of test_stream_cpu.CONFIGS are checked against the oracle on the CPU.
GPU_CONFIGS = dict(small=dict(CONFIGS["small"], causal=False), v1_16k=dict(V1_16K, channels=64, causal=False),
                   v1_16k_full=dict(V1_16K, causal=False))
LENGTHS = [23, 17]


def _setup(name, B=2, T=23, seed=3):
    torch.manual_seed(seed)
    g = K.Generator(**GPU_CONFIGS[name]).eval()
    cin = GPU_CONFIGS[name].get("in_channels", 80)
    mel = torch.randn(B, cin, T, generator=torch.Generator().manual_seed(5))
    return g, mel


def _schedule(name, T):
    if name == "fours":
        return [4] * (T // 4) + ([T % 4] if T % 4 else [])
    if name == "ones":
        return [1] * T
    s, out = SCHEDULES["irregular"], []
    while sum(out) < T:
        out.append(min(s[len(out) % len(s)], T - sum(out)))
    return out


def _stream(g, mel, schedule, lengths, max_frames=None):
    st = g.streamer(batch=mel.shape[0], max_frames=max_frames or max(schedule), lengths=lengths)
    outs = [st.push(c) for c in torch.split(mel, schedule, -1)] + [st.finish()]
    return torch.cat(outs, -1), st


def _cut(wav, st, lengths):
    return [wav[b:b + 1, :, st.delay:st.delay + n * st.hop] for b, n in enumerate(lengths)]


@pytest.mark.parametrize("schedule", sorted(SCHEDULES))
@pytest.mark.parametrize("name", sorted(GPU_CONFIGS))
def test_stream_equals_per_utterance_forward(name, schedule):
    from oracle import hifigan as O
    g, mel = _setup(name)
    sched = _schedule(schedule, mel.shape[-1])
    sd = {k: v.detach().clone() for k, v in g.state_dict().items()}
    wav_o = [O.generator_forward(sd, mel[b:b + 1, :, :n], **GPU_CONFIGS[name]) for b, n in enumerate(LENGTHS)]
    g, x = g.cuda(), mel.cuda()
    with torch.no_grad():
        ops.set_force_ffma(True)
        try:
            want = [g(x[b:b + 1, :, :n]) for b, n in enumerate(LENGTHS)]
            wav, st = _stream(g, x, sched, LENGTHS)
        finally:
            ops.set_force_ffma(False)
        got = _cut(wav, st, LENGTHS)
        err = max(float((a - b).abs().max()) for a, b in zip(got, want))
        print(f"{name}/{schedule} exact path: delay {st.delay}, max |stream - forward| = {err:.3e} (bitwise equal: {err == 0.0})")
        assert all(a.shape == b.shape for a, b in zip(got, want)) and err <= 1e-6
        for b, n in enumerate(LENGTHS):                                 # outside the utterance: zeros
            assert float(wav[b, :, :st.delay].abs().max()) == 0.0
            assert float(wav[b, :, st.delay + n * st.hop:].abs().max()) == 0.0
        want = [g(x[b:b + 1, :, :n]) for b, n in enumerate(LENGTHS)]
        wav, st = _stream(g, x, sched, torch.tensor(LENGTHS, device="cuda"))
        for a, w, o in zip(_cut(wav, st, LENGTHS), want, wav_o):
            assert rel_l2(a.cpu(), w.cpu()) <= 1e-4
            assert float((a.cpu() - o).pow(2).mean().sqrt()) <= 1e-3


def test_reset_after_drain_starts_an_exact_utterance_in_one_slot_only():
    g, a = _setup("v1_16k", B=3, T=12)
    u = torch.randn(1, a.shape[1], 9, generator=torch.Generator().manual_seed(9))
    g, a, u = g.cuda(), a.cuda(), u.cuda()
    with torch.no_grad():
        ops.set_force_ffma(True)
        try:
            want_a = [g(a[b:b + 1]) for b in range(3)]
            want_u = g(u)
            st = g.streamer(batch=3, max_frames=4, lengths=[12, 12, 12])
            outs = [st.push(a[:, :, t:t + 4]) for t in (0, 4, 8)]
            drain = st.finish()
            outs.append(drain)
            st.reset([1], [9])
            pad = torch.zeros(3, a.shape[1], 12, device="cuda")
            pad[1, :, :9] = u[0]
            after = [st.push(pad[:, :, t:t + 4]) for t in (0, 4, 8)] + [st.finish()]
        finally:
            ops.set_force_ffma(False)
    first, second = torch.cat(outs, -1), torch.cat(after, -1)
    L, hop = st.delay, st.hop
    for b in range(3):
        assert float((first[b:b + 1, :, L:L + 12 * hop] - want_a[b]).abs().max()) <= 1e-6
    assert float((second[1:2, :, L:L + 9 * hop] - want_u).abs().max()) <= 1e-6
    for b in (0, 2):                                   # drained slots keep streaming silence past their utterance
        assert float(second[b].abs().max()) == 0.0


def test_rejected_reset_leaves_the_stream_as_it_was():
    g, mel = _setup("v1_16k", B=2, T=12)
    g, mel = g.cuda(), mel.cuda()
    with torch.no_grad():
        ops.set_force_ffma(True)
        try:
            want, _ = _stream(g, mel, [4, 4, 4], [12, 12])
            st = g.streamer(batch=2, max_frames=4, lengths=[12, 12])
            outs = [st.push(mel[:, :, :4])]
            with pytest.raises(ValueError, match="distinct"):
                st.reset([0, 0], [12, 12])
            with pytest.raises(ValueError, match="expected 1 lengths"):
                st.reset([1], [9, 9])
            outs += [st.push(mel[:, :, t:t + 4]) for t in (4, 8)] + [st.finish()]
        finally:
            ops.set_force_ffma(False)
    assert torch.equal(torch.cat(outs, -1), want)


def test_graph_replay_equals_eager_bitwise():
    g, mel = _setup("v1_16k", B=2, T=14)
    g, mel = g.cuda(), mel.cuda()
    sched = [4, 4, 4, 2]
    with torch.no_grad():
        graphed, st = _stream(g, mel, sched, [14, 9], max_frames=4)     # replayed full chunks, eager tails
        eager, _ = _stream(g, mel, sched, [14, 9], max_frames=5)        # every chunk eager
    assert graphed.shape == eager.shape and graphed.shape[-1] >= (14 + st.drain_frames) * st.hop
    assert torch.equal(graphed, eager)


def test_push_and_finish_do_not_synchronise():
    g, mel = _setup("small", B=2, T=12)
    g, mel = g.cuda(), mel.cuda()
    with torch.no_grad():
        st = g.streamer(batch=2, max_frames=4, lengths=torch.tensor([12, 7], device="cuda"))
        st.push(mel[:, :, :4])
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            st.push(mel[:, :, 4:8])
            st.push(mel[:, :, 8:11])
            st.push(mel[:, :, 11:12])
            st.finish()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


def test_full_width_v1_16k_tensor_core_path():
    """The shipped non-causal 16 kHz structure at full width on the bf16x3 tensor-core route, chunks of 4 frames."""
    from oracle import hifigan as O
    g, mel = _setup("v1_16k_full", B=2, T=20)
    lengths = [20, 13]
    sd = {k: v.detach().clone() for k, v in g.state_dict().items()}
    g, x = g.cuda(), mel.cuda()
    n_tc = ops.tc_launch_count()
    with torch.no_grad():
        want = [g(x[b:b + 1, :, :n]) for b, n in enumerate(lengths)]
        wav, st = _stream(g, x, [4] * 5, lengths)
    assert ops.tc_launch_count() > n_tc
    assert st.delay == 3424 and st.drain_frames == 18
    for b, n in enumerate(lengths):
        got = wav[b:b + 1, :, st.delay:st.delay + n * st.hop]
        assert rel_l2(got.cpu(), want[b].cpu()) <= 1e-4
        o = O.generator_forward(sd, mel[b:b + 1, :, :n], causal=False, **V1_16K)
        assert float((got.cpu() - o).pow(2).mean().sqrt()) <= 1e-3
