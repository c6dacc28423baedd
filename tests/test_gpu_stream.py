"""Streaming synthesis on the GPU (Generator.streamer): the concatenated chunk outputs equal the whole-utterance forward
for any chunk schedule, batch slots are independent streams, graph-replayed chunks equal eager ones bit for bit, and a
push never synchronises the host."""
import pytest
import torch

import kantts_b200 as K
from kantts_b200 import ops
from conftest import rel_l2
from test_stream_cpu import CONFIGS, SCHEDULES

pytestmark = [pytest.mark.gpu]

GPU_CONFIGS = dict(CONFIGS, full={})        # + the full-width class-default generator


def _setup(name, B=2, T=23, seed=3):
    torch.manual_seed(seed)
    g = K.Generator(**GPU_CONFIGS[name]).eval()
    cin = GPU_CONFIGS[name].get("in_channels", 80)
    T = 32 if name == "full" else T
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


def _stream(g, mel, schedule, max_frames=None):
    st = g.streamer(batch=mel.shape[0], max_frames=max_frames or max(schedule))
    return torch.cat([st.push(c) for c in torch.split(mel, schedule, -1)], -1)


@pytest.mark.parametrize("schedule", sorted(SCHEDULES))
@pytest.mark.parametrize("name", sorted(GPU_CONFIGS))
def test_stream_equals_whole_forward(name, schedule):
    from oracle import hifigan as O
    g, mel = _setup(name)
    sched = _schedule(schedule, mel.shape[-1])
    sd = {k: v.detach().clone() for k, v in g.state_dict().items()}
    wav_o = O.generator_forward(sd, mel, **GPU_CONFIGS[name])
    g = g.cuda()
    x = mel.cuda()
    with torch.no_grad():
        ops.set_force_ffma(True)
        try:
            want, got = g(x), _stream(g, x, sched)
        finally:
            ops.set_force_ffma(False)
        err = float((got - want).abs().max())
        print(f"{name}/{schedule} exact path: max |stream - forward| = {err:.3e} (bitwise equal: {err == 0.0})")
        assert got.shape == want.shape and err <= 1e-6
        want, got = g(x), _stream(g, x, sched)
        assert rel_l2(got.cpu(), want.cpu()) <= 1e-4
        assert float((got.cpu() - wav_o).pow(2).mean().sqrt()) <= 1e-3
        if schedule == "irregular":
            g.remove_weight_norm()
            want, got = g(x), _stream(g, x, sched)
            assert rel_l2(got.cpu(), want.cpu()) <= 1e-4
            assert float((got.cpu() - wav_o).pow(2).mean().sqrt()) <= 1e-3


def test_reset_starts_a_new_utterance_in_one_slot_only():
    g, a = _setup("small", B=3, T=16)
    u = torch.randn(1, a.shape[1], 8, generator=torch.Generator().manual_seed(9))
    g, a, u = g.cuda(), a.cuda(), u.cuda()
    with torch.no_grad():
        want_a, want_u = g(a), g(u)
        st = g.streamer(batch=3, max_frames=4)
        outs = [st.push(a[:, :, 0:4]), st.push(a[:, :, 4:8])]
        st.reset([1])
        for t in (0, 4):
            chunk = a[:, :, 8 + t:12 + t].clone()
            chunk[1] = u[0, :, t:t + 4]
            outs.append(st.push(chunk))
    got = torch.cat(outs, -1)
    hop = st.hop
    for b in (0, 2):
        assert rel_l2(got[b].cpu(), want_a[b].cpu()) <= 1e-4
    assert rel_l2(got[1, :, 8 * hop:].cpu(), want_u[0].cpu()) <= 1e-4


def test_graph_replay_equals_eager_bitwise():
    g, mel = _setup("24k", B=2, T=14)
    g, mel = g.cuda(), mel.cuda()
    sched = [4, 4, 4, 2]
    with torch.no_grad():
        graphed = _stream(g, mel, sched, max_frames=4)       # three replayed chunks, then an eager tail
        eager = _stream(g, mel, sched, max_frames=5)         # every chunk eager
    assert torch.equal(graphed, eager)


def test_push_does_not_synchronise():
    g, mel = _setup("small", B=2, T=12)
    g, mel = g.cuda(), mel.cuda()
    with torch.no_grad():
        st = g.streamer(batch=2, max_frames=4)
        st.push(mel[:, :, :4])                                # graph capture
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            st.push(mel[:, :, 4:8])
            st.push(mel[:, :, 8:11])
            st.push(mel[:, :, 11:12])
        finally:
            torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


def test_push_rejects_bad_chunks():
    g, mel = _setup("small", B=2, T=6)
    g, mel = g.cuda(), mel.cuda()
    st = g.streamer(batch=2, max_frames=4)
    with pytest.raises(ValueError):
        st.push(mel[:, :, :5])
    with pytest.raises(ValueError):
        st.push(mel[:, :, :0])
    with pytest.raises(ValueError):
        st.push(mel[:1, :, :2])
