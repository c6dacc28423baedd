"""The seeded NSF excitation and streamed NSF generators on the GPU: kt_nsf_excitation equals the oracle's definition;
forward(x, nsf_seeds) equals the oracle's forward with that excitation and does not mix slots; streamed chunks equal the
seeded forward bit for bit on the exact path (cut per slot for a non-causal generator), within tolerance on the
tensor-core path; a reset slot restarts with its new seed alone; graph replay equals eager; push never synchronises; and
stream_synthesize with an NSF acoustic model gives synthesize()'s waveforms (bit for bit across chunk sizes)."""
import pytest
import torch

import kantts_b200 as K
from kantts_b200 import ops
from kantts_b200.hifigan import SourceModule
from conftest import rel_l2
from oracle import hifigan as O
from oracle import nsf as N
from test_gpu_stream import _schedule
from test_nsf_stream_cpu import NC_NSF_16K, NSF16, SEEDS, V1_NSF_24K, _f0uv
from test_stream_cpu import CONFIGS, SCHEDULES

pytestmark = [pytest.mark.gpu]
DEV = "cuda"
# non-causal structures whose whole-utterance forward runs on the GPU (deconvs with k - s even)
GPU_CONFIGS = {
    "small": dict(CONFIGS["small"], nsf_params=NSF16),
    "small_nc": dict(CONFIGS["small"], nsf_params=NSF16, causal=False),
    "24k": dict(V1_NSF_24K, channels=32),
    "16k_nc": dict(NC_NSF_16K, channels=32),
}
LENGTHS = [23, 17]


class _exact:
    def __enter__(self):
        ops.set_force_ffma(True)

    def __exit__(self, *exc):
        ops.set_force_ffma(False)


def _setup(cfg, B=2, T=23, seed=3):
    torch.manual_seed(seed)
    g = K.Generator(**cfg).eval()
    mel = torch.randn(B, cfg.get("in_channels", 80), T, generator=torch.Generator().manual_seed(5))
    return g, torch.cat([mel, *(t.float() for t in _f0uv(B, T))], 1)


def _stream(g, x, schedule, seeds, lengths=None, max_frames=None):
    st = g.streamer(batch=x.shape[0], max_frames=max_frames or max(schedule), lengths=lengths, seeds=seeds)
    outs = [st.push(c) for c in torch.split(x, schedule, -1)] + [st.finish()]
    return torch.cat(outs, -1), st


@pytest.mark.parametrize("hop,sr,frames", [(8, 16000, 23), (240, 24000, 37), (300, 24000, 1000)])
def test_kernel_excitation_equals_the_oracle(hop, sr, frames):
    seeds = [0, SEEDS[0], SEEDS[1], 2 ** 63 - 1]
    f0, uv = _f0uv(len(seeds), frames, seed=frames)
    sm = SourceModule(7, hop, sr).to(DEV)
    e = sm.excitation(f0.float().to(DEV), uv.float().to(DEV), seeds).cpu()             # (B, samples, 8)
    want = torch.from_numpy(N.batch_excitation(f0, uv, seeds, hop, sr, 7)).transpose(1, 2)
    err = float((e - want).abs().max())
    print(f"hop {hop}, {frames} frames: max |kernel - oracle| = {err:.3e}")
    assert e.shape == want.shape and err <= 1e-6
    dev_seeds = torch.tensor(seeds, dtype=torch.int64, device=DEV)
    assert torch.equal(sm.excitation(f0.float().to(DEV), uv.float().to(DEV), dev_seeds).cpu(), e)


@pytest.mark.parametrize("name", sorted(GPU_CONFIGS))
def test_seeded_forward_matches_the_oracle_and_keeps_slots_apart(name):
    cfg = GPU_CONFIGS[name]
    g, x = _setup(cfg)
    sd = {k: v.detach().clone() for k, v in g.state_dict().items()}
    hop = 1
    for s in cfg["upsample_scales"]:
        hop *= s
    exc = torch.from_numpy(N.batch_excitation(x[:, -2:-1], x[:, -1:], SEEDS, hop, cfg["nsf_params"]["sampling_rate"], 7))
    wav_o = N.generator_forward(sd, x, exc, **cfg)
    g, xd = g.to(DEV), x.to(DEV)
    with torch.no_grad():
        got = g(xd, nsf_seeds=SEEDS).cpu()
        assert float((got - wav_o).pow(2).mean().sqrt()) < 1e-3 and rel_l2(got, wav_o) < 1e-4
        with _exact():
            both = g(xd, nsf_seeds=torch.tensor(SEEDS, device=DEV))
            alone = g(xd[1:], nsf_seeds=SEEDS[1:])
        assert torch.equal(both[1:], alone)
        assert not torch.equal(g(xd, nsf_seeds=SEEDS), g(xd, nsf_seeds=[7, 8]))


@pytest.mark.parametrize("schedule", sorted(SCHEDULES))
@pytest.mark.parametrize("name", sorted(GPU_CONFIGS))
def test_stream_equals_the_seeded_forward(name, schedule):
    cfg = GPU_CONFIGS[name]
    g, x = _setup(cfg)
    g, x = g.to(DEV), x.to(DEV)
    causal = cfg.get("causal", True)
    lengths = None if causal else LENGTHS
    sched = _schedule(schedule, x.shape[-1])
    with torch.no_grad():
        for exact in (True, False):
            ops.set_force_ffma(exact)
            try:
                if causal:
                    want = [g(x, nsf_seeds=SEEDS)[b:b + 1] for b in range(2)]
                else:
                    want = [g(x[b:b + 1, :, :n], nsf_seeds=SEEDS[b:b + 1]) for b, n in enumerate(LENGTHS)]
                wav, st = _stream(g, x, sched, SEEDS, lengths)
            finally:
                ops.set_force_ffma(False)
            ns = [x.shape[-1]] * 2 if causal else LENGTHS
            got = [wav[b:b + 1, :, st.delay:st.delay + n * st.hop] for b, n in enumerate(ns)]
            err = max(float((a - w).abs().max()) for a, w in zip(got, want))
            print(f"{name}/{schedule} exact={exact}: delay {st.delay}, max |stream - forward| = {err:.3e}")
            assert all(a.shape == w.shape for a, w in zip(got, want))
            if exact:
                assert err == 0.0
            else:
                assert max(rel_l2(a.cpu(), w.cpu()) for a, w in zip(got, want)) <= 1e-4


def test_full_size_24k_nsf_tensor_core_path():
    """hifigan_v1_nsf_24k.yaml at full width on the bf16x3 tensor-core route, chunks of 4 frames."""
    g, x = _setup(V1_NSF_24K, T=20)
    sd = {k: v.detach().clone() for k, v in g.state_dict().items()}
    g, xd = g.to(DEV), x.to(DEV)
    n_tc = ops.tc_launch_count()
    with torch.no_grad():
        want = g(xd, nsf_seeds=SEEDS)
        wav, st = _stream(g, xd, [4] * 5, SEEDS)
    assert ops.tc_launch_count() > n_tc and st.delay == 0
    assert rel_l2(wav.cpu(), want.cpu()) <= 1e-4
    exc = torch.from_numpy(N.batch_excitation(x[:, -2:-1], x[:, -1:], SEEDS, 240, 24000, 7))
    o = N.generator_forward(sd, x, exc, **V1_NSF_24K)
    assert float((wav.cpu() - o).pow(2).mean().sqrt()) <= 1e-3


@pytest.mark.parametrize("name", ["small", "16k_nc"])
def test_reset_with_a_new_seed_touches_one_slot_only(name):
    cfg = GPU_CONFIGS[name]
    causal = cfg.get("causal", True)
    g, a = _setup(cfg, B=3, T=12)
    _, u = _setup(cfg, B=1, T=9, seed=4)
    u = u + 0.1 * torch.randn(u.shape, generator=torch.Generator().manual_seed(9))
    g, a, u = g.to(DEV), a.to(DEV), u.to(DEV)
    seeds = [3, 4, 5]
    with torch.no_grad(), _exact():
        want_a = [g(a[b:b + 1], nsf_seeds=seeds[b:b + 1]) for b in range(3)]
        want_u = g(u, nsf_seeds=[99])
        st = g.streamer(batch=3, max_frames=4, lengths=None if causal else [12] * 3, seeds=seeds)
        first = torch.cat([st.push(a[:, :, t:t + 4]) for t in (0, 4, 8)] + [st.finish()], -1)
        with pytest.raises(ValueError, match="seeds"):
            st.reset([1], None if causal else [9])
        st.reset([1], None if causal else [9], seeds=[99])
        cont = a.clone()
        cont[1, :, :9] = u[0]
        second = torch.cat([st.push(cont[:, :, t:t + 4]) for t in (0, 4, 8)] + [st.finish()], -1)
    L, hop = st.delay, st.hop
    for b in range(3):
        assert torch.equal(first[b:b + 1, :, L:L + 12 * hop], want_a[b])
    assert torch.equal(second[1:2, :, L:L + 9 * hop], want_u)
    if causal:              # the other slots carry on: their 24 frames are one utterance
        with torch.no_grad(), _exact():
            for b in (0, 2):
                whole = g(torch.cat([a[b:b + 1], cont[b:b + 1]], -1), nsf_seeds=seeds[b:b + 1])
                assert torch.equal(torch.cat([first[b:b + 1], second[b:b + 1]], -1), whole)
    else:                   # drained slots stream silence past their utterance
        assert float(second[0].abs().max()) == 0.0 and float(second[2].abs().max()) == 0.0


@pytest.mark.parametrize("name", ["24k", "16k_nc"])
def test_graph_replay_equals_eager_bitwise(name):
    cfg = GPU_CONFIGS[name]
    g, x = _setup(cfg, T=14)
    g, x = g.to(DEV), x.to(DEV)
    lengths = None if cfg.get("causal", True) else [14, 9]
    with torch.no_grad():
        graphed, st = _stream(g, x, [4, 4, 4, 2], SEEDS, lengths, max_frames=4)
        eager, _ = _stream(g, x, [4, 4, 4, 2], SEEDS, lengths, max_frames=5)
    assert torch.equal(graphed, eager)


def test_push_does_not_synchronise():
    g, x = _setup(GPU_CONFIGS["16k_nc"], T=12)
    g, x = g.to(DEV), x.to(DEV)
    with torch.no_grad():
        st = g.streamer(batch=2, max_frames=4, lengths=torch.tensor([12, 7], device=DEV),
                        seeds=torch.tensor(SEEDS, device=DEV))
        st.push(x[:, :, :4])
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            st.push(x[:, :, 4:8])
            st.push(x[:, :, 8:11])
            st.finish()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    with pytest.raises(ValueError, match="mel \\+ f0 \\+ uv"):
        st.push(x[:, :-2, :4])


def test_stream_synthesize_with_an_nsf_acoustic_model_equals_synthesize(golden):
    from golden.make_batch import make_sambert_batch
    g = golden("sambert_small_infer")
    cfg = dict(g.cfg, num_mels=82)
    torch.manual_seed(1234)
    am = K.KanTtsSAMBERT(cfg)
    with torch.no_grad():
        am.variance_adaptor.duration_predictor.fc.bias.fill_(1.5)
    am = am.to(DEV).eval()
    batch = make_sambert_batch(cfg, B=3, L=9, gen=torch.Generator().manual_seed(31), short=3)
    inputs = [batch[k].to(DEV) for k in ("inputs_ling", "inputs_emotion", "inputs_speaker", "input_lengths")]
    torch.manual_seed(7)
    gen = K.Generator(**dict(CONFIGS["small"], nsf_params=NSF16)).to(DEV).eval()
    nsf_f0, seeds = ("mean_std", 180.0, 40.0), [11, 12, 13]
    with torch.no_grad(), _exact(), torch.backends.cudnn.flags(enabled=False):
        wavs, _ = K.synthesize(am, gen, *inputs, nsf_f0=nsf_f0, nsf_seeds=seeds)
        got = {}
        for cs in (1, 4, 16):
            st = K.stream_synthesize(am, gen, *inputs, chunk_steps=cs, nsf_f0=nsf_f0, nsf_seeds=seeds)
            assert st.lengths == [w.shape[0] for w in wavs]
            got[cs] = torch.cat([w for _, w in st], -1)
    assert len({w.shape[0] for w in wavs}) > 1
    # the streamed post-net rows equal the whole post-net's to rounding (test_gpu_tts_stream.py): the vocoder stream is
    # exact on them (test_stream_equals_the_seeded_forward), so the waveforms are bitwise equal across chunk sizes and
    # within that rounding of synthesize()
    for cs, w in got.items():
        assert torch.equal(w, got[1]), cs
    for b, want in enumerate(wavs):
        err = rel_l2(got[1][b, 0, :want.shape[0]].cpu(), want.cpu())
        print(f"slot {b}: {want.shape[0]} samples, rel err vs synthesize {err:.3e}")
        assert err <= 1e-5
