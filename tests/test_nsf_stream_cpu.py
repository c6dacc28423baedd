"""CPU checks of the seeded NSF excitation and of streaming NSF generators: the oracle's Philox4x32-10 reproduces the
Random123 known answers; the oracle excitation is the same bit for bit whole and chunked, per slot, and its sinusoid is the
reference's formula; the stream plan's windows, lags, histories, delay and launch count follow from the shapes (strided
source convs included); a chunk-by-chunk restatement over the oracle's layer functions equals the oracle's forward with the
same excitation, causal and non-causal; and what cannot be streamed is rejected before any device is needed."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import kantts_b200 as K
from kantts_b200.hifigan import StreamPlan, stream_history, stream_lag, stream_spec
from kantts_b200.ops import ConvSpec
from oracle import hifigan as O
from oracle import nsf as N
from test_stream_cpu import CONFIGS, SCHEDULES, T

NSF16 = dict(nb_harmonics=7, sampling_rate=16000)
NSF24 = dict(nb_harmonics=7, sampling_rate=24000)
V1_NSF_24K = dict(channels=512, upsample_scales=[8, 5, 3, 2], upsample_kernal_sizes=[16, 10, 6, 4], nsf_params=NSF24)
NC_NSF_16K = dict(channels=256, upsample_scales=[10, 5, 2, 2], upsample_kernal_sizes=[20, 11, 4, 4],
                  resblock_dilations=[[1, 3, 5, 7]] * 3, causal=False, nsf_params=NSF16)
# reduced widths of the shipped NSF structures and the small generator, causal and not
STREAM_CONFIGS = {
    "small": dict(CONFIGS["small"], nsf_params=NSF16),
    "small_nc": dict(CONFIGS["small"], nsf_params=NSF16, causal=False),
    "24k": dict(V1_NSF_24K, channels=16),
    "16k_nc": dict(NC_NSF_16K, channels=16),
}
LENGTHS = [23, 17]
SEEDS = [12345, 2 ** 40 + 7]


def _generator(cfg, seed=3):
    torch.manual_seed(seed)
    return K.Generator(**cfg).eval()


def _f0uv(B, frames, seed=11):
    g = torch.Generator().manual_seed(seed)
    f0 = 80 + 220 * torch.rand(B, 1, frames, generator=g, dtype=torch.float64)
    uv = (torch.rand(B, 1, frames, generator=g, dtype=torch.float64) > 0.3).double()
    return f0.float().double(), uv


# ---- Philox and the oracle excitation ---------------------------------------------------------------------------------

@pytest.mark.parametrize("counter,key,want", [
    ((0, 0, 0, 0), (0, 0), "6627e8d5 e169c58d bc57ac4c 9b00dbd8"),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, "408f276d 41c83b0e a20bc7c6 6d5451fd"),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0), "d16cfe09 94fdcceb 5001e420 24126ea1"),
])
def test_philox_known_answers(counter, key, want):
    assert " ".join("%08x" % int(w) for w in N.philox4x32_10(counter, key)) == want


def _chunked(f0, uv, seed, split, hop, sr):
    st = N.ExcitationState(seed, 7)
    out, j = [], 0
    for n in split:
        out.append(N.excitation(f0[j:j + n], uv[j:j + n], st, hop, sr))
        j += n
    return np.concatenate(out)


@pytest.mark.parametrize("split", [[1] * 12, [4, 4, 4], [5, 1, 2, 3, 1], [12]])
def test_oracle_excitation_whole_equals_chunks_bitwise(split):
    f0, uv = _f0uv(1, 12)
    f0, uv = f0[0, 0].numpy(), uv[0, 0].numpy()
    whole = N.excitation(f0, uv, N.ExcitationState(SEEDS[1], 7), 240, 24000)
    assert whole.shape == (12 * 240, 8) and whole.dtype == np.float32
    assert np.array_equal(_chunked(f0, uv, SEEDS[1], split, 240, 24000), whole)


def test_oracle_excitation_slots_are_independent():
    f0, uv = _f0uv(3, 6)
    e = N.batch_excitation(f0, uv, [5, 6, 7], 8, 16000, 7)
    alone = N.batch_excitation(f0[1:2], uv[1:2], [6], 8, 16000, 7)
    assert np.array_equal(e[1:2], alone)
    assert not np.array_equal(e[0], e[2])


def test_oracle_excitation_statistics():
    phi = N.initial_phases(SEEDS[0], 7)
    assert phi[0] == 0 and np.all(phi >= -np.pi) and np.all(phi < np.pi) and len(set(phi[1:].tolist())) == 7
    z = N.normal_noise(SEEDS[0], np.arange(40000), 7)
    assert abs(float(z.mean())) < 0.01 and abs(float(z.std()) - 1.0) < 0.01
    # unvoiced: alpha / (3 sigma) * sigma * z; voiced: alpha * sin + sigma * z
    e = N.excitation(np.full(100, 200.0), np.zeros(100), N.ExcitationState(1, 7), 200, 16000)
    assert abs(float(e.std()) - 0.1 / 3) < 1e-3
    e = N.excitation(np.full(100, 200.0), np.ones(100), N.ExcitationState(1, 7), 200, 16000)
    assert float(np.abs(e).max()) < 0.1 + 6 * 0.003


def test_oracle_sinusoid_matches_the_reference_formula_in_float64():
    """The reference's theta = 2 pi (cumsum(f0_s * (h + 1) / sr) % 1), evaluated with a float64 cumsum: the carried-phase
    definition gives the same sinusoid to 1e-6 over 3 s at 24 kHz (with sigma -> 0 to isolate it)."""
    hop, sr, frames = 300, 24000, 240
    f0, uv = _f0uv(1, frames)
    f0 = f0[0, 0].numpy()
    e = N.excitation(f0, np.ones(frames), N.ExcitationState(SEEDS[0], 7), hop, sr, alpha=1.0, sigma=1e-30)
    f0s = np.repeat(f0.astype(np.float32).astype(np.float64), hop)
    theta = 2 * np.pi * (np.cumsum(f0s[:, None] * np.arange(1, 9)[None, :] / sr, axis=0) % 1)
    want = np.sin(theta + N.initial_phases(SEEDS[0], 7)[None, :].astype(np.float64))
    assert float(np.abs(e - want).max()) <= 1e-6


# ---- strided convs in the stream plan ---------------------------------------------------------------------------------

@pytest.mark.parametrize("u", [2, 4, 6, 20, 30])
def test_strided_source_conv_lag_and_history(u):
    nc = ConvSpec(c_in=1, c_out=8, kernel=2 * u, stride=u, pad_left=u // 2, pad_right=u // 2)
    assert stream_lag(nc) == 1                               # one output row late, from an input of lag 0
    cf = stream_spec(nc)
    assert cf.pad_left == u + u // 2 == stream_history(cf) and cf.pad_left + cf.pad_right == 2 * u - 1
    assert cf.t_out(5 * u) == 5
    for lag_in in (1, u - 1, u, 3 * u + 1):                  # an input that trails: whole output rows, rounded up
        lag = stream_lag(nc, lag_in)
        assert lag == -(-(lag_in + u - u // 2) // u)
        assert stream_spec(nc, lag_in).pad_left == lag * u + u // 2 - lag_in
    causal = ConvSpec(c_in=1, c_out=8, kernel=2 * u, stride=u, pad_left=2 * u - 1)
    assert stream_history(causal) == 2 * u - 1


def test_stride_one_rules_are_unchanged():
    for spec in (ConvSpec(8, 8, 7, pad_left=3, pad_right=3), ConvSpec(8, 8, 11, dilation=5, pad_left=25, pad_right=25),
                 ConvSpec(8, 8, 7, pad_left=3, pad_right=3, upsample=5)):
        r = (spec.kernel - 1) * spec.dilation
        assert stream_lag(spec) == r - spec.pad_left and stream_lag(spec, 4) == 4 * spec.upsample + r - spec.pad_left
        assert stream_spec(spec, 4).pad_left == r and stream_spec(spec, 4).pad_right == 0


# ---- plans -------------------------------------------------------------------------------------------------------------

def test_plan_of_the_causal_24k_nsf_generator():
    plan = StreamPlan(_generator(V1_NSF_24K))
    win = {w["name"]: w for w in plan.windows}
    assert plan.nsf and plan.causal and plan.delay == 0 and plan.hop == 240
    assert (win["f0uv"]["channels"], win["f0uv"]["rows_per_frame"], win["f0uv"]["history"]) == (2, 1, 0)
    assert (win["exc"]["channels"], win["exc"]["rows_per_frame"], win["exc"]["history"]) == (8, 240, 0)
    # the source is read by source_downs with u = 30, 6, 2 (kernel 2u, all padding on the left) and the 1x1 conv
    assert (win["source"]["channels"], win["source"]["rows_per_frame"], win["source"]["history"]) == (1, 240, 59)
    assert [plan.layer_history[f"source_downs.{i}"] for i in range(4)] == [59, 11, 3, 0]
    assert [win[f"e{i}"]["rows_per_frame"] for i in range(4)] == [8, 40, 120, 240]
    # up + (e + rep): the repeat conv, the source conv adding it, the deconv adding that
    for i in range(4):
        convs = [st for st in plan.steps if type(st).__name__ == "ConvStep" and st.dst in (f"rep{i}", f"e{i}", f"up{i}")]
        assert [(st.dst, st.resid) for st in convs] == [(f"rep{i}", None), (f"e{i}", f"rep{i}"), (f"up{i}", f"e{i}")]
    assert not any(type(st).__name__ == "MeanStep" and st.scale == 1.0 for st in plan.steps)
    # 91 of the same generator without NSF + the excitation, the ffn and 4 source convs
    assert plan.launches_per_chunk == 91 + 1 + 1 + 4


def test_plan_of_the_noncausal_16k_nsf_generator():
    g = _generator(NC_NSF_16K)
    plan = StreamPlan(g)
    base = StreamPlan(_generator(dict(NC_NSF_16K, nsf_params=None)))
    lag, win = plan.lags, {w["name"]: w for w in plan.windows}
    # the source convs (u = 20, 4, 2: one output row late; the 1x1: none) never trail the stage: the delay stays 3424
    assert [lag[f"e{i}"] for i in range(4)] == [1, 1, 1, 0]
    assert plan.delay == base.delay == 3424 and plan.hop == 200
    assert plan.layer_history["source_downs.0"] == 30 and plan.layer_history["source_downs.1"] == 6
    assert win["source"]["history"] == 30 and lag["source"] == lag["exc"] == 0
    # stages 0 and 1: the deconv trails (or ties) the repeat conv and chains up + (e + rep); stages 2 and 3 (k 4, s 2, p 1
    # against the k 7 repeat conv) form (e + rep) + up in one three-way add at the repeat conv's lag
    adds = [st for st in plan.steps if type(st).__name__ == "MeanStep" and st.scale == 1.0]
    assert [st.dst for st in adds] == ["sum2", "sum3"]
    for st in adds:
        i = st.dst[-1]
        assert st.srcs == [f"e{i}", f"rep{i}", f"up{i}"] and lag[st.dst] == lag[f"rep{i}"]
        assert st.offsets == [lag[st.dst] - lag[s] for s in st.srcs]
        assert len({win[s]["history"] for s in st.srcs}) == 1 and win[st.srcs[0]]["history"] == max(st.offsets)
    for name in ("rep0", "up0", "mean3"):
        assert lag[name] == base.lags[name]
    assert plan.launches_per_chunk == base.launches_per_chunk + 1 + 1 + 4 + 2


def test_nsf_does_not_change_the_noncausal_look_ahead():
    """A positive-weight probe (as test_stream_noncausal_cpu._probe) of the excitation path: a one-sample excitation
    impulse reaches no output sample earlier than the mel path's 3424-sample look-ahead."""
    cfg = dict(NC_NSF_16K, channels=16)
    g = _generator(cfg)
    sd = {k: v.detach().double().abs() if "weight" in k else torch.zeros_like(v, dtype=torch.float64)
          for k, v in g.state_dict().items()}
    frames, hop = 40, 200
    x = torch.zeros(1, 82, frames, dtype=torch.float64)
    exc = torch.zeros(1, 8, frames * hop, dtype=torch.float64)
    at = 30 * hop
    exc[0, :, at] = 1.0
    y = N.generator_forward(sd, x, exc, **cfg).flatten()
    look_ahead = at - int(y.nonzero()[0])
    assert 0 < look_ahead <= StreamPlan(g).delay == 3424


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_plans_without_nsf_keep_their_windows(name):
    plan = StreamPlan(_generator(CONFIGS[name]))
    assert not plan.nsf and not {"f0uv", "exc", "source"} & {w["name"] for w in plan.windows}


# ---- chunk-by-chunk restatement ----------------------------------------------------------------------------------------

def generator_stream_nsf(sd, x_chunks, lengths, seeds, **cfg):
    """The oracle's generator_forward of an NSF generator with the seeded excitation (oracle/nsf.py), restated chunk by
    chunk as in test_stream_noncausal_cpu.generator_stream_nc: every tensor trails the pushed frames by a lag (0 throughout
    for a causal generator), every layer runs unpadded over [history | chunk] with the rows outside each slot's utterance
    zeroed.  The excitation of a chunk continues each slot's carried state.  -> (waveform, lag, {layer: H}, {stage: e lag})."""
    c = dict(O.GENERATOR_DEFAULTS)
    c.update(cfg)
    causal, nsf = c["causal"], c["nsf_params"]
    slope = c["nonlinear_activation_params"]["negative_slope"]
    nk = len(c["resblock_kernel_sizes"])
    scales = list(c["upsample_scales"])
    hop = int(np.prod(scales))
    lens = torch.tensor(lengths, dtype=torch.float64)
    states = [N.ExcitationState(s, nsf["nb_harmonics"]) for s in seeds]
    state, hist, elag = {}, {}, {}
    pushed = 0

    def window(name, x, h):
        prev = state.get(name, x.new_zeros(x.shape[0], x.shape[1], h))
        full = torch.cat([prev, x], -1)
        state[name] = full[:, :, full.shape[-1] - h:]
        return full

    def masked(full, lag, rate, h):
        u = pushed * rate - lag - h + torch.arange(full.shape[-1], dtype=torch.float64)
        keep = (u[None, :] >= 0) & (u[None, :] < lens[:, None] * rate)
        return full * keep[:, None, :]

    def delayed(name, x, d):
        return window(name, x, d)[:, :, :x.shape[-1]]

    def conv(name, x, lag, rate, dilation=1, act=None):
        k = O._resolve_weight(sd, name + ".conv1d.").shape[-1]
        h = (k - 1) * dilation
        hist[name] = h
        full = masked(window(name, x, h), lag, rate, h)
        if act is not None:
            full = F.leaky_relu(full, act)
        return O.conv1d(sd, name + ".", full, False, 0, dilation), lag + (0 if causal else h // 2)

    def add(key, terms):
        """the sum of (tensor, lag) terms at the latest lag"""
        lag = max(lt for _, lt in terms)
        return sum(delayed(f"{key}.{n}", t, lag - lt) for n, (t, lt) in enumerate(terms)), lag

    outs = []
    for xc in x_chunks:
        f = xc.shape[-1]
        mel, f0, uv = xc[:, :-2], xc[:, -2], xc[:, -1]
        exc = torch.from_numpy(np.stack([N.excitation(f0[b].numpy(), uv[b].numpy(), states[b], hop, nsf["sampling_rate"]).T
                                         for b in range(xc.shape[0])])).double()
        source = N.source_ffn(sd, exc)                                   # lag 0, hop rows per frame
        rate = 1
        x, lag = conv("conv_pre", mel, 0, 1)
        for i, (s, uk) in enumerate(zip(scales, c["upsample_kernal_sizes"])):
            x = torch.sin(x) + x
            name = f"repeat_upsamples.{i}.2"
            k = O._resolve_weight(sd, name + ".conv1d.").shape[-1]
            h = -(-(k - 1) // s)
            hist[name] = h
            rep = F.leaky_relu(F.interpolate(masked(window(name, x, h), lag, rate, h), scale_factor=s, mode="nearest"), slope)
            rep = O.conv1d(sd, name + ".", rep, False, 0)[:, :, -f * s:]
            lrep = lag * s + (0 if causal else (k - 1) // 2)
            name = f"transpose_upsamples.{i}.1"
            h = (uk - 1) // s
            hist[name] = h
            up = F.leaky_relu(masked(window(name, x, h), lag, rate, h), slope)
            up = O.conv_transpose1d(sd, name + ".", up, False, s, 0)[:, :, h * s:(h + f) * s]
            lup = lag * s + (0 if causal else (uk - s) // 2)
            f, rate = f * s, rate * s
            u = hop // rate
            name = f"source_downs.{i}"
            if u == 1:
                e, le = O.conv1d(sd, name + ".", source, False, 0), 0
                hist[name] = 0
            else:
                le = 0 if causal else 1
                h = 2 * u - 1 if causal else u + u // 2                   # stream_spec's left padding
                hist[name] = h
                e = O.conv1d(sd, name + ".", masked(window(name, source, h), 0, hop, h), False, 0, 1, u)
            elag[i] = le
            x, lag = add(f"sum{i}", [(up, lup), (e, le), (rep, lrep)])
            branches = []
            for j in range(nk):
                r, lr = x, lag
                for p, d in enumerate(c["resblock_dilations"][j]):
                    xt, lt = conv(f"conv_blocks.{i * nk + j}.convs1.{p}", r, lr, rate, d, slope)
                    xt, lt = conv(f"conv_blocks.{i * nk + j}.convs2.{p}", xt, lt, rate, 1, slope)
                    r, lr = add(f"res{i}.{j}.{p}", [(xt, lt), (r, lr)])
                branches.append((r, lr))
            x, lag = add(f"mean{i}", branches)
            x = x / nk
        y, lag = conv("conv_post", x, lag, rate, 1, 0.01)
        outs.append(masked(torch.tanh(y), lag, rate, 0))
        pushed += xc.shape[-1]
    hist["source_module.ffn.0"] = 0
    return torch.cat(outs, -1), lag, hist, elag


@pytest.mark.parametrize("schedule", sorted(SCHEDULES))
@pytest.mark.parametrize("name", sorted(STREAM_CONFIGS))
def test_oracle_stream_equals_the_seeded_forward(name, schedule):
    cfg = STREAM_CONFIGS[name]
    g = _generator(cfg)
    plan = StreamPlan(g)
    sd = {k: v.detach().double() for k, v in g.state_dict().items()}
    mel = torch.randn(2, 80, T, generator=torch.Generator().manual_seed(5), dtype=torch.float64)
    x = torch.cat([mel, *_f0uv(2, T)], 1)
    lengths = LENGTHS if not plan.causal else [T, T]
    drain = -(-plan.delay // plan.hop)
    chunks = list(torch.split(x, SCHEDULES[schedule], -1))
    if drain:
        chunks.append(torch.cat([torch.randn(2, 80, drain, dtype=torch.float64), *_f0uv(2, drain, 13)], 1))
    got, lag, hist, elag = generator_stream_nsf(sd, chunks, lengths, SEEDS, **cfg)
    assert lag == plan.delay and plan.layer_history == hist
    assert [plan.lags[f"e{i}"] for i in range(len(elag))] == [elag[i] for i in range(len(elag))]
    for b, n in enumerate(lengths):
        exc = torch.from_numpy(N.batch_excitation(x[b:b + 1, -2:-1, :n], x[b:b + 1, -1:, :n], [SEEDS[b]], plan.hop,
                                                  cfg["nsf_params"]["sampling_rate"], 7))
        want = N.generator_forward(sd, x[b:b + 1, :, :n], exc, **cfg)
        out = got[b:b + 1, :, lag:lag + n * plan.hop]
        assert out.shape == want.shape
        assert float((out - want).abs().max()) <= 1e-6, (name, schedule, b)


# ---- rejections --------------------------------------------------------------------------------------------------------

def test_seeds_are_rejected_where_they_do_not_belong():
    plain = K.Generator(channels=32).eval()
    with pytest.raises(ValueError, match="NSF"):
        plain(torch.zeros(1, 80, 4), nsf_seeds=[1])
    with pytest.raises(ValueError, match="NSF"):
        plain.streamer(batch=1, max_frames=4, seeds=[1])
    nsf = K.Generator(channels=32, nsf_params=NSF16).eval()
    with pytest.raises(ValueError, match="expected 2 NSF seeds"):
        nsf.streamer(batch=2, max_frames=4, seeds=[1])
    with pytest.raises(ValueError, match="int64"):
        nsf.streamer(batch=1, max_frames=4, seeds=torch.zeros(1, dtype=torch.int32))
    with pytest.raises(ValueError, match="NSF"):                         # no seeds: the streamer refuses before the device
        K.Generator(channels=32, causal=False, nsf_params=NSF16).eval().streamer(batch=1, max_frames=4, lengths=[4])
    with pytest.raises(RuntimeError, match="CUDA"):                      # no CPU fallback
        nsf.streamer(batch=1, max_frames=4, seeds=[1])


def test_nsf_f0_needs_matching_models(golden):
    from kantts_b200.infer import denorm_f0
    g = golden("sambert_small_infer")
    am = K.KanTtsSAMBERT(g.cfg)
    am.load_state_dict(g.group("sd/"), strict=True)
    am.eval()
    n = g.cfg["num_mels"]
    inputs = (torch.zeros(1, 4, 4, dtype=torch.long), torch.zeros(1, 4, dtype=torch.long), torch.zeros(1, 4, dtype=torch.long),
              torch.tensor([4]))
    gen = K.Generator(in_channels=n, channels=32, upsample_scales=[4, 2], upsample_kernal_sizes=[8, 4],
                      nsf_params=NSF16).eval()                         # takes n + 2 channels: the model makes n
    for fn in (K.synthesize, K.stream_synthesize):
        with pytest.raises(ValueError, match="mel channels"):
            fn(am, gen, *inputs, nsf_f0=("mean_std", 200.0, 50.0), nsf_seeds=[1])
        with pytest.raises(ValueError, match="nsf_f0 and nsf_seeds"):
            fn(am, gen, *inputs, nsf_f0=("mean_std", 200.0, 50.0))
        with pytest.raises(ValueError, match="NSF generator"):
            fn(am, K.Generator(in_channels=n, channels=32).eval(), *inputs, nsf_f0=("global", 30.0, 730.0), nsf_seeds=[1])
    with pytest.raises(ValueError, match="NSF"):                         # streaming an NSF generator needs both
        K.stream_synthesize(am, gen, *inputs)
    rows = torch.tensor([[[0.5, 1.0, 0.59], [0.5, -9.0, 0.6]]])
    out = denorm_f0(rows, ("mean_std", 200.0, 50.0))
    assert out.tolist() == [[[0.5, 250.0, 0.0], [0.5, 30.0, 1.0]]]
    assert denorm_f0(rows, ("global", 30.0, 730.0))[0, 0, 1] == 730.0


@pytest.mark.parametrize("name", ["small", "small_nc", "24k"])
def test_given_excitation_forward_equals_the_oracle_forward(name):
    """oracle/nsf.generator_forward fed the reference's own random draw (the raw excitation oracle.hifigan.nsf_excitation
    makes under the same torch seed) equals oracle.hifigan.generator_forward: the restatement with a given excitation is
    the same network."""
    from torch.distributions.normal import Normal
    from torch.distributions.uniform import Uniform
    cfg = STREAM_CONFIGS[name]
    g = _generator(cfg)
    sd = {k: v.detach().double() for k, v in g.state_dict().items()}
    mel = torch.randn(2, 80, 9, generator=torch.Generator().manual_seed(5), dtype=torch.float64)
    f0, uv = _f0uv(2, 9)
    x = torch.cat([mel, f0, uv], 1)
    hop = int(np.prod(cfg["upsample_scales"]))
    torch.manual_seed(21)
    want = O.generator_forward(sd, x, **cfg)
    torch.manual_seed(21)                                  # the same draws, in the reference's order (layers.py:266-279)
    f0s, uvs = F.interpolate(f0, scale_factor=hop, mode="nearest"), F.interpolate(uv, scale_factor=hop, mode="nearest")
    harm = torch.arange(1, 9, dtype=f0s.dtype)[None, :, None]
    theta = 2 * np.pi * (torch.cumsum(f0s * harm / cfg["nsf_params"]["sampling_rate"], dim=-1) % 1)
    phase = Uniform(low=-np.pi, high=np.pi).sample(sample_shape=(2, 8, 1))
    phase[:, 0, :] = 0
    noise = Normal(loc=0.0, scale=0.003).sample(sample_shape=(2, 8, f0s.shape[-1]))
    e = (0.1 * torch.sin(theta + phase) + noise) * uvs + (0.1 / 3 / 0.003 * noise) * (1 - uvs)
    got = N.generator_forward(sd, x, e, **cfg)
    assert got.shape == want.shape and float((got - want).abs().max()) <= 1e-12
