"""CPU checks of streaming a non-causal generator (Generator.streamer with lengths): a chunk-by-chunk restatement over the
oracle's layer functions, with every tensor trailing the pushed mel by a lag and every layer input masked to its slot's
utterance, equals the oracle's per-utterance forward; the plan's lags, histories and delay agree with it and with a
perturbation probe of the oracle; causal plans keep their windows; and the new descriptors match the header."""
import ctypes
import os
import re

import pytest
import torch
import torch.nn.functional as F

import kantts_b200 as K
from kantts_b200 import _lib
from kantts_b200.hifigan import StreamPlan
from oracle import hifigan as O
from test_stream_cpu import CONFIGS, SCHEDULES, T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NC_CONFIGS = {name: dict(cfg, causal=False) for name, cfg in CONFIGS.items()}
LENGTHS = [23, 17]                    # ragged: slot 1 ends 6 frames before the pushed mel does


def generator_stream_nc(sd, mel_chunks, lengths, **cfg):
    """The oracle's generator_forward of a non-causal generator without NSF, restated chunk by chunk.  Every tensor of a
    chunk trails the pushed mel by a lag: its chunk row t of slot b is utterance row u = pushed * rate - lag + t.  Every
    layer runs in causal form, UNPADDED over [history | chunk] with the rows outside [0, lengths[b] * rate) of its input
    zeroed (the whole-utterance zero padding, per slot), and its output trails its input by the layer's right reach.  A sum
    of two tensors at different lags reads the earlier one from as many rows back.  -> (the concatenated waveform, the
    waveform's lag in samples, {layer name: H})."""
    c = dict(O.GENERATOR_DEFAULTS)
    c.update(cfg)
    assert not c["causal"] and c["nsf_params"] is None and c["repeat_upsample"]
    slope = c["nonlinear_activation_params"]["negative_slope"]
    nk = len(c["resblock_kernel_sizes"])
    lens = torch.tensor(lengths, dtype=torch.float64)
    state, hist = {}, {}
    pushed = 0

    def window(name, x, h):
        prev = state.get(name, x.new_zeros(x.shape[0], x.shape[1], h))
        full = torch.cat([prev, x], -1)
        state[name] = full[:, :, full.shape[-1] - h:]
        return full

    def masked(full, lag, rate, h):
        """zero the rows of [history | chunk] outside each slot's utterance"""
        u = pushed * rate - lag - h + torch.arange(full.shape[-1], dtype=torch.float64)
        keep = (u[None, :] >= 0) & (u[None, :] < lens[:, None] * rate)
        return full * keep[:, None, :]

    def delayed(name, x, d):
        """x read d rows back"""
        return window(name, x, d)[:, :, :x.shape[-1]]

    def conv(name, x, lag, rate, dilation=1, act=None):
        k = O._resolve_weight(sd, name + ".conv1d.").shape[-1]
        h = (k - 1) * dilation
        hist[name] = h
        full = masked(window(name, x, h), lag, rate, h)
        if act is not None:
            full = F.leaky_relu(full, act)
        return O.conv1d(sd, name + ".", full, False, 0, dilation), lag + h // 2

    def add(key, a, la, b, lb):
        """a + b, at the later of their lags"""
        if la >= lb:
            return a + delayed(key, b, la - lb), la
        return delayed(key, a, lb - la) + b, lb

    outs = []
    for mel in mel_chunks:
        f = mel.shape[-1]
        rate = 1
        x, lag = conv("conv_pre", mel, 0, 1)
        for i, (s, uk) in enumerate(zip(c["upsample_scales"], c["upsample_kernal_sizes"])):
            x = torch.sin(x) + x
            name = f"repeat_upsamples.{i}.2"
            k = O._resolve_weight(sd, name + ".conv1d.").shape[-1]
            h = -(-(k - 1) // s)
            hist[name] = h
            rep = F.leaky_relu(F.interpolate(masked(window(name, x, h), lag, rate, h), scale_factor=s, mode="nearest"), slope)
            rep = O.conv1d(sd, name + ".", rep, False, 0)[:, :, -f * s:]
            name = f"transpose_upsamples.{i}.1"
            h = (uk - 1) // s
            hist[name] = h
            up = F.leaky_relu(masked(window(name, x, h), lag, rate, h), slope)
            up = O.conv_transpose1d(sd, name + ".", up, False, s, 0)[:, :, h * s:(h + f) * s]
            x, lag = add(f"sum{i}", rep, lag * s + (k - 1) // 2, up, lag * s + (uk - s) // 2)
            f, rate = f * s, rate * s
            branches = []
            for j in range(nk):
                r, lr = x, lag
                for p, d in enumerate(c["resblock_dilations"][j]):
                    xt, lt = conv(f"conv_blocks.{i * nk + j}.convs1.{p}", r, lr, rate, d, slope)
                    xt, lt = conv(f"conv_blocks.{i * nk + j}.convs2.{p}", xt, lt, rate, 1, slope)
                    r, lr = add(f"res{i}.{j}.{p}", xt, lt, r, lr)
                branches.append((r, lr))
            lag = max(lr for _, lr in branches)
            x = sum(delayed(f"mean{i}.{j}", r, lag - lr) for j, (r, lr) in enumerate(branches)) / nk
        y, lag = conv("conv_post", x, lag, rate, 1, 0.01)
        outs.append(masked(torch.tanh(y), lag, rate, 0))
        pushed += mel.shape[-1]
    return torch.cat(outs, -1), lag, hist


def _generator(cfg, seed=3):
    torch.manual_seed(seed)
    return K.Generator(**cfg).eval()


@pytest.mark.parametrize("schedule", sorted(SCHEDULES))
@pytest.mark.parametrize("name", sorted(NC_CONFIGS))
def test_oracle_stream_equals_per_utterance_forward(name, schedule):
    cfg = NC_CONFIGS[name]
    g = _generator(cfg)
    plan = StreamPlan(g)
    sd = {k: v.detach().double() for k, v in g.state_dict().items()}
    mel = torch.randn(2, cfg.get("in_channels", 80), T, generator=torch.Generator().manual_seed(5), dtype=torch.float64)
    drain = -(-plan.delay // plan.hop)
    # the slots' mel past their lengths and the drained frames are garbage: the masks must make them irrelevant
    chunks = list(torch.split(mel, SCHEDULES[schedule], -1)) + [torch.randn(2, mel.shape[1], drain, dtype=torch.float64)]
    got, lag, hist = generator_stream_nc(sd, chunks, LENGTHS, **cfg)
    assert lag == plan.delay
    assert plan.layer_history == hist
    for b, n in enumerate(LENGTHS):
        want = O.generator_forward(sd, mel[b:b + 1, :, :n], **cfg)
        out = got[b:b + 1, :, lag:lag + n * plan.hop]
        assert out.shape == want.shape
        assert float((out - want).abs().max()) <= 1e-6, (name, schedule, b)
        assert float(got[b, :, :lag].abs().max()) == 0.0 and float(got[b, :, lag + n * plan.hop:].abs().max()) == 0.0


def _probe(cfg, frames=40, frame=30):
    """Look-ahead of the oracle's non-causal forward in output samples: perturb one mel frame and find the first output
    sample that changes.  The weights are made positive and the biases zero, with a one-hot mel: every path from the frame
    to a sample then adds a positive amount, so no dependency cancels or falls below float64 resolution.  (With random
    weights the longest paths run through the edge taps of some twenty layers, a product far below 1e-16 of the output,
    and such a probe finds a smaller look-ahead that changes with the seed and the frame.)"""
    g = _generator(cfg)
    sd = {k: v.detach().double().abs() if "weight" in k else torch.zeros_like(v, dtype=torch.float64)
          for k, v in g.state_dict().items()}
    mel = torch.zeros(1, cfg.get("in_channels", 80), frames, dtype=torch.float64)
    mel[..., frame] = 1.0
    y = O.generator_forward(sd, mel, **cfg).flatten()
    hop = y.numel() // frames
    return frame * hop - int(y.nonzero()[0])


PROBE_CONFIGS = {
    # hifigan_noncausal_v1_16k.yaml's structure (channels reduced: the look-ahead does not depend on them)
    "noncausal_v1_16k": (dict(channels=16, upsample_scales=[10, 5, 2, 2], upsample_kernal_sizes=[20, 11, 4, 4],
                              resblock_dilations=[[1, 3, 5, 7]] * 3, causal=False), 3424, 200),
    "defaults": (dict(channels=16, causal=False), 3264, 256),
    "8-5-3-2": (dict(channels=16, upsample_scales=[8, 5, 3, 2], upsample_kernal_sizes=[16, 10, 6, 4], causal=False), 3210, 240),
}


@pytest.mark.parametrize("name", sorted(PROBE_CONFIGS))
def test_delay_equals_the_oracle_look_ahead(name):
    cfg, delay, hop = PROBE_CONFIGS[name]
    plan = StreamPlan(_generator(cfg))
    assert (plan.delay, plan.hop) == (delay, hop)
    assert _probe(cfg) == plan.delay
    assert plan.lags["wav"] == plan.delay


def test_plan_lags_and_histories():
    plan = StreamPlan(_generator(dict(channels=16, causal=False)))
    lag, win = plan.lags, {w["name"]: w for w in plan.windows}
    assert lag["mel"] == 0 and lag["x"] == 3                         # conv_pre, k 7: right padding 3
    assert lag["rep0"] == 3 * 8 + 3 and lag["up0"] == 3 * 8 + 4      # the deconv (k 16, s 8, padding 4) is the later
    assert win["rep0"]["history"] == 1                               # up0 = deconv + rep0 one row back
    # the three ResBlocks (k 3 / 7 / 11, dilations 1-3-5) end 12 / 36 / 60 rows after their input
    assert [lag[f"rb0.{j}.x3"] - lag["up0"] for j in range(3)] == [12, 36, 60]
    assert lag["mean0"] == lag["up0"] + 60
    assert all(win[f"rb0.{j}.x3"]["history"] == 48 for j in range(3))
    mean = next(st for st in plan.steps if type(st).__name__ == "MeanStep")
    assert mean.offsets == [48, 24, 0]
    # stage 2 (k 4, s 2, padding 1): the repeat conv (right padding 3) is the later one and adds the deconv
    assert lag["rep2"] == 2 * lag["mean1"] + 3 and lag["up2"] == 2 * lag["mean1"] + 1
    assert win["up2"]["history"] == 2
    conv = [st for st in plan.steps if type(st).__name__ == "ConvStep" and st.dst == "rep2"][0]
    assert conv.resid == "up2" and conv.res_lag == 2
    assert plan.delay == lag["mean3"] + 3
    assert plan.launches_per_chunk == 82 + 4 + 4 + 1 + 1             # + the output mask


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_causal_plan_is_unchanged(name):
    """A causal plan has no lags: every window, history, residual and mean read is as before non-causal streaming."""
    plan = StreamPlan(_generator(CONFIGS[name]))
    assert plan.causal and plan.delay == 0 and set(plan.lags.values()) == {0}
    for st in plan.steps:
        if type(st).__name__ == "ConvStep":
            assert st.res_lag == 0 and st.spec is st.conv.spec
        if type(st).__name__ == "MeanStep":
            assert set(st.offsets) == {0}
    assert {w["name"]: w["history"] for w in plan.windows}["wav"] == 0


def test_stream_mask_descriptor_and_argument_match_header():
    assert ctypes.sizeof(_lib.KtStreamMask) == 8 + 8 + 4 + 4
    header = open(os.path.join(ROOT, "include", "kantts_b200.h")).read()
    body = re.search(r"typedef struct KtStreamMask \{([^}]*)\} KtStreamMask;", header).group(1)
    fields = re.findall(r"(\w+)(?:,|;)", body)
    assert fields == [f for f, _ in _lib.KtStreamMask._fields_]
    assert "kt_stream_mask_advance" in _lib.PROTOTYPES and re.search(r"^int kt_stream_mask_advance\(", header, flags=re.M)
    # the utterance mask is the optional third argument of the one stream forward per route
    for name in ("kt_conv1d_fwd_stream", "kt_conv1d_fwd_tc_stream"):
        params = re.search(rf"^int {name}\(([^)]*)\);", header, flags=re.M).group(1).split(",")
        assert " ".join(params[2].split()) == "const KtStreamMask* m", (name, params)
        assert _lib.PROTOTYPES[name][2] is ctypes.POINTER(_lib.KtStreamMask), name
    for name in ("kt_conv1d_fwd_stream_masked", "kt_conv1d_fwd_tc_stream_masked", "kt_l1_sum_acc"):
        assert name not in _lib.PROTOTYPES and not re.search(rf"\b{name}\b", header), name


def test_streamer_rejects_what_it_cannot_stream():
    nc = K.Generator(channels=32, causal=False).eval()
    with pytest.raises(ValueError, match="non-causal generator needs per-slot lengths"):
        nc.streamer(batch=1, max_frames=4)
    with pytest.raises(ValueError, match="causal generator streams without lengths"):
        K.Generator(channels=32).eval().streamer(batch=1, max_frames=4, lengths=[4])
    with pytest.raises(ValueError, match="NSF"):
        K.Generator(channels=32, causal=False, nsf_params=dict(nb_harmonics=7, sampling_rate=16000)).eval().streamer(
            batch=1, max_frames=4, lengths=[4])
    with pytest.raises(RuntimeError, match="CUDA"):                     # no CPU fallback
        nc.streamer(batch=1, max_frames=4, lengths=[4])


def test_stream_synthesize_stays_causal():
    from kantts_b200.infer import stream_synthesize

    class _AM:
        training = False
    with pytest.raises(ValueError, match="causal"):
        stream_synthesize(_AM(), K.Generator(channels=32, causal=False).eval(), None, None, None, None)
