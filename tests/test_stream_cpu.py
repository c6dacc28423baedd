"""CPU checks of streaming synthesis (Generator.streamer): a chunk-by-chunk restatement over the oracle's layer functions
(generator_stream below) equals the oracle's whole-utterance forward for every chunk schedule, the streamer's window plan
keeps the history each layer reads, the launch count per chunk follows from the shapes, and the stream descriptors match
the header."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

import kantts_b200 as K
from kantts_b200 import _lib
from kantts_b200.hifigan import StreamPlan
from oracle import hifigan as O

# the small causal generator of test_gpu_pipeline.py and reduced-width copies of the shipped causal configs' structure
CONFIGS = {
    "small": dict(in_channels=80, channels=32, upsample_scales=[4, 2], upsample_kernal_sizes=[8, 4],
                  resblock_kernel_sizes=[3, 7], resblock_dilations=[[1, 3], [1, 3]]),
    "16k": dict(channels=64, upsample_scales=[10, 5, 2, 2], upsample_kernal_sizes=[20, 10, 4, 4]),
    "24k": dict(channels=64, upsample_scales=[8, 5, 3, 2], upsample_kernal_sizes=[16, 10, 6, 4]),
    "8k": dict(channels=64, upsample_scales=[5, 5, 2, 2], upsample_kernal_sizes=[10, 10, 4, 4]),
    "48k": dict(in_channels=128, channels=128, upsample_scales=[10, 5, 3, 2, 2], upsample_kernal_sizes=[20, 10, 6, 4, 4],
                resblock_dilations=[[1, 3, 5, 7]] * 3),
}
T = 23
SCHEDULES = {"ones": [1] * T, "fours": [4] * (T // 4) + [T % 4], "irregular": [5, 1, 2, 9, 3, 3]}


def generator_stream(sd, mel_chunks, **cfg):
    """The oracle's generator_forward of a causal generator without NSF, restated chunk by chunk with the oracle's own
    layer functions: every layer keeps the last H rows of its input between chunks (zeros before the first one, which is
    the causal zero padding) and runs UNPADDED over
    [history | chunk], H being what it reads before a chunk: (k-1)*d for a conv, ceil((k-1)*d / s) input rows for the
    conv over the nearest-upsampled input, floor((k-1) / s) for the transposed conv (whose outputs of the chunk are the
    rows [H*s, (H+f)*s) of its uncropped output).  -> (the concatenated waveform, {layer name: H})."""
    c = dict(O.GENERATOR_DEFAULTS)
    c.update(cfg)
    assert c["causal"] and c["nsf_params"] is None and c["repeat_upsample"]
    slope = c["nonlinear_activation_params"]["negative_slope"]
    nk = len(c["resblock_kernel_sizes"])
    state, hist = {}, {}

    def window(name, x, h):
        """[history | x] of layer `name`; its last h rows become the layer's history."""
        hist[name] = h
        prev = state.get(name, x.new_zeros(x.shape[0], x.shape[1], h))
        full = torch.cat([prev, x], -1)
        state[name] = full[:, :, full.shape[-1] - h:]
        return full

    def conv(name, x, dilation=1, act=None):
        k = O._resolve_weight(sd, name + ".conv1d.").shape[-1]
        full = window(name, x, (k - 1) * dilation)
        if act is not None:                                              # act(0) = 0: a zero history stays the padding
            full = F.leaky_relu(full, act)
        return O.conv1d(sd, name + ".", full, False, 0, dilation)

    outs = []
    for mel in mel_chunks:
        f = mel.shape[-1]
        x = conv("conv_pre", mel)
        for i, (s, uk) in enumerate(zip(c["upsample_scales"], c["upsample_kernal_sizes"])):
            x = torch.sin(x) + x
            name = f"repeat_upsamples.{i}.2"
            k = O._resolve_weight(sd, name + ".conv1d.").shape[-1]
            full = window(name, x, -(-(k - 1) // s))
            rep = F.leaky_relu(F.interpolate(full, scale_factor=s, mode="nearest"), slope)
            rep = O.conv1d(sd, name + ".", rep, False, 0)[:, :, -f * s:]
            name = f"transpose_upsamples.{i}.1"
            h = (uk - 1) // s
            up = F.leaky_relu(window(name, x, h), slope)
            up = O.conv_transpose1d(sd, name + ".", up, False, s, 0)[:, :, h * s:(h + f) * s]
            x = rep + up
            xs = None
            for j in range(nk):
                r = x
                for p, d in enumerate(c["resblock_dilations"][j]):
                    xt = conv(f"conv_blocks.{i * nk + j}.convs1.{p}", r, d, slope)
                    xt = conv(f"conv_blocks.{i * nk + j}.convs2.{p}", xt, 1, slope)
                    r = xt + r
                xs = r if xs is None else xs + r
            x = xs / nk
            f *= s
        outs.append(torch.tanh(conv("conv_post", x, 1, 0.01)))
    return torch.cat(outs, -1), hist


def _generator(name, seed=3):
    torch.manual_seed(seed)
    return K.Generator(**CONFIGS[name]).eval()


@pytest.mark.parametrize("schedule", sorted(SCHEDULES))
@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_oracle_stream_equals_whole_forward(name, schedule):
    cfg = CONFIGS[name]
    g = _generator(name)
    sd = {k: v.detach().double() for k, v in g.state_dict().items()}
    mel = torch.randn(2, cfg.get("in_channels", 80), T, generator=torch.Generator().manual_seed(5), dtype=torch.float64)
    want = O.generator_forward(sd, mel, **cfg)
    got, hist = generator_stream(sd, list(torch.split(mel, SCHEDULES[schedule], -1)), **cfg)
    assert got.shape == want.shape
    assert float((got - want).abs().max()) <= 1e-6
    assert StreamPlan(g).layer_history == hist


def test_plan_windows_keep_the_largest_history_of_their_readers():
    plan = StreamPlan(_generator("24k"))
    win = {w["name"]: w for w in plan.windows}
    # stage 0: sin(x)+x feeds the repeat conv (k 7 over x8 up-sampled rows: ceil(6 / 8) = 1) and the deconv (k 16, s 8: 1)
    assert win["sin0"]["history"] == 1 and win["sin0"]["rows_per_frame"] == 1
    # the ResBlock input feeds three first convs (k 3 / 7 / 11, dilation 1: 2 / 6 / 10) and the residual adds (0)
    assert win["up0"]["history"] == 10 and win["up0"]["rows_per_frame"] == 8
    assert win["rb0.2.h0"]["history"] == 10 and win["rb0.2.x1"]["history"] == 30      # k 11: c2 (d 1), next c1 (d 3)
    assert win["rb0.2.x3"]["history"] == 0                                             # read by the mean only
    assert win["mel"]["history"] == 6 and win["mean3"]["history"] == 6                 # conv_pre / conv_post, k 7
    assert win["wav"]["rows_per_frame"] == 240 and plan.hop == 240
    assert plan.layer_history["transpose_upsamples.2.1"] == 1                          # k 6, s 3
    assert plan.layer_history["repeat_upsamples.1.2"] == 2                             # ceil(6 / 5)


def test_launches_per_chunk_follow_from_the_shapes():
    # class defaults: conv_pre + 4 x (repeat conv + deconv + 3 ResBlocks x 3 pairs x 2) + conv_post = 82 convs,
    # 4 sin-adds, 4 means, 1 window advance
    assert StreamPlan(K.Generator().eval()).launches_per_chunk == 82 + 4 + 4 + 1
    for name, cfg in CONFIGS.items():
        pairs = sum(len(d) for d in cfg.get("resblock_dilations", [[1, 3, 5]] * 3))
        n = len(cfg["upsample_scales"])
        assert StreamPlan(_generator(name)).launches_per_chunk == 2 + n * (2 + 2 * pairs) + 2 * n + 1, name


def test_stream_descriptor_sizes_match_header():
    assert ctypes.sizeof(_lib.KtStreamWin) == 6 * 4
    assert ctypes.sizeof(_lib.KtWindow) == 8 + 4 * 4
    assert _lib.KT_PLAN_STREAM == 16


def test_stream_plan_takes_the_register_staged_route():
    """A layer the TMA-fed route would take for a whole sequence runs register-staged as a stream chunk."""
    from kantts_b200.ops import ConvSpec
    _lib.build_library()
    lib = _lib.load()
    spec = ConvSpec(c_in=256, c_out=256, kernel=3, pad_left=2)
    d = spec.desc(64, 1, 512)
    whole, stream = (ctypes.c_int64 * 9)(), (ctypes.c_int64 * 9)()
    assert lib.kt_debug_conv_tc_plan(ctypes.byref(d), 0, whole) == 0
    assert lib.kt_debug_conv_tc_plan(ctypes.byref(d), _lib.KT_PLAN_STREAM, stream) == 0
    assert whole[0] > 0 and whole[1] == 1                     # N tile, TMA route
    assert stream[0] > 0 and stream[1] == 0 and stream[8] == 0
    assert lib.kt_conv1d_tc_workspace(ctypes.byref(d), _lib.KT_PLAN_STREAM) == 0
    assert lib.kt_conv1d_tc_plan(ctypes.byref(spec.desc(4, 3, 64)), _lib.KT_PLAN_STREAM) == 0    # nsub > 1: no stream


def test_streamer_rejects_what_it_cannot_stream():
    with pytest.raises(ValueError, match="causal"):
        K.Generator(channels=32, causal=False).eval().streamer(batch=1, max_frames=4)
    with pytest.raises(ValueError, match="NSF"):
        K.Generator(channels=32, nsf_params=dict(nb_harmonics=7, sampling_rate=16000)).eval().streamer(batch=1, max_frames=4)
    with pytest.raises(ValueError, match="eval"):
        K.Generator(channels=32).train().streamer(batch=1, max_frames=4)
    with pytest.raises(RuntimeError, match="CUDA"):                     # no CPU fallback
        K.Generator(channels=32).eval().streamer(batch=1, max_frames=4)
