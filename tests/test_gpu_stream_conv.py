"""The stream conv forward (kt_conv1d_fwd_stream: exact fp32, conv_core_kernel<RN, RM, KC, true, MASK>;
kt_conv1d_fwd_tc_stream: bf16x3 tensor cores, conv_tc_kernel<ROUTE, true, MASK>) of one chunk against a plain float64
reference, and the window kernels it relies on (advance, reset, mask advance, sin-add and three-way add into a window).

The cases are every distinct stream conv of the shipped streamers at full width -- the causal class-default generator, the
non-causal 16 kHz one, the causal NSF 24 kHz one and the SAM-BERT post-net -- plus synthetic edges: a persistent grid that
wraps past the SMs, partial tiles and K chunks, odd channel counts, taps before the history and past the chunk, a residual
window of its own pitch, up-sampling by 8, 10 and 32, transposed convs reading history.  Each case runs on the exact route
and on its default route, and the kernel nodes of a CUDA graph captured around a second launch confirm that the conv
kernels it launches are exactly the instances it is named for.  up32_masked is the regression
case of an int overflow: a slot whose utterance starts 2^26 rows ahead, scaled by 32, read its whole window as data.

Masked cases give every batch slot its own utterance state (MASK_STATES).  Rows outside a slot's utterance must read as
zero whatever the window holds there: NaN, 1e30 and zeros give the same bits, which are the bits of the unmasked instance
of the same route on the zero-filled window.  Every call must leave the rows outside its output chunk, its input and its
residual untouched (guard rows and guard items inside the same allocations).

Accuracy is checked per element, |y - ref| <= c * scale with scale = sum_j |w_j| |x_j| + |bias| + |resid| (the bound of
any summation order), so that one wrong row cannot hide under a global relative L2; the global relative L2 is bounded too.
"""
import ctypes
import dataclasses
import math
from dataclasses import dataclass

import pytest
import torch

from conftest import rel_l2

DEV = "cuda"
F64 = torch.float64
KT_ACT_LRELU, KT_ACT_TANH = 1, 2

# Per-element error over the error scale.  Worst over all cases on an H100 80GB HBM3 (700 W power limit): exact fp32
# 4.95e-7 (grid_wrap_masked), bf16x3 1.53e-5 (thin_cin2_masked); the bounds are just under 4x those.  Exact fp32 sums up to
# k * c_in products; bf16x3 drops the lo * lo product and each operand's bits below its 16-bit hi + lo split.  Relative L2:
# the suite's bounds for the two paths (worst measured 1.0e-6 and 1.2e-5, both gen:512-256k7s1d1p6u8).
ELEM_BOUND = {"ffma": 1.9e-6, "tc": 6e-5}
L2_BOUND = {"ffma": 2e-5, "tc": 1e-4}


def _ops():
    from kantts_b200 import ops
    return ops


# ------------------------------------------------------------------------------------------------
# float64 reference of one chunk
# ------------------------------------------------------------------------------------------------


def _chunk_rows(x_win, in_first, t_in, t, mask):
    """Chunk rows t (int64 (n,)) of every item, (B, n, C): window row in_first + t for -in_first <= t < t_in, else 0.  With
    a mask (lengths, frames_done, rows_per_frame, lag), row t of item b is kept only when its utterance row
    u = frames_done[b] * rows_per_frame - lag + t lies in [0, lengths[b] * rows_per_frame); a selection, so whatever a
    dropped row holds (NaN included) never reaches the output."""
    B = x_win.shape[0]
    keep = ((t >= -in_first) & (t < t_in))[None, :].expand(B, -1)
    if mask is not None:
        lengths, frames_done, rpf, lag = mask
        u = frames_done.long()[:, None] * rpf - lag + t[None, :]
        keep = keep & (u >= 0) & (u < lengths.long()[:, None] * rpf)
    rows = x_win[:, (in_first + t).clamp(0, x_win.shape[1] - 1)]
    return torch.where(keep[..., None], rows, torch.zeros((), dtype=rows.dtype))


def ref_stream_conv(spec, x_win, in_first, t_in, w, bias, resid_win, res_first, mask):
    """One chunk of the conv `spec` (ConvSpec semantics) in float64 -> (y, scale), each (B, t_out, c_out).
    x_win (B, pitch, c_in): chunk row t is window row in_first + t; w in the reference layout ((c_out, c_in / groups, k), a
    transposed conv (c_in, c_out, k)); bias (c_out,) or None; resid_win (B, pitch', c_out) or None, output row to adds its
    row res_first + to; mask as _chunk_rows.  scale = sum_j |w_j| |x_j| + |bias| + |resid| per output element."""
    x = x_win.to(F64)
    if spec.act_in == KT_ACT_LRELU:
        x = torch.where(x > 0, x, x * spec.act_in_slope)
    W = w.to(F64)
    B, G = x.shape[0], spec.groups
    t_out = spec.t_out(t_in)
    cig, cog = spec.c_in // G, spec.c_out // G
    to = torch.arange(t_out)
    y = torch.zeros(B, t_out, spec.c_out, dtype=F64)
    s = torch.zeros_like(y)
    for j in range(spec.kernel):
        if spec.transposed:
            # y[ti * stride + j * dilation - pad_left] += w[:, :, j]^T x[ti]
            num = to + spec.pad_left - j * spec.dilation
            ti = torch.div(num, spec.stride, rounding_mode="floor")
            xs = _chunk_rows(x, in_first, t_in, ti, mask)
            xs = torch.where((num % spec.stride == 0)[None, :, None], xs, torch.zeros((), dtype=F64))
            wj = W[:, :, j]                                               # (c_in, c_out)
        else:
            # input row floor((to * stride + j * dilation - pad_left) / upsample) of the nearest-upsampled input
            pos = to * spec.stride + j * spec.dilation - spec.pad_left
            xs = _chunk_rows(x, in_first, t_in, torch.div(pos, spec.upsample, rounding_mode="floor"), mask)
            wj = W[:, :, j].t()                                           # (c_in / groups, c_out)
        for g in range(G):
            xg, wg = xs[..., g * cig:(g + 1) * cig], wj[:, g * cog:(g + 1) * cog]
            y[..., g * cog:(g + 1) * cog] += xg @ wg
            s[..., g * cog:(g + 1) * cog] += xg.abs() @ wg.abs()
    if bias is not None:
        y += bias.to(F64)
        s += bias.to(F64).abs()
    if spec.act_out == KT_ACT_LRELU:
        y = torch.where(y > 0, y, y * spec.act_out_slope)
    elif spec.act_out == KT_ACT_TANH:
        y = torch.tanh(y)
    if resid_win is not None:
        r = resid_win[:, res_first:res_first + t_out].to(F64)
        y = y + r
        s = s + r.abs()
    return y, s


# ------------------------------------------------------------------------------------------------
# CPU self-check of the reference against the whole-utterance oracle
# ------------------------------------------------------------------------------------------------


def _oracle_kw(spec):
    act_out = None
    if spec.act_out == KT_ACT_LRELU:
        act_out = spec.act_out_slope
    elif spec.act_out == KT_ACT_TANH:
        act_out = "tanh"
    return dict(stride=spec.stride, dilation=spec.dilation, pad_left=spec.pad_left, pad_right=spec.pad_right,
                groups=spec.groups, transposed=spec.transposed, upsample=spec.upsample, crop=spec.crop,
                act_in=spec.act_in_slope if spec.act_in == KT_ACT_LRELU else None, act_out=act_out)


def _spec(**kw):
    from kantts_b200.ops import ConvSpec
    return ConvSpec(**kw)


def _stream_history(spec):
    from kantts_b200.hifigan import stream_history
    return stream_history(spec)


# causal specs: a chunk of t_in input rows (divisible by the stride) gives out_rate * t_in output rows
SELF_CHECK_SPECS = {
    "conv": dict(c_in=6, c_out=5, kernel=7, pad_left=6, act_in=KT_ACT_LRELU, act_in_slope=0.1),
    "strided": dict(c_in=3, c_out=4, kernel=8, stride=4, pad_left=5, pad_right=2),
    "dilated": dict(c_in=4, c_out=6, kernel=3, dilation=5, pad_left=10, act_out=KT_ACT_LRELU, act_out_slope=0.2),
    "upsampled": dict(c_in=5, c_out=3, kernel=7, pad_left=6, upsample=8, act_in=KT_ACT_LRELU, act_in_slope=0.1),
    "transposed": dict(c_in=5, c_out=4, kernel=16, stride=8, transposed=True, crop=8, act_in=KT_ACT_LRELU,
                       act_in_slope=0.1),
    "transposed_k11_s5": dict(c_in=3, c_out=2, kernel=11, stride=5, transposed=True, crop=6, act_out=KT_ACT_TANH),
}


def _out_rate(spec):
    return spec.stride if spec.transposed else spec.upsample / spec.stride


@pytest.mark.parametrize("masked", [False, True], ids=["plain", "masked"])
@pytest.mark.parametrize("name", sorted(SELF_CHECK_SPECS))
def test_reference_chunks_equal_whole_utterance_oracle(name, masked):
    """Chunks cut from a whole utterance, each with the history its spec needs, give the rows of oracle.convref.conv_layer
    on the whole zero-padded utterance.  Masked: the utterance (rows_per_frame 3, lag 4) sits inside a longer sequence
    whose rows outside it hold garbage, and the chunks are cut from that sequence."""
    from oracle import convref
    spec = _spec(**SELF_CHECK_SPECS[name])
    g = torch.Generator().manual_seed(len(name) * 7 + masked)
    B, rpf, lag = 2, 3, 4
    L = 12 * rpf                                           # utterance rows
    a = 17 if masked else 0                                # sequence row of utterance row 0
    seq = torch.randn(B, a + L + (23 if masked else 0), spec.c_in, generator=g, dtype=F64)
    if masked:
        seq[:, :a] = 1e6 * torch.randn(B, a, spec.c_in, generator=g, dtype=F64)
        seq[:, a + L:] = float("nan")
    w_shape = (spec.c_in, spec.c_out, spec.kernel) if spec.transposed else (spec.c_out, spec.c_in, spec.kernel)
    w = torch.randn(w_shape, generator=g, dtype=F64)
    bias = torch.randn(spec.c_out, generator=g, dtype=F64)
    rate = _out_rate(spec)
    whole = convref.conv_layer(seq[:, a:a + L].transpose(1, 2), w, bias, **_oracle_kw(spec)).transpose(1, 2)
    assert whole.shape[1] == L * rate
    resid_whole = torch.randn(B, whole.shape[1] + 5, spec.c_out, generator=g, dtype=F64)
    hist = _stream_history(spec)
    # chunk starts d = c0 - a (utterance rows) and rows: multiples of 4 (the strided spec's stride); masked, also
    # d + lag = frames_done * rpf
    chunks = [(-16, 12), (-4, 12), (8, 12), (20, 12), (32, 12)] if masked else [(-8, 8), (0, 4), (4, 8), (12, 12), (24, 8),
                                                                               (32, 12)]
    checked = 0
    for d, t_in in chunks:
        c0 = a + d
        lo = c0 - hist
        x_win = torch.zeros(B, hist + t_in, spec.c_in, dtype=F64)
        src = torch.arange(lo, c0 + t_in)
        ok = (src >= 0) & (src < seq.shape[1]) if masked else (src >= a) & (src < a + L)
        x_win[:, ok] = seq[:, src[ok]]
        mask = None
        if masked:
            # chunk row t is sequence row c0 + t = utterance row d + t = frames_done * rpf - lag + t
            assert (d + lag) % rpf == 0
            mask = (torch.full((B,), L // rpf), torch.full((B,), (d + lag) // rpf), rpf, lag)
        o0 = int(d * rate)
        t_out = spec.t_out(t_in)
        assert t_out == t_in * rate
        res_first = 2
        resid_win = torch.zeros(B, res_first + t_out, spec.c_out, dtype=F64)
        rows = torch.arange(o0, o0 + t_out)
        inside = (rows >= 0) & (rows < whole.shape[1])
        resid_win[:, res_first:][:, inside] = resid_whole[:, rows[inside]]
        y, s = ref_stream_conv(spec, x_win, hist, t_in, w, bias, resid_win, res_first, mask)
        want = whole[:, rows[inside]] + resid_whole[:, rows[inside]]
        assert torch.allclose(y[:, inside], want, rtol=1e-12, atol=1e-9), (name, c0, t_in)
        assert bool((s >= y.abs() - 1e-9).all())
        checked += int(inside.sum())
    assert checked >= L * rate * 0.6


# ------------------------------------------------------------------------------------------------
# cases
# ------------------------------------------------------------------------------------------------


@dataclass
class Case:
    name: str
    spec: object
    t_in: int
    hist: int                      # in_first: rows of history before the chunk
    B: int = 2
    masked: bool = False
    rpf: int = 1                   # mask: rows per frame of the input window
    lag: int = 0                   # mask: rows the input window trails its frames by
    out_first: int = 3
    res_first: int = -1            # < 0: no residual
    res_pitch_extra: int = 0       # residual window rows after its chunk


# Mask states: slot b of a masked case takes MASK_STATES[b % 8]; _mask_table turns each into (lengths, frames_done) for the
# case's rows per frame, lag, history and chunk rows.
MASK_STATES = ("inside", "starts_mid_chunk", "ended_in_history", "ends_mid_chunk", "idle", "starts_past_2^26",
               "long_running_mid", "long_running_ended")


def _mask_table(c, B):
    """-> (lengths, frames_done) int32 (B,) for case c: slot b takes state MASK_STATES[b % 8]."""
    H, n, rpf, lag = c.hist, c.t_in, c.rpf, c.lag
    # frames_done of a long-running slot (frames_done * rpf > 2^31 for rpf > 1)
    big = 2 ** 31 - 1 - (n + H + lag) // rpf - 16
    span = (n + H + lag) // rpf + 16                         # frames that reach past the whole window

    def start_at(t0):                                        # frames_done that puts utterance row 0 at chunk row ~t0
        return math.floor((lag - t0) / rpf)

    def end_at(e):                                           # frames_done that ends a span-frame utterance at row ~e (<= e)
        return -math.floor((e - lag - span * rpf) / rpf)

    states = {
        "inside": (start_at(-H - 2 * rpf), span + 4),
        "starts_mid_chunk": (start_at(n // 2), span),
        "ended_in_history": (end_at(0), span),
        "ends_mid_chunk": (end_at(n // 2), span),
        "idle": (5, 0),
        "starts_past_2^26": (start_at(2 ** 26 + 5), 100),
        "long_running_mid": (big, 2 ** 31 - 1),
        "long_running_ended": (big, big - span),
    }
    fd, ln = zip(*(states[MASK_STATES[b % len(MASK_STATES)]] for b in range(B)))
    return torch.tensor(ln, dtype=torch.int32), torch.tensor(fd, dtype=torch.int32)


def _tc_route(c):
    """-> the tensor-core route (0 register-staged simple, 1 generic) of case c's stream plan, None for the exact kernel."""
    from kantts_b200 import _lib
    d = c.spec.desc(c.B, 1, c.t_in)
    if not _lib.load().kt_conv1d_tc_plan(ctypes.byref(d), _lib.KT_PLAN_STREAM):
        return None
    s = c.spec
    assert s.groups == 1, s
    # run_tc's `simple` predicate for a stream forward (nsub 1, no accumulation, no data-gradient mask)
    return 0 if s.upsample == 1 and s.c_in % 8 == 0 and s.c_out % 4 == 0 and s.act_out != KT_ACT_TANH else 1


def tc_instance(c):
    route = _tc_route(c)
    return None if route is None else f"conv_tc_kernel<{route}, true, {'true' if c.masked else 'false'}>"


def conv_phase_rows(spec, t_in, direction):
    """The output rows M of each phase conv_phases makes for direction 0 (forward) or 1 (data gradient) of layer spec over
    t_in input rows: a scatter (transposed forward, strided data gradient) has one phase per output residue mod stride,
    an up-sampled data gradient one accumulating phase per up-sampled row."""
    t_out = spec.t_out(t_in)
    s = spec.stride

    def scatter(n):
        return [(n - r + s - 1) // s for r in range(min(s, n))]

    if direction == 0:
        return scatter(t_out) if spec.transposed else [t_out]
    if spec.transposed:
        return [t_in]
    return scatter(t_in) if spec.upsample == 1 else [t_in] * spec.upsample


def core_instance(M, cin_g, cout_g, groups, batch, stream=False, masked=False):
    """The conv_core_kernel instance run_core launches for one phase of M output rows: cin_g / cout_g channels per group on
    the contracted / produced side, batch items (x sub-sequences)."""
    rn = 4 if cout_g > 64 else (2 if cout_g > 32 else 1)
    kc = 4 if cin_g <= 4 else 16

    def ctas(rm):
        return -(-M // (8 * rm)) * groups * -(-cout_g // (32 * rn)) * batch

    rm = 16
    while rm > 4 and (ctas(rm) < 296 or M <= 4 * rm):
        rm >>= 1
    return f"conv_core_kernel<{rn}, {rm}, {kc}, {'true' if stream else 'false'}, {'true' if masked else 'false'}>"


def core_instances(c):
    """The conv_core_kernel instances run_core launches for case c, one per phase (a transposed conv has `stride`)."""
    s = c.spec
    return sorted({core_instance(M, s.c_in // s.groups, s.c_out // s.groups, s.groups, c.B, True, c.masked)
                   for M in conv_phase_rows(s, c.t_in, 0)})


def _spec_key(spec):
    return tuple(getattr(spec, f.name) for f in dataclasses.fields(spec) if not f.name.startswith("_"))


def _streamer_cases():
    """One case per distinct (spec, masked, route) of the shipped streamers' stream convs, at full width."""
    import kantts_b200 as K
    from kantts_b200.hifigan import ConvStep, StreamPlan
    from kantts_b200.sambert import PostNet, PostNetStreamPlan
    torch.manual_seed(0)
    nsf24 = dict(channels=512, upsample_scales=[8, 5, 3, 2], upsample_kernal_sizes=[16, 10, 6, 4],
                 nsf_params=dict(nb_harmonics=7, sampling_rate=24000))
    nc16 = dict(channels=256, upsample_scales=[10, 5, 2, 2], upsample_kernal_sizes=[20, 11, 4, 4],
                resblock_dilations=[[1, 3, 5, 7]] * 3, causal=False)
    out, seen = [], set()

    def add(src, spec, hist, rpf, lag, masked, f, res_lag, res_hist):
        c = Case(f"{src}:{spec.c_in}-{spec.c_out}k{spec.kernel}s{spec.stride}d{spec.dilation}p{spec.pad_left}"
                 f"{'T' if spec.transposed else ''}{f'u{spec.upsample}' if spec.upsample > 1 else ''}",
                 spec, t_in=f * rpf, hist=hist, B=8 if masked else 2, masked=masked, rpf=rpf, lag=lag,
                 res_first=-1 if res_lag is None else res_hist - res_lag)
        key = (_spec_key(spec), masked, _tc_route(c), c.res_first >= 0)
        if key not in seen:
            seen.add(key)
            out.append(c)

    for src, cfg in (("gen", {}), ("nc16k", nc16), ("nsf24k", nsf24)):
        plan = StreamPlan(K.Generator(**cfg).eval())
        win = {w["name"]: w for w in plan.windows}
        for st in plan.steps:
            if type(st) is ConvStep:
                wi = win[st.src]
                add(src, st.spec, wi["history"], wi["rows_per_frame"], plan.lags[st.src], not plan.causal, 2,
                    None if st.resid is None else st.res_lag, None if st.resid is None else win[st.resid]["history"])
    pn = PostNetStreamPlan(PostNet(K.sambert_24k_config()).eval())
    win = {w["name"]: w for w in pn.windows}
    for st in pn.steps:
        if st.kind == "conv":
            mod = st.module
            spec = _spec(c_in=mod.input_size, c_out=4 * mod.hidden_size, kernel=1) if hasattr(mod, "hidden_size") else mod.spec
            add("postnet", spec, win[st.src]["history"], 1, 0, False, 16,
                None if st.resid is None else st.res_lag, None if st.resid is None else win[st.resid]["history"])
    return out


def _synthetic_cases():
    L = dict(act_in=KT_ACT_LRELU, act_in_slope=0.1)
    cases = [
        # 16 items x 5 M tiles x 2 N tiles = 160 tiles: the persistent grid wraps past 132 CTAs; 2 N tiles: weights streamed
        Case("grid_wrap", _spec(c_in=256, c_out=256, kernel=3, pad_left=2, **L), t_in=600, hist=2, B=16),
        Case("grid_wrap_masked", _spec(c_in=256, c_out=256, kernel=3, pad_left=2, **L), t_in=600, hist=2, B=16,
             masked=True, rpf=4, lag=6),
        Case("partial_m_tile", _spec(c_in=64, c_out=64, kernel=5, pad_left=4), t_in=200, hist=4, res_first=4),
        Case("one_row_chunk", _spec(c_in=128, c_out=64, kernel=7, pad_left=6, **L), t_in=1, hist=6),
        Case("one_row_chunk_masked", _spec(c_in=128, c_out=64, kernel=7, pad_left=6, **L), t_in=1, hist=6, masked=True),
        Case("cin80_k_chunks", _spec(c_in=80, c_out=96, kernel=3, pad_left=2), t_in=130, hist=2),
        Case("cin80_k_chunks_masked", _spec(c_in=80, c_out=96, kernel=3, pad_left=2), t_in=130, hist=2, masked=True,
             lag=140),
        Case("odd_36_30", _spec(c_in=36, c_out=30, kernel=3, dilation=2, pad_left=4, act_out=KT_ACT_LRELU,
                                act_out_slope=0.2), t_in=150, hist=4, res_first=1),
        Case("odd_36_30_masked", _spec(c_in=36, c_out=30, kernel=3, dilation=2, pad_left=4), t_in=150, hist=4,
             masked=True, rpf=3, lag=5),
        Case("odd_7_5", _spec(c_in=7, c_out=5, kernel=4, pad_left=3), t_in=70, hist=3),
        # taps before the history read 0: pad_left 6 against 2 rows of history
        Case("pad_left_past_history", _spec(c_in=64, c_out=64, kernel=7, pad_left=6), t_in=140, hist=2),
        # taps past the chunk read 0 (the input window's rows after the chunk hold NaN)
        Case("pad_right", _spec(c_in=64, c_out=48, kernel=5, pad_left=2, pad_right=2), t_in=140, hist=2),
        Case("pad_right_masked", _spec(c_in=64, c_out=48, kernel=5, pad_left=2, pad_right=2), t_in=140, hist=2,
             masked=True, rpf=2, lag=3),
        Case("resid_own_pitch", _spec(c_in=64, c_out=64, kernel=3, pad_left=2, act_out=KT_ACT_LRELU, act_out_slope=0.1),
             t_in=260, hist=2, out_first=1, res_first=6, res_pitch_extra=9),
        Case("resid_own_pitch_masked", _spec(c_in=64, c_out=64, kernel=3, pad_left=2), t_in=260, hist=2, out_first=0,
             res_first=5, res_pitch_extra=2, masked=True, rpf=2, lag=1),
        Case("up8", _spec(c_in=64, c_out=32, kernel=7, pad_left=6, upsample=8, **L), t_in=40, hist=1),
        Case("up8_masked", _spec(c_in=64, c_out=32, kernel=7, pad_left=6, upsample=8, **L), t_in=40, hist=1,
             masked=True, rpf=8, lag=12),
        Case("up10", _spec(c_in=64, c_out=32, kernel=11, pad_left=10, upsample=10, **L), t_in=30, hist=1),
        Case("up32_masked", _spec(c_in=64, c_out=64, kernel=7, pad_left=6, upsample=32, **L), t_in=12, hist=1,
             masked=True),
        Case("up32", _spec(c_in=64, c_out=64, kernel=7, pad_left=6, upsample=32, **L), t_in=12, hist=1),
        Case("deconv_k16_s8", _spec(c_in=128, c_out=64, kernel=16, stride=8, transposed=True, crop=8, **L), t_in=40,
             hist=1, res_first=2),
        Case("deconv_k16_s8_masked", _spec(c_in=128, c_out=64, kernel=16, stride=8, transposed=True, crop=8, **L),
             t_in=40, hist=1, masked=True, rpf=2, lag=1),
        Case("deconv_k11_s5", _spec(c_in=64, c_out=32, kernel=11, stride=5, transposed=True, crop=6, **L), t_in=60,
             hist=2),
        Case("deconv_k4_s2", _spec(c_in=64, c_out=32, kernel=4, stride=2, transposed=True, crop=2, **L), t_in=150, hist=1),
        Case("deconv_k4_s2_masked", _spec(c_in=64, c_out=32, kernel=4, stride=2, transposed=True, crop=2, **L),
             t_in=150, hist=1, masked=True, lag=2),
        Case("tanh_out_masked", _spec(c_in=32, c_out=1, kernel=7, pad_left=6, act_out=KT_ACT_TANH, **L), t_in=300,
             hist=6, masked=True, rpf=4, lag=9),
        # thin inputs: K chunks of 4 channels on the exact kernel
        Case("thin_cin2", _spec(c_in=2, c_out=64, kernel=4, stride=2, pad_left=3), t_in=200, hist=3),
        Case("thin_cin2_masked", _spec(c_in=2, c_out=64, kernel=4, stride=2, pad_left=3), t_in=200, hist=3,
             masked=True, rpf=2, lag=3),
        # enough rows x items for 16-row-per-warp tiles (RM 16) of the exact kernel
        Case("rows_4800", _spec(c_in=64, c_out=64, kernel=3, pad_left=2, **L), t_in=4800, hist=2, B=8),
        Case("rows_4800_masked", _spec(c_in=64, c_out=128, kernel=3, pad_left=2, **L), t_in=4800, hist=2, B=8,
             masked=True, rpf=8, lag=20),
        Case("rows_4800_n32_masked", _spec(c_in=32, c_out=32, kernel=3, pad_left=2), t_in=4800, hist=2, B=8,
             masked=True),
    ]
    for c in cases:
        if c.masked and c.B < len(MASK_STATES):
            c.B = len(MASK_STATES)
    return cases


_CASES = None


def all_cases():
    global _CASES
    if _CASES is None:
        _CASES = {c.name: c for c in _synthetic_cases() + _streamer_cases()}
    return _CASES


# ------------------------------------------------------------------------------------------------
# running one case
# ------------------------------------------------------------------------------------------------


class _Alloc:
    """B windows of `pitch` rows x C channels inside one allocation that also holds a guard block before and after them
    (16-byte aligned): .win is the (B, pitch, C) view the kernel gets, .buf all of it."""

    def __init__(self, B, pitch, C, fill):
        self.g = -(-pitch * C // 4) * 4
        self.buf = torch.full((2 * self.g + B * pitch * C,), fill, device=DEV)
        self.win = self.buf[self.g:self.g + B * pitch * C].view(B, pitch, C)


def _outside_utterance(c, lengths, frames_done):
    """(B, hist + t_in) bool: the input window rows outside each slot's utterance."""
    t = torch.arange(-c.hist, c.t_in)
    u = frames_done.long()[:, None] * c.rpf - c.lag + t[None, :]
    return (u < 0) | (u >= lengths.long()[:, None] * c.rpf)


class _Run:
    """Inputs of one case (seeded from its name) and the library call through ops.stream_conv."""

    def __init__(self, c):
        from kantts_b200 import _lib
        from kantts_b200.stream import own_weight
        self.c = c
        s = c.spec
        g = torch.Generator().manual_seed(sum(map(ord, c.name)))
        self.t_out = s.t_out(c.t_in)
        self.in_pitch = c.hist + c.t_in + 2
        self.x = torch.randn(c.B, c.hist + c.t_in, s.c_in, generator=g)
        fan = s.kernel * (s.c_in // s.groups)
        w_shape = (s.c_in, s.c_out, s.kernel) if s.transposed else (s.c_out, s.c_in // s.groups, s.kernel)
        self.w = torch.randn(w_shape, generator=g) / math.sqrt(fan)
        self.bias = 0.3 * torch.randn(s.c_out, generator=g)
        self.resid = None
        if c.res_first >= 0:
            self.res_pitch = c.res_first + self.t_out + c.res_pitch_extra
            self.resid = torch.randn(c.B, self.res_pitch, s.c_out, generator=g)
        self.out_pitch = c.out_first + self.t_out + 2
        self.mask = None
        if c.masked:
            self.lengths, self.frames_done = _mask_table(c, c.B)
            self.outside = _outside_utterance(c, self.lengths, self.frames_done)
            self.mask = (self.lengths, self.frames_done, c.rpf, c.lag)
        self.pw, self.bias_dev = own_weight(s, self.w.to(DEV), None, self.bias.to(DEV))
        self.win = _lib.KtStreamWin(in_pitch=self.in_pitch, in_first=c.hist, out_pitch=self.out_pitch,
                                    out_first=c.out_first, res_pitch=self.res_pitch if self.resid is not None else 0,
                                    res_first=max(c.res_first, 0))

    def window(self, fill):
        """The input window: the chunk and its history, `fill` in the rows outside each slot's utterance (masked cases)
        and NaN in the guard rows after the chunk and around the windows."""
        x = self.x.clone()
        if self.c.masked and fill is not None:
            x[self.outside] = fill
        a = _Alloc(self.c.B, self.in_pitch, self.c.spec.c_in, float("nan"))
        a.win[:, :x.shape[1]] = x.to(DEV)
        return a

    def reference(self, fill=0.0):
        x = self.x.clone()
        if self.c.masked:
            x[self.outside] = fill
        return ref_stream_conv(self.c.spec, x, self.c.hist, self.c.t_in, self.w, self.bias, self.resid,
                               max(self.c.res_first, 0), self.mask)

    def __call__(self, fill=None, masked=None, capture=False):
        """Run the chunk -> (output window (B, out_pitch, c_out) on the CPU, whether everything outside the output chunk
        and both inputs are untouched).  capture: only capture the launch -> the names of the kernels it launches."""
        from kantts_b200._lib import KtStreamMask
        ops, c = _ops(), self.c
        masked = c.masked if masked is None else masked
        xa = self.window(fill)
        x0 = xa.buf.clone()
        ra = r0 = None
        if self.resid is not None:
            ra = _Alloc(c.B, self.res_pitch, c.spec.c_out, float("nan"))
            ra.win.copy_(self.resid.to(DEV))
            r0 = ra.buf.clone()
        sentinel = -7.5e33
        ya = _Alloc(c.B, self.out_pitch, c.spec.c_out, sentinel)
        m = None
        if masked:
            lengths, frames_done = self.lengths.to(DEV), self.frames_done.to(DEV)
            m = KtStreamMask(lengths.data_ptr(), frames_done.data_ptr(), c.rpf, c.lag)
        def launch():
            ops.stream_conv(c.spec, self.pw, self.bias_dev, xa.win, ya.win, c.t_in, self.win,
                            None if ra is None else ra.win, m)
        if capture:
            return _launched_kernels(launch)
        launch()
        torch.cuda.synchronize()
        if masked:   # the conv only reads the utterance record
            assert torch.equal(frames_done.cpu(), self.frames_done) and torch.equal(lengths.cpu(), self.lengths)
        ybuf = ya.buf.cpu()
        written = torch.zeros(ya.buf.numel(), dtype=torch.bool)
        wv = written[ya.g:ya.g + ya.win.numel()].view(ya.win.shape)
        wv[:, c.out_first:c.out_first + self.t_out] = True
        bits = lambda t: t.view(torch.int32)
        untouched = (torch.equal(bits(ybuf[~written]), bits(torch.full((int((~written).sum()),), sentinel)))
                     and torch.equal(bits(xa.buf), bits(x0)) and (ra is None or torch.equal(bits(ra.buf), bits(r0))))
        return ybuf[ya.g:ya.g + ya.win.numel()].view(ya.win.shape)[:, c.out_first:c.out_first + self.t_out], untouched


class _KernelNodeParams(ctypes.Structure):      # CUDA_KERNEL_NODE_PARAMS_v2 of cuda.h
    _fields_ = ([("func", ctypes.c_void_p)] + [(n, ctypes.c_uint) for n in ("gx", "gy", "gz", "bx", "by", "bz", "smem")] +
                [(n, ctypes.c_void_p) for n in ("kernel_params", "extra", "kern", "ctx")])


def _launched_kernels(fn):
    """-> the (mangled) names of the kernels fn launches, read from the kernel nodes of a CUDA graph captured around fn and
    never run.  torch.profiler's kernel records are not used for this: late in a long test session they can be missing
    from many consecutive short sessions, while a captured graph holds every launch."""
    drv = ctypes.CDLL("libcuda.so.1")

    def ok(rc):
        assert rc == 0, f"CUDA driver error {rc}"

    g = torch.cuda.CUDAGraph(keep_graph=True)
    with torch.cuda.graph(g):
        fn()
    graph, n = ctypes.c_void_p(g.raw_cuda_graph()), ctypes.c_size_t(0)
    ok(drv.cuGraphGetNodes(graph, None, ctypes.byref(n)))
    nodes = (ctypes.c_void_p * n.value)()
    ok(drv.cuGraphGetNodes(graph, nodes, ctypes.byref(n)))
    names = []
    for node in nodes:
        kind = ctypes.c_int()
        ok(drv.cuGraphNodeGetType(ctypes.c_void_p(node), ctypes.byref(kind)))
        if kind.value != 0:                                 # CU_GRAPH_NODE_TYPE_KERNEL
            continue
        prm, name = _KernelNodeParams(), ctypes.c_char_p()
        ok(drv.cuGraphKernelNodeGetParams_v2(ctypes.c_void_p(node), ctypes.byref(prm)))
        ok(drv.cuFuncGetName(ctypes.byref(name), ctypes.c_void_p(prm.func)) if prm.func else
           drv.cuKernelGetName(ctypes.byref(name), ctypes.c_void_p(prm.kern)))
        names.append(name.value.decode())
    return names


def _mangled(name):
    """'conv_core_kernel<1, 16, 16, true, false>' -> 'conv_core_kernelILi1ELi16ELi16ELb1ELb0EE', how the instance's template
    arguments (int and bool values) appear in its Itanium-mangled name."""
    base, args = name[:-1].split("<")
    return base + "I" + "".join({"true": "Lb1E", "false": "Lb0E"}.get(a, f"Li{a}E") for a in args.split(", ")) + "E"


def _routes(c):
    """-> [(route name, force_ffma, expected kernel names)]: the exact route, and the default one when it differs."""
    out = [("ffma", True, core_instances(c))]
    tc = tc_instance(c)
    if tc is not None:
        out.append(("tc", False, [tc]))
    return out


# ------------------------------------------------------------------------------------------------
# GPU tests of the stream conv
# ------------------------------------------------------------------------------------------------


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(all_cases()))
def test_stream_conv_matches_float64(name):
    ops = _ops()
    c = all_cases()[name]
    run = _Run(c)
    fill = float("nan") if c.masked else None
    want, scale = run.reference()
    try:
        for route, force, kernels in _routes(c):
            ops.set_force_ffma(force)
            y, untouched = run(fill)
            assert untouched, (route, "wrote outside its output chunk or changed an input")
            # the conv kernels of the call are exactly the instances the case is named for
            convs = [k for k in run(fill, capture=True) if "conv_core_kernelI" in k or "conv_tc_kernelI" in k]
            named = [_mangled(k) for k in kernels]
            assert (all(any(w in k for k in convs) for w in named) and all(any(w in k for w in named) for k in convs)), \
                (route, kernels, convs)
            if c.masked:
                # selection, bit for bit: NaN / 1e30 / zeros outside the utterances, and the unmasked instance on zeros
                y_big, ok1 = run(1e30)
                y_zero, ok2 = run(0.0)
                y_plain, ok3 = run(0.0, masked=False)
                assert ok1 and ok2 and ok3
                for other, what in ((y_big, "1e30"), (y_zero, "zeros"), (y_plain, "unmasked on zeros")):
                    assert torch.equal(y.view(torch.int32), other.view(torch.int32)), (route, what)
                # a slot none of whose window rows lies in its utterance writes act_out(bias) + resid, in fp32
                empty = run.outside.all(1)
                assert bool(empty[[MASK_STATES.index("idle") + k for k in range(0, c.B, len(MASK_STATES))]].all())
                b = run.bias.to(DEV)
                if c.spec.act_out == KT_ACT_LRELU:
                    b = torch.where(b > 0, b, b * c.spec.act_out_slope)
                elif c.spec.act_out == KT_ACT_TANH:
                    b = torch.tanh(b)
                idle = b.expand(c.B, run.t_out, -1)
                if run.resid is not None:
                    idle = idle + run.resid[:, c.res_first:c.res_first + run.t_out].to(DEV)
                assert torch.equal(y[empty].view(torch.int32), idle.cpu()[empty].view(torch.int32)), route
            err = (y.to(F64) - want).abs()
            ratio = float((err / scale.clamp_min(1e-300)).max())
            l2 = rel_l2(y, want)
            print(f"stream_conv {name} {route} {' '.join(kernels)} elem {ratio:.3e} rel_l2 {l2:.3e}")
            assert bool((err <= ELEM_BOUND[route] * scale).all()), (route, ratio)
            assert l2 <= L2_BOUND[route], (route, l2)
    finally:
        ops.set_force_ffma(False)


def test_cases_cover_every_stream_instance():
    """Together the cases launch all four stream conv_tc_kernel instances and, masked and unmasked, conv_core_kernel with
    every RN, both KC and RM 4 and 16 (each case's own test confirms its instances from a captured launch)."""
    cases = all_cases().values()
    tc = {tc_instance(c) for c in cases} - {None}
    assert tc == {f"conv_tc_kernel<{r}, true, {m}>" for r in (0, 1) for m in ("false", "true")}, tc
    core = {k for c in cases for k in core_instances(c)}
    for m in ("false", "true"):
        mine = [k[len("conv_core_kernel<"):-1].split(", ") for k in core if k.endswith(f"{m}>")]
        assert {rn for rn, *_ in mine} == {"1", "2", "4"}, (m, mine)
        assert {kc for _, _, kc, *_ in mine} == {"4", "16"}, (m, mine)
        assert {"4", "16"} <= {rm for _, rm, *_ in mine}, (m, mine)
    # the case the int overflow of an up-sampled utterance bound needs: a masked tensor-core conv up-sampling by 32
    assert tc_instance(all_cases()["up32_masked"]) == "conv_tc_kernel<1, true, true>"


def test_mask_table_states():
    """Each mask state is what its name says, for the synthetic cases' rows per frame and lags."""
    for c in all_cases().values():
        if not c.masked:
            continue
        lengths, fd = _mask_table(c, len(MASK_STATES))
        t = torch.arange(-c.hist, c.t_in)
        u = fd.long()[:, None] * c.rpf - c.lag + t[None, :]
        inside = (u >= 0) & (u < lengths.long()[:, None] * c.rpf)
        st = dict(zip(MASK_STATES, inside))
        assert bool(st["inside"].all()) and bool(st["long_running_mid"].all()), c.name
        for k in ("idle", "starts_past_2^26", "long_running_ended"):
            assert not bool(st[k].any()), (c.name, k)
        assert int(fd[MASK_STATES.index("long_running_mid")]) * c.rpf > 2 ** 31 or c.rpf == 1
        assert int(fd[MASK_STATES.index("starts_past_2^26")]) * c.rpf - c.lag <= -(2 ** 26)
        H, n = c.hist, c.t_in
        if n >= 2 * c.rpf:
            assert bool(st["starts_mid_chunk"][-1]) and not bool(st["starts_mid_chunk"][:H + n // 2].any()), c.name
            assert bool(st["ends_mid_chunk"][:H + 1].all()) and not bool(st["ends_mid_chunk"][H + n // 2:].any()), c.name
        e = st["ended_in_history"]
        assert not bool(e[H:].any()) and (H < c.rpf or bool(e[:H].any())), c.name


# ------------------------------------------------------------------------------------------------
# window kernels: advance, reset, mask advance, sin-add and three-way add into a window
# ------------------------------------------------------------------------------------------------


def _window_table(specs, B, g):
    """-> (windows [(base tensor (B, pitch, C)) ...], device KtWindow table) for specs [(channels, history, rpf, pitch)]."""
    from kantts_b200._lib import KtWindow
    bufs = [torch.randn(B, pitch, ch, generator=g).to(DEV) for ch, _, _, pitch in specs]
    table = (KtWindow * len(specs))(*[KtWindow(base=b.data_ptr(), pitch=p, channels=ch, history=h, rows_per_frame=r)
                                      for b, (ch, h, r, p) in zip(bufs, specs)])
    return bufs, torch.frombuffer(bytearray(bytes(table)), dtype=torch.uint8).to(DEV)


# (channels, history, rows per frame, pitch): with 3 frames a chunk is 3 * rpf rows, so the histories sit below (5 < 6,
# 100 < 240), at (24 = 24) and above (300 > 30, 7 > 3) the chunk's rows; channels 300 needs three 128-channel blocks
ADV_WINDOWS = [(300, 5, 2, 5 + 6 + 3), (64, 24, 8, 24 + 24), (3, 300, 10, 300 + 30 + 1), (129, 7, 1, 7 + 3),
               (17, 100, 80, 100 + 240)]


@pytest.mark.gpu
def test_stream_advance_matches_torch():
    from kantts_b200._lib import ptr
    g = torch.Generator().manual_seed(11)
    B, frames = 3, 3
    bufs, table = _window_table(ADV_WINDOWS, B, g)
    before = [b.cpu() for b in bufs]
    _ops().call("kt_stream_advance", ptr(table, True), len(ADV_WINDOWS), B, frames, 400)
    torch.cuda.synchronize()
    for (ch, h, rpf, _), b0, b in zip(ADV_WINDOWS, before, bufs):
        want = b0.clone()
        r = frames * rpf
        want[:, :h] = b0[:, r:r + h]
        assert torch.equal(b.cpu(), want), (ch, h, rpf)


@pytest.mark.gpu
def test_stream_reset_zeroes_only_the_selected_slots_history():
    from kantts_b200._lib import ptr
    g = torch.Generator().manual_seed(12)
    B = 5
    bufs, table = _window_table(ADV_WINDOWS, B, g)
    before = [b.cpu() for b in bufs]
    slots = torch.tensor([1, 0, 0, 1, 1], dtype=torch.uint8)
    _ops().call("kt_stream_reset", ptr(table, True), len(ADV_WINDOWS), B, ptr(slots.to(DEV), True), 400)
    torch.cuda.synchronize()
    for (ch, h, _, _), b0, b in zip(ADV_WINDOWS, before, bufs):
        want = b0.clone()
        want[slots.bool(), :h] = 0
        assert torch.equal(b.cpu(), want), (ch, h)


@pytest.mark.gpu
@pytest.mark.parametrize("rpf,lag", [(1, 0), (1, 30), (4, 6), (8, 3)])
def test_stream_mask_advance_matches_torch(rpf, lag):
    """Rows [first, first + rows) of each slot are zeroed outside its utterance (the MASK_STATES table), every other row
    is untouched, and frames_done += frames for every slot."""
    from kantts_b200._lib import KtStreamMask, ptr
    g = torch.Generator().manual_seed(rpf * 100 + lag)
    frames, first, ch = 3, 5, 33
    rows = frames * rpf
    c = Case("mask_advance", None, t_in=rows, hist=first, rpf=rpf, lag=lag)
    B = 2 * len(MASK_STATES)
    lengths, fd = _mask_table(c, B)
    y0 = torch.randn(B, first + rows + 4, ch, generator=g)
    y = y0.to(DEV)
    ld, fdd = lengths.to(DEV), fd.to(DEV)
    m = KtStreamMask(ld.data_ptr(), fdd.data_ptr(), rpf, lag)
    _ops().call("kt_stream_mask_advance", ctypes.byref(m), ptr(y), B, rows, ch, y.shape[1], first, frames)
    torch.cuda.synchronize()
    t = torch.arange(rows)
    u = fd.long()[:, None] * rpf - lag + t[None, :]
    out = (u < 0) | (u >= lengths.long()[:, None] * rpf)
    want = y0.clone()
    want[:, first:first + rows][out] = 0
    assert bool(out.any()) and not bool(out.all())
    assert torch.equal(y.cpu(), want)
    assert torch.equal(fdd.cpu(), fd + frames) and torch.equal(ld.cpu(), lengths)


@pytest.mark.gpu
@pytest.mark.parametrize("B,rows,ch,x_pitch,y_pitch,y_first", [(3, 37, 5, 40, 45, 6), (2, 1, 128, 9, 3, 2),
                                                             (4, 200, 64, 200, 210, 10)])
def test_sinadd_win_within_sinf_accuracy(B, rows, ch, x_pitch, y_pitch, y_first):
    """y = v + sinf(v): CUDA documents sinf to 2 ulp, and the sum rounds once more (half an ulp of y).  Measured on an H100:
    at most 1.11 ulp of y."""
    from kantts_b200._lib import ptr
    g = torch.Generator().manual_seed(rows + ch)
    x = (3 * torch.randn(B, x_pitch, ch, generator=g))
    y0 = torch.randn(B, y_pitch, ch, generator=g)
    y = y0.to(DEV)
    _ops().call("kt_sinadd_fwd_win", ptr(x.to(DEV)), ptr(y), B, rows, ch, x_pitch, y_pitch, y_first)
    got = y.cpu()
    want = y0.clone()
    v = x[:, :rows].to(F64)
    exact = v + torch.sin(v)
    inside = got[:, y_first:y_first + rows]

    def ulp(t):
        t = t.float()
        return (torch.nextafter(t.abs(), torch.tensor(float("inf"))) - t.abs()).to(F64)

    err = (inside.to(F64) - exact).abs()
    assert bool((err <= 0.5 * ulp(inside) + 2 * ulp(torch.sin(v))).all()), float((err / ulp(exact)).max())
    want[:, y_first:y_first + rows] = inside
    assert torch.equal(got, want)                          # the rest of the window untouched


@pytest.mark.gpu
@pytest.mark.parametrize("nb", [1, 2, 3])
@pytest.mark.parametrize("B,rows,ch,x_pitch,y_pitch,y_first", [(3, 37, 5, 40, 45, 6), (2, 300, 64, 310, 305, 4)])
def test_add3_scale_win_matches_torch(nb, B, rows, ch, x_pitch, y_pitch, y_first):
    from kantts_b200._lib import ptr
    g = torch.Generator().manual_seed(nb * 1000 + rows)
    srcs = [torch.randn(B, x_pitch, ch, generator=g) for _ in range(nb)]
    y0 = torch.randn(B, y_pitch, ch, generator=g)
    y = y0.to(DEV)
    dev = [s.to(DEV) for s in srcs] + [None] * (3 - nb)
    scale = 1.0 / 3.0
    _ops().call("kt_add3_scale_win", ptr(dev[0]), ptr(dev[1]), ptr(dev[2]), scale, ptr(y), B, rows, ch, x_pitch, y_pitch,
                y_first)
    zero = torch.zeros(B, rows, ch)
    a, b, c = [s[:, :rows] for s in srcs] + [zero] * (3 - nb)
    want = y0.clone()
    want[:, y_first:y_first + rows] = torch.tensor(scale, dtype=torch.float32) * ((a + b) + c)
    assert torch.equal(y.cpu(), want)
