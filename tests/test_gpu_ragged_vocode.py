"""Ragged batches through the whole-utterance generator: the masked forward instances (kt_conv1d_fwd_masked,
kt_conv1d_fwd_tc_masked, kt_resblock_fwd_masked, kt_rows_mask) and Generator.forward(..., lengths=) /
PQMF.synthesis(..., lengths=).

Kernel level: every route of the masked conv forward -- exact fp32 (conv_core_kernel<..., false, true>), the TMA-fed
tensor-core route (split_planes_masked_kernel + the unmasked TMA instance), the register-staged simple and generic instances
(conv_tc[_bf16]_kernel<ROUTE, false, true>), the transposed-conv phases and the fused ResBlock pair -- on both tensor-core
precisions.  Each masked call must give the bits of the unmasked call of the same route on the input whose rows past each
item's end are zeroed, whatever those rows hold (NaN included), and both must lie within the path's bound of a float64
reference.  The instance each case runs is pinned: the route by kt_debug_conv_tc_plan, simple against generic by the
host's instance predicate (launch_route in conv_tc.cu) on the planned N tile.

Module level: each item of a permuted ragged batch -- one short item against a long one, one shorter than the receptive
field -- against the same item alone, bit for bit on all three paths: every route and N tile sums each output's products in
the same order whatever the batch, so a batch of one and a batch of four give the same bits even where they plan different
routes.  Samples past each item's end are zero, and lengths = [T] * B gives the unmasked forward's bits.  And
synthesize(per_item=True) gives each utterance the generator (and the PQMF) on exactly its own post-net frames.
"""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import kantts_b200 as K
from kantts_b200 import _lib, ops
from kantts_b200._lib import KT_ACT_LRELU, KT_ACT_TANH, KT_PATH_AUTO, KT_PATH_BF16, KT_PATH_FFMA

pytestmark = pytest.mark.gpu
DEV = "cuda"
F64 = torch.float64
PATHS = {"ffma": KT_PATH_FFMA, "bf16x3": KT_PATH_AUTO, "bf16": KT_PATH_BF16}
# per-element error over the error scale sum |w| |x| + |bias| + |resid| (any summation order meets it): the suite's bounds
ELEM_BOUND = {"ffma": 2e-6, "bf16x3": 6e-5, "bf16": 2 * 2.0 ** -8}
OBSERVED = {}


def _record(key, value):
    """Print the largest observed difference per key (run with -s to see the worst case of each path)."""
    OBSERVED[key] = max(OBSERVED.get(key, 0.0), float(value))
    print(f"observed {key}: {OBSERVED[key]:.3e}")


def _zero_tail(x, lengths, rate):
    t = torch.arange(x.shape[1], device=x.device)[None, :, None]
    return torch.where(t < (lengths.long() * rate)[:, None, None], x, torch.zeros((), dtype=x.dtype, device=x.device))


def _ref_conv(spec, x, w, bias, resid):
    """float64 (y, scale) of ConvSpec `spec` on channels-last x (B, T, C); w in the reference layout."""
    def run(xx, ww, bb):
        xx = xx.transpose(1, 2)
        if spec.upsample > 1:
            xx = xx.repeat_interleave(spec.upsample, dim=2)
        if spec.transposed:
            y = F.conv_transpose1d(xx, ww, bb, stride=spec.stride, padding=spec.pad_left)
            y = y[:, :, : spec.t_out(x.shape[1])]
        else:
            xx = F.pad(xx, (spec.pad_left, spec.pad_right))
            y = F.conv1d(xx, ww, bb, stride=spec.stride, dilation=spec.dilation, groups=spec.groups)
        return y.transpose(1, 2)
    x64 = x.to(F64)
    if spec.act_in == KT_ACT_LRELU:
        x64 = torch.where(x64 > 0, x64, x64 * spec.act_in_slope)
    b64 = None if bias is None else bias.to(F64)
    y = run(x64, w.to(F64), b64)
    scale = run(x64.abs(), w.to(F64).abs(), None if b64 is None else b64.abs())
    if spec.act_out == KT_ACT_TANH:
        y = torch.tanh(y)
    if resid is not None:
        y, scale = y + resid.to(F64), scale + resid.to(F64).abs()
    return y, scale


# name: (ConvSpec kwargs, batch, T, rows per frame of the input, residual, expected tensor-core instance:
# "tma" | "simple" | "generic")
CONV_CASES = {
    # the 16 kHz generator's first stage: 256 -> 128 x10 repeat-upsample conv (generic register-staged instance)
    "upsample_generic": (dict(c_in=256, c_out=128, kernel=7, pad_left=3, pad_right=3, upsample=10, act_in=KT_ACT_LRELU,
                              act_in_slope=0.1), 3, 60, 1, True, "generic"),
    # a resblock conv at 64 channels (register-staged simple instance: too few elements for the split pass)
    "resblock_simple": (dict(c_in=64, c_out=64, kernel=7, dilation=3, pad_left=9, pad_right=9, act_in=KT_ACT_LRELU,
                             act_in_slope=0.1), 2, 3000, 100, False, "simple"),
    # conv_pre of the 24 kHz generator at 1700 frames x 4 items (TMA-fed: split pass masked)
    "conv_pre_tma": (dict(c_in=80, c_out=512, kernel=7, pad_left=3, pad_right=3), 4, 1700, 1, False, "tma"),
    # a resblock conv at 256 channels (TMA-fed, two N tiles)
    "wide_tma": (dict(c_in=256, c_out=256, kernel=3, dilation=5, pad_left=5, pad_right=5, act_in=KT_ACT_LRELU,
                      act_in_slope=0.1), 3, 1200, 40, True, "tma"),
    # the non-causal transposed upsampler 512 -> 256, k 16 s 8 (polyphase phases, register-staged simple instance)
    "transposed": (dict(c_in=512, c_out=256, kernel=16, stride=8, pad_left=4, transposed=True, act_in=KT_ACT_LRELU,
                        act_in_slope=0.1), 3, 70, 1, True, "simple"),
    # NSF source_downs: c_in = 1, kernel 2u stride u, with the residual (exact fp32 core)
    "source_down": (dict(c_in=1, c_out=64, kernel=20, stride=10, pad_left=5, pad_right=5), 3, 800, 80, True, "ffma"),
    # conv_post 32 -> 1 with the fused tanh (register-staged generic instance)
    "conv_post": (dict(c_in=32, c_out=1, kernel=7, pad_left=3, pad_right=3, act_in=KT_ACT_LRELU, act_in_slope=0.01,
                       act_out=KT_ACT_TANH), 3, 4000, 200, False, "generic"),
}


def _instance(spec, batch, t):
    """The tensor-core instance a forward of `spec` runs: "ffma" off the tensor cores, "tma", or the register-staged "simple" /
    "generic" instance -- launch_route's predicate (nsub 1, no up-sampling, contraction channels % 8, channel counts and N
    tile % 4, no tanh; a forward never accumulates) on the plan's N tile (a dense layer's N stride)."""
    if spec.plan(batch, 1, t).tile(0) == 0:
        return "ffma"
    d = spec.desc(batch, 1, t)
    out = (ctypes.c_int64 * 9)()
    _lib.load().kt_debug_conv_tc_plan(ctypes.byref(d), 0, out)
    if out[1]:
        return "tma"
    assert spec.groups == 1
    simple = (spec.upsample == 1 and spec.c_in % 8 == 0 and spec.c_out % 4 == 0 and out[0] % 4 == 0
              and spec.act_out != KT_ACT_TANH)
    return "simple" if simple else "generic"


@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("case", list(CONV_CASES))
def test_masked_conv_instance(case, path):
    kw, B, T, rate, with_resid, route = CONV_CASES[case]
    spec = ops.ConvSpec(**kw, path=PATHS[path])
    assert _instance(spec, B, T) == ("ffma" if path == "ffma" else route), (case, path, _instance(spec, B, T))
    g = torch.Generator().manual_seed(7)
    wshape = (spec.c_in, spec.c_out, spec.kernel) if spec.transposed else (spec.c_out, spec.c_in // spec.groups, spec.kernel)
    w = (torch.randn(wshape, generator=g) / (spec.c_in * spec.kernel) ** 0.5).to(DEV)
    bias = (0.1 * torch.randn(spec.c_out, generator=g)).to(DEV)
    x = torch.randn(B, T, spec.c_in, generator=g).to(DEV)
    frames = T // rate
    lengths = torch.tensor([frames, 1, max(1, frames // 3)][:B] + [frames - 1] * (B - 3), dtype=torch.int32, device=DEV)[:B]
    t_out = spec.t_out(T)
    resid = torch.randn(B, t_out, spec.c_out, generator=g).to(DEV) if with_resid else None
    xz = _zero_tail(x, lengths, rate)
    keep = _zero_tail(torch.ones_like(x), lengths, rate) != 0
    x_nan = torch.where(keep, x, torch.full_like(x, float("nan")))     # rows past an item's end must never be read
    cache = ops.PreparedWeight()
    m = ops.utterance_mask(lengths, rate)
    with torch.no_grad():
        ym = ops.conv(x_nan, spec, cache, w, None, bias, resid, mask=m)
        yu = ops.conv(xz, spec, cache, w, None, bias, resid)
    torch.cuda.synchronize()
    assert torch.equal(ym, yu), (case, path, (ym - yu).abs().max().item())
    ref, scale = _ref_conv(spec, xz.cpu(), w.cpu(), bias.cpu(), None if resid is None else resid.cpu())
    err = ((ym.cpu().to(F64) - ref).abs() / scale.clamp_min(1e-30)).max().item()
    _record(f"conv:{path}", err)
    assert err <= ELEM_BOUND[path], (case, path, err)


@pytest.mark.parametrize("path", ["bf16x3", "bf16"])
@pytest.mark.parametrize("channels,kernel,dilation", [(32, 11, 5), (64, 7, 3), (32, 3, 1)])
def test_masked_resblock_pair_matches_item_alone(channels, kernel, dilation, path):
    """The fused pair masked over a ragged batch: each item's rows before its end are the bits of the pair on that item
    alone (the same tiles), and both lie within the path's bound of the float64 pair on the zero-padded item."""
    ps = PATHS[path]
    s1 = ops.ConvSpec(c_in=channels, c_out=channels, kernel=kernel, dilation=dilation, pad_left=(kernel - 1) * dilation // 2,
                      pad_right=(kernel - 1) * dilation // 2, act_in=KT_ACT_LRELU, act_in_slope=0.1, path=ps)
    s2 = ops.ConvSpec(c_in=channels, c_out=channels, kernel=kernel, pad_left=(kernel - 1) // 2, pad_right=(kernel - 1) // 2,
                      act_in=KT_ACT_LRELU, act_in_slope=0.1, path=ps)
    g = torch.Generator().manual_seed(3)
    w1, w2 = [(torch.randn(channels, channels, kernel, generator=g) / (channels * kernel) ** 0.5).to(DEV) for _ in range(2)]
    b1, b2 = [(0.1 * torch.randn(channels, generator=g)).to(DEV) for _ in range(2)]
    B, T = 4, 700
    lengths = [700, 9, 333, 121]
    x = torch.randn(B, T, channels, generator=g).to(DEV)
    c1, c2 = ops.PreparedWeight(), ops.PreparedWeight()
    rd = ops.resblock_desc(s1, s2, B, T)
    assert rd is not None
    with torch.no_grad():
        L = torch.tensor(lengths, dtype=torch.int32, device=DEV)
        y = ops.resblock(x, s1, c1, w1, None, b1, s2, c2, w2, None, b2, rd, ops.utterance_mask(L, 1))
        for b, n in enumerate(lengths):
            rd1 = ops.resblock_desc(s1, s2, 1, n)
            assert rd1 is not None
            ya = ops.resblock(x[b:b + 1, :n].contiguous(), s1, c1, w1, None, b1, s2, c2, w2, None, b2, rd1)
            assert torch.equal(y[b, :n], ya[0]), (b, (y[b, :n] - ya[0]).abs().max().item())
            xa = x[b:b + 1, :n].cpu()
            h, sh = _ref_conv(s1, xa, w1.cpu(), b1.cpu(), None)
            yr, sy = _ref_conv(s2, h, w2.cpu(), b2.cpu(), xa)
            err = ((ya[0].cpu().to(F64) - yr[0]).abs() / (sy[0] + sh.abs().max()).clamp_min(1e-30)).max().item()
            _record(f"resblock:{path}", err)
            assert err <= 4 * ELEM_BOUND[path], (b, err)


def test_rows_mask_zeroes_past_each_end():
    y = torch.randn(3, 50, 4, device=DEV)
    L = torch.tensor([10, 1, 5], dtype=torch.int32, device=DEV)
    want = _zero_tail(y, L, 5)
    ops.rows_mask(y, ops.utterance_mask(L, 5))
    assert torch.equal(y, want)


# ------------------------------------------------------------------------------------------------
# generators
# ------------------------------------------------------------------------------------------------
_LRELU = {"nonlinear_activation": "LeakyReLU", "nonlinear_activation_params": {"negative_slope": 0.1}}
GENERATORS = {
    "class_default": dict(),
    "v1_24k": dict(channels=512, upsample_scales=[8, 5, 3, 2], upsample_kernal_sizes=[16, 10, 6, 4],
                   resblock_kernel_sizes=[3, 7, 11], resblock_dilations=[[1, 3, 5]] * 3, **_LRELU),
    "noncausal_v1_16k": dict(channels=256, upsample_scales=[10, 5, 2, 2], upsample_kernal_sizes=[20, 11, 4, 4],
                             resblock_kernel_sizes=[3, 7, 11], resblock_dilations=[[1, 3, 5, 7]] * 3, causal=False, **_LRELU),
    "nsf_24k": dict(channels=512, upsample_scales=[8, 5, 3, 2], upsample_kernal_sizes=[16, 10, 6, 4],
                    resblock_kernel_sizes=[3, 7, 11], resblock_dilations=[[1, 3, 5]] * 3,
                    nsf_params={"nb_harmonics": 7, "sampling_rate": 24000}, **_LRELU),
    "noncausal_nsf_global_16k": dict(channels=256, upsample_scales=[10, 5, 2, 2], upsample_kernal_sizes=[20, 11, 4, 4],
                                     resblock_kernel_sizes=[3, 7, 11], resblock_dilations=[[1, 3, 5, 7]] * 3, causal=False,
                                     nsf_params={"nb_harmonics": 7, "sampling_rate": 16000}, **_LRELU),
    "multiband_24k": dict(out_channels=4, channels=512, upsample_scales=[5, 3, 2, 2], upsample_kernal_sizes=[10, 6, 4, 4],
                          resblock_kernel_sizes=[3, 7, 11], resblock_dilations=[[1, 3, 5]] * 3, **_LRELU),
}
# permuted: a long item, one shorter than the receptive field, one short against the long one, one in between
LENGTHS = [3, 41, 17, 2]


def _gen(name, path):
    torch.manual_seed(11)
    gen = K.Generator(**GENERATORS[name]).to(DEV).eval()
    with torch.no_grad():      # weights of a trained scale: the random init's weight_g gives near-silent output
        for p in gen.parameters():
            p.mul_(1.0 + 0.5 * torch.rand_like(p))
    if path == "bf16":
        K.set_precision(gen, "bf16")
    pq = K.PQMF(4).to(DEV) if gen.out_channels > 1 else None
    return gen, pq


def _mel(gen, B, T):
    g = torch.Generator().manual_seed(5)
    cin = gen.conv_pre.conv1d.spec.c_in
    mel = torch.randn(B, cin, T, generator=g)
    if gen.nsf_enable:
        f0 = 100 + 200 * torch.rand(B, 1, T, generator=g)
        uv = (torch.rand(B, 1, T, generator=g) > 0.3).float()
        mel = torch.cat([mel, f0, uv], 1)
    return mel.to(DEV)


def _vocode(gen, pq, x, seeds, lengths=None):
    y = gen(x, nsf_seeds=seeds, lengths=lengths)
    if pq is not None:
        y = pq.synthesis(y, None if lengths is None else [int(n) * int(np.prod(gen.upsample_scales)) for n in lengths])
    return y


@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("name", list(GENERATORS))
def test_ragged_generator_matches_each_item_alone(name, path):
    gen, pq = _gen(name, path)
    B, T = len(LENGTHS), max(LENGTHS)
    x = _mel(gen, B, T)
    seeds = [101, 7, 55, 3] if gen.nsf_enable else None
    hop = int(np.prod(gen.upsample_scales)) * gen.out_channels
    ops.set_force_ffma(path == "ffma")
    try:
        with torch.no_grad():
            y = _vocode(gen, pq, x, seeds, LENGTHS)
            assert y.shape == (B, 1, T * hop)
            full = _vocode(gen, pq, x, seeds, [T] * B)
            plain = _vocode(gen, pq, x, seeds)
            assert torch.equal(full, plain), (full - plain).abs().max().item()
            for b, n in enumerate(LENGTHS):
                alone = _vocode(gen, pq, x[b:b + 1, :, :n].contiguous(), None if seeds is None else [seeds[b]])
                got = y[b:b + 1, :, : alone.shape[2]]
                assert alone.shape[2] == n * hop
                assert not torch.any(y[b, :, alone.shape[2]:]), (b, "samples past the item's end")
                assert torch.equal(got, alone), (name, path, b, n, (got - alone).abs().max().item())
            assert alone.abs().max() > 1e-3        # the comparison is not between silences
    finally:
        ops.set_force_ffma(False)


def test_masked_forward_refuses_autograd():
    gen, _ = _gen("class_default", "bf16x3")
    x = _mel(gen, 2, 6)
    with pytest.raises(RuntimeError, match="inference only"):
        gen(x, lengths=[6, 3])


# ------------------------------------------------------------------------------------------------
# synthesize(per_item=True)
# ------------------------------------------------------------------------------------------------
SYN_GENERATORS = {
    # a non-causal full-band generator, a non-causal NSF one (mel + f0 + uv) and a causal multi-band one with its PQMF
    "noncausal": dict(channels=32, upsample_scales=[4, 2], upsample_kernal_sizes=[8, 4], resblock_kernel_sizes=[3, 7],
                      resblock_dilations=[[1, 3], [1, 3]], causal=False),
    "nsf_noncausal": dict(channels=32, upsample_scales=[4, 2], upsample_kernal_sizes=[8, 4], resblock_kernel_sizes=[3, 7],
                          resblock_dilations=[[1, 3], [1, 3]], causal=False,
                          nsf_params={"nb_harmonics": 7, "sampling_rate": 16000}),
    "multiband": dict(out_channels=4, channels=32, upsample_scales=[5, 3, 2, 2], upsample_kernal_sizes=[10, 6, 4, 4],
                      resblock_kernel_sizes=[3, 7], resblock_dilations=[[1, 3], [1, 3]]),
}


@pytest.mark.parametrize("path", ["ffma", "bf16x3"])
@pytest.mark.parametrize("name", list(SYN_GENERATORS))
def test_synthesize_per_item_is_the_generator_on_each_items_own_frames(golden, name, path):
    """Each waveform of synthesize(per_item=True) is the generator -- with the same seed and the denormalised f0 for NSF, then
    the PQMF for multi-band -- on exactly that utterance's post-net frames, bit for bit; and for the non-causal generators
    the padded default differs from it in a shorter utterance's last samples."""
    from golden.make_batch import make_sambert_batch
    from kantts_b200.infer import denorm_f0
    g = golden("sambert_small_infer")
    nsf = "nsf" in name
    cfg = dict(g.cfg, num_mels=g.cfg["num_mels"] + 2) if nsf else g.cfg
    torch.manual_seed(1234)
    am = K.KanTtsSAMBERT(cfg)
    if nsf:
        with torch.no_grad():
            am.variance_adaptor.duration_predictor.fc.bias.fill_(1.5)
    else:
        am.load_state_dict(g.group("sd/"), strict=True)
    am = am.to(DEV).eval()
    batch = make_sambert_batch(cfg, B=3, L=9, gen=torch.Generator().manual_seed(31), short=3)
    inputs = [batch[k].to(DEV) for k in ("inputs_ling", "inputs_emotion", "inputs_speaker", "input_lengths")]
    torch.manual_seed(7)
    gen = K.Generator(in_channels=g.cfg["num_mels"], **SYN_GENERATORS[name]).to(DEV).eval()
    with torch.no_grad():
        for p in gen.parameters():
            p.mul_(1.0 + 0.5 * torch.rand_like(p))
    if gen.out_channels > 1:
        gen.pqmf = K.PQMF(4).to(DEV)
    kw = dict(nsf_f0=("mean_std", 180.0, 40.0), nsf_seeds=[11, 12, 13]) if nsf else {}
    ops.set_force_ffma(path == "ffma")
    try:
        with torch.no_grad(), torch.backends.cudnn.flags(enabled=False):
            wavs, res = K.synthesize(am, gen, *inputs, per_item=True, **kw)
            padded, _ = K.synthesize(am, gen, *inputs, **kw)
            frames = [int(n) for n in res["LR_length_rounded"].tolist()]
            assert len(set(frames)) > 1, frames
            mel = res["postnet_outputs"]
            x = (denorm_f0(mel, kw["nsf_f0"]) if nsf else mel).transpose(1, 2)
            hop = int(np.prod(gen.upsample_scales)) * gen.out_channels
            tails_differ = False
            for b, n in enumerate(frames):
                alone = gen(x[b:b + 1, :, :n].contiguous(), nsf_seeds=[kw["nsf_seeds"][b]] if nsf else None)
                if gen.out_channels > 1:
                    alone = gen.pqmf.synthesis(alone)
                assert wavs[b].shape == (n * hop,)
                assert torch.equal(wavs[b], alone[0, 0]), (b, (wavs[b] - alone[0, 0]).abs().max().item())
                tails_differ |= not torch.equal(padded[b], wavs[b])
            assert alone.abs().max() > 1e-3
            assert tails_differ    # the padded batch reads past a shorter utterance's end (every generator here looks ahead)
    finally:
        ops.set_force_ffma(False)
