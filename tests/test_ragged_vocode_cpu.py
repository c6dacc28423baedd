"""CPU: ragged batches through the whole-utterance generator (Generator.forward(..., lengths=)) as far as they go without a
GPU -- the validation of ``lengths``, the inference-only refusals, and the rows-per-frame bound each conv of every shipped
vocoder reads its input under (recorded through stand-ins for the library calls, which need a device): every layer's input
has lengths[b] * rate rows for item b, and with ``lengths=None`` no call sees a mask."""
import json
import os

import pytest
import torch

import kantts_b200 as K
from kantts_b200 import hifigan, ops, pqmf

_LRELU = {"nonlinear_activation": "LeakyReLU", "nonlinear_activation_params": {"negative_slope": 0.1}}
_NSF16 = {"nb_harmonics": 7, "sampling_rate": 16000}
# Model.Generator.params of the shipped vocoder yamls (kantts/configs/hifigan_*.yaml), plus the multi-band 24 kHz generator
# the multi-band tests build (out_channels = 4, with a PQMF)
GENERATORS = {
    "v1_8k": dict(channels=256, upsample_scales=[5, 5, 2, 2], upsample_kernal_sizes=[10, 10, 4, 4],
                  resblock_dilations=[[1, 3, 5, 7]] * 3, causal=True),
    "v1_16k": dict(channels=256, upsample_scales=[10, 5, 2, 2], upsample_kernal_sizes=[20, 10, 4, 4],
                   resblock_dilations=[[1, 3, 5, 7]] * 3, causal=True),
    "noncausal_v1_16k": dict(channels=256, upsample_scales=[10, 5, 2, 2], upsample_kernal_sizes=[20, 11, 4, 4],
                             resblock_dilations=[[1, 3, 5, 7]] * 3, causal=False),
    "noncausal_nsf_v1_16k": dict(channels=256, upsample_scales=[10, 5, 2, 2], upsample_kernal_sizes=[20, 11, 4, 4],
                                 resblock_dilations=[[1, 3, 5, 7]] * 3, causal=False, nsf_params=_NSF16),
    "v1_24k": dict(channels=512, upsample_scales=[8, 5, 3, 2], upsample_kernal_sizes=[16, 10, 6, 4],
                   resblock_dilations=[[1, 3, 5]] * 3, causal=True),
    "v1_nsf_24k": dict(channels=512, upsample_scales=[8, 5, 3, 2], upsample_kernal_sizes=[16, 10, 6, 4],
                       resblock_dilations=[[1, 3, 5]] * 3, causal=True, nsf_params={"nb_harmonics": 7, "sampling_rate": 24000}),
    "v1_48k": dict(in_channels=128, channels=512, upsample_scales=[10, 5, 3, 2, 2], upsample_kernal_sizes=[20, 10, 6, 4, 4],
                   resblock_dilations=[[1, 3, 5, 7]] * 3, causal=True),
    "multiband_24k": dict(out_channels=4, channels=512, upsample_scales=[5, 3, 2, 2], upsample_kernal_sizes=[10, 6, 4, 4],
                          resblock_dilations=[[1, 3, 5]] * 3, causal=True),
}


def _generator(name):
    p = GENERATORS[name]
    return K.Generator(in_channels=p.get("in_channels", 80), kernel_size=7, resblock_kernel_sizes=[3, 7, 11], bias=True,
                       use_weight_norm=True, **_LRELU, **{k: v for k, v in p.items() if k != "in_channels"}).eval()


class _Recorder:
    """Stand-ins for the library-backed ops: each conv / fused pair records (layer spec, input rows, mask rate), the
    element-wise steps pass shapes through, and rows_mask records its rate."""

    def __init__(self, monkeypatch):
        self.calls = []
        rec = self

        class Conv:
            @staticmethod
            def apply(x, resid, bias, v, g, spec, cache, reuse=None, mask=None):
                rec.calls.append(("conv", spec, x.shape[1], mask))
                return torch.zeros(x.shape[0], spec.t_out(x.shape[1]), spec.c_out)

        class Resblock:
            @staticmethod
            def apply(x, b1, v1, g1, b2, v2, g2, spec1, cache1, spec2, cache2, rd, mask=None):
                rec.calls.append(("resblock", spec1, x.shape[1], mask))
                return x

        class Same:
            @staticmethod
            def apply(*args):
                return next(a for a in args if torch.is_tensor(a))

        monkeypatch.setattr(ops, "ConvFn", Conv)
        monkeypatch.setattr(ops, "ResblockFn", Resblock)
        monkeypatch.setattr(ops, "SinAddFn", Same)
        monkeypatch.setattr(ops, "Mean3Fn", Same)
        monkeypatch.setattr(ops, "utterance_mask", lambda lengths, rate: ("mask", rate))
        monkeypatch.setattr(ops, "rows_mask", lambda y, m: rec.calls.append(("rows_mask", None, y.shape[1], m)) or y)
        monkeypatch.setattr(hifigan, "_PARALLEL_STREAMS", False)
        # the fused pair's descriptor needs the library's planner: plan every pair as fused
        monkeypatch.setattr(ops, "resblock_desc", lambda s1, s2, b, t: object())


def _run(gen, frames, lengths):
    cin = gen.conv_pre.conv1d.spec.c_in + (2 if gen.nsf_enable else 0)
    x = torch.zeros(2, cin, frames)
    excitation = None
    if gen.nsf_enable:    # the excitation kernel needs a device: hand its rows in directly
        excitation = torch.zeros(2, frames * int(torch.tensor(gen.upsample_scales).prod()), gen.source_module.nb_harmonics + 1)
        x = x[:, :-2]
    with torch.no_grad():
        return gen.forward_rows(x.transpose(1, 2).contiguous(), excitation, lengths)


@pytest.mark.parametrize("name", sorted(GENERATORS))
def test_every_layer_reads_its_own_rows_per_frame(monkeypatch, name):
    """Each masked conv's mask rate is its input's rows per mel frame (input rows / frames), for every layer: so item b's
    rows [0, lengths[b] * rate) are exactly the rows it has alone.  The output is masked at the samples per frame."""
    gen = _generator(name)
    rec = _Recorder(monkeypatch)
    frames = 7
    y = _run(gen, frames, torch.tensor([7, 3], dtype=torch.int32))
    hop = int(torch.tensor(gen.upsample_scales).prod())
    assert y.shape[1] == frames * hop
    convs = [c for c in rec.calls if c[0] != "rows_mask"]
    pairs = sum(len(block.convs1) for block in gen.conv_blocks)
    assert len(convs) == 2 + gen.num_upsamples * (2 + (1 if gen.nsf_enable else 0)) + pairs
    for kind, spec, t_in, mask in convs:
        assert mask is not None and mask[0] == "mask", (kind, spec)
        assert t_in == frames * mask[1], (kind, spec, t_in, mask)
    assert rec.calls[-1] == ("rows_mask", None, frames * hop, ("mask", hop))


def _signature(spec):
    return [spec.c_in, spec.c_out, spec.kernel, spec.stride, spec.dilation, spec.pad_left, int(spec.transposed), spec.upsample]


def _parent_calls():
    """The layer calls (kind, layer signature, input rows) of the unmasked forwards as the commit before ragged batches made
    them -- recorded there with this file's stand-ins, 5 frames, every ResBlock pair planned as fused."""
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ragged_unmasked_calls_parent.json")) as f:
        return json.load(f)


@pytest.mark.parametrize("name", sorted(GENERATORS))
def test_no_lengths_means_no_mask(monkeypatch, name):
    """lengths=None is the unmasked forward: the layer calls of the commit before ragged batches, in the same order, none of
    them masked, no output mask; and the masked forward makes the same calls."""
    gen = _generator(name)
    rec = _Recorder(monkeypatch)
    _run(gen, 5, None)
    assert [[k] + _signature(s) + [t] for k, s, t, m in rec.calls] == _parent_calls()[name]
    plain = [(k, id(s), t) for k, s, t, m in rec.calls]
    assert all(m is None for _, _, _, m in rec.calls) and not any(k == "rows_mask" for k, _, _, _ in rec.calls)
    rec.calls.clear()
    _run(gen, 5, torch.tensor([5, 2], dtype=torch.int32))
    assert [(k, id(s), t) for k, s, t, m in rec.calls if k != "rows_mask"] == plain


def test_pqmf_synthesis_masks_at_subband_rate(monkeypatch):
    rec = _Recorder(monkeypatch)
    p = pqmf.PQMF(4)
    with torch.no_grad():
        p.synthesis(torch.zeros(2, 4, 6))
        assert [[k] + _signature(s) + [t] for k, s, t, m in rec.calls] == _parent_calls()["pqmf_synthesis"]
        rec.calls.clear()
        y = p.synthesis(torch.zeros(2, 4, 6), lengths=[6, 2])
    assert y.shape == (2, 1, 24)
    assert [(k, t, m) for k, _, t, m in rec.calls] == [("conv", 6, ("mask", 1)), ("rows_mask", 24, ("mask", 4))]


def test_lengths_validation():
    cpu = torch.device("cpu")
    assert ops.ragged_lengths([3, 1], 2, 3, cpu).dtype == torch.int32
    assert ops.ragged_lengths(torch.tensor([3, 1]), 2, 3, cpu).tolist() == [3, 1]
    with pytest.raises(ValueError, match="expected 2 values"):
        ops.ragged_lengths([3], 2, 3, cpu)
    with pytest.raises(ValueError, match=r"in \[1, 3\]"):
        ops.ragged_lengths([4, 1], 2, 3, cpu)
    with pytest.raises(ValueError, match=r"in \[1, 3\]"):
        ops.ragged_lengths([0, 1], 2, 3, cpu)
    with pytest.raises(ValueError, match="shape"):
        ops.ragged_lengths(torch.tensor([3, 1, 2]), 2, 3, cpu)
    with pytest.raises(ValueError, match="int32 / int64"):
        ops.ragged_lengths(torch.tensor([3.0, 1.0]), 2, 3, cpu)
    with pytest.raises(ValueError, match="on cuda"):
        ops.ragged_lengths(torch.tensor([3, 1]), 2, 3, torch.device("cuda", 0))


def test_generator_refuses_ragged_training_and_unseeded_nsf():
    gen = K.Generator(channels=32).train()
    with pytest.raises(RuntimeError, match="inference only"):
        gen(torch.zeros(2, 80, 4), lengths=[4, 2])
    with pytest.raises(ValueError, match="expected 2 values"):
        gen.eval()(torch.zeros(2, 80, 4), lengths=[4])
    nsf = K.Generator(channels=32, nsf_params={"nb_harmonics": 7, "sampling_rate": 24000}).eval()
    with pytest.raises(ValueError, match="nsf_seeds"):
        nsf(torch.zeros(2, 82, 4), lengths=[4, 2])


def test_masked_conv_refuses_autograd():
    w = torch.zeros(3, requires_grad=True)
    with pytest.raises(RuntimeError, match="inference only"):
        ops._refuse_masked_grad("conv", torch.zeros(2), w)
    with torch.no_grad():
        ops._refuse_masked_grad("conv", torch.zeros(2), w)
    ops._refuse_masked_grad("conv", torch.zeros(2), None)
