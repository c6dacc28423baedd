"""GPU: the speaker-embedding extractor (csrc/speaker.cu + the conv kernels) against the goldens of torchaudio and the
unmodified reference (tests/golden/make_golden_se.py), batch isolation and run-to-run determinism, on both compute paths.

Tolerances.  The fbank is exact fp32 against torchaudio's fp32: the spectrum's rounding (~1e-7 relative) is amplified by the
log only where a mel energy is tiny; 1e-3 absolute on the log energies.  The D-TDNN on the exact-fp32 path differs from the
reference's fp32 CPU forward by summation order alone, over about 60 layers: embedding relative L2 1e-4.  The tensor-core
path keeps about 16 mantissa bits per product term (split bf16), so 1e-3.  From wavs, the fbank's error enters as well.
"""
import pytest
import torch

import kantts_b200 as K
from conftest import rel_l2
from kantts_b200 import ops
from oracle import dtdnn as od

pytestmark = pytest.mark.gpu
DEV = "cuda"
EMB_TOL = {True: 1e-4, False: 1e-3}     # exact fp32 path, tensor-core path


@pytest.fixture
def exact_path(request):
    ops.set_force_ffma(request.param)
    yield request.param
    ops.set_force_ffma(False)


def seeded_model():
    torch.manual_seed(0)
    m = K.DTDNN()
    od.seed_bn_stats(m, seed=7)
    return m.eval().to(DEV)


def golden_batch(g):
    lens = g.cfg["lengths"]
    wav = torch.zeros(len(lens), max(lens))
    for i, n in enumerate(lens):
        wav[i, :n] = g.t(f"wav_{i}")
    return wav.to(DEV), lens


def test_kaldi_fbank_matches_torchaudio(golden):
    g = golden("se_dtdnn")
    wav, lens = golden_batch(g)
    feats, frames = K.kaldi_fbank(wav, lens)
    torch.cuda.synchronize()
    assert frames == [K.speaker.fbank_frames(n) for n in lens]
    worst = 0.0
    for i, nf in enumerate(frames):
        want = g.t(f"feat_{i}")
        assert want.shape[0] == nf
        worst = max(worst, float((feats[i, :nf].cpu() - want).abs().max()))
        assert not feats[i, nf:].any()
    print(f"fbank (CMN) max abs error {worst:.3e}")
    assert worst < 1e-3


@pytest.mark.parametrize("exact_path", [True, False], indirect=True)
def test_embeddings_match_reference(golden, exact_path):
    g = golden("se_dtdnn")
    m = seeded_model()
    lens = g.cfg["lengths"]
    nfs = [K.speaker.fbank_frames(n) for n in lens]
    feats = torch.zeros(len(lens), max(nfs), 80)
    for i, nf in enumerate(nfs):
        feats[i, :nf] = g.t(f"feat_{i}")
    emb = m(feats.to(DEV), nfs).cpu()
    errs = [rel_l2(emb[i], g.t("emb")[i]) for i in range(len(lens))]
    wav, _ = golden_batch(g)
    emb_w = K.speaker_embedding(m, wav, lens).cpu()
    errs_w = [rel_l2(emb_w[i], g.t("emb")[i]) for i in range(len(lens))]
    print(f"exact={exact_path}: embedding rel L2 from features {max(errs):.3e}, from wavs {max(errs_w):.3e}")
    assert max(errs) < EMB_TOL[exact_path]
    assert max(errs_w) < 10 * EMB_TOL[exact_path]


@pytest.mark.parametrize("exact_path", [True, False], indirect=True)
def test_each_item_of_a_mixed_batch_equals_its_wav_alone(exact_path):
    m = seeded_model()
    gen = torch.Generator().manual_seed(5)
    lens = [16000, 9000, 40130, 4000, 25610]
    wav = (0.1 * torch.randn(len(lens), max(lens), generator=gen)).to(DEV)
    batch = K.speaker_embedding(m, wav, lens)
    worst = 0.0
    for i, n in enumerate(lens):
        alone = K.speaker_embedding(m, wav[i:i + 1, :n].contiguous())
        if exact_path:
            assert torch.equal(batch[i], alone[0]), i
        worst = max(worst, rel_l2(batch[i].cpu(), alone[0].cpu()))
    print(f"exact={exact_path}: batched vs alone rel L2 {worst:.3e}")
    assert worst < 1e-5


@pytest.mark.parametrize("exact_path", [True, False], indirect=True)
def test_two_runs_are_bit_identical(exact_path):
    m = seeded_model()
    gen = torch.Generator().manual_seed(6)
    lens = [32000, 12345]
    wav = (0.1 * torch.randn(2, max(lens), generator=gen)).to(DEV)
    a = K.speaker_embedding(m, wav, lens)
    b = K.speaker_embedding(m, wav, lens)
    assert torch.equal(a, b)


def test_folded_weights_follow_a_new_state_dict():
    m = seeded_model()
    gen = torch.Generator().manual_seed(8)
    wav = (0.1 * torch.randn(1, 20000, generator=gen)).to(DEV)
    a = K.speaker_embedding(m, wav)
    torch.manual_seed(1)
    other = K.DTDNN()
    od.seed_bn_stats(other, seed=2)
    m.load_state_dict(other.state_dict())
    b = K.speaker_embedding(m, wav)
    feats, _ = K.kaldi_fbank(wav)
    want = od.dtdnn_forward({k: v.to(DEV) for k, v in other.state_dict().items()}, feats)
    assert not torch.equal(a, b)
    assert rel_l2(b.cpu(), want.cpu()) < EMB_TOL[False]
