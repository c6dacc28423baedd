"""CPU: the speaker-embedding extractor of the SE flow.  The oracle restatement (oracle/dtdnn.py) against the goldens of
torchaudio and the unmodified reference (tests/golden/make_golden_se.py), DTDNN's state_dict contract and seeded init, the
install patch and the host-side checks."""
import json
import os

import numpy as np
import pytest
import torch

import kantts_b200 as K
from conftest import GOLDEN, rel_l2
from oracle import dtdnn as od
from oracle.ref_shims import REF_ROOT, reference_available

needs_reference = pytest.mark.skipif(not reference_available(), reason="reference checkout not available")


def seeded_model():
    """The goldens' model: DTDNN() after torch.manual_seed(0), BatchNorms set by seed_bn_stats(seed=7), eval mode."""
    torch.manual_seed(0)
    m = K.DTDNN()
    od.seed_bn_stats(m, seed=7)
    return m.eval()


def test_oracle_fbank_matches_torchaudio(golden):
    g = golden("se_dtdnn")
    for i, n in enumerate(g.cfg["lengths"]):
        fb = od.kaldi_fbank(g.arrays[f"wav_{i}"])
        assert fb.shape == (K.speaker.fbank_frames(n), 80)
        # float64 here against torchaudio's float32 spectrum and log
        assert np.abs(fb - g.arrays[f"fbank_{i}"]).max() < 1e-3
        assert np.abs(od.cmn(fb) - g.arrays[f"feat_{i}"]).max() < 1e-3


def test_oracle_dtdnn_matches_reference_embeddings(golden):
    g = golden("se_dtdnn")
    sd = seeded_model().state_dict()
    for i in range(len(g.cfg["lengths"])):
        e = od.dtdnn_forward(sd, g.t(f"feat_{i}")[None])[0]
        assert rel_l2(e, g.t("emb")[i]) < 1e-5


def test_dtdnn_state_dict_and_seeded_init_match_reference():
    from golden.make_golden_disc_init import checksums
    with open(os.path.join(GOLDEN, "se_dtdnn_init_checksums.json")) as f:
        want = json.load(f)["DTDNN"]
    torch.manual_seed(0)
    got = checksums(K.DTDNN().state_dict())
    assert got[0] == want[0]
    assert got[1] == pytest.approx(want[1], rel=1e-12) and got[2] == pytest.approx(want[2], rel=1e-12)


def test_dtdnn_reference_layout_checkpoint_loads_strictly(tmp_path):
    torch.manual_seed(3)
    src = K.DTDNN()
    od.seed_bn_stats(src, seed=1)
    path = tmp_path / "se.model"
    torch.save(src.state_dict(), path)
    dst = K.DTDNN()
    dst.load_state_dict(torch.load(path), strict=True)
    for (k, a), (k2, b) in zip(src.state_dict().items(), dst.state_dict().items()):
        assert k == k2 and torch.equal(a, b)


@needs_reference
def test_reference_dtdnn_loads_strictly():
    import sys
    if REF_ROOT not in sys.path:
        sys.path.insert(0, REF_ROOT)
    from kantts.preprocess.se_processor.D_TDNN import DTDNN as RefDTDNN
    torch.manual_seed(4)
    ref = RefDTDNN()
    ours = K.DTDNN()
    ours.load_state_dict(ref.state_dict(), strict=True)
    assert list(ours.state_dict()) == list(ref.state_dict())


def test_dtdnn_is_inference_only():
    m = K.DTDNN()
    with pytest.raises(RuntimeError, match="inference only"):
        m(torch.zeros(1, 50, 80))


def test_kaldi_fbank_rejects_a_wav_shorter_than_one_frame():
    with pytest.raises(ValueError, match="shorter than one"):
        K.kaldi_fbank(torch.zeros(2, 1000), [1000, 399])
    with pytest.raises(ValueError):
        K.kaldi_fbank(torch.zeros(2, 1000), [1000, 1001])


def test_fbank_frames_and_block_widths():
    assert [K.speaker.fbank_frames(n) for n in (399, 400, 559, 560, 16000)] == [0, 1, 1, 2, 98]
    m = K.DTDNN()
    widths = []
    for bi in (1, 2, 3):
        block = getattr(m.xvector, f"block{bi}")
        first = block.tdnnd1.nonlinear1.batchnorm.num_features
        widths.append((first, first + sum(l.se.linear_stem.out_channels for l in block)))
    assert widths == [(128, 512), (256, 1024), (512, 1024)]


def test_install_patches_the_speaker_processor():
    fake_loss = type("L", (), {"loss_dict": {}})()
    se = type("S", (), {})()
    K.install(kantts_models=type("M", (), {})(), kantts_loss=fake_loss, kantts_audio=type("A", (), {})(), kantts_se=se)
    assert se.DTDNN is K.DTDNN
