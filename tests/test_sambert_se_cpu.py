"""CPU: the speaker-embedding (SE) SAM-BERT variant.  Its config, its state_dict and seeded init against the unmodified
reference (tests/golden/make_golden_sambert_se.py), and the variants that stay unbuilt."""
import json
import os

import pytest
import torch

import kantts_b200 as K
from conftest import GOLDEN
from oracle.ref_shims import REF_ROOT, reference_available


def test_se_nsf_global_16k_config():
    cfg = K.sambert_se_nsf_global_16k_config()
    assert cfg["SE"] is True and cfg["speaker_units"] == 192 and cfg["num_mels"] == 82
    assert cfg["NSF"] is True and cfg["nsf_norm_type"] == "global"
    assert (cfg["nsf_f0_global_minimum"], cfg["nsf_f0_global_maximum"]) == (30.0, 730.0)
    assert "speaker" not in cfg
    same = {k: v for k, v in K.sambert_24k_config().items() if k not in ("speaker", "speaker_units", "num_mels")}
    assert {k: cfg[k] for k in same} == same


@pytest.mark.skipif(not reference_available(), reason="reference checkout not available")
def test_se_config_matches_the_shipped_yaml():
    import yaml
    with open(os.path.join(REF_ROOT, "kantts", "configs", "sambert_se_nsf_global_16k.yaml")) as f:
        params = yaml.safe_load(f)["Model"]["KanTtsSAMBERT"]["params"]
    cfg = K.sambert_se_nsf_global_16k_config()
    assert {k: cfg[k] for k in params} == params


def test_se_model_state_dict_and_seeded_init_match_reference(golden):
    from golden.make_golden_disc_init import checksums
    with open(os.path.join(GOLDEN, "se_init_checksums.json")) as f:
        want = json.load(f)["KanTtsSAMBERT"]
    torch.manual_seed(5)
    m = K.KanTtsSAMBERT(golden("sambert_se_small").cfg)
    assert not hasattr(m, "spk_tokenizer") and m.se_enable
    got = checksums(m.state_dict())
    assert got[0] == want[0]
    assert got[1] == pytest.approx(want[1], rel=1e-12) and got[2] == pytest.approx(want[2], rel=1e-12)
    m.load_state_dict(golden("sambert_se_small").group("sd/"), strict=True)


def test_full_size_se_model_constructs():
    m = K.KanTtsSAMBERT(K.sambert_se_nsf_global_16k_config())
    assert not hasattr(m, "spk_tokenizer") and m.mel_postnet.num_mels == 82
    assert not any(k.startswith("spk_tokenizer") for k in m.state_dict())


def test_se_with_fp_or_mas_stays_unbuilt():
    cfg = K.sambert_se_nsf_global_16k_config()
    for extra in ({"FP": True}, {"MAS": True}):
        with pytest.raises(NotImplementedError):
            K.KanTtsSAMBERT(dict(cfg, **extra))
