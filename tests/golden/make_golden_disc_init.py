"""Writes tests/golden/disc_init_checksums.json: for the reference's MultiPeriodDiscriminator() and
MultiScaleDiscriminator(follow_official_norm=True) built after torch.manual_seed(5), a digest of the state_dict layout (keys
in order and shapes) and two float64 checksums of the values (see checksums()).  Needs an importable KAN-TTS checkout (KANTTS_REFERENCE).
python tests/golden/make_golden_disc_init.py"""
import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from oracle.ref_shims import import_reference  # noqa: E402

CASES = (("MultiPeriodDiscriminator", {}), ("MultiScaleDiscriminator", {"follow_official_norm": True}))


def checksums(sd):
    """-> [sha256 of the (key, shape) list, sum_i (i + 1) * sum(entry_i), sum_i sum(|entry_i|)] (float64)"""
    import hashlib
    layout = hashlib.sha256(repr([(k, list(v.shape)) for k, v in sd.items()]).encode()).hexdigest()
    s = sum((i + 1) * float(v.double().sum()) for i, v in enumerate(sd.values()))
    a = sum(float(v.double().abs().sum()) for v in sd.values())
    return [layout, s, a]


def main():
    import_reference()
    from kantts.models.hifigan import hifigan as R
    out = {}
    for name, kw in CASES:
        torch.manual_seed(5)
        sd = getattr(R, name)(**kw).state_dict()
        out[name] = checksums(sd)
    with open(os.path.join(HERE, "disc_init_checksums.json"), "w") as f:
        json.dump(out, f)


if __name__ == "__main__":
    main()
