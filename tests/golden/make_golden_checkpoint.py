"""Writes tests/golden/checkpoint_reference.pth: a checkpoint in GAN_Trainer's layout (kantts/train/trainer.py:591-632) written
by the UNMODIFIED reference classes (the TINY configs of tests/test_checkpoint_cpu.py, one Adam step on synthetic gradients).
Needs an importable KAN-TTS checkout (KANTTS_REFERENCE).  python tests/golden/make_golden_checkpoint.py"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import ref_shims  # noqa: E402
import test_checkpoint_cpu as T  # noqa: E402


def main():
    ref_shims.import_reference()
    import kantts.models.hifigan.hifigan as R
    rm, ro, rs = T._build(R, T.TINY)
    T._fake_train(rm, ro)
    T._save(rm, ro, rs, 4, os.path.join(HERE, "checkpoint_reference.pth"))


if __name__ == "__main__":
    main()
