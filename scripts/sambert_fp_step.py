"""Time the filled-pause (FP) SAM-BERT train step at sambert_fp_8k.yaml sizes (batch 16, 256 symbols, about 10 % of
them labelled) against the same model with FP off, and the insertion forward + backward against the oracle's
per-position restatement (the shape of the reference's insert_fp loop) on the same GPU tensors.  Prints one JSON
line with the card name and power limit.

    python scripts/sambert_fp_step.py [--steps 10] [--warmup 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import kantts_b200 as K  # noqa: E402
from kantts_b200 import sambert, sambert_ops  # noqa: E402
from oracle import sambert_fp as ofp  # noqa: E402
from test_gpu_sambert_fp import make_fp_batch  # noqa: E402

DEV = "cuda"


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def _time(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps * 1e3


def _step(cfg, batch, fp_dict):
    torch.manual_seed(1234)
    model = sambert.KanTtsSAMBERT(cfg).to(DEV).train()
    if fp_dict is not None:
        model.fp_dict = {k: v.to(DEV) for k, v in fp_dict.items()}
    opt = torch.optim.Adam(model.parameters(), lr=1e-4, betas=(0.9, 0.98), eps=1e-9)
    crit = {"MelReconLoss": sambert.MelReconLoss(), "ProsodyReconLoss": sambert.ProsodyReconLoss()}
    if fp_dict is not None:
        crit["FpCELoss"] = sambert.FpCELoss().to(DEV)
    step = K.SambertStep(model, opt, K.train.NoamLR(opt, warmup_steps=4000), crit)
    return lambda: step.step(batch)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sambert_fp_step.py measures on the GPU; no CUDA device found")
    cfg = K.sambert_fp_8k_config()
    gen = torch.Generator().manual_seed(1234)
    fp_dict = {k: torch.stack([torch.randint(0, cfg[n], (1, 3), generator=gen)
                               for n in ("sy", "tone", "syllable_flag", "word_segment")], -1) for k in (1, 2, 3)}
    batch = {k: v.to(DEV) for k, v in make_fp_batch(cfg, gen).items()}
    B, L = batch["input_lings"].shape[:2]
    plain = make_fp_batch(cfg, gen, frac=0.0)
    plain.pop("fp_label")
    plain = {k: v.to(DEV) for k, v in plain.items()}
    res = {"card": _card(), "batch": B, "symbols": L,
           "labelled": int((batch["fp_label"] > 0).sum()), "steps": args.steps, "warmup": args.warmup}
    res["fp_step_ms"] = _time(_step(cfg, batch, fp_dict), args.steps, args.warmup)
    res["no_fp_step_ms"] = _time(_step(dict(cfg, FP=False), plain, None), args.steps, args.warmup)

    C = cfg["encoder_projection_units"]
    text = torch.randn(B, L, C, device=DEV, requires_grad=True)
    enc = torch.randn(3, 3, C, device=DEV, requires_grad=True)
    lab, in_len = batch["fp_label"], batch["valid_input_lengths"]

    def kernels():
        codes, rows, _, t_ins = sambert_ops.fp_insert_plan(in_len, L, fp_label=lab)
        out = sambert_ops.FpInsertFn.apply(text, enc, codes, rows, t_ins)
        out.backward(torch.ones_like(out))

    def per_position():
        out, _, _ = ofp.fp_insert(text, enc, in_len, fp_label=lab)
        out.backward(torch.ones_like(out))

    res["insert_fwd_bwd_kernels_ms"] = _time(kernels, 20 * args.steps, args.warmup)
    res["insert_fwd_bwd_per_position_ms"] = _time(per_position, args.steps, 1)
    codes, rows, _, t_ins = sambert_ops.fp_insert_plan(in_len, L, fp_label=lab)
    with torch.no_grad():
        same = torch.equal(sambert_ops.FpInsertFn.apply(text, enc, codes, rows, t_ins),
                           ofp.fp_insert(text, enc, in_len, fp_label=lab)[0])
    res["insert_outputs_equal"] = same
    print(json.dumps(res))


if __name__ == "__main__":
    main()
