"""Time the syBERT train step at sybert.yaml sizes (batch 32 of 64-256 symbols, masked on the device by BertMasker), the
SeqCELoss kernels (forward + backward: the wall time of a call and, from torch.profiler, the device time of its kernels)
against the torch composite of the reference's formulation on the same GPU tensors, and BertMasker against the
reference's per-utterance masking loop on the host (restated in oracle/sybert.py) for the same batch.  Checks that the
kernel loss agrees with the composite within 1e-6 relative.  Prints one JSON line with the card name and power limit.

    python scripts/sybert_step.py [--steps 20] [--warmup 5]
"""
import argparse
import json
import os
import random
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import kantts_b200 as K  # noqa: E402
from oracle import sybert as osy  # noqa: E402
from test_gpu_sybert import make_sybert_batch  # noqa: E402

DEV = "cuda"


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def _event_times(fn, steps, warmup):
    """-> per-call milliseconds from CUDA events around each call."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return times


def _kernel_us(fn, iters=20):
    """-> (microseconds of device kernel time per call, the kernels' names) from torch.profiler over ``iters`` calls."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    kernels = [e for e in prof.key_averages() if e.device_type == DeviceType.CUDA]
    return sum(e.self_device_time_total for e in kernels) / iters, sorted({e.key[:60] for e in kernels})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sybert_step.py measures on the GPU; no CUDA device found")
    cfg = K.sybert_config()
    torch.manual_seed(1234)
    config = {"Model": {"KanTtsTextsyBERT": {"params": cfg, "optimizer": {"type": "Adam", "params": {
        "lr": 1e-4, "betas": [0.9, 0.98], "eps": 1e-9, "weight_decay": 0.0}},
        "scheduler": {"type": "NoamLR", "params": {"warmup_steps": 10000}}}}}
    model, opt, sch = K.sybert_model_builder(config, DEV)
    model.train()
    crit = K.criterion_builder({"Loss": {"SeqCELoss": {"enable": True, "params": {"loss_type": "ce"}}}}, DEV)
    step = K.SybertStep(model, opt, sch, crit)
    raw = {k: v.to(DEV) for k, v in make_sybert_batch(cfg, torch.Generator().manual_seed(1234)).items()}
    masker = K.BertMasker(cfg["mask_ratio"], cfg["sy"], seed=1234)
    B, L = raw["input_lings"].shape[:2]
    symbols = int((raw["valid_input_lengths"] + 1).sum())
    res = {"card": _card(), "batch": B, "max_symbols": L, "symbols": symbols, "steps": args.steps, "warmup": args.warmup}

    step_ms = _event_times(lambda: step.step(masker(raw)), args.steps, args.warmup)
    res["step_ms_median"] = statistics.median(step_ms)
    res["symbols_per_s"] = symbols / (res["step_ms_median"] / 1e3)

    # SeqCELoss on the logits of this batch: kernels against the reference's composite, same GPU tensors
    batch = masker(raw)
    with torch.no_grad():
        logits0 = model(batch["input_lings"], batch["valid_input_lengths"])["logits"].detach()
    targets, masks = batch["targets"], batch["bert_masks"]
    x = logits0.clone().requires_grad_(True)
    out = {}

    def kernels():
        x.grad = None
        loss, err = crit["SeqCELoss"](x, targets, masks)
        loss.backward()
        out["kernels"] = (loss.detach(), err)

    def composite():
        x.grad = None
        loss, err = osy.seq_ce_loss(x, targets, masks)
        loss.backward()
        out["composite"] = (loss.detach(), err)

    # a call's wall time (events around the host code of one forward + backward) and its device kernel time
    res["seq_ce_kernels_call_ms"] = statistics.median(_event_times(kernels, 50, 10))
    res["seq_ce_composite_call_ms"] = statistics.median(_event_times(composite, 50, 10))
    res["seq_ce_kernels_device_us"], res["seq_ce_kernels_names"] = _kernel_us(kernels)
    res["seq_ce_composite_device_us"], res["seq_ce_composite_names"] = _kernel_us(composite)
    lk, lc = float(out["kernels"][0]), float(out["composite"][0])
    res["seq_ce_loss_rel_diff"] = abs(lk - lc) / abs(lc)
    res["seq_ce_err_equal"] = float(out["kernels"][1]) == float(out["composite"][1])
    assert res["seq_ce_loss_rel_diff"] <= 1e-6, res

    res["bert_masker_call_ms"] = statistics.median(_event_times(lambda: masker(raw), 50, 10))
    res["bert_masker_device_us"], _ = _kernel_us(lambda: masker(raw))
    seqs = [s[: int(n) + 1] for s, n in zip(raw["input_lings"][:, :, 0].cpu().numpy(), raw["valid_input_lengths"].cpu())]
    np.random.seed(0)
    random.seed(0)
    host = []
    for _ in range(5):
        t0 = time.perf_counter()
        for s in seqs:
            osy.reference_bert_masking(s, cfg["mask_ratio"], cfg["sy"], cfg["sy"] - 1)
        host.append((time.perf_counter() - t0) * 1e3)
    res["reference_masking_host_ms"] = statistics.median(host)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
