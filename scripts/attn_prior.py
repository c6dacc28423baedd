"""Time the alignment prior of a MAS training batch at the sizes of scripts/sambert_mas_step.py (batch 16, up to 200
symbols, up to 1000 frames, tests/test_gpu_sambert_mas.py::make_mas_batch): ``AttnPriors`` per call (CUDA events, median
over the calls), the kt_attn_prior kernel alone (torch.profiler, a separate run), and the reference's formulation for the
same lengths on one host core -- one scipy.stats.betabinom per mel frame (kantts/datasets/dataset.py:20-31, restated
here) and the collate's copy into a zero float32 pad (dataset.py:816-827).  Reports the largest difference from the
float64 oracle (oracle/attn_prior.py) in float32 units in the last place, and how many elements differ from it at all.
Prints one JSON line with the card name and power limit.

    python scripts/attn_prior.py [--calls 200] [--warmup 20]
"""
import argparse
import json
import os
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
from oracle import attn_prior as oap  # noqa: E402
from test_gpu_sambert_mas import make_mas_batch  # noqa: E402

DEV = "cuda"


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def _event_times(fn, calls, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(calls):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return times


def _kernel_us(fn, name, iters=50):
    """-> microseconds per call of the device kernels whose name contains ``name``, from torch.profiler."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    kernels = [e for e in prof.key_averages() if e.device_type == DeviceType.CUDA and name in e.key]
    assert sum(e.count for e in kernels) == iters, [(e.key, e.count) for e in kernels]
    return sum(e.self_device_time_total for e in kernels) / iters


def _ulps(got, want):
    w = want.numpy().astype(np.float32)
    return np.abs(got.numpy().astype(np.float64) - w.astype(np.float64)) / np.spacing(np.abs(w)).astype(np.float64)


def _reference_collate(il, ol, t_mel, t_text):
    """The reference's prior for each utterance (one betabinom per frame) copied into the collate's zero pad."""
    from scipy.stats import betabinom
    priors = torch.zeros(len(il), t_mel, t_text)
    for i, (n, m) in enumerate(zip(il.tolist(), ol.tolist())):
        P, M = n + 1, m
        x = np.arange(0, P)
        p = torch.tensor(np.array([betabinom(P, j, M + 1 - j).pmf(x) for j in range(1, M + 1)]))
        priors[i, : p.shape[0], : p.shape[1]] = p
    return priors


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("attn_prior.py measures on the GPU; no CUDA device found")
    batch = make_mas_batch(K.sambert_16k_mas_config(), torch.Generator().manual_seed(1234))
    il, ol = batch["valid_input_lengths"], batch["valid_output_lengths"]
    dev = {k: v.to(DEV) for k, v in batch.items() if v is not None}
    B, T = dev["mel_targets"].shape[:2]
    L = dev["input_lings"].shape[1]
    priors = K.AttnPriors()
    res = {"card": _card(), "batch": B, "frames": T, "symbols": L, "valid_elements": int(((il + 1) * ol).sum()),
           "calls": args.calls, "warmup": args.warmup}

    res["attn_priors_call_ms_median"] = statistics.median(_event_times(lambda: priors(dev), args.calls, args.warmup))
    res["kt_attn_prior_kernel_us"] = _kernel_us(lambda: priors(dev), "attn_prior_kernel")

    got = priors(dev)["attn_priors"].cpu()
    want = oap.attn_priors(il, ol, T, L)
    u = _ulps(got, want)
    res["max_ulps_vs_oracle"] = float(u.max())
    res["elements_differing_from_oracle"] = int((u > 0).sum())

    try:
        import scipy  # noqa: F401
    except ImportError:
        res["reference_host_ms"] = "not measured"
    else:
        os.sched_setaffinity(0, {min(os.sched_getaffinity(0))})      # one host core
        t0 = time.perf_counter()
        ref = _reference_collate(il, ol, T, L)
        res["reference_host_ms"] = (time.perf_counter() - t0) * 1e3
        res["max_ulps_vs_reference"] = float(_ulps(got, ref.double()).max())
    print(json.dumps(res))


if __name__ == "__main__":
    main()
