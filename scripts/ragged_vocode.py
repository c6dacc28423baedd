"""Time vocoding a ragged batch four ways: the padded whole-batch forward, the masked forward (Generator.forward(...,
lengths=)), a loop over the utterances one at a time, and the one-chunk streamer (push + finish of each utterance's whole
mel).  B = 16 seeded lengths of 100-800 frames, random weights at a trained scale, for the non-causal 16 kHz and the causal
24 kHz generators, in bf16x3 and single-pass bf16.  The variants alternate within each round; each time is one round's CUDA
events around the variant, after a warm-up of every variant.  Prints the card and its power limit, then one JSON line per
(generator, precision) with the median and spread of each variant in ms, and the masked forward's largest difference from
the per-utterance loop over the valid samples.

    python scripts/ragged_vocode.py [--rounds 5] [--batch 16]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import kantts_b200 as K  # noqa: E402

_LRELU = {"nonlinear_activation": "LeakyReLU", "nonlinear_activation_params": {"negative_slope": 0.1}}
GENERATORS = {
    "hifigan_noncausal_v1_16k": dict(channels=256, upsample_scales=[10, 5, 2, 2], upsample_kernal_sizes=[20, 11, 4, 4],
                                     resblock_kernel_sizes=[3, 7, 11], resblock_dilations=[[1, 3, 5, 7]] * 3, causal=False,
                                     **_LRELU),
    "hifigan_v1_24k": dict(channels=512, upsample_scales=[8, 5, 3, 2], upsample_kernal_sizes=[16, 10, 6, 4],
                           resblock_kernel_sizes=[3, 7, 11], resblock_dilations=[[1, 3, 5]] * 3, causal=True, **_LRELU),
}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--batch", type=int, default=16)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ragged_vocode.py needs a CUDA device")
    name, limit = card()
    print(f"card: {name}, power limit {limit}", flush=True)
    dev = "cuda"
    rng = np.random.default_rng(2026)
    lengths = [int(v) for v in rng.integers(100, 801, size=args.batch)]
    T = max(lengths)
    for gname, params in GENERATORS.items():
        for precision in ("bf16x3", "bf16"):
            torch.manual_seed(0)
            gen = K.Generator(**params).to(dev).eval()
            with torch.no_grad():
                for p in gen.parameters():
                    p.mul_(1.0 + 0.5 * torch.rand_like(p))
            if precision == "bf16":
                K.set_precision(gen, "bf16")
            mel = torch.randn(args.batch, 80, T, generator=torch.Generator().manual_seed(1)).to(dev)
            items = [mel[b:b + 1, :, :n].contiguous() for b, n in enumerate(lengths)]
            hop = int(np.prod(gen.upsample_scales))
            L = torch.tensor(lengths, dtype=torch.int32, device=dev)
            causal = params["causal"]
            st = gen.streamer(1, T, lengths=None if causal else [T])

            def stream_one(b):
                st.reset([0], lengths=None if causal else [lengths[b]])
                return st.push(items[b]), st.finish()

            variants = {
                "padded": lambda: gen(mel),
                "masked": lambda: gen(mel, lengths=L),
                "loop": lambda: [gen(x) for x in items],
                "stream_1chunk": lambda: [stream_one(b) for b in range(args.batch)],
            }
            times = {k: [] for k in variants}
            with torch.no_grad():
                for fn in variants.values():      # warm-up: plans, images, workspaces, the streamer's graph
                    fn()
                torch.cuda.synchronize()
                for _ in range(args.rounds):
                    for k, fn in variants.items():
                        times[k].append(timed(fn)[0])
                ym = gen(mel, lengths=L)
                diff = max(float((ym[b, :, : n * hop] - gen(items[b])[0]).abs().max()) for b, n in enumerate(lengths))
            res = {"generator": gname, "precision": precision, "batch": args.batch, "frames": sum(lengths),
                   "max_abs_diff_masked_vs_loop": diff}
            for k, v in times.items():
                res[k + "_ms"] = round(float(np.median(v)), 3)
                res[k + "_spread_ms"] = round(float(max(v) - min(v)), 3)
            print(json.dumps(res), flush=True)
            del st, gen
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
