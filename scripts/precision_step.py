"""bf16x3 against single-pass bf16 (hifigan.set_precision) on the GPU:
  1. the bench.py GAN workload (HiFi-GAN v1 G + MPD + MSD train step, batch 16 x 8192 samples, CUDA graph), the two
     precisions in alternating rounds, each timed over --steps steps with device events after --warmup steps;
  2. the tensor-core kernels' time per step by torch.profiler (one profiled step per precision, in its own run after
     the timed rounds), summed per kernel and, for the largest conv / weight-gradient / resblock kernels, per launch;
  3. the streamed generator's latency per 16-frame chunk at batch 1 / 16 / 64 (class-default generator, eval).
Prints the GPU's name, power limit and clocks first, then one JSON line per measurement; writes them to --out."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import kantts_b200 as K  # noqa: E402
from bench import CONFIG, synth_batch  # noqa: E402

PRECISIONS = ("bf16x3", "bf16")


def gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm,clocks.mem"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
        return out.stdout.strip()
    except OSError as e:
        return f"nvidia-smi unavailable: {e}"


def build_step(prec, dev):
    torch.manual_seed(1234)
    model, opt, sched = K.hifigan_model_builder(CONFIG, dev, precision=prec)
    crit = K.criterion_builder(CONFIG, dev)
    return K.GanStep(model, opt, sched, crit, CONFIG, cuda_graph=True)


def time_steps(step, batch, steps, warmup):
    for _ in range(warmup):
        step.step(batch)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        step.step(batch)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def profile_step(step, batch):
    from torch.profiler import ProfilerActivity, profile
    step.step(batch)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step.step(batch)
        torch.cuda.synchronize()
    per = {}
    for ev in prof.events():
        if ev.device_type.name != "CUDA":
            continue
        n = ev.name
        if not any(k in n for k in ("conv_tc", "wgrad_t", "resblock_tc", "split_planes", "wgrad_reduce")):
            continue
        d = per.setdefault(n, [0, 0.0, 0.0])
        d[0] += 1
        d[1] += ev.device_time_total / 1e3 if hasattr(ev, "device_time_total") else ev.cuda_time_total / 1e3
        d[2] = max(d[2], (ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total) / 1e3)
    return per


def stream_latency(prec, dev, batch, chunks=40, frames=16):
    torch.manual_seed(0)
    g = K.set_precision(K.Generator().to(dev).eval(), prec)
    st = g.streamer(batch, frames)
    mel = torch.randn(batch, 80, frames, device=dev)
    for _ in range(5):
        st.push(mel)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(chunks):
        st.push(mel)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / chunks * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--skip-stream", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "precision_step.py measures on a GPU"
    dev = torch.device("cuda:0")
    lines = []

    def emit(d):
        print(json.dumps(d), flush=True)
        lines.append(d)

    emit({"gpu": gpu_info()})
    y, x = (t.to(dev) for t in synth_batch(16, 1234))
    steps = {p: build_step(p, dev) for p in PRECISIONS}
    for r in range(args.rounds):
        for p in (PRECISIONS if r % 2 == 0 else PRECISIONS[::-1]):
            ms = time_steps(steps[p], (y, x), args.steps, args.warmup if r == 0 else 2)
            emit({"measure": "gan_step_ms", "precision": p, "round": r, "ms": round(ms, 3)})
    for p in PRECISIONS:
        ms = {d["round"]: d["ms"] for d in lines if d.get("precision") == p and d.get("measure") == "gan_step_ms"}
        v = list(ms.values())
        emit({"measure": "gan_step_ms_summary", "precision": p, "min": min(v), "max": max(v), "mean": sum(v) / len(v)})
    for p in PRECISIONS:
        per = profile_step(steps[p], (y, x))
        total = sum(v[1] for v in per.values())
        top = sorted(per.items(), key=lambda kv: -kv[1][1])[:12]
        emit({"measure": "tc_kernels_per_step", "precision": p, "total_ms": round(total, 3),
              "top": [{"kernel": k[:120], "launches": v[0], "ms": round(v[1], 3), "max_launch_ms": round(v[2], 3)} for k, v in top]})
    del steps
    torch.cuda.empty_cache()
    if not args.skip_stream:
        for b in (1, 16, 64):
            for p in PRECISIONS:
                emit({"measure": "stream_chunk_ms", "precision": p, "batch": b, "frames": 16,
                      "ms": round(stream_latency(p, dev, b), 3)})
    emit({"gpu_after": gpu_info()})
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for d in lines:
                f.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
