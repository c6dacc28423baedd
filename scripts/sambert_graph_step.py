"""Time SambertStep eager against SambertStep(cuda_graph=True), alternating the two in one process, on two workloads:
  ragged  seeded collate batches of 16 utterances of 64-256 symbols (the sambert_fp_step.py workload without FP), right-
          padded with data.pad_sambert_batch to multiples of 64 symbols and 192 frames, so a few shapes repeat;
  c4      batch 32 x 256 symbols x 768 frames (BASELINE config C4), one shape.
Per workload: ms per step of each mode, library launches per step (ops.launch_count; a replayed step makes none), the peak
memory of each mode, and the graphs captured.  Also the number of distinct shapes -- graphs -- that 1000 seeded ragged
batches padded the same way need.  Then, in a separate torch.profiler run, the four LSTMs' GPU time per step of the c4
shape: the new kernels (input projections, recurrences, gradients) against cuDNN's nn.LSTM forward + backward over the
same shapes, the pitch / energy BiLSTMs packed.  Prints one JSON line with the card name and power limit.

    python scripts/sambert_graph_step.py [--steps 10] [--warmup 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import kantts_b200 as K  # noqa: E402
from kantts_b200 import data, ops, sambert  # noqa: E402
from kantts_b200 import sambert_ops as sops  # noqa: E402
from golden.make_batch import make_c4_batch  # noqa: E402

DEV = "cuda"


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def ragged_batch(cfg, gen, B=16, lo=64, hi=256):
    """A collate batch of B utterances of lo..hi symbols (the trailing '~' included), 1-5 frames per symbol: padded to the
    batch's longest item, the padding frames on the symbol after each item's last (AM_Dataset.collate_fn)."""
    r = cfg["outputs_per_step"]
    n = torch.randint(lo, hi + 1, (B,), generator=gen)
    L = int(n.max())
    pad = torch.arange(L)[None, :] >= n[:, None]
    dur = torch.randint(1, 6, (B, L), generator=gen).masked_fill(pad, 0)
    out_len = dur.sum(1)
    T = -(-int(out_len.max()) // r) * r
    dur = dur.scatter_add(1, n.clamp_max(L - 1)[:, None], (T - out_len)[:, None])
    ling = torch.stack([torch.randint(0, cfg[k], (B, L), generator=gen)
                        for k in ("sy", "tone", "syllable_flag", "word_segment")], -1)
    return dict(input_lings=ling, input_emotions=torch.randint(0, cfg["emotion"], (B, L), generator=gen),
                input_speakers=torch.randint(0, cfg["speaker"], (B, L), generator=gen), valid_input_lengths=n - 1,
                valid_output_lengths=out_len, mel_targets=torch.randn(B, T, cfg["num_mels"], generator=gen),
                durations=dur, pitch_contours=torch.randn(B, L, generator=gen), energy_contours=torch.randn(B, L, generator=gen))


def _pad(cfg, b):
    # ragged_batch draws its ids from the whole tables; pad id 0 stands for the linguistic unit's "_" ids
    return data.pad_sambert_batch(b, 64, 192, cfg["outputs_per_step"], (0, 0, 0, 0), 0, 0)


def _make_step(cfg, cuda_graph, warmup):
    torch.manual_seed(1234)
    model = sambert.KanTtsSAMBERT(cfg).to(DEV).train()
    opt = torch.optim.Adam(model.parameters(), lr=1e-4, betas=(0.9, 0.98), eps=1e-9)
    crit = {"MelReconLoss": sambert.MelReconLoss(), "ProsodyReconLoss": sambert.ProsodyReconLoss()}
    return K.SambertStep(model, opt, K.train.NoamLR(opt, warmup_steps=4000), crit, cuda_graph=cuda_graph,
                         graph_warmup=warmup)


def _timed(step, batches):
    torch.cuda.synchronize()
    n0 = ops.launch_count()
    t0 = time.perf_counter()
    for b in batches:
        step.step(b)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / len(batches) * 1e3, (ops.launch_count() - n0) / len(batches)


def compare(cfg, batches, steps, warmup):
    """Eager and graph steps alternating in blocks of ``steps``: each mode is warmed up over every shape of ``batches`` first
    (the graph mode also captures), then two timed blocks of each."""
    modes = {}
    for name, g in (("eager", False), ("graph", True)):
        torch.cuda.reset_peak_memory_stats()
        step = _make_step(cfg, g, warmup)
        for _ in range(warmup + 1):
            for b in batches:
                step.step(b)
        torch.cuda.synchronize()
        modes[name] = dict(step=step, peak_mb=torch.cuda.max_memory_allocated() / 2 ** 20, ms=[], launches=0.0)
    seq = [batches[i % len(batches)] for i in range(steps)]
    for _ in range(2):
        for name in ("eager", "graph"):
            ms, launches = _timed(modes[name]["step"], seq)
            modes[name]["ms"].append(ms)
            modes[name]["launches"] = launches
    out = {f"{name}_ms_per_step": [round(v, 2) for v in m["ms"]] for name, m in modes.items()}
    out.update({f"{name}_library_launches_per_step": m["launches"] for name, m in modes.items()})
    out.update({f"{name}_peak_mb": round(m["peak_mb"], 1) for name, m in modes.items()})
    out["graphs_captured"] = len(modes["graph"]["step"]._graphs)
    out["shapes"] = sorted({(b["input_lings"].shape[1], b["mel_targets"].shape[1]) for b in batches})
    return out


def _lstm_jobs(cfg, B, L, T):
    """The four LSTMs of one c4 step: (nn.LSTM, input (B, rows, C), lengths or None), the NAR ones with every item's
    length L - 1."""
    torch.manual_seed(5)
    u = cfg["predictor_lstm_units"]
    cond = cfg["encoder_projection_units"] + cfg["emotion_units"] + cfg["speaker_units"]
    jobs = []
    lens = torch.full((B,), L - 1, dtype=torch.int32, device=DEV)
    for _ in range(2):
        jobs.append((nn.LSTM(cfg["predictor_num_memory_units"], u, batch_first=True, bidirectional=True).to(DEV),
                     torch.randn(B, L, cfg["predictor_num_memory_units"], device=DEV), lens))
    jobs.append((nn.LSTM(cfg["dur_pred_prenet_units"][-1] + cond, cfg["dur_pred_lstm_units"], num_layers=2,
                         batch_first=True).to(DEV), torch.randn(B, L, cfg["dur_pred_prenet_units"][-1] + cond, device=DEV),
                 None))
    jobs.append((nn.LSTM(cfg["postnet_num_memory_units"], cfg["postnet_lstm_units"], batch_first=True).to(DEV),
                 torch.randn(B, T, cfg["postnet_num_memory_units"], device=DEV), None))
    return jobs


def _ours(jobs):
    for lstm, x, lens in jobs:
        h = x.requires_grad_(True)
        for layer in range(lstm.num_layers):
            h, _ = sops.lstm_layer(h, lstm, layer, lens)
        h.sum().backward()


def _cudnn(jobs):
    for lstm, x, lens in jobs:
        x = x.requires_grad_(True)
        if lens is not None:
            p = nn.utils.rnn.pack_padded_sequence(x, lens.cpu(), batch_first=True, enforce_sorted=False)
            h, _ = nn.utils.rnn.pad_packed_sequence(lstm(p)[0], batch_first=True, total_length=x.shape[1])
        else:
            h, _ = lstm(x)
        h.sum().backward()


def profile_lstms(cfg, reps=3):
    """torch.profiler: GPU time per step of the four LSTMs, ours (and of it the two recurrence kernels) against cuDNN."""
    from torch.profiler import ProfilerActivity, profile
    jobs = _lstm_jobs(cfg, 32, 256, 768)
    res = {}
    for name, fn in (("ours", _ours), ("cudnn", _cudnn)):
        fn(jobs)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                fn(jobs)
            torch.cuda.synchronize()
        total = rec = 0.0
        for e in prof.key_averages():
            t = getattr(e, "self_device_time_total", None)
            t = e.self_cuda_time_total if t is None else t
            total += t
            if "lstm_rows_kernel" in e.key or "lstm_bwd_kernel" in e.key:
                rec += t
        res[f"{name}_lstm_ms_per_step"] = round(total / reps / 1e3, 3)
        if name == "ours":
            res["ours_recurrence_kernels_ms_per_step"] = round(rec / reps / 1e3, 3)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sambert_graph_step.py measures on the GPU; no CUDA device found")
    cfg = K.sambert_24k_config()
    res = {"card": _card(), "steps": args.steps, "warmup": args.warmup}
    gen = torch.Generator().manual_seed(1234)
    res["graphs_for_1000_ragged_batches"] = len({(b["input_lings"].shape[1], b["mel_targets"].shape[1])
                                                 for b in (_pad(cfg, ragged_batch(cfg, gen)) for _ in range(1000))})
    gen = torch.Generator().manual_seed(1234)
    ragged = [{k: v.to(DEV) for k, v in _pad(cfg, ragged_batch(cfg, gen)).items()} for _ in range(4)]
    res["ragged"] = compare(cfg, ragged, args.steps, args.warmup)
    del ragged
    c4 = [{k: v.to(DEV) for k, v in make_c4_batch(cfg, torch.Generator().manual_seed(1234)).items()}]
    res["c4"] = compare(cfg, c4, args.steps, args.warmup)
    res["lstm_profile_c4"] = profile_lstms(cfg)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
