#!/usr/bin/env python
"""bench.py -- HiFi-GAN v1 train-step audio-samples/sec (BASELINE.json `metric`).

Workload (BASELINE config 2, SURVEY.md 8d "C2"): synthetic "v1 @ 22.05 kHz" -- class-default
Generator (512 ch, scales 8-8-2-2, causal), MultiScaleDiscriminator (yaml: scales 3, DWT pooling,
downsample [4,4,4,4,1], follow_official_norm) + MultiPeriodDiscriminator, mel (45) + LSGAN adversarial
+ feature-matching (2) losses, Adam 2e-4 (0.5, 0.9); batch 16 x 8192-sample segments per GPU; one
"step" = one full GAN train step (generator phase + discriminator phase), fp32 parameters/activations.

  python bench.py [--gpus N --steps K --warmup W]          # this repo's CUDA path
  python bench.py --impl reference ...                      # the reference's CPU path (oracle port)
  torchrun --nproc-per-node N bench.py --gpus N ...         # N > 1: one rank per GPU, NCCL all-reduce

Prints ONE JSON line (rank 0).  `value` = whole-job samples/s with inputs resident in HBM, device-timed
(CUDA events, max over ranks); `e2e` = the same through the public API from pinned HOST buffers with the
loss read back every step.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

B_PER_GPU = 16
T_WAV = 8192
HOP = 256
MSD_PARAMS = dict(
    scales=3, downsample_pooling="DWT", downsample_pooling_params={"kernel_size": 4, "stride": 2, "padding": 2},
    discriminator_params=dict(in_channels=1, out_channels=1, kernel_sizes=[15, 41, 5, 3], channels=128,
                              max_downsample_channels=1024, max_groups=16, bias=True,
                              downsample_scales=[4, 4, 4, 4, 1], nonlinear_activation="LeakyReLU",
                              nonlinear_activation_params={"negative_slope": 0.1}),
    follow_official_norm=True)
MPD_PARAMS = dict(
    periods=[2, 3, 5, 7, 11],
    discriminator_params=dict(in_channels=1, out_channels=1, kernel_sizes=[5, 3], channels=32,
                              downsample_scales=[3, 3, 3, 3, 1], max_downsample_channels=1024, bias=True,
                              nonlinear_activation="LeakyReLU", nonlinear_activation_params={"negative_slope": 0.1},
                              use_spectral_norm=False))
G_PARAMS = dict(in_channels=80, out_channels=1, channels=512, kernel_size=7, upsample_scales=[8, 8, 2, 2],
                upsample_kernal_sizes=[16, 16, 4, 4], resblock_kernel_sizes=[3, 7, 11],
                resblock_dilations=[[1, 3, 5], [1, 3, 5], [1, 3, 5]], bias=True, causal=True,
                nonlinear_activation="LeakyReLU", nonlinear_activation_params={"negative_slope": 0.1},
                use_weight_norm=True)
LOSS = {
    "generator_adv_loss": {"enable": True, "params": {"average_by_discriminators": False}, "weights": 1.0},
    "discriminator_adv_loss": {"enable": True, "params": {"average_by_discriminators": False}, "weights": 1.0},
    "stft_loss": {"enable": False},
    "mel_loss": {"enable": True, "params": dict(fs=22050, fft_size=1024, hop_size=256, win_length=1024,
                                                window="hann", num_mels=80, fmin=0, fmax=8000, log_base=None),
                 "weights": 45.0},
    "subband_stft_loss": {"enable": False},
    "feat_match_loss": {"enable": True, "params": {"average_by_discriminators": False, "average_by_layers": False},
                        "weights": 2.0},
}
ADAM = {"type": "Adam", "params": {"lr": 2.0e-4, "betas": [0.5, 0.9], "weight_decay": 0.0}}
SCHED = {"type": "MultiStepLR", "params": {"gamma": 0.5, "milestones": [200000, 400000, 600000, 800000]}}
CONFIG = {
    "Model": {"Generator": {"params": G_PARAMS, "optimizer": ADAM, "scheduler": SCHED},
              "MultiScaleDiscriminator": {"params": MSD_PARAMS, "optimizer": ADAM, "scheduler": SCHED},
              "MultiPeriodDiscriminator": {"params": MPD_PARAMS, "optimizer": ADAM, "scheduler": SCHED}},
    "Loss": LOSS, "generator_train_start_steps": 1, "discriminator_train_start_steps": 0,
    "generator_grad_norm": -1, "discriminator_grad_norm": -1,
}
FLOP_PER_SAMPLE = 25.37e6          # as executed by the reference (SURVEY.md 8d); this repo skips the unused D wgrad
WORKLOAD = "HiFi-GAN v1 G+MPD+MSD full train step, batch=16/GPU, 8192-sample segments (BASELINE configs[1])"


def synth_batch(batch, seed):
    g = torch.Generator().manual_seed(seed)
    y = (0.1 * torch.randn(batch, 1, T_WAV, generator=g)).clamp(-1, 1)
    x = torch.randn(batch, 80, T_WAV // HOP, generator=g)
    return y, x


# ---------------------------------------------------------------------------------------------------
# reference arm: the reference's own CPU implementation of the path (oracle port, torch CPU kernels)
# ---------------------------------------------------------------------------------------------------

def build_oracle_gan(seed=1234):
    """Reference-constructed weights: identical RNG stream to the reference's constructors."""
    import kantts_b200 as K
    from oracle import hifigan as O
    torch.manual_seed(seed)
    g = K.Generator(**G_PARAMS)
    msd = K.MultiScaleDiscriminator(**MSD_PARAMS)
    mpd = K.MultiPeriodDiscriminator(**MPD_PARAMS)
    return O.OracleGAN(g.state_dict(), {"MultiScaleDiscriminator": msd.state_dict(),
                                       "MultiPeriodDiscriminator": mpd.state_dict()},
                       G_PARAMS, {"MultiScaleDiscriminator": MSD_PARAMS, "MultiPeriodDiscriminator": MPD_PARAMS}, LOSS)


def cpu_reference_run(steps, warmup, sample_batch, budget_s=150.0):
    """Times the oracle port of GAN_Trainer.train_step on the host cores.  A full B=16 step takes
    minutes on CPU, so each step is a BOUNDED sample of the workload: `sample_batch` of the 16
    segments (same models, same segment length); samples/s = sample_batch * 8192 / t.
    Threads: torch-CPU convolutions stop scaling (and regress badly) past a few dozen threads on the
    many-core hosts of the GPU boxes, so min(cores, 32) threads are used and reported.  The loop is
    time-boxed: once `budget_s` is exceeded no further step is started (the steps measured so far, warm-up
    included if nothing else exists, are what is reported -- and `sample` says so)."""
    cores = min(os.cpu_count() or 1, 32)
    torch.set_num_threads(cores)
    gan = build_oracle_gan()
    y, x = synth_batch(sample_batch, 1234)
    t_begin = time.perf_counter()
    all_times = []
    for i in range(warmup + steps):
        if i > 0 and time.perf_counter() - t_begin > budget_s:
            break
        t0 = time.perf_counter()
        gan.train_step(y, x)
        all_times.append(time.perf_counter() - t0)
    timed = all_times[warmup:] if len(all_times) > warmup else all_times
    used_warm = min(warmup, len(all_times) - len(timed)) if len(all_times) > warmup else 0
    t = sum(timed) / len(timed)
    return {"value": sample_batch * T_WAV / t, "unit": "samples/s", "cores": cores, "kind": "port",
            "sample": f"{len(timed)} timed full GAN train step(s) (after {used_warm} warm-up) on {sample_batch} of the 16 "
                      f"segments x {T_WAV} samples, oracle/hifigan.py OracleGAN.train_step, torch-CPU fp32, "
                      f"{cores} threads (host has {os.cpu_count()}); {t:.2f} s/step; time-boxed at {budget_s:.0f} s"}, t


def reference_main(args, rank):
    if rank != 0:
        return
    steps = max(1, min(args.steps, 3))
    cb, t = cpu_reference_run(steps, min(args.warmup, 1), args.cpu_sample_batch)
    line = {"impl": "reference", "metric": "hifigan_train_step_audio_samples_per_sec", "value": cb["value"],
            "unit": "samples/s", "n_gpus": args.gpus, "steps": steps, "warmup": min(args.warmup, 1),
            "ms_per_step": 1e3 * t, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "f32", "data": "synthetic",
            "config": {"workload": WORKLOAD, "global_batch": B_PER_GPU * args.gpus, "segment": T_WAV,
                       "note": "CPU arm: one process on the host cores whatever N is; each step = cpu_baseline.sample "
                               "(the full 16-segment batch by default)"},
            "cpu_baseline": cb,
            "e2e": {"value": cb["value"], "unit": "samples/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
    print(json.dumps(line), flush=True)


def torch_gpu_main(args, rank, local_rank):
    """BASELINE.md section 3: the same workload on stock PyTorch library kernels (cuDNN / cuBLAS / cuFFT, fp32, TF32 off,
    cudnn.benchmark) on ONE GPU -- "the practical kernel to beat".  Informational: printed with impl = torch_gpu and the
    key gpu_library_baseline; never part of the product path."""
    if rank != 0:
        return
    from baseline.torch_gan import TorchGanStep
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    torch.manual_seed(1234)
    st = TorchGanStep(dev)
    y, x = synth_batch(B_PER_GPU, 1234)
    y, x = y.to(dev), x.to(dev)
    flush = torch.empty(256 * 1024 * 1024 // 4, device=dev, dtype=torch.float32)
    W = max(3, args.warmup)
    for _ in range(W):
        st.step((y, x))
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        flush.zero_()
        gl, dl = st.step((y, x))
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.steps
    val = B_PER_GPU * T_WAV / (ms * 1e-3)
    print(json.dumps({"impl": "torch_gpu", "metric": "hifigan_train_step_audio_samples_per_sec", "value": val,
                      "unit": "samples/s", "n_gpus": 1, "steps": args.steps, "warmup": W, "ms_per_step": ms,
                      "higher_is_better": True, "dtype": "f32", "data": "synthetic",
                      "config": {"workload": WORKLOAD, "global_batch": B_PER_GPU, "segment": T_WAV,
                                 "note": "stock torch.nn modules (baseline/torch_gan.py), cuDNN fp32, TF32 disabled, "
                                         "cudnn.benchmark on, eager; 256 MB L2 flush between steps"},
                      "gpu_library_baseline": {"value": val, "unit": "samples/s", "ms_per_step": ms,
                                               "torch": torch.__version__, "cudnn": torch.backends.cudnn.version()},
                      "losses": {"generator": float(gl), "discriminator": float(dl)}}), flush=True)


def side_workload_main(args, rank, local_rank):
    """BASELINE configs[0] / configs[3] (SURVEY.md 8d C1 / C4) on one GPU: informational lines (the driver's headline is
    the default workload).  C1: class-default Generator, eval, weight norm removed, mel (1, 80, 32) -> 8192 samples,
    audio samples / s.  C4: SAM-BERT (sambert_24k.yaml sizes) train step, B = 32, 256 symbols, 768 mel frames, mel frames / s;
    roofline = algorithmic forward + backward FLOPs (3 x 136.4 GMAC x 2, SURVEY.md 8a row S4) against the bf16x3 tensor peak."""
    if rank != 0:
        return
    import kantts_b200 as K
    from kantts_b200 import ops
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    torch.manual_seed(1234)
    W = max(3, args.warmup)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    peaks_path = os.path.join(ROOT, "MEASURED_PEAKS.json")
    bf16 = json.load(open(peaks_path)).get("bf16_tflops_sustained", 989.0) if os.path.exists(peaks_path) else 989.0   # H100 SXM data sheet, dense
    if args.workload == "c1":
        g = K.Generator(**G_PARAMS).to(dev).eval()
        g.remove_weight_norm()
        x = torch.randn(1, 80, 32, generator=torch.Generator().manual_seed(1234)).to(dev)
        with torch.no_grad():
            for _ in range(W):
                y = g(x)
            torch.cuda.synchronize()
            n0 = ops.launch_count()
            e0.record()
            for _ in range(args.steps):
                y = g(x)
            e1.record()
            torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.steps
        flops = 2 * 10.88e9
        line = {"metric": "hifigan_generator_forward_audio_samples_per_sec", "value": 8192 / (ms * 1e-3), "unit": "samples/s",
                "config": {"workload": "HiFi-GAN v1 generator forward, batch=1, 80-mel x 32 frames (BASELINE configs[0])",
                           "note": "eval, remove_weight_norm, eager launches (latency-bound: one utterance, ~100 launches)"},
                "roofline": {"bound": "tensor", "achieved": flops / (ms * 1e-3) / 1e12, "peak": bf16 / 3, "unit": "TFLOP/s",
                             "frac": flops / (ms * 1e-3) / 1e12 / (bf16 / 3), "traffic": None},
                "gpu_launches": ops.launch_count() - n0}
    else:
        from kantts_b200 import sambert
        cfg = K.sambert_24k_config()
        model = sambert.KanTtsSAMBERT(cfg).to(dev).train()
        opt = torch.optim.Adam(model.parameters(), lr=1e-3, betas=(0.9, 0.98), eps=1e-9)
        sch = K.train.NoamLR(opt, warmup_steps=4000)
        step = K.SambertStep(model, opt, sch, {"MelReconLoss": sambert.MelReconLoss(), "ProsodyReconLoss": sambert.ProsodyReconLoss()})
        gen = torch.Generator().manual_seed(1234)
        B, L, dur = 32, 256, 3
        ling = torch.stack([torch.randint(0, cfg[k], (B, L), generator=gen) for k in ("sy", "tone", "syllable_flag", "word_segment")], -1)
        batch = dict(input_lings=ling, input_emotions=torch.randint(0, cfg["emotion"], (B, L), generator=gen),
                     input_speakers=torch.randint(0, cfg["speaker"], (B, L), generator=gen),
                     valid_input_lengths=torch.full((B,), L - 1, dtype=torch.long),
                     valid_output_lengths=torch.full((B,), L * dur, dtype=torch.long),
                     mel_targets=torch.randn(B, L * dur, cfg["num_mels"], generator=gen), durations=torch.full((B, L), dur, dtype=torch.long),
                     pitch_contours=torch.randn(B, L, generator=gen), energy_contours=torch.randn(B, L, generator=gen))
        batch = {k: v.to(dev) for k, v in batch.items()}
        for _ in range(W):
            out = step.step(batch)
        torch.cuda.synchronize()
        n0 = ops.launch_count()
        e0.record()
        for _ in range(args.steps):
            out = step.step(batch)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.steps
        flops = 3 * 2 * 136.4e9
        line = {"metric": "sambert_train_step_mel_frames_per_sec", "value": B * L * dur / (ms * 1e-3), "unit": "mel frames/s",
                "config": {"workload": "SAM-BERT acoustic model fwd/bwd + Adam, batch=32, seq_len=256, 768 x 80-mel targets (BASELINE configs[3])",
                           "note": "train() mode (dropout on), eager launches, the four LSTMs on cuDNN (SURVEY 2c)"},
                "roofline": {"bound": "tensor", "achieved": flops / (ms * 1e-3) / 1e12, "peak": bf16 / 3, "unit": "TFLOP/s",
                             "frac": flops / (ms * 1e-3) / 1e12 / (bf16 / 3), "traffic": None},
                "gpu_launches": (ops.launch_count() - n0) // args.steps, "loss": float(out["TotalLoss"])}
    line.update({"n_gpus": 1, "steps": args.steps, "warmup": W, "ms_per_step": ms, "higher_is_better": True, "dtype": "f32",
                 "data": "synthetic", "vs_baseline": None})
    print(json.dumps(line), flush=True)


# ---------------------------------------------------------------------------------------------------
# clocks
# ---------------------------------------------------------------------------------------------------

class ClockSampler(threading.Thread):
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, index):
        super().__init__(daemon=True)
        self.index, self.samples, self.stop_flag = index, [], False

    def run(self):
        while not self.stop_flag:
            try:
                out = subprocess.run(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                                      "-i", str(self.index)], capture_output=True, text=True, timeout=5).stdout
                f = [s.strip() for s in out.strip().split(",")]
                if len(f) >= 9:
                    self.samples.append(f)
            except Exception:
                pass
            time.sleep(0.1)

    def summary(self):
        if not self.samples:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        sm = sorted(int(float(s[1])) for s in self.samples)
        reasons = set()
        for s in self.samples:
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), s[5:9]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        return {"sm_mhz": sm[len(sm) // 2], "sm_max_mhz": int(float(self.samples[0][2])), "reasons": sorted(reasons),
                "samples": len(sm)}


# ---------------------------------------------------------------------------------------------------
# CUDA arm
# ---------------------------------------------------------------------------------------------------

def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="native", choices=["native", "reference", "torch_gpu"],
                    help="native: this repo's CUDA path; reference: the reference's CPU path (oracle port) on the host cores; "
                         "torch_gpu: stock PyTorch (cuDNN fp32, TF32 off) on the same GPU -- informational baseline")
    ap.add_argument("--workload", default="c2", choices=["c2", "c1", "c4"],
                    help="c2 (default, the headline: BASELINE configs[1]); c1: generator forward B = 1 (configs[0]); c4: SAM-BERT "
                         "train step B = 32 x 256 symbols x 768 frames (configs[3]) -- informational lines with their own metric")
    ap.add_argument("--cpu-sample-batch", type=int, default=16,
                    help="segments per CPU step (16 = the full batch of the workload: same config as the CUDA arm)")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-roofline", action="store_true")
    ap.add_argument("--launch", default="auto", choices=["auto", "graph", "eager"],
                    help="graph: replay the step as 2 CUDA graphs; eager: per-kernel launches from Python; auto (default): "
                         "graph if a capture+replay self-test in a child process succeeds, else eager")
    ap.add_argument("--graph", action="store_true", help="same as --launch graph")
    ap.add_argument("--graph-selftest", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--ncu", action="store_true", help="profiling mode: 1 warm-up + K steps, nothing else (not a bench number)")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write what the last timed step computed (its losses, a fixed sample of every "
                         "model's updated parameters) as DIR/<name>.npy")
    args = ap.parse_args()

    rank = int(os.environ.get("RANK", 0))
    world = int(os.environ.get("WORLD_SIZE", 1))
    local_rank = int(os.environ.get("LOCAL_RANK", rank))
    if args.impl == "reference":
        return reference_main(args, rank)
    if args.impl == "torch_gpu":
        return torch_gpu_main(args, rank, local_rank)
    if args.workload != "c2":
        return side_workload_main(args, rank, local_rank)
    if world != args.gpus:
        raise SystemExit(f"--gpus {args.gpus} but WORLD_SIZE={world}: launch N>1 with torchrun (one rank per GPU)")
    if not torch.cuda.is_available():
        raise SystemExit("bench.py: no CUDA device (the CUDA arm has no CPU fallback; use --impl reference)")

    import torch.distributed as dist
    import kantts_b200 as K
    from kantts_b200 import ops

    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    if args.graph_selftest:
        return graph_selftest(dev)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=dev)
    W = max(3, args.warmup)

    launch = "graph" if args.graph else args.launch
    launch_note = ""
    if args.ncu:
        launch = "eager"
    if launch == "auto":
        # CUDA-graph replay of the full-size step crashed inside cudaGraphLaunch in earlier builds of this round:
        # prove capture + replay in a CHILD process on this device first, fall back to eager launches otherwise
        env = {k: v for k, v in os.environ.items() if k not in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR", "MASTER_PORT")}
        env["LOCAL_RANK"] = str(local_rank)
        try:
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--graph-selftest"], env=env, capture_output=True,
                               text=True, timeout=300)
            ok = r.returncode == 0 and "GRAPH_SELFTEST_OK" in r.stdout
        except Exception:
            ok = False
        flag = torch.tensor([1 if ok else 0], device=dev)
        if world > 1:
            dist.all_reduce(flag, op=dist.ReduceOp.MIN)
        launch = "graph" if int(flag) == 1 else "eager"
        launch_note = " (auto: graph self-test %s)" % ("passed" if launch == "graph" else "FAILED -> eager fallback")

    torch.manual_seed(1234)                      # identical replicas on every rank (reference RNG stream)
    use_graph = launch == "graph"
    model, opt, sched = K.hifigan_model_builder(CONFIG, dev)
    crit = K.criterion_builder(CONFIG, dev)
    step = K.GanStep(model, opt, sched, crit, CONFIG, cuda_graph=use_graph)
    y_h, x_h = synth_batch(B_PER_GPU, 1234 + rank)
    y_h, x_h = y_h.pin_memory(), x_h.pin_memory()
    y_d, x_d = y_h.to(dev), x_h.to(dev)
    flush = torch.empty(256 * 1024 * 1024 // 4, device=dev, dtype=torch.float32)   # > 50 MB L2

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    if args.ncu:
        step.step((y_d, x_d))
        torch.cuda.synchronize()
        torch.cuda.profiler.start()
        for _ in range(args.steps):
            step.step((y_d, x_d))
        torch.cuda.synchronize()
        torch.cuda.profiler.stop()
        print(json.dumps({"ncu_mode": True, "steps": args.steps, "launches": ops.launch_count()}))
        return
    launches_per_step = None
    for i in range(W + (3 if use_graph else 0)):     # graph mode: W eager steps, 1 capture step, 2 replays
        l0 = ops.launch_count()
        log = step.step((y_d, x_d))
        if ops.launch_count() > l0:
            launches_per_step = ops.launch_count() - l0   # kernels issued by one (eager / captured) step
    barrier()

    # ---- timed region 1: inputs resident in HBM ----
    sampler = ClockSampler(local_rank)
    sampler.start()
    n0 = ops.launch_count()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    barrier()
    e0.record()
    for _ in range(args.steps):
        flush.zero_()                             # L2 flush between timed iterations (256 MB write)
        log = step.step((y_d, x_d))
    e1.record()
    barrier()
    sampler.stop_flag = True
    ms = e0.elapsed_time(e1)
    launches = (ops.launch_count() - n0 + args.steps) if not use_graph else (launches_per_step + 1) * args.steps
    t_ms = torch.tensor([ms], device=dev)
    if world > 1:
        dist.all_reduce(t_ms, op=dist.ReduceOp.MAX)
    ms_per_step = float(t_ms) / args.steps
    value = world * B_PER_GPU * T_WAV / (ms_per_step * 1e-3)

    # ---- timed region 2: end to end from pinned host buffers, loss read back each step ----
    barrier()
    e0.record()
    for _ in range(args.steps):
        flush.zero_()
        if use_graph:
            log = step.step((y_h, x_h))               # pinned host -> the graph's static input buffers (H2D inside)
        else:
            yb = y_h.to(dev, non_blocking=True)
            xb = x_h.to(dev, non_blocking=True)
            log = step.step((yb, xb))
        g_loss = float(log["generator_loss"])     # D2H read of the step's result
        d_loss = float(log["discriminator_loss"])
    e1.record()
    barrier()
    t2 = torch.tensor([e0.elapsed_time(e1)], device=dev)
    if world > 1:
        dist.all_reduce(t2, op=dist.ReduceOp.MAX)
    e2e_value = world * B_PER_GPU * T_WAV / (float(t2) / args.steps * 1e-3)
    clocks = sampler.summary()
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, log, model)

    line = {
        "metric": "hifigan_train_step_audio_samples_per_sec", "value": value, "unit": "samples/s",
        "n_gpus": world, "steps": args.steps, "warmup": W, "ms_per_step": ms_per_step, "higher_is_better": True,
        "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": WORKLOAD, "global_batch": B_PER_GPU * world, "segment": T_WAV, "parallelism": f"dp{world}",
                   "precision": "fp32 storage; tensor-core layers bf16x3 split (fp32-equivalent), others exact fp32 FFMA",
                   "l2": "explicit 256 MB flush write between timed iterations",
                   "launch": ("2 CUDA graphs per step (replay) + eager Adam / NCCL between them" if use_graph else
                              "eager launches; independent sub-discriminators / parallel resblocks on side streams") + launch_note,
                   "gflop_per_step_as_reference_executes": FLOP_PER_SAMPLE * B_PER_GPU * T_WAV / 1e9},
        "e2e": {"value": e2e_value, "unit": "samples/s", "h2d_bytes_per_step": (y_h.numel() + x_h.numel()) * 4,
                "d2h_bytes_per_step": 8},
        "gpu_launches": launches, "tc_launches_total": ops.tc_launch_count(), "clocks": clocks,
        "losses": {"generator": g_loss, "discriminator": d_loss},
    }

    if not args.no_roofline:
        # every rank runs the instrumented step (it contains the gradient all-reduces); rank 0 reports
        roof, shares = roofline_leg(step, (y_d, x_d), ops, ms_per_step)
        if rank == 0:
            line["roofline"], line["kernel_shares"] = roof, shares
    if world > 1:
        dist.barrier()
    if rank == 0 and world == 1 and not args.no_cpu_baseline:
        line["cpu_baseline"], _ = cpu_reference_run(2, 1, args.cpu_sample_batch)      # ~15-20 s of CPU work
    if rank == 0:
        print(json.dumps(line), flush=True)
    if world > 1:
        dist.destroy_process_group()


def dump_outputs(out_dir, log, model, param_sample=1 << 20):
    """What the last timed step computed, for comparing two builds output for output: every tensor of the step's log
    (the losses, float64) and a fixed, seeded sample of `param_sample` parameters of every model after that step's
    optimizer update (float32; the generator and each discriminator, 4 MB each)."""
    import re
    import numpy as np
    os.makedirs(out_dir, exist_ok=True)
    for k, v in log.items():
        if torch.is_tensor(v):
            np.save(os.path.join(out_dir, re.sub(r"[^A-Za-z0-9_.-]", "_", k) + ".npy"), v.detach().double().cpu().numpy())
    mods = {"generator": model["generator"], **{f"discriminator_{k}": v for k, v in model["discriminator"].items()}}
    for name, m in mods.items():
        flat = torch.cat([p.detach().reshape(-1).float().cpu() for p in m.parameters()])
        idx = torch.randperm(flat.numel(), generator=torch.Generator().manual_seed(0))[:param_sample].sort().values
        np.save(os.path.join(out_dir, f"{name}_params_sample.npy"), flat[idx].numpy())


def graph_selftest(dev):
    """Child-process check: eager warm-up, capture, a few replays, finite losses."""
    import kantts_b200 as K
    torch.manual_seed(1234)
    model, opt, sched = K.hifigan_model_builder(CONFIG, dev)
    crit = K.criterion_builder(CONFIG, dev)
    step = K.GanStep(model, opt, sched, crit, CONFIG, cuda_graph=True)
    y, x = synth_batch(B_PER_GPU, 1234)
    y, x = y.to(dev), x.to(dev)
    log = None
    for _ in range(step.graph_warmup + 4):
        log = step.step((y, x))
    torch.cuda.synchronize()
    vals = [float(v) for v in log.values() if torch.is_tensor(v)]
    assert step._graphs is not None and all(v == v and abs(v) < 1e6 for v in vals), vals
    print("GRAPH_SELFTEST_OK", vals, flush=True)


def roofline_leg(step, batch, ops, ms_per_step):
    """One extra instrumented step: every conv library call is bracketed by CUDA events on the
    launching stream; the dominant kernel class's achieved algorithmic rate is reported against the
    measured peak (MEASURED_PEAKS.json, else the H100 SXM data-sheet figures)."""
    from kantts_b200 import hifigan
    step.invalidate_weight_caches()        # eager launches after graph replays: prepared weights must be rebuilt
    # side streams OFF for this step: with concurrent streams an event pair around one launch also measures the
    # time the kernel spent queued behind other streams' kernels, i.e. not that kernel's own duration
    par, hifigan._PARALLEL_STREAMS = hifigan._PARALLEL_STREAMS, False
    wga, ops._WGRAD_ASYNC = ops._WGRAD_ASYNC, False          # (the weight-gradient side streams as well)
    pf = os.environ.get("KANTTS_B200_PREFETCH")
    os.environ["KANTTS_B200_PREFETCH"] = "0"
    try:
        prof = ops.set_profiler(True)
        step._eager_step(*batch)
        summ = prof.summary()
    finally:
        ops.set_profiler(False)
        hifigan._PARALLEL_STREAMS, ops._WGRAD_ASYNC = par, wga
        if pf is None:
            os.environ.pop("KANTTS_B200_PREFETCH", None)
        else:
            os.environ["KANTTS_B200_PREFETCH"] = pf
    peaks_path = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(peaks_path):
        pk = json.load(open(peaks_path))
        bf16, hbm, src = pk.get("bf16_tflops_sustained", 989.0), pk.get("hbm_gbs", 3350.0), "measured"
    else:
        bf16, hbm, src = 989.0, 3350.0, "H100 SXM data sheet (not reached)"
    total_ms = sum(v["ms"] for v in summ.values())
    shares = {k: {"calls": v["calls"], "ms": round(v["ms"], 3), "share_of_instrumented": round(v["ms"] / total_ms, 4),
                  "tflops_algorithmic": round(v["flops"] / (v["ms"] * 1e-3) / 1e12, 2) if v["ms"] > 0 else None,
                  "gbs_layer_boundary": round(v["bytes"] / (v["ms"] * 1e-3) / 1e9, 1) if v["ms"] > 0 else None}
              for k, v in sorted(summ.items(), key=lambda kv: -kv[1]["ms"])}
    top = max(summ, key=lambda k: summ[k]["ms"])
    v = summ[top]
    achieved = v["flops"] / (v["ms"] * 1e-3) / 1e12
    peak = bf16 / 3.0                      # bf16x3: three tensor MACs per algorithmic MAC
    traffic = None
    tp = os.path.join(ROOT, "profiles", "traffic.json")
    if os.path.exists(tp):
        traffic = json.load(open(tp)).get(top)
    roof = {"bound": "tensor", "kernel": top, "achieved": achieved, "peak": peak, "unit": "TFLOP/s",
            "frac": achieved / peak, "traffic": traffic,
            "note": f"algorithmic fp32-equivalent FLOPs (2*MAC) per launch / CUDA-event duration, averaged over "
                    f"{v['calls']} launches of one instrumented step; peak = {src} bf16 sustained {bf16} TF/s / 3 "
                    f"(bf16x3 issues 3 tensor MACs per MAC); HBM peak {hbm} GB/s ({src})",
            "avg_launch_ms": v["ms"] / v["calls"], "flops_per_launch": v["flops"] / v["calls"],
            "instrumented_conv_ms": total_ms, "step_ms": ms_per_step}
    return roof, shares


if __name__ == "__main__":
    main()
