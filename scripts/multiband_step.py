"""Time the multi-band HiFi-GAN against the full-band one at hifigan_v1_24k.yaml sizes.

Multi-band config: hifigan_v1_24k.yaml with ``out_channels: 4``, ``upsample_scales [5, 3, 2, 2]``,
``upsample_kernal_sizes [10, 6, 4, 4]`` (hop 60 per sub-band, 240 at the full rate) and its ``subband_stft_loss`` section
enabled (FFT sizes 384 / 683 / 171).  Measures, on one GPU, with the card name and power limit read in the same run:
  step      the CUDA-graph GAN step (GanStep(cuda_graph=True)) at batch 16 x 9600 samples, multi-band against full-band,
            alternating, ``--runs`` runs of ``--steps`` steps each (CUDA events around each run)
  synth     the generator forward (eval, no grad) plus PQMF synthesis against the full-band generator forward, for
            1 x 800 and 16 x 800 mel frames
  kernels   (a separate torch.profiler run) the device time of PQMF analysis + synthesis, forward and backward, and of the
            sub-band STFT loss forward + backward, against the reference's F.conv1d / torch.stft composites on the same
            tensors; also their relative difference
Prints one JSON line.

    python scripts/multiband_step.py [--steps 20] [--runs 3]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import kantts_b200 as K  # noqa: E402

DEV = "cuda"
BATCH, T_WAV, HOP = 16, 9600, 240
SUB_STFT = dict(fft_sizes=[384, 683, 171], hop_sizes=[35, 75, 15], win_lengths=[150, 300, 60], window="hann_window")
MSD = dict(scales=3, downsample_pooling="DWT", downsample_pooling_params={"kernel_size": 4, "stride": 2, "padding": 2},
           discriminator_params=dict(in_channels=1, out_channels=1, kernel_sizes=[15, 41, 5, 3], channels=128,
                                     max_downsample_channels=1024, max_groups=16, bias=True,
                                     downsample_scales=[4, 4, 4, 4, 1], nonlinear_activation="LeakyReLU",
                                     nonlinear_activation_params={"negative_slope": 0.1}),
           follow_official_norm=True)
MPD = dict(periods=[2, 3, 5, 7, 11],
           discriminator_params=dict(in_channels=1, out_channels=1, kernel_sizes=[5, 3], channels=32,
                                     downsample_scales=[3, 3, 3, 3, 1], max_downsample_channels=1024, bias=True,
                                     nonlinear_activation="LeakyReLU", nonlinear_activation_params={"negative_slope": 0.1},
                                     use_spectral_norm=False))
G_FULL = dict(in_channels=80, out_channels=1, channels=512, kernel_size=7, upsample_scales=[8, 5, 3, 2],
              upsample_kernal_sizes=[16, 10, 6, 4], resblock_kernel_sizes=[3, 7, 11],
              resblock_dilations=[[1, 3, 5], [1, 3, 5], [1, 3, 5]], bias=True, causal=True,
              nonlinear_activation="LeakyReLU", nonlinear_activation_params={"negative_slope": 0.1}, use_weight_norm=True)
G_MB = dict(G_FULL, out_channels=4, upsample_scales=[5, 3, 2, 2], upsample_kernal_sizes=[10, 6, 4, 4])


def config(multiband):
    adam = {"type": "Adam", "params": {"lr": 2.0e-4, "betas": [0.5, 0.9], "weight_decay": 0.0}}
    sched = {"type": "MultiStepLR", "params": {"gamma": 0.5, "milestones": [200000, 400000, 600000, 800000]}}
    loss = {
        "generator_adv_loss": {"enable": True, "params": {"average_by_discriminators": False}, "weights": 1.0},
        "discriminator_adv_loss": {"enable": True, "params": {"average_by_discriminators": False}, "weights": 1.0},
        "stft_loss": {"enable": False},
        "mel_loss": {"enable": True, "params": dict(fs=24000, fft_size=1024, hop_size=240, win_length=1024, window="hann",
                                                    num_mels=80, fmin=0, fmax=8000, log_base=None), "weights": 45.0},
        "subband_stft_loss": {"enable": multiband, "params": SUB_STFT},
        "feat_match_loss": {"enable": True, "params": {"average_by_discriminators": False, "average_by_layers": False},
                            "weights": 2.0},
    }
    return {"Model": {"Generator": {"params": G_MB if multiband else G_FULL, "optimizer": adam, "scheduler": sched},
                      "MultiScaleDiscriminator": {"params": MSD, "optimizer": adam, "scheduler": sched},
                      "MultiPeriodDiscriminator": {"params": MPD, "optimizer": adam, "scheduler": sched}},
            "Loss": loss, "generator_train_start_steps": 1, "discriminator_train_start_steps": 0,
            "generator_grad_norm": -1, "discriminator_grad_norm": -1}


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def _batch(seed):
    g = torch.Generator().manual_seed(seed)
    y = (0.1 * torch.randn(BATCH, 1, T_WAV, generator=g)).clamp(-1, 1).to(DEV)
    x = torch.randn(BATCH, 80, T_WAV // HOP, generator=g).to(DEV)
    return y, x


def _timed(fn, n):
    """-> milliseconds per call over n calls, from CUDA events around the whole run"""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / n


def measure_steps(steps, runs):
    batches = [_batch(s) for s in range(4)]
    legs = {}
    for name, mb in (("multiband", True), ("fullband", False)):
        cfg = config(mb)
        torch.manual_seed(1234)
        model, opt, sched = K.hifigan_model_builder(cfg, DEV, capturable=True)
        step = K.GanStep(model, opt, sched, K.criterion_builder(cfg, DEV), cfg, cuda_graph=True, graph_warmup=2)
        it = iter(range(10 ** 9))
        legs[name] = (step, lambda s=step, it=it: s.step(batches[next(it) % len(batches)]))
        for _ in range(5):                                   # eager warm-up, capture, replays
            log = legs[name][1]()
        torch.cuda.synchronize()
        legs[name] += (sorted(K.train.losses_to_float(log)),)
    times = {name: [] for name in legs}
    for _ in range(runs):                                    # alternating, so drift hits both legs alike
        for name, (_, fn, _) in legs.items():
            times[name].append(_timed(fn, steps))
    out = {}
    for name, ts in times.items():
        out[name] = dict(ms_per_step=[round(t, 3) for t in ts], median_ms=round(statistics.median(ts), 3),
                         spread_pct=round(100 * (max(ts) - min(ts)) / statistics.median(ts), 2),
                         samples_per_s=round(BATCH * T_WAV / (statistics.median(ts) / 1e3)), losses=legs[name][2])
    out["multiband_over_fullband"] = round(out["multiband"]["median_ms"] / out["fullband"]["median_ms"], 3)
    del legs
    torch.cuda.empty_cache()
    return out


def measure_synthesis(reps):
    torch.manual_seed(1234)
    g_mb = K.Generator(**G_MB).to(DEV).eval()
    g_mb.pqmf = K.PQMF().to(DEV)
    g_fb = K.Generator(**G_FULL).to(DEV).eval()
    out = {}
    with torch.no_grad():
        for b in (1, 16):
            x = torch.randn(b, 80, 800, device=DEV)
            fns = {"multiband": lambda: g_mb.pqmf.synthesis(g_mb(x)), "fullband": lambda: g_fb(x)}
            for fn in fns.values():
                fn()
            torch.cuda.synchronize()
            ts = {k: [] for k in fns}
            for _ in range(3):
                for k, fn in fns.items():
                    ts[k].append(_timed(fn, reps))
            out[f"{b}x800"] = {k: dict(ms=[round(t, 3) for t in v], median_ms=round(statistics.median(v), 3))
                               for k, v in ts.items()}
            out[f"{b}x800"]["multiband_over_fullband"] = round(out[f"{b}x800"]["multiband"]["median_ms"] /
                                                               out[f"{b}x800"]["fullband"]["median_ms"], 3)
    return out


def _kernel_us(fn, iters=20):
    """-> microseconds of device kernel time per call, from torch.profiler over ``iters`` calls"""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    return round(sum(e.self_device_time_total for e in prof.key_averages() if e.device_type == DeviceType.CUDA) / iters, 1)


def _torch_pqmf(p):
    """the reference's two-conv formulation (kantts/models/pqmf.py:107-134) on the module's buffers"""
    pad = p.taps // 2

    def analysis(x):
        return F.conv1d(F.conv1d(F.pad(x, (pad, pad)), p.analysis_filter), p.updown_filter, stride=p.subbands)

    def synthesis(x):
        y = F.conv_transpose1d(x, p.updown_filter * p.subbands, stride=p.subbands)
        return F.conv1d(F.pad(y, (pad, pad)), p.synthesis_filter)
    return analysis, synthesis


def _torch_stft_loss(x, y):
    """audio_torch.stft + loss.py:314-441 (MultiResolutionSTFTLoss over sub-bands) with torch.stft"""
    x, y = x.reshape(-1, x.size(2)), y.reshape(-1, y.size(2))
    sc = mag = 0.0
    for n, h, w in zip(SUB_STFT["fft_sizes"], SUB_STFT["hop_sizes"], SUB_STFT["win_lengths"]):
        win = torch.hann_window(w, device=x.device)
        m = [torch.sqrt(torch.clamp(torch.view_as_real(torch.stft(s, n, h, w, win, return_complex=True)).pow(2).sum(-1),
                                    min=1e-7)).transpose(2, 1) for s in (x, y)]
        sc = sc + torch.linalg.vector_norm(m[1] - m[0]) / torch.linalg.vector_norm(m[1])
        mag = mag + torch.mean(torch.abs(torch.log(m[1]) - torch.log(m[0])))
    k = len(SUB_STFT["fft_sizes"])
    return sc / k, mag / k


def measure_kernels():
    p = K.PQMF().to(DEV)
    t_an, t_syn = _torch_pqmf(p)
    y, _ = _batch(7)
    y_mb = (0.1 * torch.randn(BATCH, 4, T_WAV // 4, device=DEV)).requires_grad_(True)
    r = torch.randn(BATCH, 1, T_WAV, device=DEV)
    r_mb = torch.randn(BATCH, 4, T_WAV // 4, device=DEV)
    yg = y.clone().requires_grad_(True)

    def pqmf_run(an, syn):
        def fn():
            yg.grad = y_mb.grad = None
            ((an(yg) * r_mb).sum() + (syn(y_mb) * r).sum()).backward()
        return fn
    k_fn, t_fn = pqmf_run(p.analysis, p.synthesis), pqmf_run(t_an, t_syn)
    k_fn()
    gk = (yg.grad.clone(), y_mb.grad.clone())
    t_fn()
    gt = (yg.grad.clone(), y_mb.grad.clone())
    with torch.no_grad():
        pairs = [(p.analysis(y), t_an(y)), (p.synthesis(y_mb), t_syn(y_mb)), *zip(gk, gt)]
        err_pqmf = max(float((a - b).norm() / b.norm()) for a, b in pairs)
    crit = K.MultiResolutionSTFTLoss(**SUB_STFT).to(DEV)
    y_sb = p.analysis(y).detach()

    def loss_run(f):
        def fn():
            y_mb.grad = None
            sc, mag = f(y_mb, y_sb)
            (sc + mag).backward()
        return fn
    with torch.no_grad():
        a, b = crit(y_mb, y_sb), _torch_stft_loss(y_mb, y_sb)
    err_loss = max(abs(float(a[0]) - float(b[0])) / abs(float(b[0])), abs(float(a[1]) - float(b[1])) / abs(float(b[1])))
    return dict(
        pqmf_fwd_bwd_us=dict(kernels=_kernel_us(k_fn), torch_conv=_kernel_us(t_fn), max_rel_diff=f"{err_pqmf:.2e}"),
        subband_stft_loss_fwd_bwd_us=dict(kernels=_kernel_us(loss_run(crit)), torch_stft=_kernel_us(loss_run(_torch_stft_loss)),
                                          max_rel_diff=f"{err_loss:.2e}"),
        shapes=dict(waveform=[BATCH, 1, T_WAV], subbands=[BATCH, 4, T_WAV // 4]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--skip-step", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("multiband_step.py measures on the GPU; no CUDA device found")
    res = {"card": _card(), "batch": [BATCH, T_WAV], "steps_per_run": args.steps, "runs": args.runs}
    res["kernels"] = measure_kernels()
    res["synthesis"] = measure_synthesis(10)
    if not args.skip_step:
        res["step"] = measure_steps(args.steps, args.runs)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
