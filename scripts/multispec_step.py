"""Time the multi-resolution spectrogram discriminator (MultiSpecDiscriminator, "MRD") in the bench.py workload.

Configuration C2 of bench.py (v1 generator, MSD + MPD, batch 16 x 8192 samples), alone and with an MRD added at the
reference's resolutions (FFT 1024 / 2048 / 512, hop 120 / 240 / 50, window 600 / 1200 / 240), in two sizes:
  defaults   the reference's discriminator_params with kernel_size 11 (channels 15, init_kernel 1)
  wide       SpecDiscriminator's own defaults (channels 32, init_kernel 15, kernel_size 11)
Measures, on one GPU, with the card name and power limit read in the same run:
  step       the CUDA-graph GAN step (GanStep(cuda_graph=True)) of each configuration, alternating, ``--runs`` runs of
             ``--steps`` steps each (CUDA events around each run)
  launches   kernels per eager step (torch.profiler), and the library calls among them (ops.launch_count)
  kernels    (torch.profiler, a separate pass) the device time of the MRD's forward + backward on the pair batch (2 x 16
             waveforms), with its most expensive kernels, against the reference's formulation (torch.stft + weight-normed
             F.conv2d, torch's default TF32 convolutions) on the same tensors and weights; and the largest relative
             difference between the two, with the reference's formulation in full fp32
Prints one JSON line.

    python scripts/multispec_step.py [--steps 20] [--runs 3]
"""
import argparse
import copy
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (the workload's configuration)
import kantts_b200 as K  # noqa: E402
from kantts_b200 import ops  # noqa: E402

DEV = "cuda"
RESOLUTIONS = dict(fft_sizes=[1024, 2048, 512], hop_sizes=[120, 240, 50], win_lengths=[600, 1200, 240])
MRD = {
    "defaults": dict(RESOLUTIONS, discriminator_params={
        "channels": 15, "init_kernel": 1, "kernel_size": 11, "stride": 2, "use_spectral_norm": False,
        "window": "hann_window", "nonlinear_activation": "LeakyReLU", "nonlinear_activation_params": {"negative_slope": 0.1}}),
    "wide": dict(RESOLUTIONS, discriminator_params={"channels": 32, "init_kernel": 15, "kernel_size": 11, "stride": 2}),
}


def config(mrd):
    cfg = copy.deepcopy(bench.CONFIG)
    if mrd is not None:
        cfg["Model"]["MultiSpecDiscriminator"] = {"params": MRD[mrd], "optimizer": bench.ADAM, "scheduler": bench.SCHED}
    return cfg


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def _batch(seed):
    y, x = bench.synth_batch(bench.B_PER_GPU, seed)
    return y.to(DEV), x.to(DEV)


def _timed(fn, n):
    """-> milliseconds per call over n calls, from CUDA events around the whole run"""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / n


def _build(mrd, **kw):
    cfg = config(mrd)
    torch.manual_seed(1234)
    model, opt, sched = K.hifigan_model_builder(cfg, DEV, capturable=kw.get("cuda_graph", False))
    return K.GanStep(model, opt, sched, K.criterion_builder(cfg, DEV), cfg, **kw)


LEGS = (("base", None), ("mrd_defaults", "defaults"), ("mrd_wide", "wide"))


def measure_steps(steps, runs):
    batches = [_batch(s) for s in range(4)]
    legs = {}
    for name, mrd in LEGS:
        step = _build(mrd, cuda_graph=True, graph_warmup=2)
        it = iter(range(10 ** 9))
        fn = lambda s=step, it=it: s.step(batches[next(it) % len(batches)])  # noqa: E731
        for _ in range(5):                                   # eager warm-up, capture, replays
            log = fn()
        torch.cuda.synchronize()
        legs[name] = (step, fn, {k: round(v, 5) for k, v in K.train.losses_to_float(log).items()})
    times = {name: [] for name in legs}
    for _ in range(runs):                                    # alternating, so drift hits all legs alike
        for name, (_, fn, _) in legs.items():
            times[name].append(_timed(fn, steps))
    out = {}
    for name, ts in times.items():
        med = statistics.median(ts)
        out[name] = dict(ms_per_step=[round(t, 3) for t in ts], median_ms=round(med, 3),
                         spread_pct=round(100 * (max(ts) - min(ts)) / med, 2),
                         samples_per_s=round(bench.B_PER_GPU * bench.T_WAV / (med / 1e3)), losses=legs[name][2])
    for name in ("mrd_defaults", "mrd_wide"):
        out[f"{name}_over_base"] = round(out[name]["median_ms"] / out["base"]["median_ms"], 4)
    del legs
    torch.cuda.empty_cache()
    return out


def measure_launches():
    """Kernels per eager step: all device kernels (torch.profiler) and the library calls among them."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    y, x = _batch(0)
    out = {}
    for name, mrd in LEGS:
        step = _build(mrd)
        step.step((y, x))
        torch.cuda.synchronize()
        n0 = ops.launch_count()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            step.step((y, x))
            torch.cuda.synchronize()
        kernels = sum(e.count for e in prof.key_averages() if e.device_type == DeviceType.CUDA)
        out[name] = dict(device_kernels=kernels, library_launches=ops.launch_count() - n0)
        del step
        torch.cuda.empty_cache()
    for name in ("mrd_defaults", "mrd_wide"):
        out[f"{name}_added"] = {k: out[name][k] - out["base"][k] for k in out["base"]}
    return out


def _kernel_us(fn, iters=20, top=0):
    """-> microseconds of device kernel time per call, from torch.profiler over ``iters`` calls (and, with ``top``, the
    ``top`` kernels that took the most of it: [name, us per call])"""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    events = sorted((e for e in prof.key_averages() if e.device_type == DeviceType.CUDA),
                    key=lambda e: -e.self_device_time_total)
    total = round(sum(e.self_device_time_total for e in events) / iters, 1)
    if not top:
        return total
    return total, [[e.key[:60], round(e.self_device_time_total / iters, 1)] for e in events[:top]]


def _torch_mrd(m):
    """The reference's formulation (hifigan.py:481-617 on audio_torch.stft): torch.stft and weight-normed F.conv2d on
    (B, F, frames, 1), with its own leaf copies of the module's parameters.  -> (forward, parameters)"""
    params = {k: v.detach().clone().requires_grad_(True) for k, v in m.named_parameters()}

    def conv(prefix, x, stride, pad):
        v, g, b = params[prefix + "weight_v"], params[prefix + "weight_g"], params[prefix + "bias"]
        w = v * (g / v.norm(2, dim=(1, 2, 3), keepdim=True))
        return F.conv2d(x, w, b, stride=stride, padding=pad)

    def forward(y):
        outs, fmaps = [], []
        for i, d in enumerate(m.discriminators):
            with torch.no_grad():
                s = torch.stft(y.squeeze(1), d.fft_size, d.shift_size, d.win_length, d.window, return_complex=True)
                x = torch.sqrt(torch.clamp(s.real ** 2 + s.imag ** 2, min=1e-7)).unsqueeze(-1)
            fm = []
            for l, seq in enumerate(d.convs):
                spec = seq[0].spec
                x = F.leaky_relu(conv(f"discriminators.{i}.convs.{l}.0.", x, (spec.stride, 1), seq[0].pad_width), 0.1)
                fm.append(x)
            x = conv(f"discriminators.{i}.conv_post.", x, 1, (1, 0))
            fm.append(x)
            outs.append(x)
            fmaps.append(fm)
        return outs, fmaps
    return forward, list(params.values())


def measure_kernels(mrd):
    torch.manual_seed(1234)
    m = K.MultiSpecDiscriminator(**MRD[mrd]).to(DEV)
    ref_fwd, ref_params = _torch_mrd(m)
    y = torch.cat([_batch(7)[0], _batch(8)[0]])                # the pair batch of one phase
    outs, fmaps = m(y)
    rs = [torch.randn_like(t) for t in outs + [f for fm in fmaps for f in fm]]

    def run(fwd, params):
        def fn():
            for p in params:
                p.grad = None
            o, fm = fwd(y)
            sum((t * r).sum() for t, r in zip(o + [f for f_ in fm for f in f_], rs)).backward()
            K.hifigan.join_side_streams(y.device)
        return fn
    k_fn, t_fn = run(m, list(m.parameters())), run(ref_fwd, ref_params)
    # the differences against the reference's formulation in full fp32 (torch's default runs cuDNN convolutions in TF32)
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    k_fn()
    t_fn()
    torch.cuda.synchronize()
    with torch.no_grad():
        (ko, kf), (to, tf) = m(y), ref_fwd(y)
        outs = list(zip(ko + [f for fm in kf for f in fm], to + [f for fm in tf for f in fm]))
        grads = list(zip([p.grad for p in m.parameters()], [p.grad for p in ref_params]))
        diff = lambda pairs: f"{max(float((a - b).norm() / b.norm()) for a, b in pairs):.2e}"  # noqa: E731
        err = dict(outputs_and_maps=diff(outs), parameter_gradients=diff(grads))
    torch.backends.cudnn.allow_tf32 = tf32
    k_us, k_top = _kernel_us(k_fn, top=6)
    return dict(kernels_us=k_us, top_kernels=k_top, torch_stft_conv2d_us=_kernel_us(t_fn),
                max_rel_diff_fp32=err, pair_batch=list(y.shape))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--skip-step", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("multispec_step.py measures on the GPU; no CUDA device found")
    res = {"card": _card(), "batch": [bench.B_PER_GPU, bench.T_WAV], "steps_per_run": args.steps, "runs": args.runs}
    res["kernels"] = {name: measure_kernels(name) for name in MRD}
    res["launches"] = measure_launches()
    if not args.skip_step:
        res["step"] = measure_steps(args.steps, args.runs)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
