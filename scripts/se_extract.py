"""Throughput of the speaker-embedding extractor: batches of seeded 1-10 s wavs at 16 kHz through
kantts_b200.speaker_embedding (Kaldi fbank + D-TDNN, seeded weights, eval-mode BatchNorm set by oracle.dtdnn.seed_bn_stats).

Per batch size it reports the per-call time (CUDA events, median of --reps calls after a warm-up), seconds of audio per wall
second, the kernel launches per call and per dense layer, the time of the separate input BatchNorm + ReLU passes replayed
alone, and the FLOPs per second of audio from the layer shapes (oracle formulation: the
reference's layer shapes, not the extra shortcut channels of our head convs).  The comparison is the oracle's torch
formulation of the D-TDNN (oracle/dtdnn.py, cuDNN convs) run one wav at a time on the same GPU, on the same features; its
time excludes the fbank, which the reference computes on the CPU.  Prints the card and its power limit with the numbers.

python scripts/se_extract.py [--batches 1 8 32] [--reps 10]"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import kantts_b200 as K  # noqa: E402
from kantts_b200 import ops  # noqa: E402
from oracle import dtdnn as od  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name() + ", power limit unknown"


def flops(model, frames):
    """Multiply-adds x 2 of one utterance of `frames` fbank frames, from the reference's layer shapes."""
    macs, f, t = 0, 80, frames
    h = model.head
    macs += f * t * h.conv1.out_channels * 9
    for layer in (h.layer1, h.layer2):
        for blk in layer:
            fo = (f - 1) // blk.stride + 1
            c = blk.conv1.out_channels
            macs += fo * t * c * blk.conv1.in_channels * 9 + fo * t * c * c * 9
            if len(blk.shortcut):
                macs += fo * t * c * blk.conv1.in_channels
            f = fo
    f = (f - 1) // 2 + 1
    macs += f * t * h.conv2.out_channels * h.conv2.in_channels * 9
    xv = model.xvector
    t2 = (t - 1) // 2 + 1
    tdnn = xv.tdnn.linear
    macs += t2 * tdnn.out_channels * tdnn.in_channels * tdnn.kernel_size[0]
    nseg = (t2 + 99) // 100
    for bi in (1, 2, 3):
        for layer in getattr(xv, f"block{bi}"):
            l1, se = layer.linear1, layer.se
            macs += t2 * l1.out_channels * l1.in_channels
            macs += t2 * se.linear_stem.out_channels * se.linear_stem.in_channels * se.linear_stem.kernel_size[0]
            macs += nseg * (se.linear1.out_channels * se.linear1.in_channels + se.linear2.out_channels * se.linear2.in_channels)
        tr = getattr(xv, f"transit{bi}").linear
        macs += t2 * tr.out_channels * tr.in_channels
    macs += xv.dense.linear.out_channels * xv.dense.linear.in_channels
    return 2.0 * macs


def dense_layer_launches(model, wav, lens):
    """{launches: dense layers} of one call: five library calls per layer, plus one operand pre-pass for each of its two
    convs that takes the TMA-fed tensor-core route (the route depends on the layer's shape)."""
    counts = {}
    orig = K.speaker.DTDNN._dense_layer

    def counted(self, *a, **kw):
        n0 = ops.launch_count()
        out = orig(self, *a, **kw)
        n = ops.launch_count() - n0
        counts[n] = counts.get(n, 0) + 1
        return out
    K.speaker.DTDNN._dense_layer = counted
    try:
        K.speaker_embedding(model, wav, lens)
    finally:
        K.speaker.DTDNN._dense_layer = orig
    return dict(sorted(counts.items()))


def nonlinear1_passes(model, frames, reps):
    """Median ms of the separate input BatchNorm + ReLU passes of one call (kt_se_affine_rows, every dense layer and
    transit at this batch's shapes), replayed alone: what fusing them into the convs' operand reads could at most save."""
    from kantts_b200._lib import ptr
    dev = next(model.parameters()).device
    B, T2 = len(frames), (max(frames) - 1) // 2 + 1
    lg = torch.tensor([(n - 1) // 2 + 1 for n in frames], dtype=torch.int32, device=dev)
    bufs, shapes = [], []
    for bi in (1, 2, 3):
        block = getattr(model.xvector, f"block{bi}")
        c0 = block.tdnnd1.nonlinear1.batchnorm.num_features
        c_final = c0 + sum(layer.se.linear_stem.out_channels for layer in block)
        slab = torch.randn(B, T2, c_final, device=dev)
        for c in [c0 + 32 * i for i in range(len(block))] + [c_final]:
            bufs.append((slab, torch.empty(B, T2, c, device=dev), torch.ones(c, device=dev), torch.zeros(c, device=dev)))
            shapes.append((c_final, c))

    def run():
        for (slab, xn, a, sh), (pitch, c) in zip(bufs, shapes):
            ops.call("kt_se_affine_rows", ptr(slab), pitch, ptr(a), ptr(sh), 1, ptr(lg, True), ptr(xn), c, B, T2, c)
    return time_calls(run, reps)[0], len(bufs)


def time_calls(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2], ts[0], ts[-1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 8, 32])
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("se_extract.py measures on a GPU; none found")
    dev = torch.device("cuda")
    torch.manual_seed(0)
    model = K.DTDNN()
    od.seed_bn_stats(model, seed=7)
    model = model.eval().to(dev)
    sd = {k: v.to(dev) for k, v in model.state_dict().items()}
    print(f"card: {card()}")
    results = []
    for B in args.batches:
        gen = torch.Generator().manual_seed(args.seed + B)
        lens = torch.randint(16000, 160001, (B,), generator=gen).tolist()
        wav = (0.1 * torch.randn(B, max(lens), generator=gen)).to(dev)
        audio_s = sum(lens) / 16000.0
        with torch.no_grad():
            n0 = ops.launch_count()
            K.speaker_embedding(model, wav, lens)
            launches = ops.launch_count() - n0
            med, lo, hi = time_calls(lambda: K.speaker_embedding(model, wav, lens), args.reps)
            feats, frames = K.kaldi_fbank(wav, lens)
            one = [feats[i:i + 1, :nf].contiguous() for i, nf in enumerate(frames)]

            def oracle():
                for x in one:
                    od.dtdnn_forward(sd, x)
            o_med, o_lo, o_hi = time_calls(oracle, max(3, args.reps // 2))
            per_layer = dense_layer_launches(model, wav, lens)
            nl1_ms, nl1_calls = nonlinear1_passes(model, frames, args.reps)
        fl = sum(flops(model, nf) for nf in frames)
        r = dict(batch=B, audio_s=round(audio_s, 2), ms_per_call=round(med, 3), ms_min=round(lo, 3), ms_max=round(hi, 3),
                 audio_s_per_s=round(audio_s / (med / 1e3), 1), launches_per_call=launches,
                 gflop_per_audio_s=round(fl / audio_s / 1e9, 3), achieved_tflops=round(fl / (med / 1e3) / 1e12, 2),
                 oracle_one_by_one_ms=round(o_med, 3), oracle_audio_s_per_s=round(audio_s / (o_med / 1e3), 1),
                 speedup_vs_oracle=round(o_med / med, 2),
                 dense_layer_launches={str(k): v for k, v in per_layer.items()},
                 nonlinear1_passes=nl1_calls, nonlinear1_ms=round(nl1_ms, 3))
        results.append(r)
        print(json.dumps(r))
    print(json.dumps({"card": card(), "results": results}))


if __name__ == "__main__":
    main()
