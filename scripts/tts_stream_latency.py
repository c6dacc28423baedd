"""Latency of streamed text-to-speech (infer.stream_synthesize) on the GPU.

SAM-BERT with the sambert_24k.yaml network (seeded weights) and the hifigan_v1_24k.yaml generator (hop 240 at 24 kHz), over
B in {1, 8} utterances x chunk_steps in {1, 4, 16} decoder steps (3 frames each) per chunk.  ``--vocoder noncausal_16k``:
the same network (sambert_16k.yaml differs only in its data) into the non-causal hifigan_noncausal_v1_16k.yaml generator
(hop 200 at 16 kHz), streamed with ``allow_lookahead=True``: its audio waits for 3424 samples (214 ms) of look-ahead.
``--vocoder multiband_24k``: the causal multi-band generator of scripts/multiband_step.py (4 sub-bands, hop 240 at 24 kHz)
with its PQMF, whose synthesis adds 31 samples (1.3 ms) of look-ahead.
Per setting:
  ttfa_ms            time to first audio: host clock from the stream_synthesize call to a synchronize after the first chunk
                     (with a non-causal vocoder, the first chunk holding audio)
  chunk_ms           device time per chunk after the first (CUDA events at each yielded chunk; includes the device idling
                     while the host runs the per-step decoder loop)
  stream_ms          host clock from the call to a synchronize after the last chunk
  rtf                real-time factor per slot: audio seconds of the longest slot / stream seconds (> 1: faster than real time)
  dec_launches_per_step  library launches of one decoder step
  synth_ms           the same input through synthesize(), host clock to a synchronize
Seeded weights predict near-zero durations, so the duration predictor's output bias is set to give about DUR frames per
symbol: the utterances are then as long as real ones.  Prints the card and its power limit, read in the same run, and all
rows as one JSON line.

    python scripts/tts_stream_latency.py [--vocoder causal_24k|noncausal_16k|multiband_24k] [--symbols 64] [--repeats 3]
                                         [--out DIR]"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import kantts_b200 as K  # noqa: E402
from kantts_b200 import ops  # noqa: E402

DUR = 5.0
# generator structure and sample rate of each vocoder
VOCODERS = {
    "causal_24k": (dict(upsample_scales=[8, 5, 3, 2], upsample_kernal_sizes=[16, 10, 6, 4]), 24000),    # hifigan_v1_24k.yaml
    "noncausal_16k": (dict(channels=256, upsample_scales=[10, 5, 2, 2], upsample_kernal_sizes=[20, 11, 4, 4],
                           resblock_dilations=[[1, 3, 5, 7]] * 3, causal=False), 16000),      # hifigan_noncausal_v1_16k.yaml
    # G_MB of scripts/multiband_step.py: 4 sub-bands at 6 kHz, with its PQMF (hop 240 at 24 kHz)
    "multiband_24k": (dict(out_channels=4, upsample_scales=[5, 3, 2, 2], upsample_kernal_sizes=[10, 6, 4, 4]), 24000),
}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def models(vocoder="causal_24k"):
    """-> (SAM-BERT, the ``vocoder``'s generator, its sample rate)"""
    torch.manual_seed(0)
    am = K.KanTtsSAMBERT(K.sambert_24k_config())
    with torch.no_grad():
        am.variance_adaptor.duration_predictor.fc.bias.fill_(math.log(DUR + 1))
    gcfg, sr = VOCODERS[vocoder]
    gen = K.Generator(**gcfg).cuda().eval()
    if gen.out_channels > 1:
        gen.pqmf = K.PQMF(gen.out_channels).cuda()
    return am.cuda().eval(), gen, sr


def inputs(cfg, B, L):
    g = torch.Generator().manual_seed(1)
    ling = torch.stack([torch.randint(0, cfg[k], (B, L), generator=g) for k in ("sy", "tone", "syllable_flag", "word_segment")], -1)
    emo = torch.randint(0, cfg["emotion"], (B, L), generator=g)
    spk = torch.randint(0, cfg["speaker"], (B, L), generator=g)
    return [t.cuda() for t in (ling, emo, spk, torch.full((B,), L))]


def run_stream(am, gen, x, cs):
    """-> (ttfa s, per-chunk device ms, stream s, lengths in samples)"""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    st = K.stream_synthesize(am, gen, *x, chunk_steps=cs, allow_lookahead=True)       # (no-op for a causal generator)
    it = iter(st)
    next(it)
    torch.cuda.synchronize()
    ttfa = time.perf_counter() - t0
    events = [torch.cuda.Event(enable_timing=True)]
    events[0].record()
    for _ in it:
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        events.append(e)
    torch.cuda.synchronize()
    total = time.perf_counter() - t0
    chunk_ms = [a.elapsed_time(b) for a, b in zip(events, events[1:])]
    return ttfa, chunk_ms, total, st.lengths


def measure(am, gen, sr, B, cs, L, repeats):
    x = inputs(K.sambert_24k_config(), B, L)
    with torch.no_grad():
        run_stream(am, gen, x, cs)                                  # warm-up: plans, weight images, graph capture
        runs = [run_stream(am, gen, x, cs) for _ in range(repeats)]
        f = am.front_half(*x)
        n0 = ops.launch_count()
        steps = sum(1 for _ in am.mel_decoder.infer_steps(f["memory"], f["x_band_width"], f["x_band_width"]))
        dec_launches = (ops.launch_count() - n0) / steps
        K.synthesize(am, gen, *x)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(repeats):
            K.synthesize(am, gen, *x)
        torch.cuda.synchronize()
        synth = (time.perf_counter() - t0) / repeats
    ttfa = sorted(r[0] for r in runs)[len(runs) // 2]
    total = sorted(r[2] for r in runs)[len(runs) // 2]
    chunks = [c for r in runs for c in r[1]]
    audio_s = max(runs[0][3]) / sr
    return dict(B=B, chunk_steps=cs, frames_per_chunk=3 * cs, decoder_steps=steps, audio_s=round(audio_s, 3),
                ttfa_ms=round(1e3 * ttfa, 2), chunk_ms=round(sum(chunks) / max(1, len(chunks)), 3),
                chunk_ms_max=round(max(chunks, default=0.0), 3), stream_ms=round(1e3 * total, 1),
                rtf=round(audio_s / total, 2), dec_launches_per_step=dec_launches, synth_ms=round(1e3 * synth, 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--vocoder", choices=sorted(VOCODERS), default="causal_24k")
    ap.add_argument("--symbols", type=int, default=64)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the result as DIR/tts_stream_latency[_<vocoder>].json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tts_stream_latency: needs a CUDA device")
    info = card()
    am, gen, sr = models(args.vocoder)
    rows = []
    for B in (1, 8):
        for cs in (1, 4, 16):
            rows.append(measure(am, gen, sr, B, cs, args.symbols, args.repeats))
    lookahead = K.hifigan.StreamPlan(gen).delay
    result = dict(card=info, vocoder=args.vocoder, sample_rate=sr, lookahead_ms=round(1e3 * lookahead / sr, 1),
                  symbols=args.symbols, rows=rows)
    print(json.dumps(result), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        name = "tts_stream_latency" + ("" if args.vocoder == "causal_24k" else "_" + args.vocoder)
        with open(os.path.join(args.out, name + ".json"), "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
