"""Per-chunk latency of streaming synthesis (Generator.streamer) on the GPU.

For the class-default generator (hop 256 at 22.05 kHz) and the hifigan_v1_24k.yaml generator (hop 240 at 24 kHz), over
B in {1, 16, 64} slots x F in {1, 4, 16} frames per chunk: the device time per graph-replayed chunk (CUDA events over
--chunks chunks after warm-up), the host time to enqueue one push, the library launches per chunk, the real-time factor
(audio seconds per chunk / chunk time; > 1 is faster than real time), and for comparison the whole-utterance forward of
the same frames.  Prints the card and its power limit, read in the same run.

--config noncausal: the same over the non-causal hifigan_noncausal_v1_16k.yaml generator (hop 200 at 16 kHz), streamed
with per-slot lengths long enough that no utterance ends during the run; its rows also give the stream's look-ahead
(delay_ms: the audio a sample waits for) on top of the chunk's own audio.

--config nsf / nsf_noncausal: the NSF generators hifigan_v1_nsf_24k.yaml (causal, hop 240 at 24 kHz) and
hifigan_noncausal_nsf_v1_16k.yaml (hop 200 at 16 kHz), streamed with per-slot seeds; each chunk carries f0 and the voiced
flag after the mel, and the whole-utterance forward takes the same seeds.

--config multiband: the multi-band generator of scripts/multiband_step.py (G_MB: 4 sub-bands at 6 kHz, upsample_scales
[5, 3, 2, 2], 512 channels) with its PQMF synthesis as the last stream stage (hop 240 at 24 kHz; the synthesis's 31 samples
of look-ahead: per-slot lengths, one drain frame), next to the full-band v1_24k generator (hop 240 at 24 kHz).  The
whole-utterance forward of the multi-band generator includes PQMF.synthesis.

--runs N repeats the config's generators N times, alternating them, so that the spread between runs of one generator can
be set against the difference between generators.

    python scripts/stream_latency.py [--config causal|noncausal|nsf|nsf_noncausal|multiband] [--chunks 200] [--runs 1]
                                     [--out DIR]"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import kantts_b200 as K  # noqa: E402

GENERATORS = {
    "causal": {
        "default_22k": (dict(), 22050),
        "v1_24k": (dict(upsample_scales=[8, 5, 3, 2], upsample_kernal_sizes=[16, 10, 6, 4]), 24000),
    },
    "noncausal": {
        "noncausal_v1_16k": (dict(channels=256, upsample_scales=[10, 5, 2, 2], upsample_kernal_sizes=[20, 11, 4, 4],
                                  resblock_dilations=[[1, 3, 5, 7]] * 3, causal=False), 16000),
    },
    "nsf": {
        "v1_nsf_24k": (dict(upsample_scales=[8, 5, 3, 2], upsample_kernal_sizes=[16, 10, 6, 4],
                            nsf_params=dict(nb_harmonics=7, sampling_rate=24000)), 24000),
    },
    "multiband": {
        "v1_24k": (dict(upsample_scales=[8, 5, 3, 2], upsample_kernal_sizes=[16, 10, 6, 4]), 24000),
        "multiband_24k": (dict(out_channels=4, upsample_scales=[5, 3, 2, 2], upsample_kernal_sizes=[10, 6, 4, 4]), 24000),
    },
    "nsf_noncausal": {
        "noncausal_nsf_v1_16k": (dict(channels=256, upsample_scales=[10, 5, 2, 2], upsample_kernal_sizes=[20, 11, 4, 4],
                                      resblock_dilations=[[1, 3, 5, 7]] * 3, causal=False,
                                      nsf_params=dict(nb_harmonics=7, sampling_rate=16000)), 16000),
    },
}


def frames_input(gen, B, F):
    """(B, in_channels, F) on the device: a random mel, and for an NSF generator f0 in [80, 300) Hz and a voiced flag."""
    mel = torch.randn(B, 80, F, device="cuda")
    if not gen.nsf_enable:
        return mel
    f0 = 80 + 220 * torch.rand(B, 1, F, device="cuda")
    return torch.cat([mel, f0, (torch.rand(B, 1, F, device="cuda") > 0.3).float()], 1)
# the whole-utterance forward keeps every activation of the utterance: longer ones are timed at this many frames
WHOLE_MAX_ROWS = 64 * 256


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def measure(gen, sr, B, F, chunks):
    # a generator streamed with a look-ahead (non-causal, or multi-band) takes lengths that outlast the run
    lengths = [1 << 24] * B if K.hifigan.StreamPlan(gen).delay else None
    seeds = list(range(B)) if gen.nsf_enable else None
    st = gen.streamer(batch=B, max_frames=F, lengths=lengths, seeds=seeds)
    mel = frames_input(gen, B, F)
    for _ in range(10):                                  # the first push captures the graph
        st.push(mel)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    host = 0.0
    e0.record()
    for _ in range(chunks):
        t0 = time.perf_counter()
        st.push(mel)
        host += time.perf_counter() - t0
    e1.record()
    torch.cuda.synchronize()
    chunk_ms = e0.elapsed_time(e1) / chunks
    # whole-utterance forward of the same frames (capped, see WHOLE_MAX_ROWS)
    frames = min(chunks * F, max(F, WHOLE_MAX_ROWS // B))
    whole = frames_input(gen, B, frames)
    kw = dict(nsf_seeds=seeds) if seeds else {}
    forward = (lambda: gen.pqmf.synthesis(gen(whole))) if gen.out_channels > 1 else (lambda: gen(whole, **kw))
    with torch.no_grad():
        forward()
        torch.cuda.synchronize()
        w0, w1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        w0.record()
        for _ in range(3):
            forward()
        w1.record()
        torch.cuda.synchronize()
    whole_ms = w0.elapsed_time(w1) / 3
    audio_s = F * st.hop / sr
    return dict(B=B, F=F, chunk_ms=round(chunk_ms, 4), host_enqueue_ms=round(1e3 * host / chunks, 4),
                launches_per_chunk=st.plan.launches_per_chunk, rtf=round(audio_s / (chunk_ms / 1e3), 2),
                latency_audio_ms=round(1e3 * audio_s, 2), whole_frames=frames, whole_ms=round(whole_ms, 3),
                whole_rtf=round(frames * st.hop / sr / (whole_ms / 1e3), 2), delay_ms=round(1e3 * st.delay / sr, 2))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", choices=sorted(GENERATORS), default="causal")
    ap.add_argument("--chunks", type=int, default=200)
    ap.add_argument("--runs", type=int, default=1, help="measure the config's generators this many times, alternating")
    ap.add_argument("--out", default=None, help="also write the rows as DIR/stream_latency.json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("stream_latency: needs a CUDA device")
    info = card()
    print(f"card: {info}")
    rows, gens = [], {}
    for name, (cfg, sr) in GENERATORS[args.config].items():
        torch.manual_seed(0)
        gens[name] = K.Generator(**cfg).cuda().eval()
        if gens[name].out_channels > 1:
            gens[name].pqmf = K.PQMF(gens[name].out_channels).cuda()
    for run in range(args.runs):
        for name, (cfg, sr) in GENERATORS[args.config].items():
            for B in (1, 16, 64):
                for F in (1, 4, 16):
                    r = dict(generator=name, **measure(gens[name], sr, B, F, args.chunks))
                    if args.runs > 1:
                        r["run"] = run
                    rows.append(r)
                    print(json.dumps(r), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        suffix = "" if args.config == "causal" else "_" + args.config
        with open(os.path.join(args.out, f"stream_latency{suffix}.json"), "w") as f:
            json.dump(dict(card=info, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
