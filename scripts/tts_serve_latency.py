"""Continuous batching (infer.TtsServer) against lockstep batches (infer.stream_synthesize) on the GPU.

SAM-BERT with the sambert_24k.yaml network (seeded weights, about DUR frames per symbol) and the hifigan_v1_24k.yaml
generator, or with ``--vocoder noncausal_16k`` the non-causal hifigan_noncausal_v1_16k.yaml generator (hop 200 at 16 kHz,
served and streamed with ``allow_lookahead=True``: every request's audio waits for 214 ms of look-ahead), or with
``--vocoder multiband_24k`` the causal multi-band generator of scripts/multiband_step.py with its PQMF (hop 240 at 24 kHz,
1.3 ms of look-ahead: the synthesis's 31 samples).  N requests of
16..96 symbols arrive at seeded Poisson times (mean gap --gap ms).  Both servers run on one host thread and deliver
each chunk's audio to the host (a synchronize after each chunk):
  serve     TtsServer with B slots: requests are submitted when their arrival time has passed, one step() per chunk
  lockstep  whenever the previous batch has finished, the arrived requests (up to B) go through stream_synthesize as one batch
Per server: time to first audio per request (arrival -> the first chunk holding its audio, p50 / p95, ms) and aggregate
audio seconds per wall second (all requests' audio / time from the first arrival to the last audio).  Also the admission
cost: front_half of B requests one by one (as TtsServer admits them) against one padded batch.  Prints the card and
its power limit, read in the same run, and the result as one JSON line.

    python scripts/tts_serve_latency.py [--vocoder causal_24k|noncausal_16k|multiband_24k] [--requests 32] [--slots 8] [--chunk-steps 4]
                                        [--gap 150] [--out DIR]"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import kantts_b200 as K  # noqa: E402
from tts_stream_latency import VOCODERS, card, models  # noqa: E402


def requests(n, gap_ms, seed=1):
    cfg = K.sambert_24k_config()
    g = torch.Generator().manual_seed(seed)
    rng = np.random.default_rng(seed)
    arrive = np.cumsum(rng.exponential(gap_ms / 1e3, n))
    arrive -= arrive[0]
    out = []
    for i in range(n):
        L = int(rng.integers(16, 97))
        ling = torch.stack([torch.randint(0, cfg[k], (L,), generator=g) for k in ("sy", "tone", "syllable_flag", "word_segment")], -1)
        out.append(dict(arrive=float(arrive[i]), inputs=(ling, torch.randint(0, cfg["emotion"], (L,), generator=g),
                                                         torch.randint(0, cfg["speaker"], (L,), generator=g), L)))
    return out


def run_serve(am, gen, reqs, slots, cs):
    """-> (ttfa per request in s, audio samples, wall s)"""
    server = K.TtsServer(am, gen, slots=slots, chunk_steps=cs, max_steps=256, allow_lookahead=True)   # (no-op for a causal one)
    first, ids, samples, nxt = {}, {}, 0, 0
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    while nxt < len(reqs) or not server.idle:
        now = time.perf_counter() - t0
        while nxt < len(reqs) and reqs[nxt]["arrive"] <= now:
            ids[server.submit(*reqs[nxt]["inputs"])] = nxt
            nxt += 1
        if server.idle:
            time.sleep(max(0.0, reqs[nxt]["arrive"] - now))
            continue
        audio, _ = server.step()
        torch.cuda.synchronize()
        now = time.perf_counter() - t0
        for rid, _, w in audio:
            i = ids[rid]
            first.setdefault(i, now - reqs[i]["arrive"])
            samples += w.shape[0]
    return [first[i] for i in range(len(reqs))], samples, time.perf_counter() - t0


def run_lockstep(am, gen, reqs, slots, cs):
    first, samples, nxt = {}, 0, 0
    dev = next(am.parameters()).device
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    while nxt < len(reqs):
        now = time.perf_counter() - t0
        if reqs[nxt]["arrive"] > now:
            time.sleep(reqs[nxt]["arrive"] - now)
            now = time.perf_counter() - t0
        batch = [i for i in range(nxt, min(len(reqs), nxt + slots)) if reqs[i]["arrive"] <= now]
        nxt = batch[-1] + 1
        L = max(reqs[i]["inputs"][3] for i in batch)
        pad = lambda t: torch.nn.functional.pad(t, (0, 0, 0, L - t.shape[0]) if t.dim() == 2 else (0, L - t.shape[0]))
        x = [torch.stack([pad(reqs[i]["inputs"][k]) for i in batch]).to(dev) for k in range(3)]
        x.append(torch.tensor([reqs[i]["inputs"][3] for i in batch], device=dev))
        st = K.stream_synthesize(am, gen, *x, chunk_steps=cs, allow_lookahead=True)
        for start, w in st:
            torch.cuda.synchronize()
            now = time.perf_counter() - t0
            for j, i in enumerate(batch):
                if start < st.lengths[j]:
                    first.setdefault(i, now - reqs[i]["arrive"])
        samples += sum(st.lengths)
    return [first[i] for i in range(len(reqs))], samples, time.perf_counter() - t0


def front_half_cost(am, reqs, repeats=5):
    """-> (ms for front_half of every request on its own, as TtsServer admits them, ms for one padded batch of them): the
    median over ``repeats``, host clock to a synchronize."""
    dev = next(am.parameters()).device
    L = max(r["inputs"][3] for r in reqs)
    pad = lambda t: torch.nn.functional.pad(t, (0, 0, 0, L - t.shape[0]) if t.dim() == 2 else (0, L - t.shape[0]))
    one = [[r["inputs"][k][None].to(dev) for k in range(3)] + [torch.tensor([r["inputs"][3]], device=dev)] for r in reqs]
    batch = [torch.stack([pad(r["inputs"][k]) for r in reqs]).to(dev) for k in range(3)]
    batch.append(torch.tensor([r["inputs"][3] for r in reqs], device=dev))

    def clock(fn):
        times = []
        for _ in range(repeats + 1):                                  # the first run warms up
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t0)
        return round(1e3 * sorted(times[1:])[repeats // 2], 2)
    return clock(lambda: [am.front_half(*x) for x in one]), clock(lambda: am.front_half(*batch))


def summary(name, sr, ttfa, samples, wall):
    ms = np.array(ttfa) * 1e3
    return dict(server=name, ttfa_p50_ms=round(float(np.percentile(ms, 50)), 1),
                ttfa_p95_ms=round(float(np.percentile(ms, 95)), 1), audio_s=round(samples / sr, 2), wall_s=round(wall, 2),
                audio_s_per_wall_s=round(samples / sr / wall, 2))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--vocoder", choices=sorted(VOCODERS), default="causal_24k")
    ap.add_argument("--requests", type=int, default=32)
    ap.add_argument("--slots", type=int, default=8)
    ap.add_argument("--chunk-steps", type=int, default=4)
    ap.add_argument("--gap", type=float, default=150.0, help="mean gap between arrivals, ms")
    ap.add_argument("--out", default=None, help="also write the result as DIR/tts_serve_latency[_<vocoder>].json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tts_serve_latency: needs a CUDA device")
    info = card()
    am, gen, sr = models(args.vocoder)
    reqs = requests(args.requests, args.gap)
    with torch.no_grad():
        warm = requests(args.slots, 0.0, seed=2)                     # plans, weight images, graph captures
        run_serve(am, gen, warm, args.slots, args.chunk_steps)
        run_lockstep(am, gen, warm, args.slots, args.chunk_steps)
        rows = [summary("serve", sr, *run_serve(am, gen, reqs, args.slots, args.chunk_steps)),
                summary("lockstep", sr, *run_lockstep(am, gen, reqs, args.slots, args.chunk_steps))]
        alone, batched = front_half_cost(am, reqs[:args.slots])
    result = dict(card=info, vocoder=args.vocoder, lookahead_ms=round(1e3 * K.hifigan.StreamPlan(gen).delay / sr, 1),
                  requests=args.requests, slots=args.slots, chunk_steps=args.chunk_steps, mean_gap_ms=args.gap,
                  rows=rows, front_half_ms=dict(requests=args.slots, one_by_one=alone, one_batch=batched))
    print(json.dumps(result), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        name = "tts_serve_latency" + ("" if args.vocoder == "causal_24k" else "_" + args.vocoder)
        with open(os.path.join(args.out, name + ".json"), "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
