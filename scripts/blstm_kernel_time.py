"""Kernel time of the pitch / energy predictors' BiLSTM in inference: kt_blstm_ragged against cuDNN's packed nn.LSTM
(pack_padded_sequence -> nn.LSTM(bidirectional=True) -> pad_packed_sequence) on the same tensors, from torch.profiler's CUDA
activities.  sambert_24k.yaml's predictor (256 memory units, 128 LSTM units), seeded weights, a ragged batch of B sequences
of 16..L symbols.  The input projection (one k = 1 conv of 8H channels for the kernel, inside cuDNN's LSTM for the other) is
counted with each.  Prints the card and its power limit, read in the same run, and one JSON line.

    python scripts/blstm_kernel_time.py [--batch 8] [--length 96] [--iters 50] [--out DIR]"""
import argparse
import json
import os
import sys

import torch
import torch.nn as nn
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import kantts_b200 as K  # noqa: E402
from tts_stream_latency import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--length", type=int, default=96)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = "cuda"
    cfg = K.sambert_24k_config()
    torch.manual_seed(0)
    units, H = cfg["predictor_num_memory_units"], cfg["predictor_lstm_units"]
    pred = K.sambert.VarFsmnRnnNARPredictor(units, cfg["predictor_filter_size"], 1, units, 16, 0.0, 0, H).to(dev).eval()
    g = torch.Generator().manual_seed(1)
    B, L = a.batch, a.length
    lens = torch.randint(16, L + 1, (B,), generator=g)
    lens[0] = L
    x = torch.randn(B, L, units, generator=g).to(dev)
    masks = (torch.arange(L)[None, :] >= lens[:, None]).to(dev)

    def ours():
        return pred.blstm_infer(x, masks)

    def cudnn():
        packed = nn.utils.rnn.pack_padded_sequence(x, lens, batch_first=True, enforce_sorted=False)
        return nn.utils.rnn.pad_packed_sequence(pred.blstm(packed)[0], batch_first=True, total_length=L)[0]

    res = {"card": card(), "batch": B, "length": L, "hidden": H, "lengths": lens.tolist()}
    with torch.no_grad():
        err = float((ours() - cudnn()).abs().max())
        for name, fn in (("kt_blstm_ragged", ours), ("cudnn_packed", cudnn)):
            for _ in range(5):
                fn()
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(a.iters):
                    fn()
                torch.cuda.synchronize()
            kernels = {}
            for e in prof.key_averages():
                if e.device_type.name == "CUDA" and e.device_time_total > 0:
                    kernels[e.key] = e.device_time_total / a.iters
            res[name] = {"us_per_call": sum(kernels.values()), "kernels_us": kernels}
    res["max_abs_diff"] = err
    print(res["card"])
    for name in ("kt_blstm_ragged", "cudnn_packed"):
        print(f"{name}: {res[name]['us_per_call']:.1f} us of kernel time per call")
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "blstm_kernel_time.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
