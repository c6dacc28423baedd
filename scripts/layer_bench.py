"""Micro-benchmark of single conv layers through the C ABI (development aid; also the ncu target for the heavy
MultiPeriodDiscriminator layers).  python scripts/layer_bench.py [--iters 20] [--only NAME]"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from kantts_b200 import ops  # noqa: E402
from kantts_b200._lib import KT_ACT_LRELU  # noqa: E402

# name: (ConvSpec kwargs, B, T_in, period)
LAYERS = {
    "mpd_1024_1024_k5_p3": (dict(c_in=1024, c_out=1024, kernel=5, pad_left=2, pad_right=2), 16, 34, 3),
    "mpd_1024_1024_k5_p11": (dict(c_in=1024, c_out=1024, kernel=5, pad_left=2, pad_right=2), 16, 10, 11),
    "mpd_512_1024_k5s3_p3": (dict(c_in=512, c_out=1024, kernel=5, stride=3, pad_left=2, pad_right=2), 16, 102, 3),
    "mpd_128_512_k5s3_p5": (dict(c_in=128, c_out=512, kernel=5, stride=3, pad_left=2, pad_right=2), 16, 547, 5),
    "msd_1024_1024_k5": (dict(c_in=1024, c_out=1024, kernel=5, pad_left=2, pad_right=2), 16, 33, 0),
    # scale discriminator at its shorter scales and pair batch (32 items): packed M tiles, several items per tile
    "msd_1024_1024_k5_t17": (dict(c_in=1024, c_out=1024, kernel=5, pad_left=2, pad_right=2), 32, 17, 0),
    "msd_1024_1024_k5_t9": (dict(c_in=1024, c_out=1024, kernel=5, pad_left=2, pad_right=2), 32, 9, 0),
    "msd_1024_1024_k41_g16_t33": (dict(c_in=1024, c_out=1024, kernel=41, groups=16, pad_left=20, pad_right=20), 32, 33, 0),
    "msd_1024_1024_k41_g16_t17": (dict(c_in=1024, c_out=1024, kernel=41, groups=16, pad_left=20, pad_right=20), 32, 17, 0),
    "msd_1024_1024_k41_g16_t9": (dict(c_in=1024, c_out=1024, kernel=41, groups=16, pad_left=20, pad_right=20), 32, 9, 0),
    "msd_512_1024_k41_g16_s4_t9": (dict(c_in=512, c_out=1024, kernel=41, stride=4, groups=16, pad_left=20, pad_right=20),
                                   32, 33, 0),
    "msd_512_1024_k41_g16_s4_t32": (dict(c_in=512, c_out=1024, kernel=41, stride=4, groups=16, pad_left=20, pad_right=20),
                                    16, 128, 0),
    "msd_256_512_k41_g16_s4_t128": (dict(c_in=256, c_out=512, kernel=41, stride=4, groups=16, pad_left=20, pad_right=20),
                                    16, 512, 0),
    "gen_conv_pre_80_512_k7": (dict(c_in=80, c_out=512, kernel=7, pad_left=3, pad_right=3), 16, 32, 0),
    "gen_128_128_k11": (dict(c_in=128, c_out=128, kernel=11, pad_left=10, pad_right=0), 16, 2048, 0),
    "gen_32_32_k7": (dict(c_in=32, c_out=32, kernel=7, pad_left=6, pad_right=0), 16, 8192, 0),
    # one shape per MMA tile width N: 16 (single-channel output; the data gradient of a 1-channel input layer),
    # 32 / 64 (generator stages 4 / 3), 64 (N split of a 256-channel layer with 32 M tiles; grouped k41), 128 (above)
    "msd_post_1024_1_k3": (dict(c_in=1024, c_out=1, kernel=3, pad_left=1, pad_right=1), 16, 33, 0),
    "msd_pre_1_128_k15": (dict(c_in=1, c_out=128, kernel=15, pad_left=7, pad_right=7), 16, 8192, 0),
    "gen_64_64_k7": (dict(c_in=64, c_out=64, kernel=7, pad_left=6, pad_right=0), 16, 4096, 0),
    "gen_256_256_k11": (dict(c_in=256, c_out=256, kernel=11, pad_left=10, pad_right=0), 16, 256, 0),
    "msd_128_128_k41_g4_s4": (dict(c_in=128, c_out=128, kernel=41, stride=4, groups=4, pad_left=20, pad_right=20), 16, 8192, 0),
    "sambert_ffn_128_1024_k3": (dict(c_in=128, c_out=1024, kernel=3, pad_left=1, pad_right=1), 32, 256, 0),
    "sambert_ffn_1024_128_k1": (dict(c_in=1024, c_out=128, kernel=1), 32, 256, 0),
}


def run(name, iters):
    kw, B, T, period = LAYERS[name]
    spec = ops.ConvSpec(**kw)
    spec.act_out, spec.act_out_slope = KT_ACT_LRELU, 0.1
    g = torch.Generator().manual_seed(1)
    wshape = (spec.c_out, spec.c_in // spec.groups, spec.kernel)
    v = torch.nn.Parameter((torch.randn(wshape, generator=g) * 0.05).cuda())
    gg = torch.nn.Parameter(v.detach().norm(2, dim=(1, 2), keepdim=True).clone())
    bias = torch.zeros(spec.c_out, device="cuda", requires_grad=True)
    xs = (B, T, period, spec.c_in) if period else (B, T, spec.c_in)
    x = torch.randn(xs, generator=g).cuda().requires_grad_(True)
    cache = ops.PreparedWeight()
    y = ops.conv(x, spec, cache, v, gg, bias)
    r = torch.randn(y.shape, device="cuda")
    for _ in range(3):
        y = ops.conv(x, spec, cache, v, gg, bias)
        y.backward(r)
    torch.cuda.synchronize()
    prof = ops.set_profiler(True)
    for _ in range(iters):
        y = ops.conv(x, spec, cache, v, gg, bias)
        y.backward(r)
    by = prof.by_layer()
    ops.set_profiler(False)
    for (kind, det), (calls, ms, flops) in sorted(by.items()):
        print(f"{name:26s} {kind:16s} {ms / calls * 1e3:9.1f} us  {flops / ms / 1e9 if ms else 0:7.1f} TF/s  {det}")


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--only", default=None)
    a = ap.parse_args()
    only = None if a.only is None else a.only.split(",")
    for n in LAYERS:
        if only is None or n in only:
            run(n, a.iters)
