"""Full-size per-layer parity sweep of the generator's layer shapes: tensor-core (default) and FFMA (exact) paths vs the CPU layer
oracle -- y, dx, dv, dg, db (development aid for the full-size train-step parity test)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from kantts_b200 import ops
from kantts_b200._lib import KT_ACT_LRELU, KT_ACT_TANH
from oracle import convref

torch.set_num_threads(32)
rel = lambda a, b: float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))
B = 16
# name: (spec kwargs, T_in, use_resid)
L = {
    "conv_pre 80->512 k7": (dict(c_in=80, c_out=512, kernel=7, pad_left=6), 32, False),
    "up0 T 512->256 k16 s8": (dict(c_in=512, c_out=256, kernel=16, stride=8, transposed=True, crop=8), 32, True),
    "rep0 512->256 k7 up8": (dict(c_in=512, c_out=256, kernel=7, pad_left=6, upsample=8), 32, False),
    "rb256 k3 d1": (dict(c_in=256, c_out=256, kernel=3, pad_left=2, act_in=0.1), 256, True),
    "rb256 k11 d5": (dict(c_in=256, c_out=256, kernel=11, dilation=5, pad_left=50, act_in=0.1), 256, True),
    "up1 T 256->128 k16 s8": (dict(c_in=256, c_out=128, kernel=16, stride=8, transposed=True, crop=8), 256, True),
    "rep1 256->128 k7 up8": (dict(c_in=256, c_out=128, kernel=7, pad_left=6, upsample=8), 256, False),
    "rb128 k7 d3": (dict(c_in=128, c_out=128, kernel=7, dilation=3, pad_left=18, act_in=0.1), 2048, True),
    "up2 T 128->64 k4 s2": (dict(c_in=128, c_out=64, kernel=4, stride=2, transposed=True, crop=2), 2048, True),
    "rep2 128->64 k7 up2": (dict(c_in=128, c_out=64, kernel=7, pad_left=6, upsample=2), 2048, False),
    "rb64 k11 d1": (dict(c_in=64, c_out=64, kernel=11, pad_left=10, act_in=0.1), 4096, True),
    "up3 T 64->32 k4 s2": (dict(c_in=64, c_out=32, kernel=4, stride=2, transposed=True, crop=2), 4096, True),
    "rep3 64->32 k7 up2": (dict(c_in=64, c_out=32, kernel=7, pad_left=6, upsample=2), 4096, False),
    "rb32 k3 d1": (dict(c_in=32, c_out=32, kernel=3, pad_left=2, act_in=0.1), 8192, True),
    "rb32 k11 d5": (dict(c_in=32, c_out=32, kernel=11, dilation=5, pad_left=50, act_in=0.1), 8192, True),
    "conv_post 32->1 k7 tanh": (dict(c_in=32, c_out=1, kernel=7, pad_left=6, act_in=0.01, act_out="tanh"), 8192, False),
}
D = {
    "msd0 1->128 k15": (dict(c_in=1, c_out=128, kernel=15, pad_left=7, act_out=0.1), 8192, False),
    "msd1 128->128 k41 s4 g4": (dict(c_in=128, c_out=128, kernel=41, stride=4, pad_left=20, groups=4, act_out=0.1), 8192, False),
    "msd2 128->256 k41 s4 g16": (dict(c_in=128, c_out=256, kernel=41, stride=4, pad_left=20, groups=16, act_out=0.1), 2048, False),
    "msd3 256->512 k41 s4 g16": (dict(c_in=256, c_out=512, kernel=41, stride=4, pad_left=20, groups=16, act_out=0.1), 512, False),
    "msd4 512->1024 k41 s4 g16": (dict(c_in=512, c_out=1024, kernel=41, stride=4, pad_left=20, groups=16, act_out=0.1), 128, False),
    "msd5 1024->1024 k41 g16": (dict(c_in=1024, c_out=1024, kernel=41, pad_left=20, groups=16, act_out=0.1), 32, False),
    "msd6 1024->1024 k5": (dict(c_in=1024, c_out=1024, kernel=5, pad_left=2, act_out=0.1), 32, False),
    "msd7 1024->1 k3": (dict(c_in=1024, c_out=1, kernel=3, pad_left=1), 32, False),
    "aux 2->1 k15": (dict(c_in=2, c_out=1, kernel=15, pad_left=7, act_out=0.1), 4098, False),
    "msd0 scale1 1->128 k15 T4098": (dict(c_in=1, c_out=128, kernel=15, pad_left=7, act_out=0.1), 4098, False),
    "msd1 scale1 k41 s4 g4 T4098": (dict(c_in=128, c_out=128, kernel=41, stride=4, pad_left=20, groups=4, act_out=0.1), 4098, False),
    "msd1 scale2 k41 s4 g4 T2051": (dict(c_in=128, c_out=128, kernel=41, stride=4, pad_left=20, groups=4, act_out=0.1), 2051, False),
}
import sys as _sys
if len(_sys.argv) > 1 and _sys.argv[1] == "msd":
    L = D
for name, (kw, T, use_resid) in L.items():
    kw = dict(kw)
    act_in, act_out = kw.pop("act_in", None), kw.pop("act_out", None)
    if name in D:
        kw["pad_right"] = kw["pad_left"]
    spec = ops.ConvSpec(**kw)
    if act_in is not None:
        spec.act_in, spec.act_in_slope = KT_ACT_LRELU, act_in
    if act_out == "tanh":
        spec.act_out = KT_ACT_TANH
    elif act_out is not None:
        spec.act_out, spec.act_out_slope = KT_ACT_LRELU, act_out
    g = torch.Generator().manual_seed(hash(name) % 1000)
    wshape = (spec.c_in, spec.c_out, spec.kernel) if spec.transposed else (spec.c_out, spec.c_in // spec.groups, spec.kernel)
    v = torch.randn(wshape, generator=g) / (wshape[1] * spec.kernel) ** 0.5
    gdim = (1, 2)
    wg = v.norm(2, dim=gdim, keepdim=True) * (1 + 0.1 * torch.randn(wshape[0], 1, 1, generator=g))
    b = 0.1 * torch.randn(spec.c_out, generator=g)
    x = torch.randn(B, spec.c_in, T, generator=g)
    t_out = spec.t_out(T)
    resid = torch.randn(B, spec.c_out, t_out, generator=g) if use_resid else None
    r = torch.randn(B, spec.c_out, t_out, generator=g)
    xo, vo, go, bo = (t.clone().requires_grad_(True) for t in (x, v, wg, b))
    w = go * vo / vo.norm(2, dim=gdim, keepdim=True)
    yo = convref.conv_layer(xo, w, bo, resid, stride=spec.stride, dilation=spec.dilation, pad_left=spec.pad_left,
                            pad_right=spec.pad_right if spec.stride > 1 or spec.groups > 1 or spec.c_out == 1 or spec.c_in <= 2 or "k5" in name else (spec.dilation * (spec.kernel - 1) - spec.pad_left if not spec.transposed else 0),
                            groups=spec.groups, transposed=spec.transposed, upsample=spec.upsample, crop=spec.crop, act_in=act_in, act_out=act_out)
    (yo * r).sum().backward()
    out = []
    for ffma in (False, True):
        ops.set_force_ffma(ffma)
        xg = x.permute(0, 2, 1).contiguous().cuda().requires_grad_(True)
        pv, pg, pb = (torch.nn.Parameter(t.clone().cuda()) for t in (v, wg, b))
        y = ops.conv(xg, spec, ops.PreparedWeight(), pv, pg, pb, None if resid is None else resid.permute(0, 2, 1).contiguous().cuda())
        (y * r.permute(0, 2, 1).contiguous().cuda()).sum().backward()
        torch.cuda.synchronize()
        out.append("%s y %.1e dx %.1e dv %.1e dg %.1e db %.1e" % ("FFMA" if ffma else "TC  ", rel(y.detach().cpu().permute(0, 2, 1), yo.detach()),
                   rel(xg.grad.cpu().permute(0, 2, 1), xo.grad), rel(pv.grad.cpu(), vo.grad), rel(pg.grad.cpu(), go.grad), rel(pb.grad.cpu(), bo.grad)))
    ops.set_force_ffma(False)
    print(f"{name:26s} | " + " | ".join(out), flush=True)
