"""Per-layer timing breakdown of one C2 train step (development aid, not a bench number)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bench
import kantts_b200 as K
from kantts_b200 import ops

dev = torch.device("cuda", 0)
torch.manual_seed(1234)
model, opt, sched = K.hifigan_model_builder(bench.CONFIG, dev)
crit = K.criterion_builder(bench.CONFIG, dev)
step = K.GanStep(model, opt, sched, crit, bench.CONFIG)
y, x = bench.synth_batch(bench.B_PER_GPU, 1234)
y, x = y.to(dev), x.to(dev)
for _ in range(2):
    step.step((y, x))
torch.cuda.synchronize()
from kantts_b200 import hifigan
hifigan._PARALLEL_STREAMS, ops._WGRAD_ASYNC = False, False     # serialise: an event pair must bracket only its own kernels
step.step((y, x))
torch.cuda.synchronize()
prof = ops.set_profiler(True)
step.step((y, x))
by = prof.by_layer()
ops.set_profiler(False)
tot = sum(v[1] for v in by.values())
print(f"instrumented total {tot:.2f} ms")
classes = {}
for (name, _), (calls, ms, flops) in by.items():
    c = classes.setdefault(name, [0, 0.0, 0.0])
    c[0] += calls; c[1] += ms; c[2] += flops
for name, (calls, ms, flops) in sorted(classes.items(), key=lambda kv: -kv[1][1]):
    print(f"class {name:16s} {ms:8.3f} ms {100*ms/tot:5.1f}% x{calls:4d} {flops/ms/1e9 if ms else 0:7.1f} TF/s")
for (name, det), (calls, ms, flops) in sorted(by.items(), key=lambda kv: -kv[1][1])[:140]:
    print(f"{ms:8.3f} ms {100*ms/tot:5.1f}% x{calls:3d} {flops/ms/1e9 if ms else 0:7.1f} TF/s  {name:16s} {det}")
