"""torch.autograd.Function wrappers over the C ABI (include/kantts_b200.h).

Internal activation layout: channels-last rows, ``(B, T, C)`` contiguous fp32 (``(B, T, p, C)``
for the period discriminator).  The nn.Modules in hifigan.py convert at their boundary only.
Backward functions run on the autograd engine thread; every call passes the thread's current
stream explicitly and the library keeps no global state.
"""
import ctypes
from dataclasses import dataclass, field, replace

import torch

from . import _lib
from ._lib import (KT_ACT_LRELU, KT_ACT_NONE, KT_ACT_TANH, KT_PATH_AUTO, KT_PATH_BF16, KT_PATH_FFMA, KT_PATH_TC, KT_PLAN_STREAM,
                   KtConv1dDesc,
                   KtMelDesc, KtResblockDesc, KtStreamMask, check, ptr, stream_ptr)

_launches = 0          # kernels-launched counter (bench.py reports it as gpu_launches)


def launch_count():
    return _launches


def _count(n=1):
    global _launches
    _launches += n


def call(fn, *args, launches=1):
    """Call entry point ``fn`` of the library with ``args`` and the calling thread's current stream (every launching entry
    point takes its stream last), raise on a failed return code, and count ``launches`` kernel launches.  Eager steps make
    thousands of these calls from the host, so the success path makes no further Python call."""
    global _launches
    rc = getattr(_lib.load(), fn)(*args, stream_ptr())
    if rc:
        check(rc, fn)
    _launches += launches


class _Profiler:
    """Optional per-call CUDA-event timing (bench.py's roofline leg): each instrumented library call
    is bracketed by two events on the launching stream and tagged with its algorithmic work."""

    def __init__(self):
        self.records = []
        self.details = []

    def by_layer(self):
        """{(kernel class, layer signature): [calls, ms, flops]} -- development breakdown."""
        torch.cuda.synchronize()
        out = {}
        for (name, e0, e1, flops, _), det in zip(self.records, self.details):
            d = out.setdefault((name, det), [0, 0.0, 0.0])
            d[0] += 1
            d[1] += e0.elapsed_time(e1)
            d[2] += flops
        return out

    def summary(self):
        torch.cuda.synchronize()
        out = {}
        for name, e0, e1, flops, nbytes in self.records:
            d = out.setdefault(name, {"calls": 0, "ms": 0.0, "flops": 0.0, "bytes": 0.0})
            d["calls"] += 1
            d["ms"] += e0.elapsed_time(e1)
            d["flops"] += flops
            d["bytes"] += nbytes
        return out


_profiler = None


def set_profiler(enabled):
    """-> the active _Profiler (or None).  Timing adds host overhead: never on during a timed run."""
    global _profiler
    _profiler = _Profiler() if enabled else None
    return _profiler


def _sig(spec, d):
    return (f"{spec.c_in}->{spec.c_out} k{spec.kernel} s{spec.stride} d{spec.dilation} g{spec.groups}"
            f"{' T' if spec.transposed else ''}{f' up{spec.upsample}' if spec.upsample > 1 else ''}"
            f" B{d.batch}x{d.nsub} t{d.t_in}")


def _run(name, spec, d, launches, tc, *calls):
    """Make the library calls ``(entry point, *args)`` through ``call`` as one unit of kernel class ``name``: timed by the
    profiler (when on) against the work of layer ``spec`` at descriptor ``d``, and counted as ``launches`` kernel
    launches, ``tc`` of them on the tensor cores."""
    global _tc_launches
    if _profiler is not None:
        e0 = torch.cuda.Event(enable_timing=True)
        e0.record()
    for fn, *args in calls:
        call(fn, *args, launches=0)
    if _profiler is not None:
        e1 = torch.cuda.Event(enable_timing=True)
        e1.record()
        _profiler.records.append((name, e0, e1, *_conv_work(spec, d)))
        _profiler.details.append(_sig(spec, d))
    _count(launches)
    _tc_launches += tc


def _conv_work(spec, d):
    """(algorithmic FLOPs, layer-boundary HBM bytes) of one pass over the layer (SURVEY.md 8d)."""
    rows_out = d.batch * d.nsub * d.t_out
    rows_in = d.batch * d.nsub * d.t_in
    if spec.transposed:
        macs = rows_in * spec.kernel * spec.c_in * spec.c_out
    else:
        macs = rows_out * spec.kernel * (spec.c_in // spec.groups) * spec.c_out
    nbytes = 4.0 * (rows_in * spec.c_in + rows_out * spec.c_out + spec.w_numel)
    return 2.0 * macs, nbytes


@dataclass
class ConvSpec:
    """Static description of one conv layer (forward semantics), see KtConv1dDesc.  ``path`` KT_PATH_BF16 runs the layer's
    tensor-core passes in single-pass bf16 (hifigan.set_precision sets it for a whole model)."""
    c_in: int
    c_out: int
    kernel: int
    stride: int = 1
    dilation: int = 1
    pad_left: int = 0
    pad_right: int = 0          # only used to derive t_out
    groups: int = 1
    transposed: bool = False
    upsample: int = 1
    crop: int = 0               # transposed: samples cropped from the end (causal variant, layers.py:161)
    act_in: int = KT_ACT_NONE
    act_in_slope: float = 0.0
    act_out: int = KT_ACT_NONE
    act_out_slope: float = 0.0
    path: int = KT_PATH_AUTO
    _plans: dict = field(default_factory=dict, init=False, repr=False, compare=False)
    _rb_cache: dict = field(default_factory=dict, init=False, repr=False, compare=False)

    def t_out(self, t_in):
        if self.transposed:
            return (t_in - 1) * self.stride - 2 * self.pad_left + self.dilation * (self.kernel - 1) + 1 - self.crop
        t = t_in * self.upsample
        return (t + self.pad_left + self.pad_right - self.dilation * (self.kernel - 1) - 1) // self.stride + 1

    def plan(self, batch, nsub, t_in, stream=False):
        """-> the ConvPlan of this layer for one input shape, cached per shape, exact-path flag (the tests toggle
        set_force_ffma at run time), stream flag (the forward of a stream chunk, see stream_conv) and compute path (the
        precision a model is switched to).  Every other field of the spec must be set before its first plan."""
        key = (batch, nsub, t_in, _exact(self), stream, self.path)
        p = self._plans.get(key)
        if p is None:
            p = self._plans[key] = ConvPlan(self, batch, nsub, t_in, key[3], stream)
        return p

    def desc(self, batch, nsub, t_in):
        """-> a new KtConv1dDesc of this layer for one input shape (the plan keeps the one the layer runs with)."""
        return KtConv1dDesc(batch=batch, nsub=nsub, t_in=t_in, t_out=self.t_out(t_in), c_in=self.c_in, c_out=self.c_out,
                            groups=self.groups, kernel=self.kernel, stride=self.stride, dilation=self.dilation,
                            pad_left=self.pad_left, transposed=int(self.transposed), upsample=self.upsample,
                            act_in=self.act_in, act_in_slope=self.act_in_slope, act_out=self.act_out,
                            act_out_slope=self.act_out_slope, path=self.path)

    @property
    def w_numel(self):
        return self.kernel * (self.c_in // self.groups) * self.c_out


class ConvPlan:
    """Which kernel runs each pass of one conv layer for one input shape.  An N tile or workspace of 0 means the
    exact-fp32 (FFMA) kernel.
      d                        the layer's descriptor
      nt_fwd                   forward N tile
      d_bwd, nt_bwd, up_bwd    data gradient: descriptor, N tile, and whether it runs over the up-sampled rows
      ws_fwd, ws_bwd           tensor-core forward / data-gradient workspace (operand planes of the TMA-fed route), in floats
      wg_ws                    tensor-core weight-gradient workspace, in floats
    A stream plan (stream=True) plans the forward of a stream chunk only: the register-staged route, no workspace."""

    __slots__ = ("spec", "d", "nt_fwd", "d_bwd", "nt_bwd", "up_bwd", "ws_fwd", "ws_bwd", "wg_ws")

    def __init__(self, spec, batch, nsub, t_in, exact, stream=False):
        self.spec = spec
        self.d = self.d_bwd = d = spec.desc(batch, nsub, t_in)
        self.nt_fwd = self.nt_bwd = self.ws_fwd = self.ws_bwd = self.wg_ws = 0
        self.up_bwd = False
        if exact:
            return
        lib = _lib.load()
        if stream:
            self.nt_fwd = lib.kt_conv1d_tc_plan(ctypes.byref(d), KT_PLAN_STREAM)
            return
        self.nt_fwd = lib.kt_conv1d_tc_plan(ctypes.byref(d), 0)
        self.nt_bwd = lib.kt_conv1d_tc_plan(ctypes.byref(d), 1)
        if (not self.nt_bwd and spec.path in (KT_PATH_AUTO, KT_PATH_BF16) and spec.upsample > 1 and spec.c_in % 4 == 0
                and not spec.transposed):
            # the nearest-upsampled conv has no tensor-core data gradient of its own: run the same conv over the
            # up-sampled rows (upsample = 1, no fused pre-activation) and fold it back with kt_upsample_grad_reduce
            d2 = replace(spec, upsample=1, act_in=KT_ACT_NONE, act_in_slope=0.0).desc(batch, nsub, t_in * spec.upsample)
            nt2 = lib.kt_conv1d_tc_plan(ctypes.byref(d2), 1)
            if nt2:
                self.d_bwd, self.nt_bwd, self.up_bwd = d2, nt2, True
        if self.nt_fwd:
            self.ws_fwd = int(lib.kt_conv1d_tc_workspace(ctypes.byref(d), 0))
        if self.nt_bwd:
            self.ws_bwd = int(lib.kt_conv1d_tc_workspace(ctypes.byref(self.d_bwd), 1))
        self.wg_ws = int(lib.kt_conv1d_bwd_weight_tc_workspace(ctypes.byref(d)))

    def tile(self, direction):
        """N tile of direction 0 (forward) or 1 (data gradient), for a pass that runs: a KT_PATH_TC layer raises here
        when the tensor cores cannot run it (unless set_force_ffma put every layer on the exact path)."""
        nt = self.nt_bwd if direction else self.nt_fwd
        if nt == 0 and self.spec.path == KT_PATH_TC and not _exact(self.spec):
            raise RuntimeError(f"kantts_b200: layer {self.spec} cannot run on the tensor-core path")
        return nt


class PreparedWeight:
    """Kernel-layout copies of one layer's effective weight (w_fwd, w_bwd) + the weight-norm
    row norms, valid for one (parameter version) -- see kt_weight_prepare."""

    __slots__ = ("w_fwd", "w_bwd", "norm", "key", "img", "img_stale", "conv_used")

    def __init__(self):
        self.w_fwd = self.w_bwd = self.norm = None
        self.key = None
        self.img = {}          # key -> (packed weight image, descriptor it is packed for), see image()
        self.img_stale = set()
        self.conv_used = False  # a ConvFn forward ran on it: hifigan.prefetch_weights re-prepares it

    def image(self, key, d):
        """A packed weight image: hi/lo SWIZZLE_128B tiles for the tensor-core conv kernels (kt_weight_pack_tc, key
        (direction, N tile, path): the tiling can depend on the sequence length, hence the key on the N tile, and a
        single-pass bf16 image holds the hi tiles only, hence the key on the descriptor's path) or the fused resblock's
        (kt_resblock_pack, key ("rb", C, k, path), d a KtResblockDesc).  Packed for
        descriptor d on first use and re-packed in place once the weights changed; the image depends on its key only,
        so a re-pack reuses that first descriptor (prefetch_weight passes none)."""
        img = self.img.get(key)
        if img is not None and key not in self.img_stale:
            return img[0]
        lib = _lib.load()
        rb = key[0] == "rb"
        if img is None:
            nbytes = lib.kt_resblock_image_bytes(ctypes.byref(d)) if rb else lib.kt_conv1d_tc_image_bytes(ctypes.byref(d), key[0])
            img = (torch.empty(int(nbytes) // 2, device=self.w_fwd.device, dtype=torch.bfloat16), d)
            self.img[key] = img
        img, d = img
        if rb:
            call("kt_resblock_pack", ctypes.byref(d), ptr(self.w_fwd), ptr(img, True))
        else:
            src = self.w_fwd if key[0] == 0 else self.w_bwd
            call("kt_weight_pack_tc", ctypes.byref(d), key[0], ptr(src), ptr(img, True))
        self.img_stale.discard(key)
        return img


def prefetch_weight(cache, spec, v, g):
    """Re-prepare (weight norm + layouts + packed images) a layer's weights ahead of its next forward, for every image
    it holds -- a no-op when nothing changed.  train.GanStep runs this for a whole model on side streams right after
    that model's optimizer step, off the critical path of the other model's forward."""
    pw = prepare_weight(cache, spec, v, g)
    for key in [k for k in pw.img if k in pw.img_stale]:
        pw.image(key, None)


def prepare_weight(cache, spec, v, g):
    """v: reference-layout weight (weight_v for weight-norm, the effective weight otherwise);
    g: weight_g or None.  Re-runs the prepare kernel only when a parameter changed."""
    # only nn.Parameters have a trustworthy (data_ptr, version) identity.  A recomputed spectral-norm weight
    # (`weight_orig / sigma`) is a fresh temporary every forward -- and it IS a leaf whenever weight_orig is frozen or the
    # call runs under no_grad, so `is_leaf` must not decide this: such a weight is never cached and always gets fresh
    # buffers (a pending backward of the other half of a (generated, real) pair still holds the previous ones).
    cacheable = isinstance(v, torch.nn.Parameter) and (g is None or isinstance(g, torch.nn.Parameter))
    # (_version alone is not enough: torch's fused Adam -- and any optimizer that updates through its own kernels -- leaves it
    #  untouched, so every optimizer step also bumps a per-parameter epoch, see _bump_param_epochs)
    key = (v.data_ptr(), v._version, getattr(v, "_kt_epoch", 0),
           None if g is None else (g.data_ptr(), g._version, getattr(g, "_kt_epoch", 0))) if cacheable else None
    if key is not None and cache.key == key and cache.w_fwd is not None and cache.w_fwd.device == v.device:
        return cache
    d0 = v.shape[0]
    d1 = v.shape[1]
    k = spec.kernel
    assert v.numel() == d0 * d1 * k, (v.shape, spec)
    vd = v.detach()
    if not vd.is_contiguous():
        vd = vd.contiguous()
    # The buffers are allocated ONCE and rewritten in place: under CUDA-graph replay the forward of the next
    # step must read the very memory the captured prepare / pack kernels of this step wrote.
    mode = 0 if g is None else 1
    # (A recomputed spectral-norm weight differs between two forwards of the same step whose backward is
    # still pending, so it always gets fresh buffers.)
    if key is None or cache.w_fwd is None or cache.w_fwd.device != v.device or cache.w_fwd.numel() != spec.w_numel:
        cache.w_fwd = torch.empty(spec.w_numel, device=v.device, dtype=torch.float32)
        cache.w_bwd = torch.empty(spec.w_numel, device=v.device, dtype=torch.float32)
        cache.norm = torch.empty(d0, device=v.device, dtype=torch.float32) if mode else None
        cache.img = {}
    gd = None if g is None else g.detach().contiguous()
    call("kt_weight_prepare", ptr(vd), ptr(gd), None, mode, d0, d1, k, int(spec.transposed), spec.groups, ptr(cache.w_fwd),
         ptr(cache.w_bwd), ptr(cache.norm), None)
    cache.key = key
    cache.img_stale = set(cache.img)      # packed tensor-core tiles are re-packed (in place) on next use
    return cache


def _bump_param_epochs(optimizer, args, kwargs):
    """Global optimizer-step post hook: every parameter the optimizer owns gets a new epoch, which invalidates the prepared
    (kernel-layout) copies of its layer.  Found by tests/test_gpu_graph.py: with ``torch.optim.Adam(fused=True)`` the eager
    step kept running on the weights of step 0 (``Tensor._version`` does not move) while the CUDA-graph step, which
    re-prepares unconditionally, was right."""
    for group in optimizer.param_groups:
        for p in group["params"]:
            p._kt_epoch = getattr(p, "_kt_epoch", 0) + 1


from torch.optim.optimizer import register_optimizer_step_post_hook as _register_post_hook  # noqa: E402

_register_post_hook(_bump_param_epochs)

_grad_items = None


class grad_items:
    """Inside this context every op built by this module propagates gradient only for the FIRST ``n`` batch
    items: the caller guarantees that nothing differentiable hangs off the outputs of the remaining items
    (train.GanStep batches the generated and the real waveforms through the discriminators in one call; the
    real half is the reference's ``torch.no_grad()`` pass, trainer.py:527-531).  Backward then runs the data- /
    weight-gradient kernels on ``n`` items and leaves the rest of every input gradient unwritten."""

    def __init__(self, n):
        self.n = n

    def __enter__(self):
        global _grad_items
        self.prev, _grad_items = _grad_items, self.n
        return self

    def __exit__(self, *exc):
        global _grad_items
        _grad_items = self.prev
        return False


def mark_direct_grad(param, flag=True):
    """``param.grad`` is a persistent, pre-zeroed buffer (train.FlatGrads): ConvFn.backward accumulates into it
    inside the gradient kernel (kt_weight_grad_accum) and hands autograd no gradient for it, which removes the
    engine's one ``grad += new`` launch per parameter per backward.  Unmarked parameters (DistributedDataParallel,
    plain ``loss.backward()`` users) receive their gradients through autograd as usual."""
    param._kt_direct = bool(flag)


_WGRAD_ASYNC = True   # False: the chains stay on the calling stream (bench.py's per-launch event timings)
_WG_POOL = {}
_wg_next = 0


def wgrad_pool(device):
    """The per-device pool of weight-gradient side streams (created on first use)."""
    pool = _WG_POOL.setdefault((device.type, device.index), [])
    if not pool:
        pool.extend(torch.cuda.Stream(device=device) for _ in range(4))
    return pool


def _wgrad_stream(device, param):
    """A small per-device pool of streams for the weight-gradient chains (wgrad, split-K reduce, bias column sums,
    weight-norm backward + accumulation): they are leaves of the backward graph, so only the data gradients stay on
    the critical path and the weight gradients fill otherwise idle SMs.  Every parameter is PINNED to one stream of
    the pool (assigned round-robin at its first use): the accumulation into ``param.grad`` is a plain read-modify-write,
    so two chains of the same parameter in one backward (a discriminator applied to y and to y_ in the same graph)
    must be ordered -- the same stream orders them."""
    global _wg_next
    pool = wgrad_pool(device)
    idx = getattr(param, "_kt_wg_stream", None)
    if idx is None:
        _wg_next = (_wg_next + 1) % len(pool)
        idx = param._kt_wg_stream = _wg_next
    return pool[idx % len(pool)]


def join_wgrad_streams(device=None):
    """The current stream waits for the weight-gradient streams (call after backward, before reading .grad)."""
    for (dev_type, dev_index), pool in _WG_POOL.items():
        if device is not None and (dev_type, dev_index) != (device.type, device.index):
            continue
        cur = torch.cuda.current_stream(torch.device(dev_type, dev_index))
        for s in pool:
            cur.wait_stream(s)


def _is_direct(p):
    return p is None or (getattr(p, "_kt_direct", False) and p.grad is not None and p.grad.is_contiguous())


_FORCE_FFMA = False
_tc_launches = 0


def tc_launch_count():
    return _tc_launches


def set_force_ffma(flag):
    """Route every conv through the exact-fp32 FFMA kernels (the reference the tensor-core path is tested against)."""
    global _FORCE_FFMA
    _FORCE_FFMA = bool(flag)


def _exact(spec):
    """Does this layer run on the exact-fp32 (FFMA) kernels only?"""
    return _FORCE_FFMA or spec.path == KT_PATH_FFMA


def _weight_backward(spec, plan, x_, dy, y_, v, g, params, norm, need_v, need_g, need_b):
    """Weight-gradient chain of one conv layer (wgrad kernel -> split-K reduce -> bias column sums -> weight-norm backward),
    shared by ConvFn.backward and ResblockFn.backward.  x_, dy, y_: the layer's input, output gradient and (when it has a
    fused output activation) output, already restricted to the batch items of `plan`.  -> (dbias, dv, dg): the
    gradients to hand to autograd, None for parameters whose .grad the kernels accumulated into directly (mark_direct_grad)."""
    dbias = dv = dg = None
    need_w = need_v or need_g
    if not (need_w or need_b):
        return dbias, dv, dg
    has_g = g is not None
    pv, pg, pb = params
    direct = (need_w and pv.is_leaf and _is_direct(pv) and _is_direct(pg) and (not need_b or _is_direct(pb))
              and need_v and (not has_g or need_g))
    side = _wgrad_stream(x_.device, pv) if (direct and _WGRAD_ASYNC) else None
    if side is not None:
        # nothing of this chain is handed back to autograd (the kernels accumulate into param.grad), so it
        # runs on a side stream; join_wgrad_streams() orders it before the optimizer
        side.wait_stream(torch.cuda.current_stream())
        for t in (x_, dy, y_):
            if t is not None:
                t.record_stream(side)
        cm = torch.cuda.stream(side)
        cm.__enter__()
    try:
        dw = torch.empty(spec.w_numel, device=x_.device, dtype=torch.float32)
        if need_b:
            dbias = torch.empty(spec.c_out, device=x_.device, dtype=torch.float32)
        d, ws_floats, n = plan.d, plan.wg_ws, 4 if need_b else 2
        if ws_floats:
            ws = torch.empty(ws_floats, device=x_.device, dtype=torch.float32)
            _run("conv_wgrad_tc", spec, d, n, 1, ("kt_conv1d_bwd_weight_tc", ctypes.byref(d), ptr(x_), ptr(dy), ptr(y_),
                                                  ptr(dw), ptr(dbias), ptr(ws), ws_floats))
        else:
            _run("conv_wgrad_ffma", spec, d, n, 0, ("kt_conv1d_bwd_weight", ctypes.byref(d), ptr(x_), ptr(dy), ptr(y_),
                                                    ptr(dw), ptr(dbias)))
        if need_w:
            vd = v.detach().contiguous()
            gd = None if g is None else g.detach().contiguous()
            mode = 1 if has_g else 0
            if direct:
                # AccumulateGrad folded into the kernel: param.grad += (train.FlatGrads buffers, pre-zeroed)
                call("kt_weight_grad_accum", ptr(dw), ptr(vd), ptr(gd), ptr(norm), None, mode, vd.shape[0], vd.shape[1],
                     spec.kernel, int(spec.transposed), spec.groups, ptr(pv.grad), None if pg is None else ptr(pg.grad),
                     ptr(dbias) if need_b else None, ptr(pb.grad) if need_b else None, spec.c_out if need_b else 0)
                dbias = None
            else:
                dv = torch.empty_like(vd)
                if has_g:
                    dg = torch.empty_like(g)
                call("kt_weight_grad", ptr(dw), ptr(vd), ptr(gd), ptr(norm), None, mode, vd.shape[0], vd.shape[1],
                     spec.kernel, int(spec.transposed), spec.groups, ptr(dv), ptr(dg))
    finally:
        if side is not None:
            cm.__exit__(None, None, None)
    return dbias, dv, dg


def _workspace(floats, device):
    """Scratch of a tensor-core conv call (None when it needs none), from the caching allocator on the launching stream: it is
    free again for later work on that stream once the call's kernels ran (and under graph capture it comes from the graph's
    pool)."""
    return torch.empty(floats, device=device, dtype=torch.float32) if floats else None


def ragged_lengths(lengths, n, t, device):
    """-> ``lengths`` (each item's rows: a host sequence of ints, or a device integer tensor (n,)) as a contiguous device
    int32 tensor (n,).  ValueError on a wrong count, dtype or device, or a host value outside [1, t]."""
    if torch.is_tensor(lengths):
        if lengths.dtype not in (torch.int32, torch.int64) or lengths.dim() != 1 or lengths.numel() != n:
            raise ValueError(f"lengths: expected an int32 / int64 tensor of shape ({n},), got {lengths.dtype} "
                             f"{tuple(lengths.shape)}")
        if lengths.device != device:
            raise ValueError(f"lengths: expected a tensor on {device}, got {lengths.device}")
        return lengths.to(torch.int32).contiguous()
    vals = [int(v) for v in lengths]
    if len(vals) != n:
        raise ValueError(f"lengths: expected {n} values (one per batch item), got {len(vals)}")
    bad = [v for v in vals if not 1 <= v <= t]
    if bad:
        raise ValueError(f"lengths: every value must lie in [1, {t}], got {bad}")
    return torch.tensor(vals, dtype=torch.int32).to(device)


def utterance_mask(lengths, rows_per_frame):
    """-> the whole-utterance KtStreamMask of a ragged batch: item b's input rows [0, lengths[b] * rows_per_frame) are data,
    later rows read as zeros (kt_conv1d_fwd_masked).  ``lengths``: device int32 (B,), kept alive by the caller."""
    return KtStreamMask(ptr(lengths, True), None, int(rows_per_frame), 0)


def _refuse_masked_grad(what, *tensors):
    """A masked forward has no backward: refuse it where autograd would record it (an autograd.Function's forward always runs
    without grad mode, so the check belongs to the caller)."""
    if torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in tensors):
        raise RuntimeError(f"kantts_b200: a masked {what} forward is inference only (run it under torch.no_grad())")


def rows_mask(y, mask):
    """Zero rows t >= lengths[b] * rows_per_frame of each item b of the (B, T, C) rows ``y``, in place (kt_rows_mask)."""
    call("kt_rows_mask", ctypes.byref(mask), ptr(y), y.shape[0], y.shape[1], y.shape[2])
    return y


class ConvFn(torch.autograd.Function):
    """y = act_out(conv(act_in(x)) + bias) + resid   on channels-last rows.  ``mask`` (utterance_mask, inference only):
    each item's input rows past its utterance read as zeros."""

    @staticmethod
    def forward(ctx, x, resid, bias, v, g, spec, cache, reuse=None, mask=None):
        if mask is not None:
            assert reuse is None and x.dim() == 3, "a masked conv runs whole batches of (B, T, C) rows"
        x = x.contiguous()
        nsub = x.shape[2] if x.dim() == 4 else 1
        B, t_in = x.shape[0], x.shape[1]
        assert x.shape[-1] == spec.c_in, (x.shape, spec)
        full = spec.plan(B, nsub, t_in)
        pw = prepare_weight(cache, spec, v, g)
        shape = (B, full.d.t_out, nsub, spec.c_out) if x.dim() == 4 else (B, full.d.t_out, spec.c_out)
        if reuse is not None:
            # pair_reuse: the output of this layer for the batch items [nb_run, B) is already in `y_buf` (same weights, same
            # inputs, computed earlier in the step); only the first nb_run items are computed, in place
            y_buf, nb_run = reuse
            assert tuple(y_buf.shape) == tuple(shape) and y_buf.is_contiguous() and resid is None, (y_buf.shape, shape)
            y = y_buf.detach()
            run = spec.plan(nb_run, nsub, t_in)
        else:
            y = torch.empty(shape, device=x.device, dtype=torch.float32)
            run = full
        if resid is not None:
            resid = resid.contiguous()
            assert resid.shape == y.shape, (resid.shape, y.shape)
        bd = None if bias is None else bias.detach()
        d, nt, n = run.d, run.tile(0), (spec.stride if spec.transposed else 1)
        # the masked calls take the unmasked call's route, N tile, image and workspace (kt_conv1d_fwd_tc_masked), so the plan
        # and image caches need no key on the mask
        m = () if mask is None else (ctypes.byref(mask),)
        if nt:
            img = pw.image((0, nt, d.path), d)
            ws = _workspace(run.ws_fwd, x.device)
            _run("conv_fwd_tc", spec, d, n + (ws is not None), n,
                 ("kt_conv1d_fwd_tc_masked" if m else "kt_conv1d_fwd_tc", ctypes.byref(d), *m, ptr(x), ptr(img, True),
                  ptr(bd), ptr(resid), ptr(y), ptr(ws), run.ws_fwd))
        else:
            _run("conv_fwd_ffma", spec, d, n, 0, ("kt_conv1d_fwd_masked" if m else "kt_conv1d_fwd", ctypes.byref(d), *m, ptr(x),
                                                  ptr(pw.w_fwd), ptr(bd), ptr(resid), ptr(y)))
        pw.conv_used = True
        if mask is not None:
            return y
        nb = B if _grad_items is None else min(_grad_items, B)     # batch items that carry gradient
        ctx.spec, ctx.nb = spec, nb
        ctx.plan = full if nb == B else spec.plan(nb, nsub, t_in)
        ctx.w_bwd, ctx.norm = pw.w_bwd, pw.norm
        nt_b = ctx.plan.tile(1) if x.requires_grad else 0
        ctx.img_bwd = pw.image((1, nt_b, ctx.plan.d_bwd.path), ctx.plan.d_bwd) if nt_b else None
        ctx.has_resid, ctx.has_bias, ctx.has_g = resid is not None, bias is not None, g is not None
        ctx.params = (v, g, bias)
        ctx.save_for_backward(x, y if spec.act_out != KT_ACT_NONE else None, v, g)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, y, v, g = ctx.saved_tensors
        spec, plan = ctx.spec, ctx.plan
        d = plan.d
        dy = dy.contiguous()
        dx = dres = dbias = dv = dg = None
        dy_full = dy
        if ctx.nb < x.shape[0]:          # grad_items: only the leading items carry gradient (contiguous slices)
            x_, dy = x[:ctx.nb], dy[:ctx.nb]
            y_ = None if y is None else y[:ctx.nb]
        else:
            x_, y_ = x, y
        if ctx.needs_input_grad[0]:
            dx = torch.empty_like(x)     # items >= nb stay unwritten: nothing differentiable consumes them
            n = max(spec.stride if not spec.transposed else 1, spec.upsample)
            # the forward packs the plan's tensor-core image only when its x requires grad; a non-contiguous x is copied
            # there without grad, and its data gradient then runs on the exact kernel
            if ctx.img_bwd is None:
                _run("conv_dgrad_ffma", spec, d, n, 0, ("kt_conv1d_bwd_data", ctypes.byref(d), ptr(dy), ptr(y_),
                                                        ptr(ctx.w_bwd), ptr(x_), ptr(dx)))
            elif plan.up_bwd:
                d2 = plan.d_bwd
                dxu = torch.empty((ctx.nb, d2.t_in * d2.nsub, spec.c_in), device=x.device, dtype=torch.float32)
                ws = _workspace(plan.ws_bwd, x.device)
                _run("conv_dgrad_tc", spec, d, n + 1 + (ws is not None), 1,
                     ("kt_conv1d_bwd_data_tc", ctypes.byref(d2), ptr(dy), ptr(y_), ptr(ctx.img_bwd, True), None, ptr(dxu),
                      ptr(ws), plan.ws_bwd),
                     ("kt_upsample_grad_reduce", ptr(dxu), ptr(x_), spec.act_in, spec.act_in_slope, ptr(dx),
                      ctx.nb * d.t_in * d.nsub, spec.upsample, spec.c_in))
            else:
                ws = _workspace(plan.ws_bwd, x.device)
                _run("conv_dgrad_tc", spec, d, n + (ws is not None), 1,
                     ("kt_conv1d_bwd_data_tc", ctypes.byref(d), ptr(dy), ptr(y_), ptr(ctx.img_bwd, True), ptr(x_), ptr(dx),
                      ptr(ws), plan.ws_bwd))
        if ctx.has_resid and ctx.needs_input_grad[1]:
            # NOT the incoming tensor itself: the autograd engine accumulates gradients arriving at the same input IN PLACE
            # into the first arrival when it holds the last reference (input_buffer.cpp: can_accumulate_inplace), and
            # `dy_full` is still being read -- by this layer's weight-gradient chain on its side stream and, when it is the
            # shared output of Mean3Fn.backward, by the other parallel resblocks on THEIR streams.  Returning the alias let
            # the engine overwrite it under those readers: parameter gradients of the generator were off by ~5 % with the
            # (slow) exact-fp32 kernels and side streams on (test_full_size_c2_train_step_matches_oracle).
            dres = dy_full.clone()
        dbias, dv, dg = _weight_backward(spec, plan, x_, dy, y_, v, g, ctx.params, ctx.norm, ctx.needs_input_grad[3],
                                         ctx.has_g and ctx.needs_input_grad[4], ctx.has_bias and ctx.needs_input_grad[2])
        return dx, dres, dbias, dv, dg, None, None, None, None


def conv(x, spec, cache, v, g=None, bias=None, resid=None, reuse=None, mask=None):
    if mask is not None:
        _refuse_masked_grad("conv", x, v, g, bias, resid)
    return ConvFn.apply(x, resid, bias, v, g, spec, cache, reuse, mask)


def stream_conv(spec, pw, bias, x, y, t_in, win, resid=None, mask=None):
    """One chunk of a causal layer in a stream (no autograd): x, y and resid are the layer's (B, pitch, C) windows, placed
    by ``win`` (a KtStreamWin), and ``t_in`` is the chunk's input rows; the taps before the chunk read the window's history.
    ``pw``: the layer's PreparedWeight, prepared by the caller.  Planned once per chunk shape (ConvSpec.plan, stream=True);
    the tensor-core image of the plan's N tile is packed from ``pw`` on its first use.  ``mask`` (a KtStreamMask): the
    input rows outside each item's utterance read as zeros."""
    plan = spec.plan(x.shape[0], 1, t_in, stream=True)
    d, nt = plan.d, plan.tile(0)
    m = None if mask is None else ctypes.byref(mask)
    if nt:
        img = pw.image((0, nt, d.path), d)
        _run("conv_fwd_tc", spec, d, 1, 1, ("kt_conv1d_fwd_tc_stream", ctypes.byref(d), ctypes.byref(win), m, ptr(x),
                                            ptr(img, True), ptr(bias), ptr(resid), ptr(y)))
    else:
        n = spec.stride if spec.transposed else 1
        _run("conv_fwd_ffma", spec, d, n, 0, ("kt_conv1d_fwd_stream", ctypes.byref(d), ctypes.byref(win), m, ptr(x),
                                              ptr(pw.w_fwd), ptr(bias), ptr(resid), ptr(y)))


# ---- pair_reuse: one (generated, real) pair batch per phase, the real half computed once per step -----------------------
# The trainer evaluates every discriminator on the real waveforms twice per step with the SAME weights: in the generator
# phase (feature-matching targets, trainer.py:527-531) and in the discriminator phase (trainer.py:560).  With
# pair_state("record") the conv layers of the discriminators keep their pair-batch outputs ([generated | real]); with
# pair_state("reuse", B) they compute only the first B items (the re-generated waveforms) into those buffers and reuse the
# real half as is.  Layers whose weights change between two forwards (spectral norm: power iteration) never take part.
_pair_state = None


class pair_state:
    def __init__(self, mode, nb=None):
        self.state = None if mode is None else (mode, nb)

    def __enter__(self):
        global _pair_state
        self.prev, _pair_state = _pair_state, self.state
        return self

    def __exit__(self, *exc):
        global _pair_state
        _pair_state = self.prev
        return False


def pair_conv(owner, x, spec, cache, v, g, bias, resid=None):
    """ops.conv for a layer object `owner` that may record / reuse its pair-batch output (see pair_state)."""
    st = _pair_state
    if st is None or resid is not None or not x.is_cuda:
        return conv(x, spec, cache, v, g, bias, resid)
    mode, nb = st
    if mode == "record":
        y = conv(x, spec, cache, v, g, bias)
        owner._pair_out = y.detach()
        return y
    buf = getattr(owner, "_pair_out", None)
    if buf is None or buf.shape[0] != x.shape[0] or buf.shape[1] != spec.t_out(x.shape[1]) or buf.device != x.device:
        return conv(x, spec, cache, v, g, bias)
    return conv(x, spec, cache, v, g, bias, None, (buf, nb))


# ---- fused ResidualBlock unit (csrc/resblock_tc.cu) -------------------------------------------------------------------
def resblock_desc(spec1, spec2, batch, t):
    """-> KtResblockDesc when the pair (dilated conv, dilation-1 conv; same channels / kernel; fused input LeakyReLU, no
    output activation) can run on the fused kernel for this shape, else None (also on the exact path).  Cached per
    shape and path on spec1; the pair runs in single-pass bf16 when both convs do (set_precision)."""
    if _exact(spec1) or _exact(spec2):
        return None
    key = (batch, t, spec1.path, spec2.path)
    d = spec1._rb_cache.get(key, False)
    if d is not False:
        return d
    d = None
    ok = (spec1.c_in == spec1.c_out == spec2.c_in == spec2.c_out and spec1.kernel == spec2.kernel and spec2.dilation == 1
          and spec1.stride == spec2.stride == 1 and spec1.groups == spec2.groups == 1 and not spec1.transposed
          and not spec2.transposed and spec1.upsample == spec2.upsample == 1 and spec1.act_in == spec2.act_in == KT_ACT_LRELU
          and spec1.act_in_slope == spec2.act_in_slope and spec1.act_out == spec2.act_out == KT_ACT_NONE
          and spec1.t_out(t) == t and spec2.t_out(t) == t)
    if ok:
        cand = KtResblockDesc(batch=batch, t=t, channels=spec1.c_in, kernel=spec1.kernel, dilation=spec1.dilation,
                              pad_left1=spec1.pad_left, pad_left2=spec2.pad_left, slope=spec1.act_in_slope,
                              path=KT_PATH_BF16 if spec1.path == spec2.path == KT_PATH_BF16 else KT_PATH_AUTO)
        if _lib.load().kt_resblock_plan(ctypes.byref(cand)) == 1:
            d = cand
    spec1._rb_cache[key] = d
    return d


class ResblockFn(torch.autograd.Function):
    """y = x + c2(lrelu(c1(lrelu(x)) + b1)) + b2  (layers.py:213-220) in ONE launch; backward = kt_resblock_bwd (both data
    gradients) + the two convs' weight-gradient chains, from the saved (x, h)."""

    @staticmethod
    def forward(ctx, x, b1, v1, g1, b2, v2, g2, spec1, cache1, spec2, cache2, rd, mask=None):
        x = x.contiguous()
        B, T = x.shape[0], x.shape[1]
        pw1 = prepare_weight(cache1, spec1, v1, g1)
        pw2 = prepare_weight(cache2, spec2, v2, g2)
        key = ("rb", rd.channels, rd.kernel, rd.path)
        img1, img2 = pw1.image(key, rd), pw2.image(key, rd)
        need_grad = any(ctx.needs_input_grad[:7])
        y = torch.empty_like(x)
        h = torch.empty_like(x) if need_grad else None
        m = () if mask is None else (ctypes.byref(mask),)
        _run("resblock_fwd_tc", spec1, spec1.plan(B, 1, T).d, 1, 1,
             ("kt_resblock_fwd_masked" if m else "kt_resblock_fwd", ctypes.byref(rd), *m, ptr(x), ptr(img1, True),
              ptr(None if b1 is None else b1.detach()), ptr(img2, True), ptr(None if b2 is None else b2.detach()), ptr(h),
              ptr(y)))
        if need_grad:
            nb = B if _grad_items is None else min(_grad_items, B)
            p1, p2 = spec1.plan(nb, 1, T), spec2.plan(nb, 1, T)
            ctx.nb, ctx.plans, ctx.specs = nb, (p1, p2), (spec1, spec2)
            nt1, nt2 = p1.tile(1), p2.tile(1)
            assert nt1 and nt2, "fused resblock: the data gradients run on the tensor-core kernels"
            ctx.img_bwd = (pw1.image((1, nt1, p1.d.path), p1.d), pw2.image((1, nt2, p2.d.path), p2.d))
            ctx.norms = (pw1.norm, pw2.norm)
            ctx.params = ((v1, g1, b1), (v2, g2, b2))
            ctx.save_for_backward(x, h, v1, g1, v2, g2)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, h, v1, g1, v2, g2 = ctx.saved_tensors
        spec1, spec2 = ctx.specs
        p1, p2 = ctx.plans
        dy = dy.contiguous()
        dy_full = dy
        if ctx.nb < x.shape[0]:
            x_, h_, dy = x[:ctx.nb], h[:ctx.nb], dy[:ctx.nb]
        else:
            x_, h_ = x, h
        dh = torch.empty_like(x_)
        dx = torch.empty_like(x)
        _run("conv_dgrad_tc", spec1, p1.d, 3, 2,
             ("kt_resblock_bwd", ctypes.byref(p1.d), ctypes.byref(p2.d), ptr(x_), ptr(h_), ptr(dy), ptr(ctx.img_bwd[0], True),
              ptr(ctx.img_bwd[1], True), ptr(dh), ptr(dx if ctx.nb == x.shape[0] else dx[:ctx.nb])))
        ni = ctx.needs_input_grad
        (pv1, pg1, pb1), (pv2, pg2, pb2) = ctx.params
        db2, dv2, dg2 = _weight_backward(spec2, p2, h_, dy, None, v2, g2, (pv2, pg2, pb2), ctx.norms[1], ni[5],
                                         g2 is not None and ni[6], pb2 is not None and ni[4])
        db1, dv1, dg1 = _weight_backward(spec1, p1, x_, dh, None, v1, g1, (pv1, pg1, pb1), ctx.norms[0], ni[2],
                                         g1 is not None and ni[3], pb1 is not None and ni[1])
        return (dx if ni[0] else None), db1, dv1, dg1, db2, dv2, dg2, None, None, None, None, None, None


def resblock(x, spec1, cache1, v1, g1, b1, spec2, cache2, v2, g2, b2, rd, mask=None):
    if mask is not None:
        _refuse_masked_grad("resblock", x, v1, g1, b1, v2, g2, b2)
    return ResblockFn.apply(x, b1, v1, g1, b2, v2, g2, spec1, cache1, spec2, cache2, rd, mask)


class SinAddFn(torch.autograd.Function):
    """hifigan.py:157  x = sin(x) + x"""

    @staticmethod
    def forward(ctx, x):
        x = x.contiguous()
        y = torch.empty_like(x)
        call("kt_sinadd_fwd", ptr(x), ptr(y), x.numel())
        ctx.save_for_backward(x)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, = ctx.saved_tensors
        dy = dy.contiguous()
        dx = torch.empty_like(x)
        call("kt_sinadd_bwd", ptr(x), ptr(dy), ptr(dx), x.numel())
        return dx


class Mean3Fn(torch.autograd.Function):
    """hifigan.py:170-176  mean over the parallel resblocks: scale * (a + b + c)."""

    @staticmethod
    def forward(ctx, scale, a, b, c):
        a = a.contiguous()
        b = None if b is None else b.contiguous()
        c = None if c is None else c.contiguous()
        y = torch.empty_like(a)
        call("kt_add3_scale", ptr(a), ptr(b), ptr(c), float(scale), ptr(y), a.numel())
        ctx.scale, ctx.nb, ctx.nc = scale, b is not None, c is not None
        return y

    @staticmethod
    def backward(ctx, dy):
        dy = dy.contiguous()
        g = torch.empty_like(dy)
        call("kt_add3_scale", ptr(dy), None, None, float(ctx.scale), ptr(g), dy.numel())
        return None, g, (g if ctx.nb else None), (g if ctx.nc else None)


class DwtFn(torch.autograd.Function):
    """db3 analysis + channel concat: (B, T) -> (B, (T+5)//2, 2)   (hifigan.py:469-470)"""

    @staticmethod
    def forward(ctx, x):
        x = x.contiguous()
        B, T = x.shape
        y = torch.empty(B, (T + 5) // 2, 2, device=x.device, dtype=torch.float32)
        call("kt_dwt_db3_fwd", ptr(x), ptr(y), B, T)
        ctx.shape = (B, T)
        return y

    @staticmethod
    def backward(ctx, dy):
        B, T = ctx.shape
        dy = dy.contiguous()
        dx = torch.empty(B, T, device=dy.device, dtype=torch.float32)
        call("kt_dwt_db3_bwd", ptr(dy), ptr(dx), B, T)
        return dx


def spec_columns_desc(batch, t, c, reach):
    """-> the KtSpecColumnsDesc of ``batch`` items whose column classes reach ``reach`` (increasing) from the centre."""
    assert len(reach) <= _lib.KT_SPEC_MAX_CLASSES, reach
    return _lib.KtSpecColumnsDesc(batch, t, c, len(reach), (ctypes.c_int32 * _lib.KT_SPEC_MAX_CLASSES)(*reach))


class SpecColumnsFn(torch.autograd.Function):
    """rows (batch + classes, T, C) -> the spectrogram discriminator's feature map (batch, T, width, C), see
    kt_spec_columns_fwd."""

    @staticmethod
    def forward(ctx, rows, batch, reach):
        rows = rows.contiguous()
        _, t, c = rows.shape
        assert rows.shape[0] == batch + len(reach), (rows.shape, batch, reach)
        d = spec_columns_desc(batch, t, c, reach)
        width = 2 * reach[-1] + 1 if reach else 1
        out = torch.empty(batch, t, width, c, device=rows.device, dtype=torch.float32)
        call("kt_spec_columns_fwd", ctypes.byref(d), ptr(rows), ptr(out))
        ctx.d = d
        return out

    @staticmethod
    def backward(ctx, dout):
        d = ctx.d
        dout = dout.contiguous()
        drows = torch.empty(d.batch + d.classes, d.t, d.c, device=dout.device, dtype=torch.float32)
        call("kt_spec_columns_bwd", ctypes.byref(d), ptr(dout), ptr(drows))
        return drows, None, None


class StftMelFn(torch.autograd.Function):
    """Fused framing/window/rFFT/magnitude(/mel/log-normalise).  Returns mel (B, n_mels, frames)
    when ``melmat`` is given, else the magnitude (B, frames, n_bins)."""

    @staticmethod
    def forward(ctx, wav, window, melmat, n_fft, hop, pad_mode, eps, norm=(20.0, -100.0, 8.0, 4.0, -4.0, 4.0)):
        wav = wav.contiguous()
        B, T = wav.shape
        frames = (T - n_fft % 2) // hop + 1           # torch.stft(center=True): n_fft // 2 samples of padding per side
        nb = n_fft // 2 + 1
        n_mels = 0 if melmat is None else melmat.shape[1]
        d = KtMelDesc(batch=B, t=T, n_fft=n_fft, hop=hop, n_mels=n_mels, frames=frames, pad_mode=pad_mode, eps=eps,
                      ref_db=norm[0], min_db=norm[1], norm_scale=norm[2], norm_shift=norm[3], norm_lo=norm[4],
                      norm_hi=norm[5])
        spec = torch.empty(B, frames, nb, 2, device=wav.device, dtype=torch.float32) \
            if ctx.needs_input_grad[0] else None
        mel = amp = None
        if melmat is not None:
            mel = torch.empty(B, n_mels, frames, device=wav.device, dtype=torch.float32)
        else:
            amp = torch.empty(B, frames, nb, device=wav.device, dtype=torch.float32)
        call("kt_stft_mel_fwd", ctypes.byref(d), ptr(wav), ptr(window), ptr(melmat), ptr(mel), ptr(amp), ptr(spec))
        ctx.d = d
        ctx.is_mel = melmat is not None
        ctx.save_for_backward(spec, window, melmat)
        return mel if melmat is not None else amp

    @staticmethod
    def backward(ctx, dout):
        spec, window, melmat = ctx.saved_tensors
        d = ctx.d
        dout = dout.contiguous()
        dwav = torch.empty(d.batch, d.t, device=dout.device, dtype=torch.float32)
        dmel, damp = (dout, None) if ctx.is_mel else (None, dout)
        call("kt_stft_mel_bwd", ctypes.byref(d), ptr(dmel), ptr(damp), ptr(spec), ptr(window), ptr(melmat), ptr(dwav),
             launches=2)
        return dwav, None, None, None, None, None, None, None


def l1_sum_acc(out, a, b, scale):
    """out += scale * sum|a - b| (0-dim device accumulator zeroed by the caller; one launch)."""
    a, b = a.contiguous(), b.contiguous()
    call("kt_l1_sum", ptr(a), ptr(b), a.numel(), float(scale), ptr(out), 1)


def l1_sum(a, b, scale=1.0):
    """scale * sum|a - b| -> 0-dim tensor (no autograd; feature-matching value, loss.py:249)."""
    a, b = a.contiguous(), b.contiguous()
    out = torch.empty((), device=a.device, dtype=torch.float32)
    call("kt_l1_sum", ptr(a), ptr(b), a.numel(), float(scale), ptr(out), 0, launches=2)
    return out
