"""ctypes binding of libkantts_b200.so (the C ABI declared in include/kantts_b200.h).

The library is built in-tree by ``__graft_entry__.build()`` / ``kantts_b200.build_library()``
(nvcc, sm_90a).  There is NO fallback: if the shared object is missing or a call fails, a
RuntimeError is raised -- the product path never routes through PyTorch library kernels or
the CPU oracle.
"""
import ctypes
import os
import subprocess
import sys

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libkantts_b200.so")
CSRC = os.path.join(_HERE, "csrc")
SOURCES = ["api.cu", "conv_ffma.cu", "conv_tc.cu", "resblock_tc.cu", "wgrad_tc.cu", "weights.cu", "misc.cu", "stft_mel.cu", "sambert.cu", "thin.cu"]

KT_ACT_NONE, KT_ACT_LRELU, KT_ACT_TANH = 0, 1, 2
KT_PATH_AUTO, KT_PATH_FFMA, KT_PATH_TC = 0, 1, 2


class KtConv1dDesc(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int32) for n in
                ("batch", "nsub", "t_in", "t_out", "c_in", "c_out", "groups", "kernel", "stride",
                 "dilation", "pad_left", "transposed", "upsample", "act_in")] + \
               [("act_in_slope", ctypes.c_float), ("act_out", ctypes.c_int32),
                ("act_out_slope", ctypes.c_float), ("path", ctypes.c_int32)]


class KtResblockDesc(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int32) for n in ("batch", "t", "channels", "kernel", "dilation", "pad_left1", "pad_left2")] + \
               [("slope", ctypes.c_float), ("path", ctypes.c_int32)]


class KtMelDesc(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int32) for n in ("batch", "t", "n_fft", "hop", "n_mels", "frames", "pad_mode")] + \
               [(n, ctypes.c_float) for n in ("eps", "ref_db", "min_db", "norm_scale", "norm_shift", "norm_lo", "norm_hi")]


class KtAttnDesc(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int32) for n in ("batch", "heads", "d_head", "lq", "lk", "q_stride", "k_stride",
                                              "v_stride", "o_stride", "mask_q_stride")] + \
               [("mask_b_stride", ctypes.c_int64), ("scale", ctypes.c_float), ("keep_scale", ctypes.c_float)]


_P = ctypes.c_void_p
_I = ctypes.c_int32
_L = ctypes.c_int64
_F = ctypes.c_float

# name -> argtypes; mirrors include/kantts_b200.h one to one
PROTOTYPES = {
    "kt_weight_prepare": [_P, _P, _P, _I, _I, _I, _I, _I, _I, _P, _P, _P, _P, _P],
    "kt_weight_grad": [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _P, _P, _P],
    "kt_weight_grad_accum": [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _P, _P, _P, _P, _I, _P],
    "kt_conv1d_fwd": [ctypes.POINTER(KtConv1dDesc), _P, _P, _P, _P, _P, _P],
    "kt_conv1d_bwd_data": [ctypes.POINTER(KtConv1dDesc), _P, _P, _P, _P, _P, _P],
    "kt_conv1d_bwd_weight": [ctypes.POINTER(KtConv1dDesc), _P, _P, _P, _P, _P, _P],
    "kt_sinadd_fwd": [_P, _P, _L, _P],
    "kt_sinadd_bwd": [_P, _P, _P, _L, _P],
    "kt_add3_scale": [_P, _P, _P, _F, _P, _L, _P],
    "kt_upsample_grad_reduce": [_P, _P, _I, _F, _P, _L, _I, _I, _P],
    "kt_dwt_db3_fwd": [_P, _P, _I, _I, _P],
    "kt_dwt_db3_bwd": [_P, _P, _I, _I, _P],
    "kt_stft_mel_fwd": [ctypes.POINTER(KtMelDesc), _P, _P, _P, _P, _P, _P, _P],
    "kt_stft_mel_bwd": [ctypes.POINTER(KtMelDesc), _P, _P, _P, _P, _P, _P, _P],
    "kt_l1_sum": [_P, _P, _L, _F, _P, _P],
    "kt_l1_sum_acc": [_P, _P, _L, _F, _P, _P],
    "kt_conv1d_tc_plan": [ctypes.POINTER(KtConv1dDesc), _I],
    "kt_conv1d_tc_image_bytes": [ctypes.POINTER(KtConv1dDesc), _I],
    "kt_weight_pack_tc": [ctypes.POINTER(KtConv1dDesc), _I, _P, _P, _P],
    "kt_conv1d_fwd_tc": [ctypes.POINTER(KtConv1dDesc), _P, _P, _P, _P, _P, _P],
    "kt_conv1d_bwd_data_tc": [ctypes.POINTER(KtConv1dDesc), _P, _P, _P, _P, _P, _P],
    "kt_conv1d_bwd_weight_tc_workspace": [ctypes.POINTER(KtConv1dDesc)],
    "kt_conv1d_bwd_weight_tc": [ctypes.POINTER(KtConv1dDesc), _P, _P, _P, _P, _P, _P, _L, _P],
    "kt_ar_duration_infer": [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _F, _P, _I, _I, _I, _I, _I, _P],
    "kt_resblock_plan": [ctypes.POINTER(KtResblockDesc)],
    "kt_resblock_image_bytes": [ctypes.POINTER(KtResblockDesc)],
    "kt_resblock_pack": [ctypes.POINTER(KtResblockDesc), _P, _P, _P],
    "kt_resblock_fwd": [ctypes.POINTER(KtResblockDesc), _P, _P, _P, _P, _P, _P, _P, _P],
    "kt_resblock_bwd": [ctypes.POINTER(KtConv1dDesc), ctypes.POINTER(KtConv1dDesc), _P, _P, _P, _P, _P, _P, _P, _P],
    "kt_layernorm_fwd": [_P, _P, _P, _P, _P, _P, _I, _I, _F, _P],
    "kt_layernorm_bwd_workspace": [_I, _I],
    "kt_layernorm_bwd": [_P, _P, _P, _P, _P, _P, _P, _P, _P, _L, _I, _I, _P],
    "kt_attention_fwd": [ctypes.POINTER(KtAttnDesc), _P, _P, _P, _P, _P, _P, _P, _P, _P],
    "kt_attention_bwd": [ctypes.POINTER(KtAttnDesc), _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I, _P],
    "kt_fsmn_fwd": [_P, _P, _P, _P, _I, _I, _I, _I, _I, _P],
    "kt_fsmn_bwd_workspace": [_I, _I, _I, _I],
    "kt_fsmn_bwd": [_P, _P, _P, _P, _P, _P, _P, _L, _I, _I, _I, _I, _I, _P],
    "kt_rows_gather_fwd": [_P, _P, _P, _I, _I, _I, _I, _P],
    "kt_rows_gather_bwd": [_P, _P, _P, _P, _P, _I, _I, _I, _I, _P],
    "kt_debug_set_trace": [_P],
    "kt_debug_set_flags": [_I],
    "kt_debug_wgrad_plan": [ctypes.POINTER(KtConv1dDesc), _P],
    "kt_version": [],
    "kt_has_tc": [],
}

_lib = None


def nvcc_command(out_path=LIB_PATH):
    srcs = [os.path.join(CSRC, s) for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    return ["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
            "-Xcompiler", "-fPIC", "-shared", "-o", out_path] + srcs + ["-lcuda"]


def build_library(force=False, verbose=False):
    """Compile libkantts_b200.so in-tree for sm_90a (cross-compiles without a GPU)."""
    srcs = [os.path.join(CSRC, s) for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    deps = srcs + [os.path.join(CSRC, h) for h in ("common.cuh", "tc_common.cuh", "tma.cuh", "wgmma.cuh")] + [
                   os.path.join(os.path.dirname(_HERE), "include", "kantts_b200.h")]
    deps = [d for d in deps if os.path.exists(d)]
    if not force and os.path.exists(LIB_PATH) and all(os.path.getmtime(LIB_PATH) >= os.path.getmtime(d) for d in deps):
        return LIB_PATH
    cmd = nvcc_command()
    if verbose:
        print(" ".join(cmd), file=sys.stderr)
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + res.stdout + res.stderr)
    return LIB_PATH


def load():
    """-> the ctypes library handle; raises if the shared object is absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). kantts_b200 has no CPU / PyTorch fallback.")
    lib = ctypes.CDLL(LIB_PATH)
    for name, argtypes in PROTOTYPES.items():
        fn = getattr(lib, name)            # AttributeError here = header / library mismatch
        fn.argtypes = argtypes
        fn.restype = ctypes.c_int64 if name.endswith(("_workspace", "_bytes")) else ctypes.c_int
    lib.kt_last_error.argtypes = []
    lib.kt_last_error.restype = ctypes.c_char_p
    _lib = lib
    return lib


def check(rc, what):
    if rc != 0:
        msg = load().kt_last_error().decode(errors="replace")
        raise RuntimeError(f"{what} failed (code {rc}): {msg}")


_PTR_DTYPES = (torch.float32,)
_AUX_DTYPES = (torch.uint8, torch.int32, torch.bfloat16)   # masks / keep-masks, gather indices, packed tensor-core weight tiles


def ptr(t, aux=False):
    """device pointer of a tensor (None -> NULL).  The tensor must be contiguous fp32 on the CURRENT CUDA device (the
    kernels are launched on the current device's stream and read raw fp32); ``aux=True`` admits the integer / byte /
    packed-bf16 side arguments of the ABI (masks, indices, weight tile images).  A float64 / half tensor here would be
    silently reinterpreted (or read out of bounds), so it is an error -- cast at the module boundary."""
    if t is None:
        return None
    if not (t.is_cuda and t.is_contiguous()):
        raise RuntimeError(f"kantts_b200: expected a contiguous CUDA tensor, got device={t.device} "
                           f"contiguous={t.is_contiguous()} (no CPU fallback)")
    if t.dtype not in _PTR_DTYPES and not (aux and t.dtype in _AUX_DTYPES):
        raise RuntimeError(f"kantts_b200: expected a float32 tensor, got {t.dtype} (cast at the module boundary; the "
                           "kernels read raw fp32)")
    if t.device.index != torch.cuda.current_device():
        raise RuntimeError(f"kantts_b200: tensor on {t.device} but the current device is cuda:{torch.cuda.current_device()} "
                           "(wrap the call in torch.cuda.device(...))")
    return t.data_ptr()


_raw_stream = getattr(torch._C, "_cuda_getCurrentRawStream", None)


def stream_ptr():
    """cudaStream_t of the calling thread's current stream (raw accessor: ~15x cheaper than
    torch.cuda.current_stream(), which matters at ~3000 library calls per train step)."""
    if _raw_stream is not None:
        return _raw_stream(torch.cuda.current_device())
    return torch.cuda.current_stream().cuda_stream
