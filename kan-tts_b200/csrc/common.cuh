// Shared helpers for libkantts_b200 (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <atomic>
#include <vector>

#include "../../include/kantts_b200.h"

// Each entry point of kantts_b200.h is defined as extern "C" inside namespace kt, in the file that holds its kernels.  A
// C-linkage function is the same function whichever namespace declares it, so the compiler checks every definition against
// its header declaration; inside a namespace a mismatch is only warning 338, so make it an error.
#pragma nv_diag_error 338

namespace kt {

// The calling thread's error string, returned by kt_last_error (api.cu)
void set_error(const char* fmt, ...);

// variadic: the expression may contain a template-id with commas (allow_dyn_smem<kernel<A, B>>(...))
#define KT_CHECK_CUDA(...)                                                           \
  do {                                                                               \
    cudaError_t _e = (__VA_ARGS__);                                                  \
    if (_e != cudaSuccess) {                                                         \
      kt::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #__VA_ARGS__, cudaGetErrorString(_e)); \
      return KT_ERR_CUDA;                                                            \
    }                                                                                \
  } while (0)

#define KT_REQUIRE(cond, ...)            \
  do {                                   \
    if (!(cond)) {                       \
      kt::set_error(__VA_ARGS__);        \
      return KT_ERR_INVALID;             \
    }                                    \
  } while (0)

inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

// SMs of the current device, queried once per process; 132 (an H100) without a device, so that the host-logic tests plan
// for an H100.  A failed query's error is cleared: a later cudaGetLastError() must not report it as a launch failure.
inline int device_sm_count() {
  static const int n = [] {
    int dev = 0, v = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) {
      cudaGetLastError();
      v = 132;
    }
    return v;
  }();
  return n;
}

// Allow launches of `Kernel` with up to `bytes` of dynamic shared memory (use: KT_CHECK_CUDA(allow_dyn_smem<k>(bytes))
// before the launch).  The attribute belongs to the function, so it is set once per process per kernel instance and never
// lowered later.  A caller returns only after the attribute is set (concurrent first callers each set the same value);
// a failed call is returned and retried by the next caller.
template <auto Kernel>
cudaError_t allow_dyn_smem(int bytes) {
  static std::atomic<bool> done{false};
  if (done.load(std::memory_order_acquire)) return cudaSuccess;
  const cudaError_t e = cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e == cudaSuccess) done.store(true, std::memory_order_release);
  return e;
}

// floor division for b > 0
__host__ __device__ inline int fdiv(int a, int b) { return a >= 0 ? a / b : -((-a + b - 1) / b); }

// How a tensor element is transformed while it is staged into shared memory.
//   PLAIN      v
//   LRELU      leaky_relu(v)                       (fused pre-activation, layers.py:214,216)
//   DLRELU     v * leaky_relu'(aux)                (gradient through a fused output LeakyReLU)
//   DTANH      v * (1 - aux^2)                     (gradient through the fused tanh, hifigan.py:180)
enum SideMode { SIDE_PLAIN = 0, SIDE_LRELU = 1, SIDE_DLRELU = 2, SIDE_DTANH = 3 };

struct Side {
  const float* p;
  const float* aux;
  int mode;
  float slope;
};

// The Side of a tensor with a fused activation `act`: the pre-activation applied to the layer input (derivative = false, aux
// unused), or the activation's derivative at aux applied to a gradient (derivative = true, aux = the activation's output)
inline Side make_side(const float* p, const float* aux, int act, float slope, bool derivative) {
  Side s{p, aux, SIDE_PLAIN, slope};
  if (act == KT_ACT_LRELU) s.mode = derivative ? SIDE_DLRELU : SIDE_LRELU;
  else if (act == KT_ACT_TANH) s.mode = derivative ? SIDE_DTANH : SIDE_PLAIN;
  if (s.mode < SIDE_DLRELU) s.aux = nullptr;
  return s;
}

// The data gradient's output mask: leaky_relu'(x) of a fused input LeakyReLU, else none
inline Side dgrad_mask(const KtConv1dDesc* d, const float* x) {
  return d->act_in == KT_ACT_LRELU ? Side{x, nullptr, SIDE_DLRELU, d->act_in_slope} : Side{nullptr, nullptr, 0, 0.f};
}

__device__ __forceinline__ float side_apply(float v, float aux, int mode, float slope) {
  switch (mode) {
    case SIDE_LRELU: return v > 0.f ? v : v * slope;
    case SIDE_DLRELU: return aux > 0.f ? v : v * slope;
    case SIDE_DTANH: return v * (1.f - aux * aux);
    default: return v;
  }
}

// Deterministic reductions.  Float atomics from many blocks add in scheduling order, so two runs on the same inputs
// would differ in the last bits (and a training run amplifies that).  Instead every block writes its partial sums to its
// own slot of stream-ordered scratch memory (cudaMallocAsync / cudaFreeAsync on the launch stream: safe with concurrent
// streams and inside CUDA-graph capture) and split_sum adds the slots in a fixed order.
int scratch_alloc(float** p, long long floats, cudaStream_t st);
int scratch_free(float* p, cudaStream_t st);
// out[i] = (accumulate ? out[i] : 0) + sum_{s = 0, 1, ..., nsplit - 1} part[s * stride + i]   for i < n
int split_sum(const float* part, long long n, int nsplit, long long stride, float* out, bool accumulate, cudaStream_t st);

constexpr int kMaxTaps = 64;
constexpr int kMaxDynSmem = 227 * 1024;  // opt-in dynamic shared memory per CTA on sm_90

// One "phase" of a generalised 1-D convolution (see conv_ffma.cu for the decomposition):
//   out[bb][o_off + o_step*m][co] (+)= epi( sum_n sum_ci W[tap_j[n]][ci][co] * in[bb][ floor((m*i_step + tap_ioff[n]) / up) ][ci] )
struct Phase {
  int M, o_off, o_step, i_step, up;
  int ntaps;
  int tap_j[kMaxTaps];
  int tap_ioff[kMaxTaps];
  int min_ioff, max_ioff;
  int accumulate;
};

// The taps of a phase split into the residue classes of an input step (<= kMaxResidues): tap n reads time
// q * step + rho of the input, with q = floor(tap_ioff[n] / step) and rho = tap_ioff[n] - q * step.  Class rho holds taps
// [first[rho], first[rho + 1]) in phase order, so in a gather phase (tap_ioff increasing with j) by increasing (q, j).
// The placeholder tap of an output residue no real tap reaches goes to class 0 at a q far outside every tensor: it
// reads only zeros.
constexpr int kMaxResidues = 8;
struct ResidueTaps {
  int first[kMaxResidues + 1];
  int q[kMaxTaps], j[kMaxTaps];
};

inline ResidueTaps residue_taps(const Phase& ph, int step) {
  ResidueTaps rt;
  int n = 0;
  for (int r = 0; r < step; ++r) {
    rt.first[r] = n;
    for (int t = 0; t < ph.ntaps; ++t) {
      const bool placeholder = ph.tap_ioff[t] < -(1 << 24);
      const int q = placeholder ? -(1 << 20) : fdiv(ph.tap_ioff[t], step);
      if ((placeholder ? 0 : ph.tap_ioff[t] - q * step) == r) { rt.q[n] = q; rt.j[n] = ph.tap_j[t]; ++n; }
    }
  }
  rt.first[step] = n;
  return rt;
}

// Chunk rows [lo, hi) of item b's window described by m (KtStreamMask) that lie inside the item's utterance; clamped to
// +-2^26 (far beyond any chunk) to fit an int.  A caller that scales them (by an up-sampling factor) clamps them to its
// window's rows first: 2^26 * 32 is already past INT_MAX.
__device__ __forceinline__ void stream_utterance_rows(const KtStreamMask& m, int b, int& lo, int& hi) {
  const long long l = (long long)m.lag - (long long)__ldg(m.frames_done + b) * m.rows_per_frame;
  const long long h = l + (long long)__ldg(m.lengths + b) * m.rows_per_frame;
  lo = (int)max(-(1LL << 26), min(l, 1LL << 26));
  hi = (int)max(-(1LL << 26), min(h, 1LL << 26));
}

// Whole-utterance masked forwards (kt_conv1d_fwd_masked and friends): item b's input rows [0, the returned bound) are data,
// the bound being lengths[b] * rows_per_frame clamped into [0, t] (the lengths are device data the host never checks: a
// negative one means no rows, never a row before the item's first)
__device__ __forceinline__ int utterance_rows(const KtStreamMask& m, int b, int t) {
  return (int)max(0LL, min((long long)__ldg(m.lengths + b) * m.rows_per_frame, (long long)t));
}

// ---- host functions shared between files ----
// conv_ffma.cu
int validate_conv(const KtConv1dDesc* d);
// the KtStreamMask of a whole-utterance masked forward: lengths and rows_per_frame only (no frames_done, lag 0)
int validate_utterance_mask(const KtStreamMask* m, const char* what);
// validate_conv plus the window placement of one stream chunk (kt_conv1d_fwd_stream / kt_conv1d_fwd_tc_stream)
int validate_stream(const KtConv1dDesc* d, const KtStreamWin* w, const float* resid, const char* what);
// the KtStreamMask of a masked stream call
int validate_stream_mask(const KtStreamMask* m, const char* what);
Phase gather_phase(int t_out, int kernel, int stride, int dil, int pad, int up);
std::vector<Phase> conv_phases(const KtConv1dDesc* d, int dir);
// out[c] = the sum of the Side's values of channel c over `rows` rows, in a fixed order (the bias gradient)
int colsum_bias(const Side& s, long long rows, int c, float* out, cudaStream_t st);
// thin.cu: the single-input-channel layers
bool thin_cin1_ok(const KtConv1dDesc* d);
int thin_cin1_fwd(const KtConv1dDesc* d, const float* x, const float* w_fwd, const float* bias, float* y, cudaStream_t st);
int thin_cin1_wgrad(const KtConv1dDesc* d, const float* x, const float* dy, const float* y, float* dw, float* dbias,
                    cudaStream_t st);
// conv_tc.cu
int tc_pack_layer(const KtConv1dDesc* d, int dir, const float* w, void* out, cudaStream_t st);
// allow_tma = false: the register-staged route, which needs no workspace (kt_resblock_bwd)
int conv1d_bwd_data_tc(const KtConv1dDesc* d, const float* dy, const float* y, const void* wimg, const float* x, float* dx,
                       float* ws, long long ws_floats, cudaStream_t st, bool allow_tma);

}  // namespace kt
