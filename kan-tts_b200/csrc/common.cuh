// Shared helpers for libkantts_b200 (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/kantts_b200.h"

namespace kt {

void set_error(const char* fmt, ...);

#define KT_CHECK_CUDA(expr)                                                          \
  do {                                                                               \
    cudaError_t _e = (expr);                                                         \
    if (_e != cudaSuccess) {                                                         \
      kt::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
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

}  // namespace kt
