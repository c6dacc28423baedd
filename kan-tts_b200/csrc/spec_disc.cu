// Column bookkeeping of the multi-resolution spectrogram discriminator (SpecDiscriminator, hifigan.py:481-582).
// Its (k, 1) Conv2d layers pad the width-1 frequency axis as well, so every layer adds p zero columns on each side; each
// column is an independent sequence over frames.  The module computes every distinct column once -- the signal column of
// each item and one row block per column class (the columns born as zeros at one layer, identical across positions and
// items) -- and these kernels expand them into the reference's feature maps and fold the gradient back.
#include "common.cuh"

namespace kt {

static inline int columns_grid(long long n_items, int threads) {
  long long blocks = (n_items + threads - 1) / threads;
  const long long cap = 132LL * 16;
  return (int)(blocks < 1 ? 1 : (blocks > cap ? cap : blocks));
}

// Class of the column at distance dist > 0 from the centre: the first class whose reach covers it.
__device__ __forceinline__ int column_class(const KtSpecColumnsDesc& d, int dist) {
  int k = 0;
  while (d.reach[k] < dist) ++k;
  return k;
}

__global__ void spec_columns_fwd_kernel(KtSpecColumnsDesc d, const float* __restrict__ rows, float* __restrict__ out) {
  const int width = d.classes ? 2 * d.reach[d.classes - 1] + 1 : 1;
  const int centre = width / 2;
  const long long n = (long long)d.batch * d.t * width * d.c;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % d.c);
    long long r = i / d.c;
    const int w = (int)(r % width);
    r /= width;
    const int t = (int)(r % d.t);
    const int b = (int)(r / d.t);
    const int dist = abs(w - centre);
    const int item = dist ? d.batch + column_class(d, dist) : b;
    out[i] = __ldg(rows + ((long long)item * d.t + t) * d.c + c);
  }
}

constexpr int kColumnsBwdThreads = 256;

// Blocks [0, class_blocks): one block per (class, frame, 32-channel group).  Its min(C, 32) channel lanes times S slices
// split the class's N * 2 * (columns per side) terms, enumerated item by item, distance by distance, left before right; slice
// s takes terms s, s + S, ... in order, and one thread per channel adds the S partial sums in slice order.  The remaining
// blocks copy each item's centre column into its signal row.  Every sum runs in a fixed order (no atomics: reproducible
// bits).
__global__ void __launch_bounds__(kColumnsBwdThreads) spec_columns_bwd_kernel(KtSpecColumnsDesc d, int class_blocks,
                                                                              const float* __restrict__ dout,
                                                                              float* __restrict__ drows) {
  __shared__ float partial[kColumnsBwdThreads];
  const int width = d.classes ? 2 * d.reach[d.classes - 1] + 1 : 1;
  const int centre = width / 2;
  const int groups = (d.c + 31) / 32;
  if ((int)blockIdx.x >= class_blocks) {
    const long long n = (long long)d.batch * d.t * d.c;
    const long long stride = (long long)(gridDim.x - class_blocks) * blockDim.x;
    for (long long i = (blockIdx.x - class_blocks) * (long long)blockDim.x + threadIdx.x; i < n; i += stride) {
      const int c = (int)(i % d.c);
      const long long r = i / d.c;                        // item * t + frame
      drows[i] = __ldg(dout + (r * width + centre) * d.c + c);
    }
    return;
  }
  const int k = blockIdx.x / (d.t * groups);
  const int t = (blockIdx.x / groups) % d.t;
  const int c0 = (blockIdx.x % groups) * 32;
  const int lanes = min(d.c - c0, 32);
  const int slices = kColumnsBwdThreads / lanes;
  const int lane = threadIdx.x % lanes, slice = threadIdx.x / lanes;
  const int lo = k ? d.reach[k - 1] : 0;
  const int per_item = 2 * (d.reach[k] - lo);
  if (slice < slices) {
    float s = 0.f;
    for (int i = slice; i < d.batch * per_item; i += slices) {
      const int b = i / per_item, j = i % per_item;
      const int w = centre + (j & 1 ? 1 : -1) * (lo + 1 + j / 2);
      s += __ldg(dout + (((long long)b * d.t + t) * width + w) * d.c + c0 + lane);
    }
    partial[threadIdx.x] = s;
  }
  __syncthreads();
  if (threadIdx.x < lanes) {
    float s = 0.f;
    for (int j = 0; j < slices; ++j) s += partial[j * lanes + threadIdx.x];
    drows[((long long)(d.batch + k) * d.t + t) * d.c + c0 + threadIdx.x] = s;
  }
}

static int check_columns(const KtSpecColumnsDesc* d) {
  KT_REQUIRE(d && d->batch > 0 && d->t > 0 && d->c > 0 && d->classes >= 0 && d->classes <= KT_SPEC_MAX_CLASSES,
             "spec_columns: bad descriptor");
  for (int k = 0; k < d->classes; ++k)
    KT_REQUIRE(d->reach[k] > (k ? d->reach[k - 1] : 0), "spec_columns: reach must increase from 1");
  return KT_OK;
}

extern "C" int kt_spec_columns_fwd(const KtSpecColumnsDesc* d, const float* rows, float* out, void* stream) {
  int rc = check_columns(d);
  if (rc) return rc;
  KT_REQUIRE(rows && out, "spec_columns_fwd: bad arguments");
  const int width = d->classes ? 2 * d->reach[d->classes - 1] + 1 : 1;
  spec_columns_fwd_kernel<<<columns_grid((long long)d->batch * d->t * width * d->c, 256), 256, 0,
                            static_cast<cudaStream_t>(stream)>>>(*d, rows, out);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

extern "C" int kt_spec_columns_bwd(const KtSpecColumnsDesc* d, const float* dout, float* drows, void* stream) {
  int rc = check_columns(d);
  if (rc) return rc;
  KT_REQUIRE(dout && drows, "spec_columns_bwd: bad arguments");
  const int class_blocks = d->classes * d->t * ((d->c + 31) / 32);
  const int copy_blocks = columns_grid((long long)d->batch * d->t * d->c, kColumnsBwdThreads);
  spec_columns_bwd_kernel<<<class_blocks + copy_blocks, kColumnsBwdThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      *d, class_blocks, dout, drows);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

}  // namespace kt
