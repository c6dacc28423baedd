// Small HBM-bound kernels of the HiFi-GAN hot path: sin(x)+x, resblock mean, db3 DWT pooling,
// L1 reduction.  All are pure streaming kernels (one read / one write per element, float4 where
// the shape allows), grid sized to a multiple of the 132 SMs.
#include <algorithm>

#include "common.cuh"

namespace kt {

static inline int stream_grid(long long n_items, int threads) {
  long long blocks = (n_items + threads - 1) / threads;
  const long long cap = 132LL * 16;
  return (int)(blocks < 1 ? 1 : (blocks > cap ? cap : blocks));
}

// hifigan.py:157  x = torch.sin(x) + x
__global__ void sinadd_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, long long n) {
  const long long n4 = n / 4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 v = __ldg(reinterpret_cast<const float4*>(x) + i);
    v.x += sinf(v.x); v.y += sinf(v.y); v.z += sinf(v.z); v.w += sinf(v.w);
    reinterpret_cast<float4*>(y)[i] = v;
  }
  for (long long i = n4 * 4 + blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    y[i] = x[i] + sinf(x[i]);
}

__global__ void sinadd_bwd_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ dx, long long n) {
  const long long n4 = n / 4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(x) + i);
    float4 g = __ldg(reinterpret_cast<const float4*>(dy) + i);
    g.x *= 1.f + cosf(v.x); g.y *= 1.f + cosf(v.y); g.z *= 1.f + cosf(v.z); g.w *= 1.f + cosf(v.w);
    reinterpret_cast<float4*>(dx)[i] = g;
  }
  for (long long i = n4 * 4 + blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    dx[i] = dy[i] * (1.f + cosf(x[i]));
}

// hifigan.py:170-176  x = (r0 + r1 + r2) / num_kernels
__global__ void add3_scale_kernel(const float* __restrict__ a, const float* __restrict__ b, const float* __restrict__ c,
                                  float scale, float* __restrict__ y, long long n) {
  const long long n4 = n / 4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 v = __ldg(reinterpret_cast<const float4*>(a) + i);
    if (b) { const float4 t = __ldg(reinterpret_cast<const float4*>(b) + i); v.x += t.x; v.y += t.y; v.z += t.z; v.w += t.w; }
    if (c) { const float4 t = __ldg(reinterpret_cast<const float4*>(c) + i); v.x += t.x; v.y += t.y; v.z += t.z; v.w += t.w; }
    v.x *= scale; v.y *= scale; v.z *= scale; v.w *= scale;
    reinterpret_cast<float4*>(y)[i] = v;
  }
  for (long long i = n4 * 4 + blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    y[i] = scale * (a[i] + (b ? b[i] : 0.f) + (c ? c[i] : 0.f));
}

// Data gradient of `nn.Upsample(nearest, scale) -> LeakyReLU -> conv` (hifigan.py:82-97) in two steps: the plain
// conv data gradient wrt the (never materialised in forward) up-sampled rows runs on the tensor-core kernel, then
//   dx[r][c] = act_in'(x[r][c]) * sum_{u < up} dxu[r*up + u][c]
// folds the `up` replicated rows back (bound: HBM, reads up*rows*C + rows*C floats once).
__global__ void upsample_grad_reduce_kernel(const float* __restrict__ dxu, const float* __restrict__ x, int act,
                                            float slope, float* __restrict__ dx, long long rows, int up, int c4) {
  const long long total = rows * c4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / c4;
    const int q = (int)(i % c4);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int u = 0; u < up; ++u) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(dxu) + (r * up + u) * c4 + q);
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    if (act == KT_ACT_LRELU) {
      const float4 xv = __ldg(reinterpret_cast<const float4*>(x) + i);
      acc.x = xv.x > 0.f ? acc.x : acc.x * slope; acc.y = xv.y > 0.f ? acc.y : acc.y * slope;
      acc.z = xv.z > 0.f ? acc.z : acc.z * slope; acc.w = xv.w > 0.f ? acc.w : acc.w * slope;
    }
    reinterpret_cast<float4*>(dx)[i] = acc;
  }
}

int upsample_grad_reduce(const float* dxu, const float* x, int act, float slope, float* dx, long long rows, int up, int c,
                         cudaStream_t st) {
  KT_REQUIRE(dxu && dx && rows > 0 && up >= 1 && c > 0 && (c & 3) == 0, "upsample_grad_reduce: bad arguments (C %% 4 == 0 required)");
  KT_REQUIRE(act == KT_ACT_NONE || (act == KT_ACT_LRELU && x), "upsample_grad_reduce: act must be NONE or LRELU (with x)");
  upsample_grad_reduce_kernel<<<stream_grid(rows * (c / 4), 256), 256, 0, st>>>(dxu, x, act, slope, dx, rows, up, c / 4);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

// db3 analysis filters (PyWavelets Wavelet('db3').dec_lo / dec_hi)
__constant__ float c_dec_lo[6] = {0.035226291882100656f, -0.08544127388224149f, -0.13501102001039084f,
                                  0.4598775021193313f, 0.8068915093133388f, 0.3326705529509569f};
__constant__ float c_dec_hi[6] = {-0.3326705529509569f, 0.8068915093133388f, -0.4598775021193313f,
                                  -0.13501102001039084f, 0.08544127388224149f, 0.035226291882100656f};

// y[b][n][0] = sum_j lo[j] x[b][2n+1-j],  y[b][n][1] = sum_j hi[j] x[b][2n+1-j]   (zero outside [0,T))
__global__ void dwt_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, int batch, int t, int t2) {
  const long long total = (long long)batch * t2;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int b = (int)(i / t2), n = (int)(i % t2);
    const float* xb = x + (long long)b * t;
    float lo = 0.f, hi = 0.f;
#pragma unroll
    for (int j = 0; j < 6; ++j) {
      const int s = 2 * n + 1 - j;
      const float v = (s >= 0 && s < t) ? __ldg(xb + s) : 0.f;
      lo = fmaf(c_dec_lo[j], v, lo);
      hi = fmaf(c_dec_hi[j], v, hi);
    }
    reinterpret_cast<float2*>(y)[i] = make_float2(lo, hi);
  }
}

// adjoint: dx[b][s] = sum_n dy[b][n][0] lo[2n+1-s] + dy[b][n][1] hi[2n+1-s]
__global__ void dwt_bwd_kernel(const float* __restrict__ dy, float* __restrict__ dx, int batch, int t, int t2) {
  const long long total = (long long)batch * t;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int b = (int)(i / t), s = (int)(i % t);
    const float2* db = reinterpret_cast<const float2*>(dy) + (long long)b * t2;
    float acc = 0.f;
    // j = 2n + 1 - s in [0, 5]  ->  n in [ceil((s-1)/2), floor((s+4)/2)]
    const int n_lo = s >= 1 ? (s - 1 + 1) / 2 : 0;
    const int n_hi = min((s + 4) / 2, t2 - 1);
    for (int n = n_lo; n <= n_hi; ++n) {
      const int j = 2 * n + 1 - s;
      if (j < 0 || j > 5) continue;
      const float2 g = __ldg(db + n);
      acc = fmaf(g.x, c_dec_lo[j], acc);
      acc = fmaf(g.y, c_dec_hi[j], acc);
    }
    dx[i] = acc;
  }
}

// one thread per output, slots in ascending order
__global__ void split_sum_kernel(const float* __restrict__ part, long long n, int nsplit, long long stride, float* __restrict__ out,
                                 int accumulate) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float acc = 0.f;
    for (int s = 0; s < nsplit; ++s) acc += __ldg(part + (long long)s * stride + i);
    out[i] = accumulate ? out[i] + acc : acc;
  }
}

// few outputs, many slots: one block per output; thread t sums the slots t, t + 256, ... in order, then a fixed tree
__global__ void split_sum_wide_kernel(const float* __restrict__ part, long long n, int nsplit, long long stride, float* __restrict__ out,
                                      int accumulate) {
  __shared__ float red[256];
  for (long long i = blockIdx.x; i < n; i += gridDim.x) {
    float acc = 0.f;
    for (int s = threadIdx.x; s < nsplit; s += 256) acc += __ldg(part + (long long)s * stride + i);
    red[threadIdx.x] = acc;
    __syncthreads();
    for (int w = 128; w > 0; w >>= 1) {
      if ((int)threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
      __syncthreads();
    }
    if (threadIdx.x == 0) out[i] = accumulate ? out[i] + red[0] : red[0];
    __syncthreads();
  }
}

int scratch_alloc(float** p, long long floats, cudaStream_t st) {
  KT_CHECK_CUDA(cudaMallocAsync(reinterpret_cast<void**>(p), (size_t)std::max<long long>(floats, 1) * sizeof(float), st));
  return KT_OK;
}
int scratch_free(float* p, cudaStream_t st) {
  KT_CHECK_CUDA(cudaFreeAsync(p, st));
  return KT_OK;
}

int split_sum(const float* part, long long n, int nsplit, long long stride, float* out, bool accumulate, cudaStream_t st) {
  if (n <= 0) return KT_OK;
  if (nsplit >= 64 && n <= 4096)
    split_sum_wide_kernel<<<(int)std::min<long long>(n, 132LL * 8), 256, 0, st>>>(part, n, nsplit, stride, out, accumulate ? 1 : 0);
  else
    split_sum_kernel<<<stream_grid(n, 256), 256, 0, st>>>(part, n, nsplit, stride, out, accumulate ? 1 : 0);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

// per-block partial sums of scale * |a - b| -> part[blockIdx.x] (summed in order by split_sum)
__global__ void l1_sum_kernel(const float* __restrict__ a, const float* __restrict__ b, long long n, float scale, float* part) {
  float acc = 0.f;
  const long long gtid = blockIdx.x * (long long)blockDim.x + threadIdx.x, gsz = (long long)gridDim.x * blockDim.x;
  const bool vec = ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b)) & 15) == 0;
  const long long n4 = vec ? n / 4 : 0;
  for (long long i = gtid; i < n4; i += gsz) {
    const float4 u = __ldg(reinterpret_cast<const float4*>(a) + i), v = __ldg(reinterpret_cast<const float4*>(b) + i);
    acc += fabsf(u.x - v.x) + fabsf(u.y - v.y) + fabsf(u.z - v.z) + fabsf(u.w - v.w);
  }
  for (long long i = n4 * 4 + gtid; i < n; i += gsz)
    acc += fabsf(__ldg(a + i) - __ldg(b + i));
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  __shared__ float red[8];
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) t += red[i];
    part[blockIdx.x] = t * scale;
  }
}

int sinadd_fwd(const float* x, float* y, long long n, cudaStream_t st) {
  KT_REQUIRE(x && y && n >= 0, "sinadd_fwd: bad arguments");
  if (n == 0) return KT_OK;
  sinadd_fwd_kernel<<<stream_grid(n / 4 + 1, 256), 256, 0, st>>>(x, y, n);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}
int sinadd_bwd(const float* x, const float* dy, float* dx, long long n, cudaStream_t st) {
  KT_REQUIRE(x && dy && dx && n >= 0, "sinadd_bwd: bad arguments");
  if (n == 0) return KT_OK;
  sinadd_bwd_kernel<<<stream_grid(n / 4 + 1, 256), 256, 0, st>>>(x, dy, dx, n);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}
int add3_scale(const float* a, const float* b, const float* c, float scale, float* y, long long n, cudaStream_t st) {
  KT_REQUIRE(a && y && n >= 0, "add3_scale: bad arguments");
  if (n == 0) return KT_OK;
  add3_scale_kernel<<<stream_grid(n / 4 + 1, 256), 256, 0, st>>>(a, b, c, scale, y, n);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}
int dwt_fwd(const float* x, float* y, int batch, int t, cudaStream_t st) {
  KT_REQUIRE(x && y && batch > 0 && t > 0, "dwt_fwd: bad arguments");
  const int t2 = (t + 5) / 2;
  dwt_fwd_kernel<<<stream_grid((long long)batch * t2, 256), 256, 0, st>>>(x, y, batch, t, t2);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}
int dwt_bwd(const float* dy, float* dx, int batch, int t, cudaStream_t st) {
  KT_REQUIRE(dy && dx && batch > 0 && t > 0, "dwt_bwd: bad arguments");
  const int t2 = (t + 5) / 2;
  dwt_bwd_kernel<<<stream_grid((long long)batch * t, 256), 256, 0, st>>>(dy, dx, batch, t, t2);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}
int l1_sum(const float* a, const float* b, long long n, float scale, float* out, cudaStream_t st, bool accumulate) {
  KT_REQUIRE(a && b && out && n >= 0, "l1_sum: bad arguments");
  if (n == 0) {
    if (!accumulate) KT_CHECK_CUDA(cudaMemsetAsync(out, 0, sizeof(float), st));
    return KT_OK;
  }
  const int blocks = stream_grid(n / 4 + 1, 256);
  float* part = nullptr;
  int rc = scratch_alloc(&part, blocks, st);
  if (rc) return rc;
  l1_sum_kernel<<<blocks, 256, 0, st>>>(a, b, n, scale, part);
  KT_CHECK_CUDA(cudaGetLastError());
  rc = split_sum(part, 1, blocks, 1, out, accumulate, st);
  if (rc) return rc;
  return scratch_free(part, st);
}

}  // namespace kt
