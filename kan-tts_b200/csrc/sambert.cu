// SAM-BERT (kantts/models/sambert) kernels that are not convolutions / GEMMs: LayerNorm, the masked
// multi-head scaled-dot-product attention with d_head <= 64 (probabilities materialised, as the reference
// returns them), the FSMN depthwise memory block and the LengthRegulator gather.  The GEMM-shaped work of
// the model (QKV / output projections, conv feed-forward, prenets, FSMN feed-forward) runs through the
// conv kernels (conv_tc.cu / conv_ffma.cu) as kernel-size-1/3 convolutions over the same (B, L, C) rows.
//
// Everything here is exact fp32 on CUDA cores: with d_head = 16 (sambert_24k.yaml) one attention head is a
// K=16 contraction -- a single wgmma k-step -- and the kernels are bound by the probability-matrix
// traffic (B*H*Lq*Lk*4 bytes written in forward, read twice in backward), not by math.
#include <type_traits>

#include "common.cuh"

namespace kt {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ------------------------------------------------------------------------------------------------
// LayerNorm over the last dim, one warp per row (sambert/__init__.py:64,131,197; kantts_sambert.py:58,129)
// ------------------------------------------------------------------------------------------------
template <int NC>  // columns per lane, c <= 32*NC
__global__ void layernorm_fwd_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                                     const float* __restrict__ beta, float* __restrict__ y, float* __restrict__ mean_out,
                                     float* __restrict__ rstd_out, int rows, int c, float eps) {
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int r = warp; r < rows; r += nwarps) {
    const float* xr = x + (long long)r * c;
    float v[NC];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NC; ++i) {
      const int col = lane + 32 * i;
      v[i] = col < c ? __ldg(xr + col) : 0.f;
      s += v[i];
    }
    const float mean = warp_sum(s) / (float)c;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < NC; ++i) {
      const int col = lane + 32 * i;
      const float d = col < c ? v[i] - mean : 0.f;
      q = fmaf(d, d, q);
    }
    const float rstd = rsqrtf(warp_sum(q) / (float)c + eps);
#pragma unroll
    for (int i = 0; i < NC; ++i) {
      const int col = lane + 32 * i;
      if (col < c) y[(long long)r * c + col] = fmaf((v[i] - mean) * rstd, __ldg(gamma + col), __ldg(beta + col));
    }
    if (lane == 0) {
      mean_out[r] = mean;
      rstd_out[r] = rstd;
    }
  }
}

// dx = rstd * (g*dy - mean_c(g*dy) - xhat * mean_c(g*dy*xhat));  per-CTA partial column sums of
// dy*xhat (dgamma) and dy (dbeta) go to `partial` [gridDim.x][2][c], reduced by colsum2_kernel.
template <int NC>
__global__ void layernorm_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ x,
                                     const float* __restrict__ gamma, const float* __restrict__ mean,
                                     const float* __restrict__ rstd, float* __restrict__ dx, float* __restrict__ partial,
                                     int rows, int c) {
  extern __shared__ float sm[];  // [warps][2][c]
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  float g[NC], ag[NC], ab[NC];
#pragma unroll
  for (int i = 0; i < NC; ++i) {
    const int col = lane + 32 * i;
    g[i] = col < c ? __ldg(gamma + col) : 0.f;
    ag[i] = ab[i] = 0.f;
  }
  for (int r = blockIdx.x * nw + w; r < rows; r += gridDim.x * nw) {
    const float mu = __ldg(mean + r), rs = __ldg(rstd + r);
    float xh[NC], gd[NC];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < NC; ++i) {
      const int col = lane + 32 * i;
      const float d = col < c ? __ldg(dy + (long long)r * c + col) : 0.f;
      xh[i] = col < c ? (__ldg(x + (long long)r * c + col) - mu) * rs : 0.f;
      gd[i] = g[i] * d;
      s1 += gd[i];
      s2 = fmaf(gd[i], xh[i], s2);
      ag[i] = fmaf(d, xh[i], ag[i]);
      ab[i] += d;
    }
    s1 = warp_sum(s1) / (float)c;
    s2 = warp_sum(s2) / (float)c;
#pragma unroll
    for (int i = 0; i < NC; ++i) {
      const int col = lane + 32 * i;
      if (col < c) dx[(long long)r * c + col] = rs * (gd[i] - s1 - xh[i] * s2);
    }
  }
#pragma unroll
  for (int i = 0; i < NC; ++i) {
    const int col = lane + 32 * i;
    if (col < c) {
      sm[(w * 2 + 0) * c + col] = ag[i];
      sm[(w * 2 + 1) * c + col] = ab[i];
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 2 * c; i += blockDim.x) {
    float t = 0.f;
    for (int ww = 0; ww < nw; ++ww) t += sm[ww * 2 * c + i];
    partial[(long long)blockIdx.x * 2 * c + i] = t;
  }
}

// out[i] = sum_p partial[p][i]   (deterministic second stage of the column reductions)
__global__ void colsum_partials_kernel(const float* __restrict__ partial, float* __restrict__ out, int nparts, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float t = 0.f;
  for (int p = 0; p < nparts; ++p) t += __ldg(partial + (long long)p * n + i);
  out[i] = t;
}

// partial rows are [2][c]: dgamma then dbeta
__global__ void ln_reduce_kernel(const float* __restrict__ partial, float* __restrict__ dgamma, float* __restrict__ dbeta,
                                 int nparts, int c) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 2 * c) return;
  float t = 0.f;
  for (int p = 0; p < nparts; ++p) t += __ldg(partial + (long long)p * 2 * c + i);
  if (i < c) dgamma[i] = t; else dbeta[i - c] = t;
}

static int ln_grid(int rows, int warps_per_block) {
  const int want = (rows + warps_per_block - 1) / warps_per_block;
  return want < 1 ? 1 : (want > 148 * 2 ? 148 * 2 : want);
}

extern "C" int64_t kt_layernorm_bwd_workspace(int32_t rows, int32_t c) { return (int64_t)ln_grid(rows, 8) * 2 * c; }

template <int NC>
static int ln_fwd_launch(const float* x, const float* g, const float* b, float* y, float* mean, float* rstd, int rows,
                         int c, float eps, cudaStream_t st) {
  const int blocks = (rows + 7) / 8;
  layernorm_fwd_kernel<NC><<<blocks > 148 * 8 ? 148 * 8 : blocks, 256, 0, st>>>(x, g, b, y, mean, rstd, rows, c, eps);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

extern "C" int kt_layernorm_fwd(const float* x, const float* gamma, const float* beta, float* y, float* mean, float* rstd,
                                int32_t rows, int32_t c, float eps, void* stream) {
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  KT_REQUIRE(x && gamma && beta && y && mean && rstd, "layernorm_fwd: null pointer");
  KT_REQUIRE(rows >= 0 && c >= 1 && c <= 1024, "layernorm_fwd: need 1 <= C <= 1024 (got %d)", c);
  if (rows == 0) return KT_OK;
  if (c <= 32) return ln_fwd_launch<1>(x, gamma, beta, y, mean, rstd, rows, c, eps, st);
  if (c <= 64) return ln_fwd_launch<2>(x, gamma, beta, y, mean, rstd, rows, c, eps, st);
  if (c <= 128) return ln_fwd_launch<4>(x, gamma, beta, y, mean, rstd, rows, c, eps, st);
  if (c <= 256) return ln_fwd_launch<8>(x, gamma, beta, y, mean, rstd, rows, c, eps, st);
  if (c <= 512) return ln_fwd_launch<16>(x, gamma, beta, y, mean, rstd, rows, c, eps, st);
  return ln_fwd_launch<32>(x, gamma, beta, y, mean, rstd, rows, c, eps, st);
}

template <int NC>
static int ln_bwd_launch(const float* dy, const float* x, const float* g, const float* mean, const float* rstd,
                         float* dx, float* ws, int rows, int c, int grid, cudaStream_t st) {
  const size_t smem = (size_t)8 * 2 * c * sizeof(float);   // up to 64 KB at C = 1024: above the 48 KB default
  if (smem > 48 * 1024) KT_CHECK_CUDA(allow_dyn_smem<layernorm_bwd_kernel<NC>>(64 * 1024));
  layernorm_bwd_kernel<NC><<<grid, 256, smem, st>>>(dy, x, g, mean, rstd, dx, ws, rows, c);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

extern "C" int kt_layernorm_bwd(const float* dy, const float* x, const float* gamma, const float* mean, const float* rstd,
                                float* dx, float* dgamma, float* dbeta, float* workspace, int64_t workspace_floats, int32_t rows,
                                int32_t c, void* stream) {
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  KT_REQUIRE(dy && x && gamma && mean && rstd && dx && dgamma && dbeta && workspace, "layernorm_bwd: null pointer");
  KT_REQUIRE(rows >= 1 && c >= 1 && c <= 1024, "layernorm_bwd: need rows >= 1, 1 <= C <= 1024");
  const int grid = ln_grid(rows, 8);
  if (workspace_floats < (long long)grid * 2 * c) {
    set_error("layernorm_bwd: workspace too small");
    return KT_ERR_WORKSPACE;
  }
  int rc;
  if (c <= 32) rc = ln_bwd_launch<1>(dy, x, gamma, mean, rstd, dx, workspace, rows, c, grid, st);
  else if (c <= 64) rc = ln_bwd_launch<2>(dy, x, gamma, mean, rstd, dx, workspace, rows, c, grid, st);
  else if (c <= 128) rc = ln_bwd_launch<4>(dy, x, gamma, mean, rstd, dx, workspace, rows, c, grid, st);
  else if (c <= 256) rc = ln_bwd_launch<8>(dy, x, gamma, mean, rstd, dx, workspace, rows, c, grid, st);
  else if (c <= 512) rc = ln_bwd_launch<16>(dy, x, gamma, mean, rstd, dx, workspace, rows, c, grid, st);
  else rc = ln_bwd_launch<32>(dy, x, gamma, mean, rstd, dx, workspace, rows, c, grid, st);
  if (rc) return rc;
  ln_reduce_kernel<<<(2 * c + 127) / 128, 128, 0, st>>>(workspace, dgamma, dbeta, grid, c);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

// ------------------------------------------------------------------------------------------------
// Attention.  q/k/v/out are (B, L, *) row tensors addressed with explicit row strides and a per-head
// column offset h*D, so the (n*b, L, d) permute copies of the reference (sambert/__init__.py:85-100)
// never exist.  probs is the reference's `attn`: (H*B, Lq, Lk), head-major.
// ------------------------------------------------------------------------------------------------
constexpr int kKeyTile = 256;

struct AttnArgs {
  const float *q, *k, *v;
  const unsigned char* mask;
  float *out, *probs;
  const unsigned char* keep;   // attention dropout keep mask [(h*B+b)][Lq][Lk] or null
  float* probs_dropped;        // optional copy of the dropped probabilities (what the reference returns)
  float keep_scale;
  int B, H, Lq, Lk;
  int q_stride, k_stride, v_stride, o_stride;
  long long mask_b_stride;
  int mask_q_stride;
  float scale;
};

// Sum N per-lane partials across the warp so that every element ends up, fully reduced, in exactly one lane:
// N >= 32: lane l holds elements [l*N/32, (l+1)*N/32) in v[0 .. N/32);  N == 16: lanes 2m and 2m+1 hold element m
// in v[0].  N-1 shuffles instead of 5*N for a butterfly per element.
template <int n, int N>
__device__ __forceinline__ void rs_stage(float (&v)[N], int lane, int off) {
  if constexpr (n >= 1) {
    const bool upper = (lane & off) != 0;
#pragma unroll
    for (int i = 0; i < n; ++i) {
      const float send = upper ? v[i] : v[i + n];
      const float keep = upper ? v[i + n] : v[i];
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
    }
  } else {
    v[0] += __shfl_xor_sync(0xffffffffu, v[0], off);
  }
}
template <int N>
__device__ __forceinline__ void warp_reduce_scatter(float (&v)[N], int lane) {
  rs_stage<N / 2>(v, lane, 16);
  rs_stage<N / 4>(v, lane, 8);
  rs_stage<N / 8>(v, lane, 4);
  rs_stage<N / 16>(v, lane, 2);
  rs_stage<N / 32>(v, lane, 1);
}

// cooperative copy of nk rows of D floats (row stride `stride` floats) into shared rows of DP floats
template <int D, int DP>
__device__ __forceinline__ void stage_rows_smem(float* dst, const float* src, int nk, int stride) {
  const bool vec = (stride % 4 == 0) && ((reinterpret_cast<uintptr_t>(src) & 15) == 0);
  if (vec) {
    for (int i = threadIdx.x; i < nk * (D / 4); i += blockDim.x) {
      const int j = i / (D / 4), e = i % (D / 4);
      *reinterpret_cast<float4*>(dst + j * DP + 4 * e) =
          __ldg(reinterpret_cast<const float4*>(src + (long long)j * stride) + e);
    }
  } else {
    for (int i = threadIdx.x; i < nk * D; i += blockDim.x) {
      const int j = i / D, d = i % D;
      dst[j * DP + d] = __ldg(src + (long long)j * stride + d);
    }
  }
}

// Forward.  CTA = 8 warps x RW query rows of one (batch, head); lanes run over the keys.  A key / value row is
// read from shared memory once (D/4 LDS.128, rows padded to D+4 floats: conflict-free) and used for all RW rows.
template <int D, int RW>
__global__ void __launch_bounds__(256) attn_fwd_kernel(AttnArgs a) {
  extern __shared__ __align__(16) float sm[];
  constexpr int DP = D + 4;
  constexpr int QT = 8 * RW;
  constexpr int N = RW * D;
  float* s_kv = sm;                        // [kKeyTile][DP]
  float* s_sc = sm + kKeyTile * DP;        // [QT][Lk]  scores -> probabilities
  const int bh = blockIdx.y, h = bh / a.B, b = bh % a.B;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int r0 = blockIdx.x * QT + w * RW;          // first query row of this warp
  const float* qb = a.q + (long long)b * a.Lq * a.q_stride + h * D;
  const float* kb = a.k + (long long)b * a.Lk * a.k_stride + h * D;
  const float* vb = a.v + (long long)b * a.Lk * a.v_stride + h * D;
  float* sc0 = s_sc + (size_t)(w * RW) * a.Lk;
  {
    float qr[RW][D];
#pragma unroll
    for (int rr = 0; rr < RW; ++rr) {
      const int r = min(r0 + rr, a.Lq - 1);
#pragma unroll
      for (int d = 0; d < D; ++d) qr[rr][d] = __ldg(qb + (long long)r * a.q_stride + d) * a.scale;
    }
    for (int kt = 0; kt < a.Lk; kt += kKeyTile) {
      const int nk = min(kKeyTile, a.Lk - kt);
      __syncthreads();
      stage_rows_smem<D, DP>(s_kv, kb + (long long)kt * a.k_stride, nk, a.k_stride);
      __syncthreads();
      for (int j = lane; j < nk; j += 32) {
        float kk[D];
#pragma unroll
        for (int e = 0; e < D / 4; ++e) {
          const float4 t = *reinterpret_cast<const float4*>(s_kv + j * DP + 4 * e);
          kk[4 * e] = t.x; kk[4 * e + 1] = t.y; kk[4 * e + 2] = t.z; kk[4 * e + 3] = t.w;
        }
#pragma unroll
        for (int rr = 0; rr < RW; ++rr) {
          float acc = 0.f;
#pragma unroll
          for (int d = 0; d < D; ++d) acc = fmaf(qr[rr][d], kk[d], acc);
          if (a.mask) {
            const int r = min(r0 + rr, a.Lq - 1);
            if (a.mask[b * a.mask_b_stride + (long long)r * a.mask_q_stride + kt + j]) acc = -INFINITY;
          }
          sc0[(size_t)rr * a.Lk + kt + j] = acc;
        }
      }
    }
  }
  __syncwarp();
  // softmax per row (each warp owns its rows), probabilities to HBM
  for (int rr = 0; rr < RW; ++rr) {
    const int r = r0 + rr;
    float* sc = sc0 + (size_t)rr * a.Lk;
    float m = -INFINITY;
    for (int j = lane; j < a.Lk; j += 32) m = fmaxf(m, sc[j]);
    m = warp_max(m);
    float s = 0.f;
    for (int j = lane; j < a.Lk; j += 32) {
      const float e = expf(sc[j] - m);
      sc[j] = e;
      s += e;
    }
    s = warp_sum(s);
    const float inv = 1.f / s;
    const bool live = r < a.Lq;
    const long long prow = ((long long)bh * a.Lq + (live ? r : 0)) * a.Lk;
    for (int j = lane; j < a.Lk; j += 32) {
      float p = sc[j] * inv;
      if (live) a.probs[prow + j] = p;
      if (a.keep) {
        p = a.keep[prow + j] ? p * a.keep_scale : 0.f;
        if (live && a.probs_dropped) a.probs_dropped[prow + j] = p;
      }
      sc[j] = p;
    }
  }
  // out = P V: per-lane partial sums over the lane's keys for all RW x D outputs, then one reduce-scatter
  float acc[N];
#pragma unroll
  for (int i = 0; i < N; ++i) acc[i] = 0.f;
  for (int kt = 0; kt < a.Lk; kt += kKeyTile) {
    const int nk = min(kKeyTile, a.Lk - kt);
    __syncthreads();
    stage_rows_smem<D, DP>(s_kv, vb + (long long)kt * a.v_stride, nk, a.v_stride);
    __syncthreads();
    for (int j = lane; j < nk; j += 32) {
      float vv[D];
#pragma unroll
      for (int e = 0; e < D / 4; ++e) {
        const float4 t = *reinterpret_cast<const float4*>(s_kv + j * DP + 4 * e);
        vv[4 * e] = t.x; vv[4 * e + 1] = t.y; vv[4 * e + 2] = t.z; vv[4 * e + 3] = t.w;
      }
#pragma unroll
      for (int rr = 0; rr < RW; ++rr) {
        const float p = sc0[(size_t)rr * a.Lk + kt + j];
#pragma unroll
        for (int d = 0; d < D; ++d) acc[rr * D + d] = fmaf(p, vv[d], acc[rr * D + d]);
      }
    }
  }
  warp_reduce_scatter<N>(acc, lane);
  constexpr int PER = N >= 32 ? N / 32 : 1;
  const int e0 = N >= 32 ? lane * PER : lane >> 1;
  const int r = r0 + e0 / D;
  if (r < a.Lq && (N >= 32 || (lane & 1) == 0)) {
    float* o = a.out + ((long long)b * a.Lq + r) * a.o_stride + h * D + e0 % D;
#pragma unroll
    for (int i = 0; i < PER; ++i) o[i] = acc[i];
  }
}

struct AttnBwdArgs {
  const float *q, *k, *v, *probs, *dout;
  const unsigned char* keep;
  float keep_scale;
  float *dq, *dk, *dv, *delta;
  int B, H, Lq, Lk;
  int q_stride, k_stride, v_stride, o_stride;   // strides of q/dq, k/dk, v/dv, dout
  float scale;
  int accum_dq;
};

// per query row: dP[j] = dO . V[j] (through the dropout), delta = sum_j P dP, dQ = scale * sum_j P (dP - delta) K[j]
// same work split as the forward kernel: 8 warps x RW rows, lanes over keys, one reduce-scatter for dQ.
template <int D, int RW>
__global__ void __launch_bounds__(256) attn_bwd_q_kernel(AttnBwdArgs a) {
  extern __shared__ __align__(16) float sm[];
  constexpr int DP = D + 4;
  constexpr int QT = 8 * RW;
  constexpr int N = RW * D;
  float* s_kv = sm;                       // [kKeyTile][DP]  V, then K
  float* s_dp = sm + kKeyTile * DP;       // [QT][Lk]
  const int bh = blockIdx.y, h = bh / a.B, b = bh % a.B;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int r0 = blockIdx.x * QT + w * RW;
  const float* kb = a.k + (long long)b * a.Lk * a.k_stride + h * D;
  const float* vb = a.v + (long long)b * a.Lk * a.v_stride + h * D;
  float* dp0 = s_dp + (size_t)(w * RW) * a.Lk;
  long long prow[RW];
  float delta[RW];
#pragma unroll
  for (int rr = 0; rr < RW; ++rr) {
    prow[rr] = ((long long)bh * a.Lq + min(r0 + rr, a.Lq - 1)) * a.Lk;
    delta[rr] = 0.f;
  }
  {
    float dor[RW][D];
#pragma unroll
    for (int rr = 0; rr < RW; ++rr) {
      const int r = min(r0 + rr, a.Lq - 1);
#pragma unroll
      for (int d = 0; d < D; ++d) dor[rr][d] = __ldg(a.dout + ((long long)b * a.Lq + r) * a.o_stride + h * D + d);
    }
    for (int kt = 0; kt < a.Lk; kt += kKeyTile) {
      const int nk = min(kKeyTile, a.Lk - kt);
      __syncthreads();
      stage_rows_smem<D, DP>(s_kv, vb + (long long)kt * a.v_stride, nk, a.v_stride);
      __syncthreads();
      for (int j = lane; j < nk; j += 32) {
        float vv[D];
#pragma unroll
        for (int e = 0; e < D / 4; ++e) {
          const float4 t = *reinterpret_cast<const float4*>(s_kv + j * DP + 4 * e);
          vv[4 * e] = t.x; vv[4 * e + 1] = t.y; vv[4 * e + 2] = t.z; vv[4 * e + 3] = t.w;
        }
#pragma unroll
        for (int rr = 0; rr < RW; ++rr) {
          float acc = 0.f;
#pragma unroll
          for (int d = 0; d < D; ++d) acc = fmaf(dor[rr][d], vv[d], acc);
          if (a.keep) acc = a.keep[prow[rr] + kt + j] ? acc * a.keep_scale : 0.f;   // d/dP through the dropout
          dp0[(size_t)rr * a.Lk + kt + j] = acc;
          delta[rr] = fmaf(__ldg(a.probs + prow[rr] + kt + j), acc, delta[rr]);
        }
      }
    }
  }
#pragma unroll
  for (int rr = 0; rr < RW; ++rr) {
    delta[rr] = warp_sum(delta[rr]);
    if (lane == 0 && r0 + rr < a.Lq) a.delta[(long long)bh * a.Lq + r0 + rr] = delta[rr];
  }
  float acc[N];
#pragma unroll
  for (int i = 0; i < N; ++i) acc[i] = 0.f;
  for (int kt = 0; kt < a.Lk; kt += kKeyTile) {
    const int nk = min(kKeyTile, a.Lk - kt);
    __syncthreads();
    stage_rows_smem<D, DP>(s_kv, kb + (long long)kt * a.k_stride, nk, a.k_stride);
    __syncthreads();
    for (int j = lane; j < nk; j += 32) {
      float kk[D];
#pragma unroll
      for (int e = 0; e < D / 4; ++e) {
        const float4 t = *reinterpret_cast<const float4*>(s_kv + j * DP + 4 * e);
        kk[4 * e] = t.x; kk[4 * e + 1] = t.y; kk[4 * e + 2] = t.z; kk[4 * e + 3] = t.w;
      }
#pragma unroll
      for (int rr = 0; rr < RW; ++rr) {
        const float ds = __ldg(a.probs + prow[rr] + kt + j) * (dp0[(size_t)rr * a.Lk + kt + j] - delta[rr]);
#pragma unroll
        for (int d = 0; d < D; ++d) acc[rr * D + d] = fmaf(ds, kk[d], acc[rr * D + d]);
      }
    }
  }
  warp_reduce_scatter<N>(acc, lane);
  constexpr int PER = N >= 32 ? N / 32 : 1;
  const int e0 = N >= 32 ? lane * PER : lane >> 1;
  const int r = r0 + e0 / D;
  if (r < a.Lq && (N >= 32 || (lane & 1) == 0)) {
    float* o = a.dq + ((long long)b * a.Lq + r) * a.q_stride + h * D + e0 % D;
#pragma unroll
    for (int i = 0; i < PER; ++i) o[i] = a.accum_dq ? o[i] + acc[i] * a.scale : acc[i] * a.scale;
  }
}

// per key j (one thread each, 128 keys per CTA): dV[j] = sum_i Pd[i,j] dO[i],
// dK[j] = scale * sum_i P[i,j] (dPd[i,j] - delta[i]) Q[i]; the query rows stream through shared memory and the
// probability column is fetched 8 rows at a time so that 8 coalesced loads are in flight per thread.
constexpr int kBwdKeys = 128;
constexpr int kBwdQTile = 32;

template <int D>
__global__ void __launch_bounds__(kBwdKeys) attn_bwd_kv_kernel(AttnBwdArgs a) {
  __shared__ __align__(16) float s_q[kBwdQTile][D];
  __shared__ __align__(16) float s_do[kBwdQTile][D];
  __shared__ float s_delta[kBwdQTile];
  const int bh = blockIdx.y, h = bh / a.B, b = bh % a.B;
  const int j = blockIdx.x * kBwdKeys + threadIdx.x;
  const bool live = j < a.Lk;
  float vr[D], dkr[D], dvr[D];
#pragma unroll
  for (int d = 0; d < D; ++d) {
    vr[d] = live ? __ldg(a.v + ((long long)b * a.Lk + j) * a.v_stride + h * D + d) : 0.f;
    dkr[d] = dvr[d] = 0.f;
  }
  for (int i0 = 0; i0 < a.Lq; i0 += kBwdQTile) {
    const int nq = min(kBwdQTile, a.Lq - i0);
    __syncthreads();
    for (int t = threadIdx.x; t < kBwdQTile * D; t += blockDim.x) {
      const int i = t / D, d = t % D;
      const bool in = i < nq;
      s_q[i][d] = in ? __ldg(a.q + ((long long)b * a.Lq + i0 + i) * a.q_stride + h * D + d) : 0.f;
      s_do[i][d] = in ? __ldg(a.dout + ((long long)b * a.Lq + i0 + i) * a.o_stride + h * D + d) : 0.f;
    }
    if (threadIdx.x < kBwdQTile)
      s_delta[threadIdx.x] = threadIdx.x < nq ? __ldg(a.delta + (long long)bh * a.Lq + i0 + threadIdx.x) : 0.f;
    __syncthreads();
    if (live) {
      const long long pofs = ((long long)bh * a.Lq + i0) * a.Lk + j;
#pragma unroll 1
      for (int ib = 0; ib < kBwdQTile; ib += 8) {
        if (ib >= nq) break;
        float p[8], ks[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const bool in = ib + u < nq;
          p[u] = in ? __ldg(a.probs + pofs + (long long)(ib + u) * a.Lk) : 0.f;
          ks[u] = (a.keep && in) ? (a.keep[pofs + (long long)(ib + u) * a.Lk] ? a.keep_scale : 0.f) : 1.f;
        }
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const int i = ib + u;
          float dov[D], qv[D];
#pragma unroll
          for (int e = 0; e < D / 4; ++e) {
            const float4 t = *reinterpret_cast<const float4*>(&s_do[i][4 * e]);
            dov[4 * e] = t.x; dov[4 * e + 1] = t.y; dov[4 * e + 2] = t.z; dov[4 * e + 3] = t.w;
            const float4 s = *reinterpret_cast<const float4*>(&s_q[i][4 * e]);
            qv[4 * e] = s.x; qv[4 * e + 1] = s.y; qv[4 * e + 2] = s.z; qv[4 * e + 3] = s.w;
          }
          const float pd = p[u] * ks[u];
          float dpv = 0.f;
#pragma unroll
          for (int d = 0; d < D; ++d) {
            dpv = fmaf(dov[d], vr[d], dpv);
            dvr[d] = fmaf(pd, dov[d], dvr[d]);
          }
          const float ds = p[u] * (dpv * ks[u] - s_delta[i]);
#pragma unroll
          for (int d = 0; d < D; ++d) dkr[d] = fmaf(ds, qv[d], dkr[d]);
        }
      }
    }
  }
  if (live) {
    float* ok = a.dk + ((long long)b * a.Lk + j) * a.k_stride + h * D;
    float* ov = a.dv + ((long long)b * a.Lk + j) * a.v_stride + h * D;
#pragma unroll
    for (int d = 0; d < D; ++d) {
      ok[d] = dkr[d] * a.scale;
      ov[d] = dvr[d];
    }
  }
}

static int attn_check(const KtAttnDesc* d) {
  KT_REQUIRE(d, "attention: null descriptor");
  KT_REQUIRE(d->batch >= 1 && d->heads >= 1 && d->lq >= 1 && d->lk >= 1, "attention: bad sizes");
  KT_REQUIRE(d->d_head == 8 || d->d_head == 16 || d->d_head == 32 || d->d_head == 64,
             "attention: d_head must be 8, 16, 32 or 64 (got %d)", d->d_head);
  KT_REQUIRE(d->lk <= 2048, "attention: Lk <= 2048 (got %d)", d->lk);
  const int hd = d->heads * d->d_head;
  KT_REQUIRE(d->q_stride >= hd && d->k_stride >= hd && d->v_stride >= hd && d->o_stride >= hd,
             "attention: row strides smaller than heads*d_head");
  KT_REQUIRE((long long)d->heads * d->batch <= 65535, "attention: heads*batch <= 65535");
  return KT_OK;
}

// rows per warp: RW*D per-lane accumulators (<= 64) and a [8*RW][Lk] fp32 score buffer in shared memory.  d_head 32 keeps
// RW = 2 up to the Lk <= 2048 limit, so the dispatchers have no <32, 1> arm.
static_assert(((size_t)8 * 2 * 2048 + (size_t)kKeyTile * (32 + 4)) * sizeof(float) <= (size_t)kMaxDynSmem,
              "attention: d_head 32 at Lk 2048 no longer fits RW = 2; add a <32, 1> dispatch arm");
static int attn_rows_per_warp(int d_head, int lk) {
  int rw = d_head <= 16 ? 4 : (d_head == 32 ? 2 : 1);
  while (rw > 1 && ((size_t)8 * rw * lk + (size_t)kKeyTile * (d_head + 4)) * sizeof(float) > (size_t)kMaxDynSmem) rw >>= 1;
  return rw;
}

template <int D, int RW>
static int attn_fwd_launch(const KtAttnDesc* d, const AttnArgs& a, cudaStream_t st) {
  constexpr int QT = 8 * RW;
  const size_t smem = ((size_t)QT * d->lk + (size_t)kKeyTile * (D + 4)) * sizeof(float);
  KT_REQUIRE(smem <= (size_t)kMaxDynSmem, "attention: shared memory budget exceeded (Lk too long)");
  KT_CHECK_CUDA(allow_dyn_smem<attn_fwd_kernel<D, RW>>(kMaxDynSmem));
  dim3 grid((d->lq + QT - 1) / QT, d->heads * d->batch);
  attn_fwd_kernel<D, RW><<<grid, 256, smem, st>>>(a);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

extern "C" int kt_attention_fwd(const KtAttnDesc* d, const float* q, const float* k, const float* v, const uint8_t* mask,
                                const uint8_t* keep, float* out, float* probs, float* probs_dropped, void* stream) {
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  int rc = attn_check(d);
  if (rc) return rc;
  KT_REQUIRE(q && k && v && out && probs, "attention_fwd: null pointer");
  KT_REQUIRE(!keep || (d->keep_scale >= 1.f), "attention_fwd: keep mask given but keep_scale < 1");
  AttnArgs a{q, k, v, mask, out, probs, keep, probs_dropped, d->keep_scale, d->batch, d->heads, d->lq, d->lk,
             d->q_stride, d->k_stride, d->v_stride, d->o_stride, d->mask_b_stride, d->mask_q_stride, d->scale};
  const int rw = attn_rows_per_warp(d->d_head, d->lk);
  switch (d->d_head * 8 + rw) {
    case 8 * 8 + 4: return attn_fwd_launch<8, 4>(d, a, st);
    case 8 * 8 + 2: return attn_fwd_launch<8, 2>(d, a, st);
    case 16 * 8 + 4: return attn_fwd_launch<16, 4>(d, a, st);
    case 16 * 8 + 2: return attn_fwd_launch<16, 2>(d, a, st);
    case 32 * 8 + 2: return attn_fwd_launch<32, 2>(d, a, st);
    case 64 * 8 + 1: return attn_fwd_launch<64, 1>(d, a, st);
    default: break;
  }
  set_error("attention_fwd: unsupported (d_head=%d, Lk=%d)", d->d_head, d->lk);
  return KT_ERR_INVALID;
}

template <int D, int RW>
static int attn_bwd_launch(const KtAttnDesc* d, const AttnBwdArgs& a, cudaStream_t st) {
  constexpr int QT = 8 * RW;
  const size_t smem = ((size_t)QT * d->lk + (size_t)kKeyTile * (D + 4)) * sizeof(float);
  KT_REQUIRE(smem <= (size_t)kMaxDynSmem, "attention: shared memory budget exceeded (Lk too long)");
  KT_CHECK_CUDA(allow_dyn_smem<attn_bwd_q_kernel<D, RW>>(kMaxDynSmem));
  dim3 gq((d->lq + QT - 1) / QT, d->heads * d->batch);
  attn_bwd_q_kernel<D, RW><<<gq, 256, smem, st>>>(a);
  KT_CHECK_CUDA(cudaGetLastError());
  dim3 gk((d->lk + kBwdKeys - 1) / kBwdKeys, d->heads * d->batch);
  attn_bwd_kv_kernel<D><<<gk, kBwdKeys, 0, st>>>(a);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

extern "C" int kt_attention_bwd(const KtAttnDesc* d, const float* q, const float* k, const float* v, const float* probs,
                                const uint8_t* keep, const float* dout, float* dq, float* dk, float* dv, float* delta,
                                int32_t accum_dq, void* stream) {
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  int rc = attn_check(d);
  if (rc) return rc;
  KT_REQUIRE(q && k && v && probs && dout && dq && dk && dv && delta, "attention_bwd: null pointer");
  AttnBwdArgs a{q, k, v, probs, dout, keep, d->keep_scale, dq, dk, dv, delta, d->batch, d->heads, d->lq, d->lk,
                d->q_stride, d->k_stride, d->v_stride, d->o_stride, d->scale, accum_dq};
  const int rw = attn_rows_per_warp(d->d_head, d->lk);
  switch (d->d_head * 8 + rw) {
    case 8 * 8 + 4: return attn_bwd_launch<8, 4>(d, a, st);
    case 8 * 8 + 2: return attn_bwd_launch<8, 2>(d, a, st);
    case 16 * 8 + 4: return attn_bwd_launch<16, 4>(d, a, st);
    case 16 * 8 + 2: return attn_bwd_launch<16, 2>(d, a, st);
    case 32 * 8 + 2: return attn_bwd_launch<32, 2>(d, a, st);
    case 64 * 8 + 1: return attn_bwd_launch<64, 1>(d, a, st);
    default: break;
  }
  set_error("attention_bwd: unsupported (d_head=%d, Lk=%d)", d->d_head, d->lk);
  return KT_ERR_INVALID;
}

// ------------------------------------------------------------------------------------------------
// FSMN memory block (fsmn.py:46-77): depthwise FIR over time with asymmetric zero padding + skip,
// padded frames zeroed on the way in and on the way out.
//   xm = x * keep;   y[b,t,c] = keep[b,t] * ( xm[b,t,c] + sum_j w[c][j] * xm[b, t + j - lp, c] )
// The data gradient is the same filter with the taps reversed (lp -> K-1-lp) applied to dy.
// CTA = 64 time steps x 64 channels of one batch item: the (64 + K - 1) x 64 input tile (masked rows zeroed)
// and the [K][64] weight tile sit in shared memory; a thread owns one channel and 16 consecutive time steps
// and slides a 16-register window over the taps (per tap: 2 LDS + 16 FMA).
// ------------------------------------------------------------------------------------------------
constexpr int kFsT = 64, kFsC = 64, kFsTT = 16;

__global__ void __launch_bounds__(256) fsmn_fir_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                       const unsigned char* __restrict__ mask, float* __restrict__ y,
                                                       int T, int C, int K, int lp, int reverse) {
  extern __shared__ float sm[];
  float* s_x = sm;                                  // [kFsT + K - 1][kFsC]
  float* s_w = sm + (size_t)(kFsT + K - 1) * kFsC;  // [K][kFsC]
  const int b = blockIdx.z, t0 = blockIdx.x * kFsT, c0 = blockIdx.y * kFsC;
  const int rows = kFsT + K - 1;
  for (int i = threadIdx.x; i < rows * kFsC; i += blockDim.x) {
    const int rr = i / kFsC, cc = i % kFsC;
    const int t = t0 + rr - lp, c = c0 + cc;
    float v = 0.f;
    if (t >= 0 && t < T && c < C && !(mask && mask[(long long)b * T + t])) v = __ldg(x + ((long long)b * T + t) * C + c);
    s_x[i] = v;
  }
  for (int i = threadIdx.x; i < K * kFsC; i += blockDim.x) {
    const int j = i / kFsC, cc = i % kFsC, c = c0 + cc;
    s_w[i] = c < C ? __ldg(w + (long long)c * K + (reverse ? K - 1 - j : j)) : 0.f;
  }
  __syncthreads();
  const int cc = threadIdx.x % kFsC, tq = (threadIdx.x / kFsC) * kFsTT;
  float acc[kFsTT], win[kFsTT];
#pragma unroll
  for (int u = 0; u < kFsTT; ++u) {
    acc[u] = s_x[(tq + u + lp) * kFsC + cc];   // the skip term xm[b,t,c]
    win[u] = s_x[(tq + u) * kFsC + cc];
  }
  for (int j = 0; j < K; ++j) {
    const float wj = s_w[j * kFsC + cc];
#pragma unroll
    for (int u = 0; u < kFsTT; ++u) acc[u] = fmaf(wj, win[u], acc[u]);
#pragma unroll
    for (int u = 0; u < kFsTT - 1; ++u) win[u] = win[u + 1];
    win[kFsTT - 1] = (j + 1 < K) ? s_x[(tq + kFsTT + j) * kFsC + cc] : 0.f;
  }
  const int c = c0 + cc;
  if (c < C) {
#pragma unroll
    for (int u = 0; u < kFsTT; ++u) {
      const int t = t0 + tq + u;
      if (t < T) y[((long long)b * T + t) * C + c] = (mask && mask[(long long)b * T + t]) ? 0.f : acc[u];
    }
  }
}

// dw[c][j] = sum_{b,t} dym[b,t,c] * xm[b, t + j - lp, c].  CTA = (batch item, 256-step time chunk, 64 channels);
// a thread owns one channel and TJ consecutive taps (a sliding TJ-register window over x: per time step 2 LDS +
// TJ FMA).  Per-CTA partials [chunk][C*K] are reduced by colsum_partials_kernel (deterministic).
constexpr int kFsmnChunk = 256;

template <int TJ>
__global__ void __launch_bounds__(256) fsmn_bwd_weight_kernel(const float* __restrict__ x, const float* __restrict__ dy,
                                                              const unsigned char* __restrict__ mask,
                                                              float* __restrict__ partial, int T, int C, int K, int lp,
                                                              int chunks_per_b) {
  extern __shared__ float sm[];
  const int rows = kFsT + 4 * TJ - 1;               // taps padded to 4*TJ >= K
  float* s_x = sm;                                  // [rows][kFsC]
  float* s_dy = sm + (size_t)rows * kFsC;           // [kFsT][kFsC]
  const int b = blockIdx.y / chunks_per_b, tc0 = (blockIdx.y % chunks_per_b) * kFsmnChunk;
  const int c0 = blockIdx.x * kFsC;
  const int cc = threadIdx.x % kFsC, j0 = (threadIdx.x / kFsC) * TJ;
  float acc[TJ];
#pragma unroll
  for (int u = 0; u < TJ; ++u) acc[u] = 0.f;
  for (int t0 = tc0; t0 < min(T, tc0 + kFsmnChunk); t0 += kFsT) {
    __syncthreads();
    for (int i = threadIdx.x; i < rows * kFsC; i += blockDim.x) {
      const int rr = i / kFsC, ci = i % kFsC;
      const int t = t0 + rr - lp, c = c0 + ci;
      float v = 0.f;
      if (t >= 0 && t < T && c < C && !(mask && mask[(long long)b * T + t])) v = __ldg(x + ((long long)b * T + t) * C + c);
      s_x[i] = v;
    }
    for (int i = threadIdx.x; i < kFsT * kFsC; i += blockDim.x) {
      const int rr = i / kFsC, ci = i % kFsC;
      const int t = t0 + rr, c = c0 + ci;
      float v = 0.f;
      if (t < T && c < C && !(mask && mask[(long long)b * T + t])) v = __ldg(dy + ((long long)b * T + t) * C + c);
      s_dy[i] = v;
    }
    __syncthreads();
    float win[TJ];
#pragma unroll
    for (int u = 0; u < TJ; ++u) win[u] = s_x[(j0 + u) * kFsC + cc];
    for (int t = 0; t < kFsT; ++t) {
      const float d = s_dy[t * kFsC + cc];
#pragma unroll
      for (int u = 0; u < TJ; ++u) acc[u] = fmaf(d, win[u], acc[u]);
#pragma unroll
      for (int u = 0; u < TJ - 1; ++u) win[u] = win[u + 1];
      win[TJ - 1] = (t + 1 < kFsT) ? s_x[(t + 1 + j0 + TJ - 1) * kFsC + cc] : 0.f;
    }
  }
  const int c = c0 + cc;
  if (c < C) {
#pragma unroll
    for (int u = 0; u < TJ; ++u)
      if (j0 + u < K) partial[(long long)blockIdx.y * C * K + (long long)c * K + j0 + u] = acc[u];
  }
}

extern "C" int64_t kt_fsmn_bwd_workspace(int32_t B, int32_t T, int32_t C, int32_t K) {
  return (int64_t)B * ((T + kFsmnChunk - 1) / kFsmnChunk) * C * K;
}

static int grid_for(long long n, int threads) {
  long long blocks = (n + threads - 1) / threads;
  const long long cap = 148LL * 16;
  return (int)(blocks < 1 ? 1 : (blocks > cap ? cap : blocks));
}

static int fsmn_fir_launch(const float* x, const float* w, const unsigned char* mask, float* y, int B, int T, int C,
                           int K, int lp, int reverse, cudaStream_t st) {
  const size_t smem = ((size_t)(kFsT + K - 1) * kFsC + (size_t)K * kFsC) * sizeof(float);
  KT_REQUIRE(K <= 256 && B <= 65535, "fsmn: need K <= 256, B <= 65535");
  KT_CHECK_CUDA(allow_dyn_smem<fsmn_fir_kernel>(kMaxDynSmem));
  dim3 grid((T + kFsT - 1) / kFsT, (C + kFsC - 1) / kFsC, B);
  fsmn_fir_kernel<<<grid, 256, smem, st>>>(x, w, mask, y, T, C, K, lp, reverse);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

extern "C" int kt_fsmn_fwd(const float* x, const float* w, const uint8_t* mask, float* y, int32_t B, int32_t T, int32_t C,
                           int32_t K, int32_t lp, void* stream) {
  KT_REQUIRE(x && w && y && B >= 1 && T >= 1 && C >= 1 && K >= 1 && lp >= 0 && lp < K, "fsmn_fwd: bad arguments");
  return fsmn_fir_launch(x, w, mask, y, B, T, C, K, lp, 0, static_cast<cudaStream_t>(stream));
}

template <int TJ>
static int fsmn_wgrad_launch(const float* x, const float* dy, const unsigned char* mask, float* ws, int B, int T, int C,
                             int K, int lp, int cpb, cudaStream_t st) {
  const size_t smem = ((size_t)(kFsT + 4 * TJ - 1) * kFsC + (size_t)kFsT * kFsC) * sizeof(float);
  KT_CHECK_CUDA(allow_dyn_smem<fsmn_bwd_weight_kernel<TJ>>(kMaxDynSmem));
  fsmn_bwd_weight_kernel<TJ><<<dim3((C + kFsC - 1) / kFsC, B * cpb), 256, smem, st>>>(x, dy, mask, ws, T, C, K, lp, cpb);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

extern "C" int kt_fsmn_bwd(const float* x, const float* dy, const float* w, const uint8_t* mask, float* dx, float* dw,
                           float* workspace, int64_t workspace_floats, int32_t B, int32_t T, int32_t C, int32_t K, int32_t lp,
                           void* stream) {
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  KT_REQUIRE(x && dy && w && B >= 1 && T >= 1 && C >= 1 && K >= 1 && lp >= 0 && lp < K, "fsmn_bwd: bad arguments");
  if (dx) {
    int rc = fsmn_fir_launch(dy, w, mask, dx, B, T, C, K, K - 1 - lp, 1, st);
    if (rc) return rc;
  }
  if (dw) {
    const int cpb = (T + kFsmnChunk - 1) / kFsmnChunk;
    if (!workspace || workspace_floats < kt_fsmn_bwd_workspace(B, T, C, K)) {
      set_error("fsmn_bwd: workspace too small");
      return KT_ERR_WORKSPACE;
    }
    KT_REQUIRE(B * cpb <= 65535 && K <= 64, "fsmn_bwd: need B * chunks <= 65535 and K <= 64");
    const int tj = (K + 3) / 4;
    int rc;
    if (tj <= 4) rc = fsmn_wgrad_launch<4>(x, dy, mask, workspace, B, T, C, K, lp, cpb, st);
    else if (tj <= 8) rc = fsmn_wgrad_launch<8>(x, dy, mask, workspace, B, T, C, K, lp, cpb, st);
    else if (tj <= 12) rc = fsmn_wgrad_launch<12>(x, dy, mask, workspace, B, T, C, K, lp, cpb, st);
    else rc = fsmn_wgrad_launch<16>(x, dy, mask, workspace, B, T, C, K, lp, cpb, st);
    if (rc) return rc;
    colsum_partials_kernel<<<(C * K + 127) / 128, 128, 0, st>>>(workspace, dw, B * cpb, C * K);
    KT_CHECK_CUDA(cudaGetLastError());
  }
  return KT_OK;
}

// ------------------------------------------------------------------------------------------------
// LengthRegulator (adaptors.py:15-37) as a row gather instead of the one-hot matmul:
//   out[b,t,:] = idx[b,t] >= 0 ? in[b, idx[b,t], :] : 0          (idx = -1: beyond the rounded durations,
//   masked output frame, or r-padding)
// backward: din[b,i,:] = sum over the token's contiguous span [start[b,i], start[b,i]+count[b,i]) of the
// frames whose idx is i (masked frames inside the span carry idx -1).
// ------------------------------------------------------------------------------------------------
__global__ void rows_gather_fwd_kernel(const float* __restrict__ in, const int* __restrict__ idx, float* __restrict__ out,
                                       int B, int T_out, int T_in, int C) {
  const long long total = (long long)B * T_out * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long long bt = i / C;
    const int b = (int)(bt / T_out);
    const int src = __ldg(idx + bt);
    out[i] = src >= 0 ? __ldg(in + ((long long)b * T_in + src) * C + c) : 0.f;
  }
}

__global__ void rows_gather_bwd_kernel(const float* __restrict__ dout, const int* __restrict__ idx,
                                       const int* __restrict__ start, const int* __restrict__ count,
                                       float* __restrict__ din, int B, int T_out, int T_in, int C) {
  const long long total = (long long)B * T_in * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long long bi = i / C;
    const int tok = (int)(bi % T_in), b = (int)(bi / T_in);
    const int s0 = __ldg(start + bi), n = __ldg(count + bi);
    float acc = 0.f;
    for (int t = s0; t < s0 + n && t < T_out; ++t)
      if (__ldg(idx + (long long)b * T_out + t) == tok) acc += __ldg(dout + ((long long)b * T_out + t) * C + c);
    din[i] = acc;
  }
}

extern "C" int kt_rows_gather_fwd(const float* in, const int32_t* idx, float* out, int32_t B, int32_t T_out, int32_t T_in,
                                  int32_t C, void* stream) {
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  KT_REQUIRE(in && idx && out && B >= 1 && T_out >= 1 && T_in >= 1 && C >= 1, "rows_gather_fwd: bad arguments");
  rows_gather_fwd_kernel<<<grid_for((long long)B * T_out * C, 256), 256, 0, st>>>(in, idx, out, B, T_out, T_in, C);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

extern "C" int kt_rows_gather_bwd(const float* dout, const int32_t* idx, const int32_t* start, const int32_t* count, float* din,
                                  int32_t B, int32_t T_out, int32_t T_in, int32_t C, void* stream) {
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  KT_REQUIRE(dout && idx && start && count && din && B >= 1 && T_out >= 1 && T_in >= 1 && C >= 1,
             "rows_gather_bwd: bad arguments");
  rows_gather_bwd_kernel<<<grid_for((long long)B * T_in * C, 256), 256, 0, st>>>(dout, idx, start, count, din, B, T_out,
                                                                                 T_in, C);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

// ------------------------------------------------------------------------------------------------
// Filled-pause insertion (KanTtsSAMBERT.insert_fp, kantts_sambert.py:766-860) as an index plan plus a row
// gather.  Row t of utterance b is row t of the stream: for j = 0 .. L-1, the 3 rows of filled pause k_j (if
// k_j > 0) then text_hid[b, j]; then the tail rows text_hid[b, q mod L], q = 0, 1, ...  A row code >= 0 is a
// text_hid row; code = -(1 + 3 (k-1) + m) is row m of filled pause k (fp_enc is [3][3][C]).
//   training  (labels):  k_j = label if 1 <= label <= 3, n_b counts every label > 0 over all L positions;
//   inference (FP_p):    flags = (p == max over the 4 classes)[1:] on valid positions, k_j = first set flag,
//                        n_b counts every set flag (an exact tie counts twice but inserts once).
// inter_lengths[b] = input_lengths[b] + 3 n_b.  rows[b, j] = the stream row of text_hid[b, j].
// ------------------------------------------------------------------------------------------------
constexpr int kFpPlanThreads = 256;

__global__ void __launch_bounds__(kFpPlanThreads) fp_plan_kernel(const void* __restrict__ labels, int label_bytes,
                                                                 const float* __restrict__ fp_p, const int* __restrict__ in_len,
                                                                 int L, int T_cap, int* __restrict__ codes,
                                                                 int* __restrict__ rows, int* __restrict__ inter) {
  __shared__ int s_w[kFpPlanThreads / 32], s_n[kFpPlanThreads / 32];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int len = __ldg(in_len + b);
  int* code = codes + (long long)b * T_cap;
  int carry_w = 0, carry_n = 0;
  for (int base = 0; base < L; base += kFpPlanThreads) {
    const int j = base + tid;
    int k = 0, cnt = 0;
    if (j < L) {
      const long long bj = (long long)b * L + j;
      if (label_bytes) {
        const long long v = label_bytes == 8 ? __ldg((const long long*)labels + bj) : (long long)__ldg((const int*)labels + bj);
        cnt = v > 0;
        k = (v >= 1 && v <= 3) ? (int)v : 0;
      } else if (j < len) {
        const float4 p = __ldg((const float4*)fp_p + bj);
        const float mx = fmaxf(fmaxf(p.x, p.y), fmaxf(p.z, p.w));
        const int f1 = p.y == mx, f2 = p.z == mx, f3 = p.w == mx;
        cnt = f1 + f2 + f3;
        k = f1 ? 1 : (f2 ? 2 : (f3 ? 3 : 0));
      }
    }
    const int w = j < L ? (k ? 4 : 1) : 0;
    int iw = w, in = cnt;                                  // inclusive block scan of the widths, block sum of the counts
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int a = __shfl_up_sync(0xffffffffu, iw, o);
      if (lane >= o) iw += a;
    }
    in = __reduce_add_sync(0xffffffffu, in);
    if (lane == 31) s_w[warp] = iw;
    if (lane == 0) s_n[warp] = in;
    __syncthreads();
    int before = 0, tot_w = 0, tot_n = 0;
#pragma unroll
    for (int i = 0; i < kFpPlanThreads / 32; ++i) {
      if (i < warp) before += s_w[i];
      tot_w += s_w[i];
      tot_n += s_n[i];
    }
    if (j < L) {
      const int off = carry_w + before + iw - w;
      for (int m = 0; m < 3 && k; ++m)
        if (off + m < T_cap) code[off + m] = -(1 + 3 * (k - 1) + m);
      const int r = off + w - 1;
      rows[(long long)b * L + j] = r;
      if (r < T_cap) code[r] = j;
    }
    carry_w += tot_w;
    carry_n += tot_n;
    __syncthreads();
  }
  for (int t = carry_w + tid; t < T_cap; t += kFpPlanThreads) code[t] = (t - carry_w) % L;
  if (tid == 0) inter[b] = len + 3 * carry_n;
}

template <int V>
__global__ void fp_insert_fwd_kernel(const float* __restrict__ text, const float* __restrict__ fp_enc,
                                     const int* __restrict__ codes, float* __restrict__ out, int B, int L, int T_cap,
                                     int T_ins, int C) {
  using vec = typename std::conditional<V == 4, float4, float>::type;
  const int cv = C / V;
  const long long total = (long long)B * T_ins * cv;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % cv);
    const long long bt = i / cv;
    const int b = (int)(bt / T_ins), t = (int)(bt % T_ins);
    const int code = __ldg(codes + (long long)b * T_cap + t);
    const float* src = code >= 0 ? text + ((long long)b * L + code) * C : fp_enc + (long long)(-code - 1) * C;
    reinterpret_cast<vec*>(out)[i] = __ldg(reinterpret_cast<const vec*>(src) + c);
  }
}

// d text_hid[b, s] = the interleaved row rows[b, s] (when it is < T_ins) + the tail rows S_b + s + q L, ascending
template <int V>
__global__ void fp_insert_bwd_text_kernel(const float* __restrict__ dout, const int* __restrict__ rows,
                                          float* __restrict__ dtext, int B, int L, int T_ins, int C) {
  using vec = typename std::conditional<V == 4, float4, float>::type;
  const int cv = C / V;
  const long long total = (long long)B * L * cv;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % cv);
    const long long bs = i / cv;
    const int b = (int)(bs / L), s = (int)(bs % L);
    const int S = __ldg(rows + (long long)b * L + L - 1) + 1;
    const vec* d = reinterpret_cast<const vec*>(dout) + (long long)b * T_ins * cv + c;
    vec acc;
    float* a = reinterpret_cast<float*>(&acc);
#pragma unroll
    for (int v = 0; v < V; ++v) a[v] = 0.f;
    const int r = __ldg(rows + bs);
    for (int t = r; t < T_ins; t = (t == r) ? S + s : t + L) {
      const vec x = __ldg(d + (long long)t * cv);
      const float* xv = reinterpret_cast<const float*>(&x);
#pragma unroll
      for (int v = 0; v < V; ++v) a[v] += xv[v];
    }
    reinterpret_cast<vec*>(dtext)[i] = acc;
  }
}

// per-utterance partial d fp_enc: partial[b][km][c] = sum over t ascending of dout[b, t, c] where code = -(km + 1)
__global__ void fp_insert_bwd_fp_partial_kernel(const float* __restrict__ dout, const int* __restrict__ codes,
                                                float* __restrict__ partial, int T_cap, int T_ins, int C) {
  const int b = blockIdx.x;
  const int* code = codes + (long long)b * T_cap;
  const float* d = dout + (long long)b * T_ins * C;
  for (int i = threadIdx.x; i < 9 * C; i += blockDim.x) {
    const int km = i / C, c = i % C;
    float acc = 0.f;
    for (int t = 0; t < T_ins; ++t)
      if (__ldg(code + t) == -(km + 1)) acc += __ldg(d + (long long)t * C + c);
    partial[(long long)b * 9 * C + i] = acc;
  }
}

__global__ void fp_insert_bwd_fp_reduce_kernel(const float* __restrict__ partial, float* __restrict__ dfp, int B, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    float acc = 0.f;
    for (int b = 0; b < B; ++b) acc += partial[(long long)b * n + i];
    dfp[i] = acc;
  }
}

extern "C" int kt_fp_insert_plan(const void* labels, int32_t label_bytes, const float* fp_p, const int32_t* in_len, int32_t B,
                                 int32_t L, int32_t T_cap, int32_t* codes, int32_t* rows, int32_t* inter, void* stream) {
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  KT_REQUIRE(in_len && codes && rows && inter && B >= 1 && L >= 1 && T_cap >= L, "fp_insert_plan: bad arguments");
  KT_REQUIRE(label_bytes ? (labels && (label_bytes == 4 || label_bytes == 8)) : (label_bytes == 0 && fp_p != nullptr),
             "fp_insert_plan: give int32 / int64 labels or the (B, L, 4) predictions");
  KT_REQUIRE(label_bytes || (reinterpret_cast<uintptr_t>(fp_p) & 15) == 0, "fp_insert_plan: predictions not 16-byte aligned");
  fp_plan_kernel<<<B, kFpPlanThreads, 0, st>>>(labels, label_bytes, fp_p, in_len, L, T_cap, codes, rows, inter);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

static bool fp_vec4(int C, const void* a, const void* b, const void* c) {
  return C % 4 == 0 && ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | reinterpret_cast<uintptr_t>(c)) & 15) == 0;
}

extern "C" int kt_fp_insert_fwd(const float* text, const float* fp_enc, const int32_t* codes, float* out, int32_t B, int32_t L,
                                int32_t T_cap, int32_t T_ins, int32_t C, void* stream) {
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  KT_REQUIRE(text && fp_enc && codes && out && B >= 1 && L >= 1 && C >= 1 && T_ins >= L && T_ins <= T_cap,
             "fp_insert_fwd: bad arguments");
  if (fp_vec4(C, text, fp_enc, out))
    fp_insert_fwd_kernel<4><<<grid_for((long long)B * T_ins * C / 4, 256), 256, 0, st>>>(text, fp_enc, codes, out, B, L, T_cap,
                                                                                        T_ins, C);
  else
    fp_insert_fwd_kernel<1><<<grid_for((long long)B * T_ins * C, 256), 256, 0, st>>>(text, fp_enc, codes, out, B, L, T_cap,
                                                                                    T_ins, C);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

extern "C" int kt_fp_insert_bwd(const float* dout, const int32_t* codes, const int32_t* rows, float* dtext, float* dfp,
                                float* partial, int64_t partial_floats, int32_t B, int32_t L, int32_t T_cap, int32_t T_ins,
                                int32_t C, void* stream) {
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  KT_REQUIRE(dout && codes && rows && B >= 1 && L >= 1 && C >= 1 && T_ins >= L && T_ins <= T_cap,
             "fp_insert_bwd: bad arguments");
  KT_REQUIRE(!dfp || (partial && partial_floats >= 9LL * B * C), "fp_insert_bwd: partials need 9 * batch * c floats");
  if (dtext) {
    if (fp_vec4(C, dout, dtext, dtext))
      fp_insert_bwd_text_kernel<4><<<grid_for((long long)B * L * C / 4, 256), 256, 0, st>>>(dout, rows, dtext, B, L, T_ins, C);
    else
      fp_insert_bwd_text_kernel<1><<<grid_for((long long)B * L * C, 256), 256, 0, st>>>(dout, rows, dtext, B, L, T_ins, C);
    KT_CHECK_CUDA(cudaGetLastError());
  }
  if (dfp) {
    fp_insert_bwd_fp_partial_kernel<<<B, 288, 0, st>>>(dout, codes, partial, T_cap, T_ins, C);
    KT_CHECK_CUDA(cudaGetLastError());
    fp_insert_bwd_fp_reduce_kernel<<<grid_for(9LL * C, 256), 256, 0, st>>>(partial, dfp, B, 9 * C);
    KT_CHECK_CUDA(cudaGetLastError());
  }
  return KT_OK;
}

// ---------------------------------------------------------------------------------------------
// Autoregressive duration predictor, whole recurrence in ONE launch (VarRnnARPredictor.infer,
// kantts/models/sambert/adaptors.py:67-83: per symbol  x -> Prenet(1 -> P1 -> P2, ReLU) -> cat(cond) -> 2-layer LSTM ->
// Linear(H -> 1) -> ReLU -> fed back as the next symbol's input).  The reference runs ~10 library launches per symbol
// from a Python loop (L = 256 symbols: ~2500 launches, pure latency); here one CTA per batch item walks the L steps,
// 4H threads = one thread per LSTM gate, activations / states in shared memory, the (transposed) weights streamed from
// L2 with coalesced loads.  The condition's share of the layer-0 input projection does not depend on the recurrence and
// arrives precomputed: g0c[b][i][4H] = cond[b][i] . W_ih0[:, P2:]^T + b_ih0 + b_hh0 (one GEMM for all symbols).
// PyTorch gate order (i, f, g, o); exact fp32.
// ---------------------------------------------------------------------------------------------
struct ArDurParams {
  const float* g0c;                 // [B][L][4H]
  const float *w1, *b1;             // [P1] (Linear(1, P1).weight[:, 0]), [P1]
  const float *w2t, *b2;            // [P1][P2] = Linear(P1, P2).weight^T, [P2]
  const float *wih0t, *whh0t;       // [P2][4H] (prenet columns of weight_ih_l0, transposed), [H][4H]
  const float *wih1t, *whh1t, *bias1;   // [H][4H], [H][4H], [4H] = b_ih1 + b_hh1
  const float* fcw;                 // [H]
  float fcb;
  float* out;                       // [B][L]
  int L, H, P1, P2;
};

__device__ __forceinline__ float sigmoid_f(float v) { return 1.f / (1.f + expf(-v)); }

__global__ void ar_duration_kernel(const ArDurParams p) {
  extern __shared__ float sm[];
  const int H = p.H, G = 4 * H;
  float* p1 = sm;            // [P1]
  float* p2 = p1 + p.P1;     // [P2]
  float* h0 = p2 + p.P2;     // [H]
  float* c0 = h0 + H;
  float* h1 = c0 + H;
  float* c1 = h1 + H;
  float* gates = c1 + H;     // [4H]
  float* xs = gates + G;     // [1]
  const int tid = threadIdx.x, b = blockIdx.x;
  for (int t = tid; t < 4 * H; t += blockDim.x) h0[t] = 0.f;     // h0, c0, h1, c1 are contiguous
  if (tid == 0) xs[0] = 0.f;
  __syncthreads();
  const float* g0 = p.g0c + (long long)b * p.L * G;
  for (int i = 0; i < p.L; ++i) {
    const float x = xs[0];
    for (int t = tid; t < p.P1; t += blockDim.x) p1[t] = fmaxf(fmaf(__ldg(p.w1 + t), x, __ldg(p.b1 + t)), 0.f);
    __syncthreads();
    for (int t = tid; t < p.P2; t += blockDim.x) {
      float acc = __ldg(p.b2 + t);
      for (int k = 0; k < p.P1; ++k) acc = fmaf(__ldg(p.w2t + k * p.P2 + t), p1[k], acc);
      p2[t] = fmaxf(acc, 0.f);
    }
    __syncthreads();
    for (int j = tid; j < G; j += blockDim.x) {
      float acc = __ldg(g0 + (long long)i * G + j);
      for (int k = 0; k < p.P2; ++k) acc = fmaf(__ldg(p.wih0t + k * G + j), p2[k], acc);
      for (int k = 0; k < H; ++k) acc = fmaf(__ldg(p.whh0t + k * G + j), h0[k], acc);
      gates[j] = acc;
    }
    __syncthreads();
    for (int t = tid; t < H; t += blockDim.x) {
      const float ig = sigmoid_f(gates[t]), fg = sigmoid_f(gates[H + t]), gg = tanhf(gates[2 * H + t]), og = sigmoid_f(gates[3 * H + t]);
      const float c = fg * c0[t] + ig * gg;
      c0[t] = c;
      h0[t] = og * tanhf(c);
    }
    __syncthreads();
    for (int j = tid; j < G; j += blockDim.x) {
      float acc = __ldg(p.bias1 + j);
      for (int k = 0; k < H; ++k) acc = fmaf(__ldg(p.wih1t + k * G + j), h0[k], acc);
      for (int k = 0; k < H; ++k) acc = fmaf(__ldg(p.whh1t + k * G + j), h1[k], acc);
      gates[j] = acc;
    }
    __syncthreads();
    for (int t = tid; t < H; t += blockDim.x) {
      const float ig = sigmoid_f(gates[t]), fg = sigmoid_f(gates[H + t]), gg = tanhf(gates[2 * H + t]), og = sigmoid_f(gates[3 * H + t]);
      const float c = fg * c1[t] + ig * gg;
      c1[t] = c;
      h1[t] = og * tanhf(c);
    }
    __syncthreads();
    if (tid < 32) {
      float acc = 0.f;
      for (int k = tid; k < H; k += 32) acc = fmaf(__ldg(p.fcw + k), h1[k], acc);
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      if (tid == 0) {
        const float y = fmaxf(acc + p.fcb, 0.f);
        xs[0] = y;
        p.out[(long long)b * p.L + i] = y;
      }
    }
    __syncthreads();
  }
}

extern "C" int kt_ar_duration_infer(const float* g0c, const float* w1, const float* b1, const float* w2t, const float* b2,
                                    const float* wih0t, const float* whh0t, const float* wih1t, const float* whh1t,
                                    const float* bias1, const float* fcw, float fcb, float* out, int32_t B, int32_t L, int32_t H,
                                    int32_t P1, int32_t P2, void* stream) {
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  KT_REQUIRE(g0c && w1 && b1 && w2t && b2 && wih0t && whh0t && wih1t && whh1t && bias1 && fcw && out, "ar_duration_infer: null pointer");
  KT_REQUIRE(B >= 1 && L >= 1 && H >= 1 && H <= 256 && P1 >= 1 && P2 >= 1 && P1 <= 1024 && P2 <= 1024, "ar_duration_infer: bad sizes");
  ArDurParams p{g0c, w1, b1, w2t, b2, wih0t, whh0t, wih1t, whh1t, bias1, fcw, fcb, out, L, H, P1, P2};
  const int threads = std::min(1024, std::max(32, ((4 * H + 31) / 32) * 32));
  const size_t smem = (size_t)(P1 + P2 + 8 * H + 1) * sizeof(float);
  ar_duration_kernel<<<B, threads, smem, st>>>(p);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

// ---------------------------------------------------------------------------------------------
// Streaming post-net (PostNet.streamer): one chunk of MemoryBlockV2 and one chunk of the post-net LSTM.  Which chunk rows
// of item b lie inside its utterance comes from the device (KtStreamMask, read by stream_utterance_rows), so every slot of
// one launch can sit at a different place in its own utterance.
//
// fsmn_stream_slots_kernel: the memory block as a causal depthwise FIR whose output lags its input by rp = K-1-lp rows.
// m describes the input window: input row u of item b's chunk (negative: the window's history) holds a frame iff
// lo <= u < hi.  Output row t is the frame of input row t - rp; its taps j < K read input rows t + j - (K-1).
// keep(u) = lo <= u < hi; xm = keep * x, by selection, so whatever a window holds outside the utterance reads as zero.
//   y[t] = keep(t - rp) * (xm[t - rp] + sum_j w[c][j] * xm[t + j - (K-1)]) + resid[t]
// The skip term first, then the taps in order, each an fmaf with the masked value: fsmn_fir_kernel's sum, so a streamed row
// equals the whole-sequence row bit for bit.  One thread per (row, channel) of one item (blockIdx.y).
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) fsmn_stream_slots_kernel(const KtStreamMask m, const float* __restrict__ x,
                                                                const float* __restrict__ w, const float* __restrict__ resid,
                                                                float* __restrict__ y, KtStreamWin win, int rows, int C, int K,
                                                                int lp) {
  const int b = blockIdx.y;
  int lo, hi;
  stream_utterance_rows(m, b, lo, hi);
  const int rp = K - 1 - lp;
  const long long n = (long long)rows * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int t = (int)(i / C), c = (int)(i - (long long)t * C);
    const float* xc = x + ((long long)b * win.in_pitch + win.in_first + t - (K - 1)) * C + c;
    const bool keep_t = t - rp >= lo && t - rp < hi;
    float acc = keep_t ? __ldg(xc + (long long)lp * C) : 0.f;
    for (int j = 0; j < K; ++j) {
      const int u = t + j - (K - 1);
      const float v = (u >= lo && u < hi) ? __ldg(xc + (long long)j * C) : 0.f;
      acc = fmaf(__ldg(w + (long long)c * K + j), v, acc);
    }
    float out = keep_t ? acc : 0.f;
    if (resid) out += __ldg(resid + ((long long)b * win.res_pitch + win.res_first + t) * C + c);
    y[((long long)b * win.out_pitch + win.out_first + t) * C + c] = out;
  }
}

extern "C" int kt_fsmn_fwd_stream_slots(const KtStreamWin* win, const KtStreamMask* m, const float* x, const float* w,
                                        const float* resid, float* y, int32_t B, int32_t rows, int32_t C, int32_t K,
                                        int32_t lp, void* stream) {
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  int rc = validate_stream_mask(m, "fsmn_fwd_stream_slots");
  if (rc) return rc;
  KT_REQUIRE(win && x && w && y, "fsmn_fwd_stream_slots: null pointer");
  KT_REQUIRE(B >= 1 && B <= 65535 && rows >= 1 && C >= 1 && K >= 1 && lp >= 0 && lp < K, "fsmn_fwd_stream_slots: bad sizes");
  KT_REQUIRE(win->in_first >= K - 1 && win->in_first + rows <= win->in_pitch,
             "fsmn_fwd_stream_slots: the input window needs K - 1 rows of history before the chunk");
  KT_REQUIRE(win->out_first >= 0 && win->out_first + rows <= win->out_pitch,
             "fsmn_fwd_stream_slots: the chunk does not fit its output window");
  KT_REQUIRE(!resid || (win->res_first >= 0 && win->res_first + rows <= win->res_pitch),
             "fsmn_fwd_stream_slots: the chunk does not fit its residual window");
  const long long n = (long long)rows * C;
  const int blocks = (int)std::min<long long>((n + 255) / 256, 1024);
  fsmn_stream_slots_kernel<<<dim3(blocks, B), 256, 0, st>>>(*m, x, w, resid, y, *win, rows, C, K, lp);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

// lstm_rows_kernel: the recurrence of a 1-layer LSTM over `rows` rows of one (item b = blockIdx.x, direction d = blockIdx.y)
// per CTA, one thread per gate: gate j of a step = gx[t][j] + sum_k W_hh^T[k][j] h[k] (W_hh^T streamed from L2, coalesced
// over j), then one thread per hidden unit updates c and h.  The CTA runs rows [lo, hi) upwards (d = 0) or downwards (d = 1)
// and writes zeros to the rows outside them.  Row t of item b, direction d, reads gx at ((b * gx_pitch + t) * D + d) * 4H
// and writes h at ((b * h_pitch + t) * D + d) * H, D = gridDim.y; W_hh^T of direction d at whh_t + d * H * 4H.
//   lengths != NULL (kt_blstm_ragged, kt_lstm_train_fwd): lo = 0, hi = min(lengths[b], rows), from (h, c) = 0.
//   m.lengths != NULL (kt_lstm_stream_slots, D = 1): with lo from m (stream_utterance_rows), row t is frame t - lo, and hi =
//   rows.  A chunk whose first row is frame 0 or earlier (lo >= 0) starts from (h, c) = 0 whatever state holds, a later
//   chunk from the carried state[b][2][H]; the rows before frame 0 are zero and (h, c) after the last row go to state.
//   neither (kt_lstm_train_fwd without lengths): every row, from (h, c) = 0.
// init (kt_lstm_train_fwd, optional): the initial (h, c) of each (item, direction) at init[((b * D + d) * 2) * H], h then c,
// in place of zeros.  c_out / act_out (training, optional): the cell state c at h's offsets (zero outside [lo, hi), as h)
// and the gate activations (sigmoid i, f, tanh g, sigmoid o) at gx's, for kt_lstm_train_bwd (not written outside [lo, hi)).
// Each step's sums run in the same order whatever the launch shape, so an item's rows depend on its own gx rows, its
// length and the weights only.  PyTorch gate order (i, f, g, o); exact fp32.
__global__ void lstm_rows_kernel(const float* __restrict__ gx, const float* __restrict__ whh_t, float* __restrict__ state,
                                 const float* __restrict__ init, float* __restrict__ h_out, float* __restrict__ c_out,
                                 float* __restrict__ act_out, const int32_t* __restrict__ lengths, const KtStreamMask m,
                                 int rows, int H, int gx_pitch, int h_pitch) {
  extern __shared__ float sm[];
  const int G = 4 * H, tid = threadIdx.x, b = blockIdx.x, d = blockIdx.y, D = gridDim.y;
  float* h = sm;             // [H]
  float* c = h + H;          // [H]
  float* gates = c + H;      // [4H]
  whh_t += (long long)d * H * G;
  int lo = 0, hi = rows, carry = 0;
  if (lengths) {
    hi = min(max(__ldg(lengths + b), 0), rows);
  } else if (m.lengths) {
    int uhi;
    stream_utterance_rows(m, b, lo, uhi);
    carry = lo < 0;
    lo = max(lo, 0);
  }
  float* s = state ? state + (long long)b * 2 * H : nullptr;
  const float* i0 = init ? init + ((long long)b * D + d) * 2 * H : nullptr;
  for (int j = tid; j < 2 * H; j += blockDim.x) sm[j] = carry ? s[j] : (i0 ? __ldg(i0 + j) : 0.f);
  for (int t = 0; t < rows; ++t) {
    if (t >= lo && t < hi) continue;
    const long long orow = ((long long)b * h_pitch + t) * D + d;
    for (int j = tid; j < H; j += blockDim.x) {
      h_out[orow * H + j] = 0.f;
      if (c_out) c_out[orow * H + j] = 0.f;
    }
  }
  __syncthreads();
  for (int n = 0; n < hi - lo; ++n) {
    const int t = d ? hi - 1 - n : lo + n;
    const long long row = ((long long)b * gx_pitch + t) * D + d;
    const float* g = gx + row * G;
    for (int j = tid; j < G; j += blockDim.x) {
      float acc = __ldg(g + j);
      for (int k = 0; k < H; ++k) acc = fmaf(__ldg(whh_t + (long long)k * G + j), h[k], acc);
      gates[j] = acc;
    }
    __syncthreads();
    const long long orow = ((long long)b * h_pitch + t) * D + d;
    float* out = h_out + orow * H;
    for (int j = tid; j < H; j += blockDim.x) {
      const float ig = sigmoid_f(gates[j]), fg = sigmoid_f(gates[H + j]), gg = tanhf(gates[2 * H + j]), og = sigmoid_f(gates[3 * H + j]);
      const float cn = fg * c[j] + ig * gg;
      const float hn = og * tanhf(cn);
      c[j] = cn;
      h[j] = hn;
      out[j] = hn;
      if (c_out) c_out[orow * H + j] = cn;
      if (act_out) {
        float* a = act_out + row * G;
        a[j] = ig;
        a[H + j] = fg;
        a[2 * H + j] = gg;
        a[3 * H + j] = og;
      }
    }
    __syncthreads();
  }
  if (s)
    for (int j = tid; j < 2 * H; j += blockDim.x) s[j] = sm[j];
}

static int launch_lstm_rows(const float* gx, const float* whh_t, float* state, const float* init, float* h, float* c,
                            float* acts, const int32_t* lengths, const KtStreamMask& m, int B, int dirs, int rows, int H,
                            int gx_pitch, int h_pitch, cudaStream_t st) {
  const int threads = std::min(1024, ((4 * H + 31) / 32) * 32);
  const size_t smem = (size_t)6 * H * sizeof(float);
  lstm_rows_kernel<<<dim3(B, dirs), threads, smem, st>>>(gx, whh_t, state, init, h, c, acts, lengths, m, rows, H,
                                                         gx_pitch, h_pitch);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

extern "C" int kt_lstm_stream_slots(const float* gx, const float* whh_t, float* state, float* h, const KtStreamMask* m,
                                    int32_t B, int32_t rows, int32_t H, int32_t gx_pitch, int32_t h_pitch, void* stream) {
  int rc = validate_stream_mask(m, "lstm_stream_slots");
  if (rc) return rc;
  KT_REQUIRE(gx && whh_t && state && h, "lstm_stream_slots: null pointer");
  KT_REQUIRE(B >= 1 && rows >= 1 && H >= 1 && H <= 256 && gx_pitch >= rows && h_pitch >= rows, "lstm_stream_slots: bad sizes");
  return launch_lstm_rows(gx, whh_t, state, nullptr, h, nullptr, nullptr, nullptr, *m, B, 1, rows, H, gx_pitch, h_pitch,
                          static_cast<cudaStream_t>(stream));
}

extern "C" int kt_blstm_ragged(const float* gx, const float* whh_t, const int32_t* lengths, float* h, int32_t B, int32_t L,
                               int32_t H, void* stream) {
  KT_REQUIRE(gx && whh_t && lengths && h, "blstm_ragged: null pointer");
  KT_REQUIRE(B >= 1 && L >= 1 && H >= 1 && H <= 256, "blstm_ragged: bad sizes");
  return launch_lstm_rows(gx, whh_t, nullptr, nullptr, h, nullptr, nullptr, lengths, KtStreamMask{}, B, 2, L, H, L, L,
                          static_cast<cudaStream_t>(stream));
}

extern "C" int kt_lstm_train_fwd(const float* gx, const float* whh_t, const int32_t* lengths, const float* init, float* h,
                                 float* c, float* acts, int32_t B, int32_t L, int32_t dirs, int32_t H, void* stream) {
  KT_REQUIRE(gx && whh_t && h, "lstm_train_fwd: null pointer");
  KT_REQUIRE(B >= 1 && L >= 1 && (dirs == 1 || dirs == 2) && H >= 1 && H <= 256,
             "lstm_train_fwd: bad sizes (batch %d, length %d, dirs %d, hidden %d)", B, L, dirs, H);
  return launch_lstm_rows(gx, whh_t, nullptr, init, h, c, acts, lengths, KtStreamMask{}, B, dirs, L, H, L, L,
                          static_cast<cudaStream_t>(stream));
}

// lstm_bwd_kernel: the backward recurrence of lstm_rows_kernel for one (item b = blockIdx.x, direction d = blockIdx.y), over
// the same rows [lo, hi) in the reverse of their forward order.  With t' the row before t in the forward order ((h, c) =
// init, or 0, there at the direction's first row), from the upstream dh[t] and dc[t] (dc optional) and the carried
// (dh_rec, dc_rec) of the row after:
//   dh = dh[t] + dh_rec;  dc = (dc_rec + dc[t]) + dh * o * (1 - tanh(c_t)^2)
//   dgates[t] = (dc * g * i (1 - i), dc * c_t' * f (1 - f), dc * i * (1 - g^2), dh * tanh(c_t) * o (1 - o))
//   dc_rec = dc * f;  dh_rec[k] = sum_j dgates[t][j] W_hh[j][k]
// The last sum runs as four partial sums over the gate blocks (one thread per (block, k), W_hh streamed from L2, coalesced
// over k), added in block order: a fixed order, so an item's rows depend on its own rows, its length and the weights only.
// Rows outside [lo, hi) get dgates = 0.  h_prev[t] = h[t'] (init's h, or 0, at the direction's first row; 0 outside [lo, hi)):
// the operand of the weight gradient dW_hh = sum_t dgates[t]^T h_prev[t].  dstate (optional, init's layout): the gradient
// of the initial (h, c), the (dh_rec, dc_rec) left after the direction's first row.
__global__ void lstm_bwd_kernel(const float* __restrict__ dh_out, const float* __restrict__ dc_out,
                                const float* __restrict__ whh, const int32_t* __restrict__ lengths,
                                const float* __restrict__ init, const float* __restrict__ h_in, const float* __restrict__ c_in,
                                const float* __restrict__ acts, float* __restrict__ dgates, float* __restrict__ h_prev,
                                float* __restrict__ dstate, int rows, int H) {
  extern __shared__ float sm[];
  const int G = 4 * H, tid = threadIdx.x, b = blockIdx.x, d = blockIdx.y, D = gridDim.y;
  float* dc = sm;            // [H]  dc_rec
  float* dg = dc + H;        // [4H] this row's gate gradients
  float* part = dg + G;      // [4H] partial sums of dh_rec, one H block per gate block
  whh += (long long)d * G * H;
  const int hi = lengths ? min(max(__ldg(lengths + b), 0), rows) : rows;
  const long long sbase = ((long long)b * D + d) * 2 * H;
  const float* i0 = init ? init + sbase : nullptr;
  for (int j = tid; j < H; j += blockDim.x) dc[j] = 0.f;
  for (int j = tid; j < G; j += blockDim.x) part[j] = 0.f;
  for (int t = hi; t < rows; ++t) {
    const long long row = ((long long)b * rows + t) * D + d;
    for (int j = tid; j < G; j += blockDim.x) dgates[row * G + j] = 0.f;
    for (int j = tid; j < H; j += blockDim.x) h_prev[row * H + j] = 0.f;
  }
  __syncthreads();
  for (int n = 0; n < hi; ++n) {
    const int t = d ? n : hi - 1 - n;
    const int tp = d ? t + 1 : t - 1;
    const bool first = d ? tp >= hi : tp < 0;
    const long long row = ((long long)b * rows + t) * D + d, prow = ((long long)b * rows + tp) * D + d;
    const float* a = acts + row * G;
    for (int j = tid; j < H; j += blockDim.x) {
      const float dh = __ldg(dh_out + row * H + j) + (((part[j] + part[H + j]) + part[2 * H + j]) + part[3 * H + j]);
      const float ig = __ldg(a + j), fg = __ldg(a + H + j), gg = __ldg(a + 2 * H + j), og = __ldg(a + 3 * H + j);
      const float tc = tanhf(__ldg(c_in + row * H + j));
      const float cp = first ? (i0 ? __ldg(i0 + H + j) : 0.f) : __ldg(c_in + prow * H + j);
      const float dcn = fmaf(dh * og, 1.f - tc * tc, dc_out ? dc[j] + __ldg(dc_out + row * H + j) : dc[j]);
      const float gi = dcn * gg * (ig * (1.f - ig)), gf = dcn * cp * (fg * (1.f - fg));
      const float gc = dcn * ig * (1.f - gg * gg), go = dh * tc * (og * (1.f - og));
      dc[j] = dcn * fg;
      dg[j] = gi;
      dg[H + j] = gf;
      dg[2 * H + j] = gc;
      dg[3 * H + j] = go;
      float* o = dgates + row * G;
      o[j] = gi;
      o[H + j] = gf;
      o[2 * H + j] = gc;
      o[3 * H + j] = go;
      h_prev[row * H + j] = first ? (i0 ? __ldg(i0 + j) : 0.f) : __ldg(h_in + prow * H + j);
    }
    __syncthreads();
    for (int e = tid; e < G; e += blockDim.x) {
      const int q = e / H, k = e - q * H;
      float acc = 0.f;
      for (int j = q * H; j < (q + 1) * H; ++j) acc = fmaf(__ldg(whh + (long long)j * H + k), dg[j], acc);
      part[e] = acc;
    }
    __syncthreads();
  }
  if (dstate)
    for (int j = tid; j < H; j += blockDim.x) {
      dstate[sbase + j] = ((part[j] + part[H + j]) + part[2 * H + j]) + part[3 * H + j];
      dstate[sbase + H + j] = dc[j];
    }
}

extern "C" int kt_lstm_train_bwd(const float* dh, const float* dc, const float* whh, const int32_t* lengths,
                                 const float* init, const float* h, const float* c, const float* acts, float* dgates,
                                 float* h_prev, float* dstate, int32_t B, int32_t L, int32_t dirs, int32_t H, void* stream) {
  KT_REQUIRE(dh && whh && h && c && acts && dgates && h_prev, "lstm_train_bwd: null pointer");
  KT_REQUIRE(B >= 1 && L >= 1 && (dirs == 1 || dirs == 2) && H >= 1 && H <= 256,
             "lstm_train_bwd: bad sizes (batch %d, length %d, dirs %d, hidden %d)", B, L, dirs, H);
  const int threads = std::min(1024, ((4 * H + 31) / 32) * 32);
  const size_t smem = (size_t)9 * H * sizeof(float);
  lstm_bwd_kernel<<<dim3(B, dirs), threads, smem, static_cast<cudaStream_t>(stream)>>>(dh, dc, whh, lengths, init, h, c, acts,
                                                                                       dgates, h_prev, dstate, L, H);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

// ---------------------------------------------------------------------------------------------
// Per-slot free-running decoder step of MultiHeadPNCAAttention (sambert.SlotDecoder): every slot b at its own step
// s = step[b], with its own bands and memory length, all read on the device.  One CTA of two warps per (head, slot):
//   warp 0  writes the step's self K / V row into x_kv at s and attends self keys [max(0, s - x_bw[b]), s]; key s is read
//           from q_row, never from the row this launch writes, and every key / value is loaded with ld.global.cg (L2,
//           coherent), not through the read-only path, since the cache is written in this launch
//   warp 1  attends memory keys [s, min(s + h_bw[b], mem_len[b] - 1)] of h_kv
// Only the band's keys are read (the masked step path scans all Lmax keys).  Each lane takes keys j = lo + lane, lo + lane +
// 32, ...: the scores' max, then p = exp(score - max) summed into the lane's D accumulators, then one butterfly per
// accumulator.  An inactive slot (or one outside its memory) writes zero outputs and leaves its cache untouched.
// ---------------------------------------------------------------------------------------------
template <int D>
__global__ void __launch_bounds__(64) pnca_step_slots_kernel(const float* __restrict__ q_row, float* x_kv,
                                                             const float* __restrict__ h_kv, const int* __restrict__ step,
                                                             const int* __restrict__ mem_len, const int* __restrict__ x_bw,
                                                             const int* __restrict__ h_bw, const uint8_t* __restrict__ active,
                                                             float* __restrict__ out_x, float* __restrict__ out_h, int H,
                                                             int max_steps, float scale) {
  const int head = blockIdx.x, b = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int hd = H * D;
  const int s = __ldg(step + b), ml = __ldg(mem_len + b);
  float* out = (warp ? out_h : out_x) + (long long)b * hd + head * D;
  const bool live = __ldg(active + b) && s >= 0 && s < max_steps && s < ml;
  if (!live) {
    if (lane < D) out[lane] = 0.f;
    return;
  }
  const float* q = q_row + (long long)b * 3 * hd + head * D;
  const float* kv;
  int lo, hi;
  if (warp == 0) {
    float* row = x_kv + ((long long)b * max_steps + s) * 2 * hd + head * D;
    if (lane < D) {
      row[lane] = __ldg(q + hd + lane);
      row[hd + lane] = __ldg(q + 2 * hd + lane);
    }
    kv = x_kv + (long long)b * max_steps * 2 * hd + head * D;
    lo = max(0, s - __ldg(x_bw + b));
    hi = s;
  } else {
    kv = h_kv + (long long)b * max_steps * 2 * hd + head * D;
    lo = s;
    hi = min(s + __ldg(h_bw + b), ml - 1);
  }
  float qr[D];
#pragma unroll
  for (int d = 0; d < D; ++d) qr[d] = __ldg(q + d) * scale;
  // key j's K at k[0, D) and V at k[hd, hd + D): a cache row, or for the self key s the step's K | V in q_row
  const int own = warp == 0 ? s : -1;
  float m = -INFINITY;
  for (int j = lo + lane; j <= hi; j += 32) {
    const float* k = j == own ? q + hd : kv + (long long)j * 2 * hd;
    float sc = 0.f;
#pragma unroll
    for (int d = 0; d < D; ++d) sc = fmaf(qr[d], __ldcg(k + d), sc);
    m = fmaxf(m, sc);
  }
  m = warp_max(m);
  float acc[D], l = 0.f;
#pragma unroll
  for (int d = 0; d < D; ++d) acc[d] = 0.f;
  for (int j = lo + lane; j <= hi; j += 32) {
    const float* k = j == own ? q + hd : kv + (long long)j * 2 * hd;
    float sc = 0.f;
#pragma unroll
    for (int d = 0; d < D; ++d) sc = fmaf(qr[d], __ldcg(k + d), sc);
    const float p = expf(sc - m);
    l += p;
#pragma unroll
    for (int d = 0; d < D; ++d) acc[d] = fmaf(p, __ldcg(k + hd + d), acc[d]);
  }
  l = warp_sum(l);
  float mine = 0.f;
#pragma unroll
  for (int d = 0; d < D; ++d) {
    const float v = warp_sum(acc[d]);
    if (lane == d) mine = v;
  }
  if (lane < D) out[lane] = hi >= lo ? mine / l : 0.f;
}

extern "C" int kt_pnca_step_slots(const float* q_row, float* x_kv, const float* h_kv, const int32_t* step, const int32_t* mem_len,
                                  const int32_t* x_bw, const int32_t* h_bw, const uint8_t* active, float* out_x, float* out_h,
                                  int32_t B, int32_t H, int32_t d_head, int32_t max_steps, void* stream) {
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  KT_REQUIRE(q_row && x_kv && h_kv && step && mem_len && x_bw && h_bw && active && out_x && out_h,
             "pnca_step_slots: null pointer");
  KT_REQUIRE(B >= 1 && B <= 65535 && H >= 1 && H <= 65535 && max_steps >= 1, "pnca_step_slots: bad sizes");
  const dim3 grid(H, B);
  const float scale = 1.f / sqrtf((float)d_head);
  switch (d_head) {
    case 8: pnca_step_slots_kernel<8><<<grid, 64, 0, st>>>(q_row, x_kv, h_kv, step, mem_len, x_bw, h_bw, active, out_x, out_h, H, max_steps, scale); break;
    case 16: pnca_step_slots_kernel<16><<<grid, 64, 0, st>>>(q_row, x_kv, h_kv, step, mem_len, x_bw, h_bw, active, out_x, out_h, H, max_steps, scale); break;
    case 32: pnca_step_slots_kernel<32><<<grid, 64, 0, st>>>(q_row, x_kv, h_kv, step, mem_len, x_bw, h_bw, active, out_x, out_h, H, max_steps, scale); break;
    default: KT_REQUIRE(false, "pnca_step_slots: d_head must be 8, 16 or 32 (got %d)", d_head);
  }
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

}  // namespace kt
