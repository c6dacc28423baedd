// Single-input-channel convolutions: the first layer of every discriminator reads the mono waveform
// (PeriodDiscriminator convs[0]: Conv2d(1, 32, (5,1), (3,1)), hifigan.py:219-224; ScaleDiscriminator
// convs[0]: Conv1d(1, 128, 15), hifigan.py:328-334).  With C_in = 1 there is no contraction to feed a tensor
// core (K = 1 padded to 16 wastes >= 94 % of every MMA and the 128-row tiles are pure staging latency); the
// layer is a k-tap FIR per output channel and is bound by writing y (forward) / reading dy (weight gradient):
// bound: HBM.  Algorithmic bytes: forward 4*(rows_in + rows_out*C_out), weight gradient 4*(rows_in + rows_out*C_out
// [+ rows_out*C_out for y when act_out != NONE]).  Exact fp32.
#include <algorithm>

#include "common.cuh"

namespace kt {

constexpr int kThinMaxK = 16;

bool thin_cin1_ok(const KtConv1dDesc* d) {
  return !d->transposed && d->groups == 1 && d->c_in == 1 && d->upsample == 1 && d->act_in == KT_ACT_NONE &&
         d->kernel <= kThinMaxK && d->c_out >= 32 && d->c_out <= 256 && 256 % d->c_out == 0 && d->act_out != KT_ACT_TANH;
}

struct ThinParams {
  const float* x;    // [B][t_in][nsub]
  const float* w;    // [k][c_out]  (w_fwd layout with C_in = 1)
  const float* bias;
  const float* dy;   // [B][t_out][nsub][c_out]
  const float* y;    // forward output (act' of the fused output LeakyReLU)
  float* out;        // forward: y;  weight gradient: dw [k][c_out]
  float* dbias;
  // weight gradient: CTA b writes its partial sums to part + b * (k + 1) * c_out ([k][c_out] dw, then [c_out] dbias),
  // summed in CTA order afterwards (deterministic, unlike float atomics)
  float* part;
  int batch, nsub, t_in, t_out, c_out, k, stride, dil, pad, act;
  float slope;
};

// thread = (output row, 4 output channels); the k input samples of a row are shared by its C_out/4 threads (L1 hits)
__global__ void __launch_bounds__(256) thin_cin1_fwd_kernel(const ThinParams p) {
  extern __shared__ float w_s[];   // [k][c_out] + [c_out] bias
  float* b_s = w_s + p.k * p.c_out;
  for (int i = threadIdx.x; i < p.k * p.c_out; i += blockDim.x) w_s[i] = p.w[i];
  for (int i = threadIdx.x; i < p.c_out; i += blockDim.x) b_s[i] = p.bias ? p.bias[i] : 0.f;
  __syncthreads();
  // thread -> fixed channel quad; rows advance by a constant stride, so (b, to, w) is carried incrementally
  // (no per-element integer division: the 64-bit div/mod sequence cost more than the FIR itself)
  const unsigned c4n = (unsigned)p.c_out >> 2;
  const unsigned nthreads = gridDim.x * blockDim.x;           // host guarantees nthreads % c4n == 0
  const unsigned gtid = blockIdx.x * blockDim.x + threadIdx.x;
  const int c = (int)(gtid % c4n) * 4;
  const unsigned rstep = nthreads / c4n;
  const unsigned rows = (unsigned)p.batch * p.t_out * p.nsub;
  const unsigned tn = (unsigned)p.t_out * p.nsub;
  const unsigned step_b = rstep / tn, step_r = rstep % tn;    // row stride split into (batch items, remainder)
  unsigned row = gtid / c4n;
  unsigned b = row / tn, rem = row % tn;                      // rem = to * nsub + w
  for (; row < rows; row += rstep) {
    const int to = (int)(rem / (unsigned)p.nsub), w = (int)(rem % (unsigned)p.nsub);
    float4 acc = *reinterpret_cast<const float4*>(b_s + c);
    const float* xb = p.x + (long long)b * p.t_in * p.nsub + w;
#pragma unroll 5
    for (int j = 0; j < p.k; ++j) {
      const int ti = to * p.stride + j * p.dil - p.pad;
      if (ti >= 0 && ti < p.t_in) {
        const float xv = __ldg(xb + (long long)ti * p.nsub);
        const float4 wv = *reinterpret_cast<const float4*>(w_s + j * p.c_out + c);
        acc.x = fmaf(xv, wv.x, acc.x); acc.y = fmaf(xv, wv.y, acc.y);
        acc.z = fmaf(xv, wv.z, acc.z); acc.w = fmaf(xv, wv.w, acc.w);
      }
    }
    if (p.act == KT_ACT_LRELU) {
      acc.x = acc.x > 0.f ? acc.x : acc.x * p.slope; acc.y = acc.y > 0.f ? acc.y : acc.y * p.slope;
      acc.z = acc.z > 0.f ? acc.z : acc.z * p.slope; acc.w = acc.w > 0.f ? acc.w : acc.w * p.slope;
    }
    *reinterpret_cast<float4*>(p.out + (long long)row * p.c_out + c) = acc;
    b += step_b; rem += step_r;
    if (rem >= tn) { rem -= tn; ++b; }
  }
}

// dW[j][co] = sum_rows x[row -> tap j] * dpre[row][co],  dbias[co] = sum_rows dpre[row][co],  dpre = dy * act'(y).
// thread = (channel c = tid % C_out, row slot = tid / C_out); a CTA walks a contiguous row range, a warp reads
// 128 contiguous bytes of dy per row; the k input samples of a row are warp-uniform loads.  Per-CTA partial sums
// are reduced in shared memory and written to the CTA's slot of p.part ((k+1)*C_out floats).
__global__ void __launch_bounds__(256) thin_cin1_wgrad_kernel(const ThinParams p, long long rows_per_cta) {
  __shared__ float red[256 * (kThinMaxK + 1)];
  const int c = threadIdx.x % p.c_out, slot = threadIdx.x / p.c_out, nslots = 256 / p.c_out;
  const long long rows = (long long)p.batch * p.t_out * p.nsub;
  const long long r_begin = blockIdx.x * rows_per_cta, r_end = min(rows, r_begin + rows_per_cta);
  float acc[kThinMaxK + 1];
#pragma unroll
  for (int j = 0; j <= kThinMaxK; ++j) acc[j] = 0.f;
  const unsigned tn = (unsigned)p.t_out * p.nsub;
  constexpr int UR = 8;   // rows in flight per thread (the loop is otherwise one dependent global load per row)
  for (long long row0 = r_begin + slot; row0 < r_end; row0 += (long long)nslots * UR) {
    float g[UR], yv[UR];
#pragma unroll
    for (int u = 0; u < UR; ++u) {
      const long long row = row0 + (long long)u * nslots;
      const bool ok = row < r_end;
      g[u] = ok ? __ldg(p.dy + row * p.c_out + c) : 0.f;
      yv[u] = (ok && p.act == KT_ACT_LRELU) ? __ldg(p.y + row * p.c_out + c) : 1.f;
    }
#pragma unroll
    for (int u = 0; u < UR; ++u) {
      const long long row = row0 + (long long)u * nslots;
      if (row >= r_end) continue;
      const float gu = yv[u] > 0.f ? g[u] : g[u] * p.slope;
      const unsigned r32 = (unsigned)row;
      const unsigned bq = r32 / tn, rem = r32 - bq * tn;
      const int to = (int)(rem / (unsigned)p.nsub), w = (int)(rem - (unsigned)to * p.nsub);
      const float* xb = p.x + (long long)bq * p.t_in * p.nsub + w;
#pragma unroll
      for (int j = 0; j < kThinMaxK; ++j) {
        if (j < p.k) {
          const int ti = to * p.stride + j * p.dil - p.pad;
          const float xv = (ti >= 0 && ti < p.t_in) ? __ldg(xb + (long long)ti * p.nsub) : 0.f;
          acc[j] = fmaf(xv, gu, acc[j]);
        }
      }
      acc[kThinMaxK] += gu;
    }
  }
  // reduce the row slots: red[j][slot][c]
#pragma unroll
  for (int j = 0; j <= kThinMaxK; ++j) red[j * 256 + threadIdx.x] = acc[j];
  __syncthreads();
  for (int i = threadIdx.x; i < (p.k + 1) * p.c_out; i += blockDim.x) {
    const int j = i / p.c_out, cc = i % p.c_out;
    const int jj = j < p.k ? j : kThinMaxK;
    float s = 0.f;
    for (int q = 0; q < nslots; ++q) s += red[jj * 256 + q * p.c_out + cc];
    p.part[(long long)blockIdx.x * (p.k + 1) * p.c_out + i] = s;
  }
}

// ---- the scale discriminator's first layer (Conv1d(1, 128, 15), stride 1, one sub-sequence) ---------------------------------
// The generic kernels above re-read the k taps' weights from shared memory (forward: 15 LDS.128 per output quad, ~1 GB of
// shared-memory traffic per launch) or the k input samples (weight gradient: 15 loads per element) for every output row:
// 91 us / 292 us per B = 16 launch against 11 us / 22 us of HBM time (call r2ak).  Here a WARP owns a run of consecutive
// rows of one item and a lane owns one channel quad for the whole kernel: weights (forward) / gradient accumulators
// (weight gradient) live in registers, the input window of a block of 8 rows is 8 + k - 1 warp-uniform loads.
constexpr int kThinRW = 64;   // rows per warp task
constexpr int kThinUR = 8;    // rows per register block

template <int K>
__global__ void __launch_bounds__(256) thin_c128_fwd_kernel(const ThinParams p) {
  const int lane = threadIdx.x & 31, c = lane * 4;
  const int gwarp = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), nwarps = (int)((gridDim.x * blockDim.x) >> 5);
  float4 w[K];
#pragma unroll
  for (int j = 0; j < K; ++j) w[j] = __ldg(reinterpret_cast<const float4*>(p.w + j * 128 + c));
  const float4 bv = p.bias ? __ldg(reinterpret_cast<const float4*>(p.bias + c)) : make_float4(0.f, 0.f, 0.f, 0.f);
  const int tasks_item = (p.t_out + kThinRW - 1) / kThinRW;
  for (int task = gwarp; task < p.batch * tasks_item; task += nwarps) {
    const int b = task / tasks_item, t0 = (task - b * tasks_item) * kThinRW;
    const float* xb = p.x + (long long)b * p.t_in;
    float* ob = p.out + ((long long)b * p.t_out) * 128 + c;
    const int t1 = min(p.t_out, t0 + kThinRW);
    for (int tb = t0; tb < t1; tb += kThinUR) {
      float xw[kThinUR + K - 1];
#pragma unroll
      for (int i = 0; i < kThinUR + K - 1; ++i) {
        const int ti = tb - p.pad + i;
        xw[i] = (ti >= 0 && ti < p.t_in) ? __ldg(xb + ti) : 0.f;
      }
#pragma unroll
      for (int u = 0; u < kThinUR; ++u) {
        if (tb + u < t1) {
          float4 acc = bv;
#pragma unroll
          for (int j = 0; j < K; ++j) {
            acc.x = fmaf(xw[u + j], w[j].x, acc.x); acc.y = fmaf(xw[u + j], w[j].y, acc.y);
            acc.z = fmaf(xw[u + j], w[j].z, acc.z); acc.w = fmaf(xw[u + j], w[j].w, acc.w);
          }
          if (p.act == KT_ACT_LRELU) {
            acc.x = acc.x > 0.f ? acc.x : acc.x * p.slope; acc.y = acc.y > 0.f ? acc.y : acc.y * p.slope;
            acc.z = acc.z > 0.f ? acc.z : acc.z * p.slope; acc.w = acc.w > 0.f ? acc.w : acc.w * p.slope;
          }
          *reinterpret_cast<float4*>(ob + (long long)(tb + u) * 128) = acc;
        }
      }
    }
  }
}

template <int K>
__global__ void __launch_bounds__(256) thin_c128_wgrad_kernel(const ThinParams p) {
  __shared__ float4 red[4][K + 1][32];   // two rounds: warps 4-7 -> 0-3, then 0-3 -> the CTA's slot of p.part
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, c = lane * 4;
  const int gwarp = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), nwarps = (int)((gridDim.x * blockDim.x) >> 5);
  float4 acc[K + 1];
#pragma unroll
  for (int j = 0; j <= K; ++j) acc[j] = make_float4(0.f, 0.f, 0.f, 0.f);
  const int tasks_item = (p.t_out + kThinRW - 1) / kThinRW;
  for (int task = gwarp; task < p.batch * tasks_item; task += nwarps) {
    const int b = task / tasks_item, t0 = (task - b * tasks_item) * kThinRW;
    const float* xb = p.x + (long long)b * p.t_in;
    const long long rb = ((long long)b * p.t_out) * 128 + c;
    const int t1 = min(p.t_out, t0 + kThinRW);
    for (int tb = t0; tb < t1; tb += kThinUR) {
      float4 g[kThinUR];
#pragma unroll
      for (int u = 0; u < kThinUR; ++u) {
        const bool ok = tb + u < t1;
        g[u] = ok ? __ldg(reinterpret_cast<const float4*>(p.dy + rb + (long long)(tb + u) * 128)) : make_float4(0.f, 0.f, 0.f, 0.f);
        if (ok && p.act == KT_ACT_LRELU) {
          const float4 yv = __ldg(reinterpret_cast<const float4*>(p.y + rb + (long long)(tb + u) * 128));
          g[u].x = yv.x > 0.f ? g[u].x : g[u].x * p.slope; g[u].y = yv.y > 0.f ? g[u].y : g[u].y * p.slope;
          g[u].z = yv.z > 0.f ? g[u].z : g[u].z * p.slope; g[u].w = yv.w > 0.f ? g[u].w : g[u].w * p.slope;
        }
      }
      float xw[kThinUR + K - 1];
#pragma unroll
      for (int i = 0; i < kThinUR + K - 1; ++i) {
        const int ti = tb - p.pad + i;
        xw[i] = (ti >= 0 && ti < p.t_in) ? __ldg(xb + ti) : 0.f;
      }
#pragma unroll
      for (int u = 0; u < kThinUR; ++u) {
#pragma unroll
        for (int j = 0; j < K; ++j) {
          acc[j].x = fmaf(xw[u + j], g[u].x, acc[j].x); acc[j].y = fmaf(xw[u + j], g[u].y, acc[j].y);
          acc[j].z = fmaf(xw[u + j], g[u].z, acc[j].z); acc[j].w = fmaf(xw[u + j], g[u].w, acc[j].w);
        }
        acc[K].x += g[u].x; acc[K].y += g[u].y; acc[K].z += g[u].z; acc[K].w += g[u].w;
      }
    }
  }
  if (warp >= 4) {
#pragma unroll
    for (int j = 0; j <= K; ++j) red[warp - 4][j][lane] = acc[j];
  }
  __syncthreads();
  if (warp < 4) {
#pragma unroll
    for (int j = 0; j <= K; ++j) {
      const float4 o = red[warp][j][lane];
      acc[j].x += o.x; acc[j].y += o.y; acc[j].z += o.z; acc[j].w += o.w;
    }
  }
  __syncthreads();
  if (warp < 4) {
#pragma unroll
    for (int j = 0; j <= K; ++j) red[warp][j][lane] = acc[j];
  }
  __syncthreads();
  for (int i = threadIdx.x; i < (K + 1) * 128; i += blockDim.x) {
    const int j = i >> 7, cc = i & 127;
    float s = 0.f;
#pragma unroll
    for (int q = 0; q < 4; ++q) s += reinterpret_cast<const float*>(&red[q][j][0])[cc];
    p.part[(long long)blockIdx.x * (K + 1) * 128 + i] = s;
  }
}

static bool thin_c128_ok(const KtConv1dDesc* d) {
  return d->nsub == 1 && d->stride == 1 && d->dilation == 1 && d->c_out == 128 && (d->kernel == 15 || d->kernel == 5 || d->kernel == 3);
}

int thin_cin1_fwd(const KtConv1dDesc* d, const float* x, const float* w_fwd, const float* bias, float* y, cudaStream_t st) {
  ThinParams p{};
  p.x = x; p.w = w_fwd; p.bias = bias; p.out = y;
  p.batch = d->batch; p.nsub = d->nsub; p.t_in = d->t_in; p.t_out = d->t_out; p.c_out = d->c_out; p.k = d->kernel;
  p.stride = d->stride; p.dil = d->dilation; p.pad = d->pad_left; p.act = d->act_out; p.slope = d->act_out_slope;
  const long long total = (long long)d->batch * d->t_out * d->nsub * (d->c_out / 4);
  KT_REQUIRE(total < (1LL << 31), "thin_cin1_fwd: tensor too large for 32-bit row indexing");
  if (thin_c128_ok(d)) {
    const long long tasks = (long long)d->batch * ((d->t_out + kThinRW - 1) / kThinRW);
    const int blocks = (int)std::max<long long>(1, std::min<long long>((tasks + 7) / 8, 148LL * 4));
    if (d->kernel == 15) thin_c128_fwd_kernel<15><<<blocks, 256, 0, st>>>(p);
    else if (d->kernel == 5) thin_c128_fwd_kernel<5><<<blocks, 256, 0, st>>>(p);
    else thin_c128_fwd_kernel<3><<<blocks, 256, 0, st>>>(p);
    KT_CHECK_CUDA(cudaGetLastError());
    return KT_OK;
  }
  const int blocks = (int)std::max<long long>(1, std::min<long long>((total + 255) / 256, 148LL * 16));   // 256 % (c_out/4) == 0
  const size_t smem = (size_t)(d->kernel + 1) * d->c_out * sizeof(float);
  thin_cin1_fwd_kernel<<<blocks, 256, smem, st>>>(p);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

int thin_cin1_wgrad(const KtConv1dDesc* d, const float* x, const float* dy, const float* y, float* dw, float* dbias,
                    cudaStream_t st) {
  ThinParams p{};
  p.x = x; p.dy = dy; p.y = y; p.out = dw; p.dbias = dbias;
  p.batch = d->batch; p.nsub = d->nsub; p.t_in = d->t_in; p.t_out = d->t_out; p.c_out = d->c_out; p.k = d->kernel;
  p.stride = d->stride; p.dil = d->dilation; p.pad = d->pad_left; p.act = d->act_out; p.slope = d->act_out_slope;
  KT_REQUIRE((long long)d->batch * d->t_out * d->nsub < (1LL << 31), "thin_cin1_wgrad: tensor too large for 32-bit row indexing");
  const long long slot = (long long)(d->kernel + 1) * d->c_out;
  const bool c128 = thin_c128_ok(d);
  long long ctas, rows_per_cta = 0;
  if (c128) {
    const long long tasks = (long long)d->batch * ((d->t_out + kThinRW - 1) / kThinRW);
    ctas = std::max<long long>(1, std::min<long long>((tasks + 7) / 8, 132LL));
  } else {
    const long long rows = (long long)d->batch * d->t_out * d->nsub;
    const int nslots = 256 / d->c_out;
    ctas = std::min<long long>(132LL * 4, std::max<long long>(1, rows / (nslots * 32LL)));
    rows_per_cta = (rows + ctas - 1) / ctas;
    ctas = (rows + rows_per_cta - 1) / rows_per_cta;
  }
  int rc = scratch_alloc(&p.part, ctas * slot, st);
  if (rc) return rc;
  if (c128) {
    if (d->kernel == 15) thin_c128_wgrad_kernel<15><<<(int)ctas, 256, 0, st>>>(p);
    else if (d->kernel == 5) thin_c128_wgrad_kernel<5><<<(int)ctas, 256, 0, st>>>(p);
    else thin_c128_wgrad_kernel<3><<<(int)ctas, 256, 0, st>>>(p);
  } else {
    thin_cin1_wgrad_kernel<<<(int)ctas, 256, 0, st>>>(p, rows_per_cta);
  }
  KT_CHECK_CUDA(cudaGetLastError());
  rc = split_sum(p.part, (long long)d->kernel * d->c_out, (int)ctas, slot, dw, false, st);
  if (!rc && dbias) rc = split_sum(p.part + (long long)d->kernel * d->c_out, d->c_out, (int)ctas, slot, dbias, false, st);
  if (rc) return rc;
  return scratch_free(p.part, st);
}

}  // namespace kt
