// Weight re-parametrisation (weight_norm / plain-with-scale) fused with the layout change from
// the reference parameter layout to the kernel layouts of conv_ffma.cu / conv_tc.cu.
// Replaces torch._weight_norm + its backward (kantts/models/hifigan/layers.py:29,67,105,139).
#include <algorithm>

#include "common.cuh"

namespace kt {

// index of reference element (a, b, j) [shape (d0, d1, k)] in the two kernel layouts
struct WLayout {
  int d0, d1, k, transposed, groups;
  __device__ __forceinline__ void map(int a, int b, int j, long long& i_fwd, long long& i_bwd) const {
    if (!transposed) {  // a = co, b = ci_l
      const int cout = d0, cin_g = d1, cout_g = d0 / groups, cin = d1 * groups;
      const int gi = a / cout_g, co_l = a % cout_g;
      i_fwd = ((long long)j * cin_g + b) * cout + a;
      i_bwd = ((long long)j * cout_g + co_l) * cin + (long long)gi * cin_g + b;
    } else {  // a = ci, b = co
      const int cin = d0, cout = d1;
      i_fwd = ((long long)j * cin + a) * cout + b;
      i_bwd = ((long long)j * cout + b) * cin + a;
    }
  }
};

__device__ __forceinline__ float block_sum(float v, float* red) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = 0.f;
  for (int i = 0; i < (int)(blockDim.x >> 5); ++i) t += red[i];
  return t;
}

__global__ void weight_prepare_kernel(const float* __restrict__ v, const float* __restrict__ g,
                                      const float* __restrict__ inv_sigma, int mode, WLayout L,
                                      float* __restrict__ w_fwd, float* __restrict__ w_bwd,
                                      float* __restrict__ norm_out, float* __restrict__ w_ref) {
  __shared__ float red[8];
  const int a = blockIdx.x;
  const int n = L.d1 * L.k;
  const float* vs = v + (long long)a * n;
  float scale;
  if (mode == 1) {
    float ss = 0.f;
    for (int i = threadIdx.x; i < n; i += blockDim.x) { const float t = vs[i]; ss = fmaf(t, t, ss); }
    const float nrm = sqrtf(block_sum(ss, red));
    if (threadIdx.x == 0 && norm_out) norm_out[a] = nrm;
    scale = g[a] / nrm;
  } else {
    scale = inv_sigma ? *inv_sigma : 1.f;
  }
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int b = i / L.k, j = i % L.k;
    const float w = vs[i] * scale;
    long long i_fwd, i_bwd;
    L.map(a, b, j, i_fwd, i_bwd);
    if (w_fwd) w_fwd[i_fwd] = w;
    if (w_bwd) w_bwd[i_bwd] = w;
    if (w_ref) w_ref[(long long)a * n + i] = w;
  }
}

__global__ void weight_grad_kernel(const float* __restrict__ dw, const float* __restrict__ v,
                                   const float* __restrict__ g, const float* __restrict__ norm,
                                   const float* __restrict__ inv_sigma, int mode, WLayout L,
                                   float* __restrict__ dv, float* __restrict__ dg, int accumulate,
                                   const float* __restrict__ dbias_src, float* __restrict__ dbias_dst, int nbias) {
  __shared__ float red[8];
  const int a = blockIdx.x;
  const int n = L.d1 * L.k;
  if (dbias_dst) {   // bias gradient hand-over (+= into the parameter's .grad when accumulating)
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nbias; i += gridDim.x * blockDim.x)
      dbias_dst[i] = accumulate ? dbias_dst[i] + dbias_src[i] : dbias_src[i];
  }
  const float* vs = v + (long long)a * n;
  float* dvs = dv + (long long)a * n;
  if (mode == 1) {
    float dot = 0.f;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      long long i_fwd, i_bwd;
      L.map(a, i / L.k, i % L.k, i_fwd, i_bwd);
      dot = fmaf(dw[L.transposed ? i_bwd : i_fwd], vs[i], dot);
    }
    dot = block_sum(dot, red);
    const float nrm = norm[a], ga = g[a];
    if (threadIdx.x == 0) dg[a] = accumulate ? dg[a] + dot / nrm : dot / nrm;
    const float c1 = ga / nrm, c2 = ga * dot / (nrm * nrm * nrm);
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      long long i_fwd, i_bwd;
      L.map(a, i / L.k, i % L.k, i_fwd, i_bwd);
      const float r = c1 * dw[L.transposed ? i_bwd : i_fwd] - c2 * vs[i];
      dvs[i] = accumulate ? dvs[i] + r : r;
    }
  } else {
    const float scale = inv_sigma ? *inv_sigma : 1.f;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      long long i_fwd, i_bwd;
      L.map(a, i / L.k, i % L.k, i_fwd, i_bwd);
      // rounded before the accumulate (no fused multiply-add into dv): the sum is param.grad += grad of the plain kernel
      const float r = __fmul_rn(dw[L.transposed ? i_bwd : i_fwd], scale);
      dvs[i] = accumulate ? dvs[i] + r : r;
    }
  }
}

// ---- tiled variants for the large layers -----------------------------------------------------------------------------
// The kernels above give one CTA one row `a` of the reference tensor (d0, d1, k) and address the kernel layouts element by
// element: every 4-byte store / load of w_fwd / w_bwd / dw is its own 32-byte sector transaction (the kernel layouts are
// contiguous along a or along b, not along (b, j)): 55 us per 1024 x 1024 x 5 layer against ~10 us of traffic, 2.7 ms
// per train step between them (ablation, call r2aq).  Here a CTA owns 8 consecutive rows x one slice of b and moves them
// through a shared-memory tile: the reference layout is read / written along (b, j) by a warp per row, the a-contiguous
// layout 8 rows (= one sector) at a time, the b-contiguous layout 32 consecutive b per warp instruction.  Row reductions
// (norm, <dw, v>) are recomputed by every slice of a row (L2-resident re-reads) so that one launch suffices.
constexpr int kWA = 8;            // rows per CTA
constexpr int kWTile = 1024;      // tile floats per row (b-tile x k)
constexpr int kWPitch = kWTile + 4;   // bank = 4 * row + column for the 8 rows x 4 columns a warp touches

// the two kernel layouts of one layer as index forms:  A[(j * PA + b) * QA + a]   B[(j * PB + rowB(a)) * QB + offB(a) + b]
struct WForms {
  int PA, QA, PB, QB, cout_g, cin_g, transposed;
  __device__ __forceinline__ void rowB(int a, int& row, int& off) const {
    if (transposed) { row = a; off = 0; }
    else { const int gi = a / cout_g; row = a - gi * cout_g; off = gi * cin_g; }
  }
};
static WForms make_forms(const WLayout& L) {
  WForms f{};
  f.transposed = L.transposed;
  if (!L.transposed) { f.cout_g = L.d0 / L.groups; f.cin_g = L.d1; f.PA = L.d1; f.QA = L.d0; f.PB = f.cout_g; f.QB = L.d1 * L.groups; }
  else { f.cout_g = 1; f.cin_g = 0; f.PA = L.d1; f.QA = L.d0; f.PB = L.d0; f.QB = L.d1; }
  return f;
}

// a-contiguous array <-> tile[al][ib], ib = bl * k + j;  thread -> (al = t & 7, ib = t >> 3, +32, ...), (bl, j) carried incrementally
template <bool STORE>
__device__ __forceinline__ void wtile_formA(float (*tile)[kWPitch], float* arr, const float* carr, const WForms& f, int a0, int na, int b0,
                                            int bt, int k) {
  const int al = threadIdx.x & (kWA - 1);
  int ib = threadIdx.x >> 3;
  int bl = ib / k, j = ib - bl * k;
  const int dq = 32 / k, dr = 32 - dq * k;
  const int nib = bt * k;
  for (; ib < nib; ib += 32) {
    if (al < na) {
      const long long idx = ((long long)j * f.PA + (b0 + bl)) * f.QA + (a0 + al);
      if (STORE) arr[idx] = tile[al][ib];
      else tile[al][ib] = carr[idx];
    }
    bl += dq; j += dr;
    if (j >= k) { j -= k; ++bl; }
  }
}
// b-contiguous array <- tile; warp -> row al, lanes -> 32 consecutive b
__device__ __forceinline__ void wtile_storeB(float (*tile)[kWPitch], float* arr, const WForms& f, int a0, int na, int b0, int bt, int k) {
  const int al = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (al >= na) return;
  int row, off;
  f.rowB(a0 + al, row, off);
  for (int j = 0; j < k; ++j) {
    const long long base = ((long long)j * f.PB + row) * f.QB + off + b0;
    for (int bl = lane; bl < bt; bl += 32) arr[base + bl] = tile[al][bl * k + j];
  }
}

__global__ void __launch_bounds__(256) weight_prepare_tiled_kernel(const float* __restrict__ v, const float* __restrict__ g,
                                                                   const float* __restrict__ inv_sigma, int mode, WLayout L, WForms f,
                                                                   float* __restrict__ w_fwd, float* __restrict__ w_bwd,
                                                                   float* __restrict__ norm_out, float* __restrict__ w_ref, int b_slice) {
  __shared__ float tile[kWA][kWPitch];
  __shared__ float scale_s[kWA];
  const int a0 = blockIdx.x * kWA, na = min(kWA, L.d0 - a0);
  const int n = L.d1 * L.k;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp < na) {
    float scale;
    if (mode == 1) {
      const float* vs = v + (long long)(a0 + warp) * n;
      float ss = 0.f;
      for (int i = lane; i < n; i += 32) { const float t = vs[i]; ss = fmaf(t, t, ss); }
      for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
      const float nrm = sqrtf(ss);
      if (lane == 0 && norm_out && blockIdx.y == 0) norm_out[a0 + warp] = nrm;
      scale = g[a0 + warp] / nrm;
    } else {
      scale = inv_sigma ? *inv_sigma : 1.f;
    }
    if (lane == 0) scale_s[warp] = scale;
  }
  __syncthreads();
  float* arrA = L.transposed ? w_bwd : w_fwd;
  float* arrB = L.transposed ? w_fwd : w_bwd;
  const int bt_max = max(1, kWTile / L.k);
  const int b_begin = blockIdx.y * b_slice, b_end = min(L.d1, b_begin + b_slice);
  for (int b0 = b_begin; b0 < b_end; b0 += bt_max) {
    const int bt = min(bt_max, b_end - b0), nib = bt * L.k;
    if (warp < na) {
      const long long row = (long long)(a0 + warp) * n + (long long)b0 * L.k;
      const float sc = scale_s[warp];
      for (int i = lane; i < nib; i += 32) {
        const float w = v[row + i] * sc;
        tile[warp][i] = w;
        if (w_ref) w_ref[row + i] = w;
      }
    }
    __syncthreads();
    if (arrA) wtile_formA<true>(tile, arrA, nullptr, f, a0, na, b0, bt, L.k);
    if (arrB) wtile_storeB(tile, arrB, f, a0, na, b0, bt, L.k);
    __syncthreads();
  }
}

__global__ void __launch_bounds__(256) weight_grad_tiled_kernel(const float* __restrict__ dw, const float* __restrict__ v,
                                                                const float* __restrict__ g, const float* __restrict__ norm,
                                                                const float* __restrict__ inv_sigma, int mode, WLayout L, WForms f,
                                                                float* __restrict__ dv, float* __restrict__ dg, int accumulate,
                                                                const float* __restrict__ dbias_src, float* __restrict__ dbias_dst, int nbias,
                                                                int b_slice) {
  __shared__ float tile[kWA][kWPitch];   // dw of the current tile, transposed to the reference layout
  __shared__ float c1_s[kWA], c2_s[kWA];
  if (dbias_dst && blockIdx.y == 0) {   // bias gradient hand-over (+= into the parameter's .grad when accumulating)
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nbias; i += gridDim.x * blockDim.x)
      dbias_dst[i] = accumulate ? dbias_dst[i] + dbias_src[i] : dbias_src[i];
  }
  const int a0 = blockIdx.x * kWA, na = min(kWA, L.d0 - a0);
  const int n = L.d1 * L.k;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int bt_max = max(1, kWTile / L.k);
  if (mode == 1) {
    // pass 1 (whole row, every slice recomputes it): dot[a] = <dw[a, :], v[a, :]>
    float dot = 0.f;
    for (int b0 = 0; b0 < L.d1; b0 += bt_max) {
      const int bt = min(bt_max, L.d1 - b0);
      wtile_formA<false>(tile, nullptr, dw, f, a0, na, b0, bt, L.k);
      __syncthreads();
      if (warp < na) {
        const float* vs = v + (long long)(a0 + warp) * n + (long long)b0 * L.k;
        for (int i = lane; i < bt * L.k; i += 32) dot = fmaf(tile[warp][i], vs[i], dot);
      }
      __syncthreads();
    }
    for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
    if (warp < na && lane == 0) {
      const int a = a0 + warp;
      const float nrm = norm[a], ga = g[a];
      if (blockIdx.y == 0) dg[a] = accumulate ? dg[a] + dot / nrm : dot / nrm;
      c1_s[warp] = ga / nrm;
      c2_s[warp] = ga * dot / (nrm * nrm * nrm);
    }
  } else if (warp < na && lane == 0) {
    c1_s[warp] = inv_sigma ? *inv_sigma : 1.f;
    c2_s[warp] = 0.f;
  }
  __syncthreads();
  // pass 2 (this slice): dv[a, :] (+)= c1 * dw[a, :] - c2 * v[a, :]
  const int b_begin = blockIdx.y * b_slice, b_end = min(L.d1, b_begin + b_slice);
  for (int b0 = b_begin; b0 < b_end; b0 += bt_max) {
    const int bt = min(bt_max, b_end - b0);
    wtile_formA<false>(tile, nullptr, dw, f, a0, na, b0, bt, L.k);
    __syncthreads();
    if (warp < na) {
      const long long row = (long long)(a0 + warp) * n + (long long)b0 * L.k;
      const float c1 = c1_s[warp], c2 = c2_s[warp];
      for (int i = lane; i < bt * L.k; i += 32) {
        // (mode 0 rounds the product before the accumulate, as weight_grad_kernel does)
        const float r = mode == 1 ? c1 * tile[warp][i] - c2 * v[row + i] : __fmul_rn(c1, tile[warp][i]);
        dv[row + i] = accumulate ? dv[row + i] + r : r;
      }
    }
    __syncthreads();
  }
}

// tiled kernels for layers of >= 256 K elements with rows of >= 256 elements; -> (row blocks, b slices, b per slice)
static bool weight_tiled_plan(int d0, int d1, int k, int& nblk, int& nsl, int& b_slice) {
  if ((long long)d0 * d1 * k < 262144 || d1 * k < 256 || k > kWTile) return false;
  nblk = (d0 + kWA - 1) / kWA;
  nsl = std::max(1, std::min(std::max(1, d1 / 32), (296 + nblk - 1) / nblk));
  b_slice = ((d1 + nsl - 1) / nsl + 31) & ~31;
  nsl = (d1 + b_slice - 1) / b_slice;
  return true;
}

extern "C" int kt_weight_prepare(const float* v, const float* g, const float* inv_sigma, int32_t mode, int32_t d0, int32_t d1,
                                 int32_t k, int32_t transposed, int32_t groups, float* w_fwd, float* w_bwd, float* norm_out,
                                 float* w_ref, void* stream) {
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  KT_REQUIRE(v && d0 > 0 && d1 > 0 && k > 0 && groups > 0, "weight_prepare: bad arguments");
  KT_REQUIRE(mode == 0 || (mode == 1 && g && norm_out), "weight_prepare: mode 1 needs g and norm_out");
  KT_REQUIRE(!transposed || groups == 1, "weight_prepare: transposed conv must have groups == 1");
  KT_REQUIRE(transposed || d0 % groups == 0, "weight_prepare: d0 %% groups != 0");
  WLayout L{d0, d1, k, transposed, groups};
  int nblk, nsl, b_slice;
  if (weight_tiled_plan(d0, d1, k, nblk, nsl, b_slice))
    weight_prepare_tiled_kernel<<<dim3(nblk, nsl), 256, 0, st>>>(v, g, inv_sigma, mode, L, make_forms(L), w_fwd, w_bwd, norm_out, w_ref, b_slice);
  else
    weight_prepare_kernel<<<d0, 256, 0, st>>>(v, g, inv_sigma, mode, L, w_fwd, w_bwd, norm_out, w_ref);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

static int weight_grad(const float* dw, const float* v, const float* g, const float* norm, const float* inv_sigma,
                       int mode, int d0, int d1, int k, int transposed, int groups, float* dv, float* dg, int accumulate,
                       const float* dbias_src, float* dbias_dst, int nbias, cudaStream_t st) {
  KT_REQUIRE(dw && v && dv && d0 > 0 && d1 > 0 && k > 0 && groups > 0, "weight_grad: bad arguments");
  KT_REQUIRE(mode == 0 || (mode == 1 && g && norm && dg), "weight_grad: mode 1 needs g, norm, dg");
  WLayout L{d0, d1, k, transposed, groups};
  KT_REQUIRE((dbias_dst == nullptr) == (dbias_src == nullptr) && nbias >= 0, "weight_grad: dbias_src / dbias_dst must come together");
  int nblk, nsl, b_slice;
  if (weight_tiled_plan(d0, d1, k, nblk, nsl, b_slice)) {
    weight_grad_tiled_kernel<<<dim3(nblk, nsl), 256, 0, st>>>(dw, v, g, norm, inv_sigma, mode, L, make_forms(L), dv, dg, accumulate, dbias_src,
                                                               dbias_dst, nbias, b_slice);
  } else {
    weight_grad_kernel<<<d0, 256, 0, st>>>(dw, v, g, norm, inv_sigma, mode, L, dv, dg, accumulate, dbias_src, dbias_dst, nbias);
  }
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

extern "C" int kt_weight_grad(const float* dw_fwd, const float* v, const float* g, const float* norm, const float* inv_sigma,
                              int32_t mode, int32_t d0, int32_t d1, int32_t k, int32_t transposed, int32_t groups, float* dv,
                              float* dg, void* stream) {
  return weight_grad(dw_fwd, v, g, norm, inv_sigma, mode, d0, d1, k, transposed, groups, dv, dg, 0, nullptr, nullptr, 0,
                     static_cast<cudaStream_t>(stream));
}

extern "C" int kt_weight_grad_accum(const float* dw_fwd, const float* v, const float* g, const float* norm, const float* inv_sigma,
                                    int32_t mode, int32_t d0, int32_t d1, int32_t k, int32_t transposed, int32_t groups,
                                    float* dv, float* dg, const float* dbias_src, float* dbias_dst, int32_t nbias,
                                    void* stream) {
  return weight_grad(dw_fwd, v, g, norm, inv_sigma, mode, d0, d1, k, transposed, groups, dv, dg, 1, dbias_src, dbias_dst, nbias,
                     static_cast<cudaStream_t>(stream));
}

}  // namespace kt
