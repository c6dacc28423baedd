// Masked-symbol pretraining of the SAM-BERT text encoder (KanTtsTextsyBERT, sybert.yaml): the masked sequence
// cross-entropy SeqCELoss (kantts/train/loss.py:444-460) and the BERT masking of BERT_Text_Dataset.bert_masking /
// MaskingActor (kantts/datasets/dataset.py:873-1030) on the device.  The definitions are in include/kantts_b200.h
// (kt_seq_ce_fwd / _bwd, kt_bert_mask); oracle/sybert.py restates them.  Fixed-order reductions, no float atomics.
#include <math.h>

#include "common.cuh"
#include "philox.cuh"

namespace kt {

namespace {

constexpr int kCeWarps = 8;            // rows in flight per CTA, one warp each
constexpr int kCeMaxCtas = 512;        // the forward's grid, a function of `rows` only: the partials and their order are fixed
constexpr int kMaskThreads = 256;
constexpr int kMaskMaxSmem = 200 * 1024;    // dynamic shared memory of kt_bert_mask: up to 22755 positions
constexpr uint32_t kUtteranceDraw = 0xFFFFFFFFu;   // counter word 0 of the per-utterance replacement draw

__host__ __device__ inline int ce_ctas(int rows) {
  const int n = (rows + kCeWarps - 1) / kCeWarps;
  return n < 1 ? 1 : (n > kCeMaxCtas ? kCeMaxCtas : n);
}

// Online max / sum of exp of one row across the warp; (m, s) of every lane merged by a butterfly (all lanes get the same).
__device__ __forceinline__ void warp_merge_lse(float& m, float& s) {
  for (int o = 16; o > 0; o >>= 1) {
    const float m2 = __shfl_xor_sync(0xffffffffu, m, o), s2 = __shfl_xor_sync(0xffffffffu, s, o);
    const float mm = fmaxf(m, m2);
    const float a = (m == -INFINITY) ? 0.f : s * expf(m - mm);
    const float b = (m2 == -INFINITY) ? 0.f : s2 * expf(m2 - mm);
    m = mm;
    s = a + b;
  }
}

// The warp's (max, first index of the max): ties go to the smaller index, torch.argmax's rule.
__device__ __forceinline__ void warp_argmax(float& v, int& i) {
  for (int o = 16; o > 0; o >>= 1) {
    const float v2 = __shfl_xor_sync(0xffffffffu, v, o);
    const int i2 = __shfl_xor_sync(0xffffffffu, i, o);
    if (v2 > v || (v2 == v && i2 < i)) {
      v = v2;
      i = i2;
    }
  }
}

__device__ __forceinline__ double warp_sum_d(double v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Grid ce_ctas(rows) x kCeWarps warps; warp w of CTA c takes rows c * kCeWarps + w, stepping by the grid.  Per row: one pass
// of an online log-sum-exp and argmax, lse[row], then the row's masked loss and error into the warp's running sums.  The
// warps' sums are added in warp order into partials[c][3] (float64).
__global__ void __launch_bounds__(kCeWarps * 32) seq_ce_rows_kernel(const float* __restrict__ logits,
                                                                   const int64_t* __restrict__ targets,
                                                                   const float* __restrict__ masks, float* __restrict__ lse,
                                                                   double* __restrict__ partials, int rows, int v) {
  __shared__ double s_part[kCeWarps][3];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  double acc_loss = 0.0, acc_err = 0.0, acc_mask = 0.0;
  for (int r = blockIdx.x * kCeWarps + warp; r < rows; r += gridDim.x * kCeWarps) {
    const float* x = logits + (long long)r * v;
    float m = -INFINITY, s = 0.f, best = -INFINITY;
    int arg = 0x7fffffff;
    for (int j = lane; j < v; j += 32) {
      const float xj = __ldg(x + j);
      if (xj > best) {                       // ascending j per lane: the first index of the lane's max
        best = xj;
        arg = j;
      }
      if (xj > m) {
        s = (m == -INFINITY) ? 1.f : s * expf(m - xj) + 1.f;
        m = xj;
      } else {
        s += expf(xj - m);
      }
    }
    warp_merge_lse(m, s);
    warp_argmax(best, arg);
    const float row_lse = m + logf(s);
    const int64_t t = __ldg(targets + r);
    const float mk = __ldg(masks + r);
    // a target outside [0, v) has no logit: its loss is NaN, which the masked sum carries
    const float xt = (t >= 0 && t < v) ? __ldg(x + t) : __int_as_float(0x7fffffff);
    if (lane == 0) {
      lse[r] = row_lse;
      acc_loss += (double)(row_lse - xt) * (double)mk;
      acc_err += (arg != t) ? (double)mk : 0.0;
      acc_mask += (double)mk;
    }
  }
  if (lane == 0) {
    s_part[warp][0] = acc_loss;
    s_part[warp][1] = acc_err;
    s_part[warp][2] = acc_mask;
  }
  __syncthreads();
  if (threadIdx.x < 3) {
    double a = 0.0;
    for (int w = 0; w < kCeWarps; ++w) a += s_part[w][threadIdx.x];
    partials[(long long)blockIdx.x * 3 + threadIdx.x] = a;
  }
}

// One warp: the partials in a fixed order (lane l sums CTAs l, l + 32, ..., then a butterfly), then
// loss = sum loss / sum mask, err = sum error / sum mask and mask_sum in float32; 0 / 0 is NaN.
__global__ void seq_ce_reduce_kernel(const double* __restrict__ partials, int ctas, float* __restrict__ loss,
                                     float* __restrict__ err, float* __restrict__ mask_sum) {
  const int lane = threadIdx.x;
  double a[3] = {0.0, 0.0, 0.0};
  for (int c = lane; c < ctas; c += 32)
    for (int k = 0; k < 3; ++k) a[k] += partials[(long long)c * 3 + k];
  for (int k = 0; k < 3; ++k) a[k] = warp_sum_d(a[k]);
  if (lane == 0) {
    *loss = (float)(a[0] / a[2]);
    *err = (float)(a[1] / a[2]);
    *mask_sum = (float)a[2];
  }
}

// dlogits[r][j] = g_r (exp(x_j - lse_r) - [j == t_r]),  g_r = d_loss * mask_r / sum(mask).  One warp per row.
__global__ void __launch_bounds__(kCeWarps * 32) seq_ce_bwd_kernel(const float* __restrict__ logits,
                                                                  const int64_t* __restrict__ targets,
                                                                  const float* __restrict__ masks,
                                                                  const float* __restrict__ lse,
                                                                  const float* __restrict__ mask_sum,
                                                                  const float* __restrict__ d_loss,
                                                                  float* __restrict__ dlogits, int rows, int v) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float scale = __ldg(d_loss) / __ldg(mask_sum);
  for (int r = blockIdx.x * kCeWarps + warp; r < rows; r += gridDim.x * kCeWarps) {
    const float* x = logits + (long long)r * v;
    float* dx = dlogits + (long long)r * v;
    const float g = scale * __ldg(masks + r), l = __ldg(lse + r);
    const int64_t t = __ldg(targets + r);
    for (int j = lane; j < v; j += 32) {
      const float p = expf(__ldg(x + j) - l);
      dx[j] = g * (j == t ? p - 1.f : p);
    }
  }
}

// One CTA per utterance; see kt_bert_mask in include/kantts_b200.h for the decisions.  Shared memory: the rank key and the
// selection flag of every position.
__global__ void __launch_bounds__(kMaskThreads) bert_mask_kernel(const int64_t* __restrict__ lings,
                                                                const int32_t* __restrict__ valid_lengths,
                                                                int64_t* __restrict__ out_lings, int64_t* __restrict__ targets,
                                                                float* __restrict__ bert_masks, int length, int n_feat,
                                                                uint32_t k0, uint32_t k1, uint32_t call_lo, uint32_t call_hi,
                                                                long long threshold, int n_sy, int mask_id) {
  extern __shared__ unsigned long long s_key[];
  unsigned char* s_sel = reinterpret_cast<unsigned char*>(s_key + length);
  __shared__ int s_n, s_rand_id;
  const int b = blockIdx.x;
  const int valid = min(max(valid_lengths[b], 0), length);
  if (threadIdx.x == 0) {
    s_n = 0;
    const Philox4 r = philox4x32_10(Philox4{{kUtteranceDraw, (uint32_t)b, call_lo, call_hi}}, k0, k1);
    s_rand_id = (int)(((uint64_t)r.v[0] * (uint64_t)n_sy) >> 32);
  }
  __syncthreads();
  int mine = 0;
  for (int i = threadIdx.x; i < length; i += blockDim.x) {
    const Philox4 r = philox4x32_10(Philox4{{(uint32_t)i, (uint32_t)b, call_lo, call_hi}}, k0, k1);
    const bool sel = i < valid && (long long)r.v[0] < threshold;
    s_key[i] = ((unsigned long long)r.v[1] << 32) | r.v[2];
    s_sel[i] = sel;
    mine += sel;
  }
  atomicAdd(&s_n, mine);                     // an integer count: the same whatever the order
  __syncthreads();
  const int n = s_n;
  const int n_mask = (int)floor((double)n * 0.8);
  const int n_rand = (int)floor((double)n * 0.1);
  const long long row0 = (long long)b * length;
  for (int i = threadIdx.x; i < length; i += blockDim.x) {
    const int64_t* in = lings + (row0 + i) * n_feat;
    int64_t* out = out_lings + (row0 + i) * n_feat;
    const int64_t sy = in[0];
    int64_t masked = sy;
    if (s_sel[i]) {
      const unsigned long long key = s_key[i];
      int rank = 0;
      for (int j = 0; j < valid; ++j)
        rank += s_sel[j] && (s_key[j] < key || (s_key[j] == key && j < i));
      if (rank < n_mask)
        masked = mask_id;
      else if (rank < n_mask + n_rand)
        masked = s_rand_id;
    }
    out[0] = masked;
    for (int f = 1; f < n_feat; ++f) out[f] = in[f];
    targets[row0 + i] = sy;
    bert_masks[row0 + i] = s_sel[i] ? 1.f : 0.f;
  }
}

}  // namespace

extern "C" int64_t kt_seq_ce_workspace_bytes(int32_t rows) {
  return rows > 0 ? (int64_t)ce_ctas(rows) * 3 * (int64_t)sizeof(double) : 0;
}

extern "C" int kt_seq_ce_fwd(const float* logits, const int64_t* targets, const float* masks, float* lse, float* loss,
                             float* err, float* mask_sum, void* workspace, int64_t workspace_bytes, int32_t rows, int32_t v,
                             void* stream) {
  KT_REQUIRE(logits && targets && masks && lse && loss && err && mask_sum && workspace, "seq_ce_fwd: null argument");
  KT_REQUIRE(rows > 0 && v > 0, "seq_ce_fwd: rows %d, v %d", rows, v);
  KT_REQUIRE(workspace_bytes >= kt_seq_ce_workspace_bytes(rows), "seq_ce_fwd: workspace %lld bytes < %lld",
             (long long)workspace_bytes, (long long)kt_seq_ce_workspace_bytes(rows));
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int ctas = ce_ctas(rows);
  double* partials = static_cast<double*>(workspace);
  seq_ce_rows_kernel<<<ctas, kCeWarps * 32, 0, st>>>(logits, targets, masks, lse, partials, rows, v);
  KT_CHECK_CUDA(cudaGetLastError());
  seq_ce_reduce_kernel<<<1, 32, 0, st>>>(partials, ctas, loss, err, mask_sum);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

extern "C" int kt_seq_ce_bwd(const float* logits, const int64_t* targets, const float* masks, const float* lse,
                             const float* mask_sum, const float* d_loss, float* dlogits, int32_t rows, int32_t v,
                             void* stream) {
  KT_REQUIRE(logits && targets && masks && lse && mask_sum && d_loss && dlogits, "seq_ce_bwd: null argument");
  KT_REQUIRE(rows > 0 && v > 0, "seq_ce_bwd: rows %d, v %d", rows, v);
  seq_ce_bwd_kernel<<<ce_ctas(rows), kCeWarps * 32, 0, static_cast<cudaStream_t>(stream)>>>(
      logits, targets, masks, lse, mask_sum, d_loss, dlogits, rows, v);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

extern "C" int kt_bert_mask(const int64_t* lings, const int32_t* valid_lengths, int64_t* out_lings, int64_t* targets,
                            float* bert_masks, int32_t batch, int32_t length, int32_t n_feat, int64_t seed, int64_t call,
                            int64_t threshold, int32_t n_sy, int32_t mask_id, void* stream) {
  KT_REQUIRE(lings && valid_lengths && out_lings && targets && bert_masks, "bert_mask: null argument");
  KT_REQUIRE(batch > 0 && batch <= 65535 && length > 0 && n_feat > 0, "bert_mask: batch %d, length %d, n_feat %d", batch,
             length, n_feat);
  KT_REQUIRE(n_sy > 0 && threshold >= 0 && threshold <= (1LL << 32), "bert_mask: n_sy %d, threshold %lld", n_sy,
             (long long)threshold);
  const size_t smem = (size_t)length * (sizeof(unsigned long long) + 1);
  KT_REQUIRE(smem <= (size_t)kMaskMaxSmem, "bert_mask: length %d exceeds the shared-memory limit", length);
  KT_CHECK_CUDA(allow_dyn_smem<bert_mask_kernel>(kMaskMaxSmem));
  const uint64_t s = (uint64_t)seed, c = (uint64_t)call;
  bert_mask_kernel<<<batch, kMaskThreads, smem, static_cast<cudaStream_t>(stream)>>>(
      lings, valid_lengths, out_lings, targets, bert_masks, length, n_feat, (uint32_t)s, (uint32_t)(s >> 32), (uint32_t)c,
      (uint32_t)(c >> 32), (long long)threshold, n_sy, mask_id);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

}  // namespace kt
