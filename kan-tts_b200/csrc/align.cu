// Alignment learning of SAM-BERT with monotonic alignment search (MAS: True, sambert_16k_MAS*.yaml): the distance attention
// of ConvAttention (kantts/models/sambert/attention.py:85-125), the width-1 MAS of alignment.py:32-71 and the forward-sum
// loss of AttentionCTCLoss (kantts/train/loss.py:481-508).  Exact fp32 on CUDA cores (the forward-sum recursions in float64),
// fixed-order reductions, no atomics.
// Also the beta-binomial alignment prior of the data path (kantts/datasets/dataset.py:20-31), evaluated in float64.
#include <math.h>

#include "common.cuh"

namespace kt {

namespace {

constexpr int kAttnRows = 8;         // query rows per CTA, one warp each
constexpr int kAttnKeys = 32;        // keys per shared-memory tile, one lane each
constexpr int kAttnMaxC = 128;       // channels: at most 4 per lane
constexpr float kDistScale = -0.0005f;

__device__ __forceinline__ float warp_sum(float v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ float warp_max(float v) {
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Row stride of a key tile in shared memory: odd, so that lane j reading channel c of key j hits distinct banks.
__host__ __device__ inline int tile_stride(int c) { return c | 1; }

// Stage keys [j0, j0 + 32) of one utterance (zeros past t_k) into `ks`; the caller synchronises.
__device__ __forceinline__ void load_key_tile(const float* __restrict__ kb, int j0, int t_k, int c, float* ks) {
  const int ldk = tile_stride(c);
  for (int e = threadIdx.x; e < kAttnKeys * c; e += blockDim.x) {
    const int jj = e / c, ch = e - jj * c;
    ks[jj * ldk + ch] = (j0 + jj < t_k) ? __ldg(kb + (long long)(j0 + jj) * c + ch) : 0.f;
  }
}

// z = -0.0005 sum_c (q_c - k_c)^2, summed over the channels in order
__device__ __forceinline__ float dist_logit(const float* qs, const float* kj, int c) {
  float s = 0.f;
  for (int ch = 0; ch < c; ++ch) {
    const float d = qs[ch] - kj[ch];
    s = fmaf(d, d, s);
  }
  return kDistScale * s;
}

// One warp per query row (b, i): z over every key (into `logprob`, as scratch), then
//   a = prior ? z - logsumexp_j(z) + log(prior + 1e-8) : z        (the log_softmax over ALL t_k keys)
//   soft = softmax over the keys j < key_len of a, 0 on the others.
__global__ void __launch_bounds__(kAttnRows * 32) align_attn_fwd_kernel(
    const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ prior,
    const int32_t* __restrict__ key_len, float* __restrict__ logprob, float* __restrict__ soft, float* __restrict__ row_lse,
    int t_q, int t_k, int c) {
  extern __shared__ float smem[];
  float* ks = smem;                                   // [32][ldk]
  float* qs = smem + kAttnKeys * tile_stride(c);      // [kAttnRows][c]
  const int b = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i0 = blockIdx.x * kAttnRows, i = i0 + warp;
  const float* kb = k + (long long)b * t_k * c;
  for (int e = threadIdx.x; e < kAttnRows * c; e += blockDim.x) {
    const int r = e / c;
    qs[e] = (i0 + r < t_q) ? __ldg(q + ((long long)b * t_q + i0 + r) * c + (e - r * c)) : 0.f;
  }
  const long long row = ((long long)b * t_q + i) * t_k;
  for (int j0 = 0; j0 < t_k; j0 += kAttnKeys) {
    __syncthreads();
    load_key_tile(kb, j0, t_k, c, ks);
    __syncthreads();
    const int j = j0 + lane;
    if (i < t_q && j < t_k) logprob[row + j] = dist_logit(qs + warp * c, ks + lane * tile_stride(c), c);
  }
  if (i >= t_q) return;
  __syncwarp();
  float* lp = logprob + row;
  const float* pr = prior ? prior + row : nullptr;
  if (pr) {
    float m = -INFINITY;
    for (int j = lane; j < t_k; j += 32) m = fmaxf(m, lp[j]);
    m = warp_max(m);
    float s = 0.f;
    for (int j = lane; j < t_k; j += 32) s += expf(lp[j] - m);
    const float lse = m + logf(warp_sum(s));
    for (int j = lane; j < t_k; j += 32) lp[j] = (lp[j] - lse) + logf(__ldg(pr + j) + 1e-8f);
    if (lane == 0 && row_lse) row_lse[(long long)b * t_q + i] = lse;
    __syncwarp();
  }
  const int n = min(max(key_len[b], 1), t_k);
  float m = -INFINITY;
  for (int j = lane; j < n; j += 32) m = fmaxf(m, lp[j]);
  m = warp_max(m);
  float s = 0.f;
  for (int j = lane; j < n; j += 32) s += expf(lp[j] - m);
  const float inv = 1.f / warp_sum(s);
  float* so = soft + row;
  for (int j = lane; j < t_k; j += 32) so[j] = j < n ? expf(lp[j] - m) * inv : 0.f;
}

// Backward, one warp per query row: with s = soft, g = d_soft, l = d_logprob,
//   da_j = l_j + s_j (g_j - sum_j' s_j' g_j')                (softmax backward; s = 0 on the masked keys)
//   dz_j = prior ? da_j - exp(z_j - lse) sum_j' da_j' : da_j  (log_softmax backward over all keys)
//   dq_c = -0.001 sum_j dz_j (q_c - k_jc), in key order; dz goes to `dz` for the per-key pass.
__global__ void __launch_bounds__(kAttnRows * 32) align_attn_bwd_rows_kernel(
    const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ prior,
    const float* __restrict__ soft, const float* __restrict__ row_lse, const float* __restrict__ d_soft,
    const float* __restrict__ d_logprob, float* __restrict__ dz, float* __restrict__ dq, int t_q, int t_k, int c) {
  extern __shared__ float smem[];
  float* ks = smem;
  float* qs = smem + kAttnKeys * tile_stride(c);
  float* zs = qs + kAttnRows * c;                     // [kAttnRows][32] this tile's dz per row
  const int b = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i0 = blockIdx.x * kAttnRows, i = i0 + warp;
  const bool live = i < t_q;
  const float* kb = k + (long long)b * t_k * c;
  for (int e = threadIdx.x; e < kAttnRows * c; e += blockDim.x) {
    const int r = e / c;
    qs[e] = (i0 + r < t_q) ? __ldg(q + ((long long)b * t_q + i0 + r) * c + (e - r * c)) : 0.f;
  }
  const long long row = ((long long)b * t_q + (live ? i : 0)) * t_k;
  float dot = 0.f, sum_da = 0.f;
  if (live && d_soft) {
    for (int j = lane; j < t_k; j += 32) dot = fmaf(__ldg(soft + row + j), __ldg(d_soft + row + j), dot);
    dot = warp_sum(dot);
  }
  auto da_at = [&](int j) {
    float v = d_logprob ? __ldg(d_logprob + row + j) : 0.f;
    if (d_soft) v += __ldg(soft + row + j) * (__ldg(d_soft + row + j) - dot);
    return v;
  };
  if (live && prior) {
    for (int j = lane; j < t_k; j += 32) sum_da += da_at(j);
    sum_da = warp_sum(sum_da);
  }
  const float lse = (live && prior) ? row_lse[(long long)b * t_q + i] : 0.f;
  float acc[kAttnMaxC / 32] = {0.f, 0.f, 0.f, 0.f};
  const float* qw = qs + warp * c;
  for (int j0 = 0; j0 < t_k; j0 += kAttnKeys) {
    __syncthreads();
    load_key_tile(kb, j0, t_k, c, ks);
    __syncthreads();
    const int j = j0 + lane;
    float d = 0.f;
    if (live && j < t_k) {
      d = da_at(j);
      if (prior) d -= expf(dist_logit(qw, ks + lane * tile_stride(c), c) - lse) * sum_da;
      dz[row + j] = d;
    }
    zs[warp * 32 + lane] = d;
    __syncwarp();
    const int nj = min(kAttnKeys, t_k - j0);
#pragma unroll
    for (int u = 0; u < kAttnMaxC / 32; ++u) {
      const int ch = lane + 32 * u;
      if (ch < c) {
        const float qc = qw[ch];
        for (int jj = 0; jj < nj; ++jj) acc[u] = fmaf(zs[warp * 32 + jj], qc - ks[jj * tile_stride(c) + ch], acc[u]);
      }
    }
    __syncwarp();
  }
  if (!live) return;
#pragma unroll
  for (int u = 0; u < kAttnMaxC / 32; ++u) {
    const int ch = lane + 32 * u;
    if (ch < c) dq[((long long)b * t_q + i) * c + ch] = -0.001f * acc[u];
  }
}

constexpr int kDkKeys = 32;     // keys per CTA
constexpr int kDkRows = 32;     // query rows per shared-memory tile
constexpr int kDkGroups = 8;    // channel groups: thread (key, group) owns channels group, group + 8, ...

// dk_jc = 0.001 sum_i dz_ij (q_ic - k_jc), in query order
__global__ void __launch_bounds__(kDkKeys * kDkGroups) align_attn_bwd_keys_kernel(
    const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ dz, float* __restrict__ dk, int t_q,
    int t_k, int c) {
  extern __shared__ float smem[];
  float* qs = smem;                          // [kDkRows][c]
  float* zs = smem + kDkRows * c;            // [kDkRows][kDkKeys + 1]
  const int b = blockIdx.y, j0 = blockIdx.x * kDkKeys;
  const int jj = threadIdx.x / kDkGroups, grp = threadIdx.x % kDkGroups, j = j0 + jj;
  float kreg[kAttnMaxC / kDkGroups], acc[kAttnMaxC / kDkGroups];
#pragma unroll
  for (int u = 0; u < kAttnMaxC / kDkGroups; ++u) {
    const int ch = grp + kDkGroups * u;
    kreg[u] = (j < t_k && ch < c) ? __ldg(k + ((long long)b * t_k + j) * c + ch) : 0.f;
    acc[u] = 0.f;
  }
  for (int r0 = 0; r0 < t_q; r0 += kDkRows) {
    __syncthreads();
    for (int e = threadIdx.x; e < kDkRows * c; e += blockDim.x) {
      const int r = e / c;
      qs[e] = (r0 + r < t_q) ? __ldg(q + ((long long)b * t_q + r0 + r) * c + (e - r * c)) : 0.f;
    }
    for (int e = threadIdx.x; e < kDkRows * kDkKeys; e += blockDim.x) {
      const int r = e / kDkKeys, kk = e - r * kDkKeys;
      zs[r * (kDkKeys + 1) + kk] =
          (r0 + r < t_q && j0 + kk < t_k) ? __ldg(dz + ((long long)b * t_q + r0 + r) * t_k + j0 + kk) : 0.f;
    }
    __syncthreads();
    const int nr = min(kDkRows, t_q - r0);
    for (int r = 0; r < nr; ++r) {
      const float d = zs[r * (kDkKeys + 1) + jj];
#pragma unroll
      for (int u = 0; u < kAttnMaxC / kDkGroups; ++u) {
        const int ch = grp + kDkGroups * u;
        if (ch < c) acc[u] = fmaf(d, qs[r * c + ch] - kreg[u], acc[u]);
      }
    }
  }
  if (j >= t_k) return;
#pragma unroll
  for (int u = 0; u < kAttnMaxC / kDkGroups; ++u) {
    const int ch = grp + kDkGroups * u;
    if (ch < c) dk[((long long)b * t_k + j) * c + ch] = 0.001f * acc[u];
  }
}


// ---- MAS ----------------------------------------------------------------------------------------------------------------
constexpr int kMasThreads = 256;
constexpr int kMasStageRows = 8;                  // rows of log(soft) staged per pass
constexpr long long kMasSmemBits = 96 * 1024;     // decision bits stay in shared memory up to this size
constexpr int kMasSmemMax = 200 * 1024;

inline int mas_words(int t_k) { return (t_k + 31) / 32; }
inline bool mas_bits_in_smem(int t_q, int t_k) { return (long long)t_q * mas_words(t_k) * 4 <= kMasSmemBits; }
inline long long mas_smem_bytes(int t_q, int t_k) {
  const long long cols = 32LL * mas_words(t_k);
  long long bytes = (2 + kMasStageRows) * cols * 4 + cols * 4;      // log_p (two rows), staged rows, per-key counts
  if (mas_bits_in_smem(t_q, t_k)) bytes += (long long)t_q * mas_words(t_k) * 4;
  return bytes;
}

// mas_width1 on soft[b, :T, :N], T = out_len[b], N = in_len[b]: row 0 keeps only key 0; for i >= 1
//   log_p[i][j] = log(soft[i][j]) + (j >= 1 && log_p[i-1][j-1] >= log_p[i-1][j] ? log_p[i-1][j-1] : log_p[i-1][j])
// with one decision bit per cell (a warp ballot per 32 keys), then the backtrack from (T-1, N-1) and the reference's final
// write of hard[0][0].  Thread j owns keys j, j + 256, ...; one __syncthreads per row.
__global__ void __launch_bounds__(kMasThreads) mas_kernel(const float* __restrict__ soft, const int32_t* __restrict__ in_len,
                                                          const int32_t* __restrict__ out_len, float* __restrict__ hard,
                                                          float* __restrict__ durations, uint32_t* __restrict__ gbits,
                                                          int t_q, int t_k, int bits_in_smem) {
  extern __shared__ float smem[];
  const int words = (t_k + 31) / 32, cols = 32 * words;
  float* lp0 = smem;
  float* lp1 = lp0 + cols;
  float* stage = lp1 + cols;                                       // [kMasStageRows][cols]
  int* counts = reinterpret_cast<int*>(stage + kMasStageRows * cols);
  uint32_t* bits = bits_in_smem ? reinterpret_cast<uint32_t*>(counts + cols)
                                : gbits + (long long)blockIdx.x * t_q * words;
  const int b = blockIdx.x, tid = threadIdx.x;
  const int T = min(out_len[b], t_q), N = min(in_len[b], t_k);
  const int ncols = 32 * ((max(N, 0) + 31) / 32);
  const float* sb = soft + (long long)b * t_q * t_k;
  float* hb = hard + (long long)b * t_q * t_k;
  for (long long e = tid; e < (long long)t_q * t_k; e += blockDim.x) hb[e] = 0.f;
  for (int j = tid; j < cols; j += blockDim.x) {
    counts[j] = 0;
    lp0[j] = (j == 0 && N > 0 && T > 0) ? logf(sb[0]) : -INFINITY;
  }
  __syncthreads();
  if (T > 0 && N > 0) {
    float* prev = lp0;
    float* cur = lp1;
    for (int i0 = 1; i0 < T; i0 += kMasStageRows) {
      const int nr = min(kMasStageRows, T - i0);
      for (int e = tid; e < nr * N; e += blockDim.x) {
        const int r = e / N, j = e - r * N;
        stage[r * cols + j] = logf(__ldg(sb + (long long)(i0 + r) * t_k + j));
      }
      __syncthreads();
      for (int r = 0; r < nr; ++r) {
        const int i = i0 + r;
        for (int j = tid; j < ncols; j += blockDim.x) {          // whole warps: ncols is a multiple of 32
          bool left = false;
          if (j < N) {
            const float stay = prev[j];
            left = j >= 1 && prev[j - 1] >= stay;
            cur[j] = stage[r * cols + j] + (left ? prev[j - 1] : stay);
          }
          const uint32_t word = __ballot_sync(0xffffffffu, left);
          if ((tid & 31) == 0) bits[(long long)i * words + (j >> 5)] = word;
        }
        __syncthreads();
        float* t = prev;
        prev = cur;
        cur = t;
      }
    }
    if (tid == 0) {
      int j = N - 1;
      for (int i = T - 1; i >= 1; --i) {
        hb[(long long)i * t_k + j] = 1.f;
        ++counts[j];
        if ((bits[(long long)i * words + (j >> 5)] >> (j & 31)) & 1u) --j;
      }
      hb[j] = 1.f;
      ++counts[j];
      if (j != 0) {                              // the reference's opt[0, prev_ind[0, j]] = opt[0, 0] = 1 after the loop
        hb[0] = 1.f;
        ++counts[0];
      }
    }
    __syncthreads();
  }
  for (int j = tid; j < t_k; j += blockDim.x) durations[(long long)b * t_k + j] = (float)counts[j];
}

// ---- forward-sum (CTC) loss ---------------------------------------------------------------------------------------------
// The alpha / beta recursions run in float64.  Their log-probabilities grow like -(frames x per-frame cost), thousands at
// a training utterance's length, and each gradient element's posterior exp(alpha + beta - y + nll) cancels them: in fp32
// that cancellation leaves a relative error near 1e-3 at 1000 frames x 200 symbols.  The frame normalisers and the
// log-softmax inputs stay fp32; a normaliser's rounding shifts every path through its frame alike, so it cancels in the
// posteriors.  Loss and gradient are stored as fp32.
constexpr int kCtcThreads = 256;
constexpr int kCtcSmemMax = 96 * 1024;       // the two state rows of 2 t_k + 1 doubles: t_k <= 3071

struct CtcWs {
  double* alpha;   // [batch][t_q][2 t_k + 1]   first, so that the doubles are 8-byte aligned
  double* nll;     // [batch]        -log p of each utterance
  float* lse;      // [batch][t_q]   log-sum-exp of the frame's [blank, keys < N]
  float* losses;   // [batch]        nll / N, 0 when infinite
};

inline long long ctc_ws_bytes(int batch, int t_q, int t_k) {
  return 8 * ((long long)batch * t_q * (2LL * t_k + 1) + batch) + 4 * ((long long)batch * t_q + batch);
}

inline CtcWs ctc_ws(void* ws, int batch, int t_q, int t_k) {
  CtcWs w;
  w.alpha = static_cast<double*>(ws);
  w.nll = w.alpha + (long long)batch * t_q * (2LL * t_k + 1);
  w.lse = reinterpret_cast<float*>(w.nll + batch);
  w.losses = w.lse + (long long)batch * t_q;
  return w;
}

inline size_t ctc_smem_bytes(int t_k) { return (size_t)2 * (2 * t_k + 1) * sizeof(double); }

__device__ __forceinline__ double lse2(double a, double b) {
  const double m = fmax(a, b);
  return m == -INFINITY ? -INFINITY : m + log(exp(a - m) + exp(b - m));
}

__device__ __forceinline__ double lse3(double a, double b, double c) {
  const double m = fmax(fmax(a, b), c);
  return m == -INFINITY ? -INFINITY : m + log(exp(a - m) + exp(b - m) + exp(c - m));
}

// log-probability of extended label s (even: the blank column, odd: key (s - 1) / 2) at frame row `lp`
__device__ __forceinline__ double ctc_y(const float* lp, int s, float blank, float lse) {
  return (double)((s & 1) ? __ldg(lp + (s >> 1)) : blank) - (double)lse;
}

// One CTA per utterance: the frame log-softmax normalisers, then the alpha recursion over S = 2N + 1 states (stored for the
// backward), the loss -log p and its share nll / N (0 when infinite: zero_infinity).
__global__ void __launch_bounds__(kCtcThreads) ctc_fwd_kernel(const float* __restrict__ logprob,
                                                              const int32_t* __restrict__ in_len,
                                                              const int32_t* __restrict__ out_len, CtcWs w, int t_q,
                                                              int t_k, float blank) {
  extern __shared__ double ctc_state[];
  const int S_max = 2 * t_k + 1;
  double* a0 = ctc_state;
  double* a1 = ctc_state + S_max;
  const int b = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int T = min(out_len[b], t_q), N = min(in_len[b], t_k), S = 2 * N + 1;
  const float* lpb = logprob + (long long)b * t_q * t_k;
  double* alpha = w.alpha + (long long)b * t_q * S_max;
  float* lse = w.lse + (long long)b * t_q;
  if (T < 1 || N < 1) {
    if (tid == 0) {
      w.nll[b] = INFINITY;
      w.losses[b] = 0.f;
    }
    return;
  }
  for (int t = warp; t < T; t += blockDim.x / 32) {
    const float* row = lpb + (long long)t * t_k;
    float m = blank;
    for (int j = lane; j < N; j += 32) m = fmaxf(m, row[j]);
    m = warp_max(m);
    float s = lane == 0 ? expf(blank - m) : 0.f;
    for (int j = lane; j < N; j += 32) s += expf(row[j] - m);
    s = warp_sum(s);
    if (lane == 0) lse[t] = m + logf(s);
  }
  __syncthreads();
  for (int s = tid; s < S; s += blockDim.x) {
    const double v = s < 2 ? ctc_y(lpb, s, blank, lse[0]) : -INFINITY;
    a0[s] = v;
    alpha[s] = v;
  }
  __syncthreads();
  double* prev = a0;
  double* cur = a1;
  for (int t = 1; t < T; ++t) {
    const float* row = lpb + (long long)t * t_k;
    const float l = lse[t];
    for (int s = tid; s < S; s += blockDim.x) {
      const double x = prev[s];
      const double y1 = s >= 1 ? prev[s - 1] : -INFINITY;
      const double y2 = ((s & 1) && s >= 3) ? prev[s - 2] : -INFINITY;
      const double v = ctc_y(row, s, blank, l) + lse3(x, y1, y2);
      cur[s] = v;
      alpha[(long long)t * S_max + s] = v;
    }
    __syncthreads();
    double* tmp = prev;
    prev = cur;
    cur = tmp;
  }
  if (tid == 0) {
    const double nll = -lse2(prev[S - 1], prev[S - 2]);
    w.nll[b] = nll;
    w.losses[b] = isinf(nll) ? 0.f : (float)(nll / N);
  }
}

// loss = (sum over the utterances in order of nll_b / N_b) / batch
__global__ void ctc_mean_kernel(CtcWs w, float* __restrict__ loss, int batch) {
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int b = 0; b < batch; ++b) s += w.losses[b];
    loss[0] = s / (float)batch;
  }
}

// One CTA per utterance: the beta recursion from the last frame and, per frame, the gradient of the loss with respect to
// logprob[b][t][j] = d_loss / (batch N) (softmax_t(key j) - posterior of state 2j + 1), zero outside t < T, j < N and for an
// utterance whose loss was infinite.
__global__ void __launch_bounds__(kCtcThreads) ctc_bwd_kernel(const float* __restrict__ logprob,
                                                              const int32_t* __restrict__ in_len,
                                                              const int32_t* __restrict__ out_len,
                                                              const float* __restrict__ d_loss, CtcWs w,
                                                              float* __restrict__ d_logprob, int batch, int t_q, int t_k,
                                                              float blank) {
  extern __shared__ double ctc_state[];
  const int S_max = 2 * t_k + 1;
  double* b0 = ctc_state;
  double* b1 = ctc_state + S_max;
  const int b = blockIdx.x, tid = threadIdx.x;
  const int T = min(out_len[b], t_q), N = min(in_len[b], t_k), S = 2 * N + 1;
  const double nll = (T >= 1 && N >= 1) ? w.nll[b] : INFINITY;
  const bool live = !isinf(nll);
  float* gb = d_logprob + (long long)b * t_q * t_k;
  for (long long e = tid; e < (long long)t_q * t_k; e += blockDim.x) {
    const int t = (int)(e / t_k), j = (int)(e - (long long)t * t_k);
    if (!live || t >= T || j >= N) gb[e] = 0.f;
  }
  if (!live) return;
  const double g = (double)d_loss[0] / ((double)batch * (double)N);
  const float* lpb = logprob + (long long)b * t_q * t_k;
  const double* alpha = w.alpha + (long long)b * t_q * S_max;
  const float* lse = w.lse + (long long)b * t_q;
  double* next = b0;
  double* cur = b1;
  for (int t = T - 1; t >= 0; --t) {
    const float* row = lpb + (long long)t * t_k;
    const float l = lse[t];
    for (int s = tid; s < S; s += blockDim.x) {
      const double y = ctc_y(row, s, blank, l);
      double v;
      if (t == T - 1) {
        v = s >= S - 2 ? y : -INFINITY;
      } else {
        const double x1 = s + 1 < S ? next[s + 1] : -INFINITY;
        const double x2 = ((s & 1) && s + 2 < S) ? next[s + 2] : -INFINITY;
        v = y + lse3(next[s], x1, x2);
      }
      cur[s] = v;
      if (s & 1) {
        const double post = exp(alpha[(long long)t * S_max + s] + v - y + nll);
        gb[(long long)t * t_k + (s >> 1)] = (float)(g * (exp(y) - post));
      }
    }
    __syncthreads();
    double* tmp = next;
    next = cur;
    cur = tmp;
  }
}

// ---- alignment prior ----------------------------------------------------------------------------------------------------
constexpr int kPriorThreads = 256;
constexpr int kPriorRows = 32;       // mel frames per CTA
constexpr int kPriorCols = 128;      // symbols per pass over the CTA's rows

// beta_binomial_prior_distribution (kantts/datasets/dataset.py:20-31) of utterance b = blockIdx.y, rows
// [t0, t0 + kPriorRows): with n = P = in_len[b] + 1, M = out_len[b], alpha = t + 1, beta = M - t and s = t + k,
//   ln prior[t][k] = lnC(n, k) + lnB(k + alpha, n - k + beta) - lnB(alpha, beta)
//                  = col[k] + diag[s] + row[t]
//   col[k]  = lg(n + 1) - lg(k + 1) - lg(n - k + 1)
//   diag[s] = lg(s + 1) + lg(n + M - s)                       (k + alpha = s + 1, n - k + beta = n + M - s)
//   row[t]  = -(lg(t + 1) + lg(M - t) - lg(M + 1)) - lg(n + M + 1)
// with lg = the float64 lgamma.  Each term is computed once per CTA (the diagonal once per pass), in shared memory; an
// element costs two adds and an exp.  Zero outside t < M, k < P.
__global__ void __launch_bounds__(kPriorThreads) attn_prior_kernel(const int64_t* __restrict__ in_len,
                                                                   const int64_t* __restrict__ out_len,
                                                                   float* __restrict__ prior, int t_q, int t_k) {
  __shared__ double row[kPriorRows];
  __shared__ double col[kPriorCols];
  __shared__ double diag[kPriorRows + kPriorCols - 1];
  const int b = blockIdx.y, t0 = blockIdx.x * kPriorRows, tid = threadIdx.x;
  const long long P = in_len[b] + 1, M = out_len[b];
  const double n = (double)P, m = (double)M;
  const double lg_n1 = lgamma(n + 1.0), lg_nm1 = lgamma(n + m + 1.0), lg_m1 = lgamma(m + 1.0);
  const int rows = min(kPriorRows, t_q - t0);
  const int live_rows = (int)max(0LL, min((long long)rows, M - t0));     // rows t < M
  const int live_cols = (int)max(0LL, min((long long)t_k, P));            // columns k < P
  for (int r = tid; r < live_rows; r += blockDim.x) {
    const double t = (double)(t0 + r);
    row[r] = -(lgamma(t + 1.0) + lgamma(m - t) - lg_m1) - lg_nm1;
  }
  float* out = prior + ((long long)b * t_q + t0) * t_k;
  for (int k0 = 0; k0 < t_k; k0 += kPriorCols) {
    const int cols = min(kPriorCols, t_k - k0);
    const int live = max(0, min(cols, live_cols - k0));
    if (live_rows > 0 && live > 0) {
      __syncthreads();                                  // the previous pass has read col and diag
      for (int c = tid; c < live; c += blockDim.x) {
        const double k = (double)(k0 + c);
        col[c] = lg_n1 - lgamma(k + 1.0) - lgamma(n - k + 1.0);
      }
      for (int d = tid; d < live_rows + live - 1; d += blockDim.x) {
        const double s = (double)(t0 + k0 + d);
        diag[d] = lgamma(s + 1.0) + lgamma(n + m - s);
      }
      __syncthreads();
    }
    for (int e = tid; e < rows * cols; e += blockDim.x) {
      const int r = e / cols, c = e - r * cols;
      float v = 0.f;
      if (r < live_rows && c < live) v = __double2float_rn(exp(col[c] + diag[r + c] + row[r]));
      out[(long long)r * t_k + k0 + c] = v;
    }
  }
}

}  // namespace

extern "C" int kt_attn_prior(const int64_t* valid_input_lengths, const int64_t* valid_output_lengths, float* prior,
                             int32_t batch, int32_t t_mel, int32_t t_text, void* stream) {
  KT_REQUIRE(valid_input_lengths && valid_output_lengths && prior, "attn_prior: null argument");
  KT_REQUIRE(batch > 0 && batch <= 65535 && t_mel > 0 && t_text > 0, "attn_prior: bad shape (batch %d, t_mel %d, t_text %d)",
             batch, t_mel, t_text);
  const dim3 grid((unsigned)ceil_div(t_mel, kPriorRows), (unsigned)batch);
  attn_prior_kernel<<<grid, kPriorThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      valid_input_lengths, valid_output_lengths, prior, t_mel, t_text);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

extern "C" int kt_align_attn_fwd(const float* q, const float* k, const float* prior, const int32_t* key_lengths,
                                 float* logprob, float* soft, float* row_lse, int32_t batch, int32_t t_q, int32_t t_k,
                                 int32_t c, void* stream) {
  KT_REQUIRE(q && k && key_lengths && logprob && soft, "align_attn_fwd: null argument");
  KT_REQUIRE(!prior || row_lse, "align_attn_fwd: a prior needs row_lse");
  KT_REQUIRE(batch > 0 && batch <= 65535 && t_q > 0 && t_k > 0 && c > 0 && c <= kAttnMaxC,
             "align_attn_fwd: bad shape (batch %d, t_q %d, t_k %d, c %d; c <= %d)", batch, t_q, t_k, c, kAttnMaxC);
  const size_t smem = (size_t)(kAttnKeys * tile_stride(c) + kAttnRows * c) * sizeof(float);
  const dim3 grid((unsigned)ceil_div(t_q, kAttnRows), (unsigned)batch);
  align_attn_fwd_kernel<<<grid, kAttnRows * 32, smem, static_cast<cudaStream_t>(stream)>>>(
      q, k, prior, key_lengths, logprob, soft, row_lse, t_q, t_k, c);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

extern "C" int kt_align_attn_bwd(const float* q, const float* k, const float* prior, const float* soft,
                                 const float* row_lse, const float* d_soft, const float* d_logprob, float* dz, float* dq,
                                 float* dk, int32_t batch, int32_t t_q, int32_t t_k, int32_t c, void* stream) {
  KT_REQUIRE(q && k && soft && dz && dq && dk, "align_attn_bwd: null argument");
  KT_REQUIRE(!prior || row_lse, "align_attn_bwd: a prior needs row_lse");
  KT_REQUIRE(batch > 0 && batch <= 65535 && t_q > 0 && t_k > 0 && c > 0 && c <= kAttnMaxC,
             "align_attn_bwd: bad shape (batch %d, t_q %d, t_k %d, c %d; c <= %d)", batch, t_q, t_k, c, kAttnMaxC);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t smem = (size_t)(kAttnKeys * tile_stride(c) + kAttnRows * c + kAttnRows * 32) * sizeof(float);
  align_attn_bwd_rows_kernel<<<dim3((unsigned)ceil_div(t_q, kAttnRows), (unsigned)batch), kAttnRows * 32, smem, st>>>(
      q, k, prior, soft, row_lse, d_soft, d_logprob, dz, dq, t_q, t_k, c);
  KT_CHECK_CUDA(cudaGetLastError());
  const size_t smem_k = (size_t)(kDkRows * c + kDkRows * (kDkKeys + 1)) * sizeof(float);
  align_attn_bwd_keys_kernel<<<dim3((unsigned)ceil_div(t_k, kDkKeys), (unsigned)batch), kDkKeys * kDkGroups, smem_k, st>>>(
      q, k, dz, dk, t_q, t_k, c);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

extern "C" int64_t kt_mas_workspace_bytes(int32_t batch, int32_t t_q, int32_t t_k) {
  if (batch <= 0 || t_q <= 0 || t_k <= 0 || mas_bits_in_smem(t_q, t_k)) return 0;
  return (int64_t)batch * t_q * mas_words(t_k) * 4;
}

extern "C" int kt_mas(const float* soft, const int32_t* in_lengths, const int32_t* out_lengths, float* hard,
                      float* durations, uint32_t* workspace, int64_t workspace_bytes, int32_t batch, int32_t t_q,
                      int32_t t_k, void* stream) {
  KT_REQUIRE(soft && in_lengths && out_lengths && hard && durations, "mas: null argument");
  KT_REQUIRE(batch > 0 && batch <= 65535 && t_q > 0 && t_k > 0, "mas: bad shape (batch %d, t_q %d, t_k %d)", batch, t_q, t_k);
  const bool in_smem = mas_bits_in_smem(t_q, t_k);
  const long long need = in_smem ? 0 : (long long)batch * t_q * mas_words(t_k) * 4;
  if (workspace_bytes < need || (need > 0 && !workspace)) {
    set_error("mas: workspace too small (%lld < %lld bytes)", (long long)workspace_bytes, need);
    return KT_ERR_WORKSPACE;
  }
  const long long smem = mas_smem_bytes(t_q, t_k);
  KT_REQUIRE(smem <= kMasSmemMax, "mas: %d keys need %lld bytes of shared memory (at most %d)", t_k, smem, kMasSmemMax);
  KT_CHECK_CUDA(allow_dyn_smem<mas_kernel>(kMasSmemMax));
  mas_kernel<<<batch, kMasThreads, (size_t)smem, static_cast<cudaStream_t>(stream)>>>(
      soft, in_lengths, out_lengths, hard, durations, workspace, t_q, t_k, in_smem ? 1 : 0);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

extern "C" int64_t kt_attn_ctc_workspace_bytes(int32_t batch, int32_t t_q, int32_t t_k) {
  if (batch <= 0 || t_q <= 0 || t_k <= 0) return 0;
  return (int64_t)ctc_ws_bytes(batch, t_q, t_k);
}

static int ctc_check(const float* logprob, const int32_t* in_lengths, const int32_t* out_lengths, const void* workspace,
                     int64_t workspace_bytes, int32_t batch, int32_t t_q, int32_t t_k, const char* what) {
  KT_REQUIRE(logprob && in_lengths && out_lengths && workspace, "%s: null argument", what);
  KT_REQUIRE(batch > 0 && batch <= 65535 && t_q > 0 && t_k > 0, "%s: bad shape (batch %d, t_q %d, t_k %d)", what, batch,
             t_q, t_k);
  KT_REQUIRE(ctc_smem_bytes(t_k) <= (size_t)kCtcSmemMax, "%s: %d keys exceed the shared-memory state rows (at most %d)",
             what, t_k, (kCtcSmemMax / (int)sizeof(double) / 2 - 1) / 2);
  const long long need = ctc_ws_bytes(batch, t_q, t_k);
  if (workspace_bytes < need) {
    set_error("%s: workspace too small (%lld < %lld bytes)", what, (long long)workspace_bytes, need);
    return KT_ERR_WORKSPACE;
  }
  return KT_OK;
}

extern "C" int kt_attn_ctc_fwd(const float* logprob, const int32_t* in_lengths, const int32_t* out_lengths, float* loss,
                               void* workspace, int64_t workspace_bytes, int32_t batch, int32_t t_q, int32_t t_k,
                               float blank_logprob, void* stream) {
  const int rc = ctc_check(logprob, in_lengths, out_lengths, workspace, workspace_bytes, batch, t_q, t_k, "attn_ctc_fwd");
  if (rc != KT_OK) return rc;
  KT_REQUIRE(loss, "attn_ctc_fwd: null loss");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const CtcWs w = ctc_ws(workspace, batch, t_q, t_k);
  KT_CHECK_CUDA(allow_dyn_smem<ctc_fwd_kernel>(kCtcSmemMax));
  ctc_fwd_kernel<<<batch, kCtcThreads, ctc_smem_bytes(t_k), st>>>(logprob, in_lengths, out_lengths, w, t_q, t_k, blank_logprob);
  KT_CHECK_CUDA(cudaGetLastError());
  ctc_mean_kernel<<<1, 32, 0, st>>>(w, loss, batch);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

extern "C" int kt_attn_ctc_bwd(const float* logprob, const int32_t* in_lengths, const int32_t* out_lengths,
                               const float* d_loss, const void* workspace, int64_t workspace_bytes, float* d_logprob,
                               int32_t batch, int32_t t_q, int32_t t_k, float blank_logprob, void* stream) {
  const int rc = ctc_check(logprob, in_lengths, out_lengths, workspace, workspace_bytes, batch, t_q, t_k, "attn_ctc_bwd");
  if (rc != KT_OK) return rc;
  KT_REQUIRE(d_loss && d_logprob, "attn_ctc_bwd: null argument");
  const CtcWs w = ctc_ws(const_cast<void*>(workspace), batch, t_q, t_k);
  KT_CHECK_CUDA(allow_dyn_smem<ctc_bwd_kernel>(kCtcSmemMax));
  ctc_bwd_kernel<<<batch, kCtcThreads, ctc_smem_bytes(t_k), static_cast<cudaStream_t>(stream)>>>(
      logprob, in_lengths, out_lengths, d_loss, w, d_logprob, batch, t_q, t_k, blank_logprob);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

}  // namespace kt
