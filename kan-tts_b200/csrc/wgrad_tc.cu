// wgmma weight-gradient kernel (bf16x3 split precision, fp32 accumulation in registers).
//
//   G[tap j][ca][cb] = sum_{batch, w, m}  fa(A[b][(m*step + ioff_j)/up, w][ca]) * fb(Bm[b][m, w][cb])
//   conv layer      : A = act_in(x)  (ca = C_in),  Bm = dy * act_out'(y) (cb = C_out), step = stride
//   transposed conv : A = dy * act'  (ca = C_out), Bm = act_in(x)        (cb = C_in),  step = stride
//
// The contraction runs over the flattened (time, sub-sequence) index, so both MMA operands are
// "MN-major" views of the same kind of shared-memory image the forward kernel uses ([flattened rows]
// [64 channels] bf16, SWIZZLE_128B): K = 16 consecutive rows per wgmma, M / N = channels
// (64-element groups, LBO apart).  A conv tap (q, rho) is again a pure descriptor row shift (q * nsub)
// of the staged residue image rho.  Two ways to fill M = 128 (two warpgroups of M = 64):
//   mode 0 (ca % 128 == 0): two 64-channel images of one tap
//   mode 1 (ca == 64)     : ONE image, two taps of the same residue, (q_{n+1} - q_n) * nsub rows apart
// Each CTA owns (ca tile, cb tile, a group of <= U "units" of one residue class = U*NT <= 128 accumulator
// columns) for a slice of the (batch, flattened time) range (split-K); partial tiles go to a workspace
// with plain stores and a second kernel reduces over the splits in order (deterministic, and cheaper than ~10^7 atomics).
#include <algorithm>
#include <atomic>
#include <cstdlib>
#include <vector>

#include "common.cuh"
#include "tc_common.cuh"
#include "tma.cuh"

namespace kt {

using namespace tc;

constexpr int kWgTK = 64;        // flattened rows per staged chunk
constexpr int kWgMaxUnits = 8;
constexpr int kWgMaxGroups = 24;

struct WgTcParams {
  Side a, b;
  float* ws;
  int batch, nsub, t_a, t_b, ca, cb, taps_total;   // ca / cb = tensor widths (all groups)
  int groups, ca_g, cb_g;                           // channels per (super-)group (= ca, cb when groups == 1)
  // thin groups: `gt` consecutive conv groups form one super-group whose dense (gt*ca_g0) x (gt*cb_g0) product is
  // computed and only the gt diagonal (ca_g0 x cb_g0) blocks are stored (cf. the block-diagonal tiles of conv_tc.cu)
  int gt, ca_g0, cb_g0;
  int M;                       // base rows m per sub-sequence
  int step, up;
  int mode, NT, n_cb_tiles, n_ca_tiles;
  int nsplit, chunks_per_batch;
  int a_groups, b_groups;      // 64-channel images per stage on each side
  int rows_a;                  // A image rows (max over unit groups), multiple of 8
  int ngroups;                 // unit groups (grid.y)
  int grp_rho[kWgMaxGroups], grp_qlo[kWgMaxGroups];
  int grp_first_unit[kWgMaxGroups + 1];
  int unit_tap0[kMaxTaps];     // first tap (index into tap_j / tap_q) of each unit
  int unit_ntaps[kMaxTaps];    // 1 or 2
  int tap_j[kMaxTaps];
  int tap_q[kMaxTaps];
  // bias gradient in the split-K workspace at `bias_off` (bias_grp >= 0) -- not produced by these kernels (bias_grp = -1): the
  // bias gradient is the column-sum kernel's
  int bias_grp;
  long long bias_off, split_stride;
  float* bias_direct;   // nsplit == 1: the kernel writes dw / dbias itself (ws = dw, no reduce pass); else nullptr
};

// Consumers: two warpgroups, warpgroup cw owns rows [64 cw, 64 cw + 64) of the M = 128 accumulator block of every unit (U =
// 128 / NT units of NT columns: 64 fp32 registers per thread).  Mode 0: rows = channels [128 ca_tile + 64 cw, +64) -- the
// second 64-channel image; mode 1: rows = channels of tap 2u + cw of the unit -- the image row-shifted by the tap distance.
constexpr int kWgConsumerArrivals = 8;   // one per consumer warp

// MMAs of one staged chunk for one unit (accumulators acc[OFF, OFF + NT / 2)): A (M = 64 channels x K rows) and B (K rows x
// NT channels) are MN-major images, the hi / lo planes img16 apart, K = 16 rows = 128 descriptor units per slice
template <int NT, int OFF>
__device__ __forceinline__ void wg_unit_mma(float (&acc)[kWgmmaMaxRegs], uint32_t a_hi, uint32_t img_a16, uint32_t b_hi, uint32_t img_b16,
                                            int kslices) {
  for (int ks = 0; ks < kslices; ++ks) {
    const uint32_t ko = (uint32_t)ks * 128u;
    wgmma_bf16_n<NT, 1, 1, OFF>(acc, desc_lo(a_hi + ko + img_a16), desc_lo(b_hi + ko), 1u);
    wgmma_bf16_n<NT, 1, 1, OFF>(acc, desc_lo(a_hi + ko), desc_lo(b_hi + ko + img_b16), 1u);
    wgmma_bf16_n<NT, 1, 1, OFF>(acc, desc_lo(a_hi + ko), desc_lo(b_hi + ko), 1u);
  }
}

// all units of one staged chunk, then wait for the MMAs (the stage is released by the caller)
template <int NT>
__device__ __forceinline__ void wg_chunk_mma(float (&acc)[kWgmmaMaxRegs], uint32_t sbase16, uint32_t b_hi, uint32_t img_a16, uint32_t img_b16,
                                             const uint32_t* s_shift, const uint32_t* s_half, int nu, int cw, int kslices) {
  wgmma_fence();
  wg_unit_mma<NT, 0>(acc, sbase16 + s_shift[0] + (cw ? s_half[0] : 0u), img_a16, b_hi, img_b16, kslices);
  if constexpr (kWgmmaMaxN / NT > 1) {
    if (nu > 1) wg_unit_mma<NT, NT / 2>(acc, sbase16 + s_shift[1] + (cw ? s_half[1] : 0u), img_a16, b_hi, img_b16, kslices);
  }
  wgmma_commit();
  wgmma_wait<0>();
  acc_fence(acc);
}

// registers -> workspace partial tiles (or dw itself when there is one split)
template <int NT>
__device__ __forceinline__ void wg_store(const WgTcParams& p, const float (&acc)[kWgmmaMaxRegs], int cw, int wq, int lane, int cb_tile,
                                         int ca_tile, int cgrp, int u0, int nu, int split) {
  const bool vec = ((p.cb | p.cb_g0) & 1) == 0;
#pragma unroll
  for (int u = 0; u < kWgmmaMaxN / NT; ++u) {
    if (u >= nu) break;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = cw * 64 + wq * 16 + (lane >> 2) + 8 * h;   // M index inside the unit
      int tap_n, ca_idx;
      bool valid;
      if (p.mode == 0) { tap_n = p.unit_tap0[u0 + u]; ca_idx = ca_tile * 128 + row; valid = true; }
      else { tap_n = p.unit_tap0[u0 + u] + (row >> 6); ca_idx = row & 63; valid = (row >> 6) < p.unit_ntaps[u0 + u]; }
      valid = valid && ca_idx < p.ca_g;
      if (!valid) continue;
      const int col0 = cb_tile * NT;                                      // first column inside the (super-)group
      // columns [c_lo, c_hi) of this tile are stored, column n at obase + n
      int c_lo = 0, c_hi = min(NT, p.cb_g - col0);
      long long obase;
      if (p.gt > 1) {   // block diagonal: row of conv group gl keeps only that group's cb_g0 columns
        const int gl = ca_idx / p.ca_g0, ci_l = ca_idx - gl * p.ca_g0;
        c_lo = gl * p.cb_g0; c_hi = c_lo + p.cb_g0;
        obase = (long long)split * p.split_stride + (((long long)p.tap_j[tap_n]) * p.ca_g0 + ci_l) * p.cb +
                ((long long)cgrp * p.gt + gl) * p.cb_g0 - c_lo;
      } else {
        obase = (long long)split * p.split_stride + (((long long)p.tap_j[tap_n]) * p.ca_g + ca_idx) * p.cb + (long long)cgrp * p.cb_g + col0;
      }
#pragma unroll
      for (int i = 0; i < NT / 8; ++i) {
        const int n = i * 8 + 2 * (lane & 3);
        const float v0 = acc[u * (NT / 2) + 4 * i + 2 * h], v1 = acc[u * (NT / 2) + 4 * i + 2 * h + 1];
        const bool ok0 = n >= c_lo && n < c_hi, ok1 = n + 1 >= c_lo && n + 1 < c_hi;
        if (vec && ok0 && ok1) {
          *reinterpret_cast<float2*>(p.ws + obase + n) = make_float2(v0, v1);
        } else {
          if (ok0) p.ws[obase + n] = v0;
          if (ok1) p.ws[obase + n + 1] = v1;
        }
      }
    }
  }
}

// per unit of this CTA: A-side row shift and the offset of the second warpgroup's 64 rows, in 16-byte descriptor units
__device__ __forceinline__ void wg_unit_table(const WgTcParams& p, int u0, int nu, int qlo, int img_a, uint32_t* s_shift, uint32_t* s_half) {
  for (int u = threadIdx.x; u < nu; u += blockDim.x) {
    const int n_a = p.unit_tap0[u0 + u];
    uint32_t half;
    if (p.mode == 0) half = 2u * (uint32_t)img_a;
    // mode 1: second half of M = the next tap of the same residue (rows 64..127 are discarded when the unit has one tap)
    else half = p.unit_ntaps[u0 + u] == 2 ? (uint32_t)((p.tap_q[n_a + 1] - p.tap_q[n_a]) * p.nsub) * 128u : 128u;
    s_shift[u] = ((uint32_t)((p.tap_q[n_a] - qlo) * p.nsub) * 128u) >> 4;
    s_half[u] = half >> 4;
  }
}

// warpgroups 0 / 3: producers of the even / odd chunks; warpgroups 1 / 2: consumers (MMAs + epilogue).  The kernel is bound
// by the ISSUE rate of the fp32 -> split-bf16 staging (~80 instructions per 8 elements), so the producers are 8 warps.
constexpr int kWgThreads = 512;

template <int NT>
__global__ void __launch_bounds__(kWgThreads, 1) wgrad_tc_kernel(const __grid_constant__ WgTcParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // (pointer arithmetic on the __shared__ array, not integer casts: the compiler must keep the shared address space)
  uint8_t* smem = smem_raw + ((1024u - (tc::smem_u32(smem_raw) & 1023u)) & 1023u);
  const int img_a = p.rows_a * 128;            // one plane of one A image
  const int img_b = kWgTK * 128;               // one plane of one B image
  const int stage_bytes = 2 * (p.a_groups * img_a + p.b_groups * img_b);
  uint8_t* stage0 = smem;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + 2 * (size_t)stage_bytes);
  uint64_t* full = bars;        // [2] producers -> MMA
  uint64_t* empty = bars + 2;   // [2] MMA -> producers
  uint32_t* s_shift = reinterpret_cast<uint32_t*>(bars + 4);   // [kWgMaxUnits]
  uint32_t* s_half = s_shift + kWgMaxUnits;                    // [kWgMaxUnits]

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int cb_tile = blockIdx.x % p.n_cb_tiles;
  const int ca_tile = (blockIdx.x / p.n_cb_tiles) % p.n_ca_tiles;
  const int cgrp = blockIdx.x / (p.n_cb_tiles * p.n_ca_tiles);   // conv group
  const int grp = blockIdx.y;
  const int u0 = p.grp_first_unit[grp];
  const int nu = p.grp_first_unit[grp + 1] - u0;
  const int qlo = p.grp_qlo[grp];
  const int split = blockIdx.z;
  const long long units = (long long)p.batch * p.chunks_per_batch;
  const long long c_begin = units * split / p.nsplit;
  const long long c_end = units * (split + 1) / p.nsplit;

  if (tid == 0) {
    for (int s = 0; s < 2; ++s) { mbar_init(&full[s], 128); mbar_init(&empty[s], kWgConsumerArrivals); }
    mbar_fence_init();
    fence_proxy_async();
  }
  wg_unit_table(p, u0, nu, qlo, img_a, s_shift, s_half);
  __syncthreads();

  if (warp < 4 || warp >= 12) {
    // ===================== producers =====================
    const int pg = warp < 4 ? 0 : 1;                                       // pipeline stage this group fills
    const int ptid = tid & 127;
    int it = 0;
    for (long long c = c_begin; c < c_end; ++c, ++it) {
      const int s = it & 1;
      if (s != pg) continue;
      mbar_wait(&empty[s], ((it >> 1) & 1) ^ 1);
      const int bb = (int)(c / p.chunks_per_batch);
      const int f0 = (int)(c % p.chunks_per_batch) * kWgTK;
      uint8_t* st = stage0 + (size_t)s * stage_bytes;
      RowMap ra;  // gathered side: residue image of this unit group
      ra.base_row = (long long)bb * p.t_a * p.nsub;
      ra.fv0 = f0 + qlo * p.nsub;
      ra.nsub = p.nsub; ra.step = p.step; ra.rho = p.grp_rho[grp]; ra.up = p.up; ra.t_lim = p.t_a * p.up;
      for (int g = 0; g < p.a_groups; ++g) {
        uint8_t* hi = st + (size_t)g * 2 * img_a;
        const int c_lo = ca_tile * (p.mode == 0 ? 128 : 64) + g * 64;           // channel offset inside the group
        stage_rows<4, false, 2>(hi, hi + img_a, p.a, p.a.p, p.a.aux, p.ca, cgrp * p.ca_g + c_lo, min(64, p.ca_g - c_lo), true, ra,
                                p.rows_a, ptid);
      }
      RowMap rb;  // base side: rows m (flattened with w), zero beyond M
      rb.base_row = (long long)bb * p.t_b * p.nsub;
      rb.fv0 = f0; rb.nsub = p.nsub; rb.step = 1; rb.rho = 0; rb.up = 1; rb.t_lim = min(p.M, p.t_b);
      uint8_t* bst = st + (size_t)p.a_groups * 2 * img_a;
      for (int g = 0; g < p.b_groups; ++g) {
        uint8_t* hi = bst + (size_t)g * 2 * img_b;
        const int c_lo = cb_tile * NT + g * 64;
        stage_rows<2, false, 2>(hi, hi + img_b, p.b, p.b.p, p.b.aux, p.cb, cgrp * p.cb_g + c_lo, min(64, p.cb_g - c_lo), true, rb,
                                kWgTK, ptid);
      }
      fence_proxy_async();
      mbar_arrive(&full[s]);
    }
  } else {
    // ===================== consumers =====================
    const int cw = (warp - 4) >> 2, wq = warp & 3;
    const uint32_t lbo_b16 = ((2u * (uint32_t)img_b) >> 4) << 16;
    const uint32_t img_a16 = (uint32_t)img_a >> 4, img_b16 = (uint32_t)img_b >> 4;
    const uint32_t st16[2] = {smem_u32(stage0) >> 4, smem_u32(stage0 + stage_bytes) >> 4};
    const uint32_t boff16 = (uint32_t)(p.a_groups * 2 * img_a) >> 4;
    float acc[kWgmmaMaxRegs];
#pragma unroll
    for (int i = 0; i < kWgmmaMaxRegs; ++i) acc[i] = 0.f;
    int it = 0;
    for (long long c = c_begin; c < c_end; ++c, ++it) {
      const int s = it & 1;
      mbar_wait(&full[s], (it >> 1) & 1);
      wg_chunk_mma<NT>(acc, st16[s], (st16[s] + boff16) | lbo_b16, img_a16, img_b16, s_shift, s_half, nu, cw, kWgTK / 16);
      if (lane == 0) mbar_arrive(&empty[s]);
    }
    wg_store<NT>(p, acc, cw, wq, lane, cb_tile, ca_tile, cgrp, u0, nu, split);
  }
}

// ---- TMA-fed variant (plain convs, no nearest-upsampling, channel counts % 8 == 0) -------------------------------------
// The register-staged kernel above is bound by its producers: every CTA converts its fp32 operand rows to split bf16
// itself (a 1024-channel layer converts each element ~23 times, once per (channel tile, unit group) CTA) with ~2 loads
// in flight per thread -- 11 us per 64-row chunk against 1.6 us of MMAs (call r2y).  Here one elementwise pre-pass writes
// each operand ONCE as hi / lo bf16 planes ([plane][batch][time][sub-sequence][channel], the activation layout), and the
// weight-gradient CTAs pull their tiles with cp.async.bulk.tensor (SWIZZLE_128B boxes of 64 channels x `nsub` x `tt`
// time steps land as exactly the MN-major images the MMAs read; rows outside [0, T) are the TMA unit's zero fill), so the
// main loop is one elected producer thread, two consumer warpgroups and an `nstages`-deep mbarrier ring.
// A chunk = `tt` base time steps x all sub-sequences = R rows, padded to Rp = ceil16(R) (K = 16 per MMA) with rows that
// are zeroed once and never written again.  A strided conv reads one residue class of the input per unit group: each
// residue rho has its own tensor map (base + rho rows, time stride = step), so no element strides are needed.
constexpr int kWgTmaThreads = 288;   // warpgroups 0 / 1 consumers (MMAs + epilogue), warp 8 TMA producer
constexpr int kWgTmaMaxStages = 4;

struct WgTmaExtra {
  int tt, R, Rp, nstages;
  int rows_a_p;        // rows of one A image plane (multiple of 8): Rp + tap span
  int a_box_t;         // time steps per A box = tt + (largest tap span of a unit group)
  int chunks_per_batch;
  alignas(64) CUtensorMap map_b;
  alignas(64) CUtensorMap map_a[8];   // one per residue class of the input
};

// fp32 operand -> hi / lo bf16 planes, with the operand's fused transform (pre-activation / activation-derivative mask)
// (both operands of a layer in ONE launch: CTAs [0, blocks_a) convert operand A, the rest operand B)
__global__ void split_planes_kernel(Side sa, long long n8a, __nv_bfloat16* __restrict__ hia, Side sb, long long n8b,
                                    __nv_bfloat16* __restrict__ hib, int blocks_a) {
  const bool first = (int)blockIdx.x < blocks_a;
  const Side s = first ? sa : sb;
  const long long n8 = first ? n8a : n8b;
  __nv_bfloat16* hi = first ? hia : hib;
  __nv_bfloat16* lo = hi + n8 * 8;
  const long long b0 = first ? blockIdx.x : blockIdx.x - blocks_a, nb = first ? blocks_a : (long long)gridDim.x - blocks_a;
  const bool has_aux = s.mode >= SIDE_DLRELU;
  for (long long i = b0 * (long long)blockDim.x + threadIdx.x; i < n8; i += nb * blockDim.x) {
    const float4 v0 = __ldg(reinterpret_cast<const float4*>(s.p) + 2 * i), v1 = __ldg(reinterpret_cast<const float4*>(s.p) + 2 * i + 1);
    float x[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
    if (has_aux) {
      const float4 a0 = __ldg(reinterpret_cast<const float4*>(s.aux) + 2 * i), a1 = __ldg(reinterpret_cast<const float4*>(s.aux) + 2 * i + 1);
      const float ax[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
#pragma unroll
      for (int e = 0; e < 8; ++e) x[e] = side_apply(x[e], ax[e], s.mode, s.slope);
    } else if (s.mode == SIDE_LRELU) {
#pragma unroll
      for (int e = 0; e < 8; ++e) x[e] = x[e] > 0.f ? x[e] : x[e] * s.slope;
    }
    uint4 h, l;
    split8(x, h, l);
    reinterpret_cast<uint4*>(hi)[i] = h;
    reinterpret_cast<uint4*>(lo)[i] = l;
  }
}

template <int NT>
__global__ void __launch_bounds__(kWgTmaThreads, 1) wgrad_tma_kernel(const __grid_constant__ WgTcParams p, const __grid_constant__ WgTmaExtra x) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (tc::smem_u32(smem_raw) & 1023u)) & 1023u);
  const int img_a = x.rows_a_p * 128;          // one plane of one A image
  const int img_b = x.Rp * 128;                // one plane of one B image
  const int stage_bytes = 2 * (p.a_groups * img_a + p.b_groups * img_b);
  uint8_t* stage0 = smem;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)x.nstages * stage_bytes);
  uint64_t* full = bars;                        // [nstages] TMA -> MMA
  uint64_t* empty = bars + kWgTmaMaxStages;     // [nstages] MMA -> TMA
  uint32_t* s_shift = reinterpret_cast<uint32_t*>(bars + 2 * kWgTmaMaxStages);   // [kWgMaxUnits]
  uint32_t* s_half = s_shift + kWgMaxUnits;                                     // [kWgMaxUnits]

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int cb_tile = blockIdx.x % p.n_cb_tiles;
  const int ca_tile = (blockIdx.x / p.n_cb_tiles) % p.n_ca_tiles;
  const int cgrp = blockIdx.x / (p.n_cb_tiles * p.n_ca_tiles);
  const int grp = blockIdx.y;
  const int u0 = p.grp_first_unit[grp];
  const int nu = p.grp_first_unit[grp + 1] - u0;
  const int qlo = p.grp_qlo[grp];
  const int split = blockIdx.z;
  const long long units = (long long)p.batch * x.chunks_per_batch;
  const long long c_begin = units * split / p.nsplit;
  const long long c_end = units * (split + 1) / p.nsplit;

  if (tid == 0) {
    for (int s = 0; s < x.nstages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], kWgConsumerArrivals); }
    mbar_fence_init();
  }
  {  // padding rows of every image (never written by the TMA boxes): zero, so that a partial last K slice contributes nothing
    const int a_box_rows = x.a_box_t * p.nsub;
    const int n_img = 2 * (p.a_groups + p.b_groups);
    for (int s = 0; s < x.nstages; ++s)
      for (int i = 0; i < n_img; ++i) {
        const bool is_a = i < 2 * p.a_groups;
        uint8_t* img = stage0 + (size_t)s * stage_bytes + (is_a ? (size_t)i * img_a : (size_t)2 * p.a_groups * img_a + (size_t)(i - 2 * p.a_groups) * img_b);
        const int r0 = is_a ? a_box_rows : x.R, r1 = is_a ? x.rows_a_p : x.Rp;
        for (int o = r0 * 128 + tid * 16; o < r1 * 128; o += kWgTmaThreads * 16) *reinterpret_cast<uint4*>(img + o) = make_uint4(0u, 0u, 0u, 0u);
      }
  }
  wg_unit_table(p, u0, nu, qlo, img_a, s_shift, s_half);
  fence_proxy_async();
  __syncthreads();

  if (warp == 8) {
    // ===================== TMA producer =====================
    if (elect_one()) {
      const uint32_t tx = 2u * (uint32_t)(p.a_groups * x.a_box_t * p.nsub + p.b_groups * x.R) * 128u;
      const CUtensorMap* ma = &x.map_a[p.grp_rho[grp]];
      const int ca0 = cgrp * p.ca_g + ca_tile * (p.mode == 0 ? 128 : 64);
      const int cb0 = cgrp * p.cb_g + cb_tile * NT;
      int it = 0;
      for (long long c = c_begin; c < c_end; ++c, ++it) {
        const int s = it % x.nstages;
        mbar_wait(&empty[s], ((it / x.nstages) & 1) ^ 1);
        const int bb = (int)(c / x.chunks_per_batch);
        const int m0 = (int)(c % x.chunks_per_batch) * x.tt;
        uint8_t* st = stage0 + (size_t)s * stage_bytes;
        mbar_arrive_expect_tx(&full[s], tx);
        for (int g = 0; g < p.a_groups; ++g)
          for (int pl = 0; pl < 2; ++pl)
            tma_load_5d(st + (size_t)(2 * g + pl) * img_a, ma, ca0 + g * 64, 0, m0 + qlo, bb, pl, &full[s]);
        uint8_t* bst = st + (size_t)p.a_groups * 2 * img_a;
        for (int g = 0; g < p.b_groups; ++g)
          for (int pl = 0; pl < 2; ++pl)
            tma_load_5d(bst + (size_t)(2 * g + pl) * img_b, &x.map_b, cb0 + g * 64, 0, m0, bb, pl, &full[s]);
      }
      // every issued box has landed before the CTA may exit: the consumers waited for all of them
    }
    __syncwarp();
  } else {
    // ===================== consumers =====================
    const int cw = warp >> 2, wq = warp & 3;
    const uint32_t lbo_b16 = ((2u * (uint32_t)img_b) >> 4) << 16;
    const uint32_t img_a16 = (uint32_t)img_a >> 4, img_b16 = (uint32_t)img_b >> 4;
    const uint32_t st0_16 = smem_u32(stage0) >> 4, stage16 = (uint32_t)stage_bytes >> 4;
    const uint32_t boff16 = (uint32_t)(p.a_groups * 2 * img_a) >> 4;
    const int kslices = x.Rp >> 4;
    float acc[kWgmmaMaxRegs];
#pragma unroll
    for (int i = 0; i < kWgmmaMaxRegs; ++i) acc[i] = 0.f;
    int it = 0;
    for (long long c = c_begin; c < c_end; ++c, ++it) {
      const int s = it % x.nstages;
      mbar_wait(&full[s], (it / x.nstages) & 1);
      const uint32_t sbase = st0_16 + (uint32_t)s * stage16;
      wg_chunk_mma<NT>(acc, sbase, (sbase + boff16) | lbo_b16, img_a16, img_b16, s_shift, s_half, nu, cw, kslices);
      if (lane == 0) mbar_arrive(&empty[s]);
    }
    wg_store<NT>(p, acc, cw, wq, lane, cb_tile, ca_tile, cgrp, u0, nu, split);
  }
}

// sums the split-K partials: ws = [nsplit][stride] with stride >= n + nb; elements [0, n) -> dw, [bias_off, bias_off + nb) -> dbias
__global__ void wgrad_reduce_kernel(const float* __restrict__ ws, float* __restrict__ dw, long long n, int nsplit, long long stride,
                                    float* __restrict__ dbias, long long bias_off, int nb) {
  const long long gtid = blockIdx.x * (long long)blockDim.x + threadIdx.x, gsz = (long long)gridDim.x * blockDim.x;
  if (dbias) {
    for (long long i = gtid; i < nb; i += gsz) {
      float acc = 0.f;
      for (int s = 0; s < nsplit; ++s) acc += ws[(long long)s * stride + bias_off + i];
      dbias[i] = acc;
    }
  }
  if ((n & 3) || (stride & 3)) {  // thin layers: split slices are not 16-byte aligned
    for (long long i = gtid; i < n; i += gsz) {
      float acc = ws[i];
      for (int s = 1; s < nsplit; ++s) acc += ws[(long long)s * stride + i];
      dw[i] = acc;
    }
    return;
  }
  const long long n4 = n / 4;
  for (long long i = gtid; i < n4; i += gsz) {
    float4 acc = __ldg(reinterpret_cast<const float4*>(ws) + i);
    for (int s = 1; s < nsplit; ++s) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(ws + (long long)s * stride) + i);
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    reinterpret_cast<float4*>(dw)[i] = acc;
  }
}

// Many splits of a small gradient (thin layers: 147 splits of 7 K floats): one WARP per output float4, lanes stride over the splits
// and combine with shuffles -- the kernel above walks the splits serially per thread (47 us for that shape with 7 CTAs).
__global__ void wgrad_reduce_wide_kernel(const float* __restrict__ ws, float* __restrict__ dw, long long n, int nsplit, long long stride,
                                         float* __restrict__ dbias, long long bias_off, int nb) {
  const int lane = threadIdx.x & 31;
  const long long warp = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5, nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  const bool vec = ((n | stride) & 3) == 0;
  const long long items = vec ? n / 4 : n;
  const long long items_b = dbias ? nb : 0;
  for (long long i = warp; i < items + items_b; i += nwarps) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (i < items) {
      if (vec) {
        for (int s = lane; s < nsplit; s += 32) {
          const float4 v = __ldg(reinterpret_cast<const float4*>(ws + (long long)s * stride) + i);
          acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
        }
      } else {
        for (int s = lane; s < nsplit; s += 32) acc.x += ws[(long long)s * stride + i];
      }
    } else {
      for (int s = lane; s < nsplit; s += 32) acc.x += ws[(long long)s * stride + bias_off + (i - items)];
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      acc.x += __shfl_xor_sync(0xffffffffu, acc.x, o); acc.y += __shfl_xor_sync(0xffffffffu, acc.y, o);
      acc.z += __shfl_xor_sync(0xffffffffu, acc.z, o); acc.w += __shfl_xor_sync(0xffffffffu, acc.w, o);
    }
    if (lane == 0) {
      if (i >= items) dbias[i - items] = acc.x;
      else if (vec) reinterpret_cast<float4*>(dw)[i] = acc;
      else dw[i] = acc.x;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// host
// ---------------------------------------------------------------------------------------------
struct WgPlan {
  bool ok;
  WgTcParams p;
  size_t smem;
  long long ws_floats;       // whole workspace: split-K partials (+ the bf16 operand planes of the TMA variant)
  // TMA variant (tma == true): x, its shared-memory size, offsets (floats) of the operand planes inside the workspace
  bool tma;
  WgTmaExtra x;
  size_t smem_tma;
  long long part_floats, planes_a_off, planes_b_off;
  int nsplit_tma;
  int max_span_q;
};

int debug_flags();   // conv_tc.cu (kt_debug_set_flags): 256 skip the operand split, 512 skip the MMA kernel, 1024 skip the split-K reduce

// SMs of the current device (132 without one: the host-logic tests plan for an H100)
static int wg_sm_count() {
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

static bool wg_want_tma() {
  static const bool on = [] { const char* e = std::getenv("KANTTS_B200_WG_TMA"); return !(e && e[0] == '0'); }();
  return on;
}

static WgPlan make_plan(const KtConv1dDesc* d, bool allow_tma = true, bool plan_only = false) {
  WgPlan pl{};
  pl.ok = false;
  WgTcParams& p = pl.p;
  // gathered (A) side / base (B) side, see conv_ffma.cu: conv1d_bwd_weight_ffma
  const bool tr = d->transposed != 0;
  const int ca = tr ? d->c_out : d->c_in, cb = tr ? d->c_in : d->c_out;
  p.groups = d->groups;
  p.ca_g = ca / d->groups; p.cb_g = cb / d->groups;
  p.ca_g0 = p.ca_g; p.cb_g0 = p.cb_g; p.gt = 1;
  if (d->groups > 1 && (p.cb_g & 3) == 0) {   // pack thin groups into block-diagonal super-groups
    while (p.groups % 2 == 0 && p.ca_g * 2 <= 64 && p.cb_g * 2 <= 256) { p.groups /= 2; p.ca_g *= 2; p.cb_g *= 2; p.gt *= 2; }
  }
  p.batch = d->batch; p.nsub = d->nsub; p.ca = ca; p.cb = cb; p.taps_total = d->kernel;
  p.t_a = tr ? d->t_out : d->t_in;
  p.t_b = tr ? d->t_in : d->t_out;
  p.M = p.t_b;
  p.step = d->stride;
  p.up = tr ? 1 : d->upsample;
  if (p.step > 8) return pl;
  // channels are zero-padded to 64-wide images: thin / grouped layers use the same kernel
  p.mode = p.ca_g <= 64 ? 1 : 0;
  // TMA variant (see wgrad_tma_kernel): plain convs whose box coordinates (multiples of the (super-)group widths) are 16-byte
  // aligned.  Tiles are at most N = 128 wide (the accumulators of all units of a CTA are 64 registers per consumer thread).
  const bool tma_ok = allow_tma && !tr && p.up == 1 && (ca % 8) == 0 && (cb % 8) == 0 && (p.ca_g % 8) == 0 && (p.cb_g % 8) == 0 &&
                      (plan_only || (wg_want_tma() && encode_tiled_fn() != nullptr));   // plan_only: host-logic tests without a driver
  p.NT = std::min(kWgmmaMaxN, (p.cb_g + 63) & ~63);
  p.n_cb_tiles = ceil_div(p.cb_g, p.NT);
  p.n_ca_tiles = p.mode == 0 ? ceil_div(p.ca_g, 128) : 1;
  p.a_groups = p.mode == 0 ? 2 : 1;
  p.b_groups = p.NT / 64;
  const int U = std::min(kWgMaxUnits, kWgmmaMaxN / p.NT);
  const int taps_per_unit = p.mode == 1 ? 2 : 1;
  // taps sorted by (residue, q)
  int ntap = 0, nunit = 0;
  p.ngroups = 0;
  int max_span = 0;
  for (int r = 0; r < p.step; ++r) {
    std::vector<std::pair<int, int>> tq;  // (q, j)
    for (int j = 0; j < d->kernel; ++j) {
      const int ioff = j * d->dilation - d->pad_left;
      const int q = fdiv(ioff, p.step);
      if (ioff - q * p.step == r) tq.push_back({q, j});
    }
    std::sort(tq.begin(), tq.end());
    size_t i = 0;
    // the residue's units are spread EVENLY over its unit groups (5 taps, U = 4: groups of 3 + 2, not 4 + 1): every CTA loads
    // the same operand rows per chunk whatever its unit count, so the largest group sets the pace
    const int units_r = ceil_div((int)tq.size(), taps_per_unit);
    const int groups_r = std::max(1, ceil_div(units_r, U));
    const int U_r = ceil_div(units_r, groups_r);
    while (i < tq.size()) {
      // one unit group: up to U units of this residue
      if (p.ngroups >= kWgMaxGroups) return pl;
      const int g = p.ngroups++;
      p.grp_rho[g] = r;
      p.grp_qlo[g] = tq[i].first;
      p.grp_first_unit[g] = nunit;
      int qhi = tq[i].first;
      for (int u = 0; u < U_r && i < tq.size(); ++u) {
        p.unit_tap0[nunit] = ntap;
        const int nt_u = (int)std::min<size_t>(taps_per_unit, tq.size() - i);
        p.unit_ntaps[nunit] = nt_u;
        for (int e = 0; e < nt_u; ++e, ++i, ++ntap) {
          p.tap_j[ntap] = tq[i].second;
          p.tap_q[ntap] = tq[i].first;
          qhi = tq[i].first;
        }
        ++nunit;
      }
      max_span = std::max(max_span, (qhi - p.grp_qlo[g]) * p.nsub);
      pl.max_span_q = std::max(pl.max_span_q, qhi - p.grp_qlo[g]);
    }
  }
  p.grp_first_unit[p.ngroups] = nunit;
  p.rows_a = (kWgTK + max_span + 7) & ~7;
  const size_t stage = 2 * ((size_t)p.a_groups * p.rows_a * 128 + (size_t)p.b_groups * kWgTK * 128);
  pl.smem = 1024 + 2 * stage + 128;
  if (pl.smem > (size_t)kMaxDynSmem) return pl;   // (a smaller U would shrink the halo; not needed for the shipped shapes)
  p.bias_grp = -1;   // the bias gradient is the column-sum kernel's (conv1d_bwd_weight_tc)
  p.chunks_per_batch = ceil_div(p.M * p.nsub, kWgTK);
  const long long units = (long long)p.batch * p.chunks_per_batch;
  const long long base = (long long)p.groups * p.n_ca_tiles * p.n_cb_tiles * p.ngroups;
  const int sms = wg_sm_count();
  // split-K factor: CTAs run one per SM in waves of one per SM; minimise (waves x chunks per CTA) plus the cost of writing
  // and re-reading one more partial copy of the gradient (in units of one chunk ~ 10 us; ~4 TB/s effective)
  const double out_chunks = (double)p.taps_total * p.ca_g0 * cb * 8.0 / 4e12 / 10e-6;
  long long nsplit = 1;
  double best = 1e30;
  for (long long ns = 1; ns <= std::min<long long>(units, 296); ++ns) {
    const long long waves = (base * ns + sms - 1) / sms;
    const double cost = (double)waves * (double)((units + ns - 1) / ns) + (double)ns * out_chunks;
    if (cost < best - 1e-9) { best = cost; nsplit = ns; }
  }
  p.nsplit = (int)nsplit;
  const long long n_main = (long long)p.taps_total * p.ca_g0 * cb;
  p.bias_off = n_main;
  p.split_stride = n_main + (p.bias_grp >= 0 ? ((cb + 3) & ~3) : 0);
  pl.ws_floats = nsplit * p.split_stride;
  pl.ok = true;

  // ---- TMA variant: chunk = tt base time steps x nsub sub-sequences, padded to whole K = 16 slices
  pl.tma = false;
  if (tma_ok) {
    WgTmaExtra& x = pl.x;
    for (int r = 0; r < p.step; ++r)
      if (p.t_a - r <= 0) return make_plan(d, false, plan_only);
    // tt: the largest chunk (R = tt * nsub <= 128 rows, at most 20 % padding in the last K slice) that still leaves a ring of
    // three stages; else the deepest ring
    int best_tt = 0, best_ns = 0;
    for (int tt = std::max(1, 128 / p.nsub); tt >= 1; --tt) {
      const int R = tt * p.nsub, Rp = (R + 15) & ~15;
      if (tt + pl.max_span_q > 256 || R > 256 || (tt > 1 && R * 5 < Rp * 4)) continue;
      const int rows_a_p = (Rp + pl.max_span_q * p.nsub + 7) & ~7;
      const size_t stage = 2 * ((size_t)p.a_groups * rows_a_p * 128 + (size_t)p.b_groups * Rp * 128);
      const size_t fixed = 1024 + 128 + (p.bias_grp >= 0 ? (size_t)(Rp + 8) * 128 : 0);
      if (fixed + stage > (size_t)kMaxDynSmem) continue;
      const int ns = (int)std::min<size_t>(kWgTmaMaxStages, ((size_t)kMaxDynSmem - fixed) / stage);
      if (ns > best_ns) { best_ns = ns; best_tt = tt; }
      if (ns >= 3) break;
    }
    if (best_ns < 2) return make_plan(d, false, plan_only);
    x.tt = best_tt; x.R = best_tt * p.nsub; x.Rp = (x.R + 15) & ~15;
    x.a_box_t = best_tt + pl.max_span_q;
    x.rows_a_p = (x.Rp + pl.max_span_q * p.nsub + 7) & ~7;
    x.nstages = best_ns;
    {
      const size_t stage = 2 * ((size_t)p.a_groups * x.rows_a_p * 128 + (size_t)p.b_groups * x.Rp * 128);
      pl.smem_tma = 1024 + 128 + (p.bias_grp >= 0 ? (size_t)(x.Rp + 8) * 128 : 0) + (size_t)best_ns * stage;
    }
    pl.tma = true;
    x.chunks_per_batch = ceil_div(p.M, x.tt);
    const long long units_t = (long long)p.batch * x.chunks_per_batch;
    // split-K: a chunk costs ~2 us here (TMA + MMAs), one more partial copy of the gradient out_bytes / ~4 TB/s twice
    // (all in us) a chunk: the larger of its loads (~1.5 us per 70 KB at the observed ~45 GB/s per SM) and its MMAs (12 per unit
    // and 64 rows, N / 2 cycles each); one split more: one more partial copy written and read back (~4 TB/s), and the
    // reduce pass itself (~5 us) which a single split does not need at all (the kernel then writes dw directly)
    int u_max = 1;
    for (int g = 0; g < p.ngroups; ++g) u_max = std::max(u_max, p.grp_first_unit[g + 1] - p.grp_first_unit[g]);
    const double stage_kb = 2.0 * (p.a_groups * x.rows_a_p + p.b_groups * x.Rp) * 128 / 1024.0;
    const double chunk_us = std::max(stage_kb / 45.0, u_max * 3.0 * (x.Rp / 16) * (p.NT / 2) / 1900.0);
    const double out_us = (double)p.taps_total * p.ca_g0 * cb * 8.0 / 4e12 * 1e6;
    long long ns_best = 1;
    double cbest = 1e30;
    for (long long ns = 1; ns <= std::min<long long>(units_t, 296); ++ns) {
      const long long waves = (base * ns + sms - 1) / sms;
      const double cost = (double)waves * (double)((units_t + ns - 1) / ns) * chunk_us + (ns > 1 ? 5.0 + (double)ns * out_us : 0.0);
      if (cost < cbest - 1e-9) { cbest = cost; ns_best = ns; }
    }
    pl.nsplit_tma = (int)ns_best;
    pl.part_floats = (ns_best * p.split_stride + 63) & ~63LL;
    const long long fa = ((long long)p.batch * p.t_a * p.nsub * ca + 63) & ~63LL;     // floats = 2 planes x bf16
    const long long fb = ((long long)p.batch * p.t_b * p.nsub * cb + 63) & ~63LL;
    pl.planes_a_off = pl.part_floats;
    pl.planes_b_off = pl.part_floats + fa;
    pl.ws_floats = pl.part_floats + fa + fb;
  }
  return pl;
}

// development / test aid (kt_debug_wgrad_plan): the TMA variant's plan of a layer as it would be made on a GPU box
// out = {ok, tma, tt, R, Rp, nstages, smem bytes, nsplit, NT, unit groups, a_box_t, rows_a_p}
void debug_wgrad_plan(const KtConv1dDesc* d, int* out) {
  const WgPlan pl = make_plan(d, true, true);
  out[0] = pl.ok; out[1] = pl.tma; out[2] = pl.x.tt; out[3] = pl.x.R; out[4] = pl.x.Rp; out[5] = pl.x.nstages;
  out[6] = (int)(pl.tma ? pl.smem_tma : pl.smem); out[7] = pl.tma ? pl.nsplit_tma : pl.p.nsplit; out[8] = pl.p.NT; out[9] = pl.p.ngroups;
  out[10] = pl.x.a_box_t; out[11] = pl.x.rows_a_p;
}

// floats of workspace needed by conv1d_bwd_weight_tc (0 = layer not supported)
bool thin_cin1_ok(const KtConv1dDesc* d);   // thin.cu

long long wgrad_tc_workspace(const KtConv1dDesc* d) {
  if (d->path != KT_PATH_TC && thin_cin1_ok(d)) return 0;   // waveform-input layers: thin.cu
  const WgPlan pl = make_plan(d);
  return pl.ok ? pl.ws_floats : 0;
}

int colsum_bias(const Side& s, long long rows, int c, float* out, cudaStream_t st);  // conv_ffma.cu

int conv1d_bwd_weight_tc(const KtConv1dDesc* d, const float* x, const float* dy, const float* y, float* dw,
                         float* dbias, float* ws, long long ws_floats, cudaStream_t st) {
  WgPlan pl = make_plan(d);
  KT_REQUIRE(pl.ok, "conv1d_bwd_weight_tc: layer not supported by the tensor-core path");
  KT_REQUIRE(ws && ws_floats >= pl.ws_floats, "conv1d_bwd_weight_tc: workspace too small (%lld < %lld floats)", ws_floats, pl.ws_floats);
  KT_REQUIRE(d->act_out == KT_ACT_NONE || y != nullptr, "bwd_weight: y required when act_out != NONE");
  WgTcParams& p = pl.p;
  const Side sx{x, nullptr, d->act_in == KT_ACT_LRELU ? SIDE_LRELU : SIDE_PLAIN, d->act_in_slope};
  Side sdy{dy, y, SIDE_PLAIN, d->act_out_slope};
  if (d->act_out == KT_ACT_LRELU) sdy.mode = SIDE_DLRELU;
  else if (d->act_out == KT_ACT_TANH) sdy.mode = SIDE_DTANH;
  else sdy.aux = nullptr;
  if (d->transposed) { p.a = sdy; p.b = sx; }
  else { p.a = sx; p.b = sdy; }
  p.ws = ws;
  p.bias_direct = nullptr;
  if (pl.tma) p.nsplit = pl.nsplit_tma;
  if (dbias == nullptr) p.bias_grp = -1;
  const bool direct = p.nsplit == 1;      // one split: the partial tile IS the gradient
  if (direct) { p.ws = dw; p.bias_direct = dbias; }
  if (pl.tma) {
    WgTmaExtra& x = pl.x;
    __nv_bfloat16* pa = reinterpret_cast<__nv_bfloat16*>(ws + pl.planes_a_off);
    __nv_bfloat16* pb = reinterpret_cast<__nv_bfloat16*>(ws + pl.planes_b_off);
    const long long na = (long long)p.batch * p.t_a * p.nsub * p.ca, nb = (long long)p.batch * p.t_b * p.nsub * p.cb;
    auto blocks_for = [](long long n8) { return (int)std::max<long long>(1, std::min<long long>((n8 + 255) / 256, 132LL * 16)); };
    if (!(debug_flags() & 256)) {
      const int ba = blocks_for(na / 8), bb = blocks_for(nb / 8);
      split_planes_kernel<<<ba + bb, 256, 0, st>>>(p.a, na / 8, pa, p.b, nb / 8, pb, ba);
    }
    KT_CHECK_CUDA(cudaGetLastError());
    const cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    {
      const cuuint64_t gdim[5] = {(cuuint64_t)p.cb, (cuuint64_t)p.nsub, (cuuint64_t)p.t_b, (cuuint64_t)p.batch, 2};
      const cuuint64_t gstr[4] = {(cuuint64_t)p.cb * 2, (cuuint64_t)p.nsub * p.cb * 2, (cuuint64_t)p.t_b * p.nsub * p.cb * 2, (cuuint64_t)nb * 2};
      const cuuint32_t box[5] = {64, (cuuint32_t)p.nsub, (cuuint32_t)x.tt, 1, 1};
      const CUresult r = encode_tiled_fn()(&x.map_b, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, pb, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                           CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      KT_REQUIRE(r == CUDA_SUCCESS, "conv1d_bwd_weight_tc: cuTensorMapEncodeTiled(B) failed (%d)", (int)r);
    }
    for (int rho = 0; rho < p.step; ++rho) {
      const cuuint64_t gdim[5] = {(cuuint64_t)p.ca, (cuuint64_t)p.nsub, (cuuint64_t)ceil_div(p.t_a - rho, p.step), (cuuint64_t)p.batch, 2};
      const cuuint64_t gstr[4] = {(cuuint64_t)p.ca * 2, (cuuint64_t)p.step * p.nsub * p.ca * 2, (cuuint64_t)p.t_a * p.nsub * p.ca * 2, (cuuint64_t)na * 2};
      const cuuint32_t box[5] = {64, (cuuint32_t)p.nsub, (cuuint32_t)x.a_box_t, 1, 1};
      const CUresult r = encode_tiled_fn()(&x.map_a[rho], CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, pa + (long long)rho * p.nsub * p.ca, gdim, gstr, box, estr,
                                           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      KT_REQUIRE(r == CUDA_SUCCESS, "conv1d_bwd_weight_tc: cuTensorMapEncodeTiled(A, residue %d) failed (%d)", rho, (int)r);
    }
    static std::atomic<bool> cfg_t{false};
    if (!cfg_t.load(std::memory_order_acquire)) {
      KT_CHECK_CUDA(cudaFuncSetAttribute(wgrad_tma_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem));
      KT_CHECK_CUDA(cudaFuncSetAttribute(wgrad_tma_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem));
      cfg_t.store(true, std::memory_order_release);
    }
    dim3 grid(p.groups * p.n_ca_tiles * p.n_cb_tiles, p.ngroups, p.nsplit);
    if (!(debug_flags() & 512)) {
      if (p.NT == 64) wgrad_tma_kernel<64><<<grid, kWgTmaThreads, pl.smem_tma, st>>>(p, x);
      else wgrad_tma_kernel<128><<<grid, kWgTmaThreads, pl.smem_tma, st>>>(p, x);
    }
    KT_CHECK_CUDA(cudaGetLastError());
  } else {
  static std::atomic<bool> cfg{false};
  if (!cfg.load(std::memory_order_acquire)) {
    KT_CHECK_CUDA(cudaFuncSetAttribute(wgrad_tc_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem));
    KT_CHECK_CUDA(cudaFuncSetAttribute(wgrad_tc_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem));
    cfg.store(true, std::memory_order_release);
  }
  dim3 grid(p.groups * p.n_ca_tiles * p.n_cb_tiles, p.ngroups, p.nsplit);
  if (p.NT == 64) wgrad_tc_kernel<64><<<grid, kWgThreads, pl.smem, st>>>(p);
  else wgrad_tc_kernel<128><<<grid, kWgThreads, pl.smem, st>>>(p);
  KT_CHECK_CUDA(cudaGetLastError());
  }
  const long long n = (long long)p.taps_total * p.ca_g0 * p.cb;
  const int blocks = (int)std::max<long long>(1, std::min<long long>((n / 4 + 255) / 256, 132LL * 8));
  const bool fused_bias = dbias != nullptr && p.bias_grp >= 0;
  if (direct || (debug_flags() & 1024)) {
    // nothing to reduce (or ablation)
  } else if (p.nsplit >= 16) {
    const long long warps = n / 4 + d->c_out;
    const int wblocks = (int)std::max<long long>(1, std::min<long long>((warps + 7) / 8, 132LL * 8));
    wgrad_reduce_wide_kernel<<<wblocks, 256, 0, st>>>(ws, dw, n, p.nsplit, p.split_stride, fused_bias ? dbias : nullptr, p.bias_off, d->c_out);
  } else {
    wgrad_reduce_kernel<<<blocks, 256, 0, st>>>(ws, dw, n, p.nsplit, p.split_stride, fused_bias ? dbias : nullptr, p.bias_off, d->c_out);
  }
  KT_CHECK_CUDA(cudaGetLastError());
  if (dbias && !fused_bias) {
    const long long rows = (long long)d->batch * d->nsub * d->t_out;
    int rc = colsum_bias(sdy, rows, d->c_out, dbias, st);
    if (rc) return rc;
  }
  return KT_OK;
}

}  // namespace kt
