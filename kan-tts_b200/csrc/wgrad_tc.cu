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
// Single-pass bf16 (KT_PATH_BF16): the instances with PL = 1 stage / load one bf16 plane per operand and issue the hi * hi
// wgmma alone; the split-K partials, their reduces and the summation order are those of bf16x3 (PL = 2).
#include <algorithm>

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
  int planes;                  // bf16 planes per operand image: 2 bf16x3, 1 single-pass bf16 (the instance's PL)
  int nsplit, chunks_per_batch;   // chunk = kWgTK flattened rows (register-staged) or tt base time steps (TMA)
  int a_groups, b_groups;      // 64-channel images per stage on each side
  int rows_a;                  // register-staged route: A image rows (max over unit groups), multiple of 8
  int ngroups;                 // unit groups (grid.y)
  int grp_rho[kWgMaxGroups], grp_qlo[kWgMaxGroups];
  int grp_first_unit[kWgMaxGroups + 1];
  int unit_tap0[kMaxTaps];     // first tap (index into tap_j / tap_q) of each unit
  int unit_ntaps[kMaxTaps];    // 1 or 2
  int tap_j[kMaxTaps];
  int tap_q[kMaxTaps];
  long long split_stride;      // floats between two splits' partial gradients in ws
};

// The work of one CTA: (conv group cgrp, ca tile, cb tile) = blockIdx.x, unit group grp = blockIdx.y (units [u0, u0 + nu) of one
// residue class, lowest tap shift qlo), split-K slice split = blockIdx.z: chunks [c_begin, c_end) of the (batch, chunk) range
struct WgCta {
  int cb_tile, ca_tile, cgrp, grp, u0, nu, qlo, split;
  long long c_begin, c_end;
  __device__ __forceinline__ explicit WgCta(const WgTcParams& p) {
    cb_tile = blockIdx.x % p.n_cb_tiles;
    ca_tile = (blockIdx.x / p.n_cb_tiles) % p.n_ca_tiles;
    cgrp = blockIdx.x / (p.n_cb_tiles * p.n_ca_tiles);
    grp = blockIdx.y;
    u0 = p.grp_first_unit[grp];
    nu = p.grp_first_unit[grp + 1] - u0;
    qlo = p.grp_qlo[grp];
    split = blockIdx.z;
    const long long units = (long long)p.batch * p.chunks_per_batch;
    c_begin = units * split / p.nsplit;
    c_end = units * (split + 1) / p.nsplit;
  }
};

// Consumers: two warpgroups, warpgroup cw owns rows [64 cw, 64 cw + 64) of the M = 128 accumulator block of every unit (U =
// 128 / NT units of NT columns: 64 fp32 registers per thread).  Mode 0: rows = channels [128 ca_tile + 64 cw, +64) -- the
// second 64-channel image; mode 1: rows = channels of tap 2u + cw of the unit -- the image row-shifted by the tap distance.
constexpr int kWgConsumerArrivals = 8;   // one per consumer warp

// MMAs of one staged chunk for one unit (accumulators acc[OFF, OFF + NT / 2)): A (M = 64 channels x K rows) and B (K rows x
// NT channels) are MN-major images, the hi / lo planes img16 apart, K = 16 rows = 128 descriptor units per slice (PL = 1: the
// hi * hi product only)
template <int NT, int OFF, int PL>
__device__ __forceinline__ void wg_unit_mma(float (&acc)[kWgmmaMaxRegs], uint32_t a_hi, uint32_t img_a16, uint32_t b_hi, uint32_t img_b16,
                                            int kslices) {
  for (int ks = 0; ks < kslices; ++ks) {
    const uint32_t ko = (uint32_t)ks * 128u;
    if constexpr (PL == 2) {
      wgmma_bf16_n<NT, 1, 1, OFF>(acc, desc_lo(a_hi + ko + img_a16), desc_lo(b_hi + ko), 1u);
      wgmma_bf16_n<NT, 1, 1, OFF>(acc, desc_lo(a_hi + ko), desc_lo(b_hi + ko + img_b16), 1u);
    }
    wgmma_bf16_n<NT, 1, 1, OFF>(acc, desc_lo(a_hi + ko), desc_lo(b_hi + ko), 1u);
  }
}

// all units of one staged chunk, then wait for the MMAs (the stage is released by the caller)
template <int NT, int PL>
__device__ __forceinline__ void wg_chunk_mma(float (&acc)[kWgmmaMaxRegs], uint32_t sbase16, uint32_t b_hi, uint32_t img_a16, uint32_t img_b16,
                                             const uint32_t* s_shift, const uint32_t* s_half, int nu, int cw, int kslices) {
  wgmma_fence();
  wg_unit_mma<NT, 0, PL>(acc, sbase16 + s_shift[0] + (cw ? s_half[0] : 0u), img_a16, b_hi, img_b16, kslices);
  if constexpr (kWgmmaMaxN / NT > 1) {
    if (nu > 1) wg_unit_mma<NT, NT / 2, PL>(acc, sbase16 + s_shift[1] + (cw ? s_half[1] : 0u), img_a16, b_hi, img_b16, kslices);
  }
  wgmma_commit();
  wgmma_wait<0>();
  acc_fence(acc);
}

// registers -> workspace partial tiles (or dw itself when there is one split)
template <int NT>
__device__ __forceinline__ void wg_store(const WgTcParams& p, const WgCta& cta, const float (&acc)[kWgmmaMaxRegs], int cw, int wq,
                                         int lane) {
  const int cb_tile = cta.cb_tile, ca_tile = cta.ca_tile, cgrp = cta.cgrp, u0 = cta.u0, nu = cta.nu, split = cta.split;
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
// (img_a: bytes of ALL planes of one A image, the distance of two 64-channel images)
__device__ __forceinline__ void wg_unit_table(const WgTcParams& p, const WgCta& cta, int img_a, uint32_t* s_shift, uint32_t* s_half) {
  for (int u = threadIdx.x; u < cta.nu; u += blockDim.x) {
    const int n_a = p.unit_tap0[cta.u0 + u];
    uint32_t half;
    if (p.mode == 0) half = (uint32_t)img_a;
    // mode 1: second half of M = the next tap of the same residue (rows 64..127 are discarded when the unit has one tap)
    else half = p.unit_ntaps[cta.u0 + u] == 2 ? (uint32_t)((p.tap_q[n_a + 1] - p.tap_q[n_a]) * p.nsub) * 128u : 128u;
    s_shift[u] = ((uint32_t)((p.tap_q[n_a] - cta.qlo) * p.nsub) * 128u) >> 4;
    s_half[u] = half >> 4;
  }
}

// warpgroups 0 / 3: producers of the even / odd chunks; warpgroups 1 / 2: consumers (MMAs + epilogue).  The kernel is bound
// by the ISSUE rate of the fp32 -> split-bf16 staging (~80 instructions per 8 elements), so the producers are 8 warps.
constexpr int kWgThreads = 512;

// (PL: bf16 planes per operand image; kernels wgrad_tc_kernel / wgrad_tc_bf16_kernel)
template <int NT, int PL>
__device__ __forceinline__ void wgrad_tc_body(const WgTcParams& p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_align_1024(smem_raw);
  const int img_a = p.rows_a * 128;            // one plane of one A image
  const int img_b = kWgTK * 128;               // one plane of one B image
  const int stage_bytes = PL * (p.a_groups * img_a + p.b_groups * img_b);
  uint8_t* stage0 = smem;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + 2 * (size_t)stage_bytes);
  uint64_t* full = bars;        // [2] producers -> MMA
  uint64_t* empty = bars + 2;   // [2] MMA -> producers
  uint32_t* s_shift = reinterpret_cast<uint32_t*>(bars + 4);   // [kWgMaxUnits]
  uint32_t* s_half = s_shift + kWgMaxUnits;                    // [kWgMaxUnits]

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const WgCta cta(p);

  if (tid == 0) {
    for (int s = 0; s < 2; ++s) { mbar_init(&full[s], 128); mbar_init(&empty[s], kWgConsumerArrivals); }
    mbar_fence_init();
    fence_proxy_async();
  }
  wg_unit_table(p, cta, PL * img_a, s_shift, s_half);
  __syncthreads();

  if (warp < 4 || warp >= 12) {
    // ===================== producers =====================
    const int pg = warp < 4 ? 0 : 1;                                       // pipeline stage this group fills
    const int ptid = tid & 127;
    int it = 0;
    for (long long c = cta.c_begin; c < cta.c_end; ++c, ++it) {
      const int s = it & 1;
      if (s != pg) continue;
      mbar_wait(&empty[s], ((it >> 1) & 1) ^ 1);
      const int bb = (int)(c / p.chunks_per_batch);
      const int f0 = (int)(c % p.chunks_per_batch) * kWgTK;
      uint8_t* st = stage0 + (size_t)s * stage_bytes;
      RowMap ra;  // gathered side: residue image of this unit group
      ra.base_row = (long long)bb * p.t_a * p.nsub;
      ra.fv0 = f0 + cta.qlo * p.nsub;
      ra.nsub = p.nsub; ra.step = p.step; ra.rho = p.grp_rho[cta.grp]; ra.up = p.up; ra.t_lim = p.t_a * p.up;
      for (int g = 0; g < p.a_groups; ++g) {
        uint8_t* hi = st + (size_t)g * PL * img_a;
        const int c_lo = cta.ca_tile * (p.mode == 0 ? 128 : 64) + g * 64;           // channel offset inside the group
        stage_rows<4, false, 2, false, false, PL>(hi, hi + img_a, p.a, p.a.p, p.a.aux, p.ca, cta.cgrp * p.ca_g + c_lo, min(64, p.ca_g - c_lo), true, ra,
                                p.rows_a, ptid);
      }
      RowMap rb;  // base side: rows m (flattened with w), zero beyond M
      rb.base_row = (long long)bb * p.t_b * p.nsub;
      rb.fv0 = f0; rb.nsub = p.nsub; rb.step = 1; rb.rho = 0; rb.up = 1; rb.t_lim = min(p.M, p.t_b);
      uint8_t* bst = st + (size_t)p.a_groups * PL * img_a;
      for (int g = 0; g < p.b_groups; ++g) {
        uint8_t* hi = bst + (size_t)g * PL * img_b;
        const int c_lo = cta.cb_tile * NT + g * 64;
        stage_rows<2, false, 2, false, false, PL>(hi, hi + img_b, p.b, p.b.p, p.b.aux, p.cb, cta.cgrp * p.cb_g + c_lo, min(64, p.cb_g - c_lo), true, rb,
                                kWgTK, ptid);
      }
      fence_proxy_async();
      mbar_arrive(&full[s]);
    }
  } else {
    // ===================== consumers =====================
    const int cw = (warp - 4) >> 2, wq = warp & 3;
    const uint32_t lbo_b16 = (((uint32_t)PL * (uint32_t)img_b) >> 4) << 16;
    const uint32_t img_a16 = (uint32_t)img_a >> 4, img_b16 = (uint32_t)img_b >> 4;
    const uint32_t st16[2] = {smem_u32(stage0) >> 4, smem_u32(stage0 + stage_bytes) >> 4};
    const uint32_t boff16 = (uint32_t)(p.a_groups * PL * img_a) >> 4;
    float acc[kWgmmaMaxRegs];
#pragma unroll
    for (int i = 0; i < kWgmmaMaxRegs; ++i) acc[i] = 0.f;
    int it = 0;
    for (long long c = cta.c_begin; c < cta.c_end; ++c, ++it) {
      const int s = it & 1;
      mbar_wait(&full[s], (it >> 1) & 1);
      wg_chunk_mma<NT, PL>(acc, st16[s], (st16[s] + boff16) | lbo_b16, img_a16, img_b16, s_shift, s_half, cta.nu, cw, kWgTK / 16);
      if (lane == 0) mbar_arrive(&empty[s]);
    }
    wg_store<NT>(p, cta, acc, cw, wq, lane);
  }
}

template <int NT>
__global__ void __launch_bounds__(kWgThreads, 1) wgrad_tc_kernel(const __grid_constant__ WgTcParams p) { wgrad_tc_body<NT, 2>(p); }
template <int NT>
__global__ void __launch_bounds__(kWgThreads, 1) wgrad_tc_bf16_kernel(const __grid_constant__ WgTcParams p) { wgrad_tc_body<NT, 1>(p); }

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
  alignas(64) CUtensorMap map_b;
  alignas(64) CUtensorMap map_a[8];   // one per residue class of the input
};

// (the operand planes are written by split_planes, tc_common.cuh)
// (kernels wgrad_tma_kernel / wgrad_tma_bf16_kernel)
template <int NT, int PL>
__device__ __forceinline__ void wgrad_tma_body(const WgTcParams& p, const WgTmaExtra& x) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_align_1024(smem_raw);
  const int img_a = x.rows_a_p * 128;          // one plane of one A image
  const int img_b = x.Rp * 128;                // one plane of one B image
  const int stage_bytes = PL * (p.a_groups * img_a + p.b_groups * img_b);
  uint8_t* stage0 = smem;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)x.nstages * stage_bytes);
  uint64_t* full = bars;                        // [nstages] TMA -> MMA
  uint64_t* empty = bars + kWgTmaMaxStages;     // [nstages] MMA -> TMA
  uint32_t* s_shift = reinterpret_cast<uint32_t*>(bars + 2 * kWgTmaMaxStages);   // [kWgMaxUnits]
  uint32_t* s_half = s_shift + kWgMaxUnits;                                     // [kWgMaxUnits]

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const WgCta cta(p);

  if (tid == 0) {
    for (int s = 0; s < x.nstages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], kWgConsumerArrivals); }
    mbar_fence_init();
  }
  {  // padding rows of every image (never written by the TMA boxes): zero, so that a partial last K slice contributes nothing
    const int a_box_rows = x.a_box_t * p.nsub;
    const int n_img = PL * (p.a_groups + p.b_groups);
    for (int s = 0; s < x.nstages; ++s)
      for (int i = 0; i < n_img; ++i) {
        const bool is_a = i < PL * p.a_groups;
        uint8_t* img = stage0 + (size_t)s * stage_bytes + (is_a ? (size_t)i * img_a : (size_t)PL * p.a_groups * img_a + (size_t)(i - PL * p.a_groups) * img_b);
        const int r0 = is_a ? a_box_rows : x.R, r1 = is_a ? x.rows_a_p : x.Rp;
        for (int o = r0 * 128 + tid * 16; o < r1 * 128; o += kWgTmaThreads * 16) *reinterpret_cast<uint4*>(img + o) = make_uint4(0u, 0u, 0u, 0u);
      }
  }
  wg_unit_table(p, cta, PL * img_a, s_shift, s_half);
  fence_proxy_async();
  __syncthreads();

  if (warp == 8) {
    // ===================== TMA producer =====================
    if (elect_one()) {
      const uint32_t tx = (uint32_t)PL * (uint32_t)(p.a_groups * x.a_box_t * p.nsub + p.b_groups * x.R) * 128u;
      const CUtensorMap* ma = &x.map_a[p.grp_rho[cta.grp]];
      const int ca0 = cta.cgrp * p.ca_g + cta.ca_tile * (p.mode == 0 ? 128 : 64);
      const int cb0 = cta.cgrp * p.cb_g + cta.cb_tile * NT;
      RingPos r;
      for (long long c = cta.c_begin; c < cta.c_end; ++c, r.advance(x.nstages)) {
        const int s = r.slot();
        mbar_wait(&empty[s], r.phase() ^ 1u);
        const int bb = (int)(c / p.chunks_per_batch);
        const int m0 = (int)(c % p.chunks_per_batch) * x.tt;
        uint8_t* st = stage0 + (size_t)s * stage_bytes;
        mbar_arrive_expect_tx(&full[s], tx);
        for (int g = 0; g < p.a_groups; ++g)
          for (int pl = 0; pl < PL; ++pl)
            tma_load_5d(st + (size_t)(PL * g + pl) * img_a, ma, ca0 + g * 64, 0, m0 + cta.qlo, bb, pl, &full[s]);
        uint8_t* bst = st + (size_t)p.a_groups * PL * img_a;
        for (int g = 0; g < p.b_groups; ++g)
          for (int pl = 0; pl < PL; ++pl)
            tma_load_5d(bst + (size_t)(PL * g + pl) * img_b, &x.map_b, cb0 + g * 64, 0, m0, bb, pl, &full[s]);
      }
      // every issued box has landed before the CTA may exit: the consumers waited for all of them
    }
    __syncwarp();
  } else {
    // ===================== consumers =====================
    const int cw = warp >> 2, wq = warp & 3;
    const uint32_t lbo_b16 = (((uint32_t)PL * (uint32_t)img_b) >> 4) << 16;
    const uint32_t img_a16 = (uint32_t)img_a >> 4, img_b16 = (uint32_t)img_b >> 4;
    const uint32_t st0_16 = smem_u32(stage0) >> 4, stage16 = (uint32_t)stage_bytes >> 4;
    const uint32_t boff16 = (uint32_t)(p.a_groups * PL * img_a) >> 4;
    const int kslices = x.Rp >> 4;
    float acc[kWgmmaMaxRegs];
#pragma unroll
    for (int i = 0; i < kWgmmaMaxRegs; ++i) acc[i] = 0.f;
    RingPos r;
    for (long long c = cta.c_begin; c < cta.c_end; ++c, r.advance(x.nstages)) {
      const int s = r.slot();
      mbar_wait(&full[s], r.phase());
      const uint32_t sbase = st0_16 + (uint32_t)s * stage16;
      wg_chunk_mma<NT, PL>(acc, sbase, (sbase + boff16) | lbo_b16, img_a16, img_b16, s_shift, s_half, cta.nu, cw, kslices);
      if (lane == 0) mbar_arrive(&empty[s]);
    }
    wg_store<NT>(p, cta, acc, cw, wq, lane);
  }
}

template <int NT>
__global__ void __launch_bounds__(kWgTmaThreads, 1) wgrad_tma_kernel(const __grid_constant__ WgTcParams p, const __grid_constant__ WgTmaExtra x) {
  wgrad_tma_body<NT, 2>(p, x);
}
template <int NT>
__global__ void __launch_bounds__(kWgTmaThreads, 1) wgrad_tma_bf16_kernel(const __grid_constant__ WgTcParams p,
                                                                          const __grid_constant__ WgTmaExtra x) {
  wgrad_tma_body<NT, 1>(p, x);
}

// sums the split-K partials: ws = [nsplit][stride] with stride >= n; elements [0, n) -> dw
__global__ void wgrad_reduce_kernel(const float* __restrict__ ws, float* __restrict__ dw, long long n, int nsplit, long long stride) {
  const long long gtid = blockIdx.x * (long long)blockDim.x + threadIdx.x, gsz = (long long)gridDim.x * blockDim.x;
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
__global__ void wgrad_reduce_wide_kernel(const float* __restrict__ ws, float* __restrict__ dw, long long n, int nsplit, long long stride) {
  const int lane = threadIdx.x & 31;
  const long long warp = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5, nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  const bool vec = ((n | stride) & 3) == 0;
  const long long items = vec ? n / 4 : n;
  for (long long i = warp; i < items; i += nwarps) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (vec) {
      for (int s = lane; s < nsplit; s += 32) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(ws + (long long)s * stride) + i);
        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
      }
    } else {
      for (int s = lane; s < nsplit; s += 32) acc.x += ws[(long long)s * stride + i];
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      acc.x += __shfl_xor_sync(0xffffffffu, acc.x, o); acc.y += __shfl_xor_sync(0xffffffffu, acc.y, o);
      acc.z += __shfl_xor_sync(0xffffffffu, acc.z, o); acc.w += __shfl_xor_sync(0xffffffffu, acc.w, o);
    }
    if (lane == 0) {
      if (vec) reinterpret_cast<float4*>(dw)[i] = acc;
      else dw[i] = acc.x;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// host
// ---------------------------------------------------------------------------------------------
struct WgPlan {
  bool ok;
  bool tma;                  // TMA-fed kernel (x filled in), else register-staged
  WgTcParams p;
  WgTmaExtra x;
  size_t smem;
  long long ws_floats;       // whole workspace: split-K partials, then on the TMA route the bf16 planes of both operands
  long long planes_a_off, planes_b_off;   // TMA route: offsets (floats) of the operand planes inside the workspace
};

// bytes of one ring stage: the planes of the A images (rows_a rows) and of the B images (rows_b rows)
static size_t wg_stage_bytes(const WgTcParams& p, int rows_a, int rows_b) {
  return (size_t)p.planes * ((size_t)p.a_groups * rows_a * 128 + (size_t)p.b_groups * rows_b * 128);
}

// split-K factor: the ns in [1, min(units, 296)] of least cost(waves, chunks per CTA, ns), the smaller on a tie.  `ctas`
// CTAs per split run one per SM in waves of one per SM.
template <class Cost>
static int split_k(long long units, long long ctas, Cost cost) {
  const int sms = device_sm_count();
  long long best_ns = 1;
  double best = 1e30;
  for (long long ns = 1; ns <= std::min<long long>(units, 296); ++ns) {
    const long long waves = (ctas * ns + sms - 1) / sms;
    const double c = cost((double)waves, (double)((units + ns - 1) / ns), ns);
    if (c < best - 1e-9) { best = c; best_ns = ns; }
  }
  return (int)best_ns;
}

static WgPlan make_plan(const KtConv1dDesc* d, bool plan_only = false) {
  WgPlan pl{};
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
  p.planes = d->path == KT_PATH_BF16 ? 1 : 2;
  p.t_a = tr ? d->t_out : d->t_in;
  p.t_b = tr ? d->t_in : d->t_out;
  p.M = p.t_b;
  p.step = d->stride;
  p.up = tr ? 1 : d->upsample;
  if (p.step > kMaxResidues) return pl;
  // channels are zero-padded to 64-wide images: thin / grouped layers use the same kernel
  p.mode = p.ca_g <= 64 ? 1 : 0;
  p.NT = std::min(kWgmmaMaxN, (p.cb_g + 63) & ~63);
  p.n_cb_tiles = ceil_div(p.cb_g, p.NT);
  p.n_ca_tiles = p.mode == 0 ? ceil_div(p.ca_g, 128) : 1;
  p.a_groups = p.mode == 0 ? 2 : 1;
  p.b_groups = p.NT / 64;
  const int U = std::min(kWgMaxUnits, kWgmmaMaxN / p.NT);
  const int taps_per_unit = p.mode == 1 ? 2 : 1;
  // taps by (residue, q, j): the gather phase of the gradient's contraction, as conv1d_bwd_weight_ffma runs it
  const ResidueTaps rt = residue_taps(gather_phase(p.M, d->kernel, p.step, d->dilation, d->pad_left, p.up), p.step);
  std::copy(rt.j, rt.j + rt.first[p.step], p.tap_j);
  std::copy(rt.q, rt.q + rt.first[p.step], p.tap_q);
  int nunit = 0, max_span_q = 0;
  for (int r = 0; r < p.step; ++r) {
    const int end = rt.first[r + 1];
    // the residue's units are spread EVENLY over its unit groups (5 taps, U = 4: groups of 3 + 2, not 4 + 1): every CTA loads
    // the same operand rows per chunk whatever its unit count, so the largest group sets the pace
    const int units_r = ceil_div(end - rt.first[r], taps_per_unit);
    const int groups_r = std::max(1, ceil_div(units_r, U));
    const int U_r = ceil_div(units_r, groups_r);
    for (int i = rt.first[r]; i < end;) {
      // one unit group: up to U_r units of this residue
      if (p.ngroups >= kWgMaxGroups) return pl;
      const int g = p.ngroups++;
      p.grp_rho[g] = r;
      p.grp_qlo[g] = rt.q[i];
      p.grp_first_unit[g] = nunit;
      for (int u = 0; u < U_r && i < end; ++u, ++nunit) {
        p.unit_tap0[nunit] = i;
        p.unit_ntaps[nunit] = std::min(taps_per_unit, end - i);
        i += p.unit_ntaps[nunit];
      }
      max_span_q = std::max(max_span_q, rt.q[i - 1] - p.grp_qlo[g]);
    }
  }
  p.grp_first_unit[p.ngroups] = nunit;
  // Whether a layer runs on the tensor cores does not depend on the route (a driver without tensor-map encoding plans the
  // same layers): the register-staged ring must fit on both.  (A smaller U would shrink the halo; not needed for the shipped
  // shapes.)
  const int rows_a = (kWgTK + max_span_q * p.nsub + 7) & ~7;
  pl.smem = 1024 + 2 * wg_stage_bytes(p, rows_a, kWgTK) + 128;
  if (pl.smem > (size_t)kMaxDynSmem) return pl;
  p.split_stride = (long long)p.taps_total * p.ca_g0 * cb;
  const double out_bytes = (double)p.taps_total * p.ca_g0 * cb * 8.0;   // one partial copy of the gradient, written and read
  const long long ctas = (long long)p.groups * p.n_ca_tiles * p.n_cb_tiles * p.ngroups;

  // TMA route (see wgrad_tma_kernel): plain convs whose box coordinates (multiples of the (super-)group widths) are 16-byte
  // aligned, with a time step in every residue class of the input.  Chunk = tt base time steps x nsub sub-sequences (R rows),
  // padded to whole K = 16 slices (Rp rows).  tt: the largest chunk (R <= 128 rows, at most 20 % padding in the last K slice)
  // that still leaves a ring of three stages; else the deepest ring, which must have two.
  int tt = 0, nstages = 0;
  if (!tr && p.up == 1 && (ca % 8) == 0 && (cb % 8) == 0 && (p.ca_g % 8) == 0 && (p.cb_g % 8) == 0 && p.t_a >= p.step &&
      (plan_only || encode_tiled_fn() != nullptr)) {   // plan_only: host-logic tests without a driver
    for (int t = std::max(1, 128 / p.nsub); t >= 1; --t) {
      const int R = t * p.nsub, Rp = (R + 15) & ~15;
      if (t + max_span_q > 256 || R > 256 || (t > 1 && R * 5 < Rp * 4)) continue;
      const size_t stage = wg_stage_bytes(p, (Rp + max_span_q * p.nsub + 7) & ~7, Rp);
      if (1024 + 128 + stage > (size_t)kMaxDynSmem) continue;
      const int ns = (int)std::min<size_t>(kWgTmaMaxStages, ((size_t)kMaxDynSmem - 1024 - 128) / stage);
      if (ns > nstages) { nstages = ns; tt = t; }
      if (ns >= 3) break;
    }
  }
  pl.tma = nstages >= 2;
  if (pl.tma) {
    WgTmaExtra& x = pl.x;
    x.tt = tt; x.R = tt * p.nsub; x.Rp = (x.R + 15) & ~15; x.nstages = nstages;
    x.a_box_t = tt + max_span_q;
    x.rows_a_p = (x.Rp + max_span_q * p.nsub + 7) & ~7;
    pl.smem = 1024 + 128 + (size_t)nstages * wg_stage_bytes(p, x.rows_a_p, x.Rp);
    p.chunks_per_batch = ceil_div(p.M, tt);
    // split-K cost (in us) of a chunk: the larger of its loads (~1.5 us per 70 KB at the observed ~45 GB/s per SM) and its MMAs
    // (12 per unit and 64 rows, N / 2 cycles each); of one split more: one more partial copy written and read back (~4 TB/s),
    // and the reduce pass itself (~5 us) which a single split does not need at all (the kernel then writes dw directly)
    int u_max = 1;
    for (int g = 0; g < p.ngroups; ++g) u_max = std::max(u_max, p.grp_first_unit[g + 1] - p.grp_first_unit[g]);
    const double stage_kb = (double)p.planes * (p.a_groups * x.rows_a_p + p.b_groups * x.Rp) * 128 / 1024.0;
    const double mmas = p.planes == 2 ? 3.0 : 1.0;   // wgmma per unit, K = 16 slice and 64 rows
    const double chunk_us = std::max(stage_kb / 45.0, u_max * mmas * (x.Rp / 16) * (p.NT / 2) / 1900.0);
    const double out_us = out_bytes / 4e12 * 1e6;
    p.nsplit = split_k((long long)p.batch * p.chunks_per_batch, ctas, [&](double waves, double chunks, long long ns) {
      return waves * chunks * chunk_us + (ns > 1 ? 5.0 + (double)ns * out_us : 0.0);
    });
    pl.planes_a_off = (p.nsplit * p.split_stride + 63) & ~63LL;
    pl.planes_b_off = pl.planes_a_off + plane_floats(p.batch, p.t_a, p.nsub, ca, p.planes);
    pl.ws_floats = pl.planes_b_off + plane_floats(p.batch, p.t_b, p.nsub, cb, p.planes);
  } else {
    p.rows_a = rows_a;
    p.chunks_per_batch = ceil_div(p.M * p.nsub, kWgTK);
    // split-K: minimise (waves x chunks per CTA) plus the cost of writing and re-reading one more partial copy of the gradient
    // (in units of one chunk ~ 10 us; ~4 TB/s effective)
    const double out_chunks = out_bytes / 4e12 / 10e-6;
    p.nsplit = split_k((long long)p.batch * p.chunks_per_batch, ctas, [&](double waves, double chunks, long long ns) {
      return waves * chunks + (double)ns * out_chunks;
    });
    pl.ws_floats = p.nsplit * p.split_stride;
  }
  pl.ok = true;
  return pl;
}

// development / test aid (kt_debug_wgrad_plan): the plan of a layer as it would be made on a GPU box
// out = {ok, tma, tt, R, Rp, nstages, smem bytes, nsplit, NT, unit groups, a_box_t, rows_a_p} (TMA-only entries 0 on the
// register-staged route)
extern "C" int kt_debug_wgrad_plan(const KtConv1dDesc* d, int32_t* out) {
  KT_REQUIRE(d && out, "kt_debug_wgrad_plan: null pointer");
  const WgPlan pl = make_plan(d, true);
  out[0] = pl.ok; out[1] = pl.tma; out[2] = pl.x.tt; out[3] = pl.x.R; out[4] = pl.x.Rp; out[5] = pl.x.nstages;
  out[6] = (int)pl.smem; out[7] = pl.p.nsplit; out[8] = pl.p.NT; out[9] = pl.p.ngroups;
  out[10] = pl.x.a_box_t; out[11] = pl.x.rows_a_p;
  return KT_OK;
}

// floats of workspace needed by kt_conv1d_bwd_weight_tc (0 = layer not supported)
extern "C" int64_t kt_conv1d_bwd_weight_tc_workspace(const KtConv1dDesc* d) {
  if (validate_conv(d)) return 0;
  if (d->path != KT_PATH_TC && thin_cin1_ok(d)) return 0;   // waveform-input layers: thin.cu
  const WgPlan pl = make_plan(d);
  return pl.ok ? pl.ws_floats : 0;
}

// the weight-gradient instance of one call: TMA-fed or register-staged, N tile 64 / 128, PL planes
template <int PL, bool TMA>
static int launch_wgrad(const WgTcParams& p, const WgTmaExtra& x, dim3 grid, size_t smem, cudaStream_t st) {
  if constexpr (TMA) {
    constexpr auto k64 = PL == 1 ? wgrad_tma_bf16_kernel<64> : wgrad_tma_kernel<64>;
    constexpr auto k128 = PL == 1 ? wgrad_tma_bf16_kernel<128> : wgrad_tma_kernel<128>;
    KT_CHECK_CUDA(allow_dyn_smem<k64>(kMaxDynSmem));
    KT_CHECK_CUDA(allow_dyn_smem<k128>(kMaxDynSmem));
    if (p.NT == 64) k64<<<grid, kWgTmaThreads, smem, st>>>(p, x);
    else k128<<<grid, kWgTmaThreads, smem, st>>>(p, x);
  } else {
    constexpr auto k64 = PL == 1 ? wgrad_tc_bf16_kernel<64> : wgrad_tc_kernel<64>;
    constexpr auto k128 = PL == 1 ? wgrad_tc_bf16_kernel<128> : wgrad_tc_kernel<128>;
    KT_CHECK_CUDA(allow_dyn_smem<k64>(kMaxDynSmem));
    KT_CHECK_CUDA(allow_dyn_smem<k128>(kMaxDynSmem));
    if (p.NT == 64) k64<<<grid, kWgThreads, smem, st>>>(p);
    else k128<<<grid, kWgThreads, smem, st>>>(p);
  }
  return KT_OK;
}

extern "C" int kt_conv1d_bwd_weight_tc(const KtConv1dDesc* d, const float* x, const float* dy, const float* y, float* dw,
                                       float* dbias, float* ws, int64_t ws_floats, void* stream) {
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  int rc = validate_conv(d);
  if (rc) return rc;
  KT_REQUIRE(x && dy && dw, "kt_conv1d_bwd_weight_tc: null pointer");
  WgPlan pl = make_plan(d);
  KT_REQUIRE(pl.ok, "conv1d_bwd_weight_tc: layer not supported by the tensor-core path");
  KT_REQUIRE(ws && ws_floats >= pl.ws_floats, "conv1d_bwd_weight_tc: workspace too small (%lld < %lld floats)", (long long)ws_floats,
             pl.ws_floats);
  KT_REQUIRE(d->act_out == KT_ACT_NONE || y != nullptr, "bwd_weight: y required when act_out != NONE");
  WgTcParams& p = pl.p;
  const Side sx = make_side(x, nullptr, d->act_in, d->act_in_slope, false);
  const Side sdy = make_side(dy, y, d->act_out, d->act_out_slope, true);
  if (d->transposed) { p.a = sdy; p.b = sx; }
  else { p.a = sx; p.b = sdy; }
  const bool direct = p.nsplit == 1;      // one split: the partial tile IS the gradient
  p.ws = direct ? dw : ws;
  const dim3 grid(p.groups * p.n_ca_tiles * p.n_cb_tiles, p.ngroups, p.nsplit);
  if (pl.tma) {
    WgTmaExtra& x = pl.x;
    __nv_bfloat16* pa = reinterpret_cast<__nv_bfloat16*>(ws + pl.planes_a_off);
    __nv_bfloat16* pb = reinterpret_cast<__nv_bfloat16*>(ws + pl.planes_b_off);
    const long long na = (long long)p.batch * p.t_a * p.nsub * p.ca, nb = (long long)p.batch * p.t_b * p.nsub * p.cb;
    KT_CHECK_CUDA(split_planes(p.a, na, pa, p.b, nb, pb, p.planes, st));
    rc = encode_plane_map(&x.map_b, pb, p.batch, p.t_b, p.nsub, p.cb, 1, 0, 64, x.tt, "conv1d_bwd_weight_tc (operand B)", p.planes);
    for (int rho = 0; rc == KT_OK && rho < p.step; ++rho)
      rc = encode_plane_map(&x.map_a[rho], pa, p.batch, p.t_a, p.nsub, p.ca, p.step, rho, 64, x.a_box_t, "conv1d_bwd_weight_tc (operand A)",
                            p.planes);
    if (rc) return rc;
    rc = p.planes == 1 ? launch_wgrad<1, true>(p, x, grid, pl.smem, st) : launch_wgrad<2, true>(p, x, grid, pl.smem, st);
  } else {
    rc = p.planes == 1 ? launch_wgrad<1, false>(p, pl.x, grid, pl.smem, st) : launch_wgrad<2, false>(p, pl.x, grid, pl.smem, st);
  }
  if (rc) return rc;
  KT_CHECK_CUDA(cudaGetLastError());
  const long long n = (long long)p.taps_total * p.ca_g0 * p.cb;
  if (p.nsplit >= 16) {
    const int wblocks = (int)std::max<long long>(1, std::min<long long>((n / 4 + 7) / 8, 132LL * 8));
    wgrad_reduce_wide_kernel<<<wblocks, 256, 0, st>>>(ws, dw, n, p.nsplit, p.split_stride);
  } else if (!direct) {
    const int blocks = (int)std::max<long long>(1, std::min<long long>((n / 4 + 255) / 256, 132LL * 8));
    wgrad_reduce_kernel<<<blocks, 256, 0, st>>>(ws, dw, n, p.nsplit, p.split_stride);
  }
  KT_CHECK_CUDA(cudaGetLastError());
  if (dbias) {
    const long long rows = (long long)d->batch * d->nsub * d->t_out;
    rc = colsum_bias(sdy, rows, d->c_out, dbias, st);
    if (rc) return rc;
  }
  return KT_OK;
}

}  // namespace kt
