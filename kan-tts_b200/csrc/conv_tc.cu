// wgmma implicit-GEMM Conv1d (forward / data-gradient) for the GEMM-shaped HiFi-GAN layers.
//
// Precision: "bf16x3".  Every fp32 operand is split x = hi + lo (two bf16, |x - hi - lo| <~ 2^-17 |x|)
// and the product is accumulated in fp32 registers as hi*hi + hi*lo + lo*hi (the dropped lo*lo term is
// ~2^-18 relative).  A single-pass TF32/BF16 MMA does not meet the path's tolerance (mel-L1 <= 1e-4,
// SURVEY.md "hard parts"); three bf16 MMAs do, at twice the rate of 3xTF32.
//
// Tile = 128 consecutive FLATTENED outputs (time m, sub-sequence w) of one batch item x NT (<= 128) channels.
// Data flow per CTA:
//   warpgroup 0  stages the channels-last fp32 activation rows (fused pre-activation / activation
//              derivative), split them into hi / lo bf16 planes and store SWIZZLE_128B shared-memory
//              images (rows = flattened (time, sub-sequence) positions of ONE input residue class).
//              im2col-free: tap j = residue image rho_j read through a wgmma descriptor whose start
//              address is shifted by q_j * nsub rows (the 128-byte swizzle is a function of absolute
//              smem address bits, so a row shift needs no re-phasing).  Stride s convs stage s residue
//              images per 64-channel chunk; the period discriminator's (k,1) Conv2d needs nothing extra.
//   warp 12    streams the pre-swizzled bf16 weight tiles (hi + lo, one tap x 64 input channels) with
//              cp.async.bulk (TMA engine) into a ring of shared-memory stages, mbarrier complete_tx.
//   warpgroups 1 / 2  wgmma (M = 64 rows each, N = NT, K = 16) x 4 k-slices x 3 products per (chunk, tap) into
//              register accumulators, then the epilogue of their 64 rows: bias / activation / residual (or act'
//              mask for the data gradient), stores to the channels-last output.
#include <algorithm>
#include <atomic>
#include <cstdlib>
#include <vector>

#include "common.cuh"
#include "tc_common.cuh"
#include "tma.cuh"

namespace kt {

using namespace tc;

constexpr int kTcM = 128;        // output rows per CTA
constexpr int kTcKC = 64;        // input channels per K chunk (one 128-byte swizzle row of bf16)
constexpr int kTcMaxRows = 256;  // image rows (128 + halo) upper bound
constexpr int kTcMaxGroups = 8;  // residue classes (= input step) per phase

// ---------------------------------------------------------------------------------------------
// weight packing: fp32 W[taps][K][N] (kernel layout of conv_ffma.cu) -> bf16 hi/lo SWIZZLE_128B tiles
//   block (j, kc, nt) = [hi tile | lo tile], tile = NT rows (n) x 64 (k) bf16, row = 128 bytes
// ---------------------------------------------------------------------------------------------
// K (contraction rows of W) is zero-padded to a multiple of 64 and every N tile to NT rows, so thin
// (C_in = 1, 32, 80, ...), single-output and GROUPED layers use the same kernel: tile nt covers the
// columns [nt * n_stride, nt * n_stride + min(n_stride, N - nt * n_stride)) of W (n_stride = NT for a
// dense layer, C_out / groups for a grouped one, whose W already has K = C_in / groups rows).
//
// GROUPED layers with thin groups pack `gt` consecutive groups into one tile as a BLOCK-DIAGONAL weight (K = gt *
// kin_g contraction channels, n_stride = gt * pout_g produced channels, zeros off the diagonal): a 128->256 g16
// layer (8 -> 16 channels per group) becomes 2 tiles of K = 64 x N = 128 instead of 16 tiles of K = 8 (padded to
// 16) x N = 16 -- 8x fewer tiles, each restaging the activations once, at MMA shapes the tensor pipe runs well.
// w is then [taps][kin_g][N] (rows = channels of ONE group) and K = gt * kin_g; kin_g = 0 means dense.
// One thread = one 16-byte chunk (8 consecutive k) of one tile row r: the 8 source loads are coalesced across the warp (lanes =
// consecutive produced channels n), the hi / lo chunks are written with two 16-byte stores (round 1 wrote single bf16
// elements: 2-byte scattered stores and five 64-bit divisions per element made this the 4th largest kernel of the step).
__global__ void tc_pack_weights_kernel(const float* __restrict__ w, int taps, int K, int N, int NT, int n_stride,
                                       int ntiles, int kin_g, int pout_g, __nv_bfloat16* __restrict__ out) {
  const int kchunks = (K + kTcKC - 1) / kTcKC;
  const int block = blockIdx.x;                                   // (j, kc, nt)
  const int nt = block % ntiles, kc = (block / ntiles) % kchunks, j = block / (ntiles * kchunks);
  uint8_t* tile = reinterpret_cast<uint8_t*>(out) + (size_t)block * (2u * NT * kTcKC * 2u);
  for (int idx = blockIdx.y * blockDim.x + threadIdx.x; idx < NT * 8; idx += gridDim.y * blockDim.x) {
    const int q = idx / NT, r = idx - q * NT;
    const int n = nt * n_stride + r;
    const bool row_ok = r < n_stride && n < N;
    float x[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int k = kc * kTcKC + q * 8 + e;
      bool ok = row_ok && k < K;
      long long src;
      if (kin_g > 0) {   // block diagonal: contraction channel k and produced channel r must be in the same group
        ok = ok && (k / kin_g) == (r / pout_g);
        src = ((long long)j * kin_g + (k % kin_g)) * N + n;
      } else {
        src = ((long long)j * K + k) * N + n;
      }
      x[e] = ok ? __ldg(w + src) : 0.f;
    }
    uint4 hi, lo;
    split8(x, hi, lo);
    const uint32_t o = sw128_offset((uint32_t)r, (uint32_t)q);
    *reinterpret_cast<uint4*>(tile + o) = hi;
    *reinterpret_cast<uint4*>(tile + (size_t)NT * kTcKC * 2 + o) = lo;
  }
}

// ---------------------------------------------------------------------------------------------
// conv kernel
// ---------------------------------------------------------------------------------------------
struct TcParams {
  Side in;
  const __nv_bfloat16* wimg;
  const float* bias;
  const float* resid;
  Side mask;
  float* out;
  int batch, nsub, t_in, t_out, c_in, c_out;
  int out_act;
  float out_slope;
  int NT, ntiles, kchunks, rows, na_stages, nb_stages;
  // 1: every (K chunk, tap) weight tile of the layer has its own shared-memory slot (slot = c * ntaps + n), loaded
  // ONCE per CTA and reused by all of its tiles -- thin layers otherwise re-stream all taps per 128-row tile through
  // a ring whose refill round trip (release -> empty -> bulk copy -> full) bounds the MMA issue rate
  int w_resident;
  int kg;        // contraction channels per tile (C_in, or C_in / groups)
  int grouped;   // 1: N tile nt = group nt (input channels [nt * kg, +kg), outputs [nt * n_stride, +n_stride))
  int n_stride;  // output channels advanced per N tile
  // phases: out[(o_off + o_step*m), w] = sum_n W[tap_j[n]] in[(m + q_n)*i_step + rho_n, w].  All polyphase
  // phases of a layer (the `stride` output residues of a transposed conv / strided data gradient) run in ONE
  // launch: the m-tile index space is the concatenation of the phases' tiles.
  int nphases;
  int ph_M[kTcMaxGroups], ph_ooff[kTcMaxGroups];
  int ph_mt0[kTcMaxGroups + 1];       // first m-tile of each phase
  int ph_g0[kTcMaxGroups + 1];        // first residue group of each phase
  int o_step, i_step, up, accumulate;
  int ngroups;                        // residue groups over all phases
  int grp_rho[kTcMaxGroups];
  int grp_qlo[kTcMaxGroups];
  int grp_first[kTcMaxGroups + 1];    // taps of group g: [grp_first[g], grp_first[g+1])
  int ntaps;
  int tap_j[kMaxTaps];                // weight tap index, ordered by group
  int tap_shift[kMaxTaps];            // image row shift (q_n - q_lo) * nsub
};

// Warp roles (416 threads): warpgroup 0 stages activations; warpgroups 1 and 2 are the consumers -- each runs the wgmma
// of one 64-row half of the 128-row tile into its registers and that half's epilogue; warp 12 streams weights.  (Warps
// hold registers in groups of four: 13 warps keep the 128 registers per thread the consumers' accumulators need.)
constexpr int kTcThreads = 416;
constexpr int kTcConsumerArrivals = 8;   // one per consumer warp

// Persistent: gridDim.x = min(#tiles, #SMs); each CTA walks tiles blockIdx.x, +gridDim.x, ...  The activation and
// weight pipelines run continuously ACROSS tiles, so staging of tile i+1 overlaps the MMAs and the epilogue of tile i.
// SIMPLE = true: nsub == 1, up == 1, vectorisable channel counts, no tanh / accumulate -- the generator's resblock
// convs, the scale discriminator and every SAM-BERT linear / conv (see stage_rows).  false: everything else.
template <bool SIMPLE>
__global__ void __launch_bounds__(kTcThreads, 1) conv_tc_kernel(const __grid_constant__ TcParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // carve-up (all image / tile bases 1024-byte aligned)
  // (pointer arithmetic on the __shared__ array, not integer casts: the compiler must keep the shared address space)
  uint8_t* smem = smem_raw + ((1024u - (tc::smem_u32(smem_raw) & 1023u)) & 1023u);
  const int img_bytes = p.rows * 128;                 // one plane of one activation stage
  const int a_stage_bytes = 2 * img_bytes;            // hi + lo
  const int b_stage_bytes = 2 * p.NT * 128;           // hi + lo weight tile
  uint8_t* a_base = smem;
  uint8_t* b_base = a_base + (size_t)p.na_stages * a_stage_bytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(b_base + (size_t)p.nb_stages * b_stage_bytes);
  uint64_t* full_a = bars;                         // [na]
  uint64_t* empty_a = full_a + p.na_stages;        // [na]
  uint64_t* full_b = empty_a + p.na_stages;        // [nb]
  uint64_t* empty_b = full_b + p.nb_stages;        // [nb]
  // per-tap image row shift in descriptor units (16 bytes)
  uint32_t* s_tapshift = reinterpret_cast<uint32_t*>(empty_b + p.nb_stages);   // [kMaxTaps]

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int mtiles = p.ph_mt0[p.nphases];   // m-tiles of all phases (each: 128 flattened outputs m * nsub + w)
  const int total_tiles = mtiles * p.ntiles * p.batch;

  if (tid == 0) {
    for (int s = 0; s < p.na_stages; ++s) { mbar_init(&full_a[s], 128); mbar_init(&empty_a[s], kTcConsumerArrivals); }
    for (int s = 0; s < p.nb_stages; ++s) { mbar_init(&full_b[s], 1); mbar_init(&empty_b[s], kTcConsumerArrivals); }
    mbar_fence_init();
    fence_proxy_async();
  }
  if (tid < kMaxTaps) s_tapshift[tid] = (uint32_t)p.tap_shift[tid] * 8u;
  __syncthreads();

  if (warp < 4) {
    // ===================== activation producers =====================
    const int ptid = tid;
    int it = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const int gm = tile % mtiles, bb = tile / (mtiles * p.ntiles);
      int ph = 0;
      while (gm >= p.ph_mt0[ph + 1]) ++ph;
      const int ch_base = p.grouped ? ((tile / mtiles) % p.ntiles) * p.kg : 0;
      const int f0 = (gm - p.ph_mt0[ph]) * kTcM;
      for (int c = 0; c < p.kchunks; ++c) {
        for (int g = p.ph_g0[ph]; g < p.ph_g0[ph + 1]; ++g, ++it) {
          const int s = it % p.na_stages;
          mbar_wait(&empty_a[s], ((it / p.na_stages) & 1) ^ 1);
          uint8_t* img_hi = a_base + (size_t)s * a_stage_bytes;
          RowMap rm;
          rm.base_row = (long long)bb * p.t_in * p.nsub;
          rm.fv0 = f0 + p.grp_qlo[g] * p.nsub;
          rm.nsub = p.nsub; rm.step = p.i_step; rm.rho = p.grp_rho[g]; rm.up = p.up; rm.t_lim = p.t_in * p.up;
          stage_rows<5, SIMPLE, 3>(img_hi, img_hi + img_bytes, p.in, p.in.p, p.in.aux, p.c_in, ch_base + c * kTcKC,
                                   min(kTcKC, p.kg - c * kTcKC), false, rm, p.rows, ptid);
          fence_proxy_async();
          mbar_arrive(&full_a[s]);
        }
      }
    }
  } else if (warp == 12) {
    // ===================== weight stream (bulk async copies) =====================
    const bool leader = elect_one();
    if (leader && p.w_resident) {
      if ((int)blockIdx.x < total_tiles) {
        for (int c = 0; c < p.kchunks; ++c)
          for (int n = 0; n < p.ntaps; ++n) {
            const int s = c * p.ntaps + n;
            const long long block = ((long long)p.tap_j[n] * p.kchunks + c) * p.ntiles;   // ntiles == 1
            const uint8_t* src = reinterpret_cast<const uint8_t*>(p.wimg) + block * (long long)b_stage_bytes;
            mbar_arrive_expect_tx(&full_b[s], (uint32_t)b_stage_bytes);
            bulk_g2s(b_base + (size_t)s * b_stage_bytes, src, (uint32_t)b_stage_bytes, &full_b[s]);
          }
        for (int s = 0; s < p.nb_stages; ++s) mbar_wait(&full_b[s], 0);   // no bulk copy may outlive the CTA
      }
    } else if (leader) {
      int it = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int nt = (tile / mtiles) % p.ntiles;
        int ph = 0;
        while ((tile % mtiles) >= p.ph_mt0[ph + 1]) ++ph;
        const int n_begin = p.grp_first[p.ph_g0[ph]], n_end = p.grp_first[p.ph_g0[ph + 1]];
        for (int c = 0; c < p.kchunks; ++c) {
          for (int n = n_begin; n < n_end; ++n, ++it) {  // taps are ordered by group: same order as the consumers
            const int s = it % p.nb_stages;
            mbar_wait(&empty_b[s], ((it / p.nb_stages) & 1) ^ 1);
            const long long block = ((long long)p.tap_j[n] * p.kchunks + c) * p.ntiles + nt;
            const uint8_t* src = reinterpret_cast<const uint8_t*>(p.wimg) + block * (long long)b_stage_bytes;
            mbar_arrive_expect_tx(&full_b[s], (uint32_t)b_stage_bytes);
            bulk_g2s(b_base + (size_t)s * b_stage_bytes, src, (uint32_t)b_stage_bytes, &full_b[s]);
          }
        }
      }
    }
    __syncwarp();
  } else if (warp >= 4 && warp < 12) {
    // ===================== consumers: wgmma + epilogue, one 64-row half of the tile per warpgroup =====================
    // Descriptor low words + 32-bit adds only: a tap's row shift, the K = 16 slice offset (32 bytes = 2 units), the hi -> lo
    // plane distance and this warpgroup's 64-row offset (8 KB = 512 units) are integer adds on the low word.
    const int cw = (warp - 4) >> 2;                  // 0: rows 0-63, 1: rows 64-127
    const int wq = warp & 3;                         // warp inside the warpgroup: rows 16 wq .. 16 wq + 15 of the half
    const uint32_t a_base16 = (smem_u32(a_base) >> 4) + (uint32_t)cw * 512u;
    const uint32_t b_base16 = smem_u32(b_base) >> 4;
    const uint32_t a_stage16 = (uint32_t)a_stage_bytes >> 4, img16 = (uint32_t)img_bytes >> 4;
    const uint32_t b_stage16 = (uint32_t)b_stage_bytes >> 4, bplane16 = (uint32_t)(p.NT * 128) >> 4;
    const bool resident = p.w_resident != 0;
    const int NT = p.NT;
    float acc[kWgmmaMaxRegs];
#pragma unroll
    for (int i = 0; i < kWgmmaMaxRegs; ++i) acc[i] = 0.f;
    int it_a = 0, it_b = 0, ti = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x, ++ti) {
      const int gm = tile % mtiles, nt = (tile / mtiles) % p.ntiles, bb = tile / (mtiles * p.ntiles);
      int ph = 0;
      while (gm >= p.ph_mt0[ph + 1]) ++ph;
      const int g_begin = p.ph_g0[ph], g_end = p.ph_g0[ph + 1];
      uint32_t scale_d = 0;
      for (int c = 0; c < p.kchunks; ++c) {
        const int kslices = (min(kTcKC, p.kg - c * kTcKC) + 15) >> 4;   // K = 16 slices holding real channels
        for (int g = g_begin; g < g_end; ++g, ++it_a) {
          const int sa = it_a % p.na_stages;
          mbar_wait(&full_a[sa], (it_a / p.na_stages) & 1);
          const uint32_t a16 = a_base16 + (uint32_t)sa * a_stage16;
          for (int n = p.grp_first[g]; n < p.grp_first[g + 1]; ++n, ++it_b) {
            int sb;
            if (resident) {
              sb = c * p.ntaps + n;
              if (ti == 0) mbar_wait(&full_b[sb], 0u);
            } else {
              sb = it_b % p.nb_stages;
              mbar_wait(&full_b[sb], (uint32_t)((it_b / p.nb_stages) & 1));
            }
            const uint32_t a_hi = a16 + s_tapshift[n];
            const uint32_t b_hi = b_base16 + (uint32_t)sb * b_stage16;
            wgmma_fence();
            for (int ks = 0; ks < kslices; ++ks) {
              wgmma_x3<0, 0>(NT, acc, a_hi + 2u * ks, img16, b_hi + 2u * ks, bplane16, scale_d);
              scale_d = 1;
            }
            wgmma_commit();
            wgmma_wait<0>();
            acc_fence(acc);
            if (!resident && lane == 0) mbar_arrive(&empty_b[sb]);
          }
          if (lane == 0) mbar_arrive(&empty_a[sa]);
        }
      }
      // ---- epilogue: registers -> bias / activation / residual (or act' mask for the data gradient) -> output rows
      const int mt = gm - p.ph_mt0[ph];
      const int F = p.ph_M[ph] * p.nsub;
      const int c_tile = nt * p.n_stride;
      const int n_valid = min(p.n_stride, p.c_out - c_tile);   // real output channels of this tile
      const bool vec2 = ((p.c_out | p.n_stride) & 1) == 0;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int f = mt * kTcM + cw * 64 + wq * 16 + (lane >> 2) + 8 * h;
        if (f >= F) continue;
        const int m = p.nsub == 1 ? f : f / p.nsub;
        const int w = f - m * p.nsub;
        const int to = p.ph_ooff[ph] + p.o_step * m;
        const long long obase = ((long long)(bb * p.t_out + to) * p.nsub + w) * p.c_out + c_tile;
#pragma unroll
        for (int i = 0; i < kWgmmaMaxN / 8; ++i) {
          const int col = i * 8 + 2 * (lane & 3);
          if (i * 8 >= NT || col >= n_valid) continue;
          float v[2] = {acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]};
          const bool pair = vec2 && col + 1 < n_valid;
          const int ne = col + 1 < n_valid ? 2 : 1;
          float bia[2] = {0.f, 0.f}, sd[2] = {0.f, 0.f}, md[2] = {0.f, 0.f}, od[2] = {0.f, 0.f};
          const long long o = obase + col;
          if (pair) {
            if (p.bias) { const float2 t = __ldg(reinterpret_cast<const float2*>(p.bias + c_tile + col)); bia[0] = t.x; bia[1] = t.y; }
            if (p.mask.p) { const float2 t = __ldg(reinterpret_cast<const float2*>(p.mask.p + o)); md[0] = t.x; md[1] = t.y; }
            if (p.resid) { const float2 t = __ldg(reinterpret_cast<const float2*>(p.resid + o)); sd[0] = t.x; sd[1] = t.y; }
            if (!SIMPLE && p.accumulate) { const float2 t = *reinterpret_cast<const float2*>(p.out + o); od[0] = t.x; od[1] = t.y; }
          } else {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              if (e >= ne) break;
              if (p.bias) bia[e] = __ldg(p.bias + c_tile + col + e);
              if (p.mask.p) md[e] = __ldg(p.mask.p + o + e);
              if (p.resid) sd[e] = __ldg(p.resid + o + e);
              if (!SIMPLE && p.accumulate) od[e] = p.out[o + e];
            }
          }
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            float x = v[e] + bia[e];
            if (p.out_act == KT_ACT_LRELU) x = x > 0.f ? x : x * p.out_slope;
            else if (!SIMPLE && p.out_act == KT_ACT_TANH) x = tanhf(x);
            if (p.mask.p) x = side_apply(x, md[e], p.mask.mode, p.mask.slope);
            x += sd[e] + od[e];
            v[e] = x;
          }
          if (pair) *reinterpret_cast<float2*>(p.out + o) = make_float2(v[0], v[1]);
          else {
            p.out[o] = v[0];
            if (ne == 2) p.out[o + 1] = v[1];
          }
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
// Layer-level tiling of one direction (0 forward, 1 data gradient).
struct TcLayerPlan {
  bool ok;
  int kg;        // contraction channels per tile
  int n_total;   // produced channels (tensor width)
  int n_stride;  // produced channels per N tile
  int NT;        // padded N tile (multiple of 16, <= 128: the accumulators live in registers)
  int ntiles, kchunks, grouped;
  int kin_g, pout_g;   // grouped: channels of ONE group on the contraction / produced side (kg = gt * kin_g)
};

std::vector<Phase> conv_phases(const KtConv1dDesc* d, int dir);  // conv_ffma.cu
struct TcParams;

// shared memory outside the activation / weight stages: barriers and the tap-shift table (see the carve-up in conv_tc_kernel)
static int tc_fixed_smem(int slots) { return (2 * 3 + 2 * std::max(6, slots)) * 8 + kMaxTaps * 4; }

static int sm_count();

static TcLayerPlan layer_plan(const KtConv1dDesc* d, int dir) {
  TcLayerPlan L{};
  const int g = d->groups;
  const int kin = (dir == 0 ? d->c_in : d->c_out) / g;     // contraction channels per group
  const int pout = (dir == 0 ? d->c_out : d->c_in) / g;    // produced channels per group
  L.kg = kin;
  L.n_total = pout * g;
  L.kchunks = ceil_div(kin, kTcKC);
  L.grouped = g > 1;
  if (g > 1) {
    if (pout > kWgmmaMaxN) return L;
    // groups per tile: fill one 64-channel K chunk, keep the N tile <= 128 (block-diagonal tile, see tc_pack_weights_kernel)
    int gt = 1;
    while (gt * 2 <= g && g % (gt * 2) == 0 && kin * gt * 2 <= kTcKC && pout * gt * 2 <= 128) gt *= 2;
    L.kin_g = kin; L.pout_g = pout;
    L.kg = gt * kin;
    L.kchunks = ceil_div(L.kg, kTcKC);
    L.n_stride = gt * pout; L.NT = (L.n_stride + 15) & ~15; L.ntiles = g / gt;
  } else if (pout <= 2 * kWgmmaMaxN) {
    // N tiles of <= 128 channels (a 64-row half tile's accumulators are 64 registers per thread at N = 128)
    L.ntiles = ceil_div(pout, kWgmmaMaxN);
    L.n_stride = (ceil_div(pout, L.ntiles) + 15) & ~15; L.NT = L.n_stride;
    // under-filled grids (short sequences x wide layers): split N so that >= ~1 tile per SM exists
    const long long mtiles = (long long)ceil_div((dir == 0 ? d->t_out : d->t_in) * d->nsub, kTcM) * d->batch;
    while (mtiles * L.ntiles < 120 && L.NT >= 128 && L.NT % 32 == 0 && pout % (L.NT / 2) == 0) {
      L.NT /= 2; L.n_stride = L.NT; L.ntiles = pout / L.NT;
    }
  } else {
    L.NT = pout % 128 == 0 ? 128 : 0;
    if (L.NT == 0) return L;
    L.n_stride = L.NT; L.ntiles = pout / L.NT;
  }
  L.ok = true;
  return L;
}

// Append one phase (its residue groups and taps) to the launch parameters.  Returns false when the
// phase does not fit the kernel's limits.  Call reset_phases() first.
static void reset_phases(TcParams& p) {
  p.nphases = 0; p.ngroups = 0; p.ntaps = 0; p.rows = 0;
  p.ph_mt0[0] = 0; p.ph_g0[0] = 0; p.grp_first[0] = 0;
}

static bool add_phase(TcParams& p, const Phase& ph, int nsub) {
  if (ph.M <= 0) return true;
  const int s = ph.i_step;
  if (s < 1 || s > kTcMaxGroups || p.nphases >= kTcMaxGroups) return false;
  if (p.nphases > 0 && (p.o_step != ph.o_step || p.i_step != ph.i_step || p.up != ph.up)) return false;
  p.o_step = ph.o_step; p.i_step = ph.i_step; p.up = ph.up; p.accumulate = ph.accumulate;
  int q[kMaxTaps], rho[kMaxTaps];
  for (int n = 0; n < ph.ntaps; ++n) {
    if (ph.tap_ioff[n] < -(1 << 24)) {  // placeholder tap of an output residue no real tap reaches
      q[n] = -(1 << 20); rho[n] = 0;
      continue;
    }
    q[n] = fdiv(ph.tap_ioff[n], s);
    rho[n] = ph.tap_ioff[n] - q[n] * s;
  }
  int max_span = 0;
  for (int r = 0; r < s; ++r) {
    int qlo = 1 << 30, qhi = -(1 << 30), cnt = 0;
    for (int n = 0; n < ph.ntaps; ++n)
      if (rho[n] == r) { qlo = std::min(qlo, q[n]); qhi = std::max(qhi, q[n]); ++cnt; }
    if (!cnt) continue;
    if (p.ngroups >= kTcMaxGroups || p.ntaps + cnt > kMaxTaps) return false;
    const int g = p.ngroups++;
    p.grp_rho[g] = r; p.grp_qlo[g] = qlo; p.grp_first[g] = p.ntaps;
    for (int n = 0; n < ph.ntaps; ++n)
      if (rho[n] == r) {
        p.tap_j[p.ntaps] = ph.tap_j[n];
        p.tap_shift[p.ntaps] = (q[n] - qlo) * nsub;
        ++p.ntaps;
      }
    p.grp_first[p.ngroups] = p.ntaps;
    max_span = std::max(max_span, (qhi - qlo) * nsub);
  }
  const int i = p.nphases++;
  p.ph_M[i] = ph.M; p.ph_ooff[i] = ph.o_off;
  p.ph_mt0[i + 1] = p.ph_mt0[i] + ceil_div(ph.M * nsub, kTcM);
  p.ph_g0[i + 1] = p.ngroups;
  p.rows = std::max(p.rows, (kTcM + max_span + 7) & ~7);
  return p.rows <= kTcMaxRows;
}

// Split the phases of a layer into launches: phases that fit together (and do not accumulate) share one.
static bool plan_launches(const std::vector<Phase>& phases, int nsub, std::vector<TcParams>& out, const TcParams& base) {
  TcParams cur = base;
  reset_phases(cur);
  for (const Phase& ph : phases) {
    TcParams trial = cur;
    if (ph.accumulate || cur.accumulate || !add_phase(trial, ph, nsub)) {
      if (cur.nphases > 0) out.push_back(cur);
      cur = base;
      reset_phases(cur);
      if (!add_phase(cur, ph, nsub)) return false;
    } else {
      cur = trial;
    }
  }
  if (cur.nphases > 0) out.push_back(cur);
  return true;
}

// Is (direction dir: 0 fwd, 1 bwd_data) of this layer runnable on the tensor-core kernel?  -> N tile or 0
bool thin_cin1_ok(const KtConv1dDesc* d);   // thin.cu

int tc_plan(const KtConv1dDesc* d, int dir) {
  if (dir == 0 && d->path != KT_PATH_TC && thin_cin1_ok(d)) return 0;   // waveform-input layers: HBM-bound FIR kernel
  if (dir == 1 && d->upsample > 1) return 0;          // `upsample` single-tap residue phases: staging-bound, stays FFMA
  const TcLayerPlan L = layer_plan(d, dir);
  if (!L.ok) return 0;
  std::vector<TcParams> launches;
  if (!plan_launches(conv_phases(d, dir), d->nsub, launches, TcParams{})) return 0;
  return L.NT;
}

// bytes of the packed split-bf16 weight image of direction `dir` (0 when unsupported)
long long tc_image_bytes(const KtConv1dDesc* d, int dir) {
  if (tc_plan(d, dir) == 0) return 0;
  const TcLayerPlan L = layer_plan(d, dir);
  return (long long)d->kernel * L.kchunks * L.ntiles * 2LL * L.NT * kTcKC * 2LL;
}

// w = the fp32 kernel-layout weight of this direction (w_fwd for dir 0, w_bwd for dir 1): [taps][K][N]
int tc_pack_layer(const KtConv1dDesc* d, int dir, const float* w, void* out, cudaStream_t st) {
  KT_REQUIRE(w && out && tc_plan(d, dir) > 0, "tc_pack_layer: layer not supported by the tensor-core path");
  const TcLayerPlan L = layer_plan(d, dir);
  const dim3 grid((unsigned)(d->kernel * L.kchunks * L.ntiles), (unsigned)ceil_div(L.NT * 8, 256));
  tc_pack_weights_kernel<<<grid, 256, 0, st>>>(w, d->kernel, L.kg, L.n_total, L.NT, L.n_stride, L.ntiles,
                                               L.grouped ? L.kin_g : 0, L.pout_g, reinterpret_cast<__nv_bfloat16*>(out));
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

static int sm_count() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
  }
  return n;
}

static int g_dbg = 0;   // development aid (kt_debug_set_flags): ablation switches of the weight-gradient chain, see wgrad_tc.cu
void debug_set_flags(int f) { g_dbg = f; }
int debug_flags() { return g_dbg; }
void debug_set_trace(long long*) {}   // (the per-role timelines belonged to the previous tensor-core kernels)

static int run_tc(TcParams p, cudaStream_t st) {   // p: phases already planned by plan_launches
  const int a_stage = 2 * p.rows * 128;
  const int b_stage = 2 * p.NT * 128;
  const int slots = p.ntaps * p.kchunks;                                      // weight tiles of the whole layer
  const long long tiles = (long long)p.ph_mt0[p.nphases] * p.ntiles * p.batch;
  const int bar_bytes = tc_fixed_smem(slots);
  const int budget = kMaxDynSmem - 1024 /*align slack*/ - bar_bytes;
  p.w_resident = 0;
  if (p.ntiles == 1 && slots <= 160 && 2 * a_stage + slots * b_stage <= budget) {
    p.w_resident = 1;
    p.nb_stages = slots;
    p.na_stages = (budget - slots * b_stage) / a_stage >= 3 ? 3 : 2;
  } else {
    // Layers with >= 4 taps per activation image spend long enough on one image for its successor to be staged meanwhile:
    // when three image and three weight stages do not fit, they give the third image stage to the weight ring.
    int min_taps = kMaxTaps;
    for (int g = 0; g < p.ngroups; ++g) min_taps = std::min(min_taps, p.grp_first[g + 1] - p.grp_first[g]);
    p.na_stages = (3 * a_stage + 3 * b_stage <= budget) ? 3 : (min_taps >= 4 ? 2 : 3);
    if (3 * a_stage + 2 * b_stage > budget) p.na_stages = 2;
    p.nb_stages = std::min(6, (budget - p.na_stages * a_stage) / b_stage);
  }
  KT_REQUIRE(p.nb_stages >= 2 || p.w_resident, "conv_tc: shared memory budget exceeded (rows=%d NT=%d)", p.rows, p.NT);
  const size_t smem = 1024 + (size_t)p.na_stages * a_stage + (size_t)p.nb_stages * b_stage + bar_bytes;
  static std::atomic<bool> cfg{false};
  if (!cfg.load(std::memory_order_acquire)) {
    KT_CHECK_CUDA(cudaFuncSetAttribute(conv_tc_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem));
    KT_CHECK_CUDA(cudaFuncSetAttribute(conv_tc_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem));
    cfg.store(true, std::memory_order_release);
  }
  const int grid = (int)std::min<long long>(tiles, sm_count());
  const bool simple = p.nsub == 1 && p.up == 1 && (p.kg & 7) == 0 && (p.c_in & 3) == 0 && (p.c_out & 3) == 0 &&
                      (p.n_stride & 3) == 0 && p.out_act != KT_ACT_TANH && !p.accumulate &&
                      (p.in.mode < SIDE_DLRELU || p.in.aux != nullptr) && !(p.resid && p.mask.p);
  if (simple) conv_tc_kernel<true><<<grid, kTcThreads, smem, st>>>(p);
  else conv_tc_kernel<false><<<grid, kTcThreads, smem, st>>>(p);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

static Side make_side_tc(const float* p, const float* aux, int act, float slope, bool derivative) {
  Side s{p, aux, SIDE_PLAIN, slope};
  if (act == KT_ACT_LRELU) s.mode = derivative ? SIDE_DLRELU : SIDE_LRELU;
  else if (act == KT_ACT_TANH) s.mode = derivative ? SIDE_DTANH : SIDE_PLAIN;
  if (s.mode < SIDE_DLRELU) s.aux = nullptr;
  return s;
}

int conv1d_fwd_tc(const KtConv1dDesc* d, const float* x, const void* wimg, const float* bias, const float* resid,
                  float* y, cudaStream_t st) {
  KT_REQUIRE(tc_plan(d, 0) > 0, "conv1d_fwd_tc: layer not supported by the tensor-core path");
  const TcLayerPlan L = layer_plan(d, 0);
  TcParams p{};
  p.NT = L.NT; p.ntiles = L.ntiles; p.kchunks = L.kchunks; p.kg = L.kg; p.grouped = L.grouped; p.n_stride = L.n_stride;
  p.in = make_side_tc(x, nullptr, d->act_in, d->act_in_slope, false);
  p.wimg = reinterpret_cast<const __nv_bfloat16*>(wimg);
  p.bias = bias; p.resid = resid; p.mask = Side{nullptr, nullptr, 0, 0.f}; p.out = y;
  p.batch = d->batch; p.nsub = d->nsub; p.t_in = d->t_in; p.t_out = d->t_out; p.c_in = d->c_in; p.c_out = d->c_out;
  p.out_act = d->act_out; p.out_slope = d->act_out_slope;
  std::vector<TcParams> launches;
  KT_REQUIRE(plan_launches(conv_phases(d, 0), d->nsub, launches, p), "conv1d_fwd_tc: phases exceed kernel limits");
  for (const TcParams& lp : launches) {
    int rc = run_tc(lp, st);
    if (rc) return rc;
  }
  return KT_OK;
}

int conv1d_bwd_data_tc(const KtConv1dDesc* d, const float* dy, const float* y, const void* wimg, const float* x,
                       float* dx, cudaStream_t st) {
  KT_REQUIRE(tc_plan(d, 1) > 0, "conv1d_bwd_data_tc: layer not supported by the tensor-core path");
  const TcLayerPlan L = layer_plan(d, 1);
  KT_REQUIRE(d->act_out == KT_ACT_NONE || y != nullptr, "bwd_data: y required when act_out != NONE");
  KT_REQUIRE(d->act_in == KT_ACT_NONE || x != nullptr, "bwd_data: x required when act_in != NONE");
  TcParams p{};
  p.NT = L.NT; p.ntiles = L.ntiles; p.kchunks = L.kchunks; p.kg = L.kg; p.grouped = L.grouped; p.n_stride = L.n_stride;
  p.in = make_side_tc(dy, y, d->act_out, d->act_out_slope, true);
  p.wimg = reinterpret_cast<const __nv_bfloat16*>(wimg);
  p.bias = nullptr; p.resid = nullptr; p.out = dx;
  p.mask = d->act_in == KT_ACT_LRELU ? Side{x, nullptr, SIDE_DLRELU, d->act_in_slope} : Side{nullptr, nullptr, 0, 0.f};
  // roles swap: the gathered tensor is dy (c_out channels, t_out rows), the product is dx
  p.batch = d->batch; p.nsub = d->nsub; p.t_in = d->t_out; p.t_out = d->t_in; p.c_in = d->c_out; p.c_out = d->c_in;
  p.out_act = KT_ACT_NONE; p.out_slope = 0.f;
  std::vector<TcParams> launches;
  KT_REQUIRE(plan_launches(conv_phases(d, 1), d->nsub, launches, p), "conv1d_bwd_data_tc: phases exceed kernel limits");
  for (const TcParams& lp : launches) {
    int rc = run_tc(lp, st);
    if (rc) return rc;
  }
  return KT_OK;
}

}  // namespace kt
