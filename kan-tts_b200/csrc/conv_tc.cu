// wgmma implicit-GEMM Conv1d (forward / data-gradient) for the GEMM-shaped HiFi-GAN layers.
//
// Precision: "bf16x3".  Every fp32 operand is split x = hi + lo (two bf16, |x - hi - lo| <~ 2^-17 |x|)
// and the product is accumulated in fp32 registers as hi*hi + hi*lo + lo*hi (the dropped lo*lo term is
// ~2^-18 relative).  A single-pass TF32/BF16 MMA does not meet the path's tolerance (mel-L1 <= 1e-4,
// SURVEY.md "hard parts"); three bf16 MMAs do, at twice the rate of 3xTF32.
// Single-pass bf16 (KT_PATH_BF16, opt-in): every operand is rounded once to bf16 (the hi plane alone) and each K = 16
// slice is ONE wgmma hi * hi into the same fp32 accumulators.  Those instances (template argument PL = 1, "planes") stage,
// pack and move one plane per operand; PL = 2 is the bf16x3 route.
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
//              mask for the data gradient), stores to the channels-last output -- staged through a small shared-memory
//              block per warp into float4 rows when the channel counts allow (TcParams::epi_staged).
//
// TMA-fed route (plain convs, channel counts % 8 == 0, see make_tc_plan): warpgroup 0 is the bound of the layers with
// few taps per image -- every CTA converts its own copy of each image, once per N tile -- so the call first writes the
// transformed gathered operand ONCE as hi / lo bf16 planes (split_planes, the weight gradient's layout) and one elected
// thread pulls each image as two SWIZZLE_128B boxes (64 channels x nsub x a_box_t time steps, one per plane) straight into
// the stage the consumers read.  A box starts at a whole time step, so an M tile is tt whole time steps x nsub rows
// (R = tt * nsub <= 128); the consumers still issue M = 128 and the epilogue discards rows r >= R.
#include <algorithm>
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
//   block (j, kc, nt) = [hi tile | lo tile], tile = NT rows (n) x 64 (k) bf16, row = 128 bytes (PL = 1: the hi tile only)
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
template <int PL>
__global__ void tc_pack_weights_kernel(const float* __restrict__ w, int taps, int K, int N, int NT, int n_stride,
                                       int ntiles, int kin_g, int pout_g, __nv_bfloat16* __restrict__ out) {
  const int kchunks = (K + kTcKC - 1) / kTcKC;
  const int block = blockIdx.x;                                   // (j, kc, nt)
  const int nt = block % ntiles, kc = (block / ntiles) % kchunks, j = block / (ntiles * kchunks);
  uint8_t* tile = reinterpret_cast<uint8_t*>(out) + (size_t)block * ((uint32_t)PL * NT * kTcKC * 2u);
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
    store_planes8<PL>(x, tile, tile + (size_t)NT * kTcKC * 2, sw128_offset((uint32_t)r, (uint32_t)q));
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
  int planes;    // bf16 planes per operand: 2 bf16x3, 1 single-pass bf16 (the kernel instance's PL)
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
  int span_q;                         // largest tap span (q_hi - q_lo) of a residue group
  // output rows per m-tile: kTcM on the register-staged route; tt whole time steps x nsub on the TMA route
  int R, tt;
  int a_box_t;                        // TMA route: time steps per image box = tt + span_q
  // Packed tiles (register-staged route, layers whose items have few output rows): one m-tile holds `pack` consecutive items
  // of the batch, item b of the tile in image rows [b * pack_rows, (b + 1) * pack_rows) -- its M * nsub output rows and the
  // span_q * nsub halo rows their taps read, so every tap stays inside the item's block -- and output row r belongs to item
  // r / pack_rows, flattened output r % pack_rows (dropped past the phase's M * nsub).  pack_magic: the RowMap divisor of
  // pack_rows.  pack = 1, pack_magic = 0: one item per tile.  The m-tile index space is per group of `pack` items.
  int pack, pack_rows;
  uint32_t pack_magic;
  // stream instances (kt_conv1d_fwd_tc_stream, nsub == 1): windows of the input / output / residual, see KtStreamWin
  int in_pitch, in_first, out_pitch, out_first, res_pitch, res_first;
  // 1: the epilogue goes through each consumer warp's shared-memory staging block (kTcEpiWarpBytes) with float4 global
  // traffic, see conv_tc_kernel; 0: straight from the accumulator registers (stream chunks, channel counts % 4 != 0,
  // operands not 16-byte aligned)
  int epi_staged;
  // masked stream instances (kt_conv1d_fwd_tc_stream with a mask): the input window's utterance bounds per item
  KtStreamMask smask;
};

// Staged epilogue: each consumer warp turns 32 columns of its 16 accumulator rows at a time into a 16 x 32 fp32 block in
// shared memory (row pitch 40 floats: the fragment writes conflict at most 2-way, rows stay 16-byte aligned), then reads it
// back as float4 per lane -- 4 rows x 128 contiguous bytes per warp instruction, like the bias / side-operand loads and the
// output stores.
constexpr int kTcEpiPitch = 40;
constexpr int kTcEpiWarpBytes = 16 * kTcEpiPitch * 4;
constexpr int kTcEpiBytes = 8 * kTcEpiWarpBytes;   // 8 consumer warps

// TMA route: one tensor map of the gathered operand's planes per input residue class rho (base + rho rows, time stride
// i_step), as wgrad_tma_kernel's map_a[]
struct TcTmaMaps {
  alignas(64) CUtensorMap map[kTcMaxGroups];
};

// Warp roles, register-staged route (416 threads): warpgroup 0 stages activations; warpgroups 1 and 2 are the consumers --
// each runs the wgmma of one 64-row half of the 128-row tile into its registers and that half's epilogue; warp 12 streams
// weights.  (Warps hold registers in groups of four: 13 warps keep the 128 registers per thread the consumers'
// accumulators need.)  TMA route (320 threads): warpgroups 0 and 1 are the consumers, warp 8 issues the image boxes,
// warp 9 streams weights.
constexpr int kTcThreads = 416;
constexpr int kTcTmaThreads = 320;
constexpr int kTcConsumerArrivals = 8;   // one per consumer warp

// Kernel instances.  REG_SIMPLE: register-staged, nsub == 1, up == 1, vectorisable channel counts, no tanh / accumulate --
// the generator's resblock convs, the scale discriminator and every SAM-BERT linear / conv (see stage_rows); it exists
// because the generic staging code made one kernel too large for the instruction cache.  REG: every other
// register-staged layer.  TMA: the TMA-fed route (no staging code, one instance).
enum TcRoute { kTcRegSimple = 0, kTcReg = 1, kTcTma = 2 };

// Persistent: gridDim.x = min(#tiles, #SMs); each CTA walks tiles blockIdx.x, +gridDim.x, ...  The activation and
// weight pipelines run continuously ACROSS tiles, so staging of tile i+1 overlaps the MMAs and the epilogue of tile i.
// STREAM (register-staged routes only): one chunk of a stream -- rows live in the windows of KtStreamWin, and the input
// rows before the chunk (down to -in_first) are real data instead of zero padding.  MASK (with STREAM): of those, only the
// rows inside item bb's utterance (KtStreamMask) are, bounded per tile by the row map's t_lo / t_lim.  MASK without STREAM
// (kt_conv1d_fwd_tc_masked, one item per tile): item bb's input rows [0, lengths[bb] * rows_per_frame) are data, the row
// map's t_lim.  PL: bf16 planes per
// operand (2: bf16x3, three wgmma per K = 16 slice; 1: single-pass bf16, one): conv_tc_kernel / conv_tc_bf16_kernel.
template <int ROUTE, bool STREAM, bool MASK, int PL>
__device__ __forceinline__ void conv_tc_body(const TcParams& p, const TcTmaMaps& maps) {
  static_assert(!(STREAM && ROUTE == kTcTma), "stream chunks take the register-staged route");
  constexpr bool SIMPLE = ROUTE == kTcRegSimple;
  constexpr bool TMA = ROUTE == kTcTma;
  constexpr int kConsumer0 = TMA ? 0 : 4;     // first consumer warp
  constexpr int kWeightWarp = TMA ? 9 : 12;
  // rows per m-tile: a compile-time 128 on the register-staged route (those instances are at their 128-register cap)
  const int R = TMA ? p.R : kTcM;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_align_1024(smem_raw);          // carve-up: all image / tile bases 1024-byte aligned
  const int img_bytes = p.rows * 128;                 // one plane of one activation stage
  const int a_stage_bytes = PL * img_bytes;           // hi (+ lo)
  const int b_stage_bytes = PL * p.NT * 128;          // hi (+ lo) weight tile
  uint8_t* a_base = smem;
  uint8_t* b_base = a_base + (size_t)p.na_stages * a_stage_bytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(b_base + (size_t)p.nb_stages * b_stage_bytes);
  uint64_t* full_a = bars;                         // [na]
  uint64_t* empty_a = full_a + p.na_stages;        // [na]
  uint64_t* full_b = empty_a + p.na_stages;        // [nb]
  uint64_t* empty_b = full_b + p.nb_stages;        // [nb]
  // per-tap image row shift in descriptor units (16 bytes)
  uint32_t* s_tapshift = reinterpret_cast<uint32_t*>(empty_b + p.nb_stages);   // [kMaxTaps]
  // staged epilogue blocks [8][16][kTcEpiPitch] floats, 16-byte aligned, after the tap-shift table (derived from it in the
  // epilogue: a pointer kept live through the main loop would cost the register-staged instances a register)

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int mtiles = p.ph_mt0[p.nphases];   // m-tiles of all phases (each: R flattened outputs m * nsub + w)
  const int total_tiles = mtiles * p.ntiles * ((p.batch + p.pack - 1) / p.pack);   // bb below: a group of p.pack items

  if (tid == 0) {
    for (int s = 0; s < p.na_stages; ++s) { mbar_init(&full_a[s], TMA ? 1 : 128); mbar_init(&empty_a[s], kTcConsumerArrivals); }
    for (int s = 0; s < p.nb_stages; ++s) { mbar_init(&full_b[s], 1); mbar_init(&empty_b[s], kTcConsumerArrivals); }
    mbar_fence_init();
    fence_proxy_async();
  }
  if (tid < kMaxTaps) s_tapshift[tid] = (uint32_t)p.tap_shift[tid] * 8u;
  __syncthreads();

  if (!TMA && warp < 4) {
    // ===================== activation producers (register-staged) =====================
    const int ptid = tid;
    RingPos ra;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const int gm = tile % mtiles, bb = tile / (mtiles * p.ntiles);
      int ph = 0;
      while (gm >= p.ph_mt0[ph + 1]) ++ph;
      const int ch_base = p.grouped ? ((tile / mtiles) % p.ntiles) * p.kg : 0;
      const int f0 = (gm - p.ph_mt0[ph]) * kTcM;
      int t_lo = 0, t_lim = 0;   // MASK: the item's utterance rows, in the row map's (up-sampled) units
      if constexpr (MASK && STREAM) {
        stream_utterance_rows(p.smask, bb, t_lo, t_lim);
        // both bounds clamped into the window's rows [-in_first, t_in] before they are scaled: the products stay in int
        // for every up-sampling factor whose up-sampled window does
        t_lo = min(max(t_lo, -p.in_first), p.t_in) * p.up;
        t_lim = max(min(t_lim, p.t_in), -p.in_first) * p.up;
      } else if constexpr (MASK) {
        t_lim = utterance_rows(p.smask, bb, p.t_in) * p.up;   // one item per tile: the masked plan never packs
      }
      for (int c = 0; c < p.kchunks; ++c) {
        for (int g = p.ph_g0[ph]; g < p.ph_g0[ph + 1]; ++g, ra.advance(p.na_stages)) {
          const int s = ra.slot();
          mbar_wait(&empty_a[s], ra.phase() ^ 1u);
          uint8_t* img_hi = a_base + (size_t)s * a_stage_bytes;
          RowMap rm;
          if constexpr (STREAM) {
            rm.base_row = (long long)bb * p.in_pitch + p.in_first;
            rm.t_lo = -p.in_first * p.up;
          } else {
            rm.base_row = (long long)bb * p.pack * p.t_in * p.nsub;
            rm.pack_magic = p.pack_magic; rm.pack_rows = p.pack_rows; rm.pack_items = min(p.pack, p.batch - bb * p.pack);
            rm.item_rows = (long long)p.t_in * p.nsub;
          }
          rm.fv0 = f0 + p.grp_qlo[g] * p.nsub;
          rm.nsub = p.nsub; rm.step = p.i_step; rm.rho = p.grp_rho[g]; rm.up = p.up; rm.t_lim = p.t_in * p.up;
          if constexpr (MASK) { rm.t_lo = t_lo; rm.t_lim = t_lim; }
          stage_rows<5, SIMPLE, 3, STREAM, !STREAM, PL>(img_hi, img_hi + img_bytes, p.in, p.in.p, p.in.aux, p.c_in, ch_base + c * kTcKC,
                                   min(kTcKC, p.kg - c * kTcKC), false, rm, p.rows, ptid);
          fence_proxy_async();
          mbar_arrive(&full_a[s]);
        }
      }
    }
  } else if (TMA && warp == 8) {
    // ===================== activation producer (TMA) =====================
    // Image row r = (time step m0 + qlo + r / nsub of residue class rho, sub-sequence r % nsub): the register-staged row map
    // with f0 = mt * R.  Time steps outside [0, T) -- left padding included -- and channels past c_in arrive as the TMA
    // unit's zeros.  In a block-diagonal grouped tile (kg < 64) the box also brings the next tile's real channels: they meet
    // zero weight rows, and kslices stops the MMAs at the last K = 16 slice holding this tile's channels.  Rows past the box
    // keep whatever an earlier image left there: they feed only the discarded output rows r >= R, and the stage holds
    // p.rows >= 128 + span_q * nsub rows, so every row an MMA reads lies inside it.
    if (elect_one()) {
      const uint32_t box_bytes = (uint32_t)(p.a_box_t * p.nsub) * 128u;
      RingPos ra;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int gm = tile % mtiles, bb = tile / (mtiles * p.ntiles);
        int ph = 0;
        while (gm >= p.ph_mt0[ph + 1]) ++ph;
        const int ch_base = p.grouped ? ((tile / mtiles) % p.ntiles) * p.kg : 0;
        const int m0 = (gm - p.ph_mt0[ph]) * p.tt;
        for (int c = 0; c < p.kchunks; ++c) {
          for (int g = p.ph_g0[ph]; g < p.ph_g0[ph + 1]; ++g, ra.advance(p.na_stages)) {
            const int s = ra.slot();
            mbar_wait(&empty_a[s], ra.phase() ^ 1u);
            uint8_t* img_hi = a_base + (size_t)s * a_stage_bytes;
            const CUtensorMap* map = &maps.map[p.grp_rho[g]];
            mbar_arrive_expect_tx(&full_a[s], (uint32_t)PL * box_bytes);
            tma_load_5d(img_hi, map, ch_base + c * kTcKC, 0, m0 + p.grp_qlo[g], bb, 0, &full_a[s]);
            if constexpr (PL == 2) tma_load_5d(img_hi + img_bytes, map, ch_base + c * kTcKC, 0, m0 + p.grp_qlo[g], bb, 1, &full_a[s]);
          }
        }
      }
      // every issued box has landed before the CTA may exit: the consumers waited for all of them
    }
    __syncwarp();
  } else if (warp == kWeightWarp) {
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
      RingPos rb;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int nt = (tile / mtiles) % p.ntiles;
        int ph = 0;
        while ((tile % mtiles) >= p.ph_mt0[ph + 1]) ++ph;
        const int n_begin = p.grp_first[p.ph_g0[ph]], n_end = p.grp_first[p.ph_g0[ph + 1]];
        for (int c = 0; c < p.kchunks; ++c) {
          for (int n = n_begin; n < n_end; ++n, rb.advance(p.nb_stages)) {  // taps are ordered by group: same order as the consumers
            const int s = rb.slot();
            mbar_wait(&empty_b[s], rb.phase() ^ 1u);
            const long long block = ((long long)p.tap_j[n] * p.kchunks + c) * p.ntiles + nt;
            const uint8_t* src = reinterpret_cast<const uint8_t*>(p.wimg) + block * (long long)b_stage_bytes;
            mbar_arrive_expect_tx(&full_b[s], (uint32_t)b_stage_bytes);
            bulk_g2s(b_base + (size_t)s * b_stage_bytes, src, (uint32_t)b_stage_bytes, &full_b[s]);
          }
        }
      }
    }
    __syncwarp();
  } else if (warp >= kConsumer0 && warp < kConsumer0 + 8) {
    // ===================== consumers: wgmma + epilogue, one 64-row half of the tile per warpgroup =====================
    // Descriptor low words + 32-bit adds only: a tap's row shift, the K = 16 slice offset (32 bytes = 2 units), the hi -> lo
    // plane distance and this warpgroup's 64-row offset (8 KB = 512 units) are integer adds on the low word.
    const int cw = (warp - kConsumer0) >> 2;         // 0: rows 0-63, 1: rows 64-127
    const int wq = warp & 3;                         // warp inside the warpgroup: rows 16 wq .. 16 wq + 15 of the half
    const uint32_t a_base16 = (smem_u32(a_base) >> 4) + (uint32_t)cw * 512u;
    const uint32_t b_base16 = smem_u32(b_base) >> 4;
    const uint32_t a_stage16 = (uint32_t)a_stage_bytes >> 4, img16 = (uint32_t)img_bytes >> 4;
    const uint32_t b_stage16 = (uint32_t)b_stage_bytes >> 4, bplane16 = (uint32_t)(p.NT * 128) >> 4;
    const bool resident = p.w_resident != 0;
    // one consumer path per MMA width (see with_wgmma_n)
    with_wgmma_n(p.NT, [&](auto nt) {
      constexpr int NT = decltype(nt)::value;
      float acc[kWgmmaMaxRegs];
#pragma unroll
      for (int i = 0; i < kWgmmaMaxRegs; ++i) acc[i] = 0.f;
      RingPos ra, rb;
      int ti = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x, ++ti) {
        const int gm = tile % mtiles, nt = (tile / mtiles) % p.ntiles, bb = tile / (mtiles * p.ntiles);
        int ph = 0;
        while (gm >= p.ph_mt0[ph + 1]) ++ph;
        const int g_begin = p.ph_g0[ph], g_end = p.ph_g0[ph + 1];
        uint32_t scale_d = 0;
        for (int c = 0; c < p.kchunks; ++c) {
          const int kslices = warp_uniform((min(kTcKC, p.kg - c * kTcKC) + 15) >> 4);   // K = 16 slices holding real channels
          for (int g = g_begin; g < g_end; ++g, ra.advance(p.na_stages)) {
            const int sa = ra.slot();
            mbar_wait(&full_a[sa], ra.phase());
            const uint32_t a16 = a_base16 + (uint32_t)sa * a_stage16;
            for (int n = p.grp_first[g]; n < p.grp_first[g + 1]; ++n) {
              int sb;
              if (resident) {
                sb = c * p.ntaps + n;
                if (ti == 0) mbar_wait(&full_b[sb], 0u);
              } else {
                sb = rb.slot();
                mbar_wait(&full_b[sb], rb.phase());
                rb.advance(p.nb_stages);
              }
              const uint32_t a_hi = a16 + s_tapshift[n];
              const uint32_t b_hi = b_base16 + (uint32_t)sb * b_stage16;
              wgmma_fence();
              for (int ks = 0; ks < kslices; ++ks) {
                wgmma_slice<PL, NT, 0, 0>(acc, a_hi + 2u * ks, img16, b_hi + 2u * ks, bplane16, scale_d);
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
        // Element index of output row r's first column (false: the row is not written).  The residual element is the
        // output element + rdelta (0 outside streams: the residual has the output's layout); the act' mask and `out` itself
        // (accumulate) share the output's layout.
        const long long rdelta = STREAM ? ((long long)bb * (p.res_pitch - p.out_pitch) + p.res_first - p.out_first) * p.c_out : 0;
        // packed tiles: row r is row r - b * pack_rows of item b's block (RowMap); the TMA and stream instances never pack
        constexpr bool PACKED = !TMA && !STREAM;
        auto row_base = [&](int r, long long& obase) {
          const int b = PACKED ? (int)(((uint32_t)r * p.pack_magic) >> 16) : 0;
          const int item = PACKED ? bb * p.pack + b : bb;
          r -= b * p.pack_rows;
          const int f = mt * R + r;
          if ((TMA && r >= R) || f >= F || (PACKED && (b >= p.pack || item >= p.batch))) return false;
          const int m = p.nsub == 1 ? f : f / p.nsub;
          const int w = f - m * p.nsub;
          const int to = p.ph_ooff[ph] + p.o_step * m;
          obase = STREAM ? ((long long)bb * p.out_pitch + p.out_first + to) * p.c_out + c_tile
                         : ((long long)(item * p.t_out + to) * p.nsub + w) * p.c_out + c_tile;
          return true;
        };
        // Both forms do the same fp32 operations per element in the same order, so they write the same bits.
        auto finish = [&](float x, float bia, float md, float sd, float od) {
          x += bia;
          if (p.out_act == KT_ACT_LRELU) x = x > 0.f ? x : x * p.out_slope;
          else if (!SIMPLE && p.out_act == KT_ACT_TANH) x = tanhf(x);
          if (p.mask.p) x = side_apply(x, md, p.mask.mode, p.mask.slope);
          return x + (sd + od);
        };
        if (!STREAM && p.epi_staged) {
          // Staged: per 32-column chunk, registers -> this warp's shared-memory block -> float4 rows.  A warp waits for its
          // side operand 16 times per tile instead of 32, every load and store moves whole 128-byte lines, and the unrolled
          // code per chunk stays small (the register form's code per tile is several times larger).
          float* blk = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(s_tapshift + kMaxTaps) + 15) & ~(uintptr_t)15) +
                       (warp - kConsumer0) * (16 * kTcEpiPitch);
          const int c4 = (lane & 7) * 4;   // this lane's 4 columns of the chunk; rows it * 4 + lane / 8
          const float* side = p.resid ? p.resid + rdelta : p.mask.p;   // at most one (run_plan)
#pragma unroll
          for (int j = 0; j < (NT + 31) / 32; ++j) {
#pragma unroll
            for (int ii = 0; ii < 4; ++ii) {
              const int i = 4 * j + ii;
              if (i >= NT / 8) break;
#pragma unroll
              for (int h = 0; h < 2; ++h)
                *reinterpret_cast<float2*>(blk + ((lane >> 2) + 8 * h) * kTcEpiPitch + ii * 8 + 2 * (lane & 3)) =
                    make_float2(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]);
            }
            __syncwarp();
            const int col = j * 32 + c4;
            float4 bia = make_float4(0.f, 0.f, 0.f, 0.f);
            if (p.bias && col < n_valid) bia = __ldg(reinterpret_cast<const float4*>(p.bias + c_tile + col));
#pragma unroll
            for (int it = 0; it < 4; ++it) {
              long long o;
              if (col >= n_valid || !row_base(cw * 64 + wq * 16 + it * 4 + (lane >> 3), o)) continue;
              o += col;
              const float4 pre = side ? __ldg(reinterpret_cast<const float4*>(side + o)) : make_float4(0.f, 0.f, 0.f, 0.f);
              const float4 v = *reinterpret_cast<const float4*>(blk + (it * 4 + (lane >> 3)) * kTcEpiPitch + c4);
              const float4 md = p.resid ? make_float4(0.f, 0.f, 0.f, 0.f) : pre;
              const float4 sd = p.resid ? pre : make_float4(0.f, 0.f, 0.f, 0.f);
              *reinterpret_cast<float4*>(p.out + o) = make_float4(finish(v.x, bia.x, md.x, sd.x, 0.f), finish(v.y, bia.y, md.y, sd.y, 0.f),
                                                                  finish(v.z, bia.z, md.z, sd.z, 0.f), finish(v.w, bia.w, md.w, sd.w, 0.f));
            }
            __syncwarp();
          }
          continue;
        }
        const bool vec2 = ((p.c_out | p.n_stride) & 1) == 0;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          long long obase;
          if (!row_base(cw * 64 + wq * 16 + (lane >> 2) + 8 * h, obase)) continue;   // row of the M = 128 accumulator tile
#pragma unroll
          for (int i = 0; i < NT / 8; ++i) {
            const int col = i * 8 + 2 * (lane & 3);
            if (col >= n_valid) continue;
            float v[2] = {acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]};
            const bool pair = vec2 && col + 1 < n_valid;
            const int ne = col + 1 < n_valid ? 2 : 1;
            float bia[2] = {0.f, 0.f}, sd[2] = {0.f, 0.f}, md[2] = {0.f, 0.f}, od[2] = {0.f, 0.f};
            const long long o = obase + col;
            if (pair) {
              if (p.bias) { const float2 t = __ldg(reinterpret_cast<const float2*>(p.bias + c_tile + col)); bia[0] = t.x; bia[1] = t.y; }
              if (p.mask.p) { const float2 t = __ldg(reinterpret_cast<const float2*>(p.mask.p + o)); md[0] = t.x; md[1] = t.y; }
              if (p.resid) { const float2 t = __ldg(reinterpret_cast<const float2*>(p.resid + o + rdelta)); sd[0] = t.x; sd[1] = t.y; }
              if (!SIMPLE && p.accumulate) { const float2 t = *reinterpret_cast<const float2*>(p.out + o); od[0] = t.x; od[1] = t.y; }
            } else {
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                if (e >= ne) break;
                if (p.bias) bia[e] = __ldg(p.bias + c_tile + col + e);
                if (p.mask.p) md[e] = __ldg(p.mask.p + o + e);
                if (p.resid) sd[e] = __ldg(p.resid + o + rdelta + e);
                if (!SIMPLE && p.accumulate) od[e] = p.out[o + e];
              }
            }
#pragma unroll
            for (int e = 0; e < 2; ++e) v[e] = finish(v[e], bia[e], md[e], sd[e], od[e]);
            if (pair) *reinterpret_cast<float2*>(p.out + o) = make_float2(v[0], v[1]);
            else {
              p.out[o] = v[0];
              if (ne == 2) p.out[o + 1] = v[1];
            }
          }
        }
      }
    });
  }
}

template <int ROUTE, bool STREAM = false, bool MASK = false>
__global__ void __launch_bounds__(ROUTE == kTcTma ? kTcTmaThreads : kTcThreads, 1)
    conv_tc_kernel(const __grid_constant__ TcParams p, const __grid_constant__ TcTmaMaps maps) {
  conv_tc_body<ROUTE, STREAM, MASK, 2>(p, maps);
}
template <int ROUTE, bool STREAM = false, bool MASK = false>
__global__ void __launch_bounds__(ROUTE == kTcTma ? kTcTmaThreads : kTcThreads, 1)
    conv_tc_bf16_kernel(const __grid_constant__ TcParams p, const __grid_constant__ TcTmaMaps maps) {
  conv_tc_body<ROUTE, STREAM, MASK, 1>(p, maps);
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
  int pack, pack_rows; // items per packed m-tile and rows of one item's block (pack_shape); pack = 1: not packed
};

struct TcParams;

// shared memory outside the activation / weight stages: barriers and the tap-shift table (see the carve-up in conv_tc_kernel)
static int tc_fixed_smem(int slots) { return (2 * 3 + 2 * std::max(6, slots)) * 8 + kMaxTaps * 4; }

// Packing of a layer whose items have few output rows (TcParams::pack): with M output time steps per item (the largest phase)
// and taps spanning span_q steps of one residue class (the widest), an item's block is pack_rows = (M + span_q) * nsub image
// rows, and the last item's M * nsub output rows must lie in the 128-row tile: pack = (128 - M * nsub) / pack_rows + 1 items,
// at most the batch.  The last block's taps then read at most 128 + span_q * nsub rows, which every launch of the layer
// stages.  Items of more than 64 output rows never pack (pack = 1).
static void pack_shape(const KtConv1dDesc* d, const std::vector<Phase>& phases, int& pack, int& pack_rows) {
  int M = 0, span_q = 0;
  for (const Phase& ph : phases) {
    if (ph.M <= 0) continue;
    M = std::max(M, ph.M);
    const ResidueTaps rt = residue_taps(ph, ph.i_step);
    for (int r = 0; r < ph.i_step; ++r) {
      int qlo = 1 << 30, qhi = -(1 << 30);
      for (int n = rt.first[r]; n < rt.first[r + 1]; ++n) { qlo = std::min(qlo, rt.q[n]); qhi = std::max(qhi, rt.q[n]); }
      if (rt.first[r + 1] > rt.first[r]) span_q = std::max(span_q, qhi - qlo);
    }
  }
  pack = 1; pack_rows = 0;
  if (M == 0 || 2 * M * d->nsub > kTcM) return;
  pack_rows = (M + span_q) * d->nsub;
  pack = std::min(d->batch, (kTcM - M * d->nsub) / pack_rows + 1);
  if (pack < 2) { pack = 1; pack_rows = 0; }
}

static TcLayerPlan layer_plan(const KtConv1dDesc* d, int dir) {
  TcLayerPlan L{};
  pack_shape(d, conv_phases(d, dir), L.pack, L.pack_rows);
  const int g = d->groups;
  const int kin = (dir == 0 ? d->c_in : d->c_out) / g;     // contraction channels per group
  const int pout = (dir == 0 ? d->c_out : d->c_in) / g;    // produced channels per group
  L.kg = kin;
  L.n_total = pout * g;
  L.kchunks = ceil_div(kin, kTcKC);
  L.grouped = g > 1;
  // M tiles per N tile of the launch (packed: one per group of L.pack items)
  const long long mtiles = L.pack > 1 ? ceil_div(d->batch, L.pack)
                                      : (long long)ceil_div((dir == 0 ? d->t_out : d->t_in) * d->nsub, kTcM) * d->batch;
  if (g > 1) {
    if (pout > kWgmmaMaxN) return L;
    // groups per tile: fill one 64-channel K chunk, keep the N tile <= 128 (block-diagonal tile, see tc_pack_weights_kernel)
    int gt = 1;
    while (gt * 2 <= g && g % (gt * 2) == 0 && kin * gt * 2 <= kTcKC && pout * gt * 2 <= 128) gt *= 2;
    // Under-filled grids (short sequences): fewer groups per tile.  A tile's MMAs grow with gt^2 (K and N both gt-fold) of
    // which only 1 / gt is off the zero blocks, so halving gt quarters each tile's MMA time and doubles the tiles.  Each
    // output still gets its own group's K = 16 slices in the same order (the dropped slices only added zero products): the
    // same bits.  The halving keeps the N tile >= 16 (so the N tile still identifies the image layout, PreparedWeight's
    // key) and the alignment of kg and n_stride the kernel instances depend on.
    while (gt > 1 && mtiles * (g / gt) < 120 && (gt / 2) * pout >= 16 && (gt / 2) * kin % 8 == 0 && (gt / 2) * pout % 4 == 0)
      gt /= 2;
    L.kin_g = kin; L.pout_g = pout;
    L.kg = gt * kin;
    L.kchunks = ceil_div(L.kg, kTcKC);
    L.n_stride = gt * pout; L.NT = (L.n_stride + 15) & ~15; L.ntiles = g / gt;
  } else if (pout <= 2 * kWgmmaMaxN) {
    // N tiles of <= 128 channels (a 64-row half tile's accumulators are 64 registers per thread at N = 128)
    L.ntiles = ceil_div(pout, kWgmmaMaxN);
    L.n_stride = (ceil_div(pout, L.ntiles) + 15) & ~15; L.NT = L.n_stride;
    // under-filled grids (short sequences x wide layers): split N so that >= ~1 tile per SM exists
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
  p.nphases = 0; p.ngroups = 0; p.ntaps = 0; p.rows = 0; p.span_q = 0;
  p.ph_mt0[0] = 0; p.ph_g0[0] = 0; p.grp_first[0] = 0;
}

static bool add_phase(TcParams& p, const Phase& ph, int nsub) {
  if (ph.M <= 0) return true;
  const int s = ph.i_step;
  if (s < 1 || s > kTcMaxGroups || p.nphases >= kTcMaxGroups) return false;
  if (p.nphases > 0 && (p.o_step != ph.o_step || p.i_step != ph.i_step || p.up != ph.up)) return false;
  p.o_step = ph.o_step; p.i_step = ph.i_step; p.up = ph.up; p.accumulate = ph.accumulate;
  const ResidueTaps rt = residue_taps(ph, s);
  int max_span = 0;
  for (int r = 0; r < s; ++r) {
    const int n0 = rt.first[r], cnt = rt.first[r + 1] - n0;
    if (!cnt) continue;
    int qlo = 1 << 30, qhi = -(1 << 30);
    for (int n = n0; n < n0 + cnt; ++n) { qlo = std::min(qlo, rt.q[n]); qhi = std::max(qhi, rt.q[n]); }
    if (p.ngroups >= kTcMaxGroups || p.ntaps + cnt > kMaxTaps) return false;
    const int g = p.ngroups++;
    p.grp_rho[g] = r; p.grp_qlo[g] = qlo; p.grp_first[g] = p.ntaps;
    for (int n = n0; n < n0 + cnt; ++n, ++p.ntaps) {
      p.tap_j[p.ntaps] = rt.j[n];
      p.tap_shift[p.ntaps] = (rt.q[n] - qlo) * nsub;
    }
    p.grp_first[p.ngroups] = p.ntaps;
    max_span = std::max(max_span, (qhi - qlo) * nsub);
    p.span_q = std::max(p.span_q, qhi - qlo);
  }
  const int i = p.nphases++;
  p.ph_M[i] = ph.M; p.ph_ooff[i] = ph.o_off;
  p.ph_mt0[i + 1] = p.ph_mt0[i] + ceil_div(ph.M * nsub, p.R);
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

// What a call of direction dir (0 forward, 1 data gradient) of a layer runs: the tiling, the launches (phases planned,
// pointers filled in by the caller) and the route.  The gathered operand is x (c_in channels, t_in rows) for the forward
// and dy (c_out channels, t_out rows) for the data gradient.
struct TcPlan {
  bool ok;                          // the tensor-core kernel runs this direction
  bool tma;                         // TMA-fed route, else register-staged
  TcLayerPlan L;
  std::vector<TcParams> launches;
  long long ws_floats;              // TMA route: hi / lo bf16 planes of the gathered operand (one float per element)
};

// Does the split pass pay for itself?  It moves ~12 bytes per gathered element through HBM (read fp32, write and re-read
// two bf16 planes) to take the staging off the CTAs.  Measured per layer in the C2 step (H100 SXM, 700 W, both routes):
//   wins  dense layers with >= 2 N tiles (the staging was repeated per N tile): MPD 1024 -> 1024 k5 fwd / dgrad 0.29-0.38
//         -> 0.24 ms, MPD 512 -> 1024 s3 dgrad 0.41 -> 0.17 ms, 256 -> 256 k3 dgrad 0.44 -> 0.21 ms; and small gathered
//         tensors, whose planes stay in L2 (MSD 1024 -> 1 k3 fwd 0.33 -> 0.20 ms, MPD 1 -> 32 s3 dgrad 0.65 -> 0.26 ms)
//   losses one N tile over >= 4 M elements (generator 128 -> 128 k3 fwd 0.55 -> 0.78 ms, MPD 128 -> 512 s3 dgrad at
//         15 M elements 0.22 -> 0.55 ms: HBM-bound already), and grouped layers on balance (MSD g16 dgrads 0.29 -> 0.59,
//         0.61 -> 0.83, 0.29 -> 0.50 ms against g4 / g16 dgrad wins of 0.34 and 0.32 ms)
// Below 512 K gathered elements no producer is the bound (the C2 step's 1024-channel layers at 9 time steps: 0.20 vs 0.21 ms)
// and the split pass is one more launch, plus the tensor maps encoded on the host, in latency-bound calls (batch-1 inference).
static bool tma_pays(const TcParams& lp) {
  const long long elems = (long long)lp.batch * lp.t_in * lp.nsub * lp.c_in;   // gathered operand
  return !lp.grouped && elems >= (1LL << 19) && (lp.ntiles >= 2 || elems < (1LL << 22));
}

// allow_pack: false for stream chunks, whose rows live in per-slot windows (one item per tile)
static TcPlan make_tc_plan(const KtConv1dDesc* d, int dir, bool allow_tma = true, bool plan_only = false, bool allow_pack = true) {
  TcPlan P{};
  if (dir == 0 && d->path != KT_PATH_TC && thin_cin1_ok(d)) return P;   // waveform-input layers: HBM-bound FIR kernel
  if (dir == 1 && d->upsample > 1) return P;   // no direct plan: ops.ConvPlan runs it as the plain conv over the
                                               // up-sampled rows + kt_upsample_grad_reduce
  P.L = layer_plan(d, dir);
  const TcLayerPlan& L = P.L;
  if (!L.ok) return P;
  TcParams base{};
  base.NT = L.NT; base.ntiles = L.ntiles; base.kchunks = L.kchunks; base.kg = L.kg; base.grouped = L.grouped; base.n_stride = L.n_stride;
  base.batch = d->batch; base.nsub = d->nsub; base.pack = 1;
  base.planes = d->path == KT_PATH_BF16 ? 1 : 2;
  // roles swap for the data gradient: the gathered tensor is dy, the product is dx
  base.t_in = dir == 0 ? d->t_in : d->t_out; base.t_out = dir == 0 ? d->t_out : d->t_in;
  base.c_in = dir == 0 ? d->c_in : d->c_out; base.c_out = dir == 0 ? d->c_out : d->c_in;
  const std::vector<Phase> phases = conv_phases(d, dir);
  // TMA route: no nearest-upsampling (the planes hold the tensor as stored), 16-byte aligned box coordinates and strides
  // (the gathered width and the channels per tile % 8), box extents <= 256 and a time step in every residue class
  bool tma = allow_tma && d->upsample == 1 && base.c_in % 8 == 0 && L.kg % 8 == 0 && d->nsub <= kTcM &&
             (plan_only || encode_tiled_fn() != nullptr);
  if (tma) {
    base.tt = kTcM / d->nsub; base.R = base.tt * d->nsub;
    tma = plan_launches(phases, d->nsub, P.launches, base);
    for (TcParams& lp : P.launches) {
      lp.a_box_t = lp.tt + lp.span_q;
      tma = tma && lp.up == 1 && lp.a_box_t <= 256 && lp.t_in >= lp.i_step && tma_pays(lp);
    }
  }
  if (!tma) {
    P.launches.clear();
    base.tt = 0; base.R = kTcM;
    if (allow_pack && L.pack > 1) {
      // packed tiles (register-staged route only: a TMA box holds one item); every phase is one m-tile per item group
      base.pack = L.pack; base.pack_rows = L.pack_rows;
      base.pack_magic = (1u << 16) / (unsigned)L.pack_rows + 1;
    }
    if (!plan_launches(phases, d->nsub, P.launches, base)) return P;
  }
  // staged epilogue: float4 rows need output channel counts and tile offsets % 4 (run_plan also checks the pointers);
  // accumulating launches keep the register form
  for (TcParams& lp : P.launches) lp.epi_staged = lp.c_out % 4 == 0 && lp.n_stride % 4 == 0 && !lp.accumulate;
  P.ok = true;
  P.tma = tma;
  P.ws_floats = tma ? plane_floats(base.batch, base.t_in, base.nsub, base.c_in, base.planes) : 0;
  return P;
}

// dir: 0 / 1, or KT_PLAN_STREAM (the forward of a stream chunk: register-staged route, nsub == 1, register epilogue: the
// stream instances have no registers to spare)
static TcPlan make_tc_plan_flags(const KtConv1dDesc* d, int dir, bool plan_only = false) {
  if (dir == KT_PLAN_STREAM) {
    if (d->nsub != 1) return TcPlan{};
    TcPlan P = make_tc_plan(d, 0, false, plan_only, false);
    for (TcParams& lp : P.launches) lp.epi_staged = 0;
    return P;
  }
  return make_tc_plan(d, dir, true, plan_only);
}

static int tc_plan(const KtConv1dDesc* d, int dir) {
  const TcPlan P = make_tc_plan_flags(d, dir);
  return P.ok ? P.L.NT : 0;
}

extern "C" int kt_conv1d_tc_plan(const KtConv1dDesc* d, int32_t dir) {
  if (validate_conv(d)) return 0;
  return tc_plan(d, dir);
}

extern "C" int64_t kt_conv1d_tc_workspace(const KtConv1dDesc* d, int32_t dir) {
  if (validate_conv(d)) return 0;
  return make_tc_plan_flags(d, dir).ws_floats;
}

// bytes of the packed weight image of direction `dir` (0 when unsupported): two bf16 planes, one for KT_PATH_BF16
extern "C" int64_t kt_conv1d_tc_image_bytes(const KtConv1dDesc* d, int32_t dir) {
  if (validate_conv(d)) return 0;
  if (dir != 0 && dir != 1) return 0;
  if (tc_plan(d, dir) == 0) return 0;
  const TcLayerPlan L = layer_plan(d, dir);
  const long long planes = d->path == KT_PATH_BF16 ? 1 : 2;
  return (long long)d->kernel * L.kchunks * L.ntiles * planes * L.NT * kTcKC * 2LL;
}

// w = the fp32 kernel-layout weight of this direction (w_fwd for dir 0, w_bwd for dir 1): [taps][K][N]
int tc_pack_layer(const KtConv1dDesc* d, int dir, const float* w, void* out, cudaStream_t st) {
  KT_REQUIRE(w && out && tc_plan(d, dir) > 0, "tc_pack_layer: layer not supported by the tensor-core path");
  const TcLayerPlan L = layer_plan(d, dir);
  const dim3 grid((unsigned)(d->kernel * L.kchunks * L.ntiles), (unsigned)ceil_div(L.NT * 8, 256));
  auto* img = reinterpret_cast<__nv_bfloat16*>(out);
  if (d->path == KT_PATH_BF16)
    tc_pack_weights_kernel<1><<<grid, 256, 0, st>>>(w, d->kernel, L.kg, L.n_total, L.NT, L.n_stride, L.ntiles, L.grouped ? L.kin_g : 0,
                                                    L.pout_g, img);
  else
    tc_pack_weights_kernel<2><<<grid, 256, 0, st>>>(w, d->kernel, L.kg, L.n_total, L.NT, L.n_stride, L.ntiles, L.grouped ? L.kin_g : 0,
                                                    L.pout_g, img);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

extern "C" int kt_weight_pack_tc(const KtConv1dDesc* d, int32_t dir, const float* w, void* out, void* stream) {
  int rc = validate_conv(d);
  if (rc) return rc;
  return tc_pack_layer(d, dir, w, out, static_cast<cudaStream_t>(stream));
}

// Ring sizes of one launch -> its shared-memory bytes (0: the stages do not fit)
// (single-pass bf16 stages are half the bytes: the same rule gives those layers resident weights or deeper rings where they
// fit, up to the same stage caps)
static size_t size_stages(TcParams& p) {
  const int a_stage = p.planes * p.rows * 128;
  const int b_stage = p.planes * p.NT * 128;
  const int slots = p.ntaps * p.kchunks;                                      // weight tiles of the whole layer
  const int bar_bytes = tc_fixed_smem(slots) + (p.epi_staged ? 16 + kTcEpiBytes : 0);
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
  if (p.nb_stages < 2 && !p.w_resident) return 0;
  return 1024 + (size_t)p.na_stages * a_stage + (size_t)p.nb_stages * b_stage + bar_bytes;
}

// development / test aid (kt_debug_conv_tc_plan): the plan of direction dir as it would be made on a GPU box
// out = {N tile (0: not on the tensor cores), TMA route, tt, R, a_box_t, image stages, weight stages, shared-memory bytes,
// workspace floats}, the launch-dependent entries for the first launch
extern "C" int kt_debug_conv_tc_plan(const KtConv1dDesc* d, int32_t dir, int64_t* out) {
  KT_REQUIRE(d && out, "kt_debug_conv_tc_plan: null pointer");
  TcPlan P = make_tc_plan_flags(d, dir, true);
  for (int i = 0; i < 9; ++i) out[i] = 0;
  if (!P.ok) return KT_OK;
  TcParams& lp = P.launches[0];
  const size_t smem = size_stages(lp);
  out[0] = P.L.NT; out[1] = P.tma; out[2] = lp.tt; out[3] = lp.R; out[4] = lp.a_box_t;
  out[5] = lp.na_stages; out[6] = lp.nb_stages; out[7] = (int64_t)smem; out[8] = P.ws_floats;
  return KT_OK;
}

// development / test aid (kt_debug_conv_tc_pack): the tile packing of direction dir (0, 1 or KT_PLAN_STREAM) as it would be
// planned on a GPU box.  out = {items per m-tile, rows of one item's block, MMA rows issued per N tile over all launches,
// the same without packing, output rows produced per N tile}; {1, 0, 0, 0, 0} for a layer off the tensor cores
extern "C" int kt_debug_conv_tc_pack(const KtConv1dDesc* d, int32_t dir, int64_t* out) {
  KT_REQUIRE(d && out, "kt_debug_conv_tc_pack: null pointer");
  const TcPlan P = make_tc_plan_flags(d, dir, true);
  out[0] = 1;
  for (int i = 1; i < 5; ++i) out[i] = 0;
  if (!P.ok) return KT_OK;
  out[0] = P.launches[0].pack; out[1] = P.launches[0].pack_rows;
  for (const TcParams& lp : P.launches) {
    const int mt = lp.ph_mt0[lp.nphases];
    out[2] += (int64_t)kTcM * mt * ceil_div(lp.batch, lp.pack);
    out[3] += (int64_t)kTcM * mt * lp.batch;
    for (int i = 0; i < lp.nphases; ++i) out[4] += (int64_t)lp.ph_M[i] * lp.nsub * lp.batch;
  }
  return KT_OK;
}

// development / test aid: 1 when the launches of direction dir (0, 1 or KT_PLAN_STREAM) take the staged epilogue given
// 16-byte aligned operands, 0 for the register epilogue or a layer off the tensor cores
extern "C" int kt_debug_conv_tc_epilogue(const KtConv1dDesc* d, int32_t dir) {
  if (d == nullptr) return 0;
  const TcPlan P = make_tc_plan_flags(d, dir, true);
  return P.ok && P.launches[0].epi_staged ? 1 : 0;
}

template <int ROUTE, bool STREAM, bool MASK, int PL>
static int launch_tc(const TcParams& p, const TcTmaMaps& maps, int grid, size_t smem, cudaStream_t st) {
  constexpr auto kernel = PL == 1 ? conv_tc_bf16_kernel<ROUTE, STREAM, MASK> : conv_tc_kernel<ROUTE, STREAM, MASK>;
  KT_CHECK_CUDA(allow_dyn_smem<kernel>(kMaxDynSmem));
  kernel<<<grid, ROUTE == kTcTma ? kTcTmaThreads : kTcThreads, smem, st>>>(p, maps);
  return KT_OK;
}

// the instance of one launch, PL = p.planes
template <int PL>
static int launch_route(const TcParams& p, const TcTmaMaps& maps, bool tma, bool stream, bool masked, int grid, size_t smem,
                        cudaStream_t st) {
  if (tma) return launch_tc<kTcTma, false, false, PL>(p, maps, grid, smem, st);
  const bool simple = p.nsub == 1 && p.up == 1 && (p.kg & 7) == 0 && (p.c_in & 3) == 0 && (p.c_out & 3) == 0 &&
                      (p.n_stride & 3) == 0 && p.out_act != KT_ACT_TANH && !p.accumulate &&
                      (p.in.mode < SIDE_DLRELU || p.in.aux != nullptr) && !(p.resid && p.mask.p);
  if (masked && !stream && simple) return launch_tc<kTcRegSimple, false, true, PL>(p, maps, grid, smem, st);
  if (masked && !stream) return launch_tc<kTcReg, false, true, PL>(p, maps, grid, smem, st);
  if (masked && simple) return launch_tc<kTcRegSimple, true, true, PL>(p, maps, grid, smem, st);
  if (masked) return launch_tc<kTcReg, true, true, PL>(p, maps, grid, smem, st);
  if (stream && simple) return launch_tc<kTcRegSimple, true, false, PL>(p, maps, grid, smem, st);
  if (stream) return launch_tc<kTcReg, true, false, PL>(p, maps, grid, smem, st);
  if (simple) return launch_tc<kTcRegSimple, false, false, PL>(p, maps, grid, smem, st);
  return launch_tc<kTcReg, false, false, PL>(p, maps, grid, smem, st);
}

static int run_tc(TcParams p, const TcTmaMaps& maps, bool tma, bool stream, bool masked,
                  cudaStream_t st) {   // p: phases already planned
  const size_t smem = size_stages(p);
  KT_REQUIRE(smem > 0, "conv_tc: shared memory budget exceeded (rows=%d NT=%d)", p.rows, p.NT);
  const long long tiles = (long long)p.ph_mt0[p.nphases] * p.ntiles * ceil_div(p.batch, p.pack);
  const int grid = (int)std::min<long long>(tiles, device_sm_count());
  const int rc = p.planes == 1 ? launch_route<1>(p, maps, tma, stream, masked, grid, smem, st)
                               : launch_route<2>(p, maps, tma, stream, masked, grid, smem, st);
  if (rc) return rc;
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

// split_planes_kernel of one operand [batch][t][c] (nsub == 1, c % 8 == 0) for a whole-utterance masked forward: item b's rows
// at or past lengths[b] * rows_per_frame are written as zeros, so the TMA route's images need no mask of their own.  The
// other rows get split_planes_kernel's bits.
template <int PL>
__global__ void split_planes_masked_kernel(Side s, long long n8, __nv_bfloat16* __restrict__ hi, const __grid_constant__ KtStreamMask m,
                                           int t, int c) {
  __nv_bfloat16* lo = hi + n8 * 8;
  const int c8 = c / 8;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (long long)gridDim.x * blockDim.x) {
    const long long row = i / c8;
    const int b = (int)(row / t), tr = (int)(row - (long long)b * t);
    float x[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (tr < utterance_rows(m, b, t)) {
      const float4 v0 = __ldg(reinterpret_cast<const float4*>(s.p) + 2 * i), v1 = __ldg(reinterpret_cast<const float4*>(s.p) + 2 * i + 1);
      x[0] = v0.x; x[1] = v0.y; x[2] = v0.z; x[3] = v0.w; x[4] = v1.x; x[5] = v1.y; x[6] = v1.z; x[7] = v1.w;
      if (s.mode == SIDE_LRELU)
#pragma unroll
        for (int e = 0; e < 8; ++e) x[e] = x[e] > 0.f ? x[e] : x[e] * s.slope;
    }
    store_planes8<PL>(x, reinterpret_cast<uint8_t*>(hi), reinterpret_cast<uint8_t*>(lo), (size_t)i * 16);
  }
}

// Every launch of plan P with the operands of `io` (in, wimg, bias, resid, mask, out, out_act, out_slope).  The TMA route
// first writes the gathered operand's planes into ws (masked per item when io.smask is a whole-utterance mask).
static int run_plan(const TcPlan& P, const TcParams& io, float* ws, long long ws_floats, const char* what, cudaStream_t st) {
  TcTmaMaps maps{};
  __nv_bfloat16* planes = reinterpret_cast<__nv_bfloat16*>(ws);
  if (P.tma) {
    if (ws == nullptr || ws_floats < P.ws_floats) {
      set_error("%s: workspace too small (%lld < %lld floats)", what, ws_floats, P.ws_floats);
      return KT_ERR_WORKSPACE;
    }
    const TcParams& g = P.launches[0];
    const long long n = (long long)g.batch * g.t_in * g.nsub * g.c_in;
    if (io.smask.lengths != nullptr) {   // (stream chunks never take the TMA route)
      const int blocks = (int)std::max<long long>(1, std::min<long long>((n / 8 + 255) / 256, 132LL * 16));
      if (g.planes == 1) split_planes_masked_kernel<1><<<blocks, 256, 0, st>>>(io.in, n / 8, planes, io.smask, g.t_in, g.c_in);
      else split_planes_masked_kernel<2><<<blocks, 256, 0, st>>>(io.in, n / 8, planes, io.smask, g.t_in, g.c_in);
      KT_CHECK_CUDA(cudaGetLastError());
    } else {
      KT_CHECK_CUDA(split_planes(io.in, n, planes, Side{nullptr, nullptr, 0, 0.f}, 0, nullptr, g.planes, st));
    }
  }
  for (TcParams lp : P.launches) {
    lp.in = io.in; lp.wimg = io.wimg; lp.bias = io.bias; lp.resid = io.resid; lp.mask = io.mask; lp.out = io.out;
    lp.out_act = io.out_act; lp.out_slope = io.out_slope;
    lp.in_pitch = io.in_pitch; lp.in_first = io.in_first; lp.out_pitch = io.out_pitch; lp.out_first = io.out_first;
    lp.res_pitch = io.res_pitch; lp.res_first = io.res_first;
    lp.smask = io.smask;
    auto a16 = [](const void* q) { return ((uintptr_t)q & 15) == 0; };
    // the staged epilogue reads at most one side operand (a forward has no mask, a data gradient no residual): fewer live
    // values, the register-staged instances are at their cap
    lp.epi_staged = lp.epi_staged && io.in_pitch == 0 && !(io.resid && io.mask.p) && a16(io.out) && a16(io.bias) &&
                    a16(io.resid) && a16(io.mask.p);
    for (int rho = 0; P.tma && rho < lp.i_step; ++rho) {
      const int rc = encode_plane_map(&maps.map[rho], planes, lp.batch, lp.t_in, lp.nsub, lp.c_in, lp.i_step, rho, kTcKC, lp.a_box_t, what,
                                      lp.planes);
      if (rc) return rc;
    }
    const int rc = run_tc(lp, maps, P.tma, io.in_pitch > 0, io.smask.lengths != nullptr, st);
    if (rc) return rc;
  }
  return KT_OK;
}

extern "C" int kt_conv1d_fwd_tc(const KtConv1dDesc* d, const float* x, const void* wimg, const float* bias, const float* resid,
                                float* y, float* ws, int64_t ws_floats, void* stream) {
  int rc = validate_conv(d);
  if (rc) return rc;
  KT_REQUIRE(x && wimg && y, "kt_conv1d_fwd_tc: null pointer");
  const TcPlan P = make_tc_plan(d, 0);
  KT_REQUIRE(P.ok, "conv1d_fwd_tc: layer not supported by the tensor-core path");
  TcParams io{};
  io.in = make_side(x, nullptr, d->act_in, d->act_in_slope, false);
  io.wimg = reinterpret_cast<const __nv_bfloat16*>(wimg);
  io.bias = bias; io.resid = resid; io.mask = Side{nullptr, nullptr, 0, 0.f}; io.out = y;
  io.out_act = d->act_out; io.out_slope = d->act_out_slope;
  return run_plan(P, io, ws, ws_floats, "conv1d_fwd_tc", static_cast<cudaStream_t>(stream));
}

// kt_conv1d_fwd_tc with item b's input rows at or past lengths[b] * rows_per_frame read as zeros: the same route, N tile and
// workspace as the unmasked call, except that the register-staged route keeps one item per tile (the bound is per tile)
extern "C" int kt_conv1d_fwd_tc_masked(const KtConv1dDesc* d, const KtStreamMask* m, const float* x, const void* wimg,
                                       const float* bias, const float* resid, float* y, float* ws, int64_t ws_floats,
                                       void* stream) {
  int rc = validate_conv(d);
  if (!rc) rc = validate_utterance_mask(m, "kt_conv1d_fwd_tc_masked");
  if (rc) return rc;
  KT_REQUIRE(x && wimg && y, "kt_conv1d_fwd_tc_masked: null pointer");
  KT_REQUIRE(d->nsub == 1, "kt_conv1d_fwd_tc_masked: masked forwards need nsub == 1");
  const TcPlan P = make_tc_plan(d, 0, true, false, false);
  KT_REQUIRE(P.ok, "kt_conv1d_fwd_tc_masked: layer not supported by the tensor-core path");
  TcParams io{};
  io.in = make_side(x, nullptr, d->act_in, d->act_in_slope, false);
  io.wimg = reinterpret_cast<const __nv_bfloat16*>(wimg);
  io.bias = bias; io.resid = resid; io.mask = Side{nullptr, nullptr, 0, 0.f}; io.out = y;
  io.out_act = d->act_out; io.out_slope = d->act_out_slope;
  io.smask = *m;
  return run_plan(P, io, ws, ws_floats, "kt_conv1d_fwd_tc_masked", static_cast<cudaStream_t>(stream));
}

// One chunk of a stream (KtStreamWin): the register-staged route over the windows; m: the input's utterance bounds (masked
// instances), or null
extern "C" int kt_conv1d_fwd_tc_stream(const KtConv1dDesc* d, const KtStreamWin* w, const KtStreamMask* m, const float* x,
                                       const void* wimg, const float* bias, const float* resid, float* y, void* stream) {
  int rc = validate_stream(d, w, resid, "kt_conv1d_fwd_tc_stream");
  if (!rc && m) rc = validate_stream_mask(m, "kt_conv1d_fwd_tc_stream");
  if (rc) return rc;
  KT_REQUIRE(x && wimg && y, "kt_conv1d_fwd_tc_stream: null pointer");
  const TcPlan P = make_tc_plan_flags(d, KT_PLAN_STREAM);
  KT_REQUIRE(P.ok && !P.tma, "kt_conv1d_fwd_tc_stream: layer not supported by the tensor-core path");
  KT_REQUIRE(w->in_pitch > 0 && w->out_pitch > 0, "kt_conv1d_fwd_tc_stream: bad window pitch");
  TcParams io{};
  io.in = make_side(x, nullptr, d->act_in, d->act_in_slope, false);
  io.wimg = reinterpret_cast<const __nv_bfloat16*>(wimg);
  io.bias = bias; io.resid = resid; io.mask = Side{nullptr, nullptr, 0, 0.f}; io.out = y;
  io.out_act = d->act_out; io.out_slope = d->act_out_slope;
  io.in_pitch = w->in_pitch; io.in_first = w->in_first; io.out_pitch = w->out_pitch; io.out_first = w->out_first;
  io.res_pitch = w->res_pitch; io.res_first = w->res_first;
  if (m) io.smask = *m;
  return run_plan(P, io, nullptr, 0, "kt_conv1d_fwd_tc_stream", static_cast<cudaStream_t>(stream));
}

int conv1d_bwd_data_tc(const KtConv1dDesc* d, const float* dy, const float* y, const void* wimg, const float* x,
                       float* dx, float* ws, long long ws_floats, cudaStream_t st, bool allow_tma) {
  const TcPlan P = make_tc_plan(d, 1, allow_tma);
  KT_REQUIRE(P.ok, "conv1d_bwd_data_tc: layer not supported by the tensor-core path");
  KT_REQUIRE(d->act_out == KT_ACT_NONE || y != nullptr, "bwd_data: y required when act_out != NONE");
  KT_REQUIRE(d->act_in == KT_ACT_NONE || x != nullptr, "bwd_data: x required when act_in != NONE");
  TcParams io{};
  io.in = make_side(dy, y, d->act_out, d->act_out_slope, true);
  io.wimg = reinterpret_cast<const __nv_bfloat16*>(wimg);
  io.bias = nullptr; io.resid = nullptr; io.out = dx;
  io.mask = dgrad_mask(d, x);
  io.out_act = KT_ACT_NONE; io.out_slope = 0.f;
  return run_plan(P, io, ws, ws_floats, "conv1d_bwd_data_tc", st);
}

extern "C" int kt_conv1d_bwd_data_tc(const KtConv1dDesc* d, const float* dy, const float* y, const void* wimg, const float* x,
                                     float* dx, float* ws, int64_t ws_floats, void* stream) {
  int rc = validate_conv(d);
  if (rc) return rc;
  KT_REQUIRE(dy && wimg && dx, "kt_conv1d_bwd_data_tc: null pointer");
  return conv1d_bwd_data_tc(d, dy, y, wimg, x, dx, ws, ws_floats, static_cast<cudaStream_t>(stream), true);
}

}  // namespace kt
