// Fused ResidualBlock unit of the HiFi-GAN generator (kantts/models/hifigan/layers.py:213-220):
//
//     h = c1(leaky_relu(x)) + b1          c1: k taps, dilation d1      (layers.py:214-215, convs1[i])
//     y = c2(leaky_relu(h)) + b2 + x      c2: k taps, dilation 1       (layers.py:216-219, convs2[i] + the residual add)
//
// in ONE launch for the thin stages (C = 32 / 64 channels) -- unfused, each of the two convs re-stages its input
// (global fp32 -> split bf16 shared-memory image) and writes / re-reads the intermediate; the pair is bound by that
// staging and by the epilogue, not by the tensor pipe.  Here the intermediate never leaves the
// SM: epilogue 1 turns the c1 accumulators (registers) straight into the split-bf16 shared-memory image c2's MMAs read.
//
// Tile = TO = 128 - (k - 1) consecutive outputs of one batch item.  c2 needs h on the 128 rows [H0, H0 + 128),
// H0 = i * TO - p2 (one M = 128 MMA block; rows outside [0, T) are c2's zero padding); c1 needs x on
// [H0 - p1, H0 + 128 + (k - 1) * d1 - p1).  bf16x3 split precision and the im2col-free row-shift descriptors are those of
// conv_tc.cu.  C = 32 packs TWO taps per 64-wide K chunk: image row r holds [act(x[r]) | act(x[r + d])], so a tap pair is
// one dense K = 64 step and the resident weights halve (k = 11: 96 KB for both convs).
//
// Single-pass bf16 (KT_PATH_BF16): the PL = 1 instances keep one bf16 plane per image and weight tile and issue the hi * hi
// wgmma alone; the layout, the tiling and the pipeline are the bf16x3 ones (PL = 2).
//
// Warp roles: see resblock_tc_kernel.

#include <algorithm>
#include <vector>

#include "common.cuh"
#include "tc_common.cuh"
#include "tma.cuh"

namespace kt {

using namespace tc;

constexpr int kRbThreads = 416;
constexpr int kRbM = 128;

struct RbParams {
  const float* x;
  float* y;
  float* h;                         // optional: c1 output (pre-activation), saved for the backward pass
  const __nv_bfloat16* w1;
  const __nv_bfloat16* w2;
  const float* b1;
  const float* b2;
  int batch, t, c;
  int k, d1, p1, p2;
  float slope;
  int to, tiles_per_item, total_tiles;
  int rows_x, rows_h;               // image rows (multiples of 8)
  int nx;                           // x image stages (1 or 2)
  int pair;                         // C == 32: two taps per K chunk
  int nsteps;                       // MMA steps per conv: k, or ceil(k / 2) when pair
  int last_kslices;                 // K = 16 slices of the last step (pair with odd k: 2, else 4)
  int resident, nb;                 // weights: all tiles resident | ring of nb stages
  int tile_bytes;                   // one weight tile: [hi NT rows | lo NT rows] x 128 B (single-pass bf16: hi only)
  int planes;                       // bf16 planes per image / tile: 2 bf16x3, 1 single-pass bf16 (the instance's PL)
  // TMA-staged input: the fp32 x tile [rows_box][C] of every tile -- halo included, rows outside [0, T) zero-filled by the
  // TMA unit itself -- is brought into shared memory with cp.async.bulk.tensor (one box of 32 channels x rows_box rows per
  // 32 channels, nx landing stages); the producer warps then only CONVERT shared -> shared (LeakyReLU, hi / lo split,
  // swizzled image): no global-load latency, no address arithmetic, no bounds tests.
  int rows_box;                     // rows of one TMA box (rows_x, + d1 for the paired layout): at most 256
  int fstage_bytes;                 // one fp32 landing stage: (C / 32) boxes x rows_box x 128 B
  alignas(64) CUtensorMap tmx;      // 3-D map of x: (C, T, B), box (32, rows_box, 1), no swizzle, zero OOB fill
};

// Parameters of the masked instances (kt_resblock_fwd_masked): RbParams and each item's utterance rows.  A struct of its own,
// so that the unmasked instances keep their parameter block.
struct RbMaskedParams {
  RbParams p;
  KtStreamMask smask;
};

// ---- weight packing for the paired (C = 32) layout: tile p = taps (2p, 2p + 1) along K -----------------------------
// w: kernel layout [k][ci][co] (kt_weight_prepare's w_fwd).  Tile p: NT = 32 rows n = co, k index c: c < 32 -> tap 2p,
// ci = c; c >= 32 -> tap 2p + 1, ci = c - 32 (zero when 2p + 1 == k).  [hi tile | lo tile] (PL = 1: hi), SWIZZLE_128B rows.
template <int PL>
__global__ void rb_pack_pair_kernel(const float* __restrict__ w, int k, int npairs, __nv_bfloat16* __restrict__ out) {
  const int total = npairs * 32 * 64;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int c = i & 63, n = (i >> 6) & 31, p = i >> 11;
    const int tap = 2 * p + (c >> 5), ci = c & 31;
    const float v = tap < k ? w[((long long)tap * 32 + ci) * 32 + n] : 0.f;
    const __nv_bfloat16 hi = __float2bfloat16_rn(v);
    const __nv_bfloat16 lo = __float2bfloat16_rn(v - __bfloat162float(hi));
    const long long base = (long long)p * (PL * 32 * 64);
    const uint32_t off = (sw128_offset((uint32_t)n, (uint32_t)(c >> 3)) >> 1) + (uint32_t)(c & 7);
    out[base + off] = hi;
    if constexpr (PL == 2) out[base + 32 * 64 + off] = lo;
  }
}

// ---- shared fp32 landing tile -> split-bf16 SWIZZLE_128B image (fused LeakyReLU), rows [r_begin, r_end), 128 threads.
// ft: boxes of [rows_box][32 floats] (128-byte rows, linear).  PAIR (C = 32): image row r = [x[r] | x[r + d]];
// else (C = 64): image row r = channels 0..63 of row r, box q / 4.  Rows outside [0, T) arrive as zeros.
template <bool PAIR, int PL>
__device__ __forceinline__ void rb_convert_tile(uint8_t* img_hi, uint8_t* img_lo, const float* ft, int box_floats, int d, float slope,
                                                int r_begin, int r_end, int tid) {
  const int q = tid & 7;
  const float* base = PAIR ? ft + (q >> 2) * d * 32 + (q & 3) * 8 : ft + (q >> 2) * box_floats + (q & 3) * 8;
#pragma unroll 2
  for (int r = r_begin + (tid >> 3); r < r_end; r += 16) {
    const float4 a = *reinterpret_cast<const float4*>(base + r * 32);
    const float4 b = *reinterpret_cast<const float4*>(base + r * 32 + 4);
    float e[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
    for (int z = 0; z < 8; ++z) e[z] = e[z] > 0.f ? e[z] : e[z] * slope;
    store_planes8<PL>(e, img_hi, img_lo, sw128_offset((uint32_t)r, (uint32_t)q));
  }
}

// rb_convert_tile of the masked instances: source rows of the tile at or past lim_r (the item's utterance end, in
// landing-stage rows) convert as zeros
template <bool PAIR, int PL>
__device__ __forceinline__ void rb_convert_tile_masked(uint8_t* img_hi, uint8_t* img_lo, const float* ft, int box_floats, int d,
                                                       float slope, int r_begin, int r_end, int tid, int lim_r) {
  const int q = tid & 7;
  const float* base = PAIR ? ft + (q >> 2) * d * 32 + (q & 3) * 8 : ft + (q >> 2) * box_floats + (q & 3) * 8;
  if (PAIR) lim_r -= (q >> 2) * d;   // the second half of a paired row holds source row r + d
#pragma unroll 2
  for (int r = r_begin + (tid >> 3); r < r_end; r += 16) {
    const float4 a = *reinterpret_cast<const float4*>(base + r * 32);
    const float4 b = *reinterpret_cast<const float4*>(base + r * 32 + 4);
    float e[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
    for (int z = 0; z < 8; ++z) e[z] = r >= lim_r ? 0.f : (e[z] > 0.f ? e[z] : e[z] * slope);
    store_planes8<PL>(e, img_hi, img_lo, sw128_offset((uint32_t)r, (uint32_t)q));
  }
}

// Warp roles (416 threads): warpgroup 0 produces the x images, warpgroups 1 / 2 are the consumers (each: the 64-row half
// of both convs' wgmma and of both epilogues), warp 12 streams weights (bulk async copies).  (Warps hold registers in
// groups of four: 13 warps keep the 128 registers per thread the consumers' accumulators need.)
// Per tile a consumer runs c1 (x image -> registers), epilogue 1 (+b1 -> [h to global] -> lrelu -> split -> its half of
// the H image), a named barrier of both consumers, c2 (H image -> registers) and epilogue 2 (+b2 + x -> y).
constexpr int kRbConsumerArrivals = 8;   // one per consumer warp
constexpr int kRbConsumerBar = 1;        // named barrier of the 256 consumer threads

__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync %0, 256;" ::"n"(kRbConsumerBar) : "memory"); }

// NT = C (32 or 64): the MMA width is a compile-time constant of each instance; PL: bf16 planes (2 bf16x3: resblock_tc_kernel,
// 1 single-pass: resblock_tc_bf16_kernel).  MASK (resblock_tc[_bf16]_masked_kernel): item bb's rows at or past
// lengths[bb] * rows_per_frame read as zeros, both in the x tile (c1's input) and in the H image (c2's input)
template <int NT, int PL, bool MASK = false>
__device__ __forceinline__ void resblock_tc_body(const RbParams& p, const KtStreamMask& smask) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_align_1024(smem_raw);
  const int ximg = p.rows_x * 128, himg = p.rows_h * 128;            // one plane
  const int nslots = p.resident ? 2 * p.nsteps : p.nb;
  uint8_t* x_base = smem;                                            // nx stages x (hi | lo)
  uint8_t* h_base = x_base + (size_t)p.nx * PL * ximg;               // (hi | lo)
  uint8_t* w_base = h_base + PL * (size_t)himg;
  uint8_t* f_base = w_base + (size_t)nslots * p.tile_bytes;          // nx fp32 landing stages of the TMA-staged x tiles
  uint64_t* bars = reinterpret_cast<uint64_t*>(f_base + (size_t)p.nx * p.fstage_bytes);
  uint64_t* x_full = bars;                 // [2]
  uint64_t* x_empty = x_full + 2;          // [2]
  uint64_t* w_full = x_empty + 2;          // [nslots]
  uint64_t* w_empty = w_full + nslots;     // [nslots] (ring only)
  uint64_t* f_full = w_empty + nslots;     // [2] the x tile has landed
  float* s_bias = reinterpret_cast<float*>(f_full + 2);              // b1 | b2 (2 * NT floats)

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int ntile_cta = ((int)blockIdx.x < p.total_tiles) ? (p.total_tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;

  if (tid == 0) {
    for (int s = 0; s < 2; ++s) {
      mbar_init(&x_full[s], 128); mbar_init(&x_empty[s], kRbConsumerArrivals);
      mbar_init(&f_full[s], 1);
    }
    for (int s = 0; s < nslots; ++s) { mbar_init(&w_full[s], 1); mbar_init(&w_empty[s], kRbConsumerArrivals); }
    mbar_fence_init();
    fence_proxy_async();
  }
  // the H image starts as zeros: rows >= 128 (read only by discarded output rows) and, in the paired layout, the
  // second half of row 127 are never written
  for (int i = tid; i < PL * himg / 16; i += kRbThreads) reinterpret_cast<uint4*>(h_base)[i] = make_uint4(0u, 0u, 0u, 0u);
  for (int i = tid; i < 2 * NT; i += kRbThreads) s_bias[i] = i < NT ? (p.b1 ? p.b1[i] : 0.f) : (p.b2 ? p.b2[i - NT] : 0.f);
  fence_proxy_async();
  __syncthreads();

  if (warp < 4) {
    // ===================== producers: x images (fused input LeakyReLU) =====================
    // the producers convert the landed fp32 tile; thread 0 issues the TMA loads, `nx` tiles ahead, as soon as the landing
    // stage has been read
    const int ptid = tid;
    const int r0 = 0, r1 = p.rows_x;
    const int nbox = p.c / 32, box_floats = p.rows_box * 32;
    auto issue = [&](int ti, int s) {   // tile ti of this CTA -> landing stage s
      const int tile = (int)blockIdx.x + ti * (int)gridDim.x;
      const int bb = tile / p.tiles_per_item, it = tile - bb * p.tiles_per_item;
      const int x0 = it * p.to - p.p2 - p.p1;
      mbar_arrive_expect_tx(&f_full[s], (uint32_t)p.fstage_bytes);
      for (int bx = 0; bx < nbox; ++bx)
        tma_load_3d(f_base + (size_t)s * p.fstage_bytes + (size_t)bx * box_floats * 4, &p.tmx, bx * 32, x0, bb, &f_full[s]);
    };
    if (ptid == 0)
      for (int ti = 0; ti < min(p.nx, ntile_cta); ++ti) issue(ti, ti);
    RingPos rx;
    for (int ti = 0; ti < ntile_cta; ++ti, rx.advance(p.nx)) {
      const int s = rx.slot();
      mbar_wait(&x_empty[s], rx.phase() ^ 1u);
      mbar_wait(&f_full[s], rx.phase());
      uint8_t* img_hi = x_base + (size_t)s * PL * ximg;
      const float* ft = reinterpret_cast<const float*>(f_base + (size_t)s * p.fstage_bytes);
      if constexpr (MASK) {
        const int tile = (int)blockIdx.x + ti * (int)gridDim.x;
        const int bb = tile / p.tiles_per_item, it = tile - bb * p.tiles_per_item;
        const int lim_r = utterance_rows(smask, bb, p.t) - (it * p.to - p.p2 - p.p1);   // landing-stage row of the item's end
        if (p.pair) rb_convert_tile_masked<true, PL>(img_hi, img_hi + ximg, ft, box_floats, p.d1, p.slope, r0, r1, ptid, lim_r);
        else rb_convert_tile_masked<false, PL>(img_hi, img_hi + ximg, ft, box_floats, p.d1, p.slope, r0, r1, ptid, lim_r);
      } else {
        if (p.pair) rb_convert_tile<true, PL>(img_hi, img_hi + ximg, ft, box_floats, p.d1, p.slope, r0, r1, ptid);
        else rb_convert_tile<false, PL>(img_hi, img_hi + ximg, ft, box_floats, p.d1, p.slope, r0, r1, ptid);
      }
      fence_proxy_async();
      mbar_arrive(&x_full[s]);
      asm volatile("bar.sync 2, 128;" ::: "memory");          // every producer thread has read the landing stage
      if (ptid == 0 && ti + p.nx < ntile_cta) issue(ti + p.nx, s);
    }
  } else if (warp == 12) {
    // ===================== weight stream =====================
    if (elect_one() && ntile_cta > 0) {
      if (p.resident) {
        for (int s = 0; s < 2 * p.nsteps; ++s) {
          const uint8_t* src = reinterpret_cast<const uint8_t*>(s < p.nsteps ? p.w1 : p.w2) + (size_t)(s < p.nsteps ? s : s - p.nsteps) * p.tile_bytes;
          mbar_arrive_expect_tx(&w_full[s], (uint32_t)p.tile_bytes);
          bulk_g2s(w_base + (size_t)s * p.tile_bytes, src, (uint32_t)p.tile_bytes, &w_full[s]);
        }
        for (int s = 0; s < 2 * p.nsteps; ++s) mbar_wait(&w_full[s], 0);   // no bulk copy may outlive the CTA
      } else {
        // same job order as the consumers: per tile c1, c2
        RingPos rw;
        auto stream_conv = [&](const __nv_bfloat16* w) {
          for (int s = 0; s < p.nsteps; ++s, rw.advance(p.nb)) {
            const int slot = rw.slot();
            mbar_wait(&w_empty[slot], rw.phase() ^ 1u);
            mbar_arrive_expect_tx(&w_full[slot], (uint32_t)p.tile_bytes);
            bulk_g2s(w_base + (size_t)slot * p.tile_bytes, reinterpret_cast<const uint8_t*>(w) + (size_t)s * p.tile_bytes,
                     (uint32_t)p.tile_bytes, &w_full[slot]);
          }
        };
        for (int ti = 0; ti < ntile_cta; ++ti) {
          stream_conv(p.w1);
          stream_conv(p.w2);
        }
      }
    }
    __syncwarp();
  } else if (warp >= 4 && warp < 12) {
    // ===================== consumers =====================
    const int cw = (warp - 4) >> 2;                  // 0: accumulator rows 0-63, 1: rows 64-127
    const int wq = warp & 3;
    const uint32_t x16 = smem_u32(x_base) >> 4, h16 = smem_u32(h_base) >> 4, w16 = smem_u32(w_base) >> 4;
    const uint32_t half16 = (uint32_t)cw * 512u;                      // 64 rows x 128 B
    const uint32_t ximg16 = (uint32_t)ximg >> 4, himg16 = (uint32_t)himg >> 4, tile16 = (uint32_t)p.tile_bytes >> 4;
    const uint32_t bplane16 = (uint32_t)(NT * 128) >> 4;
    const uint32_t step1 = (uint32_t)((p.pair ? 2 : 1) * p.d1) * 8u;      // row shift per MMA step, 16-byte units
    const uint32_t step2 = (uint32_t)(p.pair ? 2 : 1) * 8u;
    float acc[kWgmmaMaxRegs];
#pragma unroll
    for (int i = 0; i < kWgmmaMaxRegs; ++i) acc[i] = 0.f;
    RingPos rw;   // weight ring (not used with resident weights)
    // one conv of one tile: A = image (hi plane at a16, lo plane a16 + plane16), taps = descriptor row shifts
    // One MMA group stays in flight: a step's wait retires the PREVIOUS step, whose ring slot is then released.  (Draining
    // every step instead -- wait<0> between the steps' wgmmas -- makes ptxas serialise every wgmma of the kernel, C7515.)
    auto run_conv = [&](int cv, uint32_t a16, uint32_t plane16, uint32_t astep, bool first_pass) {
      uint32_t scale_d = 0;
      int held = -1;   // ring slot read by the group in flight
      for (int s = 0; s < p.nsteps; ++s) {
        int slot;
        if (p.resident) {
          slot = cv * p.nsteps + s;
          if (first_pass) mbar_wait(&w_full[slot], 0u);
        } else {
          slot = rw.slot();
          mbar_wait(&w_full[slot], rw.phase());
          rw.advance(p.nb);
        }
        const uint32_t a_hi = a16 + (uint32_t)s * astep;
        const uint32_t b_hi = w16 + (uint32_t)slot * tile16;
        const int ks = warp_uniform((s == p.nsteps - 1) ? p.last_kslices : 4);
        wgmma_fence();
        for (int k = 0; k < ks; ++k) {
          wgmma_slice<PL, NT, 0, 0>(acc, a_hi + 2u * k, plane16, b_hi + 2u * k, bplane16, scale_d);
          scale_d = 1;
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (held >= 0 && lane == 0) mbar_arrive(&w_empty[held]);
        held = p.resident ? -1 : slot;
      }
      wgmma_wait<0>();
      acc_fence(acc);
      if (held >= 0 && lane == 0) mbar_arrive(&w_empty[held]);
    };
    RingPos rx;
    for (int ti = 0; ti < ntile_cta; ++ti, rx.advance(p.nx)) {
      const int tile = (int)blockIdx.x + ti * (int)gridDim.x;
      const int bb = tile / p.tiles_per_item, it = tile - bb * p.tiles_per_item;
      const int s = rx.slot();
      // ---------- c1 ----------
      mbar_wait(&x_full[s], rx.phase());
      run_conv(0, x16 + (uint32_t)s * (uint32_t)PL * ximg16 + half16, ximg16, step1, ti == 0);
      if (lane == 0) mbar_arrive(&x_empty[s]);
      // ---------- epilogue 1: h = acc + b1 -> [global] -> lrelu -> split -> H image ----------
      const int h0 = it * p.to - p.p2;
#pragma unroll
      for (int i = 0; i < kWgmmaMaxRegs; ++i)
        if ((i >> 2) * 8 < NT) acc[i] += s_bias[(i >> 2) * 8 + 2 * (lane & 3) + (i & 1)];
      if (p.h) {
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int r = cw * 64 + wq * 16 + (lane >> 2) + 8 * hh;
          const int t = h0 + r;
          if (!(r >= p.p2 && r < p.p2 + p.to && t < p.t)) continue;
          float* dst = p.h + ((long long)bb * p.t + t) * p.c + 2 * (lane & 3);
#pragma unroll
          for (int i = 0; i < kWgmmaMaxRegs / 4; ++i)
            if (i * 8 < NT) *reinterpret_cast<float2*>(dst + i * 8) = make_float2(acc[4 * i + 2 * hh], acc[4 * i + 2 * hh + 1]);
        }
      }
      consumer_sync();   // both consumers have finished c2 of the previous tile: the H image may be rewritten
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int r = cw * 64 + wq * 16 + (lane >> 2) + 8 * hh;
        const int t = h0 + r;
        // else: c2's zero padding (masked: also the rows past the item's end)
        const bool in_range = t >= 0 && t < (MASK ? utterance_rows(smask, bb, p.t) : p.t);
#pragma unroll
        for (int i = 0; i < kWgmmaMaxRegs / 4; ++i) {
          if (i * 8 >= NT) continue;
          float e2[2];
#pragma unroll
          for (int z = 0; z < 2; ++z) {
            const float hv = acc[4 * i + 2 * hh + z];
            e2[z] = in_range ? (hv > 0.f ? hv : hv * p.slope) : 0.f;
          }
          const __nv_bfloat162 hb = __floats2bfloat162_rn(e2[0], e2[1]);
          const float2 hf = __bfloat1622float2(hb);
          const __nv_bfloat162 lb = __floats2bfloat162_rn(e2[0] - hf.x, e2[1] - hf.y);
          const uint32_t bo = 4u * (uint32_t)(lane & 3);                // byte offset of this thread's 2 channels in the 16-byte chunk
          const uint32_t o = sw128_offset((uint32_t)r, (uint32_t)i) + bo;
          *reinterpret_cast<__nv_bfloat162*>(h_base + o) = hb;
          if constexpr (PL == 2) *reinterpret_cast<__nv_bfloat162*>(h_base + himg + o) = lb;
          if (p.pair && r > 0) {   // second half of the previous row: act(h[r]) = "row r - 1, + 1"
            const uint32_t o2 = sw128_offset((uint32_t)(r - 1), (uint32_t)i + 4u) + bo;
            *reinterpret_cast<__nv_bfloat162*>(h_base + o2) = hb;
            if constexpr (PL == 2) *reinterpret_cast<__nv_bfloat162*>(h_base + himg + o2) = lb;
          }
        }
      }
      fence_proxy_async();
      consumer_sync();   // the whole H image is written
      // ---------- c2 ----------
      run_conv(1, h16 + half16, himg16, step2, ti == 0);
      // ---------- epilogue 2: y = acc + b2 + x ----------
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int r = cw * 64 + wq * 16 + (lane >> 2) + 8 * hh;
        const int t = it * p.to + r;
        if (!(r < p.to && t < p.t)) continue;
        const long long o = ((long long)bb * p.t + t) * p.c + 2 * (lane & 3);
#pragma unroll
        for (int i = 0; i < kWgmmaMaxRegs / 4; ++i) {
          if (i * 8 >= NT) continue;
          const int col = i * 8 + 2 * (lane & 3);
          const float2 xv = __ldg(reinterpret_cast<const float2*>(p.x + o + i * 8));
          *reinterpret_cast<float2*>(p.y + o + i * 8) =
              make_float2(acc[4 * i + 2 * hh] + s_bias[NT + col] + xv.x, acc[4 * i + 2 * hh + 1] + s_bias[NT + col + 1] + xv.y);
        }
      }
    }
  }
}

template <int NT>
__global__ void __launch_bounds__(kRbThreads, 1) resblock_tc_kernel(const __grid_constant__ RbParams p) {
  resblock_tc_body<NT, 2>(p, KtStreamMask{});
}
template <int NT>
__global__ void __launch_bounds__(kRbThreads, 1) resblock_tc_bf16_kernel(const __grid_constant__ RbParams p) {
  resblock_tc_body<NT, 1>(p, KtStreamMask{});
}
template <int NT>
__global__ void __launch_bounds__(kRbThreads, 1) resblock_tc_masked_kernel(const __grid_constant__ RbMaskedParams mp) {
  resblock_tc_body<NT, 2, true>(mp.p, mp.smask);
}
template <int NT>
__global__ void __launch_bounds__(kRbThreads, 1) resblock_tc_bf16_masked_kernel(const __grid_constant__ RbMaskedParams mp) {
  resblock_tc_body<NT, 1, true>(mp.p, mp.smask);
}

// ---------------------------------------------------------------------------------------------
// host
// ---------------------------------------------------------------------------------------------
struct RbPlan {
  bool ok;
  RbParams p;
  size_t smem;
};

static int rb_fixed_smem(int nslots) { return (6 + 2 * nslots) * 8 + 2 * 64 * 4; }

// geometry only (no device query): kt_resblock_plan answers without a GPU
static RbPlan rb_plan(const KtResblockDesc* d) {
  RbPlan pl{};
  RbParams& p = pl.p;
  if (d->path == KT_PATH_FFMA) return pl;
  if (!(d->channels == 32 || d->channels == 64)) return pl;
  if (d->kernel < 1 || d->kernel > 15 || (d->kernel & 1) == 0 || d->dilation < 1 || d->batch < 1 || d->t < 1) return pl;
  const int span1 = (d->kernel - 1) * d->dilation, span2 = d->kernel - 1;
  if (d->pad_left1 < 0 || d->pad_left1 > span1 || d->pad_left2 < 0 || d->pad_left2 > span2) return pl;
  p.batch = d->batch; p.t = d->t; p.c = d->channels; p.k = d->kernel; p.d1 = d->dilation;
  p.p1 = d->pad_left1; p.p2 = d->pad_left2; p.slope = d->slope;
  p.planes = d->path == KT_PATH_BF16 ? 1 : 2;
  p.to = kRbM - span2;
  p.tiles_per_item = ceil_div(p.t, p.to);
  p.total_tiles = p.tiles_per_item * p.batch;
  p.pair = p.c == 32 ? 1 : 0;
  p.nsteps = p.pair ? (p.k + 1) / 2 : p.k;
  p.last_kslices = (p.pair && (p.k & 1)) ? 2 : 4;
  p.rows_x = (kRbM + span1 + 7) & ~7;
  p.rows_h = (kRbM + span2 + 7) & ~7;
  p.tile_bytes = p.planes * p.c * 128;
  const int himg2 = p.planes * p.rows_h * 128;
  p.rows_box = p.rows_x + (p.pair ? p.d1 : 0);
  p.fstage_bytes = (p.c / 32) * p.rows_box * 128;
  if (p.rows_box > 256) return pl;                 // TMA box limit (k >= 13 with dilation >= 9): the pair runs as two convs
  const int ximg2 = p.planes * p.rows_x * 128 + p.fstage_bytes;   // one x stage: (hi | lo) image + its fp32 landing stage
  const int cap = kMaxDynSmem - 1024;
  // preference: resident weights + 2 x stages; resident + 1; ring (>= 3 stages) + 2 x stages; ring + 1
  const int res_bytes = 2 * p.nsteps * p.tile_bytes;
  auto fits = [&](int nx, int wbytes, int nslots) { return nx * ximg2 + himg2 + wbytes + rb_fixed_smem(nslots) <= cap; };
  if (fits(2, res_bytes, 2 * p.nsteps)) { p.resident = 1; p.nx = 2; p.nb = 0; }
  else if (fits(1, res_bytes, 2 * p.nsteps)) { p.resident = 1; p.nx = 1; p.nb = 0; }
  else {
    p.resident = 0;
    p.nx = 2;
    int nb = (cap - 2 * ximg2 - himg2 - rb_fixed_smem(8)) / p.tile_bytes;
    if (nb < 3) { p.nx = 1; nb = (cap - ximg2 - himg2 - rb_fixed_smem(8)) / p.tile_bytes; }
    if (nb < 3) return pl;
    p.nb = std::min(nb, 8);
  }
  const int nslots = p.resident ? 2 * p.nsteps : p.nb;
  pl.smem = 1024 + (size_t)p.nx * ximg2 + himg2 + (size_t)nslots * p.tile_bytes + rb_fixed_smem(nslots);
  pl.ok = true;
  return pl;
}

extern "C" int kt_resblock_plan(const KtResblockDesc* d) { return d && rb_plan(d).ok ? 1 : 0; }

extern "C" int64_t kt_resblock_image_bytes(const KtResblockDesc* d) {
  if (!d) return 0;
  const RbPlan pl = rb_plan(d);
  return pl.ok ? (int64_t)pl.p.nsteps * pl.p.tile_bytes : 0;
}

// w: fp32 kernel-layout weight [k][C][C] of one of the two convs (kt_weight_prepare's w_fwd)
extern "C" int kt_resblock_pack(const KtResblockDesc* d, const float* w, void* img, void* stream) {
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  KT_REQUIRE(d, "kt_resblock_pack: null descriptor");
  const RbPlan pl = rb_plan(d);
  KT_REQUIRE(pl.ok && w && img, "resblock_pack: shape not supported by the fused kernel");
  if (pl.p.pair) {
    const int total = pl.p.nsteps * 32 * 64;
    const int blocks = std::min((total + 255) / 256, 132 * 4);
    auto* out = reinterpret_cast<__nv_bfloat16*>(img);
    if (pl.p.planes == 1) rb_pack_pair_kernel<1><<<blocks, 256, 0, st>>>(w, d->kernel, pl.p.nsteps, out);
    else rb_pack_pair_kernel<2><<<blocks, 256, 0, st>>>(w, d->kernel, pl.p.nsteps, out);
    KT_CHECK_CUDA(cudaGetLastError());
    return KT_OK;
  }
  // C = 64: one [hi 64 rows | lo 64 rows] tile per tap (hi only in single-pass bf16) == conv_tc's packed forward image of a
  // 64 -> 64 layer of the same precision
  KtConv1dDesc cd{};
  cd.batch = d->batch; cd.nsub = 1; cd.t_in = d->t; cd.t_out = d->t; cd.c_in = 64; cd.c_out = 64; cd.groups = 1;
  cd.kernel = d->kernel; cd.stride = 1; cd.dilation = 1; cd.pad_left = d->kernel - 1; cd.upsample = 1;
  cd.path = d->path == KT_PATH_BF16 ? KT_PATH_BF16 : KT_PATH_TC;
  return tc_pack_layer(&cd, 0, w, img, st);
}

template <int PL>
static int launch_resblock(const RbParams& p, int grid, size_t smem, cudaStream_t st) {
  constexpr auto k32 = PL == 1 ? resblock_tc_bf16_kernel<32> : resblock_tc_kernel<32>;
  constexpr auto k64 = PL == 1 ? resblock_tc_bf16_kernel<64> : resblock_tc_kernel<64>;
  KT_CHECK_CUDA(allow_dyn_smem<k32>(kMaxDynSmem));
  KT_CHECK_CUDA(allow_dyn_smem<k64>(kMaxDynSmem));
  if (p.c == 32) k32<<<grid, kRbThreads, smem, st>>>(p);
  else k64<<<grid, kRbThreads, smem, st>>>(p);
  return KT_OK;
}

template <int PL>
static int launch_resblock_masked(const RbMaskedParams& mp, int grid, size_t smem, cudaStream_t st) {
  constexpr auto k32 = PL == 1 ? resblock_tc_bf16_masked_kernel<32> : resblock_tc_masked_kernel<32>;
  constexpr auto k64 = PL == 1 ? resblock_tc_bf16_masked_kernel<64> : resblock_tc_masked_kernel<64>;
  KT_CHECK_CUDA(allow_dyn_smem<k32>(kMaxDynSmem));
  KT_CHECK_CUDA(allow_dyn_smem<k64>(kMaxDynSmem));
  if (mp.p.c == 32) k32<<<grid, kRbThreads, smem, st>>>(mp);
  else k64<<<grid, kRbThreads, smem, st>>>(mp);
  return KT_OK;
}

static int resblock_fwd(const KtResblockDesc* d, const KtStreamMask* m, const float* x, const void* img1, const float* b1,
                        const void* img2, const float* b2, float* h, float* y, cudaStream_t st) {
  KT_REQUIRE(d, "kt_resblock_fwd: null descriptor");
  RbPlan pl = rb_plan(d);
  KT_REQUIRE(pl.ok, "resblock_fwd: shape not supported by the fused kernel (see kt_resblock_plan)");
  KT_REQUIRE(x && img1 && img2 && y, "resblock_fwd: null pointer");
  RbParams& p = pl.p;
  p.x = x; p.y = y; p.h = h;
  p.w1 = reinterpret_cast<const __nv_bfloat16*>(img1); p.w2 = reinterpret_cast<const __nv_bfloat16*>(img2);
  p.b1 = b1; p.b2 = b2;
  const cuuint64_t gdim[3] = {(cuuint64_t)p.c, (cuuint64_t)p.t, (cuuint64_t)p.batch};
  const cuuint64_t gstr[2] = {(cuuint64_t)p.c * 4, (cuuint64_t)p.t * p.c * 4};
  const cuuint32_t box[3] = {32, (cuuint32_t)p.rows_box, 1};
  const int rc = encode_tensor_map(&p.tmx, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, x, gdim, gstr, box, CU_TENSOR_MAP_SWIZZLE_NONE,
                                   CU_TENSOR_MAP_L2_PROMOTION_L2_128B, "resblock_fwd");
  if (rc) return rc;
  const int grid = std::min(p.total_tiles, device_sm_count());
  int rc2;
  if (m) {
    RbMaskedParams mp{};
    mp.p = p;
    mp.smask = *m;
    rc2 = p.planes == 1 ? launch_resblock_masked<1>(mp, grid, pl.smem, st) : launch_resblock_masked<2>(mp, grid, pl.smem, st);
  } else {
    rc2 = p.planes == 1 ? launch_resblock<1>(p, grid, pl.smem, st) : launch_resblock<2>(p, grid, pl.smem, st);
  }
  if (rc2) return rc2;
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

extern "C" int kt_resblock_fwd(const KtResblockDesc* d, const float* x, const void* img1, const float* b1, const void* img2,
                               const float* b2, float* h, float* y, void* stream) {
  return resblock_fwd(d, nullptr, x, img1, b1, img2, b2, h, y, static_cast<cudaStream_t>(stream));
}

// kt_resblock_fwd with item b's rows at or past lengths[b] * rows_per_frame read as zeros by both convs
extern "C" int kt_resblock_fwd_masked(const KtResblockDesc* d, const KtStreamMask* m, const float* x, const void* img1,
                                      const float* b1, const void* img2, const float* b2, float* h, float* y, void* stream) {
  const int rc = validate_utterance_mask(m, "kt_resblock_fwd_masked");
  if (rc) return rc;
  return resblock_fwd(d, m, x, img1, b1, img2, b2, h, y, static_cast<cudaStream_t>(stream));
}

extern "C" int kt_resblock_bwd(const KtConv1dDesc* d1, const KtConv1dDesc* d2, const float* x, const float* h, const float* dy,
                               const void* wimg1_bwd, const void* wimg2_bwd, float* dh, float* dx, void* stream) {
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  KT_REQUIRE(d1 && d2 && x && h && dy && wimg1_bwd && wimg2_bwd && dh && dx, "kt_resblock_bwd: null pointer");
  KT_REQUIRE(d1->act_in == KT_ACT_LRELU && d2->act_in == KT_ACT_LRELU && d1->act_out == KT_ACT_NONE && d2->act_out == KT_ACT_NONE &&
                 d1->c_in == d1->c_out && d2->c_in == d2->c_out && d1->c_in == d2->c_in && d1->t_in == d2->t_in && d1->t_out == d1->t_in &&
                 d2->t_out == d2->t_in && d1->batch == d2->batch && d1->nsub == 1 && d2->nsub == 1,
             "kt_resblock_bwd: descriptors are not a (convs1[i], convs2[i]) pair of a ResidualBlock");
  // dh = c2^T(dy) * lrelu'(h);  dx = c1^T(dh) * lrelu'(x) + dy   (the residual path, layers.py:219)
  // (register-staged route: this entry point takes no workspace)
  int rc = conv1d_bwd_data_tc(d2, dy, nullptr, wimg2_bwd, h, dh, nullptr, 0, st, false);
  if (rc) return rc;
  rc = conv1d_bwd_data_tc(d1, dh, nullptr, wimg1_bwd, x, dx, nullptr, 0, st, false);
  if (rc) return rc;
  return kt_add3_scale(dx, dy, nullptr, 1.f, dx, (int64_t)d1->batch * d1->t_in * d1->c_in, stream);
}

}  // namespace kt
