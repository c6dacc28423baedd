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
// Warp roles: see resblock_tc_kernel.

#include <algorithm>
#include <atomic>
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
  int tile_bytes;                   // one weight tile: [hi NT rows | lo NT rows] x 128 B
  // TMA-staged input (north_star: "TMA-staged input tiles"): the fp32 x tile [rows_box][C] of every tile -- halo included,
  // rows outside [0, T) zero-filled by the TMA unit itself -- is brought into shared memory with cp.async.bulk.tensor (one
  // box of 32 channels x rows_box rows per 32 channels); the producer warps then only CONVERT shared -> shared
  // (LeakyReLU, hi / lo split, swizzled image): no global-load latency, no address arithmetic, no bounds tests.
  int tma;                          // 1: x tiles arrive by TMA (f stages = nx); 0: producer warps load them (LDG)
  int rows_box;                     // rows of one TMA box (rows_x, + d1 for the paired layout)
  int fstage_bytes;                 // one fp32 landing stage: (C / 32) boxes x rows_box x 128 B
  alignas(64) CUtensorMap tmx;      // 3-D map of x: (C, T, B), box (32, rows_box, 1), no swizzle, zero OOB fill
};

// ---- weight packing for the paired (C = 32) layout: tile p = taps (2p, 2p + 1) along K -----------------------------
// w: kernel layout [k][ci][co] (kt_weight_prepare's w_fwd).  Tile p: NT = 32 rows n = co, k index c: c < 32 -> tap 2p,
// ci = c; c >= 32 -> tap 2p + 1, ci = c - 32 (zero when 2p + 1 == k).  [hi tile | lo tile], SWIZZLE_128B rows.
__global__ void rb_pack_pair_kernel(const float* __restrict__ w, int k, int npairs, __nv_bfloat16* __restrict__ out) {
  const int total = npairs * 32 * 64;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int c = i & 63, n = (i >> 6) & 31, p = i >> 11;
    const int tap = 2 * p + (c >> 5), ci = c & 31;
    const float v = tap < k ? w[((long long)tap * 32 + ci) * 32 + n] : 0.f;
    const __nv_bfloat16 hi = __float2bfloat16_rn(v);
    const __nv_bfloat16 lo = __float2bfloat16_rn(v - __bfloat162float(hi));
    const long long base = (long long)p * (2 * 32 * 64);
    const uint32_t off = (sw128_offset((uint32_t)n, (uint32_t)(c >> 3)) >> 1) + (uint32_t)(c & 7);
    out[base + off] = hi;
    out[base + 32 * 64 + off] = lo;
  }
}

// ---- paired staging (C = 32): image row r = [act(x[X0 + r]) (32 ch) | act(x[X0 + r + d]) (32 ch)] ------------------
// 128 threads: thread -> (row = tid / 8 + 16 * i, chunk q = tid % 8); q < 4: channels 8q.. of source row r, q >= 4:
// channels 8(q-4).. of source row r + d.  NB rows per thread are loaded back to back before any conversion.
template <int NB>
__device__ __forceinline__ void rb_stage_pair(uint8_t* img_hi, uint8_t* img_lo, const float* x, long long base_row, int x0,
                                              int d, int t_lim, float slope, int rows, int tid) {
  const int q = tid & 7;
  const int ch = (q & 3) * 8, dsh = (q >> 2) * d;
  for (int r0 = tid >> 3; r0 < rows; r0 += 16 * NB) {
    float4 v[NB][2];
    bool ok[NB];
#pragma unroll
    for (int i = 0; i < NB; ++i) {
      const int r = r0 + 16 * i;
      const int tv = x0 + r + dsh;
      ok[i] = r < rows && tv >= 0 && tv < t_lim;
      const float* src = ok[i] ? x + (base_row + tv) * 32 + ch : x;
      v[i][0] = __ldg(reinterpret_cast<const float4*>(src));
      v[i][1] = __ldg(reinterpret_cast<const float4*>(src) + 1);
    }
#pragma unroll
    for (int i = 0; i < NB; ++i) {
      const int r = r0 + 16 * i;
      float e[8] = {v[i][0].x, v[i][0].y, v[i][0].z, v[i][0].w, v[i][1].x, v[i][1].y, v[i][1].z, v[i][1].w};
#pragma unroll
      for (int z = 0; z < 8; ++z) e[z] = ok[i] ? (e[z] > 0.f ? e[z] : e[z] * slope) : 0.f;
      uint4 hi, lo;
      split8(e, hi, lo);
      if (r < rows) {
        const uint32_t o = sw128_offset((uint32_t)r, (uint32_t)q);
        *reinterpret_cast<uint4*>(img_hi + o) = hi;
        *reinterpret_cast<uint4*>(img_lo + o) = lo;
      }
    }
  }
}

// ---- TMA: one box (32 channels x rows) of the 3-D tensor (C, T, B) -> shared memory, completion on an mbarrier (SASS UTMALDG)
__device__ __forceinline__ void tma_load_box(void* dst_smem, const CUtensorMap* map, int c0, int t0, int b, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(
          smem_u32(dst_smem)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(t0), "r"(b)
      : "memory");
}

// ---- shared fp32 landing tile -> split-bf16 SWIZZLE_128B image (fused LeakyReLU), rows [r_begin, r_end), 128 threads.
// ft: boxes of [rows_box][32 floats] (128-byte rows, linear).  PAIR (C = 32): image row r = [x[r] | x[r + d]];
// else (C = 64): image row r = channels 0..63 of row r, box q / 4.  Rows outside [0, T) arrive as zeros.
template <bool PAIR>
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
    uint4 hi, lo;
    split8(e, hi, lo);
    const uint32_t o = sw128_offset((uint32_t)r, (uint32_t)q);
    *reinterpret_cast<uint4*>(img_hi + o) = hi;
    *reinterpret_cast<uint4*>(img_lo + o) = lo;
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

__global__ void __launch_bounds__(kRbThreads, 1) resblock_tc_kernel(const __grid_constant__ RbParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int NT = p.c;
  const int ximg = p.rows_x * 128, himg = p.rows_h * 128;            // one plane
  const int nslots = p.resident ? 2 * p.nsteps : p.nb;
  uint8_t* x_base = smem;                                            // nx stages x (hi | lo)
  uint8_t* h_base = x_base + (size_t)p.nx * 2 * ximg;                // (hi | lo)
  uint8_t* w_base = h_base + 2 * (size_t)himg;
  uint8_t* f_base = w_base + (size_t)nslots * p.tile_bytes;          // fp32 landing stages of the TMA-staged x tiles (tma only)
  uint64_t* bars = reinterpret_cast<uint64_t*>(f_base + (p.tma ? (size_t)p.nx * p.fstage_bytes : 0));
  uint64_t* x_full = bars;                 // [2]
  uint64_t* x_empty = x_full + 2;          // [2]
  uint64_t* w_full = x_empty + 2;          // [nslots]
  uint64_t* w_empty = w_full + nslots;     // [nslots] (ring only)
  uint64_t* f_full = w_empty + nslots;     // [2] (tma only): the x tile has landed
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
  for (int i = tid; i < 2 * himg / 16; i += kRbThreads) reinterpret_cast<uint4*>(h_base)[i] = make_uint4(0u, 0u, 0u, 0u);
  for (int i = tid; i < 2 * NT; i += kRbThreads) s_bias[i] = i < NT ? (p.b1 ? p.b1[i] : 0.f) : (p.b2 ? p.b2[i - NT] : 0.f);
  fence_proxy_async();
  __syncthreads();

  if (warp < 4) {
    // ===================== producers: x images (fused input LeakyReLU) =====================
    const int ptid = tid;
    if (p.tma) {
      // TMA-staged: the producers convert the landed fp32 tile; thread 0 issues the loads, `nx` tiles ahead, as soon as the
      // landing stage has been read
      const int r0 = 0, r1 = p.rows_x;
      const int nbox = p.c / 32, box_floats = p.rows_box * 32;
      auto issue = [&](int ti) {
        const int tile = (int)blockIdx.x + ti * (int)gridDim.x;
        const int bb = tile / p.tiles_per_item, it = tile - bb * p.tiles_per_item;
        const int x0 = it * p.to - p.p2 - p.p1;
        const int s = ti % p.nx;
        mbar_arrive_expect_tx(&f_full[s], (uint32_t)p.fstage_bytes);
        for (int bx = 0; bx < nbox; ++bx)
          tma_load_box(f_base + (size_t)s * p.fstage_bytes + (size_t)bx * box_floats * 4, &p.tmx, bx * 32, x0, bb, &f_full[s]);
      };
      if (ptid == 0)
        for (int ti = 0; ti < min(p.nx, ntile_cta); ++ti) issue(ti);
      for (int ti = 0; ti < ntile_cta; ++ti) {
        const int s = ti % p.nx, n = ti / p.nx;
        mbar_wait(&x_empty[s], (uint32_t)((n & 1) ^ 1));
        mbar_wait(&f_full[s], (uint32_t)(n & 1));
        uint8_t* img_hi = x_base + (size_t)s * 2 * ximg;
        const float* ft = reinterpret_cast<const float*>(f_base + (size_t)s * p.fstage_bytes);
        if (p.pair) rb_convert_tile<true>(img_hi, img_hi + ximg, ft, box_floats, p.d1, p.slope, r0, r1, ptid);
        else rb_convert_tile<false>(img_hi, img_hi + ximg, ft, box_floats, p.d1, p.slope, r0, r1, ptid);
        fence_proxy_async();
        mbar_arrive(&x_full[s]);
        asm volatile("bar.sync 2, 128;" ::: "memory");          // every producer thread has read the landing stage
        if (ptid == 0 && ti + p.nx < ntile_cta) issue(ti + p.nx);
      }
    } else {
    const Side sx{p.x, nullptr, SIDE_LRELU, p.slope};
    for (int ti = 0; ti < ntile_cta; ++ti) {
      const int tile = (int)blockIdx.x + ti * (int)gridDim.x;
      const int bb = tile / p.tiles_per_item, it = tile - bb * p.tiles_per_item;
      const int x0 = it * p.to - p.p2 - p.p1;
      const int s = ti % p.nx, n = ti / p.nx;
      mbar_wait(&x_empty[s], (uint32_t)((n & 1) ^ 1));
      uint8_t* img_hi = x_base + (size_t)s * 2 * ximg;
      if (p.pair) {
        rb_stage_pair<4>(img_hi, img_hi + ximg, p.x, (long long)bb * p.t, x0, p.d1, p.t, p.slope, p.rows_x, ptid);
      } else {
        RowMap rm;
        rm.base_row = (long long)bb * p.t; rm.fv0 = x0; rm.nsub = 1; rm.step = 1; rm.rho = 0; rm.up = 1; rm.t_lim = p.t;
        stage_rows<4, true, 4>(img_hi, img_hi + ximg, sx, p.x, nullptr, p.c, 0, p.c, false, rm, p.rows_x, ptid);
      }
      fence_proxy_async();
      mbar_arrive(&x_full[s]);
    }
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
        int it = 0;
        auto stream_conv = [&](const __nv_bfloat16* w) {
          for (int s = 0; s < p.nsteps; ++s, ++it) {
            const int slot = it % p.nb;
            mbar_wait(&w_empty[slot], (uint32_t)(((it / p.nb) & 1) ^ 1));
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
    int it_w = 0;
    // one conv of one tile: A = image (hi plane at a16, lo plane a16 + plane16), taps = descriptor row shifts
    auto run_conv = [&](int cv, uint32_t a16, uint32_t plane16, uint32_t astep, bool first_pass) {
      uint32_t scale_d = 0;
      for (int s = 0; s < p.nsteps; ++s, ++it_w) {
        int slot;
        if (p.resident) {
          slot = cv * p.nsteps + s;
          if (first_pass) mbar_wait(&w_full[slot], 0u);
        } else {
          slot = it_w % p.nb;
          mbar_wait(&w_full[slot], (uint32_t)((it_w / p.nb) & 1));
        }
        const uint32_t a_hi = a16 + (uint32_t)s * astep;
        const uint32_t b_hi = w16 + (uint32_t)slot * tile16;
        const int ks = (s == p.nsteps - 1) ? p.last_kslices : 4;
        wgmma_fence();
        for (int k = 0; k < ks; ++k) {
          wgmma_x3<0, 0>(NT, acc, a_hi + 2u * k, plane16, b_hi + 2u * k, bplane16, scale_d);
          scale_d = 1;
        }
        wgmma_commit();
        wgmma_wait<0>();
        acc_fence(acc);
        if (!p.resident && lane == 0) mbar_arrive(&w_empty[slot]);
      }
    };
    for (int ti = 0; ti < ntile_cta; ++ti) {
      const int tile = (int)blockIdx.x + ti * (int)gridDim.x;
      const int bb = tile / p.tiles_per_item, it = tile - bb * p.tiles_per_item;
      const int s = ti % p.nx, n = ti / p.nx;
      // ---------- c1 ----------
      mbar_wait(&x_full[s], (uint32_t)(n & 1));
      run_conv(0, x16 + (uint32_t)s * 2u * ximg16 + half16, ximg16, step1, ti == 0);
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
        const bool in_range = t >= 0 && t < p.t;                       // else: c2's zero padding
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
          *reinterpret_cast<__nv_bfloat162*>(h_base + himg + o) = lb;
          if (p.pair && r > 0) {   // second half of the previous row: act(h[r]) = "row r - 1, + 1"
            const uint32_t o2 = sw128_offset((uint32_t)(r - 1), (uint32_t)i + 4u) + bo;
            *reinterpret_cast<__nv_bfloat162*>(h_base + o2) = hb;
            *reinterpret_cast<__nv_bfloat162*>(h_base + himg + o2) = lb;
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

// ---------------------------------------------------------------------------------------------
// host
// ---------------------------------------------------------------------------------------------
struct RbPlan {
  bool ok;
  RbParams p;
  size_t smem;
};

static int rb_fixed_smem(int nslots) { return (6 + 2 * nslots) * 8 + 2 * 64 * 4; }

// KANTTS_B200_RB_TMA=0 keeps the producer warps on global loads (A/B testing); default: TMA-staged x tiles when they fit
static bool rb_want_tma() {
  static const bool v = [] { const char* e = getenv("KANTTS_B200_RB_TMA"); return !(e && e[0] == '0'); }();
  return v;
}

static RbPlan rb_plan(const KtResblockDesc* d, bool tma = false) {
  RbPlan pl{};
  RbParams& p = pl.p;
  if (d->path == KT_PATH_FFMA) return pl;
  if (!(d->channels == 32 || d->channels == 64)) return pl;
  if (d->kernel < 1 || d->kernel > 15 || (d->kernel & 1) == 0 || d->dilation < 1 || d->batch < 1 || d->t < 1) return pl;
  const int span1 = (d->kernel - 1) * d->dilation, span2 = d->kernel - 1;
  if (d->pad_left1 < 0 || d->pad_left1 > span1 || d->pad_left2 < 0 || d->pad_left2 > span2) return pl;
  p.batch = d->batch; p.t = d->t; p.c = d->channels; p.k = d->kernel; p.d1 = d->dilation;
  p.p1 = d->pad_left1; p.p2 = d->pad_left2; p.slope = d->slope;
  p.to = kRbM - span2;
  p.tiles_per_item = ceil_div(p.t, p.to);
  p.total_tiles = p.tiles_per_item * p.batch;
  p.pair = p.c == 32 ? 1 : 0;
  p.nsteps = p.pair ? (p.k + 1) / 2 : p.k;
  p.last_kslices = (p.pair && (p.k & 1)) ? 2 : 4;
  p.rows_x = (kRbM + span1 + 7) & ~7;
  p.rows_h = (kRbM + span2 + 7) & ~7;
  p.tile_bytes = 2 * p.c * 128;
  const int himg2 = 2 * p.rows_h * 128;
  p.rows_box = p.rows_x + (p.pair ? p.d1 : 0);
  p.fstage_bytes = (p.c / 32) * p.rows_box * 128;
  if (tma && p.rows_box > 256) return pl;          // TMA box limit
  p.tma = tma ? 1 : 0;
  const int ximg2 = 2 * p.rows_x * 128 + (tma ? p.fstage_bytes : 0);   // one x stage: (hi | lo) image (+ its fp32 landing stage)
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

int resblock_plan(const KtResblockDesc* d) { return rb_plan(d).ok ? 1 : 0; }

long long resblock_image_bytes(const KtResblockDesc* d) {
  const RbPlan pl = rb_plan(d);
  return pl.ok ? (long long)pl.p.nsteps * pl.p.tile_bytes : 0;
}

// w: fp32 kernel-layout weight [k][C][C] of one of the two convs (kt_weight_prepare's w_fwd)
int resblock_pack(const KtResblockDesc* d, const float* w, void* img, cudaStream_t st) {
  const RbPlan pl = rb_plan(d);
  KT_REQUIRE(pl.ok && w && img, "resblock_pack: shape not supported by the fused kernel");
  if (pl.p.pair) {
    const int total = pl.p.nsteps * 32 * 64;
    rb_pack_pair_kernel<<<std::min((total + 255) / 256, 132 * 4), 256, 0, st>>>(w, d->kernel, pl.p.nsteps,
                                                                                reinterpret_cast<__nv_bfloat16*>(img));
    KT_CHECK_CUDA(cudaGetLastError());
    return KT_OK;
  }
  // C = 64: one [hi 64 rows | lo 64 rows] tile per tap == conv_tc's packed forward image of a 64 -> 64 layer
  KtConv1dDesc cd{};
  cd.batch = d->batch; cd.nsub = 1; cd.t_in = d->t; cd.t_out = d->t; cd.c_in = 64; cd.c_out = 64; cd.groups = 1;
  cd.kernel = d->kernel; cd.stride = 1; cd.dilation = 1; cd.pad_left = d->kernel - 1; cd.upsample = 1; cd.path = KT_PATH_TC;
  int tc_pack_layer(const KtConv1dDesc*, int, const float*, void*, cudaStream_t);
  return tc_pack_layer(&cd, 0, w, img, st);
}

int resblock_fwd(const KtResblockDesc* d, const float* x, const void* img1, const float* b1, const void* img2, const float* b2,
                 float* h, float* y, cudaStream_t st) {
  RbPlan pl = rb_plan(d, rb_want_tma() && encode_tiled_fn() != nullptr);
  if (!pl.ok) pl = rb_plan(d, false);
  KT_REQUIRE(pl.ok, "resblock_fwd: shape not supported by the fused kernel (channels 32 / 64, odd kernel)");
  KT_REQUIRE(x && img1 && img2 && y, "resblock_fwd: null pointer");
  RbParams& p = pl.p;
  p.x = x; p.y = y; p.h = h;
  p.w1 = reinterpret_cast<const __nv_bfloat16*>(img1); p.w2 = reinterpret_cast<const __nv_bfloat16*>(img2);
  p.b1 = b1; p.b2 = b2;
  if (p.tma) {
    const cuuint64_t gdim[3] = {(cuuint64_t)p.c, (cuuint64_t)p.t, (cuuint64_t)p.batch};
    const cuuint64_t gstr[2] = {(cuuint64_t)p.c * 4, (cuuint64_t)p.t * p.c * 4};
    const cuuint32_t box[3] = {32, (cuuint32_t)p.rows_box, 1};
    const cuuint32_t estr[3] = {1, 1, 1};
    const CUresult r = encode_tiled_fn()(&p.tmx, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(x), gdim, gstr, box, estr,
                                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    KT_REQUIRE(r == CUDA_SUCCESS, "resblock_fwd: cuTensorMapEncodeTiled failed (%d)", (int)r);
  }
  static std::atomic<bool> cfg{false};
  if (!cfg.load(std::memory_order_acquire)) {
    KT_CHECK_CUDA(cudaFuncSetAttribute(resblock_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem));
    cfg.store(true, std::memory_order_release);
  }
  int dev = 0, sms = 132;
  if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int grid = std::min(p.total_tiles, sms > 0 ? sms : 132);
  resblock_tc_kernel<<<grid, kRbThreads, pl.smem, st>>>(p);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

}  // namespace kt
