// sm_90a primitives used by the tensor-core kernels: mbarrier, bulk async copy (TMA engine, UBLKCP),
// wgmma shared-memory descriptors and warpgroup synchronisation.  Bit layouts follow the PTX ISA "matrix descriptor"
// table of wgmma; everything here is hand-written inline PTX.
#pragma once
#include <cuda_bf16.h>
#include <stdint.h>

#include <algorithm>

#include "common.cuh"
#include "wgmma.cuh"

namespace kt {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// One elected lane of a fully converged warp (elect.sync).  Unlike `if (lane == 0)`, the compiler knows that exactly
// one thread runs the guarded region, so bulk-copy operands move to uniform registers directly.
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

// ---- mbarrier ----
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// Bounded wait: a protocol bug must surface as a trap (launch error), never as a hung GPU.  The try_wait carries CUTLASS's
// suspend-time hint (the hardware parks the warp instead of polling) and the loop must NOT be unrolled: nvcc unrolled it
// 64x at every call site (~2 KB of SASS each, ~15 sites per kernel), and four concurrently running warp roles were
// thrashing the instruction cache (stall_no_inst).
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  uint32_t ok = 0;
#pragma unroll 1
  for (uint32_t spin = 0; spin < (1u << 22); ++spin) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(addr), "r"(parity), "r"(0x989680u)
        : "memory");
    if (ok) return;
  }
  __trap();
}

// Position in a ring of `n` stages, each with a "full" and an "empty" mbarrier: the slot and the parity of its current
// pass.  A consumer waits on full[slot()] with phase(), a producer on empty[slot()] with phase() ^ 1 (the first pass
// finds every slot empty).  Stage counts are run-time values: advance() wraps without a division.  Both live in one
// register, as the loop counter they replace did: conv_tc_kernel's consumers are at the 128-register cap.
struct RingPos {
  uint32_t v = 0;   // slot << 1 | phase
  __device__ __forceinline__ int slot() const { return (int)(v >> 1); }
  __device__ __forceinline__ uint32_t phase() const { return v & 1u; }
  __device__ __forceinline__ void advance(int n) {
    v += 2u;
    if (v >> 1 == (uint32_t)n) v = (v & 1u) ^ 1u;
  }
};

// The dynamic shared-memory base rounded up to 1024 bytes: every SWIZZLE_128B image and tile base must be 1024-byte aligned.
// (pointer arithmetic on the __shared__ array, not integer casts: the compiler must keep the shared address space)
__device__ __forceinline__ uint8_t* smem_align_1024(uint8_t* smem_raw) {
  return smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
}

// generic-proxy writes (st.shared) -> visible to the async proxy (wgmma / bulk copies)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- bulk async copy global -> shared, completion on an mbarrier (TMA engine; SASS UBLKCP) ----
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// ---- warpgroup MMA (wgmma) ----
// Every operand of this library is a SWIZZLE_128B image with 128-byte rows (64 bf16).  Shared-memory matrix descriptor:
//   bits [0,14)  start address >> 4          bits [16,30) leading byte offset >> 4
//   bits [32,46) stride byte offset >> 4     bits [49,52) matrix base offset (0)     bits [62,64) layout: 1 = SWIZZLE_128B
// K-major operand  (rows = M/N index, K contiguous):  SBO = 1024 (8 rows), LBO unused
// MN-major operand (rows = K index, M/N contiguous):  SBO = 1024 (8 K-rows), LBO = stride between 64-element M/N groups
// The high word (SBO = 1024 -> 0x40, SWIZZLE_128B -> bit 30) is a constant; the kernels keep the low word
// (address >> 4) | (LBO >> 4) << 16 and move through an image with 32-bit adds: +2 per K = 16 slice of a K-major operand,
// +128 per 16 rows of an MN-major one, +8 per 128-byte row.  The swizzle XOR acts on absolute shared-memory address bits
// [4,7) ^= [7,10), so a start address advanced by whole rows reads a ROW-SHIFTED view of the same staged image -- this is
// what makes a conv tap a descriptor offset (all image bases are 1024-byte aligned, base offset 0).
constexpr uint32_t kDescHiSw128 = 0x40000040u;
__device__ __forceinline__ uint64_t desc_lo(uint32_t lo) { return ((uint64_t)kDescHiSw128 << 32) | lo; }

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs
__device__ __forceinline__ void acc_fence(float (&d)[kWgmmaMaxRegs]) {
#pragma unroll
  for (int i = 0; i < kWgmmaMaxRegs; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// accumulator element i of thread `lane` of warp `w` (0..3) of the warpgroup: row 16 w + lane / 4 + 8 ((i >> 1) & 1),
// column 8 (i >> 2) + 2 (lane & 3) + (i & 1)

// split-bf16 ("bf16x3") product of one K = 16 slice: lo * hi + hi * lo + hi * hi into the accumulators
// (a_hi / b_hi: descriptor low words of the hi planes, a_pl / b_pl: plane distances in 16-byte units)
template <int N, int TA, int TB>
__device__ __forceinline__ void wgmma_x3(float (&d)[kWgmmaMaxRegs], uint32_t a_hi, uint32_t a_pl, uint32_t b_hi, uint32_t b_pl,
                                         uint32_t scale_d) {
  wgmma_bf16_n<N, TA, TB>(d, desc_lo(a_hi + a_pl), desc_lo(b_hi), scale_d);
  wgmma_bf16_n<N, TA, TB>(d, desc_lo(a_hi), desc_lo(b_hi + b_pl), 1u);
  wgmma_bf16_n<N, TA, TB>(d, desc_lo(a_hi), desc_lo(b_hi), 1u);
}

// One K = 16 slice of a product whose operands are PL bf16 planes (hi, then lo, plane distances a_pl / b_pl): PL = 2 the
// split-bf16 product above, PL = 1 the single-pass bf16 product hi * hi (KT_PATH_BF16)
template <int PL, int N, int TA, int TB>
__device__ __forceinline__ void wgmma_slice(float (&d)[kWgmmaMaxRegs], uint32_t a_hi, uint32_t a_pl, uint32_t b_hi, uint32_t b_pl,
                                            uint32_t scale_d) {
  static_assert(PL == 1 || PL == 2, "wgmma_slice: one or two planes");
  if constexpr (PL == 2) wgmma_x3<N, TA, TB>(d, a_hi, a_pl, b_hi, b_pl, scale_d);
  else wgmma_bf16_n<N, TA, TB>(d, desc_lo(a_hi), desc_lo(b_hi), scale_d);
}

// A value every lane of the warp already holds, in a form ptxas can prove warp-uniform.  ptxas serialises EVERY wgmma of a
// kernel (a wait for completion after each one; ptxas info C7520) when it cannot prove that all threads run the same
// number of them, and it cannot for a loop bound derived from the counter of a loop that waits on an mbarrier: the MMA
// loops take such trip counts through this.
__device__ __forceinline__ int warp_uniform(int v) { return __shfl_sync(0xffffffffu, v, 0); }

// byte offset of 16-byte chunk `q` (0..7) of row `r` inside a 1024-byte-aligned SWIZZLE_128B image
__host__ __device__ __forceinline__ uint32_t sw128_offset(uint32_t r, uint32_t q) { return r * 128u + ((q ^ (r & 7u)) << 4); }

// split 8 fp32 into bf16 hi (round-to-nearest) and bf16 lo = rn(x - hi): x ~= hi + lo to ~2^-17
__device__ __forceinline__ void split8(const float (&x)[8], uint4& hi, uint4& lo) {
  uint32_t h[4], l[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const __nv_bfloat162 hb = __floats2bfloat162_rn(x[2 * i], x[2 * i + 1]);
    const float2 hf = __bfloat1622float2(hb);
    const __nv_bfloat162 lb = __floats2bfloat162_rn(x[2 * i] - hf.x, x[2 * i + 1] - hf.y);
    h[i] = *reinterpret_cast<const uint32_t*>(&hb);
    l[i] = *reinterpret_cast<const uint32_t*>(&lb);
  }
  hi = make_uint4(h[0], h[1], h[2], h[3]);
  lo = make_uint4(l[0], l[1], l[2], l[3]);
}

// Store the planes of 8 values at byte offset o of a hi image (and of its lo image when PL = 2): PL = 1 keeps hi only, the
// round-to-nearest bf16 of each value
template <int PL>
__device__ __forceinline__ void store_planes8(const float (&x)[8], uint8_t* img_hi, uint8_t* img_lo, size_t o) {
  uint4 hi, lo;
  split8(x, hi, lo);
  *reinterpret_cast<uint4*>(img_hi + o) = hi;
  if constexpr (PL == 2) *reinterpret_cast<uint4*>(img_lo + o) = lo;
}

// fp32 operand -> hi / lo bf16 planes ([plane][batch][time][sub-sequence][channel], the activation layout), with the
// operand's fused transform (pre-activation / activation-derivative mask) -- the same arithmetic as stage_rows, so a tile
// pulled from the planes by the TMA unit holds the bits a register-staged tile would.  Two operands in ONE launch: CTAs
// [0, blocks_a) convert operand A, the rest operand B (n8b = 0: none).  Static: every kernel file that feeds its tiles
// from planes compiles its own instance of this one definition.  PL = 1 (single-pass bf16): the hi plane only.
template <int PL>
static __global__ void split_planes_kernel(Side sa, long long n8a, __nv_bfloat16* __restrict__ hia, Side sb, long long n8b,
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
    store_planes8<PL>(x, reinterpret_cast<uint8_t*>(hi), reinterpret_cast<uint8_t*>(lo), (size_t)i * 16);
  }
}

// Launch split_planes_kernel over na elements of operand a into the planes at pa and nb elements of b into pb (na, nb
// multiples of 8; nb = 0: one operand), `planes` (1 or 2) planes each.
static inline cudaError_t split_planes(const Side& a, long long na, __nv_bfloat16* pa, const Side& b, long long nb,
                                       __nv_bfloat16* pb, int planes, cudaStream_t st) {
  auto blocks_for = [](long long n8) { return (int)std::max<long long>(1, std::min<long long>((n8 + 255) / 256, 132LL * 16)); };
  const int ba = blocks_for(na / 8), bb = nb > 0 ? blocks_for(nb / 8) : 0;
  if (planes == 1) split_planes_kernel<1><<<ba + bb, 256, 0, st>>>(a, na / 8, pa, b, nb / 8, pb, ba);
  else split_planes_kernel<2><<<ba + bb, 256, 0, st>>>(a, na / 8, pa, b, nb / 8, pb, ba);
  return cudaGetLastError();
}

}  // namespace tc

// Stage `rows` time steps x 64 channels of a channels-last fp32 tensor into a hi / lo bf16
// SWIZZLE_128B image pair.  128 threads: thread -> (row = tid/8 + 16*i, 16-byte chunk q = tid%8).
// Loads are issued in batches of NB rows per thread BEFORE any conversion so that each thread keeps
// 2*NB (4*NB with an aux tensor) 16-byte loads in flight: with one CTA per SM the
// staging loop is otherwise pure DRAM/L2 latency.
//
// RowMap: image row r -> source row of the channels-last tensor.  The rows of a tile are the
// FLATTENED (time m', sub-sequence w) index fv = m' * nsub + w of one batch item (nsub = period of the
// period discriminator, else 1); the source time is t = m' * step + rho (a strided conv reads one
// residue class rho of the input per image), optionally nearest-upsampled (t / up):
//     fv = fv0 + r;  m' = floor(fv / nsub);  w = fv mod nsub;  tv = m' * step + rho  (valid iff 0 <= tv < t_lim)
//     source row = base_row + (tv / up) * nsub + w
// With this map a conv tap (q, rho) is the row shift q * nsub of residue image rho for ANY stride and
// period, so every M = 128 tile is a dense run of flattened outputs.
// STREAM (a chunk of a stream, nsub == 1): base_row is the row of time step 0 in the item's window, and the rows before it
// are real data down to tv >= t_lo (= -history * up); negative up-sampled times take the floor.
// PACK (packed tiles of the conv kernel, see TcParams::pack): the image holds consecutive blocks of pack_rows rows, block b
// belonging to item b of the tile (item_rows source rows further on); row r is row r - b * pack_rows of its block, and
// blocks past the tile's pack_items items are zero.  pack_magic = floor(2^16 / pack_rows) + 1, so that b = (r * pack_magic)
// >> 16 = r / pack_rows exactly for r * pack_rows < 2^16 (rows < 256, pack_rows <= 128); 0 when the tile holds one item.
struct RowMap {
  long long base_row;
  int fv0, nsub, step, rho, up, t_lim;
  int t_lo;   // STREAM only
  uint32_t pack_magic;
  int pack_rows, pack_items;
  long long item_rows;
  // PACK: image row r -> (row of its item's block, source-row offset of the item); false past the tile's items
  template <bool PACK>
  __device__ __forceinline__ bool block_row(int& r, long long& item) const {
    if constexpr (PACK) {
      const int b = (int)(((uint32_t)r * pack_magic) >> 16);
      if (b >= pack_items) return false;
      r -= b * pack_rows;
      item = b * item_rows;
    }
    return true;
  }
  // nsub == 1 && up == 1 (every layer but the period discriminator's and the nearest-upsampled convs): no divisions
  template <bool STREAM = false, bool PACK = false>
  __device__ __forceinline__ bool map_simple(int r, long long& row) const {
    long long item = 0;
    if (!block_row<PACK>(r, item)) return false;
    const int tv = (fv0 + r) * step + rho;
    if (tv < (STREAM ? t_lo : 0) || tv >= t_lim) return false;
    row = base_row + item + tv;
    return true;
  }
  template <bool STREAM = false, bool PACK = false>
  __device__ __forceinline__ bool map(int r, long long& row) const {
    long long item = 0;
    if (!block_row<PACK>(r, item)) return false;
    const int fv = fv0 + r;
    const int mp = nsub == 1 ? fv : fdiv(fv, nsub);
    const int w = fv - mp * nsub;
    const int tv = mp * step + rho;
    if (tv < (STREAM ? t_lo : 0) || tv >= t_lim) return false;
    row = base_row + item + (long long)(up == 1 ? tv : (STREAM ? fdiv(tv, up) : tv / up)) * nsub + w;
    return true;
  }
};

// Implementation for one (VEC, AUX) combination.  Phase 1 issues ALL global loads of a batch (NB rows x
// 32 bytes, x2 with an aux tensor) back to back with no dependent instruction in between; phase 2
// converts and stores.  The two phases are separate fully-unrolled loops without early exits: with one
// CTA per SM the staging loop is pure DRAM/L2 latency, and a fused load->convert->store loop measured
// ~1 load in flight per thread.
template <int NB, bool VEC, bool AUX, bool SIMPLE = false, bool STREAM = false, bool PACK = false, int PL = 2>
__device__ __forceinline__ void stage_rows_impl(uint8_t* img_hi, uint8_t* img_lo, const Side& s, const float* base,
                                                const float* aux_base, int c_total, int ch0, int nv, const RowMap& rm,
                                                int rows, int tid, int r_begin = 0) {
  const int q = tid & 7;
  for (int r0 = r_begin + (tid >> 3); r0 < rows; r0 += 16 * NB) {
    float4 v[NB][2], a[NB][2];
    long long off[NB];
    bool ok[NB];
#pragma unroll
    for (int i = 0; i < NB; ++i) {
      const int r = r0 + 16 * i;
      long long srow = 0;
      ok[i] = r < rows && nv > 0 && (SIMPLE ? rm.template map_simple<STREAM, PACK>(r, srow) : rm.template map<STREAM, PACK>(r, srow));
      off[i] = ok[i] ? srow * c_total + ch0 + q * 8 : 0;   // offset 0 is always a readable address
    }
#pragma unroll
    for (int i = 0; i < NB; ++i) {
      if constexpr (VEC) {
        v[i][0] = __ldg(reinterpret_cast<const float4*>(base + off[i]));
        v[i][1] = __ldg(reinterpret_cast<const float4*>(base + off[i] + 4));
        if constexpr (AUX) {
          a[i][0] = __ldg(reinterpret_cast<const float4*>(aux_base + off[i]));
          a[i][1] = __ldg(reinterpret_cast<const float4*>(aux_base + off[i] + 4));
        }
      } else {
        float t[8], u[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const long long oe = (ok[i] && e < nv) ? off[i] + e : 0;
          t[e] = __ldg(base + oe);
          u[e] = AUX ? __ldg(aux_base + oe) : 0.f;
          if (!(ok[i] && e < nv)) { t[e] = 0.f; u[e] = 0.f; }
        }
        v[i][0] = make_float4(t[0], t[1], t[2], t[3]); v[i][1] = make_float4(t[4], t[5], t[6], t[7]);
        a[i][0] = make_float4(u[0], u[1], u[2], u[3]); a[i][1] = make_float4(u[4], u[5], u[6], u[7]);
      }
    }
#pragma unroll
    for (int i = 0; i < NB; ++i) {
      const int r = r0 + 16 * i;
      float x[8] = {v[i][0].x, v[i][0].y, v[i][0].z, v[i][0].w, v[i][1].x, v[i][1].y, v[i][1].z, v[i][1].w};
      if (VEC && !ok[i]) {
#pragma unroll
        for (int e = 0; e < 8; ++e) x[e] = 0.f;
      }
      if (s.mode == SIDE_LRELU) {
#pragma unroll
        for (int e = 0; e < 8; ++e) x[e] = x[e] > 0.f ? x[e] : x[e] * s.slope;
      } else if (AUX) {
        const float ax[8] = {a[i][0].x, a[i][0].y, a[i][0].z, a[i][0].w, a[i][1].x, a[i][1].y, a[i][1].z, a[i][1].w};
#pragma unroll
        for (int e = 0; e < 8; ++e) x[e] = side_apply(x[e], ax[e], s.mode, s.slope);
      }
      if (r < rows) tc::store_planes8<PL>(x, img_hi, img_lo, tc::sw128_offset((uint32_t)r, (uint32_t)q));
    }
  }
}

// SIMPLE: the host guarantees nsub == 1, up == 1 and 16-byte-aligned 8-channel chunks (c_valid % 8 == 0, c_total % 4
// == 0): only the vectorised instantiations exist in that kernel variant, which roughly halves its code size -- the
// generic kernel (~140 KB of SASS shared by four concurrently running warp roles) does not fit the instruction cache.
// PL: bf16 planes written per image (2: hi / lo split, 1: hi only, img_lo unused)
template <int NB, bool SIMPLE = false, int NB_AUX = NB, bool STREAM = false, bool PACK = false, int PL = 2>
__device__ __forceinline__ void stage_rows(uint8_t* img_hi, uint8_t* img_lo, const Side& s, const float* base,
                                           const float* aux_base, int c_total, int ch0, int c_valid, bool fill_all,
                                           const RowMap& rm, int rows, int tid, int r_begin = 0) {
  // (r_begin, rows): this group of 128 threads stages image rows [r_begin, rows) -- several groups can share one image
  // c_valid (1..64) = real channels of this 64-wide chunk; the rest of the image row is zero padding
  // (thin / grouped layers).  When channels are the K dimension (forward / dgrad) the 16-byte chunks past
  // the last K = 16 slice the MMA reads need not be written (fill_all = false); when channels are the
  // M / N dimension (weight gradient) every chunk of the row is read and must be zero-filled.
  const int q = tid & 7;
  if (!fill_all && q * 8 >= ((c_valid + 15) & ~15)) return;
  const int nv = min(8, c_valid - q * 8);                       // valid channels of this thread's chunk (may be <= 0)
  if (nv <= 0) {
    // pure padding chunk (thin layers with fill_all): zeros, no loads.  Without this exit such lanes fell into the scalar
    // (non-vector) staging path, and every warp executed BOTH paths: ncu counted ~265 instructions per 8-element chunk for
    // the 32-channel weight gradients against ~80 for full chunks
    const uint4 z = make_uint4(0u, 0u, 0u, 0u);
    for (int r = r_begin + (tid >> 3); r < rows; r += 16) {
      const uint32_t o = tc::sw128_offset((uint32_t)r, (uint32_t)q);
      *reinterpret_cast<uint4*>(img_hi + o) = z;
      if constexpr (PL == 2) *reinterpret_cast<uint4*>(img_lo + o) = z;
    }
    return;
  }
  const bool vec = nv == 8 && (c_total & 3) == 0 && ((ch0 + q * 8) & 3) == 0;
  const bool has_aux = s.mode >= SIDE_DLRELU;
  if constexpr (SIMPLE) {
    if (has_aux) stage_rows_impl<NB_AUX, true, true, true, STREAM, PACK, PL>(img_hi, img_lo, s, base, aux_base, c_total, ch0, nv, rm, rows, tid, r_begin);
    else stage_rows_impl<NB, true, false, true, STREAM, PACK, PL>(img_hi, img_lo, s, base, aux_base, c_total, ch0, nv, rm, rows, tid, r_begin);
    return;
  }
  if (vec) {
    if (has_aux) stage_rows_impl<NB_AUX, true, true, false, STREAM, PACK, PL>(img_hi, img_lo, s, base, aux_base, c_total, ch0, nv, rm, rows, tid, r_begin);
    else stage_rows_impl<NB, true, false, false, STREAM, PACK, PL>(img_hi, img_lo, s, base, aux_base, c_total, ch0, nv, rm, rows, tid, r_begin);
  } else {
    if (has_aux) stage_rows_impl<2, false, true, false, STREAM, PACK, PL>(img_hi, img_lo, s, base, aux_base, c_total, ch0, nv, rm, rows, tid, r_begin);
    else stage_rows_impl<2, false, false, false, STREAM, PACK, PL>(img_hi, img_lo, s, base, aux_base, c_total, ch0, nv, rm, rows, tid, r_begin);
  }
}

}  // namespace kt
