// Exact-fp32 (FFMA) generalised Conv1d kernels, channels-last rows, sm_90a.
//
// Every layer-level operation of the HiFi-GAN hot path (conv / transposed conv /
// nearest-upsampled conv; forward, data gradient, weight gradient; strided, dilated,
// grouped, period-interleaved) is decomposed on the host into "phases" of ONE device
// primitive (struct kt::Phase):
//
//   out[bb][o_off + o_step*m][co] (+)= epi( sum_n sum_ci W[tap_j[n]][ci][co]
//                                            * f_in( in[bb][ floor((m*i_step + tap_ioff[n]) / up) ][ci] ) )
//
// * conv forward            : one phase, i_step = stride, tap_ioff[j] = j*dilation - pad_left
// * conv data-gradient      : `stride` polyphase phases over dy (taps flipped); stride 1 = one phase
// * transposed-conv forward : `stride` polyphase phases (only the taps that hit each output phase)
// * transposed-conv dgrad   : one strided phase
// * nearest-upsampled conv  : forward up = u (rows are gathered at pos / u); its dgrad = u accumulating phases
//
// Thread mapping (core kernel): a warp owns RM output rows x (32*RN) output channels; the lane
// index runs over output channels (contiguous, conflict-free LDS.128 of the weight tile) and the
// input values are warp-uniform broadcast LDS.128 from the channels-last activation tile, so a
// (4 x kk) step costs RM + 4*RN/... shared wavefronts for 4*RM*RN FFMAs per lane.
//
// These kernels are the exact-fp32 path (and the only path for thin layers: C_in/g < 32, C_out = 1).
// The tensor-core kernels in conv_tc.cu take over the GEMM-shaped layers.
#include <stdarg.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <vector>

#include "common.cuh"

namespace kt {

// ---------------------------------------------------------------------------------------------
// error string (thread-local: the ABI is re-entrant across forward / autograd threads)
// ---------------------------------------------------------------------------------------------
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
const char* last_error() { return g_err; }

// ---------------------------------------------------------------------------------------------
// core (forward-like) primitive
// ---------------------------------------------------------------------------------------------
struct CoreParams {
  Side in;
  const float* w;      // [k][cin_g][c_out]
  const float* bias;   // [c_out] or null
  const float* resid;  // out-shaped or null (added after the output activation)
  Side mask;           // epilogue multiply by act'(mask.p) (mode DLRELU) -- data-gradient of a fused pre-activation
  float* out;
  int batch, nsub, t_in, t_out, c_in, c_out, groups, cin_g, cout_g;
  int out_act;
  float out_slope;
  int rmax;            // rows of the activation tile the host sized shared memory for
  Phase ph;
};

__device__ __forceinline__ long long row_index(int bb, int t, int T, int nsub) {
  return ((long long)(bb / nsub) * T + t) * nsub + (bb % nsub);
}

template <int RN, int RM, int KC>
__global__ void __launch_bounds__(256, 2) conv_core_kernel(const __grid_constant__ CoreParams p) {
  constexpr int TN = 32 * RN;
  constexpr int TM = 8 * RM;
  constexpr int NTC = 4;  // taps staged per weight tile
  extern __shared__ __align__(16) float smem[];
  float* x_s = smem;                               // [rmax][KC]
  float* w_s = smem + (size_t)p.rmax * KC;         // [NTC][KC][TN]

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int ctiles = (p.cout_g + TN - 1) / TN;
  const int g = blockIdx.y / ctiles;
  const int co0 = (blockIdx.y % ctiles) * TN;
  const int bb = blockIdx.z;
  const int m0 = blockIdx.x * TM;
  const Phase& ph = p.ph;
  const int up = ph.up;

  const int m_last = min(m0 + TM - 1, ph.M - 1);
  const int pos_lo = m0 * ph.i_step + ph.min_ioff;
  const int pos_hi = m_last * ph.i_step + ph.max_ioff;
  const int row_lo = fdiv(pos_lo, up);
  const int R = min(fdiv(pos_hi, up) - row_lo + 1, p.rmax);

  float acc[RM][RN];
#pragma unroll
  for (int i = 0; i < RM; ++i)
#pragma unroll
    for (int j = 0; j < RN; ++j) acc[i][j] = 0.f;

  const bool vec_in = (p.c_in % 4 == 0) && (p.cin_g % 4 == 0);
  const bool vec_w = (p.c_out % 4 == 0) && (p.cout_g % 4 == 0);

  for (int c0 = 0; c0 < p.cin_g; c0 += KC) {
    __syncthreads();
    // ---- stage the activation tile: rows [row_lo, row_lo+R) x channels [c0, c0+KC) ----
    for (int idx = tid; idx < R * (KC / 4); idx += 256) {
      const int r = idx / (KC / 4), q = idx % (KC / 4);
      const int tin = row_lo + r;
      const int c = c0 + q * 4;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (tin >= 0 && tin < p.t_in && c < p.cin_g) {
        const long long off = row_index(bb, tin, p.t_in, p.nsub) * p.c_in + (long long)g * p.cin_g + c;
        if (vec_in && c + 3 < p.cin_g) {
          v = __ldg(reinterpret_cast<const float4*>(p.in.p + off));
          if (p.in.mode >= SIDE_DLRELU) {
            const float4 a = __ldg(reinterpret_cast<const float4*>(p.in.aux + off));
            v.x = side_apply(v.x, a.x, p.in.mode, p.in.slope);
            v.y = side_apply(v.y, a.y, p.in.mode, p.in.slope);
            v.z = side_apply(v.z, a.z, p.in.mode, p.in.slope);
            v.w = side_apply(v.w, a.w, p.in.mode, p.in.slope);
          } else if (p.in.mode == SIDE_LRELU) {
            v.x = side_apply(v.x, 0.f, SIDE_LRELU, p.in.slope);
            v.y = side_apply(v.y, 0.f, SIDE_LRELU, p.in.slope);
            v.z = side_apply(v.z, 0.f, SIDE_LRELU, p.in.slope);
            v.w = side_apply(v.w, 0.f, SIDE_LRELU, p.in.slope);
          }
        } else {
          float t[4] = {0.f, 0.f, 0.f, 0.f};
          for (int e = 0; e < 4; ++e)
            if (c + e < p.cin_g) {
              const float a = p.in.mode >= SIDE_DLRELU ? __ldg(p.in.aux + off + e) : 0.f;
              t[e] = side_apply(__ldg(p.in.p + off + e), a, p.in.mode, p.in.slope);
            }
          v = make_float4(t[0], t[1], t[2], t[3]);
        }
      }
      *reinterpret_cast<float4*>(&x_s[r * KC + q * 4]) = v;
    }

    for (int nt0 = 0; nt0 < ph.ntaps; nt0 += NTC) {
      const int ntc = min(NTC, ph.ntaps - nt0);
      if (nt0 > 0) __syncthreads();
      // ---- stage the weight tile [ntc][KC][TN] ----
      for (int idx = tid; idx < ntc * KC * (TN / 4); idx += 256) {
        const int cq = idx % (TN / 4);
        const int kk = (idx / (TN / 4)) % KC;
        const int nn = idx / (TN / 4 * KC);
        const int ci = c0 + kk, co = co0 + cq * 4;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (ci < p.cin_g && co < p.cout_g) {
          const long long off = ((long long)ph.tap_j[nt0 + nn] * p.cin_g + ci) * p.c_out + (long long)g * p.cout_g + co;
          if (vec_w && co + 3 < p.cout_g) {
            v = __ldg(reinterpret_cast<const float4*>(p.w + off));
          } else {
            float t[4] = {0.f, 0.f, 0.f, 0.f};
            for (int e = 0; e < 4; ++e)
              if (co + e < p.cout_g) t[e] = __ldg(p.w + off + e);
            v = make_float4(t[0], t[1], t[2], t[3]);
          }
        }
        *reinterpret_cast<float4*>(&w_s[(nn * KC + kk) * TN + cq * 4]) = v;
      }
      __syncthreads();

      // ---- FFMA ----
      for (int nn = 0; nn < ntc; ++nn) {
        const int ioff = ph.tap_ioff[nt0 + nn];
        int rr[RM];
#pragma unroll
        for (int i = 0; i < RM; ++i) {
          const int m = min(m0 + warp * RM + i, ph.M - 1);
          const int pos = m * ph.i_step + ioff;
          int r = (up == 1 ? pos : fdiv(pos, up)) - row_lo;
          rr[i] = min(max(r, 0), R - 1) * KC;
        }
#pragma unroll
        for (int kk = 0; kk < KC; kk += 4) {
          float b[4][RN];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const float* wp = &w_s[(nn * KC + kk + q) * TN + lane * RN];
            if constexpr (RN == 4) {
              const float4 t = *reinterpret_cast<const float4*>(wp);
              b[q][0] = t.x; b[q][1] = t.y; b[q][2] = t.z; b[q][3] = t.w;
            } else if constexpr (RN == 2) {
              const float2 t = *reinterpret_cast<const float2*>(wp);
              b[q][0] = t.x; b[q][1] = t.y;
            } else {
              b[q][0] = wp[0];
            }
          }
#pragma unroll
          for (int i = 0; i < RM; ++i) {
            const float4 a = *reinterpret_cast<const float4*>(&x_s[rr[i] + kk]);
#pragma unroll
            for (int j = 0; j < RN; ++j) {
              acc[i][j] = fmaf(a.x, b[0][j], acc[i][j]);
              acc[i][j] = fmaf(a.y, b[1][j], acc[i][j]);
              acc[i][j] = fmaf(a.z, b[2][j], acc[i][j]);
              acc[i][j] = fmaf(a.w, b[3][j], acc[i][j]);
            }
          }
        }
      }
    }
  }

  // ---- epilogue ----
#pragma unroll
  for (int i = 0; i < RM; ++i) {
    const int m = m0 + warp * RM + i;
    if (m >= ph.M) continue;
    const int to = ph.o_off + ph.o_step * m;
    const long long obase = row_index(bb, to, p.t_out, p.nsub) * p.c_out + (long long)g * p.cout_g;
#pragma unroll
    for (int j = 0; j < RN; ++j) {
      const int co = co0 + lane * RN + j;
      if (co >= p.cout_g) continue;
      const long long o = obase + co;
      float v = acc[i][j];
      if (p.bias) v += __ldg(p.bias + g * p.cout_g + co);
      if (p.out_act == KT_ACT_LRELU) v = v > 0.f ? v : v * p.out_slope;
      else if (p.out_act == KT_ACT_TANH) v = tanhf(v);
      if (p.mask.p) v = side_apply(v, __ldg(p.mask.p + o), p.mask.mode, p.mask.slope);
      if (p.resid) v += __ldg(p.resid + o);
      if (ph.accumulate) v += p.out[o];
      p.out[o] = v;
    }
  }
}

template <int RN, int RM, int KC>
static int launch_core(const CoreParams& p, cudaStream_t st) {
  constexpr int TN = 32 * RN, TM = 8 * RM, NTC = 4;
  const size_t smem = ((size_t)p.rmax * KC + (size_t)NTC * KC * TN) * sizeof(float);
  KT_REQUIRE(smem <= 200 * 1024, "conv_core: activation tile too large (%zu bytes shared)", smem);
  // opt in ONCE per process to the full 227 KB (the attribute is per function, not per thread: a
  // smaller value set later from the autograd thread would make larger launches fail)
  static std::atomic<bool> configured{false};
  if (!configured.load(std::memory_order_acquire)) {
    KT_CHECK_CUDA(cudaFuncSetAttribute(conv_core_kernel<RN, RM, KC>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem));
    configured.store(true, std::memory_order_release);
  }
  dim3 grid(ceil_div(p.ph.M, TM), p.groups * ceil_div(p.cout_g, TN), p.batch);
  conv_core_kernel<RN, RM, KC><<<grid, 256, smem, st>>>(p);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

static int run_core(CoreParams p, cudaStream_t st) {
  if (p.ph.M <= 0 || p.ph.ntaps <= 0) return KT_OK;
  const int RN = p.cout_g > 64 ? 4 : (p.cout_g > 32 ? 2 : 1);
  const int TN = 32 * RN;
  // biggest row tile that still fills the machine (>= 2 CTAs per SM on 132 SMs)
  int RM = 16;
  auto ctas = [&](int rm) { return (long long)ceil_div(p.ph.M, 8 * rm) * p.groups * ceil_div(p.cout_g, TN) * p.batch; };
  while (RM > 4 && (ctas(RM) < 296 || p.ph.M <= 4 * RM)) RM >>= 1;
  const int TM = 8 * RM;
  p.rmax = fdiv((TM - 1) * p.ph.i_step + p.ph.max_ioff - p.ph.min_ioff, p.ph.up) + 2;
  const int KC = p.cin_g <= 4 ? 4 : 16;
#define KT_CORE_CASE(rn, rm, kc) \
  if (RN == rn && RM == rm && KC == kc) return launch_core<rn, rm, kc>(p, st);
  KT_CORE_CASE(4, 16, 16) KT_CORE_CASE(4, 8, 16) KT_CORE_CASE(4, 4, 16)
  KT_CORE_CASE(2, 16, 16) KT_CORE_CASE(2, 8, 16) KT_CORE_CASE(2, 4, 16)
  KT_CORE_CASE(1, 16, 16) KT_CORE_CASE(1, 8, 16) KT_CORE_CASE(1, 4, 16)
  KT_CORE_CASE(4, 16, 4) KT_CORE_CASE(4, 8, 4) KT_CORE_CASE(4, 4, 4)
  KT_CORE_CASE(2, 16, 4) KT_CORE_CASE(2, 8, 4) KT_CORE_CASE(2, 4, 4)
  KT_CORE_CASE(1, 16, 4) KT_CORE_CASE(1, 8, 4) KT_CORE_CASE(1, 4, 4)
#undef KT_CORE_CASE
  set_error("conv_core: no kernel variant");
  return KT_ERR_INVALID;
}

// ---------------------------------------------------------------------------------------------
// weight-gradient primitive
//   G[tap_j[n]][ca][cb] += sum_bb sum_m  fa( A[bb][ floor((m*i_step + tap_ioff[n]) / up) ][ca] ) * fb( Bm[bb][o_off + o_step*m][cb] )
// ---------------------------------------------------------------------------------------------
struct WgradParams {
  Side a, b;
  float* g;  // [k][ca_g][cb_total]; split s accumulates into g + s * g_stride (g_stride = 0: one split)
  long long g_stride;
  int batch, nsub, t_a, t_b, ca_total, cb_total, groups, ca_g, cb_g;
  int rmax;
  int nsplit, npass;
  long long g_size;   // floats of g
  Phase ph;
};

template <int RN, int RMA, bool SPLITM>
__global__ void __launch_bounds__(256, 2) conv_wgrad_kernel(const __grid_constant__ WgradParams p) {
  constexpr int TN = 32 * RN;
  constexpr int TCA = SPLITM ? RMA : 8 * RMA;  // A-side channels per CTA
  constexpr int TK = 32;                       // time steps per staged chunk
  constexpr int NTW = 3;                       // taps accumulated per pass
  extern __shared__ __align__(16) float smem[];
  float* a_s = smem;                           // [rmax][TCA]
  float* b_s = smem + (size_t)p.rmax * TCA;    // [TK][TN]

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const Phase& ph = p.ph;
  const int up = ph.up;
  const int catiles = (p.ca_g + TCA - 1) / TCA;
  const int cbtiles = (p.cb_g + TN - 1) / TN;
  const int ca0 = (blockIdx.x % catiles) * TCA;
  const int g = blockIdx.y / cbtiles;
  const int cb0 = (blockIdx.y % cbtiles) * TN;
  const int pass = blockIdx.z % p.npass;
  const int split = blockIdx.z / p.npass;
  const int n0 = pass * NTW;
  const int nt = min(NTW, ph.ntaps - n0);

  int pmin = ph.tap_ioff[n0], pmax = ph.tap_ioff[n0];
  for (int n = 1; n < nt; ++n) {
    pmin = min(pmin, ph.tap_ioff[n0 + n]);
    pmax = max(pmax, ph.tap_ioff[n0 + n]);
  }

  const int nchunks = (ph.M + TK - 1) / TK;
  const long long units = (long long)p.batch * nchunks;
  const long long u_begin = units * split / p.nsplit;
  const long long u_end = units * (split + 1) / p.nsplit;

  float acc[NTW][RMA][RN];
#pragma unroll
  for (int n = 0; n < NTW; ++n)
#pragma unroll
    for (int i = 0; i < RMA; ++i)
#pragma unroll
      for (int j = 0; j < RN; ++j) acc[n][i][j] = 0.f;

  const bool vec_a = (p.ca_total % 4 == 0) && (p.ca_g % 4 == 0);
  const bool vec_b = (p.cb_total % 4 == 0) && (p.cb_g % 4 == 0);

  for (long long u = u_begin; u < u_end; ++u) {
    const int bb = (int)(u / nchunks);
    const int m0 = (int)(u % nchunks) * TK;
    const int m_last = min(m0 + TK - 1, ph.M - 1);
    const int row_lo = fdiv(m0 * ph.i_step + pmin, up);
    const int R = min(fdiv(m_last * ph.i_step + pmax, up) - row_lo + 1, p.rmax);
    __syncthreads();
    // A tile
    for (int idx = tid; idx < R * (TCA / 4); idx += 256) {
      const int r = idx / (TCA / 4), q = idx % (TCA / 4);
      const int t = row_lo + r;
      const int c = ca0 + q * 4;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (t >= 0 && t < p.t_a && c < p.ca_g) {
        const long long off = row_index(bb, t, p.t_a, p.nsub) * p.ca_total + (long long)g * p.ca_g + c;
        float tv[4] = {0.f, 0.f, 0.f, 0.f};
        if (vec_a && c + 3 < p.ca_g) {
          const float4 x = __ldg(reinterpret_cast<const float4*>(p.a.p + off));
          float4 ax = make_float4(0.f, 0.f, 0.f, 0.f);
          if (p.a.mode >= SIDE_DLRELU) ax = __ldg(reinterpret_cast<const float4*>(p.a.aux + off));
          tv[0] = side_apply(x.x, ax.x, p.a.mode, p.a.slope);
          tv[1] = side_apply(x.y, ax.y, p.a.mode, p.a.slope);
          tv[2] = side_apply(x.z, ax.z, p.a.mode, p.a.slope);
          tv[3] = side_apply(x.w, ax.w, p.a.mode, p.a.slope);
        } else {
          for (int e = 0; e < 4; ++e)
            if (c + e < p.ca_g) {
              const float ax = p.a.mode >= SIDE_DLRELU ? __ldg(p.a.aux + off + e) : 0.f;
              tv[e] = side_apply(__ldg(p.a.p + off + e), ax, p.a.mode, p.a.slope);
            }
        }
        v = make_float4(tv[0], tv[1], tv[2], tv[3]);
      }
      *reinterpret_cast<float4*>(&a_s[r * TCA + q * 4]) = v;
    }
    // B tile
    for (int idx = tid; idx < TK * (TN / 4); idx += 256) {
      const int mm = idx / (TN / 4), q = idx % (TN / 4);
      const int m = m0 + mm;
      const int c = cb0 + q * 4;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (m < ph.M && c < p.cb_g) {
        const int t = ph.o_off + ph.o_step * m;
        const long long off = row_index(bb, t, p.t_b, p.nsub) * p.cb_total + (long long)g * p.cb_g + c;
        float tv[4] = {0.f, 0.f, 0.f, 0.f};
        if (vec_b && c + 3 < p.cb_g) {
          const float4 x = __ldg(reinterpret_cast<const float4*>(p.b.p + off));
          float4 ax = make_float4(0.f, 0.f, 0.f, 0.f);
          if (p.b.mode >= SIDE_DLRELU) ax = __ldg(reinterpret_cast<const float4*>(p.b.aux + off));
          tv[0] = side_apply(x.x, ax.x, p.b.mode, p.b.slope);
          tv[1] = side_apply(x.y, ax.y, p.b.mode, p.b.slope);
          tv[2] = side_apply(x.z, ax.z, p.b.mode, p.b.slope);
          tv[3] = side_apply(x.w, ax.w, p.b.mode, p.b.slope);
        } else {
          for (int e = 0; e < 4; ++e)
            if (c + e < p.cb_g) {
              const float ax = p.b.mode >= SIDE_DLRELU ? __ldg(p.b.aux + off + e) : 0.f;
              tv[e] = side_apply(__ldg(p.b.p + off + e), ax, p.b.mode, p.b.slope);
            }
        }
        v = make_float4(tv[0], tv[1], tv[2], tv[3]);
      }
      *reinterpret_cast<float4*>(&b_s[mm * TN + q * 4]) = v;
    }
    __syncthreads();

    const int mm_begin = SPLITM ? warp : 0;
    const int mm_step = SPLITM ? 8 : 1;
    const int a_col = SPLITM ? 0 : warp * RMA;
    for (int mm = mm_begin; mm < TK; mm += mm_step) {
      float b[RN];
      const float* bp = &b_s[mm * TN + lane * RN];
      if constexpr (RN == 4) {
        const float4 t = *reinterpret_cast<const float4*>(bp);
        b[0] = t.x; b[1] = t.y; b[2] = t.z; b[3] = t.w;
      } else if constexpr (RN == 2) {
        const float2 t = *reinterpret_cast<const float2*>(bp);
        b[0] = t.x; b[1] = t.y;
      } else {
        b[0] = bp[0];
      }
      const int m = min(m0 + mm, ph.M - 1);
#pragma unroll
      for (int n = 0; n < NTW; ++n) {
        if (n < nt) {
          const int pos = m * ph.i_step + ph.tap_ioff[n0 + n];
          int r = (up == 1 ? pos : fdiv(pos, up)) - row_lo;
          r = min(max(r, 0), R - 1);
          const float* ap = &a_s[r * TCA + a_col];
#pragma unroll
          for (int i4 = 0; i4 < RMA; i4 += 4) {
            const float4 a = *reinterpret_cast<const float4*>(ap + i4);
#pragma unroll
            for (int j = 0; j < RN; ++j) {
              acc[n][i4 + 0][j] = fmaf(a.x, b[j], acc[n][i4 + 0][j]);
              acc[n][i4 + 1][j] = fmaf(a.y, b[j], acc[n][i4 + 1][j]);
              acc[n][i4 + 2][j] = fmaf(a.z, b[j], acc[n][i4 + 2][j]);
              acc[n][i4 + 3][j] = fmaf(a.w, b[j], acc[n][i4 + 3][j]);
            }
          }
        }
      }
    }
  }

  // ---- with SPLITM the eight warps hold partials of the same elements (they split the rows): fold them into warp 0 in
  // warp order through shared memory (3 * RMA * RN * 32 floats <= the TK x TN B tile), so that below every element of the
  // split's zeroed slice of G receives exactly one add -- the result does not depend on scheduling
  if constexpr (SPLITM) {
    float* red = smem;
    for (int w = 1; w < 8; ++w) {
      __syncthreads();
      if (warp == w)
#pragma unroll
        for (int e = 0; e < NTW * RMA * RN; ++e) red[e * 32 + lane] = (&acc[0][0][0])[e];
      __syncthreads();
      if (warp == 0)
#pragma unroll
        for (int e = 0; e < NTW * RMA * RN; ++e) (&acc[0][0][0])[e] += red[e * 32 + lane];
    }
    if (warp != 0) return;
  }

  // ---- reduce into G ----
  const int a_col = SPLITM ? 0 : warp * RMA;
#pragma unroll
  for (int n = 0; n < NTW; ++n) {
    if (n >= nt) continue;
    const int j_tap = ph.tap_j[n0 + n];
#pragma unroll
    for (int i = 0; i < RMA; ++i) {
      const int ca = ca0 + a_col + i;
      if (ca >= p.ca_g) continue;
#pragma unroll
      for (int j = 0; j < RN; ++j) {
        const int cb = cb0 + lane * RN + j;
        if (cb >= p.cb_g) continue;
        atomicAdd(p.g + split * p.g_stride + ((long long)j_tap * p.ca_g + ca) * p.cb_total + (long long)g * p.cb_g + cb, acc[n][i][j]);
      }
    }
  }
}

template <int RN, int RMA, bool SPLITM>
static int launch_wgrad(WgradParams p, cudaStream_t st) {
  constexpr int TN = 32 * RN, TCA = SPLITM ? RMA : 8 * RMA, TK = 32, NTW = 3;
  p.rmax = fdiv((TK - 1) * p.ph.i_step + (NTW - 1) * 0 + (p.ph.max_ioff - p.ph.min_ioff), p.ph.up) + 2;
  p.npass = ceil_div(p.ph.ntaps, NTW);
  const long long units = (long long)p.batch * ceil_div(p.ph.M, TK);
  const long long base = (long long)ceil_div(p.ca_g, TCA) * p.groups * ceil_div(p.cb_g, TN) * p.npass;
  long long nsplit = std::max<long long>(1, (132 * 4) / std::max<long long>(1, base));
  nsplit = std::min<long long>(nsplit, std::max<long long>(1, units / 4));
  nsplit = std::min<long long>(nsplit, 4096);
  // every split accumulates into its own zeroed slice of scratch (each element of a slice is added to by one CTA, in a
  // fixed order); the slices are summed in order into g
  const long long g_size = p.g_size;
  nsplit = std::max<long long>(1, std::min<long long>(nsplit, (1LL << 25) / std::max<long long>(1, g_size)));
  p.nsplit = (int)nsplit;
  const size_t smem = ((size_t)p.rmax * TCA + (size_t)TK * TN) * sizeof(float);
  KT_REQUIRE(smem <= 200 * 1024, "conv_wgrad: tile too large (%zu bytes shared)", smem);
  static std::atomic<bool> configured{false};
  if (!configured.load(std::memory_order_acquire)) {
    KT_CHECK_CUDA(cudaFuncSetAttribute(conv_wgrad_kernel<RN, RMA, SPLITM>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem));
    configured.store(true, std::memory_order_release);
  }
  dim3 grid(ceil_div(p.ca_g, TCA), p.groups * ceil_div(p.cb_g, TN), p.npass * p.nsplit);
  float* out = p.g;
  float* part = nullptr;
  p.g_stride = 0;
  if (p.nsplit > 1) {
    int rc = scratch_alloc(&part, (long long)p.nsplit * g_size, st);
    if (rc) return rc;
    KT_CHECK_CUDA(cudaMemsetAsync(part, 0, (size_t)p.nsplit * g_size * sizeof(float), st));
    p.g = part;
    p.g_stride = g_size;
  }
  conv_wgrad_kernel<RN, RMA, SPLITM><<<grid, 256, smem, st>>>(p);
  KT_CHECK_CUDA(cudaGetLastError());
  if (part) {
    int rc = split_sum(part, g_size, p.nsplit, g_size, out, true, st);
    if (rc) return rc;
    return scratch_free(part, st);
  }
  return KT_OK;
}

static int run_wgrad(const WgradParams& p, cudaStream_t st) {
  if (p.ph.M <= 0 || p.ph.ntaps <= 0) return KT_OK;
  const int RN = p.cb_g > 64 ? 4 : (p.cb_g > 32 ? 2 : 1);
  if (p.ca_g <= 4) {
    if (RN == 4) return launch_wgrad<4, 4, true>(p, st);
    if (RN == 2) return launch_wgrad<2, 4, true>(p, st);
    return launch_wgrad<1, 4, true>(p, st);
  }
  if (p.ca_g <= 8) {
    if (RN == 4) return launch_wgrad<4, 8, true>(p, st);
    if (RN == 2) return launch_wgrad<2, 8, true>(p, st);
    return launch_wgrad<1, 8, true>(p, st);
  }
  if (p.ca_g <= 32) {
    if (RN == 4) return launch_wgrad<4, 4, false>(p, st);
    if (RN == 2) return launch_wgrad<2, 4, false>(p, st);
    return launch_wgrad<1, 4, false>(p, st);
  }
  if (RN == 4) return launch_wgrad<4, 8, false>(p, st);
  if (RN == 2) return launch_wgrad<2, 8, false>(p, st);
  return launch_wgrad<1, 8, false>(p, st);
}

// column sums of one row range: part[blockIdx.y][c] = sum_rows f(v[row][c])   (bias gradient, see colsum_bias)
__global__ void colsum_kernel(Side s, long long rows, int c, float* part) {
  const int ch = blockIdx.x * 32 + (threadIdx.x & 31);
  const int rlane = threadIdx.x >> 5;  // 8 row lanes
  float acc = 0.f;
  if (ch < c) {
    for (long long r = (long long)blockIdx.y * 8 + rlane; r < rows; r += (long long)gridDim.y * 8) {
      const long long off = r * c + ch;
      const float a = s.mode >= SIDE_DLRELU ? __ldg(s.aux + off) : 0.f;
      acc += side_apply(__ldg(s.p + off), a, s.mode, s.slope);
    }
  }
  __shared__ float red[8][33];
  red[rlane][threadIdx.x & 31] = acc;
  __syncthreads();
  if (rlane == 0 && ch < c) {
    float t = 0.f;
    for (int i = 0; i < 8; ++i) t += red[i][threadIdx.x & 31];
    part[(long long)blockIdx.y * c + ch] = t;
  }
}

// ---------------------------------------------------------------------------------------------
// host-side decomposition of a layer into phases
// ---------------------------------------------------------------------------------------------
static int validate(const KtConv1dDesc* d) {
  KT_REQUIRE(d != nullptr, "null descriptor");
  KT_REQUIRE(d->batch > 0 && d->nsub > 0 && d->t_in > 0 && d->t_out > 0, "bad sizes B=%d nsub=%d t_in=%d t_out=%d", d->batch, d->nsub, d->t_in, d->t_out);
  KT_REQUIRE(d->c_in > 0 && d->c_out > 0 && d->groups > 0 && d->c_in % d->groups == 0 && d->c_out % d->groups == 0, "bad channels/groups %d %d %d", d->c_in, d->c_out, d->groups);
  KT_REQUIRE(d->kernel > 0 && d->kernel <= kMaxTaps, "kernel size %d unsupported (max %d)", d->kernel, kMaxTaps);
  KT_REQUIRE(d->stride > 0 && d->dilation > 0 && d->upsample > 0, "bad stride/dilation/upsample");
  KT_REQUIRE(!(d->transposed && (d->groups != 1 || d->upsample != 1)), "transposed conv: groups/upsample unsupported");
  KT_REQUIRE(!(d->upsample > 1 && d->stride != 1), "upsampled conv must have stride 1");
  KT_REQUIRE((long long)d->batch * d->nsub <= 65535, "batch*nsub too large");
  return KT_OK;
}

static void finish_phase(Phase& ph) {
  ph.min_ioff = ph.tap_ioff[0];
  ph.max_ioff = ph.tap_ioff[0];
  for (int n = 1; n < ph.ntaps; ++n) {
    ph.min_ioff = std::min(ph.min_ioff, ph.tap_ioff[n]);
    ph.max_ioff = std::max(ph.max_ioff, ph.tap_ioff[n]);
  }
}

// forward of a conv / data-gradient of a transposed conv: one gather phase
//   out[to] = sum_j W_j in[(to*stride + j*dil - pad) / up]
static Phase gather_phase(int t_out, int kernel, int stride, int dil, int pad, int up) {
  Phase ph{};
  ph.M = t_out; ph.o_off = 0; ph.o_step = 1; ph.i_step = stride; ph.up = up; ph.accumulate = 0;
  ph.ntaps = kernel;
  for (int j = 0; j < kernel; ++j) { ph.tap_j[j] = j; ph.tap_ioff[j] = j * dil - pad; }
  finish_phase(ph);
  return ph;
}

// scatter semantics out[ti*stride + j*dil - pad] += W_j in[ti], rewritten as `stride` gather phases
// over the outputs to = r + stride*m  (forward of a transposed conv / data-gradient of a conv)
static std::vector<Phase> scatter_phases(int t_out, int kernel, int stride, int dil, int pad) {
  std::vector<Phase> v;
  for (int r = 0; r < stride && r < t_out; ++r) {
    Phase ph{};
    ph.M = (t_out - r + stride - 1) / stride; ph.o_off = r; ph.o_step = stride; ph.i_step = 1; ph.up = 1; ph.accumulate = 0;
    ph.ntaps = 0;
    for (int j = 0; j < kernel; ++j) {
      const int num = r + pad - j * dil;  // ti*stride = to + pad - j*dil
      if (((num % stride) + stride) % stride != 0) continue;
      ph.tap_j[ph.ntaps] = j;
      ph.tap_ioff[ph.ntaps] = fdiv(num, stride);
      ++ph.ntaps;
    }
    if (ph.ntaps == 0) {  // no tap reaches this output phase: still must write bias / zeros
      ph.ntaps = 1; ph.tap_j[0] = 0; ph.tap_ioff[0] = -(1 << 28);
    }
    finish_phase(ph);
    v.push_back(ph);
  }
  return v;
}

static Side make_side(const float* p, const float* aux, int act, float slope, bool derivative) {
  Side s{p, aux, SIDE_PLAIN, slope};
  if (act == KT_ACT_LRELU) s.mode = derivative ? SIDE_DLRELU : SIDE_LRELU;
  else if (act == KT_ACT_TANH) s.mode = derivative ? SIDE_DTANH : SIDE_PLAIN;
  if (s.mode < SIDE_DLRELU) s.aux = nullptr;
  return s;
}

// Phases of a layer: dir 0 = forward, dir 1 = data gradient (roles of t_in / t_out swapped by the caller).
std::vector<Phase> conv_phases(const KtConv1dDesc* d, int dir) {
  std::vector<Phase> v;
  if (dir == 0) {
    if (!d->transposed) v.push_back(gather_phase(d->t_out, d->kernel, d->stride, d->dilation, d->pad_left, d->upsample));
    else v = scatter_phases(d->t_out, d->kernel, d->stride, d->dilation, d->pad_left);
    return v;
  }
  if (d->transposed) {
    // dx[ti] = sum_j W_j^T dy[ti*stride + j*dil - pad]
    v.push_back(gather_phase(d->t_in, d->kernel, d->stride, d->dilation, d->pad_left, 1));
  } else if (d->upsample == 1) {
    // dx[ti] = sum_j W_j^T dy[(ti + pad - j*dil) / stride]
    v = scatter_phases(d->t_in, d->kernel, d->stride, d->dilation, d->pad_left);
  } else {
    // nearest-upsampled input: dx[ti] = sum_{r<u} sum_j W_j^T dy[ti*u + r + pad - j*dil]
    const int u = d->upsample;
    for (int r = 0; r < u; ++r) {
      Phase ph{};
      ph.M = d->t_in; ph.o_off = 0; ph.o_step = 1; ph.i_step = u; ph.up = 1; ph.accumulate = r > 0;
      ph.ntaps = d->kernel;
      for (int j = 0; j < d->kernel; ++j) { ph.tap_j[j] = j; ph.tap_ioff[j] = r + d->pad_left - j * d->dilation; }
      finish_phase(ph);
      v.push_back(ph);
    }
  }
  return v;
}

bool thin_cin1_ok(const KtConv1dDesc* d);                                                                       // thin.cu
int thin_cin1_fwd(const KtConv1dDesc*, const float*, const float*, const float*, float*, cudaStream_t);
int thin_cin1_wgrad(const KtConv1dDesc*, const float*, const float*, const float*, float*, float*, cudaStream_t);

int conv1d_fwd_ffma(const KtConv1dDesc* d, const float* x, const float* w_fwd, const float* bias,
                    const float* resid, float* y, cudaStream_t st) {
  if (thin_cin1_ok(d) && resid == nullptr) return thin_cin1_fwd(d, x, w_fwd, bias, y, st);   // waveform-input layers
  CoreParams p{};
  p.in = make_side(x, nullptr, d->act_in, d->act_in_slope, false);
  p.w = w_fwd; p.bias = bias; p.resid = resid; p.mask = Side{nullptr, nullptr, 0, 0.f}; p.out = y;
  p.batch = d->batch * d->nsub; p.nsub = d->nsub; p.t_in = d->t_in; p.t_out = d->t_out;
  p.c_in = d->c_in; p.c_out = d->c_out; p.groups = d->groups; p.cin_g = d->c_in / d->groups; p.cout_g = d->c_out / d->groups;
  p.out_act = d->act_out; p.out_slope = d->act_out_slope;
  for (const Phase& ph : conv_phases(d, 0)) {
    p.ph = ph;
    int rc = run_core(p, st);
    if (rc) return rc;
  }
  return KT_OK;
}

int conv1d_bwd_data_ffma(const KtConv1dDesc* d, const float* dy, const float* y, const float* w_bwd,
                         const float* x, float* dx, cudaStream_t st) {
  CoreParams p{};
  KT_REQUIRE(d->act_out == KT_ACT_NONE || y != nullptr, "bwd_data: y required when act_out != NONE");
  KT_REQUIRE(d->act_in == KT_ACT_NONE || x != nullptr, "bwd_data: x required when act_in != NONE");
  p.in = make_side(dy, y, d->act_out, d->act_out_slope, true);
  p.w = w_bwd; p.bias = nullptr; p.resid = nullptr; p.out = dx;
  p.mask = d->act_in == KT_ACT_LRELU ? Side{x, nullptr, SIDE_DLRELU, d->act_in_slope} : Side{nullptr, nullptr, 0, 0.f};
  // roles swap: "in" = dy (c_out channels, t_out rows), "out" = dx (c_in channels, t_in rows)
  p.batch = d->batch * d->nsub; p.nsub = d->nsub; p.t_in = d->t_out; p.t_out = d->t_in;
  p.c_in = d->c_out; p.c_out = d->c_in; p.groups = d->groups; p.cin_g = d->c_out / d->groups; p.cout_g = d->c_in / d->groups;
  p.out_act = KT_ACT_NONE; p.out_slope = 0.f;
  // (a fused act_in' mask is multiplicative, so applying it in every accumulating phase is exact)
  for (const Phase& ph : conv_phases(d, 1)) {
    p.ph = ph;
    int rc = run_core(p, st);
    if (rc) return rc;
  }
  return KT_OK;
}

int colsum_bias(const Side& s, long long rows, int c, float* out, cudaStream_t st);

int conv1d_bwd_weight_ffma(const KtConv1dDesc* d, const float* x, const float* dy, const float* y,
                           float* dw, float* dbias, cudaStream_t st) {
  KT_REQUIRE(d->act_out == KT_ACT_NONE || y != nullptr, "bwd_weight: y required when act_out != NONE");
  if (thin_cin1_ok(d)) return thin_cin1_wgrad(d, x, dy, y, dw, dbias, st);
  const size_t wn = (size_t)d->kernel * (d->c_in / d->groups) * d->c_out;
  KT_CHECK_CUDA(cudaMemsetAsync(dw, 0, wn * sizeof(float), st));
  const Side sx = make_side(x, nullptr, d->act_in, d->act_in_slope, false);
  const Side sdy = make_side(dy, y, d->act_out, d->act_out_slope, true);
  WgradParams p{};
  p.g = dw; p.g_size = (long long)wn; p.batch = d->batch * d->nsub; p.nsub = d->nsub; p.groups = d->groups;
  if (!d->transposed) {
    // dW[j][ci][co] = sum x[(to*stride + j*dil - pad)/up][ci] * dpre[to][co]
    p.a = sx; p.b = sdy;
    p.t_a = d->t_in; p.t_b = d->t_out; p.ca_total = d->c_in; p.cb_total = d->c_out;
    p.ca_g = d->c_in / d->groups; p.cb_g = d->c_out / d->groups;
    p.ph = gather_phase(d->t_out, d->kernel, d->stride, d->dilation, d->pad_left, d->upsample);
  } else {
    // dW[ci][co][j] = sum_ti x[ti][ci] * dpre[ti*stride + j*dil - pad][co]: the shifted (gathered)
    // side is dpre, so A = dpre (rows co), B = x (cols ci) and dw comes out in the [k][Cout][Cin]
    // (= w_bwd) layout for transposed convs, as documented in kantts_b200.h.
    p.a = sdy; p.b = sx;
    p.t_a = d->t_out; p.t_b = d->t_in; p.ca_total = d->c_out; p.cb_total = d->c_in;
    p.ca_g = d->c_out; p.cb_g = d->c_in;
    p.ph = gather_phase(d->t_in, d->kernel, d->stride, d->dilation, d->pad_left, 1);
  }
  int rc = run_wgrad(p, st);
  if (rc) return rc;
  if (dbias) return colsum_bias(sdy, (long long)d->batch * d->nsub * d->t_out, d->c_out, dbias, st);
  return KT_OK;
}

int colsum_bias(const Side& s, long long rows, int c, float* out, cudaStream_t st) {
  const int ny = (int)std::min<long long>(std::max<long long>(1, rows / 256), 512);
  float* part = nullptr;
  int rc = scratch_alloc(&part, (long long)ny * c, st);
  if (rc) return rc;
  colsum_kernel<<<dim3(ceil_div(c, 32), ny), 256, 0, st>>>(s, rows, c, part);
  KT_CHECK_CUDA(cudaGetLastError());
  rc = split_sum(part, c, ny, c, out, false, st);
  if (rc) return rc;
  return scratch_free(part, st);
}

int validate_conv(const KtConv1dDesc* d) { return validate(d); }

}  // namespace kt
