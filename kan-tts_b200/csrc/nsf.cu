// Seeded sine-plus-noise excitation of the neural source filter (SourceModule, kantts/models/hifigan/layers.py:229-290),
// computed on the GPU as a deterministic function of (seed, f0 / voiced flag of the slot, sample index): the definition is
// in include/kantts_b200.h (kt_nsf_excitation) and restated by oracle/nsf.py.  Every floating-point operation is an
// explicitly rounded intrinsic, so that no multiply-add is contracted and the kernel computes the oracle's function.
#include "common.cuh"
#include "philox.cuh"

namespace kt {

constexpr int kNsfFramesPerCta = 4;
constexpr int kNsfMaxChannels = 32;          // nb_harmonics + 1
constexpr double kTwoPi = 6.283185307179586;  // 2 * math.pi
constexpr double kPi = 3.141592653589793;

__device__ __forceinline__ double nsf_frac(double x) { return __dsub_rn(x, floor(x)); }

// c = f0 * (h + 1) / sr, in float64
__device__ __forceinline__ double nsf_rate(float f0, int h, double sr) {
  return __ddiv_rn(__dmul_rn((double)f0, (double)(h + 1)), sr);
}

// P_{j+1} = frac(P_j + hop * c_j)
__device__ __forceinline__ double nsf_step(double p, float f0, int h, int hop, double sr) {
  return nsf_frac(__dadd_rn(p, __dmul_rn((double)hop, nsf_rate(f0, h, sr))));
}

// Grid (frame blocks of kNsfFramesPerCta, batch).  The first nch threads run the phase scan of their harmonic from the
// carried state up to the CTA's frames (the one order-dependent sum, sequential by definition), then all threads write the
// CTA's rows.  The state itself is advanced by nsf_state_kernel afterwards.
__global__ void __launch_bounds__(256) nsf_excitation_kernel(const float* __restrict__ f0uv, int f0uv_pitch, int f0uv_first,
                                                             const KtNsfState s, float* __restrict__ e, int e_pitch, int e_first,
                                                             int frames, int hop, int nch, double sr, float alpha, float sigma,
                                                             float k_unvoiced) {
  __shared__ double s_p[kNsfFramesPerCta][kNsfMaxChannels], s_c[kNsfFramesPerCta][kNsfMaxChannels];
  __shared__ float s_uv[kNsfFramesPerCta], s_phi[kNsfMaxChannels];
  const int b = blockIdx.y, j0 = blockIdx.x * kNsfFramesPerCta;
  const int nf = min(kNsfFramesPerCta, frames - j0);
  const float* rows = f0uv + ((long long)b * f0uv_pitch + f0uv_first) * 2;
  const uint64_t seed = (uint64_t)s.seeds[b];
  const uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
  const int h = threadIdx.x;
  if (h < nch) {
    double p = s.phase[(long long)b * nch + h];
    for (int j = 0; j < j0; ++j) p = nsf_step(p, __ldg(rows + 2 * j), h, hop, sr);
    for (int jj = 0; jj < nf; ++jj) {
      const float f0 = __ldg(rows + 2 * (j0 + jj));
      s_p[jj][h] = p;
      s_c[jj][h] = nsf_rate(f0, h, sr);
      p = nsf_step(p, f0, h, hop, sr);
    }
    float phi = 0.f;                                  // phi_0 = 0; phi_h ~ U[-pi, pi) from counter (0, 0, h, 1)
    if (h > 0) {
      const Philox4 r = philox4x32_10(Philox4{{0u, 0u, (uint32_t)h, 1u}}, k0, k1);
      phi = (float)__dadd_rn(-kPi, __dmul_rn(kTwoPi, __dmul_rn((double)r.v[0], 0x1p-32)));
    }
    s_phi[h] = phi;
  }
  if (h < nf) s_uv[h] = __ldg(rows + 2 * (j0 + h) + 1);
  __syncthreads();

  const long long n0 = s.samples_done[b] + (long long)j0 * hop;      // sample index of the CTA's first row
  float* out = e + ((long long)b * e_pitch + e_first + (long long)j0 * hop) * nch;
  const int total = nf * hop * nch;
  for (int idx = threadIdx.x; idx < total; idx += blockDim.x) {
    const int row = idx / nch, ch = idx - row * nch;
    const int jj = row / hop, i = row - jj * hop;
    const uint64_t n = (uint64_t)(n0 + row);
    const Philox4 r = philox4x32_10(Philox4{{(uint32_t)n, (uint32_t)(n >> 32), (uint32_t)ch, 0u}}, k0, k1);
    const double u1 = __dmul_rn(__dadd_rn((double)r.v[0], 0.5), 0x1p-32);
    const double u2 = __dmul_rn(__dadd_rn((double)r.v[1], 0.5), 0x1p-32);
    const float z = (float)__dmul_rn(sqrt(__dmul_rn(-2.0, log(u1))), cos(__dmul_rn(kTwoPi, u2)));
    const float theta = (float)__dmul_rn(kTwoPi, nsf_frac(__dadd_rn(s_p[jj][ch], __dmul_rn((double)(i + 1), s_c[jj][ch]))));
    const float noise = __fmul_rn(sigma, z);
    const float voiced = __fadd_rn(__fmul_rn(alpha, sinf(__fadd_rn(theta, s_phi[ch]))), noise);
    const float unvoiced = __fmul_rn(k_unvoiced, noise);
    const float uv = s_uv[jj];
    out[idx] = __fadd_rn(__fmul_rn(voiced, uv), __fmul_rn(unvoiced, __fsub_rn(1.f, uv)));
  }
}

// After the chunk: phase[b][h] = P_{h, frames}, samples_done[b] += frames * hop.  One CTA per item, thread h per harmonic.
__global__ void nsf_state_kernel(const float* __restrict__ f0uv, int f0uv_pitch, int f0uv_first, const KtNsfState s, int frames,
                                 int hop, int nch, double sr) {
  const int b = blockIdx.x, h = threadIdx.x;
  const float* rows = f0uv + ((long long)b * f0uv_pitch + f0uv_first) * 2;
  if (h < nch) {
    double p = s.phase[(long long)b * nch + h];
    for (int j = 0; j < frames; ++j) p = nsf_step(p, __ldg(rows + 2 * j), h, hop, sr);
    s.phase[(long long)b * nch + h] = p;
  }
  if (h == 0) s.samples_done[b] += (long long)frames * hop;
}

extern "C" int kt_nsf_excitation(const float* f0uv, int32_t f0uv_pitch, int32_t f0uv_first, const KtNsfState* s, float* e,
                                 int32_t e_pitch, int32_t e_first, int32_t batch, int32_t frames, int32_t hop,
                                 int32_t nb_harmonics, int32_t sampling_rate, float alpha, float sigma, void* stream) {
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  KT_REQUIRE(s && s->seeds && s->phase && s->samples_done, "nsf_excitation: null state");
  KT_REQUIRE(f0uv && e && batch > 0 && batch <= 65535 && frames > 0 && hop > 0, "nsf_excitation: bad arguments");
  KT_REQUIRE(nb_harmonics >= 0 && nb_harmonics < kNsfMaxChannels, "nsf_excitation: nb_harmonics %d not in [0, %d)",
             nb_harmonics, kNsfMaxChannels);
  KT_REQUIRE(f0uv_first >= 0 && f0uv_first + frames <= f0uv_pitch, "nsf_excitation: the chunk does not fit its f0 / uv window");
  KT_REQUIRE(e_first >= 0 && (long long)e_first + (long long)frames * hop <= e_pitch,
             "nsf_excitation: the chunk does not fit its excitation window");
  KT_REQUIRE(sampling_rate > 0 && sigma > 0, "nsf_excitation: bad sampling rate / sigma");
  const int nch = nb_harmonics + 1;
  const float k_unvoiced = (float)((double)alpha / 3.0 / (double)sigma);
  const dim3 grid((unsigned)ceil_div(frames, kNsfFramesPerCta), (unsigned)batch);
  nsf_excitation_kernel<<<grid, 256, 0, st>>>(f0uv, f0uv_pitch, f0uv_first, *s, e, e_pitch, e_first, frames, hop, nch,
                                              (double)sampling_rate, alpha, sigma, k_unvoiced);
  KT_CHECK_CUDA(cudaGetLastError());
  nsf_state_kernel<<<batch, kNsfMaxChannels, 0, st>>>(f0uv, f0uv_pitch, f0uv_first, *s, frames, hop, nch,
                                                     (double)sampling_rate);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

}  // namespace kt
