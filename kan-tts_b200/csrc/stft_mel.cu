// Fused STFT -> |.| -> mel projection -> log-normalise kernel (+ backward), one CTA per frame.
//
// Replaces the ~35-launch chain torch.stft (cuFFT R2C) -> pow/add/clamp/sqrt -> matmul(cuBLAS) ->
// clamp/log10/scale/clamp/transpose of kantts/utils/audio_torch.py:155-186 (MelSpectrogram.forward)
// and audio_torch.py:8-31 (stft magnitude for the multi-resolution STFT loss).
//
// Per frame: framing with centre padding (zeros for the mel variant, reflect for `stft()`), window,
// an in-shared-memory radix-2 FFT of the n_fft real samples, power -> sqrt(clamp) amplitude,
// the (n_bins x n_mels) projection and the dB normalisation -- nothing but the wav samples, the
// optional saved spectrum and the 80 mel values ever touch HBM.
// The backward runs the same FFT with conjugated twiddles on Z_k = d re_k + i d im_k and
// overlap-adds win[n] * Re(ifft) into d wav.
//
// An n_fft that is not a power of two (the sub-band STFT loss: 171, 384, 683) takes separate kernel instances
// (kAnyN) that compute the n-point DFT by Bluestein's algorithm: with the chirp c_m = exp(sign * i pi m^2 / n),
//   X_k = c_k * sum_j (x_j c_j) conj(c_{k-j}),
// a circular convolution of size M = 2^logm >= 2n - 1 done with three radix-2 FFTs of M points (the input, the
// chirp filter -- recomputed per CTA, so the route keeps no state between calls -- and the inverse).  The
// chirp's phase m^2 / n is reduced mod 2 in integers before sincospif, so large m keep full precision.
#include <algorithm>

#include "common.cuh"
#include "fft.cuh"

namespace kt {

struct MelParams {
  int batch, t, n_fft, hop, n_mels, frames, logn, pad_mode;   // logn: log2 of the radix-2 FFT length (n_fft, or M)
  float eps, ref_db, min_db, norm_scale, norm_shift, norm_lo, norm_hi;
};

__device__ __forceinline__ int src_index(int pos, int t, int pad_mode) {
  // pos relative to the un-padded signal; returns -1 for a zero sample
  if (pos >= 0 && pos < t) return pos;
  if (pad_mode == 0) return -1;
  if (pos < 0) pos = -pos;                 // reflect (no edge repeat), as F.pad(mode="reflect")
  if (pos >= t) pos = 2 * (t - 1) - pos;
  return (pos >= 0 && pos < t) ? pos : -1;
}

// exp(sign * i * pi * m^2 / n) for 0 <= m < n
__device__ __forceinline__ float2 chirp(int m, int n, float sign) {
  const int r = (int)(((long long)m * m) % (2 * n));
  float sn, cs;
  sincospif(sign * (float)r / (float)n, &sn, &cs);
  return make_float2(cs, sn);
}

__device__ __forceinline__ float2 cmul(float2 a, float2 b) {
  return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}

// fft_inplace (fft.cuh) of two M-point buffers at once: one barrier per stage for both
__device__ void fft2_inplace(float2* a, float2* b, int logm, float sign) {
  const int m = 1 << logm;
  for (int st = 1; st <= logm; ++st) {
    const int half = 1 << (st - 1);
    __syncthreads();
    for (int idx = threadIdx.x; idx < m; idx += blockDim.x) {
      float2* s = idx < m / 2 ? a : b;
      const int id = idx & (m / 2 - 1);
      const int k = id & (half - 1);
      const int i0 = ((id >> (st - 1)) << st) + k;
      const int i1 = i0 + half;
      float sn, cs;
      sincospif(sign * (float)k / (float)half, &sn, &cs);
      const float2 u = s[i0], v = s[i1];
      const float2 t = make_float2(v.x * cs - v.y * sn, v.x * sn + v.y * cs);
      s[i0] = make_float2(u.x + t.x, u.y + t.y);
      s[i1] = make_float2(u.x - t.x, u.y - t.y);
    }
  }
  __syncthreads();
}

// Bluestein's n-point DFT (see the file comment) over two M-point buffers, M = 2^logm >= 2n - 1.  On entry
// a[bitrev(j)] = x_j c_j for j < n and 0 at every other position; b is scratch.  On return
// a[k] = sum_j x_j exp(sign * 2 pi i j k / n) for k < n.
__device__ void bluestein(float2* a, float2* b, int n, int logm, float sign) {
  const int m = 1 << logm;
  for (int i = threadIdx.x; i < m; i += blockDim.x) {   // the filter conj(c_i), c_{m-i} = c_i for the negative lags
    const int l = min(i, m - i);
    b[bitrev(i, logm)] = l < n ? chirp(l, n, -sign) : make_float2(0.f, 0.f);
  }
  fft2_inplace(a, b, logm, -1.f);
  const float inv = 1.f / (float)m;
  for (int i = threadIdx.x; i < m; i += blockDim.x) {
    const float2 z = cmul(a[i], b[i]);
    b[i] = make_float2(z.x * inv, z.y * inv);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < m; i += blockDim.x) a[bitrev(i, logm)] = b[i];
  fft_inplace(a, m, logm, +1.f);
  for (int k = threadIdx.x; k < n; k += blockDim.x) a[k] = cmul(a[k], chirp(k, n, sign));
  __syncthreads();
}

// kAnyN: any n_fft by Bluestein (s and a second buffer of M points each); otherwise n_fft is a power of two
template <bool kAnyN>
__global__ void __launch_bounds__(256) stft_mel_fwd_kernel(MelParams p, const float* __restrict__ wav,
                                                           const float* __restrict__ window,
                                                           const float* __restrict__ melmat,
                                                           float* __restrict__ mel, float* __restrict__ amp_out,
                                                           float* __restrict__ spec) {
  extern __shared__ __align__(16) float smem_f[];
  float2* s = reinterpret_cast<float2*>(smem_f);          // [n_fft] | kAnyN: [M], then [M] scratch
  float* amp = smem_f + (kAnyN ? 4 << p.logn : 2 * p.n_fft);   // [n_fft/2 + 1]
  const int f = blockIdx.x % p.frames, b = blockIdx.x / p.frames;
  const int n = p.n_fft, nb = n / 2 + 1;
  const float* w = wav + (long long)b * p.t;
  const int start = f * p.hop - n / 2;
  if constexpr (kAnyN) {
    for (int i = threadIdx.x; i < (1 << p.logn); i += blockDim.x) {
      float2 v = make_float2(0.f, 0.f);
      if (i < n) {
        const int si = src_index(start + i, p.t, p.pad_mode);
        const float x = si >= 0 ? __ldg(w + si) * __ldg(window + i) : 0.f;
        const float2 c = chirp(i, n, -1.f);
        v = make_float2(x * c.x, x * c.y);
      }
      s[bitrev(i, p.logn)] = v;
    }
    bluestein(s, s + (1 << p.logn), n, p.logn, -1.f);
  } else {
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const int si = src_index(start + i, p.t, p.pad_mode);
      const float v = si >= 0 ? __ldg(w + si) * __ldg(window + i) : 0.f;
      s[bitrev(i, p.logn)] = make_float2(v, 0.f);
    }
    fft_inplace(s, n, p.logn, -1.f);
  }
  const long long fb = (long long)b * p.frames + f;
  for (int k = threadIdx.x; k < nb; k += blockDim.x) {
    const float2 z = s[k];
    const float a = sqrtf(fmaxf(z.x * z.x + z.y * z.y, p.eps));
    amp[k] = a;
    if (amp_out) amp_out[fb * nb + k] = a;
    if (spec) reinterpret_cast<float2*>(spec)[fb * nb + k] = z;
  }
  __syncthreads();
  if (mel) {
    for (int m = threadIdx.x; m < p.n_mels; m += blockDim.x) {
      float acc = 0.f;
      for (int k = 0; k < nb; ++k) acc = fmaf(amp[k], __ldg(melmat + (long long)k * p.n_mels + m), acc);
      acc = fmaxf(acc, p.eps);
      const float db = 20.f * log10f(fmaxf(acc, 1e-5f)) - p.ref_db;
      // spectral_normalize_torch (audio_torch.py:42-63) / dsp._normalize (dsp.py:66-74)
      float v = p.norm_scale * ((db - p.min_db) / (-p.min_db)) - p.norm_shift;
      v = fminf(fmaxf(v, p.norm_lo), p.norm_hi);
      mel[((long long)b * p.n_mels + m) * p.frames + f] = v;
    }
  }
}

template <bool kAnyN>
__global__ void __launch_bounds__(256) stft_mel_bwd_kernel(MelParams p, const float* __restrict__ dmel,
                                                           const float* __restrict__ damp_in,
                                                           const float* __restrict__ spec,
                                                           const float* __restrict__ window,
                                                           const float* __restrict__ melmat,
                                                           float* __restrict__ frame_grad) {
  extern __shared__ __align__(16) float smem_f[];
  float2* s = reinterpret_cast<float2*>(smem_f);          // [n_fft] | kAnyN: [M], then [M] scratch
  float* amp = smem_f + (kAnyN ? 4 << p.logn : 2 * p.n_fft);   // [nb]
  float* dm = amp + (p.n_fft / 2 + 1);                    // [n_mels]
  const int f = blockIdx.x % p.frames, b = blockIdx.x / p.frames;
  const int n = p.n_fft, nb = n / 2 + 1;
  const long long fb = (long long)b * p.frames + f;
  const float2* z = reinterpret_cast<const float2*>(spec) + fb * nb;
  for (int k = threadIdx.x; k < nb; k += blockDim.x) {
    const float2 v = __ldg(z + k);
    amp[k] = sqrtf(fmaxf(v.x * v.x + v.y * v.y, p.eps));
  }
  __syncthreads();
  if (dmel) {
    for (int m = threadIdx.x; m < p.n_mels; m += blockDim.x) {
      float acc = 0.f;
      for (int k = 0; k < nb; ++k) acc = fmaf(amp[k], __ldg(melmat + (long long)k * p.n_mels + m), acc);
      float gr = __ldg(dmel + ((long long)b * p.n_mels + m) * p.frames + f);
      const float melc = fmaxf(acc, p.eps);
      const float x = fmaxf(melc, 1e-5f);
      const float db = 20.f * log10f(x) - p.ref_db;
      const float v = p.norm_scale * ((db - p.min_db) / (-p.min_db)) - p.norm_shift;
      if (!(v >= p.norm_lo && v <= p.norm_hi) || melc < 1e-5f || acc < p.eps) gr = 0.f;
      dm[m] = gr * (p.norm_scale / (-p.min_db) * 20.f * 0.4342944819032518f) / x;  // d/dx [scale/(-min) * 20 log10 x]
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < (kAnyN ? 1 << p.logn : n); i += blockDim.x) {
    // Z_k = dre_k + i dim_k for k <= n/2, 0 above; store bit-reversed for the in-place FFT (kAnyN: times the chirp)
    float2 zk = make_float2(0.f, 0.f);
    if (i < nb) {
      float da = damp_in ? __ldg(damp_in + fb * nb + i) : 0.f;
      if (dmel) {
        const float* mr = melmat + (long long)i * p.n_mels;
        float acc = 0.f;
        for (int m = 0; m < p.n_mels; ++m) acc = fmaf(__ldg(mr + m), dm[m], acc);
        da += acc;
      }
      const float2 v = __ldg(z + i);
      const float pw = v.x * v.x + v.y * v.y;
      const float sc = pw >= p.eps ? da / amp[i] : 0.f;    // d amp / d re = re / amp  (clamp passes grad iff pw >= eps)
      zk = make_float2(v.x * sc, v.y * sc);
      if constexpr (kAnyN) zk = cmul(zk, chirp(i, n, +1.f));
    }
    s[bitrev(i, p.logn)] = zk;
  }
  if constexpr (kAnyN) bluestein(s, s + (1 << p.logn), n, p.logn, +1.f);
  else fft_inplace(s, n, p.logn, +1.f);
  // windowed frame gradient; ola_gather_kernel overlap-adds the frames (a fixed summation order, unlike float atomics)
  float* fg = frame_grad + fb * n;
  for (int i = threadIdx.x; i < n; i += blockDim.x) fg[i] = s[i].x * __ldg(window + i);
}

// dwav[b][t] = sum over the padded positions q that src_index maps to t (q = t, its left and right reflections), and over
// the frames f covering q (ascending), of frame_grad[b][f][q - f * hop + n / 2]
__global__ void ola_gather_kernel(const MelParams p, const float* __restrict__ frame_grad, float* __restrict__ dwav) {
  const int n = p.n_fft, half = n / 2;
  const long long total = (long long)p.batch * p.t;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int b = (int)(idx / p.t), t = (int)(idx - (long long)b * p.t);
    const int cand[3] = {t, -t, 2 * (p.t - 1) - t};
    float acc = 0.f;
    for (int c = 0; c < 3; ++c) {
      const int q = cand[c];
      if ((c == 1 && q == cand[0]) || (c == 2 && (q == cand[0] || q == cand[1]))) continue;
      if (src_index(q, p.t, p.pad_mode) != t) continue;
      // frames f with 0 <= q - f * hop + half < n
      const int f_lo = max(0, fdiv(q + half - n, p.hop) + 1), f_hi = min(p.frames - 1, fdiv(q + half, p.hop));
      for (int f = f_lo; f <= f_hi; ++f) acc += __ldg(frame_grad + ((long long)b * p.frames + f) * n + (q - f * p.hop + half));
    }
    dwav[idx] = acc;
  }
}

static bool any_n(int n_fft) { return (n_fft & (n_fft - 1)) != 0; }

// dynamic shared memory of a forward / backward CTA: the FFT buffer(s), the amplitudes and (backward) the mel gradient
static size_t stft_smem(const MelParams& p, int bwd) {
  const size_t fft = any_n(p.n_fft) ? 4 * ((size_t)1 << p.logn) : 2 * (size_t)p.n_fft;
  return (fft + p.n_fft / 2 + 1 + (bwd ? p.n_mels : 0)) * sizeof(float);
}

// largest stft_smem of the Bluestein instances: M = 8192 for n_fft < 4096, 256 mels
constexpr int kAnyNMaxSmem = (4 * 8192 + 2048 + 1 + 256) * 4;

static int fill(MelParams& p, const KtMelDesc* d) {
  KT_REQUIRE(d && d->batch > 0 && d->t > 0 && d->hop > 0 && d->frames > 0, "stft_mel: bad descriptor");
  KT_REQUIRE(d->n_fft >= 16 && d->n_fft <= 4096, "stft_mel: n_fft=%d must be in [16, 4096]", d->n_fft);
  // a power of two runs the radix-2 FFT of n_fft points, any other n_fft Bluestein's of M >= 2 n_fft - 1 points
  const int len = any_n(d->n_fft) ? 2 * d->n_fft - 1 : d->n_fft;
  int logn = 0;
  while ((1 << logn) < len) ++logn;
  // center=True: n_fft / 2 samples of padding on either side, so an odd n_fft has (t - 1) / hop + 1 frames (torch.stft)
  const int frames = (d->t - d->n_fft % 2) / d->hop + 1;
  KT_REQUIRE(d->frames == frames, "stft_mel: frames=%d != (t - n_fft %% 2)/hop+1=%d (center=True)", d->frames, frames);
  KT_REQUIRE(d->pad_mode == 0 || d->t > d->n_fft / 2, "stft_mel: reflect padding needs t > n_fft/2");
  KT_REQUIRE(d->n_mels >= 0 && d->n_mels <= 256, "stft_mel: n_mels=%d unsupported", d->n_mels);
  p.batch = d->batch; p.t = d->t; p.n_fft = d->n_fft; p.hop = d->hop; p.n_mels = d->n_mels; p.frames = d->frames;
  p.logn = logn; p.pad_mode = d->pad_mode; p.eps = d->eps;
  p.ref_db = d->ref_db; p.min_db = d->min_db; p.norm_scale = d->norm_scale; p.norm_shift = d->norm_shift;
  p.norm_lo = d->norm_lo; p.norm_hi = d->norm_hi;
  KT_REQUIRE(d->n_mels == 0 || d->min_db < 0.f, "stft_mel: min_db must be negative");
  return KT_OK;
}

extern "C" int kt_stft_mel_fwd(const KtMelDesc* d, const float* wav, const float* window, const float* melmat, float* mel,
                               float* amp, float* spec, void* stream) {
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  MelParams p;
  int rc = fill(p, d);
  if (rc) return rc;
  KT_REQUIRE(wav && window && (!mel || melmat), "stft_mel_fwd: null argument");
  const size_t smem = stft_smem(p, 0);
  if (any_n(p.n_fft)) {
    KT_CHECK_CUDA(allow_dyn_smem<stft_mel_fwd_kernel<true>>(kAnyNMaxSmem));
    stft_mel_fwd_kernel<true><<<p.batch * p.frames, 256, smem, st>>>(p, wav, window, melmat, mel, amp, spec);
  } else {
    KT_CHECK_CUDA(allow_dyn_smem<stft_mel_fwd_kernel<false>>(64 * 1024));
    stft_mel_fwd_kernel<false><<<p.batch * p.frames, 256, smem, st>>>(p, wav, window, melmat, mel, amp, spec);
  }
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

extern "C" int kt_stft_mel_bwd(const KtMelDesc* d, const float* dmel, const float* damp, const float* spec, const float* window,
                               const float* melmat, float* dwav, void* stream) {
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  MelParams p;
  int rc = fill(p, d);
  if (rc) return rc;
  KT_REQUIRE(spec && window && dwav && (dmel || damp) && (!dmel || melmat), "stft_mel_bwd: null argument");
  const size_t smem = stft_smem(p, 1);
  if (any_n(p.n_fft)) KT_CHECK_CUDA(allow_dyn_smem<stft_mel_bwd_kernel<true>>(kAnyNMaxSmem));
  else KT_CHECK_CUDA(allow_dyn_smem<stft_mel_bwd_kernel<false>>(64 * 1024));
  float* frame_grad = nullptr;
  rc = scratch_alloc(&frame_grad, (long long)p.batch * p.frames * p.n_fft, st);
  if (rc) return rc;
  if (any_n(p.n_fft))
    stft_mel_bwd_kernel<true><<<p.batch * p.frames, 256, smem, st>>>(p, dmel, damp, spec, window, melmat, frame_grad);
  else
    stft_mel_bwd_kernel<false><<<p.batch * p.frames, 256, smem, st>>>(p, dmel, damp, spec, window, melmat, frame_grad);
  KT_CHECK_CUDA(cudaGetLastError());
  const long long total = (long long)p.batch * p.t;
  ola_gather_kernel<<<(int)std::min<long long>((total + 255) / 256, 132LL * 16), 256, 0, st>>>(p, frame_grad, dwav);
  KT_CHECK_CUDA(cudaGetLastError());
  return scratch_free(frame_grad, st);
}

}  // namespace kt
