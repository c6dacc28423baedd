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
#include <algorithm>

#include "common.cuh"

namespace kt {

__device__ __forceinline__ int bitrev(int x, int bits) { return (int)(__brev((unsigned)x) >> (32 - bits)); }

// in-place radix-2 DIT FFT over s[0..n) (already in bit-reversed order); sign = -1 forward, +1 inverse
__device__ void fft_inplace(float2* s, int n, int logn, float sign) {
  for (int st = 1; st <= logn; ++st) {
    const int half = 1 << (st - 1);
    __syncthreads();
    for (int idx = threadIdx.x; idx < n / 2; idx += blockDim.x) {
      const int k = idx & (half - 1);
      const int i0 = ((idx >> (st - 1)) << st) + k;
      const int i1 = i0 + half;
      float sn, cs;
      sincospif(sign * (float)k / (float)half, &sn, &cs);  // exp(sign * i * pi * k / half)
      const float2 a = s[i0], b = s[i1];
      const float2 t = make_float2(b.x * cs - b.y * sn, b.x * sn + b.y * cs);
      s[i0] = make_float2(a.x + t.x, a.y + t.y);
      s[i1] = make_float2(a.x - t.x, a.y - t.y);
    }
  }
  __syncthreads();
}

struct MelParams {
  int batch, t, n_fft, hop, n_mels, frames, logn, pad_mode;
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

__global__ void __launch_bounds__(256) stft_mel_fwd_kernel(MelParams p, const float* __restrict__ wav,
                                                           const float* __restrict__ window,
                                                           const float* __restrict__ melmat,
                                                           float* __restrict__ mel, float* __restrict__ amp_out,
                                                           float* __restrict__ spec) {
  extern __shared__ __align__(16) float smem_f[];
  float2* s = reinterpret_cast<float2*>(smem_f);          // [n_fft]
  float* amp = smem_f + 2 * p.n_fft;                      // [n_fft/2 + 1]
  const int f = blockIdx.x % p.frames, b = blockIdx.x / p.frames;
  const int n = p.n_fft, nb = n / 2 + 1;
  const float* w = wav + (long long)b * p.t;
  const int start = f * p.hop - n / 2;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int si = src_index(start + i, p.t, p.pad_mode);
    const float v = si >= 0 ? __ldg(w + si) * __ldg(window + i) : 0.f;
    s[bitrev(i, p.logn)] = make_float2(v, 0.f);
  }
  fft_inplace(s, n, p.logn, -1.f);
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

__global__ void __launch_bounds__(256) stft_mel_bwd_kernel(MelParams p, const float* __restrict__ dmel,
                                                           const float* __restrict__ damp_in,
                                                           const float* __restrict__ spec,
                                                           const float* __restrict__ window,
                                                           const float* __restrict__ melmat,
                                                           float* __restrict__ frame_grad) {
  extern __shared__ __align__(16) float smem_f[];
  float2* s = reinterpret_cast<float2*>(smem_f);          // [n_fft]
  float* amp = smem_f + 2 * p.n_fft;                      // [nb]
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
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    // Z_k = dre_k + i dim_k for k <= n/2, 0 above; store bit-reversed for the in-place FFT
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
    }
    s[bitrev(i, p.logn)] = zk;
  }
  fft_inplace(s, n, p.logn, +1.f);
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

static int fill(MelParams& p, const KtMelDesc* d) {
  KT_REQUIRE(d && d->batch > 0 && d->t > 0 && d->hop > 0 && d->frames > 0, "stft_mel: bad descriptor");
  int logn = 0;
  while ((1 << logn) < d->n_fft) ++logn;
  KT_REQUIRE((1 << logn) == d->n_fft && d->n_fft >= 64 && d->n_fft <= 4096, "stft_mel: n_fft=%d must be a power of two in [64, 4096]", d->n_fft);
  KT_REQUIRE(d->frames == d->t / d->hop + 1, "stft_mel: frames=%d != t/hop+1=%d (center=True)", d->frames, d->t / d->hop + 1);
  KT_REQUIRE(d->pad_mode == 0 || d->t > d->n_fft / 2, "stft_mel: reflect padding needs t > n_fft/2");
  KT_REQUIRE(d->n_mels >= 0 && d->n_mels <= 256, "stft_mel: n_mels=%d unsupported", d->n_mels);
  p.batch = d->batch; p.t = d->t; p.n_fft = d->n_fft; p.hop = d->hop; p.n_mels = d->n_mels; p.frames = d->frames;
  p.logn = logn; p.pad_mode = d->pad_mode; p.eps = d->eps;
  p.ref_db = d->ref_db; p.min_db = d->min_db; p.norm_scale = d->norm_scale; p.norm_shift = d->norm_shift;
  p.norm_lo = d->norm_lo; p.norm_hi = d->norm_hi;
  KT_REQUIRE(d->n_mels == 0 || d->min_db < 0.f, "stft_mel: min_db must be negative");
  return KT_OK;
}

int stft_mel_fwd(const KtMelDesc* d, const float* wav, const float* window, const float* melmat, float* mel,
                 float* amp, float* spec, cudaStream_t st) {
  MelParams p;
  int rc = fill(p, d);
  if (rc) return rc;
  KT_REQUIRE(wav && window && (!mel || melmat), "stft_mel_fwd: null argument");
  const size_t smem = (2 * (size_t)p.n_fft + p.n_fft / 2 + 1) * sizeof(float);
  static bool cfg = false;
  if (!cfg) { KT_CHECK_CUDA(cudaFuncSetAttribute(stft_mel_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024)); cfg = true; }
  stft_mel_fwd_kernel<<<p.batch * p.frames, 256, smem, st>>>(p, wav, window, melmat, mel, amp, spec);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

int stft_mel_bwd(const KtMelDesc* d, const float* dmel, const float* damp, const float* spec, const float* window,
                 const float* melmat, float* dwav, cudaStream_t st) {
  MelParams p;
  int rc = fill(p, d);
  if (rc) return rc;
  KT_REQUIRE(spec && window && dwav && (dmel || damp) && (!dmel || melmat), "stft_mel_bwd: null argument");
  const size_t smem = (2 * (size_t)p.n_fft + p.n_fft / 2 + 1 + p.n_mels) * sizeof(float);
  static bool cfg = false;
  if (!cfg) { KT_CHECK_CUDA(cudaFuncSetAttribute(stft_mel_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024)); cfg = true; }
  float* frame_grad = nullptr;
  rc = scratch_alloc(&frame_grad, (long long)p.batch * p.frames * p.n_fft, st);
  if (rc) return rc;
  stft_mel_bwd_kernel<<<p.batch * p.frames, 256, smem, st>>>(p, dmel, damp, spec, window, melmat, frame_grad);
  KT_CHECK_CUDA(cudaGetLastError());
  const long long total = (long long)p.batch * p.t;
  ola_gather_kernel<<<(int)std::min<long long>((total + 255) / 256, 132LL * 16), 256, 0, st>>>(p, frame_grad, dwav);
  KT_CHECK_CUDA(cudaGetLastError());
  return scratch_free(frame_grad, st);
}

}  // namespace kt
