// Speaker-embedding extractor of the SE SAM-BERT flow (kantts/preprocess/se_processor): the Kaldi fbank with per-utterance
// mean normalisation, and the pieces of the D-TDNN forward that the conv kernels do not cover -- the masked tap gather of
// the 2-D head, the masked per-channel affine (+ ReLU) that reads and writes rows at a channel pitch (the dense blocks'
// concatenation slab), the context-aware gating of PoolingBlock and the statistics pooling.  Inference only, exact fp32.
//
// Every kernel takes per-item lengths, and an item reads only its own valid rows: rows at or past its length are written as
// zeros (the zero padding every conv of a batch-1 run sees there), and every reduction runs over the item's valid rows in a
// fixed order.  So an item computes the same bits whatever else is in its batch.  No atomics.
#include <float.h>
#include <algorithm>
#include <math.h>

#include "common.cuh"
#include "fft.cuh"

namespace kt {

namespace {

constexpr int kFrameLen = 400;    // 25 ms at 16 kHz
constexpr int kFrameShift = 160;  // 10 ms
constexpr int kFftLog = 9;        // zero-padded to 512 points (round_to_power_of_two)
constexpr int kFftN = 1 << kFftLog;
constexpr int kFbankThreads = 256;
constexpr int kRowThreads = 128;

__host__ __device__ inline int fbank_frames(int n) { return n >= kFrameLen ? 1 + (n - kFrameLen) / kFrameShift : 0; }

__device__ __forceinline__ float block_sum_256(float v, float* red) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.f;
  for (int w = 0; w < kFbankThreads / 32; ++w) s += red[w];
  return s;
}

__device__ __forceinline__ float kaldi_mel(float hz) { return 1127.f * logf(1.f + hz / 700.f); }

// One CTA per (frame, utterance): the frame's 400 samples -> DC removal -> pre-emphasis (the first sample against itself)
// -> povey window -> 512-point power spectrum -> 80 Kaldi triangles over [20 Hz, Nyquist] on the mel scale
// 1127 ln(1 + f / 700) -> log(max(e, FLT_EPSILON)).  Frames past the utterance's last full frame are written as zeros.
__global__ void __launch_bounds__(kFbankThreads) kaldi_fbank_kernel(const float* __restrict__ wav,
                                                                    const int32_t* __restrict__ lengths,
                                                                    float* __restrict__ out, int n_samples, int frames,
                                                                    int n_mels, float sample_rate, float low_hz) {
  __shared__ float2 s[kFftN];
  __shared__ float fr[kFrameLen];
  __shared__ float pw[kFftN / 2 + 1];
  __shared__ float mel_of_bin[kFftN / 2];
  __shared__ float red[kFbankThreads / 32];
  const int f = blockIdx.x, b = blockIdx.y;
  float* o = out + ((long long)b * frames + f) * n_mels;
  if (f >= fbank_frames(__ldg(lengths + b))) {
    for (int m = threadIdx.x; m < n_mels; m += blockDim.x) o[m] = 0.f;
    return;
  }
  const float* x = wav + (long long)b * n_samples + (long long)f * kFrameShift;
  float part = 0.f;
  for (int i = threadIdx.x; i < kFrameLen; i += blockDim.x) {
    const float v = __ldg(x + i);
    fr[i] = v;
    part += v;
  }
  const float mean = block_sum_256(part, red) / (float)kFrameLen;
  for (int i = threadIdx.x; i < kFftN; i += blockDim.x) {
    float v = 0.f;
    if (i < kFrameLen) {
      const float cur = fr[i] - mean, prev = fr[i > 0 ? i - 1 : 0] - mean;
      const float hann = 0.5f - 0.5f * cospif(2.f * (float)i / (float)(kFrameLen - 1));
      v = (cur - 0.97f * prev) * powf(hann, 0.85f);
    }
    s[bitrev(i, kFftLog)] = make_float2(v, 0.f);
  }
  fft_inplace(s, kFftN, kFftLog, -1.f);
  const float bin_hz = sample_rate / (float)kFftN;
  for (int k = threadIdx.x; k <= kFftN / 2; k += blockDim.x) {
    pw[k] = s[k].x * s[k].x + s[k].y * s[k].y;
    if (k < kFftN / 2) mel_of_bin[k] = kaldi_mel(bin_hz * (float)k);
  }
  __syncthreads();
  const float mel_lo = kaldi_mel(low_hz), mel_hi = kaldi_mel(0.5f * sample_rate);
  const float delta = (mel_hi - mel_lo) / (float)(n_mels + 1);
  for (int m = threadIdx.x; m < n_mels; m += blockDim.x) {
    const float left = mel_lo + (float)m * delta, center = mel_lo + (float)(m + 1) * delta;
    const float right = mel_lo + (float)(m + 2) * delta;
    float e = 0.f;
    for (int k = 0; k < kFftN / 2; ++k) {   // the Nyquist bin has no triangle
      const float mk = mel_of_bin[k];
      const float w = fminf((mk - left) / (center - left), (right - mk) / (right - center));
      if (w > 0.f) e = fmaf(pw[k], w, e);
    }
    o[m] = logf(fmaxf(e, FLT_EPSILON));
  }
}

// One CTA per utterance: subtract each mel channel's mean over the utterance's frames, summed in frame order.
__global__ void __launch_bounds__(kRowThreads) fbank_cmn_kernel(const int32_t* __restrict__ lengths, float* __restrict__ out,
                                                                int frames, int n_mels) {
  const int b = blockIdx.x, nf = fbank_frames(__ldg(lengths + b));
  float* o = out + (long long)b * frames * n_mels;
  for (int m = threadIdx.x; m < n_mels; m += blockDim.x) {
    float acc = 0.f;
    for (int f = 0; f < nf; ++f) acc += o[(long long)f * n_mels + m];
    const float mean = acc / (float)nf;
    for (int f = 0; f < nf; ++f) o[(long long)f * n_mels + m] -= mean;
  }
}

// y[b][fo][t][k][c] (row pitch y_pitch) = x[b * sb + fi * sf + t * st + c] with fi = stride * fo + k - pad, zero outside
// [0, f_in) or at t >= lengths[b]
__global__ void tap_gather_kernel(const float* __restrict__ x, long long sb, long long sf, long long st,
                                  const int32_t* __restrict__ lengths, float* __restrict__ y, int y_pitch, int f_in, int t,
                                  int c, int f_out, int taps, int stride, int pad, long long total) {
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    long long r = idx / c;
    const int ch = (int)(idx - r * c);
    const int k = (int)(r % taps);
    r /= taps;
    const int tt = (int)(r % t);
    r /= t;
    const int fo = (int)(r % f_out);
    const int b = (int)(r / f_out);
    const int fi = stride * fo + k - pad;
    float v = 0.f;
    if (tt < __ldg(lengths + b) && fi >= 0 && fi < f_in) v = __ldg(x + b * sb + fi * sf + tt * st + ch);
    y[(((long long)b * f_out + fo) * t + tt) * y_pitch + (long long)k * c + ch] = v;
  }
}

// y[b][r][c] (row pitch y_pitch) = act(scale[c] * x[b][r][c] + shift[c]) (row pitch x_pitch) for r < lengths[b], else 0
__global__ void affine_rows_kernel(const float* __restrict__ x, int x_pitch, const float* __restrict__ scale,
                                   const float* __restrict__ shift, int relu, const int32_t* __restrict__ lengths,
                                   float* __restrict__ y, int y_pitch, int t, int c, long long total) {
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const long long row = idx / c;
    const int ch = (int)(idx - row * c);
    const int b = (int)(row / t), r = (int)(row - (long long)b * t);
    float v = 0.f;
    if (r < __ldg(lengths + b)) {
      v = __ldg(x + row * x_pitch + ch);
      if (scale) v = fmaf(__ldg(scale + ch), v, __ldg(shift + ch));
      if (relu) v = fmaxf(v, 0.f);
    }
    y[row * y_pitch + ch] = v;
  }
}

// One CTA per (segment, item): the sum and the max of each channel over the segment's valid rows, in row order, into
// stats[b][j][0 / 1][c]; the segment's rows at or past the item's length are zeroed in h.
__global__ void __launch_bounds__(kRowThreads) gate_stats_kernel(float* __restrict__ h, const int32_t* __restrict__ lengths,
                                                                 float* __restrict__ stats, int t, int c, int seg,
                                                                 int nseg) {
  const int j = blockIdx.x, b = blockIdx.y, len = __ldg(lengths + b);
  const int r0 = j * seg, r1 = min(r0 + seg, t), valid = min(r1, len);
  float* hb = h + (long long)b * t * c;
  float* sb = stats + ((long long)b * nseg + j) * 2 * c;
  for (int ch = threadIdx.x; ch < c; ch += blockDim.x) {
    float sum = 0.f, mx = -INFINITY;
    for (int r = r0; r < valid; ++r) {
      const float v = hb[(long long)r * c + ch];
      sum += v;
      mx = fmaxf(mx, v);
    }
    for (int r = max(r0, valid); r < r1; ++r) hb[(long long)r * c + ch] = 0.f;
    sb[ch] = sum;
    sb[c + ch] = mx;
  }
}

// One CTA per (segment, item): the gate of PoolingBlock for the segment,
//   s = sigmoid(W2 relu(W1 (mean_valid(h) + segmax(h)) + b1) + b2),
// then out[b][r][o] (row pitch out_pitch) = y[b][r][o] * s[o] over the segment's rows, 0 at r >= lengths[b].
__global__ void __launch_bounds__(kRowThreads) gate_apply_kernel(
    const float* __restrict__ y, const float* __restrict__ stats, const float* __restrict__ w1, const float* __restrict__ b1,
    const float* __restrict__ w2, const float* __restrict__ b2, const int32_t* __restrict__ lengths, float* __restrict__ out,
    int out_pitch, int t, int c, int c_mid, int c_out, int seg, int nseg) {
  extern __shared__ float sm[];
  float* v = sm;              // [c]
  float* z = v + c;           // [c_mid]
  float* s = z + c_mid;       // [c_out]
  const int j = blockIdx.x, b = blockIdx.y, len = __ldg(lengths + b);
  const int nseg_b = (len + seg - 1) / seg;
  const int r0 = j * seg, r1 = min(r0 + seg, t);
  if (j < nseg_b) {
    const float* st = stats + (long long)b * nseg * 2 * c;
    for (int ch = threadIdx.x; ch < c; ch += blockDim.x) {
      float acc = 0.f;
      for (int jj = 0; jj < nseg_b; ++jj) acc += __ldg(st + (long long)jj * 2 * c + ch);
      v[ch] = acc / (float)len + __ldg(st + ((long long)j * 2 + 1) * c + ch);
    }
    __syncthreads();
    for (int k = threadIdx.x; k < c_mid; k += blockDim.x) {
      float acc = __ldg(b1 + k);
      for (int ch = 0; ch < c; ++ch) acc = fmaf(__ldg(w1 + (long long)k * c + ch), v[ch], acc);
      z[k] = fmaxf(acc, 0.f);
    }
    __syncthreads();
    for (int o = threadIdx.x; o < c_out; o += blockDim.x) {
      float acc = __ldg(b2 + o);
      for (int k = 0; k < c_mid; ++k) acc = fmaf(__ldg(w2 + (long long)o * c_mid + k), z[k], acc);
      s[o] = 1.f / (1.f + expf(-acc));
    }
    __syncthreads();
  }
  for (int e = threadIdx.x; e < (r1 - r0) * c_out; e += blockDim.x) {
    const int r = r0 + e / c_out, o = e % c_out;
    const long long row = (long long)b * t + r;
    out[row * out_pitch + o] = r < len ? __ldg(y + row * c_out + o) * s[o] : 0.f;
  }
}

// out[b] = [mean_c, std_c] over the item's valid rows (std unbiased, as torch.std), two passes in row order
__global__ void __launch_bounds__(kRowThreads) stats_pool_kernel(const float* __restrict__ x, const int32_t* __restrict__ lengths,
                                                                 float* __restrict__ out, int t, int c) {
  const int b = blockIdx.y, ch = blockIdx.x * blockDim.x + threadIdx.x, n = __ldg(lengths + b);
  if (ch >= c) return;
  const float* xb = x + (long long)b * t * c + ch;
  float acc = 0.f;
  for (int r = 0; r < n; ++r) acc += __ldg(xb + (long long)r * c);
  const float mean = acc / (float)n;
  float sq = 0.f;
  for (int r = 0; r < n; ++r) {
    const float d = __ldg(xb + (long long)r * c) - mean;
    sq = fmaf(d, d, sq);
  }
  out[(long long)b * 2 * c + ch] = mean;
  out[(long long)b * 2 * c + c + ch] = sqrtf(sq / (float)(n - 1));
}

int grid_for(long long total) { return (int)std::min<long long>((total + 255) / 256, 132LL * 32); }

}  // namespace

extern "C" int kt_kaldi_fbank(const float* wav, const int32_t* lengths, float* out, int32_t batch, int32_t n_samples,
                              int32_t frames, int32_t n_mels, float sample_rate, float low_hz, void* stream) {
  KT_REQUIRE(wav && lengths && out, "kaldi_fbank: null argument");
  KT_REQUIRE(batch > 0 && batch <= 65535 && n_samples >= kFrameLen && frames == fbank_frames(n_samples),
             "kaldi_fbank: bad shape (batch %d, n_samples %d, frames %d; expected %d frames)", batch, n_samples, frames,
             fbank_frames(n_samples));
  KT_REQUIRE(n_mels > 0 && n_mels <= 256 && sample_rate > 0.f && low_hz >= 0.f && low_hz < 0.5f * sample_rate,
             "kaldi_fbank: bad mel bank (n_mels %d, sample rate %g, low %g Hz)", n_mels, sample_rate, low_hz);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  kaldi_fbank_kernel<<<dim3(frames, batch), kFbankThreads, 0, st>>>(wav, lengths, out, n_samples, frames, n_mels,
                                                                    sample_rate, low_hz);
  KT_CHECK_CUDA(cudaGetLastError());
  fbank_cmn_kernel<<<batch, kRowThreads, 0, st>>>(lengths, out, frames, n_mels);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

extern "C" int kt_se_tap_gather(const float* x, int64_t sb, int64_t sf, int64_t st, const int32_t* lengths, float* y,
                                int32_t y_pitch, int32_t batch, int32_t f_in, int32_t t, int32_t c, int32_t f_out,
                                int32_t taps, int32_t stride, int32_t pad, void* stream) {
  KT_REQUIRE(x && lengths && y, "se_tap_gather: null argument");
  KT_REQUIRE(batch > 0 && f_in > 0 && t > 0 && c > 0 && f_out > 0 && taps > 0 && stride > 0 && pad >= 0 &&
             y_pitch >= taps * c, "se_tap_gather: bad shape");
  const long long total = (long long)batch * f_out * t * taps * c;
  tap_gather_kernel<<<grid_for(total), 256, 0, static_cast<cudaStream_t>(stream)>>>(x, sb, sf, st, lengths, y, y_pitch, f_in,
                                                                                     t, c, f_out, taps, stride, pad, total);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

extern "C" int kt_se_affine_rows(const float* x, int32_t x_pitch, const float* scale, const float* shift, int32_t relu,
                                 const int32_t* lengths, float* y, int32_t y_pitch, int32_t batch, int32_t t, int32_t c,
                                 void* stream) {
  KT_REQUIRE(x && lengths && y && (!scale) == (!shift), "se_affine_rows: null argument");
  KT_REQUIRE(batch > 0 && t > 0 && c > 0 && x_pitch >= c && y_pitch >= c, "se_affine_rows: bad shape");
  const long long total = (long long)batch * t * c;
  affine_rows_kernel<<<grid_for(total), 256, 0, static_cast<cudaStream_t>(stream)>>>(x, x_pitch, scale, shift, relu, lengths,
                                                                                      y, y_pitch, t, c, total);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

extern "C" int kt_se_gate_stats(float* h, const int32_t* lengths, float* stats, int32_t batch, int32_t t, int32_t c,
                                int32_t seg, void* stream) {
  KT_REQUIRE(h && lengths && stats, "se_gate_stats: null argument");
  KT_REQUIRE(batch > 0 && batch <= 65535 && t > 0 && c > 0 && seg > 0, "se_gate_stats: bad shape");
  const int nseg = ceil_div(t, seg);
  gate_stats_kernel<<<dim3(nseg, batch), kRowThreads, 0, static_cast<cudaStream_t>(stream)>>>(h, lengths, stats, t, c, seg,
                                                                                              nseg);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

extern "C" int kt_se_gate_apply(const float* y, const float* stats, const float* w1, const float* b1, const float* w2,
                                const float* b2, const int32_t* lengths, float* out, int32_t out_pitch, int32_t batch,
                                int32_t t, int32_t c, int32_t c_mid, int32_t c_out, int32_t seg, void* stream) {
  KT_REQUIRE(y && stats && w1 && b1 && w2 && b2 && lengths && out, "se_gate_apply: null argument");
  KT_REQUIRE(batch > 0 && batch <= 65535 && t > 0 && c > 0 && c_mid > 0 && c_out > 0 && seg > 0 && out_pitch >= c_out,
             "se_gate_apply: bad shape");
  const size_t smem = (size_t)(c + c_mid + c_out) * sizeof(float);
  KT_REQUIRE(smem <= 48 * 1024, "se_gate_apply: %d + %d + %d channels exceed shared memory", c, c_mid, c_out);
  const int nseg = ceil_div(t, seg);
  gate_apply_kernel<<<dim3(nseg, batch), kRowThreads, smem, static_cast<cudaStream_t>(stream)>>>(
      y, stats, w1, b1, w2, b2, lengths, out, out_pitch, t, c, c_mid, c_out, seg, nseg);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

extern "C" int kt_se_stats_pool(const float* x, const int32_t* lengths, float* out, int32_t batch, int32_t t, int32_t c,
                                void* stream) {
  KT_REQUIRE(x && lengths && out, "se_stats_pool: null argument");
  KT_REQUIRE(batch > 0 && batch <= 65535 && t > 0 && c > 0, "se_stats_pool: bad shape");
  stats_pool_kernel<<<dim3(ceil_div(c, kRowThreads), batch), kRowThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      x, lengths, out, t, c);
  KT_CHECK_CUDA(cudaGetLastError());
  return KT_OK;
}

}  // namespace kt
