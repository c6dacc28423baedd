// In-shared-memory radix-2 FFT shared by the STFT / mel kernels (stft_mel.cu) and the Kaldi fbank (speaker.cu).
#pragma once
#include <cuda_runtime.h>

namespace kt {

__device__ __forceinline__ int bitrev(int x, int bits) { return (int)(__brev((unsigned)x) >> (32 - bits)); }

// in-place radix-2 DIT FFT over s[0..n) (already in bit-reversed order); sign = -1 forward, +1 inverse
__device__ inline void fft_inplace(float2* s, int n, int logn, float sign) {
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

}  // namespace kt
