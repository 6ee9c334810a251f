// fft64.cuh — the shared-memory FP64 radix-2 transform of one CTA, shared by the FP64 STFT kernels
// (f64_kernels.cuh) and the tempogram kernel (rhythm_kernels.cuh).  Device functions only, so that any number of
// units may include it.
#pragma once
#include <cuda_runtime.h>

namespace b2l {

__device__ __forceinline__ double2 cmul64(double2 a, double2 b) {
  return make_double2(fma(a.x, b.x, -a.y * b.y), fma(a.x, b.y, a.y * b.x));
}

__device__ __forceinline__ int bitrev_rt(int x, int bits) { return (int)(__brev((unsigned)x) >> (32 - bits)); }

// In-place radix-2 decimation-in-time FFT of M = 2^log2m points already stored in bit-reversed order.
// tw[j] = exp(-2*pi*i*j/(2M)), so W_M^p = tw[2p].  All threads of the block take part.
// static: every including unit keeps its own copy (a host-side stub would otherwise be defined twice).
static __device__ void fft64_inplace(double2* z, int log2m, const double2* __restrict__ tw) {
  const int M = 1 << log2m;
  for (int s = 1; s <= log2m; ++s) {
    const int half = 1 << (s - 1), stride = M >> s;      // twiddle step: W_(2*half)^pos = W_M^(pos*stride)
    for (int b = threadIdx.x; b < M / 2; b += blockDim.x) {
      const int pos = b & (half - 1), i0 = ((b - pos) << 1) + pos, i1 = i0 + half;
      const double2 w = tw[2 * pos * stride];
      const double2 a = z[i0], t = cmul64(w, z[i1]);
      z[i0] = make_double2(a.x + t.x, a.y + t.y);
      z[i1] = make_double2(a.x - t.x, a.y - t.y);
    }
    __syncthreads();
  }
}

}  // namespace b2l
