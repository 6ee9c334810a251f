// Register-only radix-32 DFT throughput: the butterfly network of fft_engine.cuh with no memory traffic, at the
// occupancy of the production kernels (512 threads and 128 registers per thread, one CTA per SM).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o dft32_rate dft32_rate.cu
#include "../../librosa_b200/csrc/fft_engine.cuh"
#include <cstdio>
using namespace b2l;

constexpr int ITER = 2048;

template <int WITH_TW>
__global__ void __launch_bounds__(512, 1) dft_loop(float2* out, float2 seed, float2 tw) {
  float2 v[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) v[i] = make_float2(seed.x * (threadIdx.x + i), seed.y * (i - 7));
  for (int it = 0; it < ITER; ++it) {
    if constexpr (WITH_TW) {
#pragma unroll
      for (int i = 1; i < 32; ++i) v[i] = cmul(v[i], tw);     // the inter-pass twiddle product
    }
    dft_reg<32, 0>(v);
  }
  float2 s = make_float2(0.f, 0.f);
#pragma unroll
  for (int i = 0; i < 32; ++i) { s.x += v[i].x; s.y += v[i].y; }
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

template <int WITH_TW>
void run(const char* name, float2* out, int sms) {
  dft_loop<WITH_TW><<<sms, 512>>>(out, make_float2(1e-3f, 2e-3f), make_float2(0.7f, 0.7f));
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  cudaEventRecord(a);
  for (int r = 0; r < 5; ++r) dft_loop<WITH_TW><<<sms, 512>>>(out, make_float2(1e-3f, 2e-3f), make_float2(0.7f, 0.7f));
  cudaEventRecord(b); cudaEventSynchronize(b);
  float ms; cudaEventElapsedTime(&ms, a, b); ms /= 5;
  const double dfts = double(sms) * 512 * ITER;
  printf("%-34s %8.3f ms   %7.2f G radix-32 DFTs/s   %6.1f clk per DFT and sub-partition warp (1.965 GHz)\n", name, ms,
         dfts / ms * 1e-6, ms * 1e-3 * 1.965e9 / (double(ITER) * 4));
}

int main() {
  cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
  float2* out; cudaMalloc(&out, size_t(p.multiProcessorCount) * 512 * sizeof(float2));
  printf("%s\n", p.name);
  run<0>("radix-32 DFT", out, p.multiProcessorCount);
  run<1>("31 twiddle products + radix-32 DFT", out, p.multiProcessorCount);
  printf("%s\n", cudaGetErrorString(cudaDeviceSynchronize()));
  return 0;
}
