// Standalone check of contrast_kernel's tail extraction against a host sort (development aid).
//   nvcc -std=c++17 -O3 -gencode arch=compute_90a,code=sm_90a -I librosa_b200/csrc -o /tmp/contrast_test tools/micro/contrast_test.cu
#include <cstdio>
#include <cstdlib>
#include <vector>
#include <algorithm>
#include "feat_kernels.cuh"
using namespace b2l;
template <int N>
__global__ void sort_check(int* errs) {
  unsigned int v[16];
  unsigned int st = 12345u + 977u * (blockIdx.x * blockDim.x + threadIdx.x);
  for (int r = 0; r < 64; ++r) {
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      st = st * 1664525u + 1013904223u;
      v[j] = (j < N - (int)(threadIdx.x % 3)) ? (0x80000000u | (st >> 9)) : 0xffffffffu;
    }
    sort_keys<N>(v);
    bool bad = false;
#pragma unroll
    for (int j = 1; j < N; ++j) bad = bad || v[j - 1] > v[j];
    if (bad) atomicAdd(errs, 1);
  }
}
int main() {
  {
    int* d; cudaMalloc(&d, 16); cudaMemset(d, 0, 16);
    sort_check<2><<<8, 128>>>(d); sort_check<4><<<8, 128>>>(d + 1); sort_check<8><<<8, 128>>>(d + 2); sort_check<16><<<8, 128>>>(d + 3);
    int h[4]; cudaMemcpy(h, d, 16, cudaMemcpyDeviceToHost);
    printf("sort_keys errors: N=2 %d, N=4 %d, N=8 %d, N=16 %d\n", h[0], h[1], h[2], h[3]);
  }
  const int F = 1025, T = 64;
  std::vector<float> S((size_t)T * F);
  srand(1);
  for (auto& x : S) x = (float)(rand() % 100000) / 997.0f;
  ContrastArgs a;
  memset(&a, 0, sizeof(a));
  int los[] = {0, 18, 37, 74, 148, 297, 594}, cnts[] = {18, 19, 37, 74, 149, 297, 431}, ks[] = {1, 1, 1, 2, 3, 6, 9};
  a.n_bands = 7;
  for (int b = 0; b < 7; ++b) { a.lo[b] = los[b]; a.count[b] = cnts[b]; a.k[b] = ks[b]; }
  float *dS, *dp, *dv;
  cudaMalloc(&dS, S.size() * 4); cudaMalloc(&dp, 7 * T * 4); cudaMalloc(&dv, 7 * T * 4);
  cudaMemcpy(dS, S.data(), S.size() * 4, cudaMemcpyHostToDevice);
  const int cap = 512, nw = 8;
  const size_t smem = (size_t)nw * (1028 + cap) * 4;
  cudaFuncSetAttribute(contrast_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  contrast_kernel<<<4, nw * 32, smem>>>(dS, T, T, F, cap, a, dp, dv);
  std::vector<float> p(7 * T), v(7 * T);
  cudaMemcpy(p.data(), dp, p.size() * 4, cudaMemcpyDeviceToHost);
  cudaMemcpy(v.data(), dv, v.size() * 4, cudaMemcpyDeviceToHost);
  printf("cuda: %s\n", cudaGetErrorString(cudaGetLastError()));
  for (int b = 0; b < 7; ++b) {
    int bad = 0;
    for (int t = 0; t < T; ++t) {
      std::vector<float> x(S.begin() + (size_t)t * F + los[b], S.begin() + (size_t)t * F + los[b] + cnts[b]);
      std::sort(x.begin(), x.end());
      float lo = 0, hi = 0;
      for (int i = 0; i < ks[b]; ++i) { lo += x[i]; hi += x[x.size() - 1 - i]; }
      lo /= ks[b]; hi /= ks[b];
      if (fabsf(lo - v[b * T + t]) > 1e-5f * fabsf(lo) + 1e-6f || fabsf(hi - p[b * T + t]) > 1e-5f * fabsf(hi) + 1e-6f) {
        if (bad < 2) printf("  band %d frame %d: valley %g (want %g) peak %g (want %g)\n", b, t, v[b * T + t], lo, p[b * T + t], hi);
        ++bad;
      }
    }
    printf("band %d n=%d k=%d bad %d/%d\n", b, cnts[b], ks[b], bad, T);
  }
  return 0;
}
