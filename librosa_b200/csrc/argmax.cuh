// argmax.cuh — np.argmax order on the device, shared by pyin's decoder (pitch_kernels.cuh), the general HMM
// decoder (sequence_kernels.cuh) and rqa (align_kernels.cuh): the first NaN wins, else the first maximum.
//
// A partial result is a (value, index) pair; index kArgNone marks a partial that holds no element yet, so lanes or
// warps without a state merge as empty and never win a tie.
#pragma once

namespace b2l {

constexpr int kArgNone = 0x7fffffff;

__device__ __forceinline__ bool argmax_before(double va, int ia, double vb, int ib) {
  const bool na = isnan(va), nb = isnan(vb);
  if (na != nb) return na;
  if (na) return ia < ib;
  return va > vb || (va == vb && ia < ib);
}

// (bv, bi) <- the earlier of (bv, bi) and (v, i) in np.argmax order; an empty side never wins.
__device__ __forceinline__ void argmax_merge(double& bv, int& bi, double v, int i) {
  if (i != kArgNone && (bi == kArgNone || argmax_before(v, i, bv, bi))) { bv = v; bi = i; }
}

// Butterfly over groups of W lanes (all 32 lanes of the warp take part); every lane of a group ends with its result.
template <int W = 32>
__device__ __forceinline__ void warp_argmax(double& v, int& i) {
#pragma unroll
  for (int o = W / 2; o > 0; o >>= 1) {
    const double ov = __shfl_xor_sync(0xffffffffu, v, o, W);
    const int oi = __shfl_xor_sync(0xffffffffu, i, o, W);
    argmax_merge(v, i, ov, oi);
  }
}

// Whole block: thread 0 ends with the result.  s_v / s_i hold one entry per warp; the call ends with a barrier
// behind the warps' writes, so the caller may reuse them after another __syncthreads().
__device__ __forceinline__ void block_argmax(double& v, int& i, double* s_v, int* s_i) {
  warp_argmax(v, i);
  if ((threadIdx.x & 31) == 0) { s_v[threadIdx.x >> 5] = v; s_i[threadIdx.x >> 5] = i; }
  __syncthreads();
  if (threadIdx.x == 0)
    for (int w = 1; w < (int)(blockDim.x + 31) / 32; ++w) argmax_merge(v, i, s_v[w], s_i[w]);
}

// The same with 64-bit indices, for arrays of 2^31 elements or more (rqa's score matrix, align_kernels.cuh).
constexpr long long kArgNone64 = 0x7fffffffffffffffLL;

__device__ __forceinline__ bool argmax_before(double va, long long ia, double vb, long long ib) {
  const bool na = isnan(va), nb = isnan(vb);
  if (na != nb) return na;
  if (na) return ia < ib;
  return va > vb || (va == vb && ia < ib);
}

__device__ __forceinline__ void argmax_merge(double& bv, long long& bi, double v, long long i) {
  if (i != kArgNone64 && (bi == kArgNone64 || argmax_before(v, i, bv, bi))) { bv = v; bi = i; }
}

__device__ __forceinline__ void warp_argmax(double& v, long long& i) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double ov = __shfl_xor_sync(0xffffffffu, v, o);
    const long long oi = __shfl_xor_sync(0xffffffffu, i, o);
    argmax_merge(v, i, ov, oi);
  }
}

__device__ __forceinline__ void block_argmax(double& v, long long& i, double* s_v, long long* s_i) {
  warp_argmax(v, i);
  if ((threadIdx.x & 31) == 0) { s_v[threadIdx.x >> 5] = v; s_i[threadIdx.x >> 5] = i; }
  __syncthreads();
  if (threadIdx.x == 0)
    for (int w = 1; w < (int)(blockDim.x + 31) / 32; ++w) argmax_merge(v, i, s_v[w], s_i[w]);
}

}  // namespace b2l
