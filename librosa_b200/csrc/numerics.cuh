// numerics.cuh — the device primitives the area kernels share: correctly rounded arithmetic, rounding to T, NumPy's
// NaN rules, warp and block reductions and ordered (value, index) selection.  They decide bit-exactness against the
// reference (the rounding of an operation, which operand a NaN max returns, which index wins a tie), so each rule is
// written once, here.  Inline device functions, templates and functors only: every unit may include this header.
// The transform headers (fwd_kernel.cuh, inv_kernel.cuh, mr_kernel.cuh, czt_kernel.cuh) do not.
#pragma once
#include <cuda_runtime.h>
#include <math.h>

#include <type_traits>

namespace b2l {

// One correctly rounded operation in the operands' precision: explicit intrinsics keep nvcc from contracting a
// multiply and an add into an FMA, which the reference (NumPy, numba without fast-math) never does.
__device__ __forceinline__ float add_rn(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double add_rn(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ float sub_rn(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ double sub_rn(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ float div_rn(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ double div_rn(double a, double b) { return __ddiv_rn(a, b); }
__device__ __forceinline__ float sqrt_rn(float a) { return __fsqrt_rn(a); }
__device__ __forceinline__ double sqrt_rn(double a) { return __dsqrt_rn(a); }
__device__ __forceinline__ float log1p_(float x) { return log1pf(x); }
__device__ __forceinline__ double log1p_(double x) { return log1p(x); }
// |z| through hypot, as plp needs.  Not cqt's np_abs (NumPy's x86 loop, cqt_kernels.cuh) nor chroma's Mag<float2>
// (correctly rounded through double, chroma_kernels.cuh): the three round differently.
__device__ __forceinline__ float cabs_(float2 z) { return hypotf(z.x, z.y); }
__device__ __forceinline__ double cabs_(double2 z) { return hypot(z.x, z.y); }
template <class T> __device__ __forceinline__ bool finite_(T v) { return isfinite(v); }

// A float64 value rounded once to T (round to nearest even), as NumPy's cast does.
template <class T> __device__ __forceinline__ T narrow(double v);
template <> __device__ __forceinline__ float narrow<float>(double v) { return __double2float_rn(v); }
template <> __device__ __forceinline__ double narrow<double>(double v) { return v; }
// The smallest normal of T: np.finfo(T).tiny.
template <class T> __device__ __forceinline__ T tiny_of() { return sizeof(T) == 4 ? (T)1.17549435e-38f : (T)2.2250738585072014e-308; }

// np.min / np.max: NaN wins (the first NaN operand is returned)
struct MinNan { template <class T> __device__ T operator()(T a, T b) const { return a != a ? a : (b != b ? b : (b < a ? b : a)); } };
struct MaxNan { template <class T> __device__ T operator()(T a, T b) const { return a != a ? a : (b != b ? b : (b > a ? b : a)); } };

// v <- op(v, v of lane ^ o) for o = 16 .. 1: every lane of the warp ends with the warp's result.
template <class T, class Op>
__device__ __forceinline__ T warp_reduce(T v, Op op) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = op(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Whole block (blockDim.x a multiple of 32), every thread ends with the result, combined in warp order.  s_red holds
// one entry per warp.  The barrier before the warps' writes lets consecutive calls share s_red; the caller needs
// another __syncthreads() before it writes s_red for anything else.
template <class T, class Op>
__device__ __forceinline__ T block_reduce(T v, Op op, T* s_red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  v = warp_reduce(v, op);
  __syncthreads();
  if (lane == 0) s_red[warp] = v;
  __syncthreads();
  v = s_red[0];
  for (int w = 1; w < nw; ++w) v = op(v, s_red[w]);
  return v;
}

// Ordered selection of (value, index) partials.  A rule is a merge functor: merge(v, i, ov, oi) replaces (v, i) by
// (ov, oi) when (ov, oi) goes first in its order.  (A merge, not a bool predicate: nvcc emits different code for the
// same test once it is returned through a bool.)
// Butterfly over groups of W lanes (all 32 lanes of the warp take part); every lane of a group ends with its result.
template <int W = 32, class V, class I, class Merge>
__device__ __forceinline__ void warp_select(V& v, I& i, Merge merge) {
#pragma unroll
  for (int o = W / 2; o > 0; o >>= 1) {
    const V ov = __shfl_xor_sync(0xffffffffu, v, o, W);
    const I oi = __shfl_xor_sync(0xffffffffu, i, o, W);
    merge(v, i, ov, oi);
  }
}

// Whole block: thread 0 ends with the result.  s_v / s_i hold one entry per warp; the call ends with a barrier
// behind the warps' writes, so the caller may reuse them after another __syncthreads().
template <class V, class I, class Merge>
__device__ __forceinline__ void block_select(V& v, I& i, V* s_v, I* s_i, Merge merge) {
  warp_select(v, i, merge);
  if ((threadIdx.x & 31) == 0) { s_v[threadIdx.x >> 5] = v; s_i[threadIdx.x >> 5] = i; }
  __syncthreads();
  if (threadIdx.x == 0)
    for (int w = 1; w < (int)(blockDim.x + 31) / 32; ++w) merge(v, i, s_v[w], s_i[w]);
}

// np.argmax order: the first NaN wins, else the first maximum.  Index kArgNone (kArgNone64 for 64-bit indices, which
// arrays of 2^31 elements or more need) marks a partial that holds no element yet, so lanes or warps without an
// element merge as empty and never win a tie.
constexpr int kArgNone = 0x7fffffff;
constexpr long long kArgNone64 = 0x7fffffffffffffffLL;
struct ArgmaxMerge {
  template <class I>
  __device__ __forceinline__ void operator()(double& bv, I& bi, double v, I i) const {
    static_assert(std::is_same<I, int>::value || std::is_same<I, long long>::value, "int or long long indices");
    const I none = std::is_same<I, int>::value ? (I)kArgNone : (I)kArgNone64;
    if (i != none && (bi == none || before(v, i, bv, bi))) { bv = v; bi = i; }
  }
  template <class I>
  static __device__ __forceinline__ bool before(double va, I ia, double vb, I ib) {
    const bool na = isnan(va), nb = isnan(vb);
    if (na != nb) return na;
    if (na) return ia < ib;
    return va > vb || (va == vb && ia < ib);
  }
};

// 1-D librosa.util.localmax / localmin at position i of a line of n >= 2 values (librosa/util/utils.py:1029-1178):
// never at i = 0; cur > prev and cur >= next inside the line (cur < prev and cur <= next for a minimum); cur > prev
// alone at i = n - 1, where `next` is ignored.  A NaN compares false.
template <class T>
__device__ __forceinline__ bool local_extremum(bool is_max, long long i, long long n, T prev, T cur, T next) {
  if (i == 0) return false;
  if (is_max) return cur > prev && (i == n - 1 || cur >= next);
  return cur < prev && (i == n - 1 || cur <= next);
}

}  // namespace b2l
