// featutil_kernels.cuh — the feature-stacking utilities of librosa/feature/utils.py: delta and stack_memory.
//
//   delta_rows_kernel     savgol_filter along a contiguous axis (inner == 1): each warp stages a row tile plus its
//                         halo in its own shared-memory slot
//   delta_strided_kernel  savgol_filter along a strided axis (inner > 1): one output per thread, threads along inner
//   stack_memory_kernel   the gather of stack_memory: output (clip, step * d + row, i) <- input column i - step * delay
//   localext_kernel       librosa.util.localmax / localmin along one axis (librosa/util/utils.py), one byte per element
//
// delta reproduces scipy.ndimage.convolve1d (which savgol_filter calls) bit for bit: every line is widened to double,
// the reversed taps fw are applied in ndimage's fixed order with separately rounded multiplies and adds, and the sum is
// rounded once to the output type.  ndimage's three orders, with h = width / 2 and x centred on the output:
//   symmetric      acc = x[0] fw[0];  acc += (x[jj] + x[-jj]) fw[jj]  for jj = -h .. -1
//   antisymmetric  the same with (x[jj] - x[-jj])
//   neither        acc = x[h] fw[h];  acc += x[jj] fw[jj]             for jj = -h .. h-1
// Samples outside the line come from the padded-index table (pad): the source sample of each padded position, -1 for
// the constant.  mode="interp" replaces the first and last h outputs of a line by the float64 polynomial-fit map
// `edge` applied to the first or last `width` samples (ascending, unfused); a non-finite sample in such a window sets
// B2L_STATUS_NOT_FINITE_VALUE, where SciPy's fit raises.
#pragma once
#include <stdint.h>

#include "common.cuh"
#include "numerics.cuh"

namespace b2l_featutil {
using namespace b2l;

constexpr int kMaxWidth = B2L_DELTA_MAX_WIDTH;
constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
// Work items are per warp: a 431-frame MFCC row is two delta tiles or four stack_memory chunks, so many short rows
// are in flight at once instead of one row per block behind a barrier.
constexpr int kTile = 128;    // outputs of one warp's row tile (delta_rows_kernel)
constexpr int kChunk = 128;   // output columns of one warp's item (stack_memory_kernel), 4 per lane

// shared memory of delta_rows_kernel: the taps, then each warp's tile with its halo
__host__ __device__ inline int rows_smem_bytes(int h) {
  return (2 * h + 1 + kWarps * (kTile + 2 * h)) * (int)sizeof(double);
}

struct DeltaArgs {
  const void* x;          // [outer][n][inner]
  void* y;                // same geometry
  long long outer, n, inner;
  long long tiles;        // row tiles per line (delta_rows_kernel)
  int h;                  // width / 2
  int sym;                // 1 symmetric, -1 antisymmetric, 0 neither (ndimage's classification of fw)
  int interp;
  double cval;
  const double* fw;       // [2h + 1] reversed Savitzky-Golay coefficients
  const double* edge;     // [2h][2h + 1]: rows 0 .. h-1 give outputs 0 .. h-1 from x[0 .. 2h], rows h .. 2h-1 give
                          // outputs n-h .. n-1 from x[n-2h-1 .. n-1]
  const long long* pad;   // [2h]: padded positions -h .. -1, then n .. n+h-1
  int* status;
};

// Sample p (-h <= p < n + h) of the padded line starting at xr, samples `stride` apart.
template <class T>
__device__ __forceinline__ double load_line(const T* __restrict__ xr, long long stride, long long p, const DeltaArgs& a) {
  if (p < 0 || p >= a.n) {
    const long long src = __ldg(a.pad + (p < 0 ? p + a.h : p - a.n + a.h));
    if (src < 0) return a.cval;
    p = src;
  }
  return (double)__ldg(xr + p * stride);
}

// ndimage's correlation at one output; X(jj) is the sample jj positions from it, fw points at the centre tap.
template <class F>
__device__ __forceinline__ double correlate(F X, const double* fw, int h, int sym) {
  if (sym > 0) {
    double acc = __dmul_rn(X(0), fw[0]);
    for (int jj = -h; jj < 0; ++jj) acc = __dadd_rn(acc, __dmul_rn(__dadd_rn(X(jj), X(-jj)), fw[jj]));
    return acc;
  }
  if (sym < 0) {
    double acc = __dmul_rn(X(0), fw[0]);
    for (int jj = -h; jj < 0; ++jj) acc = __dadd_rn(acc, __dmul_rn(__dsub_rn(X(jj), X(-jj)), fw[jj]));
    return acc;
  }
  double acc = __dmul_rn(X(h), fw[h]);
  for (int jj = -h; jj < h; ++jj) acc = __dadd_rn(acc, __dmul_rn(X(jj), fw[jj]));
  return acc;
}

// mode="interp": output j of a line (j < h or j >= n - h) from the edge map.
template <class T>
__device__ double interp_edge(const T* __restrict__ xr, long long stride, long long j, const DeltaArgs& a) {
  const int w = 2 * a.h + 1;
  const bool left = j < a.h;
  const double* e = a.edge + (left ? j : a.h + (j - (a.n - a.h))) * (long long)w;
  const T* xw = xr + (left ? 0 : (a.n - w)) * stride;
  bool bad = false;
  double acc = 0.0;
  for (int k = 0; k < w; ++k) {
    const double v = (double)__ldg(xw + k * stride);
    bad |= !isfinite(v);
    const double t = __dmul_rn(__ldg(e + k), v);
    acc = k == 0 ? t : __dadd_rn(acc, t);
  }
  if (bad) atomicOr(a.status, B2L_STATUS_NOT_FINITE_VALUE);
  return acc;
}

template <class T>
__device__ __forceinline__ bool is_edge(const DeltaArgs& a, long long j) {
  return a.interp && (j < a.h || j >= a.n - a.h);
}

// inner == 1: warp-stride loop over (line, tile) pairs; a warp stages its tile [j0 - h, j0 + len + h) as double.
template <class T>
__global__ void __launch_bounds__(kThreads) delta_rows_kernel(DeltaArgs a) {
  extern __shared__ double smem[];
  const int h = a.h, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double* fw = smem;
  double* tile = smem + 2 * h + 1 + warp * (kTile + 2 * h);
  for (int i = threadIdx.x; i < 2 * h + 1; i += blockDim.x) fw[i] = __ldg(a.fw + i);
  __syncthreads();
  const T* x = (const T*)a.x;
  T* y = (T*)a.y;
  for (long long b = blockIdx.x * (long long)kWarps + warp; b < a.outer * a.tiles; b += (long long)gridDim.x * kWarps) {
    const long long line = b / a.tiles;
    const long long j0 = (b - line * a.tiles) * kTile;
    const int len = (int)min((long long)kTile, a.n - j0);
    const T* xr = x + line * a.n;
    T* yr = y + line * a.n;
    __syncwarp();   // the warp's previous tile is consumed
#pragma unroll 4
    for (int i = lane; i < len + 2 * h; i += 32) tile[i] = load_line(xr, 1, j0 - h + i, a);
    __syncwarp();
    for (int i = lane; i < len; i += 32) {
      const long long j = j0 + i;
      const double* c = tile + i + h;
      const double v = is_edge<T>(a, j) ? interp_edge(xr, 1, j, a)
                                        : correlate([c](int jj) { return c[jj]; }, fw + h, h, a.sym);
      yr[j] = narrow<T>(v);
    }
  }
}

// inner > 1: grid-stride loop over the outputs in memory order, so a warp reads and writes along inner.
template <class T>
__global__ void __launch_bounds__(kThreads) delta_strided_kernel(DeltaArgs a) {
  extern __shared__ double smem[];
  const int h = a.h;
  for (int i = threadIdx.x; i < 2 * h + 1; i += blockDim.x) smem[i] = __ldg(a.fw + i);
  __syncthreads();
  const T* x = (const T*)a.x;
  T* y = (T*)a.y;
  const long long total = a.outer * a.n * a.inner;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const long long k = e % a.inner;
    const long long r = e / a.inner;
    const long long j = r % a.n;
    const T* xr = x + (r - j) * a.inner + k;
    double v;
    if (is_edge<T>(a, j)) {
      v = interp_edge(xr, a.inner, j, a);
    } else {
      v = correlate([&](int jj) { return load_line(xr, a.inner, j + jj, a); }, smem + h, h, a.sym);
    }
    y[e] = narrow<T>(v);
  }
}

struct StackArgs {
  const void* x;          // [n_clips] x (d, t): element (c, r, i) at c * clip_stride + r * row_stride + i * col_stride
  long long clip_stride, row_stride, col_stride;
  void* out;              // [n_clips][n_steps * d][t], C order
  long long n_clips, d, t, delay;
  int n_steps;
  long long n_pad;        // (n_steps - 1) * |delay|
  const long long* pad;   // [n_pad]: padded positions -n_pad .. -1 (delay > 0) or t .. t + n_pad - 1 (delay < 0)
  uint4 fill;             // the constant, in the element's bytes
  long long rows;         // n_clips * n_steps * d
  long long chunks;       // column chunks of kChunk per output row
};

template <int S> struct Elem;
template <> struct Elem<1> { typedef uint8_t T; };
template <> struct Elem<2> { typedef uint16_t T; };
template <> struct Elem<4> { typedef uint32_t T; };
template <> struct Elem<8> { typedef unsigned long long T; };
template <> struct Elem<16> { typedef uint4 T; };

// Output row (clip, step * d + row) column i reads input column q = i - step * delay; columns outside [0, t) are the
// padded positions of np.pad and go through the table.  This is __stack's block order for either sign of delay.
// One warp item is kChunk columns of one output row: each lane issues its four loads before its four stores.
template <int S>
__global__ void __launch_bounds__(kThreads) stack_memory_kernel(StackArgs a) {
  typedef typename Elem<S>::T T;
  const T* __restrict__ x = (const T*)a.x;
  T* __restrict__ out = (T*)a.out;
  T fill;
  memcpy(&fill, &a.fill, S);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  constexpr int kPer = kChunk / 32;
  for (long long b = blockIdx.x * (long long)kWarps + warp; b < a.rows * a.chunks; b += (long long)gridDim.x * kWarps) {
    const long long orow = b / a.chunks;
    const long long i0 = (b - orow * a.chunks) * kChunk + lane;
    const long long c = orow / (a.n_steps * a.d);
    const long long sr = orow - c * (a.n_steps * a.d);
    const long long s = sr / a.d;
    const T* xr = x + c * a.clip_stride + (sr - s * a.d) * a.row_stride;
    T* yr = out + orow * a.t;
    const long long shift = s * a.delay;
    T v[kPer];
#pragma unroll
    for (int k = 0; k < kPer; ++k) {
      const long long i = i0 + 32 * k;
      if (i < a.t) {
        long long q = i - shift;
        if (q < 0 || q >= a.t) q = __ldg(a.pad + (q < 0 ? q + a.n_pad : q - a.t));
        v[k] = q < 0 ? fill : xr[q * a.col_stride];
      }
    }
#pragma unroll
    for (int k = 0; k < kPer; ++k)
      if (i0 + 32 * k < a.t) yr[i0 + 32 * k] = v[k];
  }
}

// librosa.util.localmax / localmin along the middle axis of x [outer][n][inner] (n >= 2) into one byte per element:
// local_extremum (numerics.cuh) of each element and its neighbours on the line.  One output per thread in memory order;
// CONTIG (inner == 1) spares the division by inner, as delta's row path does.
template <class T, bool CONTIG>
__global__ void __launch_bounds__(kThreads) localext_kernel(const T* __restrict__ x, long long total, long long n,
                                                            long long inner, bool is_max, uint8_t* __restrict__ out) {
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const long long j = CONTIG ? e % n : (e / inner) % n;
    const long long s = CONTIG ? 1 : inner;
    const T cur = x[e];
    const T prev = j > 0 ? x[e - s] : cur;
    const T next = j < n - 1 ? x[e + s] : cur;
    out[e] = local_extremum(is_max, j, n, prev, cur, next);
  }
}

}  // namespace b2l_featutil
