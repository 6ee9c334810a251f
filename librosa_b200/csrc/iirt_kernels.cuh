// iirt_kernels.cuh — the semitone filter-bank spectrogram of librosa.iirt (librosa/core/spectrum.py:1522-1713).
//
//   pad_center_kernel   np.pad(y, pad, mode) of every clip into [clip][n + 2 pad] (load_padded's index map)
//   sosfiltfilt_kernel  scipy.signal.sosfiltfilt of one (clip, band) chain per thread, FP64, in place in scratch
//   stmsp_kernel        factor * sum(x[start + arange(w)] ** 2) per (clip, band, frame), NumPy's pairwise order
//
// Chains are grouped by sampling rate: the threads of a warp serve chains of one rate, so they share the signal
// length and walk their recursions in lockstep.  A rate's scratch is [row][chain] float64 with the chains fastest
// (stride: the rate's chain count rounded up to 32), so at every step a warp reads or writes one contiguous 256-byte
// run.  Row r of chain (clip, band) holds the filtered sample r; rows n .. n + padlen - 1 belong to the odd extension
// at the end and are never read as output.
//
// Both passes reproduce SciPy's _sosfilt loop bit for bit: per sample and section, with separately rounded
// multiplies and adds (no FMA contraction),
//   x_new = b0 x + z0;   z0 = (b1 x - a1 x_new) + z1;   z1 = b2 x - a2 x_new.
// The odd extension 2 x[0] - x[k] is formed in float32, as odd_ext forms it on the float32 signal.
#pragma once
#include <stdint.h>

#include "common.cuh"

namespace b2l_iirt {

constexpr int kMaxSections = B2L_IIRT_MAX_SECTIONS;   // butter at the default Q designs 10
constexpr int kMaxRates = B2L_IIRT_MAX_RATES;
constexpr int kCoefStride = 8;     // doubles per section in the coefficient table: b0 b1 b2 a1 a2 zi0 zi1 (pad)
constexpr int kFilterThreads = 128;
constexpr int kStmspThreads = 256;
constexpr int kChunk = 8;          // samples loaded ahead of the recursion
constexpr int kMaxDepth = B2L_IIRT_MAX_DEPTH;   // pairwise-sum stack

struct Rate {
  const float* x;       // [n_clips][x_stride] float32 signal at this rate
  long long x_stride;
  long long n;          // samples per clip: the filtered length
  double* scr;          // [rows][stride] float64 scratch
  long long stride;     // chains per row: n_clips * n_bands rounded up to 32
  const int* bands;     // [n_bands] filter-bank index of each band at this rate (its output row)
  int n_bands;
  long long block0;     // first block of this rate (filter kernel)
  long long sblock0;    // first block of this rate (stmsp kernel)
  const int* starts;    // [T] frame starts in samples at this rate
  const int4* leaves;   // pairwise-sum program: (offset, length, combines after it, 0)
  int n_leaves;
  double factor;        // sr / rate
};

struct Args {
  Rate rate[kMaxRates];
  int n_rates;
  const double* coef;   // [n_bands_total][kMaxSections][kCoefStride], pass-through sections after a band's own
  const int* info;      // [n_bands_total][2]: sections, padlen
  long long n_clips;
  long long T;          // frames
  int n_out_bands;      // rows of the output
  float* out;           // [n_clips][n_out_bands][T]
};

__device__ __forceinline__ int rate_of(const Args& a, long long block, bool stmsp) {
  int r = 0;
  while (r + 1 < a.n_rates && block >= (stmsp ? a.rate[r + 1].sblock0 : a.rate[r + 1].block0)) ++r;
  return r;
}

__global__ void __launch_bounds__(256) pad_center_kernel(const float* __restrict__ x, long long n_clips, int n,
                                                         int pad, int mode, float* __restrict__ out) {
  const long long n_out = (long long)n + 2LL * pad;
  const long long total = n_clips * n_out;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long c = i / n_out, j = i - c * n_out;
    out[i] = b2l::load_padded(x + c * n, n, j - pad, mode, pad);
  }
}

// A cascade of NS second-order sections, coefficients and state in registers.  A band with fewer sections than the
// launch's largest is padded with pass-through sections (b0 = 1, everything else 0, zero state): each returns its
// input unchanged (x + 0, with at most the sign of an exact zero changed), so no thread branches per section.
template <int NS>
struct Cascade {
  double b0[NS], b1[NS], b2[NS], a1[NS], a2[NS], z0[NS], z1[NS];

  __device__ __forceinline__ void load(const double* c) {
#pragma unroll
    for (int s = 0; s < NS; ++s) {
      const double* q = c + s * kCoefStride;
      b0[s] = __ldg(q + 0);
      b1[s] = __ldg(q + 1);
      b2[s] = __ldg(q + 2);
      a1[s] = __ldg(q + 3);
      a2[s] = __ldg(q + 4);
    }
  }
  // sosfilt's zi argument: sosfilt_zi(sos) * x0, one rounding per element
  __device__ __forceinline__ void init(const double* c, double x0) {
#pragma unroll
    for (int s = 0; s < NS; ++s) {
      z0[s] = __dmul_rn(__ldg(c + s * kCoefStride + 5), x0);
      z1[s] = __dmul_rn(__ldg(c + s * kCoefStride + 6), x0);
    }
  }
  __device__ __forceinline__ double step(double x) {
#pragma unroll
    for (int s = 0; s < NS; ++s) {
      const double xn = __dadd_rn(__dmul_rn(b0[s], x), z0[s]);
      z0[s] = __dadd_rn(__dsub_rn(__dmul_rn(b1[s], x), __dmul_rn(a1[s], xn)), z1[s]);
      z1[s] = __dsub_rn(__dmul_rn(b2[s], x), __dmul_rn(a2[s], xn));
      x = xn;
    }
    return x;
  }
};

// Sample i of odd_ext(x, p): 2 x[0] - x[p - i] before the signal, 2 x[n-1] - x[2n - 2 - k] after it (float32).
__device__ __forceinline__ double ext_at(const float* __restrict__ x, long long n, int p, long long i) {
  const long long k = i - p;
  if (k < 0) return (double)__fsub_rn(__fmul_rn(2.0f, __ldg(x)), __ldg(x + p - i));
  if (k < n) return (double)__ldg(x + k);
  return (double)__fsub_rn(__fmul_rn(2.0f, __ldg(x + n - 1)), __ldg(x + 2 * n - 2 - k));
}

// sosfiltfilt(sos, x, padtype="odd", padlen=3 * ntaps) of one chain: the forward pass over the extension of
// E = n + 2p samples stores outputs p .. E-1 in rows 0 .. n+p-1; the backward pass starts from zi * y[E-1] and runs
// over those rows in reverse, overwriting rows 0 .. n-1 with the result.  Outputs 0 .. p-1 of the forward pass are
// never read by the backward pass (it stops at the crop), so they are not stored.
template <int NS>
__global__ void __launch_bounds__(kFilterThreads) sosfiltfilt_kernel(const Args a) {
  const int ri = rate_of(a, blockIdx.x, false);
  const Rate& R = a.rate[ri];
  const long long c = ((long long)blockIdx.x - R.block0) * kFilterThreads + threadIdx.x;
  if (c >= a.n_clips * R.n_bands) return;
  const long long clip = c / R.n_bands;
  const int band = __ldg(R.bands + (c - clip * R.n_bands));
  const double* coef = a.coef + (long long)band * kMaxSections * kCoefStride;
  const int p = __ldg(a.info + 2 * band + 1);
  const float* x = R.x + clip * R.x_stride;
  const long long n = R.n, E = n + 2LL * p, st = R.stride;
  double* col = R.scr + c;

  Cascade<NS> f;
  f.load(coef);
  f.init(coef, ext_at(x, n, p, 0));
  double cur[kChunk], nxt[kChunk], last = 0.0;
#pragma unroll
  for (int k = 0; k < kChunk; ++k) cur[k] = k < E ? ext_at(x, n, p, k) : 0.0;
  for (long long i0 = 0; i0 < E; i0 += kChunk) {
#pragma unroll
    for (int k = 0; k < kChunk; ++k) nxt[k] = i0 + kChunk + k < E ? ext_at(x, n, p, i0 + kChunk + k) : 0.0;
#pragma unroll
    for (int k = 0; k < kChunk; ++k) {
      const long long i = i0 + k;
      if (i < E) {
        last = f.step(cur[k]);
        if (i >= p) col[(i - p) * st] = last;
      }
      cur[k] = nxt[k];
    }
  }

  f.init(coef, last);
  const long long top = n + p - 1;   // row of y[E-1]
#pragma unroll
  for (int k = 0; k < kChunk; ++k) cur[k] = top - k >= 0 ? col[(top - k) * st] : 0.0;
  for (long long r0 = top; r0 >= 0; r0 -= kChunk) {
#pragma unroll
    for (int k = 0; k < kChunk; ++k) nxt[k] = r0 - kChunk - k >= 0 ? col[(r0 - kChunk - k) * st] : 0.0;
#pragma unroll
    for (int k = 0; k < kChunk; ++k) {
      const long long r = r0 - k;
      if (r >= 0) {
        const double yb = f.step(cur[k]);
        if (r < n) col[r * st] = yb;
      }
      cur[k] = nxt[k];
    }
  }
}

// Squares of rows [o, o + len) of one chain, summed as NumPy's pairwise_sum sums a block of at most 128: a plain loop
// below 8 terms, else eight accumulators, combined ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), then the tail.  Rows at or
// past `valid` are the zeros of util.fix_length.
__device__ __forceinline__ double sq_at(const double* __restrict__ col, long long st, long long valid, long long j) {
  const double v = j < valid ? __ldg(col + j * st) : 0.0;
  return __dmul_rn(v, v);
}

__device__ __forceinline__ double leaf_sum(const double* __restrict__ col, long long st, long long valid, long long o,
                                           int len) {
  if (len < 8) {
    double s = 0.0;
    for (int i = 0; i < len; ++i) s = __dadd_rn(s, sq_at(col, st, valid, o + i));
    return s;
  }
  double r[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) r[k] = sq_at(col, st, valid, o + k);
  int i = 8;
  for (; i < len - (len % 8); i += 8) {
#pragma unroll
    for (int k = 0; k < 8; ++k) r[k] = __dadd_rn(r[k], sq_at(col, st, valid, o + i + k));
  }
  double s = __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), __dadd_rn(r[2], r[3])),
                       __dadd_rn(__dadd_rn(r[4], r[5]), __dadd_rn(r[6], r[7])));
  for (; i < len; ++i) s = __dadd_rn(s, sq_at(col, st, valid, o + i));
  return s;
}

// One output per thread, chains fastest within a frame: a warp reads 32 neighbouring chains of the same row.  The
// window's pairwise tree (split at n/2 - (n/2 mod 8) above 128 terms) is the rate's leaf program, evaluated in
// post-order with a stack of partial sums.
__global__ void __launch_bounds__(kStmspThreads) stmsp_kernel(const Args a) {
  const int ri = rate_of(a, blockIdx.x, true);
  const Rate& R = a.rate[ri];
  const long long g = ((long long)blockIdx.x - R.sblock0) * kStmspThreads + threadIdx.x;
  const long long t = g / R.stride, c = g - t * R.stride;
  if (t >= a.T || c >= a.n_clips * R.n_bands) return;
  const long long clip = c / R.n_bands;
  const int band = __ldg(R.bands + (c - clip * R.n_bands));
  const double* col = R.scr + c;
  const long long s0 = __ldg(R.starts + t);
  double stk[kMaxDepth];
  int sp = 0;
  for (int l = 0; l < R.n_leaves; ++l) {
    const int4 q = __ldg(R.leaves + l);
    stk[sp++] = leaf_sum(col, R.stride, R.n, s0 + q.x, q.y);
    for (int k = 0; k < q.z; ++k) {
      --sp;
      stk[sp - 1] = __dadd_rn(stk[sp - 1], stk[sp]);
    }
  }
  a.out[(clip * a.n_out_bands + band) * a.T + t] = __double2float_rn(__dmul_rn(R.factor, stk[0]));
}

}  // namespace b2l_iirt
