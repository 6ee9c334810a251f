// rhythm_kernels.cuh — librosa.feature.tempogram / tempo (librosa/feature/rhythm.py:38-470).
//
//   tempogram_kernel<T>  onset envelope (T = float or double) -> normalised local autocorrelation, float64
//                        [row][frame][lag] (one CTA per (row, frame), FP64 throughout)
//   tempo_kernel<T>      tempogram (float64, or float32 when the caller hands one in) -> BPM of the first maximum
//                        of log1p(1e6 tg) + logprior over the lags, per row (time mean) or per (row, frame)
//
// A row is one envelope: every leading index of the caller's array, bands of a multi-band envelope included.
#pragma once
#include <float.h>
#include <math.h>

#include "../../include/b2l.h"
#include "fft64.cuh"
#include "numerics.cuh"

namespace b2l {

struct TempogramArgs {
  const void* x;          // [rows][n] envelope of type T
  int n, win, pad;        // pad = win / 2 when centred, else 0
  int n_frames, log2m;    // frames per row; the transform has N = 2^(log2m+1) >= 2 win - 1 real points
  const double* window;   // [win]
  const double2* tw;      // exp(-2 pi i j / N), j <= N / 2
  int norm;               // B2L_TG_NORM_*
  double norm_p;          // the exponent of B2L_TG_NORM_P
  double* out;            // [rows][n_frames][win]
  int* status;            // B2L_STATUS_NOT_FINITE_VALUE: a value of the autocorrelation is not finite
};

// Dynamic shared memory of tempogram_kernel in doubles: z [M] double2, p [M + 1], window [win], reduction [32].
__host__ __device__ inline size_t tempogram_smem_doubles(int log2m, int win) {
  const size_t M = (size_t)1 << log2m;
  return 2 * M + (M + 1) + (size_t)win + 32;
}

// One CTA per (row, frame):
//   1. frame t of np.pad(x, win // 2, mode="linear_ramp", end_values=0) when centred (the ramp value is formed in
//      double and rounded to T, as NumPy does), of x otherwise, times the float64 window;
//   2. zero-padded to N, packed real FFT, P = |X|^2;
//   3. P is real and even, so the same packed transform of P gives N r: the linear autocorrelation on lags < win;
//   4. util.normalize along the lags (threshold tiny(float64), fill=None).
template <class T>
__global__ void tempogram_kernel(const TempogramArgs a) {
  extern __shared__ __align__(16) unsigned char smem_tg[];
  const int M = 1 << a.log2m, W = a.win;
  double2* z = reinterpret_cast<double2*>(smem_tg);
  double* p = reinterpret_cast<double*>(z + M);   // power spectrum, then the autocorrelation
  double* w = p + M + 1;
  double* red = w + W;
  const long long item = blockIdx.x;
  const long long row = item / a.n_frames;
  const int t = (int)(item % a.n_frames);
  const T* x = static_cast<const T*>(a.x) + row * a.n;
  for (int i = threadIdx.x; i < W; i += blockDim.x) w[i] = a.window[i];
  __syncthreads();
  auto frame = [&](int i) -> double {
    if (i >= W) return 0.0;
    const long long j = (long long)t + i - a.pad;
    T v;
    if (j < 0 || j >= a.n) {
      const long long d = j < 0 ? -j : j - (a.n - 1);     // 1 .. pad
      v = (T)((double)(a.pad - d) * ((double)x[j < 0 ? 0 : a.n - 1] / (double)a.pad));
    } else {
      v = x[j];
    }
    return (double)v * w[i];
  };
  for (int e = threadIdx.x; e < M; e += blockDim.x) z[bitrev_rt(e, a.log2m)] = make_double2(frame(2 * e), frame(2 * e + 1));
  __syncthreads();
  fft64_inplace(z, a.log2m, a.tw);
  // real-FFT un-mix (as stft64_kernel): X[k] = E + W_N^k O, k = 0 .. M
  for (int k = threadIdx.x; k <= M; k += blockDim.x) {
    const double2 A = z[k & (M - 1)], B = z[(M - k) & (M - 1)];
    const double er = 0.5 * (A.x + B.x), ei = 0.5 * (A.y - B.y);
    const double orr = 0.5 * (A.y + B.y), oi = 0.5 * (B.x - A.x);
    const double2 tw = a.tw[k];
    const double xr = er + (tw.x * orr - tw.y * oi), xi = ei + (tw.x * oi + tw.y * orr);
    p[k] = xr * xr + xi * xi;
  }
  __syncthreads();
  for (int e = threadIdx.x; e < M; e += blockDim.x) {
    const int m0 = 2 * e, m1 = 2 * e + 1;   // P[N - m] = P[m]
    z[bitrev_rt(e, a.log2m)] = make_double2(p[m0 <= M ? m0 : 2 * M - m0], p[m1 <= M ? m1 : 2 * M - m1]);
  }
  __syncthreads();
  fft64_inplace(z, a.log2m, a.tw);
  const double inv_n = 1.0 / (double)(2 * M);
  double part = a.norm == B2L_TG_NORM_MIN ? INFINITY : 0.0;
  bool bad = false;
  for (int k = threadIdx.x; k < W; k += blockDim.x) {
    const double2 A = z[k & (M - 1)], B = z[(M - k) & (M - 1)];
    const double er = 0.5 * (A.x + B.x), orr = 0.5 * (A.y + B.y), oi = 0.5 * (B.x - A.x);
    const double2 tw = a.tw[k];
    const double r = (er + (tw.x * orr - tw.y * oi)) * inv_n;
    p[k] = r;
    bad |= !isfinite(r);
    const double m = fabs(r);
    switch (a.norm) {
      case B2L_TG_NORM_MAX: part = fmax(part, m); break;
      case B2L_TG_NORM_MIN: part = fmin(part, m); break;
      case B2L_TG_NORM_COUNT: part += m > 0.0 ? 1.0 : 0.0; break;
      case B2L_TG_NORM_P: part += pow(m, a.norm_p); break;
      default: break;
    }
  }
  // Block-wide reduction in a fixed order (the same result on every run).  Not block_reduce (numerics.cuh): this one
  // has its barrier after the read rather than before the write, and moving it changes the kernel's code.
  auto reduce = [&](double v, auto op) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    v = warp_reduce(v, op);
    if (lane == 0) red[warp] = v;
    __syncthreads();
    double r = red[0];
    for (int i = 1; i < nw; ++i) r = op(r, red[i]);
    __syncthreads();
    return r;
  };
  double length = 1.0;
  if (a.norm == B2L_TG_NORM_MAX) length = reduce(part, [](double u, double v) { return fmax(u, v); });
  else if (a.norm == B2L_TG_NORM_MIN) length = reduce(part, [](double u, double v) { return fmin(u, v); });
  else if (a.norm == B2L_TG_NORM_COUNT) length = reduce(part, [](double u, double v) { return u + v; });
  else if (a.norm == B2L_TG_NORM_P)
    length = pow(reduce(part, [](double u, double v) { return u + v; }), 1.0 / a.norm_p);
  if (length < DBL_MIN) length = 1.0;      // below tiny(float64): left as it is
  double* o = a.out + item * W;
  for (int k = threadIdx.x; k < W; k += blockDim.x) o[k] = p[k] / length;
  if (bad && a.status) atomicOr(a.status, B2L_STATUS_NOT_FINITE_VALUE);
}

struct TempoArgs {
  const void* tg;                       // tempogram of type T
  long long rows;
  int n_lags, n_frames;
  long long row_stride, lag_stride, frame_stride;   // in elements
  const double* logprior;               // [n_lags], -inf where the prior or max_tempo excludes a lag
  const double* bpms;                   // [n_lags], bpms[0] = inf
  double* out;                          // [rows] (time mean) or [rows][n_frames]
};

// log1p(1e6 tg) + logprior in the tempogram's precision, as NumPy evaluates it (float32 log1p for float32 input)
__device__ __forceinline__ double tempo_score(double v, double lp) { return log1p(1e6 * v) + lp; }
__device__ __forceinline__ double tempo_score(float v, double lp) { return (double)log1pf(1e6f * v) + lp; }

// np.argmax order: NaN first, then the larger score, then the smaller lag
struct TempoMerge {
  __device__ __forceinline__ void operator()(double& bv, int& bk, double v, int k) const {
    if (before(v, k, bv, bk)) { bv = v; bk = k; }
  }
  static __device__ __forceinline__ bool before(double v, int k, double bv, int bk) {
    const bool vn = isnan(v), bn = isnan(bv);
    if (vn != bn) return vn;
    if (!vn && v != bv) return v > bv;
    return k < bk;
  }
};

// aggregate=np.mean: one CTA per row.  Each thread owns lags and sums their frames in increasing order, so the
// result does not depend on scheduling; the mean of a float32 tempogram is rounded to float32.
template <class T>
__global__ void tempo_mean_kernel(const TempoArgs a) {
  __shared__ double s_v[32];
  __shared__ int s_k[32];
  const long long row = blockIdx.x;
  const T* g = static_cast<const T*>(a.tg) + row * a.row_stride;
  double best = -INFINITY;
  int bk = 0x7fffffff;
  for (int k = threadIdx.x; k < a.n_lags; k += blockDim.x) {
    const T* gk = g + k * a.lag_stride;
    double s = 0.0;
    for (int f = 0; f < a.n_frames; ++f) s += (double)gk[f * a.frame_stride];
    TempoMerge()(best, bk, tempo_score((T)(s / (double)a.n_frames), a.logprior[k]), k);
  }
  warp_select(best, bk, TempoMerge());
  // not block_select (numerics.cuh): its warp count rounds blockDim up, which changes this kernel's code; the merge
  // functor in the loop below changes it too, so the loop applies TempoMerge::before itself
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) { s_v[warp] = best; s_k[warp] = bk; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < (int)(blockDim.x >> 5); ++i)
      if (TempoMerge::before(s_v[i], s_k[i], best, bk)) { best = s_v[i]; bk = s_k[i]; }
    a.out[row] = a.bpms[bk];
  }
}

// aggregate=None: one warp per (row, frame), lanes stride the lags.
template <class T>
__global__ void tempo_frames_kernel(const TempoArgs a) {
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= a.rows * a.n_frames) return;
  const long long row = warp / a.n_frames;
  const int f = (int)(warp % a.n_frames);
  const T* g = static_cast<const T*>(a.tg) + row * a.row_stride + f * a.frame_stride;
  double best = -INFINITY;
  int bk = 0x7fffffff;
  for (int k = lane; k < a.n_lags; k += 32) {
    TempoMerge()(best, bk, tempo_score(g[k * a.lag_stride], a.logprior[k]), k);
  }
  warp_select(best, bk, TempoMerge());
  if (lane == 0) a.out[warp] = a.bpms[bk];
}

}  // namespace b2l
