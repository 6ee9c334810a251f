// f64_kernels.cuh — double-precision path: what librosa computes when it is handed float64 audio
// (complex128 STFT, float64 spectrogram / mel / dB / MFCC; librosa/core/spectrum.py:341 dtype_r2c, :388 rfft of
// the float64 window product, :598 irfft, feature/spectral.py:2160 einsum in the input's precision).
//
// This is the correctness path for float64 callers, not the throughput path: one CTA per frame, the transform in
// shared memory (in-place radix-2 for powers of two, a direct O(n_fft^2) DFT with an exact twiddle table for any
// other length), FP64 arithmetic throughout.  The float32 kernels (fwd_kernel / inv_kernel) remain
// the product's hot path; these kernels make `stft(float64)` mean float64 instead of a relabelled float32 result.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"
#include "fft64.cuh"
#include "numerics.cuh"

namespace b2l {

// np.pad index map in double (same modes as load_padded in common.cuh)
__device__ __forceinline__ double load_padded64(const double* __restrict__ y, int n, long long j, int mode, int pad) {
  if (j >= 0 && j < n) return y[j];
  switch (mode) {
    case PAD_EDGE:
      return y[j < 0 ? 0 : n - 1];
    case PAD_REFLECT: {
      if (n == 1) return y[0];
      long long P = 2LL * (n - 1), m = j % P;
      if (m < 0) m += P;
      if (m >= n) m = P - m;
      return y[m];
    }
    case PAD_SYMMETRIC: {
      long long P = 2LL * n, m = j % P;
      if (m < 0) m += P;
      if (m >= n) m = P - 1 - m;
      return y[m];
    }
    case PAD_LINEAR_RAMP: {
      long long d = j < 0 ? -j : j - (n - 1);
      double edge = y[j < 0 ? 0 : n - 1];
      long long i = pad - d;
      if (i <= 0) return 0.0;
      return (double)i * (edge / (double)pad);
    }
    default:
      return 0.0;
  }
}

struct F64FwdArgs {
  const double* y;          // [n_clips][y_stride]
  long long y_stride;
  int n, n_clips, n_fft, hop, pad, pad_mode, n_frames;
  int log2m;                // >= 1: n_fft = 2^(log2m+1) -> packed FFT; 0: direct DFT
  const double* window;     // [n_fft]
  const double2* tw;        // exp(-2*pi*i*j/n_fft): j <= n_fft/2 (FFT) or j < n_fft (DFT)
  double2* out;             // [n_clips][n_frames][n_fft/2 + 1]
  int* status;
  double2* zscratch;        // per-frame work area in global memory for sizes that do not fit in shared memory
                            // (n_fft/2 double2 per frame for the FFT, n_fft doubles for the DFT); NULL: shared memory
};

// One CTA per (frame, clip): windowed frame -> complex spectrum.  A sample np.isfinite rejects sets the status word
// (tested before the window product, so a zero window tap does not hide it); samples no frame reads are left to
// finite_scan64_kernel.
__global__ void stft64_kernel(const F64FwdArgs a) {
  extern __shared__ __align__(16) unsigned char smem64[];
  const long long item = blockIdx.x;
  const int clip = (int)(item / a.n_frames), frame = (int)(item % a.n_frames);
  const double* yc = a.y + (long long)clip * a.y_stride;
  const long long s0 = (long long)frame * a.hop - a.pad;
  const int N = a.n_fft, F = N / 2 + 1;
  double2* orow = a.out + ((long long)clip * a.n_frames + frame) * F;
  bool bad = false;
  if (a.log2m > 0) {
    const int M = N / 2;
    double2* z = a.zscratch ? a.zscratch + item * M : reinterpret_cast<double2*>(smem64);
    for (int e = threadIdx.x; e < M; e += blockDim.x) {
      const double v0 = load_padded64(yc, a.n, s0 + 2 * e, a.pad_mode, a.pad);
      const double v1 = load_padded64(yc, a.n, s0 + 2 * e + 1, a.pad_mode, a.pad);
      bad |= !isfinite(v0) || !isfinite(v1);
      z[bitrev_rt(e, a.log2m)] = make_double2(v0 * a.window[2 * e], v1 * a.window[2 * e + 1]);
    }
    __syncthreads();
    fft64_inplace(z, a.log2m, a.tw);
    // real-FFT un-mix: X[k] = E + W_N^k O, E = (Z[k] + conj Z[M-k]) / 2, O = (Z[k] - conj Z[M-k]) / (2i)
    for (int k = threadIdx.x; k <= M; k += blockDim.x) {
      const double2 A = z[k & (M - 1)], B = z[(M - k) & (M - 1)];
      const double er = 0.5 * (A.x + B.x), ei = 0.5 * (A.y - B.y);
      const double orr = 0.5 * (A.y + B.y), oi = 0.5 * (B.x - A.x);
      const double2 w = a.tw[k];
      orow[k] = make_double2(er + (w.x * orr - w.y * oi), ei + (w.x * oi + w.y * orr));
    }
  } else {
    double* xw = a.zscratch ? reinterpret_cast<double*>(a.zscratch) + item * N : reinterpret_cast<double*>(smem64);
    for (int i = threadIdx.x; i < N; i += blockDim.x) {
      const double v = load_padded64(yc, a.n, s0 + i, a.pad_mode, a.pad);
      bad |= !isfinite(v);
      xw[i] = v * a.window[i];
    }
    __syncthreads();
    for (int k = threadIdx.x; k < F; k += blockDim.x) {
      double re = 0.0, im = 0.0;
      int idx = 0;
      for (int i = 0; i < N; ++i) {
        const double2 w = a.tw[idx];
        re = fma(xw[i], w.x, re);
        im = fma(xw[i], w.y, im);
        idx += k;
        if (idx >= N) idx -= N;
      }
      orow[k] = make_double2(re, im);
    }
  }
  if (bad) *a.status = B2L_STATUS_NOT_FINITE_SAMPLE;
}

struct F64InvArgs {
  const double2* D;         // [n_clips][n_frames_stored][F]
  long long d_clip_stride;  // in double2
  int n_clips, n_frames, n_fft, hop, start, out_len, log2m;
  const double* window;     // [n_fft], carries nothing else (1/n is applied here)
  const double2* tw;        // as in F64FwdArgs
  double* frames;           // scratch [n_clips][n_frames][n_fft]
  const double* inv_wss;    // [out_len]
  double* y;                // [n_clips][y_stride]
  long long y_stride;
  double2* zscratch;        // as in F64FwdArgs (n_fft/2 double2 per frame for the FFT, n_fft/2+1 for the DFT)
};

// One CTA per (frame, clip): irfft (scipy semantics: Im of DC / Nyquist ignored, 1/n scaling) times the window.
__global__ void istft64_frames_kernel(const F64InvArgs a) {
  extern __shared__ __align__(16) unsigned char smem64[];
  const long long item = blockIdx.x;
  const int clip = (int)(item / a.n_frames), frame = (int)(item % a.n_frames);
  const int N = a.n_fft, F = N / 2 + 1;
  const double2* X = a.D + (long long)clip * a.d_clip_stride + (long long)frame * F;
  double* out = a.frames + ((long long)clip * a.n_frames + frame) * N;
  if (a.log2m > 0) {
    const int M = N / 2;
    double2* z = a.zscratch ? a.zscratch + item * M : reinterpret_cast<double2*>(smem64);
    // Z[k] = E + i O with E = (X[k] + conj X[M-k]) / 2, O = conj(W_N^k) (X[k] - conj X[M-k]) / 2; the inverse
    // transform is conj(FFT(conj Z)) / M, so conj(Z) goes in (bit-reversed) and the result is conjugated.
    for (int k = threadIdx.x; k < M; k += blockDim.x) {
      double2 xa = X[k], xb = X[M - k];
      if (k == 0) { xa.y = 0.0; xb.y = 0.0; }
      const double er = 0.5 * (xa.x + xb.x), ei = 0.5 * (xa.y - xb.y);
      const double pr = 0.5 * (xa.x - xb.x), pi = 0.5 * (xa.y + xb.y);
      const double2 w = a.tw[k];                         // conj(w) * P
      const double orr = w.x * pr + w.y * pi, oi = w.x * pi - w.y * pr;
      z[bitrev_rt(k, a.log2m)] = make_double2(er - oi, -(ei + orr));   // conj(E + i O)
    }
    __syncthreads();
    fft64_inplace(z, a.log2m, a.tw);
    const double scale = 1.0 / (double)M;
    for (int e = threadIdx.x; e < M; e += blockDim.x) {
      out[2 * e] = z[e].x * scale * a.window[2 * e];
      out[2 * e + 1] = -z[e].y * scale * a.window[2 * e + 1];
    }
  } else {
    double2* xs = a.zscratch ? a.zscratch + item * F : reinterpret_cast<double2*>(smem64);
    for (int k = threadIdx.x; k < F; k += blockDim.x) xs[k] = X[k];
    __syncthreads();
    const bool even = (N % 2) == 0;
    const int kmax = even ? N / 2 - 1 : N / 2;            // bins with a distinct mirror image
    for (int i = threadIdx.x; i < N; i += blockDim.x) {
      double acc = xs[0].x;
      if (even) acc += (i & 1) ? -xs[N / 2].x : xs[N / 2].x;
      int idx = 0;
      for (int k = 1; k <= kmax; ++k) {
        idx += i;
        if (idx >= N) idx -= N;
        const double2 w = a.tw[idx];                       // exp(-2 pi i k i / N); need Re(X e^{+...}) = X.x w.x + X.y w.y
        acc += 2.0 * (xs[k].x * w.x + xs[k].y * w.y);
      }
      out[i] = acc / (double)N * a.window[i];
    }
  }
}

// Overlap-add of the parked frames in increasing frame order (librosa/core/spectrum.py:629-643) and the
// window-sum-square normalisation (:606-624).
__global__ void ola64_kernel(const F64InvArgs a) {
  const int clip = blockIdx.y;
  const double* fr = a.frames + (long long)clip * a.n_frames * a.n_fft;
  double* yc = a.y + (long long)clip * a.y_stride;
  for (long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x; o < a.out_len; o += (long long)gridDim.x * blockDim.x) {
    const long long u = o + a.start;
    long long f_hi = u / a.hop;
    if (f_hi > a.n_frames - 1) f_hi = a.n_frames - 1;
    long long f_lo = (u - a.n_fft + a.hop) / a.hop;       // smallest f with u - f*hop <= n_fft - 1
    if (u - a.n_fft + 1 <= 0) f_lo = 0;
    double acc = 0.0;
    for (long long f = f_lo; f <= f_hi; ++f) {
      const long long i = u - f * a.hop;
      if (i >= 0 && i < a.n_fft) acc += fr[f * a.n_fft + i];
    }
    yc[o] = acc * a.inv_wss[o];
  }
}

// |D|**power, elementwise (power == 2: re^2 + im^2 like np.abs(D)**2 up to one rounding)
__global__ void abs_pow64_kernel(const double2* __restrict__ D, long long n, double power, double* __restrict__ S) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const double m = hypot(D[i].x, D[i].y);
    S[i] = power == 1.0 ? m : (power == 2.0 ? m * m : pow(m, power));
  }
}

// mel[c][m][t] = sum_k W[m][k] S[c][t][k]; one warp per (clip, frame), lanes stride the band of every row.
__global__ void mel64_kernel(const double* __restrict__ S, const float* __restrict__ mel_w, const MelBand* __restrict__ band,
                             int n_mels, int F, int T, long long n_rows, double* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (warp >= n_rows) return;
  const long long clip = warp / T;
  const int t = (int)(warp % T);
  const double* row = S + warp * F;
  for (int m = 0; m < n_mels; ++m) {
    const MelBand b = band[m];
    double acc = 0.0;
    for (int i = lane; i < b.len; i += 32) acc = fma((double)mel_w[b.off + i], row[b.lo + i], acc);
    acc = warp_reduce(acc, [](double u, double v) { return u + v; });
    if (lane == 0) out[(clip * n_mels + m) * T + t] = acc;
  }
}

__device__ __forceinline__ unsigned long long double_to_key(double d) {
  unsigned long long u = (unsigned long long)__double_as_longlong(d);
  return (u & 0x8000000000000000ull) ? ~u : (u | 0x8000000000000000ull);
}
__device__ __forceinline__ double key_to_double(unsigned long long k) {
  unsigned long long u = (k & 0x8000000000000000ull) ? (k & 0x7fffffffffffffffull) : ~k;
  return __longlong_as_double((long long)u);
}

// 10 log10(max(amin, x)) - 10 log10(max(amin, ref)) and the per-clip maximum (librosa/core/spectrum.py:1866-1873)
__global__ void db64_kernel(const double* __restrict__ in, long long per_clip, double amin, double db_sub,
                            double* __restrict__ out, unsigned long long* __restrict__ clip_max) {
  const int clip = blockIdx.y;
  const double* src = in + (long long)clip * per_clip;
  double* dst = out + (long long)clip * per_clip;
  double m = -INFINITY;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < per_clip; i += (long long)gridDim.x * blockDim.x) {
    const double v = 10.0 * log10(MaxNan()(amin, src[i])) - db_sub;
    dst[i] = v;
    m = MaxNan()(m, v);
  }
  m = warp_reduce(m, MaxNan());
  // a NaN maximum (np.maximum keeps a NaN cell) is the all-ones key: no finite key exceeds it, key_to_double reads NaN
  if ((threadIdx.x & 31) == 0 && !(m == -INFINITY)) atomicMax(clip_max + clip, m != m ? ~0ull : double_to_key(m));
}
// np.maximum(log_spec, log_spec.max(per clip) - top_db) (:1875-1881)
__global__ void db64_clamp_kernel(double* __restrict__ x, long long per_clip, double top_db,
                                  const unsigned long long* __restrict__ clip_max) {
  const int clip = blockIdx.y;
  double* dst = x + (long long)clip * per_clip;
  const double floor_v = key_to_double(clip_max[clip]) - top_db;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < per_clip; i += (long long)gridDim.x * blockDim.x)
    dst[i] = MaxNan()(dst[i], floor_v);
}

// C[c][k][t] = sum_m dct[k][m] L[c][m][t]   (scipy.fft.dct along the mel axis as an explicit matrix, lifter folded in)
__global__ void dct64_kernel(const double* __restrict__ L, const double* __restrict__ dct, int n_mels, int n_mfcc, int T,
                             double* __restrict__ C) {
  extern __shared__ __align__(16) unsigned char smem64[];
  double* s_dct = reinterpret_cast<double*>(smem64);
  for (int i = threadIdx.x; i < n_mfcc * n_mels; i += blockDim.x) s_dct[i] = dct[i];
  __syncthreads();
  const int clip = blockIdx.y;
  const double* Lc = L + (long long)clip * n_mels * T;
  double* Cc = C + (long long)clip * n_mfcc * T;
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < T; t += gridDim.x * blockDim.x) {
    for (int k = 0; k < n_mfcc; ++k) {
      double acc = 0.0;
      for (int m = 0; m < n_mels; ++m) acc = fma(s_dct[k * n_mels + m], Lc[(long long)m * T + t], acc);
      Cc[(long long)k * T + t] = acc;
    }
  }
}

}  // namespace b2l
