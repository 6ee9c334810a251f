// chroma_kernels.cuh — the constant-Q chroma features: librosa.feature.chroma_cqt / chroma_vqt / chroma_cens /
// tonnetz (librosa/feature/spectral.py:1296-1839) after the CQT.
//
//   chroma_fold_kernel     |C| (or a real C / chroma), the cq_to_chroma map, the threshold and util.normalize, then
//                          nothing, the CENS L1 + quantisation (+ the final normalisation), or the tonnetz L1 +
//                          6 x n_chroma projection
//   chroma_smooth_kernel   CENS's scipy.ndimage.convolve along frames (mode="constant") and the final normalisation
//
// A fold block serves one clip and `tf` consecutive frames.  It stages the tile's magnitudes in shared memory with
// reads along the contiguous axis (bins for "ft" input, frames for "c" input), so the input is read once, and the
// map's per-row (column, weight) lists next to it when they fit (else they are read through L1).  Chroma values are
// accumulated in the result precision; util.normalize follows numpy: the column length in double from |x| as
// float64, numpy's fast paths for the exponents 1, 2, 0.5, -1 and 0, lengths below tiny(dtype) replaced by 1, and
// one rounding of the float64 quotient into the result dtype.  Results are C-ordered [clip][rows][T].
#pragma once
#include <stdint.h>

#include "numerics.cuh"

namespace b2l_chroma {
using namespace b2l;

constexpr int kThreads = 256;

enum Norm { kNone = 0, kInf = 1, kNegInf = 2, kZero = 3, kP = 4 };   // enum b2l_chroma_norm
enum Epilogue { kPlain = 0, kCens = 1, kTonnetz = 2 };              // enum b2l_chroma_epilogue

struct FoldArgs {
  const void* in;          // [clip][T][n_bins] ("ft") or [clip][n_bins][T] ("c")
  int ft;                  // input layout
  int n_bins, n_chroma;
  long long T;
  int tf;                  // frames per block
  const int* row_ptr;      // [n_chroma + 1] CSR of the map
  const int* cols;
  const double* weights;
  int nnz;
  int staged_map;          // map lists copied to shared memory
  int norm;                // chroma_cqt's normalisation
  double norm_p;
  int has_threshold;
  double threshold;
  int epilogue;
  int post_norm;           // CENS: after quantisation (kNone: the quantised values)
  double post_p;
  const double* phi;       // [6][n_chroma] tonnetz
  long long clip0;
  void* out;               // [clip][n_chroma][T] chroma dtype, or [clip][6][T] double (tonnetz)
  int* status;
};

// numpy's array ** scalar: the fast paths of its scalar power, else pow
__device__ __forceinline__ double np_pow(double x, double e) {
  if (e == 1.0) return x;
  if (e == 2.0) return __dmul_rn(x, x);
  if (e == 0.5) return sqrt(x);
  if (e == -1.0) return 1.0 / x;
  if (e == 0.0) return 1.0;
  return pow(x, e);
}

// util.normalize's length of one column v[0], v[stride], ... (n values), with the tiny rule of the dtype T
template <class T>
__device__ double column_length(const T* v, int stride, int n, int kind, double p) {
  double len = 0.0;
  if (kind == kInf || kind == kNegInf) {
    len = fabs((double)v[0]);
    for (int i = 1; i < n; ++i) {
      const double m = fabs((double)v[i * stride]);
      len = kind == kInf ? fmax(len, m) : fmin(len, m);
    }
  } else if (kind == kZero) {
    for (int i = 0; i < n; ++i) len += fabs((double)v[i * stride]) > 0.0 ? 1.0 : 0.0;
  } else {
    for (int i = 0; i < n; ++i) len = __dadd_rn(len, np_pow(fabs((double)v[i * stride]), p));
    len = np_pow(len, 1.0 / p);
  }
  return len < (double)tiny_of<T>() ? 1.0 : len;
}

template <class In>
struct Mag;
// |x| of complex64, correctly rounded through double: not cqt's np_abs (NumPy's x86 loop) nor plp's cabs_ (hypotf)
template <>
struct Mag<float2> {
  typedef float R;
  static __device__ __forceinline__ float get(float2 v) {
    const double re = v.x, im = v.y;
    return __double2float_rn(sqrt(__dadd_rn(__dmul_rn(re, re), __dmul_rn(im, im))));
  }
};
template <>
struct Mag<float> {
  typedef float R;
  static __device__ __forceinline__ float get(float v) { return v; }
};
template <>
struct Mag<double> {
  typedef double R;
  static __device__ __forceinline__ double get(double v) { return v; }
};

// Normalises the tile's columns s[f * n + r] (r < n) in place with one thread per frame (f < tf), then syncs.
template <class T>
__device__ void normalize_tile(T* s, double* s_len, int tf, int n, int kind, double p) {
  if (kind == kNone) return;
  for (int f = threadIdx.x; f < tf; f += kThreads) s_len[f] = column_length(s + f * n, 1, n, kind, p);
  __syncthreads();
  for (int i = threadIdx.x; i < tf * n; i += kThreads) s[i] = (T)((double)s[i] / s_len[i / n]);
  __syncthreads();
}

template <class In, class Out>
__global__ void __launch_bounds__(kThreads) chroma_fold_kernel(const FoldArgs a) {
  typedef typename Mag<In>::R R;
  extern __shared__ __align__(16) unsigned char smem[];
  const int nb = a.n_bins, nc = a.n_chroma, tf = a.tf;
  // fold_smem_bytes (chroma_api.cu) sizes this layout: doubles first, then the chroma and magnitude tiles (each
  // rounded up to 8 bytes), then the map's integers
  double* s_len = reinterpret_cast<double*>(smem);                  // [tf]
  double* s_w = s_len + tf;                                          // [nnz] (staged map)
  Out* s_c = reinterpret_cast<Out*>(s_w + (a.staged_map ? a.nnz : 0));   // [tf][nc]
  R* s_x = reinterpret_cast<R*>(s_c + (tf * nc + 1) / 2 * 2);        // [tf][nb]
  int* s_ptr = reinterpret_cast<int*>(s_x + ((size_t)tf * nb + 1) / 2 * 2);   // [nc + 1] (staged map)
  int* s_col = s_ptr + nc + 1;                                       // [nnz]
  __shared__ int s_bad;

  const long long clip = a.clip0 + blockIdx.y;
  const long long t0 = (long long)blockIdx.x * tf;
  const int nf = (int)min((long long)tf, a.T - t0);
  const In* in = reinterpret_cast<const In*>(a.in);
  if (threadIdx.x == 0) s_bad = 0;
  if (a.ft) {   // the tile is one contiguous run of nf * nb values
    const In* src = in + (clip * a.T + t0) * nb;
    for (int i = threadIdx.x; i < nf * nb; i += kThreads) s_x[i] = Mag<In>::get(__ldg(src + i));
  } else {      // nb rows of nf contiguous frames
    const In* src = in + clip * nb * a.T + t0;
    for (int i = threadIdx.x; i < nf * nb; i += kThreads) {
      const int b = i / nf, f = i - b * nf;
      s_x[f * nb + b] = Mag<In>::get(__ldg(src + (long long)b * a.T + f));
    }
  }
  const int* ptr = a.row_ptr;
  const int* col = a.cols;
  const double* w = a.weights;
  if (a.staged_map) {
    for (int i = threadIdx.x; i <= nc; i += kThreads) s_ptr[i] = __ldg(a.row_ptr + i);
    for (int i = threadIdx.x; i < a.nnz; i += kThreads) {
      s_col[i] = __ldg(a.cols + i);
      s_w[i] = __ldg(a.weights + i);
    }
    ptr = s_ptr;
    col = s_col;
    w = s_w;
  }
  __syncthreads();

  // the map, then the threshold; a non-finite value is what util.normalize refuses
  bool bad = false;
  for (int i = threadIdx.x; i < nf * nc; i += kThreads) {
    const int f = i / nc, r = i - f * nc;
    const R* x = s_x + f * nb;
    Out acc = Out(0);
    for (int k = ptr[r]; k < ptr[r + 1]; ++k) acc += (Out)w[k] * (Out)x[col[k]];
    if (a.has_threshold && acc < (Out)a.threshold) acc = Out(0);
    bad |= !isfinite(acc);
    s_c[i] = acc;
  }
  if (bad) atomicOr(&s_bad, 1);
  __syncthreads();
  normalize_tile(s_c, s_len, nf, nc, a.norm, a.norm_p);

  if (a.epilogue == kTonnetz) {
    bad = false;   // the L1 normalisation checks the normalised chroma again
    for (int i = threadIdx.x; i < nf * nc; i += kThreads) bad |= !isfinite(s_c[i]);
    if (bad) atomicOr(&s_bad, 1);
    normalize_tile(s_c, s_len, nf, nc, kP, 1.0);
    double* out = reinterpret_cast<double*>(a.out) + clip * 6 * a.T + t0;
    for (int i = threadIdx.x; i < 6 * nf; i += kThreads) {
      const int p = i / nf, f = i - p * nf;
      double acc = 0.0;
      for (int r = 0; r < nc; ++r) acc += __ldg(a.phi + p * nc + r) * (double)s_c[f * nc + r];
      out[(long long)p * a.T + f] = acc;
    }
  } else {
    if (a.epilogue == kCens) {   // L1, the "log-like" quantisation, then the final normalisation (if fused)
      normalize_tile(s_c, s_len, nf, nc, kP, 1.0);
      for (int i = threadIdx.x; i < nf * nc; i += kThreads) {
        const Out x = s_c[i];
        Out q = Out(0);
        q += x > (Out)0.4 ? Out(0.25) : Out(0);
        q += x > (Out)0.2 ? Out(0.25) : Out(0);
        q += x > (Out)0.1 ? Out(0.25) : Out(0);
        q += x > (Out)0.05 ? Out(0.25) : Out(0);
        s_c[i] = q;
      }
      __syncthreads();
      normalize_tile(s_c, s_len, nf, nc, a.post_norm, a.post_p);
    }
    Out* out = reinterpret_cast<Out*>(a.out) + clip * nc * a.T + t0;
    for (int i = threadIdx.x; i < nf * nc; i += kThreads) {
      const int r = i / nf, f = i - r * nf;
      out[(long long)r * a.T + f] = s_c[f * nc + r];
    }
  }
  if (threadIdx.x == 0 && s_bad) atomicOr(a.status, B2L_STATUS_NOT_FINITE_VALUE);
}

struct SmoothArgs {
  const void* in;          // [clip][n_chroma][T] quantised chroma
  int n_chroma;
  long long T;
  int ts;                  // frames per block
  int reach;               // taps reach from t - reach to t - reach + L - 1
  int span;                // staged frames per row: ts + L - 1, or 0 (read through L1)
  const int* tap_off;      // [n_taps] ascending positions j of the flipped window with |w| > DBL_EPSILON
  const double* tap_w;     // their weights
  int n_taps;
  int norm;
  double norm_p;
  long long clip0;
  void* out;               // [clip][n_chroma][T]
};

// y[t] = sum_j wf[j] * x[t - reach + j] over the kept taps in ascending j (wf: the window reversed, reach:
// L - 1 - L // 2), accumulated in double with a separate multiply and add per tap and rounded once: ndimage's
// correlate with the flipped window; frames outside the clip are zero (mode="constant").  Then util.normalize.
template <class T>
__global__ void __launch_bounds__(kThreads) chroma_smooth_kernel(const SmoothArgs a) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int nc = a.n_chroma, ts = a.ts;
  double* s_len = reinterpret_cast<double*>(smem);   // [ts]
  T* s_o = reinterpret_cast<T*>(s_len + ts);          // [ts][nc]
  T* s_x = s_o + ts * nc;                             // [nc][span] (ts * nc is even)
  const long long clip = a.clip0 + blockIdx.y;
  const long long t0 = (long long)blockIdx.x * ts;
  const int nf = (int)min((long long)ts, a.T - t0);
  const T* x = reinterpret_cast<const T*>(a.in) + clip * nc * a.T;
  const long long first = t0 - a.reach;   // frame of s_x[.][0]
  if (a.span) {
    for (int i = threadIdx.x; i < nc * a.span; i += kThreads) {
      const int r = i / a.span;
      const long long t = first + (i - r * a.span);
      s_x[i] = (t >= 0 && t < a.T) ? __ldg(x + r * a.T + t) : T(0);
    }
    __syncthreads();
  }
  for (int i = threadIdx.x; i < nf * nc; i += kThreads) {
    const int r = i / nf, f = i - r * nf;
    double acc = 0.0;
    for (int k = 0; k < a.n_taps; ++k) {
      const int j = __ldg(a.tap_off + k);
      const long long t = first + f + j;
      if (t < 0 || t >= a.T) continue;
      const double v = a.span ? (double)s_x[r * a.span + f + j] : (double)__ldg(x + r * a.T + t);
      acc = __dadd_rn(acc, __dmul_rn(__ldg(a.tap_w + k), v));
    }
    s_o[f * nc + r] = (T)acc;
  }
  __syncthreads();
  normalize_tile(s_o, s_len, nf, nc, a.norm, a.norm_p);
  T* out = reinterpret_cast<T*>(a.out) + clip * nc * a.T + t0;
  for (int i = threadIdx.x; i < nf * nc; i += kThreads) {
    const int r = i / nf, f = i - r * nf;
    out[(long long)r * a.T + f] = s_o[f * nc + r];
  }
}

}  // namespace b2l_chroma
