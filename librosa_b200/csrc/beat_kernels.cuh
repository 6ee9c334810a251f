// beat_kernels.cuh — librosa.beat.beat_track's dynamic-programming tracker (librosa/beat.py:510-742) on the device.
// Included by rhythm_api.cu only.
//
//   beat_track_kernel<T, TC>  onset envelopes (T = float or double) -> dense beats, tracker intermediates and, for
//                         one clip, the compacted beat list.  TC is the DP's type: numba picks the float64 loop
//                         unless both the envelope and the frames per beat are float32
//   any_nonzero_kernel<T> np.any of a device envelope batch (beat_track's early return)
//   plp_select_kernel<C>  librosa.beat.plp's peak selection and phase normalisation of a Fourier tempogram, in place
//   plp_finish_kernel<T>  plp's np.clip(pulse, 0) and util.normalize(axis=-1), in place
//
// The tracker is discrete: one rounding difference moves a beat, so every step restates the reference's arithmetic
// (numba, no fast-math): explicit _rn intrinsics keep nvcc from contracting to FMA, and every transcendental comes
// from host tables built with libm (log(d), log(fpb) — logf for float32 envelopes — and the Gaussian windows).
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/b2l.h"
#include "numerics.cuh"

namespace b2l_beat {
using namespace b2l;

struct BeatArgs {
  const void* env;          // [clips][n]
  int n;
  int tv;                   // 1: one frames-per-beat per frame ([clips][n]); 0: one per clip ([clips][1])
  const double* fpb;        // frames per beat (integers >= 1)
  const double* logfpb;     // log(fpb): logf(float(fpb)) for a float DP
  const double* woff;       // index into wtab of w(0) for that fpb; w(d) = wtab[woff + d], |d| <= min(fpb, n-1)
  const double* wtab;       // exp(-0.5 * x * x), x = d * 32.0 / fpb
  const double* logd;       // log(d) for 1 <= d < n_logd
  double tightness;         // float32 tightness, widened
  int trim;
  void* localscore;         // [clips][n] T
  void* cumscore;           // [clips][n] TC
  int32_t* backlink;        // [clips][n]
  void* scratch;            // [clips][n] doubles: local maxima (TC), then the beat list
  uint8_t* beats;           // [clips][n]
  int units;                // compacted list of clip 0 when sparse != NULL: 0 frames, 1 samples (int64), 2 seconds
  void* sparse;
  long long* count;
  int hop_length;
  double sr;
};

// NumPy's pairwise summation (numpy/_core/src/umath/loops_utils.h.src) of f(0) .. f(n-1) in T, one thread.  The
// recursion splits at n/2 rounded down to a multiple of 8 until a block holds at most 128 elements; it is walked
// here with an explicit stack.
template <class T, class F>
__device__ T pairwise_sum(long long n, F f) {
  struct Frame { long long lo, n; int state; T left; };
  Frame st[48];
  int sp = 0;
  st[0] = {0, n, 0, T(0)};
  T ret = T(0);
  while (sp >= 0) {
    Frame& fr = st[sp];
    if (fr.n <= 128) {
      T res;
      if (fr.n < 8) {
        res = T(-0.0);
        for (long long i = 0; i < fr.n; ++i) res = add_rn(res, f(fr.lo + i));
      } else {
        T r[8];
        for (int j = 0; j < 8; ++j) r[j] = f(fr.lo + j);
        long long i = 8;
        for (; i < fr.n - (fr.n % 8); i += 8)
          for (int j = 0; j < 8; ++j) r[j] = add_rn(r[j], f(fr.lo + i + j));
        res = add_rn(add_rn(add_rn(r[0], r[1]), add_rn(r[2], r[3])), add_rn(add_rn(r[4], r[5]), add_rn(r[6], r[7])));
        for (; i < fr.n; ++i) res = add_rn(res, f(fr.lo + i));
      }
      ret = res;
      --sp;
    } else {
      long long n2 = fr.n / 2;
      n2 -= n2 % 8;
      if (fr.state == 0) {
        fr.state = 1;
        st[sp + 1] = {fr.lo, n2, 0, T(0)};
        ++sp;
        continue;
      }
      if (fr.state == 1) {
        fr.state = 2;
        fr.left = ret;
        st[sp + 1] = {fr.lo + n2, fr.n - n2, 0, T(0)};
        ++sp;
        continue;
      }
      ret = add_rn(fr.left, ret);
      --sp;
    }
  }
  return ret;
}

// round(fpb / 2) with Python's round-half-even, for integer fpb
__device__ __forceinline__ int half_even(int fpb) {
  const int k = fpb >> 1;
  return (fpb & 1) ? ((k & 1) ? k + 1 : k) : k;
}

// local_extremum (numerics.cuh) gives the same result, but its eagerly loaded neighbours change beat_track_kernel's code
template <class T>
__device__ __forceinline__ bool is_localmax(const T* x, int i, int n) {
  if (i == 0) return false;   // util.localmax pads with the edge value: x[0] > x[0] never holds
  return x[i] > x[i - 1] && (i == n - 1 ? x[i] >= x[i] : x[i] >= x[i + 1]);
}

struct Cand {
  double s;
  int loc;
};
// the reference scans loc downward and keeps the first strictly larger score: ties go to the larger loc.  Kept with
// its own butterfly below: warp_select (numerics.cuh), with this rule or a merge calling it, changes the kernel's code.
__device__ __forceinline__ Cand better(Cand a, Cand b) {
  if (b.loc < 0) return a;
  if (a.loc < 0) return b;
  if (b.s > a.s || (b.s == a.s && b.loc > a.loc)) return b;
  return a;
}

// One CTA per clip (blockDim a multiple of 32, at most 1024).
template <class T, class TC>
__global__ void __launch_bounds__(256) beat_track_kernel(BeatArgs a) {
  const long long clip = blockIdx.x;
  const int n = a.n, tid = threadIdx.x, nt = blockDim.x;
  const int lane = tid & 31, warp = tid >> 5, n_warps = nt >> 5;
  const T* env = (const T*)a.env + clip * n;
  T* ls = (T*)a.localscore + clip * n;
  TC* cum = (TC*)a.cumscore + clip * n;
  int32_t* back = a.backlink + clip * n;
  TC* lmax = (TC*)((double*)a.scratch + clip * n);
  uint8_t* beats = a.beats + clip * n;
  const long long prow = clip * (a.tv ? n : 1);

  __shared__ T s_denom;
  __shared__ double s_red[32];
  __shared__ int s_ired[32];
  __shared__ int s_count, s_tail, s_first;
  __shared__ TC s_med[2];

  // 1. __normalize_onsets: onsets / (std(ddof=1) + tiny), NumPy's pairwise sums in T; the mean and the variance
  //    are divided by the (integer) count in float64 and rounded to T, as np.true_divide by an intp does.
  if (tid == 0) {
    const T sum = pairwise_sum<T>(n, [&](long long i) { return env[i]; });
    const T mean = (T)((double)sum / (double)n);
    const T ss = pairwise_sum<T>(n, [&](long long i) {
      const T d = sub_rn(env[i], mean);
      return mul_rn(d, d);
    });
    const int dof = n - 1 > 0 ? n - 1 : 0;
    const T var = (T)((double)ss / (double)dof);
    s_denom = add_rn(sqrt_rn(var), tiny_of<T>());
    s_count = 0;
    s_first = n;
    s_med[0] = s_med[1] = TC(0);
  }
  __syncthreads();
  const T denom = s_denom;

  // 2. __beat_local_score: localscore[i] = sum over k ascending of window[k] * x[i + fpb - k], each term added in
  //    float64 and rounded to T; source frames j from min(n-1, i+fpb) down to max(1, i-fpb) (x[0] never counts).
  for (int i = tid; i < n; i += nt) {
    const long long pi = prow + (a.tv ? i : 0);
    const int fpb = (int)a.fpb[pi];
    const double* w = a.wtab + (long long)a.woff[pi];
    const int jhi = (int)min((long long)n - 1, (long long)i + fpb);
    const int jlo = max(1, i - fpb);
    T acc = T(0);
    for (int j = jhi; j >= jlo; --j) {
      const T x = env[j] / denom;
      acc = (T)__dadd_rn((double)acc, __dmul_rn(w[i - j], (double)x));
    }
    ls[i] = acc;
    beats[i] = 0;
  }
  __syncthreads();

  // 3. __beat_track_dp.  score_thresh = 0.01 * max(localscore) (numba's max: the first NaN wins); the first beat
  //    is pending until the first frame whose localscore is not below it.
  {
    double m = -INFINITY;
    bool nan = false;
    for (int i = tid; i < n; i += nt) {
      const double v = (double)ls[i];
      if (v != v) nan = true;
      else m = fmax(m, v);
    }
    m = warp_reduce(m, [](double u, double v) { return fmax(u, v); });
    nan = __any_sync(0xffffffffu, nan);
    if (lane == 0) s_red[warp] = nan ? NAN : m;
    __syncthreads();
    if (tid == 0) {
      double r = -INFINITY;
      for (int w = 0; w < n_warps; ++w) r = (s_red[w] != s_red[w] || r != r) ? NAN : fmax(r, s_red[w]);
      s_red[0] = __dmul_rn(0.01, r);
    }
    __syncthreads();
    const double thresh = s_red[0];
    int first = n;
    for (int i = tid; i < n; i += nt)
      if (!((double)ls[i] < thresh)) { first = i; break; }
    atomicMin(&s_first, first);
    __syncthreads();
  }
  const int first = s_first;
  // Frames i .. i + r - 1 (r = max(1, round(fpb/2))) read cumscore only before i, so each such block runs at once:
  // one warp per frame, lanes over the candidates i - r, i - r - 1, ... down to i - 2 fpb (and 0).  loc == i
  // (fpb == 1) is skipped: log(0) makes its score -inf or NaN, which never wins.
  for (int i0 = 0; i0 < n;) {
    int i1 = i0 + 1;
    while (i1 < n) {
      const int fpb = (int)a.fpb[prow + (a.tv ? i1 : 0)];
      if (max(half_even(fpb), 1) < i1 - i0 + 1) break;
      ++i1;
    }
    for (int i = i0 + warp; i < i1; i += n_warps) {
      const long long pi = prow + (a.tv ? i : 0);
      const int fpb = (int)a.fpb[pi];
      const double lf = a.logfpb[pi];
      const int hi = i - max(half_even(fpb), 1);
      const long long lo_ex = (long long)i - 2LL * fpb - 1;
      const int lo = (int)(lo_ex + 1 > 0 ? lo_ex + 1 : 0);
      Cand best = {-INFINITY, -1};
      for (int loc = hi - lane; loc >= lo; loc -= 32) {
        const double d = __dsub_rn(a.logd[i - loc], lf);
        const double s = __dsub_rn((double)cum[loc], __dmul_rn(a.tightness, __dmul_rn(d, d)));
        if (s > best.s) best = {s, loc};
      }
      for (int o = 16; o; o >>= 1) {
        Cand other = {__shfl_xor_sync(0xffffffffu, best.s, o), __shfl_xor_sync(0xffffffffu, best.loc, o)};
        best = better(best, other);
      }
      if (lane == 0) {
        const T si = ls[i];
        cum[i] = best.loc >= 0 ? (TC)__dadd_rn((double)si, best.s) : (TC)si;
        back[i] = i < first ? -1 : best.loc;
      }
    }
    __syncthreads();
    i0 = i1;
  }

  // 4. __last_beat: the median of cumscore over its local maxima (np.ma.median: the two middle values summed in TC
  //    and halved), threshold = 0.5 * median in TC; the last local maximum at or above it, else n - 1.
  for (int i = tid; i < n; i += nt)
    if (is_localmax(cum, i, n)) lmax[atomicAdd(&s_count, 1)] = cum[i];
  __syncthreads();
  const int m = s_count;
  if (m > 0) {
    const int k1 = (m - 1) / 2, k2 = m / 2;
    for (int u = tid; u < m; u += nt) {
      const TC v = lmax[u];
      int less = 0, le = 0;
      for (int q = 0; q < m; ++q) {
        const TC w = lmax[q];
        less += w < v;
        le += w <= v;
      }
      if (less <= k1 && k1 < le) s_med[0] = v;
      if (less <= k2 && k2 < le) s_med[1] = v;
    }
  }
  __syncthreads();
  {
    int tail = -1;
    if (m > 0) {
      const TC med = (m & 1) ? s_med[0] : mul_rn(add_rn(s_med[0], s_med[1]), TC(0.5));
      const TC thr = mul_rn(TC(0.5), med);
      for (int i = tid; i < n; i += nt)
        if (is_localmax(cum, i, n) && cum[i] >= thr) tail = i;
    }
    tail = warp_reduce(tail, [](int u, int v) { return max(u, v); });
    if (lane == 0) s_ired[warp] = tail;
    __syncthreads();
    if (tid == 0) {
      int t = -1;
      for (int w = 0; w < n_warps; ++w) t = max(t, s_ired[w]);
      s_tail = t >= 0 ? t : n - 1;
    }
    __syncthreads();
  }

  // 5. __dp_backtrack, then 6. __trim_beats, one thread: the beat list (descending) goes to the scratch row.
  if (tid == 0) {
    int* list = (int*)lmax;
    int nb = 0;
    for (int t = s_tail; t >= 0; t = back[t]) {
      beats[t] = 1;
      list[nb++] = t;
    }
    double thr = 0.0;
    if (a.trim) {
      // np.convolve(localscore[beats], np.hanning(5))[2 : n + 2]: full convolution outputs p = 2 .. 1 + cnt,
      // cnt = min(n, nb + 2); hanning(5) is exactly {0, 0.5, 1, 0.5, 0}.  Numba's mean: a plain float64 sum.
      const double hw[5] = {0.0, 0.5, 1.0, 0.5, 0.0};
      const int cnt = min(n, nb + 2);
      double ss = 0.0;
      for (int p = 2; p < 2 + cnt; ++p) {
        double c = 0.0;
        for (int q = max(0, p - 4); q <= min(nb - 1, p); ++q)
          c = __dadd_rn(c, __dmul_rn((double)ls[list[nb - 1 - q]], hw[p - q]));
        ss = __dadd_rn(ss, __dmul_rn(c, c));
      }
      thr = __dmul_rn(0.5, __dsqrt_rn(ss / (double)cnt));
    }
    // the reference's loops are unbounded; an all-zero clip clears every frame here
    int lo = 0;
    while (lo < n && (double)ls[lo] <= thr) beats[lo++] = 0;
    int hi = n - 1;
    while (hi >= 0 && (double)ls[hi] <= thr) beats[hi--] = 0;
    if (a.sparse && clip == 0) {
      long long k = 0;
      for (int q = nb - 1; q >= 0; --q) {
        const int t = list[q];
        if (!beats[t]) continue;
        if (a.units == 0) ((long long*)a.sparse)[k++] = t;
        else if (a.units == 1) ((long long*)a.sparse)[k++] = (long long)t * a.hop_length;
        else ((double*)a.sparse)[k++] = (double)((long long)t * a.hop_length) / a.sr;
      }
      *a.count = k;
    }
  }
}

// flag = 1 when any element of x [n] is not zero (np.any: NaN counts)
template <class T>
__global__ void any_nonzero_kernel(const T* __restrict__ x, long long n, int* __restrict__ flag) {
  bool hit = false;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    hit |= x[i] != T(0);
  if (__syncthreads_or(hit) && threadIdx.x == 0) atomicOr(flag, 1);
}

// ---- librosa.beat.plp (beat.py:320-507) -------------------------------------------------------------------------
// np.max with a NaN: a canonical NaN here, not MaxNan's NaN operand (numerics.cuh), which changes plp_select's code
template <class R> __device__ __forceinline__ R rmax_nan(R a, R b) { return (a != a || b != b) ? (R)NAN : (a > b ? a : b); }

// One warp per (row, frame) of a Fourier tempogram X [rows * frames][n_bins] (bins contiguous, C = float2 or
// double2):  bins with keep[b] == 0 are zeroed (the tempo range); ftmag = log1p(1e6 |X|) in the data's precision,
// plus logprior[b] added in float64 and rounded back (NumPy's in-place +=); bins whose ftmag is below the frame's
// maximum are zeroed (ties survive; a NaN maximum zeroes nothing).  Then X /= sqrt_tiny + |max(X)| with NumPy's
// complex max (lexicographic: real part, then imaginary part) over all bins, zeroed ones included, and the
// complex-by-real division re * (1/c), im * (1/c).
template <class C>
__global__ void plp_select_kernel(C* __restrict__ X, long long n_frames, int n_bins, const double* __restrict__ keep,
                                  const double* __restrict__ logprior, double sqrt_tiny) {
  using R = decltype(X->x);
  const long long f = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (f >= n_frames) return;
  C* row = X + f * n_bins;
  R peak = (R)-INFINITY;
  for (int b = lane; b < n_bins; b += 32) {
    C z = row[b];
    if (keep[b] == 0.0) z.x = z.y = (R)0;
    R m = log1p_((R)1e6 * cabs_(z));
    if (logprior) m = (R)((double)m + logprior[b]);
    peak = rmax_nan(peak, m);
  }
  peak = warp_reduce(peak, [](R u, R v) { return rmax_nan(u, v); });
  R mre = (R)-INFINITY, mim = (R)-INFINITY;
  bool first = true;
  for (int b = lane; b < n_bins; b += 32) {
    C z = row[b];
    if (keep[b] == 0.0) z.x = z.y = (R)0;
    R m = log1p_((R)1e6 * cabs_(z));
    if (logprior) m = (R)((double)m + logprior[b]);
    if (m < peak) z.x = z.y = (R)0;
    row[b] = z;
    if (first || z.x > mre || (z.x == mre && z.y > mim)) { mre = z.x; mim = z.y; }
    first = false;
  }
  // not warp_select (numerics.cuh): with this rule as its merge it changes the kernel's code
  for (int o = 16; o; o >>= 1) {
    const R ore = (R)__shfl_xor_sync(0xffffffffu, mre, o), oim = (R)__shfl_xor_sync(0xffffffffu, mim, o);
    if (ore > mre || (ore == mre && oim > mim)) { mre = ore; mim = oim; }
  }
  __syncwarp();
  const R c = (R)sqrt_tiny + cabs_(C{mre, mim});
  const R r = (R)1 / c;
  for (int b = lane; b < n_bins; b += 32) {
    C z = row[b];
    z.x = mul_rn(z.x, r);
    z.y = mul_rn(z.y, r);
    row[b] = z;
  }
}

// One CTA per row of the pulse x [rows][n]: x = max(x, 0) (NaN stays), then x / max|x| (1 when below tiny), as
// util.normalize(norm=inf, axis=-1).  A non-finite value sets B2L_STATUS_NOT_FINITE_VALUE (normalize's "Input must
// be finite").
template <class T>
__global__ void plp_finish_kernel(T* __restrict__ x, int n, int* __restrict__ status) {
  __shared__ T s_max[32];
  __shared__ int s_bad;
  T* row = x + (long long)blockIdx.x * n;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) s_bad = 0;
  T m = T(0);
  bool bad = false;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    T v = row[i];
    v = v < T(0) ? T(0) : v;
    row[i] = v;
    if (!isfinite(v)) bad = true;
    else m = v > m ? v : m;
  }
  // not warp_reduce (numerics.cuh): it changes the float instance's code
  for (int o = 16; o; o >>= 1) {
    const T other = __shfl_xor_sync(0xffffffffu, m, o);
    m = other > m ? other : m;
  }
  if (lane == 0) s_max[warp] = m;
  if (bad) atomicOr(&s_bad, 1);
  __syncthreads();
  if (threadIdx.x == 0) {
    T r = T(0);
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) r = s_max[w] > r ? s_max[w] : r;
    s_max[0] = r < tiny_of<T>() ? T(1) : r;
    if (s_bad) atomicOr(status, B2L_STATUS_NOT_FINITE_VALUE);
  }
  __syncthreads();
  const T len = s_max[0];
  for (int i = threadIdx.x; i < n; i += blockDim.x) row[i] = row[i] / len;
}

}  // namespace b2l_beat
