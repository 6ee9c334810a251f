// onset_kernels.cuh — librosa.onset.onset_detect's normaliser, librosa.util.peak_pick and librosa.onset.onset_backtrack
// (librosa/onset.py:31-214 and :370-441, librosa/util/utils.py:1188-1496, librosa/util/matching.py:215-390) on the
// device.  Included by rhythm_api.cu only.
//
//   onset_normalize_kernel<T>  one CTA per row: (x - min x) / (max(x - min x) + tiny) in T, and the call's verdict
//                              flags (some element nonzero, some element not finite) over the whole batch
//   peak_pick_kernel<T, M>     one CTA per row: the picks of the greedy or dynamic-programming peak picker as a dense
//                              bool row and / or the compacted list of one row, converted to the requested units
//   onset_backtrack_kernel<T>  one CTA: each event matched to the last local minimum of an energy row at or before it
//
// The picks are discrete decisions, so the candidate tests restate the reference's numba arithmetic: np.mean over a
// window is a left-to-right sum in T divided by the element count in float64 and compared with x[n] in float64;
// np.cumsum is sequential in T; np.max returns NaN as soon as it meets one.  Explicit _rn intrinsics keep nvcc from
// contracting anything into an FMA.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/b2l.h"
#include "numerics.cuh"

namespace b2l_onset {
using namespace b2l;

// verdict flags (word 0 of the flags pair; word 1 is the pick count)
constexpr int kNonzero = 1, kNonfinite = 2;
constexpr int kGreedy = 0, kDpCount = 1, kDpValue = 2;
constexpr int kChunk = 8192;              // frames per candidate bitmask in shared memory
constexpr int kWords = kChunk / 32;

// One CTA per row of x [rows][n].  With out != NULL the row is normalised like onset_detect(normalize=True):
// x - min(x) (NaN wins), divided by max of that difference (NaN wins) + tiny, every step in T.  flags[0] gets
// kNonzero when an element of the (normalised) batch is not zero (np.any: NaN counts) and kNonfinite when one is
// not finite.
template <class T>
__global__ void onset_normalize_kernel(const T* __restrict__ x, int n, T tiny, T* __restrict__ out,
                                       long long* __restrict__ flags) {
  __shared__ T s_red[32];
  const T* row = x + (long long)blockIdx.x * n;
  T mn = T(0), scale = T(1);
  if (out) {
    T v = row[0];
    for (long long i = threadIdx.x; i < n; i += blockDim.x) v = MinNan()(v, row[i]);
    mn = block_reduce(v, MinNan(), s_red);
    T m = sub_rn(row[0], mn);
    for (long long i = threadIdx.x; i < n; i += blockDim.x) m = MaxNan()(m, sub_rn(row[i], mn));
    scale = add_rn(block_reduce(m, MaxNan(), s_red), tiny);
  }
  int f = 0;
  for (long long i = threadIdx.x; i < n; i += blockDim.x) {
    T v = row[i];
    if (out) {
      v = div_rn(sub_rn(v, mn), scale);
      out[(long long)blockIdx.x * n + i] = v;
    }
    if (v != T(0)) f |= kNonzero;
    if (!finite_(v)) f |= kNonfinite;
  }
  f = (__syncthreads_or(f & kNonzero) ? kNonzero : 0) | (__syncthreads_or(f & kNonfinite) ? kNonfinite : 0);
  if (threadIdx.x == 0 && f) atomicOr((int*)flags, f);
}

struct PeakArgs {
  const void* x;            // [rows][n], T
  int n;
  long long pre_max, post_max, pre_avg, post_avg, wait;   // clamped to [0, n] (post_* >= 1)
  double delta;
  const long long* flags;   // NULL, or the verdict of onset_normalize_kernel: picks only when nonzero and finite
  uint8_t* dense;           // [rows][n] or NULL
  void* sparse;             // the list of row 0 (n entries) or NULL: int64 frames / samples, or float64 seconds
  long long* count;         // entries written to sparse
  int units;                // 0 frames, 1 samples, 2 seconds
  int hop_length;
  double sr;
  double* scratch;          // dynamic programming: [rows][2 (n + 1)] doubles (cumsum, values)
  uint8_t* marks;           // dynamic programming: [rows][n] (bit 0 candidate, bit 1 taken, bit 2 picked)
};

// np.max(x[max(0, i - pre_max) : min(i + post_max, n)]) with numba's NaN rule
template <class T>
__device__ __forceinline__ T window_max(const T* row, long long i, const PeakArgs& a) {
  const long long lo = i - a.pre_max > 0 ? i - a.pre_max : 0, hi = i + a.post_max < a.n ? i + a.post_max : a.n;
  T m = row[lo];
  if (m != m) return m;
  for (long long j = lo + 1; j < hi; ++j) {
    const T v = row[j];
    if (v != v) return v;
    if (v > m) m = v;
  }
  return m;
}

// greedy candidate: x[i] == max of its window and x[i] >= np.mean(x[max(0, i - pre_avg) : min(i + post_avg, n)]) + delta
template <class T>
__device__ bool greedy_candidate(const T* row, long long i, const PeakArgs& a) {
  const T xi = row[i];
  if (!(xi == window_max(row, i, a))) return false;
  const long long lo = i - a.pre_avg > 0 ? i - a.pre_avg : 0, hi = i + a.post_avg < a.n ? i + a.post_avg : a.n;
  T s = T(0);
  for (long long j = lo; j < hi; ++j) s = add_rn(s, row[j]);
  const double avg = __ddiv_rn((double)s, (double)(hi - lo));
  return (double)xi >= __dadd_rn(avg, a.delta);
}

// dynamic-programming candidate: not (x[i] < max), and x[i] >= the cumsum average + delta
template <class T>
__device__ bool dp_candidate(const T* row, const double* cum, long long i, const PeakArgs& a) {
  const T xi = row[i];
  if (xi < window_max(row, i, a)) return false;
  const long long lo = i - a.pre_avg > 0 ? i - a.pre_avg : 0, hi = i + a.post_avg < a.n ? i + a.post_avg : a.n;
  double avg;
  if (lo == 0) avg = __ddiv_rn(cum[hi - 1], (double)hi);
  else avg = __ddiv_rn((double)sub_rn((T)cum[hi - 1], (T)cum[lo - 1]), (double)(hi - lo));
  return (double)xi >= __dadd_rn(avg, a.delta);
}

__device__ __forceinline__ void put_unit(const PeakArgs& a, long long k, long long t) {
  if (a.units == 0) ((long long*)a.sparse)[k] = t;
  else if (a.units == 1) ((long long*)a.sparse)[k] = t * a.hop_length;
  else ((double*)a.sparse)[k] = (double)(t * a.hop_length) / a.sr;
}

template <class T, int METHOD>
__global__ void __launch_bounds__(256) peak_pick_kernel(PeakArgs a) {
  __shared__ unsigned s_cand[kWords], s_pick[kWords];
  const long long rowi = blockIdx.x;
  const int n = a.n, lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const T* row = (const T*)a.x + rowi * n;
  uint8_t* dense = a.dense ? a.dense + rowi * n : nullptr;
  const bool list = a.sparse && rowi == 0;
  bool pass = true;
  if (a.flags) {
    const int f = (int)*a.flags;
    pass = (f & kNonzero) && !(f & kNonfinite);
  }
  if (!pass) {
    if (dense)
      for (long long i = threadIdx.x; i < n; i += blockDim.x) dense[i] = 0;
    if (list && threadIdx.x == 0) *a.count = 0;
    return;
  }
  if (METHOD == kGreedy) {
    // candidates of one chunk as a bitmask (one ballot per 32 frames), then warp 0 walks it: the next pick is the
    // first candidate at or after last + wait + 1
    long long next = 0, k = 0;   // warp 0's state
    for (long long cs = 0; cs < n; cs += kChunk) {
      const long long ce = cs + kChunk < n ? cs + kChunk : n;
      const int words = (int)((ce - cs + 31) >> 5);
      for (int w = warp; w < words; w += nw) {
        const long long i = cs + 32LL * w + lane;
        const bool c = i < ce && greedy_candidate(row, i, a);
        const unsigned b = __ballot_sync(0xffffffffu, c);
        if (lane == 0) { s_cand[w] = b; s_pick[w] = 0; }
      }
      __syncthreads();
      if (warp == 0) {
        long long pos = next;
        while (pos < ce) {
          const int wi = (int)((pos - cs) >> 5);
          const int my = wi + lane;
          unsigned word = my < words ? s_cand[my] : 0u;
          if (lane == 0) word &= ~0u << ((pos - cs) & 31);
          const unsigned ball = __ballot_sync(0xffffffffu, word != 0);
          if (!ball) {   // no candidate in these 32 words: on to the next 32, but never past the chunk
            pos = min(cs + 32LL * (wi + 32), ce);
            continue;
          }
          const int l = __ffs(ball) - 1;
          const unsigned wl = __shfl_sync(0xffffffffu, word, l);
          const long long p = cs + 32LL * (wi + l) + (__ffs(wl) - 1);
          if (lane == 0) {
            s_pick[(p - cs) >> 5] |= 1u << ((p - cs) & 31);
            if (list) put_unit(a, k, p);
          }
          ++k;
          pos = p + a.wait + 1;
        }
        next = pos;   // past ce only by a wait, which carries into the next chunk
      }
      __syncthreads();
      if (dense)
        for (long long i = cs + threadIdx.x; i < ce; i += blockDim.x)
          dense[i] = (s_pick[(i - cs) >> 5] >> ((i - cs) & 31)) & 1u;
      __syncthreads();
    }
    if (list && threadIdx.x == 0) *a.count = k;
  } else {
    double* cum = a.scratch + rowi * 2 * (n + 1LL);
    double* values = cum + (n + 1LL);
    uint8_t* marks = a.marks + rowi * n;
    if (threadIdx.x == 0) {   // np.cumsum: sequential in T
      T c = T(0);
      for (long long i = 0; i < n; ++i) {
        c = add_rn(c, row[i]);
        cum[i] = (double)c;
      }
    }
    __syncthreads();
    for (long long i = threadIdx.x; i < n; i += blockDim.x) marks[i] = dp_candidate(row, cum, i, a) ? 1 : 0;
    __syncthreads();
    if (threadIdx.x == 0) {
      // backward DP in float64: take frame i when it is a candidate and values[next] + v > values[i + 1]
      values[n] = 0.0;
      for (long long i = n - 1; i >= 0; --i) {
        const double skip = values[i + 1];
        values[i] = skip;
        if (marks[i] & 1) {
          const long long nx = i + a.wait + 1 < n ? i + a.wait + 1 : n;
          const double v = METHOD == kDpCount ? 1.0 : (double)row[i];
          const double take = __dadd_rn(values[nx], v);
          if (take > skip) {
            values[i] = take;
            marks[i] |= 2;
          }
        }
      }
      // follow the pointers from frame 0: the taken frames on the chain are the picks
      long long k = 0;
      for (long long i = 0; i < n;) {
        if (marks[i] & 2) {
          marks[i] |= 4;
          if (list) put_unit(a, k, i);
          ++k;
          i = i + a.wait + 1 < n ? i + a.wait + 1 : n;
        } else {
          ++i;
        }
      }
      if (list) *a.count = k;
    }
    __syncthreads();
    if (dense)
      for (long long i = threadIdx.x; i < n; i += blockDim.x) dense[i] = (marks[i] >> 2) & 1;
  }
}

// One CTA.  energy [n] (T): a minimum is a frame 1 <= i <= n - 2 with e[i] <= e[i-1] and e[i] < e[i+1]; frame 0
// always counts.  last[i] = the last minimum at or before i (block max-scan in chunks with a carry), then
// out[k] = last[min(events[k], n - 1)] in the requested units.  events [n_events] int64, of which *count are used
// when count != NULL; a negative event sets B2L_STATUS_NEGATIVE_EVENT in *status and writes nothing.
template <class T>
__global__ void __launch_bounds__(1024) onset_backtrack_kernel(const T* __restrict__ e, int n,
                                                               const long long* __restrict__ events,
                                                               long long n_events, const long long* __restrict__ count,
                                                               int* __restrict__ last, int units, int hop_length,
                                                               double sr, void* __restrict__ out, int* status) {
  __shared__ int s_warp[32];
  __shared__ int s_carry;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const long long m = count ? *count : n_events;
  bool neg = false;
  for (long long k = threadIdx.x; k < m; k += blockDim.x) neg |= events[k] < 0;
  if (__syncthreads_or(neg)) {
    if (threadIdx.x == 0) atomicOr(status, B2L_STATUS_NEGATIVE_EVENT);
    return;
  }
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  for (long long cs = 0; cs < n; cs += blockDim.x) {
    const long long i = cs + threadIdx.x;
    int v = 0;
    if (i >= 1 && i + 1 < n && e[i] <= e[i - 1] && e[i] < e[i + 1]) v = (int)i;
    for (int o = 1; o < 32; o <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, v, o);
      if (lane >= o) v = max(v, u);
    }
    if (lane == 31) s_warp[warp] = v;
    __syncthreads();
    int pre = s_carry;
    for (int w = 0; w < warp; ++w) pre = max(pre, s_warp[w]);
    v = max(v, pre);
    if (i < n) last[i] = v;
    __syncthreads();
    if (threadIdx.x == blockDim.x - 1) s_carry = v;
    __syncthreads();
  }
  for (long long k = threadIdx.x; k < m; k += blockDim.x) {
    const long long ev = events[k];
    const long long t = n > 0 ? last[ev < n - 1 ? ev : n - 1] : 0;
    if (units == 0) ((long long*)out)[k] = t;
    else if (units == 1) ((long long*)out)[k] = t * hop_length;
    else ((double*)out)[k] = (double)(t * hop_length) / sr;
  }
}

}  // namespace b2l_onset
