// align_kernels.cuh — librosa.sequence.dtw, dtw_backtracking and rqa (librosa/sequence.py:185-1075).
//
//   dtw_cost_kernel<T, METRIC>   cdist(X, Y, metric) in float64, one thread per cell of C, and the NaN verdict flag
//   nan_flag_kernel<T>           the NaN verdict of a cost matrix the caller supplies
//   wave_kernel<TILE, Rule>      one anti-diagonal of TILE x TILE tiles of a 2-D dynamic programme; Rule is
//                                DtwRule (accumulated cost and step index) or RqaRule<T> (alignment score and pointer)
//   dtw_walk_kernel              the dtw warping path, walked from the end cell by one warp
//   rqa_argmax_kernel<T>         np.argmax over the whole score matrix, per block (64-bit flat indices)
//   rqa_walk_kernel              the last reduction step and the rqa path, start to end
//
// The tile wavefront is exact for any dependency (a, b) with a, b >= 0 and a + b >= 1: such a predecessor lies on an
// earlier anti-diagonal, of cells and of tiles.  Tiles of one anti-diagonal are independent CTAs of one launch; inside
// a tile the cell anti-diagonals are separated by block barriers, and every predecessor is read from global memory
// (the tile's own cells after the barrier, earlier tiles after the launch boundary).
#pragma once
#include <float.h>
#include <stdint.h>

#include "numerics.cuh"

namespace b2l_align {
using namespace b2l;

#ifndef B2L_ALIGN_TILE
#define B2L_ALIGN_TILE 32
#endif
constexpr int kTile = B2L_ALIGN_TILE;

enum Metric { kEuclidean = 0, kSqEuclidean = 1, kCityblock = 2, kChebyshev = 3, kCosine = 4 };

// ------------------------------------------------------------------ cost matrix
struct CostArgs {
  const void* x;              // X, C order (..., K, N): feature f of frame n is x[x_off[f] + n]
  const void* y;              // Y likewise, M frames
  const long long* x_off;     // [K]
  const long long* y_off;     // [K]
  long long K, N, M;
  int transpose;              // write C.T: C[m][n] ([M][N]); else C[n][m] ([N][M])
  double* C;
  int* flags;                 // bit 0: some cost is NaN
};

__device__ __forceinline__ double ld(const float* p, long long i) { return (double)__ldg(p + i); }
__device__ __forceinline__ double ld(const double* p, long long i) { return __ldg(p + i); }

// scipy 1.18's cdist: the sums run over the features in order, unfused; cosine keeps two interleaved partial sums
// (even and odd features, added at the end, an odd last feature after them) for the dot product and each squared
// norm, divides by the product of the two square roots and clamps the cosine to [-1, 1].
template <class T, int METRIC>
__global__ void __launch_bounds__(256) dtw_cost_kernel(CostArgs a) {
  const T* x = (const T*)a.x;
  const T* y = (const T*)a.y;
  const long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  bool nan = false;
  for (long long n = blockIdx.y; n < a.N; n += gridDim.y) {
    if (m < a.M) {
      double r;
      if (METRIC == kCosine) {
        double xy[2] = {0.0, 0.0}, xx[2] = {0.0, 0.0}, yy[2] = {0.0, 0.0};
        const long long pairs = a.K / 2 * 2;
        for (long long f = 0; f < pairs; ++f) {
          const double u = ld(x, __ldg(a.x_off + f) + n), v = ld(y, __ldg(a.y_off + f) + m);
          xy[f & 1] = __dadd_rn(xy[f & 1], __dmul_rn(u, v));
          xx[f & 1] = __dadd_rn(xx[f & 1], __dmul_rn(u, u));
          yy[f & 1] = __dadd_rn(yy[f & 1], __dmul_rn(v, v));
        }
        double sxy = __dadd_rn(xy[0], xy[1]), sxx = __dadd_rn(xx[0], xx[1]), syy = __dadd_rn(yy[0], yy[1]);
        if (pairs < a.K) {
          const double u = ld(x, __ldg(a.x_off + pairs) + n), v = ld(y, __ldg(a.y_off + pairs) + m);
          sxy = __dadd_rn(sxy, __dmul_rn(u, v));
          sxx = __dadd_rn(sxx, __dmul_rn(u, u));
          syy = __dadd_rn(syy, __dmul_rn(v, v));
        }
        double c = __ddiv_rn(sxy, __dmul_rn(__dsqrt_rn(sxx), __dsqrt_rn(syy)));
        if (fabs(c) > 1.0) c = copysign(1.0, c);
        r = __dsub_rn(1.0, c);
      } else {
        r = 0.0;
        for (long long f = 0; f < a.K; ++f) {
          const double d = __dsub_rn(ld(x, __ldg(a.x_off + f) + n), ld(y, __ldg(a.y_off + f) + m));
          if (METRIC == kCityblock) r = __dadd_rn(r, fabs(d));
          else if (METRIC == kChebyshev) r = r < fabs(d) ? fabs(d) : r;   // std::max: a NaN difference is skipped
          else r = __dadd_rn(r, __dmul_rn(d, d));
        }
        if (METRIC == kEuclidean) r = __dsqrt_rn(r);
      }
      nan |= isnan(r);
      a.C[a.transpose ? m * a.N + n : n * a.M + m] = r;
    }
  }
  if (__any_sync(0xffffffffu, nan) && (threadIdx.x & 31) == 0) atomicOr(a.flags, 1);
}

template <class T>
__global__ void __launch_bounds__(256) nan_flag_kernel(const T* c, long long n, int* flags) {
  bool nan = false;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    nan |= isnan((double)c[i]);
  if (__any_sync(0xffffffffu, nan) && (threadIdx.x & 31) == 0) atomicOr(flags, 1);
}

// ------------------------------------------------------------------ wavefront
// Cells of tile (ti, tj): rows ti*TILE + r (thread r), columns tj*TILE + s - r at step s.
template <int TILE, class Rule>
__global__ void __launch_bounds__(TILE) wave_kernel(Rule rule, long long wave, long long ti0) {
  const long long ti = ti0 + blockIdx.x, tj = wave - ti;
  const long long i = ti * TILE + threadIdx.x, j0 = tj * TILE;
  if (rule.skip_tile(ti * TILE, j0, TILE)) {
    if (i < rule.n)
      for (int c = 0; c < TILE && j0 + c < rule.m; ++c) rule.fill_outside(i, j0 + c);
    return;
  }
  for (int s = 0; s < 2 * TILE - 1; ++s) {
    const long long j = j0 + s - (int)threadIdx.x;
    if (i < rule.n && j >= j0 && j < j0 + TILE && j < rule.m) rule.cell(i, j);
    __syncthreads();
  }
}

// D[i][j] = min over the steps k, in table order, of D[i - a_k][j - b_k] + (w_mul[k] * C[i][j] + w_add[k]), a step
// taken only when strictly better; predecessors outside the matrix are +inf.  Starting values D[0][0] = C[0][0] (with
// subseq: D[0][j] = C[0][j]), +inf elsewhere, and the step scan runs over them too.  Outside the Sakoe-Chiba band
// (band_lo < j - i < band_hi) C counts as +inf.
template <class TC>
struct DtwRule {
  const TC* C;
  double* D;
  int* steps;
  const long long* sa;        // [n_steps] step along rows
  const long long* sb;        // [n_steps] step along columns
  const double* w_add;
  const double* w_mul;
  long long n, m;
  int n_steps, subseq, band, skip_outside;   // skip_outside: every w_mul > 0, so a cell outside the band is +inf
  long long band_lo, band_hi;

  __device__ bool inside(long long i, long long j) const {
    const long long d = j - i;
    return !band || (d > band_lo && d < band_hi);
  }
  __device__ bool skip_tile(long long i0, long long j0, int t) const {
    if (!band || !skip_outside) return false;
    // j - i over the tile spans [j0 - (i0 + t - 1), j0 + t - 1 - i0]
    return j0 + t - 1 - i0 <= band_lo || j0 - (i0 + t - 1) >= band_hi;
  }
  __device__ void fill_outside(long long i, long long j) const {
    D[i * m + j] = __longlong_as_double(0x7ff0000000000000LL);
    steps[i * m + j] = 0;
  }
  __device__ void cell(long long i, long long j) const {
    const double inf = __longlong_as_double(0x7ff0000000000000LL);
    const double c = inside(i, j) ? (double)C[i * m + j] : inf;
    double best = (i == 0 && (j == 0 || subseq)) ? c : inf;
    int st = 0;
    for (int k = 0; k < n_steps; ++k) {
      const long long a = __ldg(sa + k), b = __ldg(sb + k);
      double pred;
      if (a == 0 && b == 0) pred = best;
      else if (a > i || b > j) pred = inf;
      else pred = D[(i - a) * m + (j - b)];
      const double cost = __dadd_rn(pred, __dadd_rn(__dmul_rn(__ldg(w_mul + k), c), __ldg(w_add + k)));
      if (cost < best) { best = cost; st = k; }
    }
    D[i * m + j] = best;
    steps[i * m + j] = st;
  }
};

// librosa's __rqa_dp: score in sim's dtype, candidates and gap arithmetic in float64 rounded once on store, int8
// pointers (0 diagonal, 1 / 2 knight moves, -1 reset, -2 inclusive reset).
template <class T>
struct RqaRule {
  const T* sim;
  T* score;
  signed char* ptr;
  long long n, m;
  double gap_onset, gap_extend;
  int knight;

  __device__ bool skip_tile(long long, long long, int) const { return false; }
  __device__ void fill_outside(long long, long long) const {}
  __device__ void cell(long long i, long long j) const {
    const long long at = i * m + j;
    const T s = sim[at];
    if (i == 0 || j == 0) {
      score[at] = s;
      ptr[at] = s != (T)0 ? -2 : -1;    // truthiness: NaN counts as a link
      return;
    }
    if (i == 1 && j == 1) {
      if (s > (T)0) {
        score[at] = (T)((double)score[0] + (double)s);
        ptr[at] = 0;
      } else {
        const double link = sim[0] > (T)0 ? 1.0 : 0.0;
        const double v = __dsub_rn(__dsub_rn((double)score[0], __dmul_rn(link, gap_onset)),
                                   __dmul_rn(1.0 - link, gap_extend));
        const T out = (T)(v > 0.0 ? v : 0.0);
        score[at] = out;
        ptr[at] = out > (T)0 ? 0 : -1;
      }
      return;
    }
    // candidates: (i-1, j-1), (i-1, j-2), (i-2, j-1); the second row and column take the first two (in their own
    // order: the second column's second candidate is (i-2, j-1), stored as pointer 1)
    long long at_c[3];
    int limit;
    if (i == 1) { at_c[0] = at - m - 1; at_c[1] = at - m - 2; limit = knight ? 2 : 1; }
    else if (j == 1) { at_c[0] = at - m - 1; at_c[1] = at - 2 * m - 1; limit = knight ? 2 : 1; }
    else { at_c[0] = at - m - 1; at_c[1] = at - m - 2; at_c[2] = at - 2 * m - 1; limit = knight ? 3 : 1; }
    double bv = 0.0;
    int bi = kArgNone;
    if (s > (T)0) {
      for (int k = 0; k < limit; ++k) ArgmaxMerge()(bv, bi, (double)score[at_c[k]], k);
      score[at] = (T)__dadd_rn(bv, (double)s);
      ptr[at] = (signed char)bi;
    } else {
      for (int k = 0; k < limit; ++k) {
        const double t = sim[at_c[k]] > (T)0 ? 1.0 : 0.0;
        const double v = __dsub_rn(__dsub_rn((double)score[at_c[k]], __dmul_rn(t, gap_onset)),
                                   __dmul_rn(1.0 - t, gap_extend));
        ArgmaxMerge()(bv, bi, v, k);
      }
      const T out = (T)(bv > 0.0 ? bv : 0.0);
      score[at] = out;
      ptr[at] = out == (T)0 ? -1 : (signed char)bi;
    }
  }
};

// ------------------------------------------------------------------ dtw path
// Status of a walk, as the negative of the length word.
enum WalkStatus {
  kWalkAllInf = 1,      // subseq: the last row of D is all +-inf
  kWalkInfEnd = 2,      // the end cell of D is +-inf
  kWalkNotOrigin = 3,   // the path does not reach (0, 0)
  kWalkZeroStep = 4,    // a (0, 0) step: the reference's walk never ends
  kWalkBadStep = 5,     // a step index outside the table
  kWalkNan = 6,         // the cost matrix holds NaN (the verdict flag)
};

struct WalkArgs {
  const int* steps;           // [n][m]
  const double* D;            // [n][m], subseq without start / end-cell checks (NULL: none)
  const long long* sa;
  const long long* sb;
  int n_steps;
  long long n, m;
  int subseq;
  long long start;            // end column; < 0: the last column, or with D and subseq the first argmin of D's last row
  int check_end;              // dtw's checks: +-inf end cell or last row, and reaching (0, 0)
  int flip;                   // write (m, n) pairs
  const int* flags;           // verdict flags of the cost matrix (NULL: none)
  long long* wp;              // [n + m][2], walk order
  long long* len;             // path length, or -WalkStatus
};

__global__ void __launch_bounds__(32) dtw_walk_kernel(WalkArgs a) {
  const int lane = threadIdx.x;
  const double inf = __longlong_as_double(0x7ff0000000000000LL);
  if (a.flags && (a.flags[0] & 1)) {
    if (lane == 0) *a.len = -kWalkNan;
    return;
  }
  long long j = a.start < 0 ? a.m - 1 : a.start;
  if (a.D && a.subseq && a.start < 0) {
    // np.argmin of the last row (the first NaN, else the first minimum), as an argmax of -D
    const double* row = a.D + (a.n - 1) * a.m;
    double bv = 0.0;
    long long bi = kArgNone64;
    bool all_inf = true;
    for (long long c = lane; c < a.m; c += 32) {
      all_inf &= isinf(row[c]);
      ArgmaxMerge()(bv, bi, -row[c], c);
    }
    warp_select(bv, bi, ArgmaxMerge());
    all_inf = __all_sync(0xffffffffu, all_inf);
    if (a.check_end && all_inf) {
      if (lane == 0) *a.len = -kWalkAllInf;
      return;
    }
    j = bi;
  } else if (a.D && a.check_end && isinf(a.D[a.n * a.m - 1])) {
    if (lane == 0) *a.len = -kWalkInfEnd;
    return;
  }
  if (lane != 0) return;
  long long i = a.n - 1, len = 0;
  const int fi = a.flip ? 1 : 0;
  a.wp[0 + fi] = i;
  a.wp[1 - fi] = j;
  len = 1;
  while (a.subseq ? i > 0 : (i != 0 || j != 0)) {
    const int k = a.steps[i * a.m + j];
    if (k < 0 || k >= a.n_steps) { *a.len = -kWalkBadStep; return; }
    const long long di = a.sa[k], dj = a.sb[k];
    if (di == 0 && dj == 0) { *a.len = -kWalkZeroStep; return; }
    i -= di;
    j -= dj;
    if (i < 0 || j < 0) break;
    a.wp[2 * len + fi] = i;
    a.wp[2 * len + 1 - fi] = j;
    ++len;
  }
  if (a.check_end && !a.subseq && (a.wp[2 * (len - 1)] != 0 || a.wp[2 * (len - 1) + 1] != 0)) {
    *a.len = -kWalkNotOrigin;
    return;
  }
  *a.len = len;
}

// ------------------------------------------------------------------ rqa path
constexpr int kArgThreads = 256;

// Block b reduces cells [b * per_block, (b + 1) * per_block) to (value, flat index) in np.argmax order.
template <class T>
__global__ void __launch_bounds__(kArgThreads) rqa_argmax_kernel(const T* score, long long total, long long per_block,
                                                                 double* part_v, long long* part_i) {
  __shared__ double s_v[kArgThreads / 32];
  __shared__ long long s_i[kArgThreads / 32];
  const long long lo = (long long)blockIdx.x * per_block, hi = min(total, lo + per_block);
  double v = 0.0;
  long long idx = kArgNone64;
  for (long long k = lo + threadIdx.x; k < hi; k += kArgThreads) ArgmaxMerge()(v, idx, (double)score[k], k);
  block_select(v, idx, s_v, s_i, ArgmaxMerge());
  if (threadIdx.x == 0) { part_v[blockIdx.x] = v; part_i[blockIdx.x] = idx; }
}

// One block: the argmax over the partials, then thread 0 walks the pointers from it twice — to count, then to write
// the path start to end.  Column indices follow the reference's Python indexing: the second column's pointer 1 steps
// to column -1, read as the last column and stored as that negative value in uint64.  len: the path length, or -1
// when a column index passes -m (the reference raises IndexError there).
__global__ void __launch_bounds__(kArgThreads) rqa_walk_kernel(const signed char* ptr, long long n, long long m,
                                                               const double* part_v, const long long* part_i,
                                                               int n_parts, unsigned long long* path, long long* len) {
  __shared__ double s_v[kArgThreads / 32];
  __shared__ long long s_i[kArgThreads / 32];
  double v = 0.0;
  long long idx = kArgNone64;
  for (int k = threadIdx.x; k < n_parts; k += kArgThreads) ArgmaxMerge()(v, idx, part_v[k], part_i[k]);
  block_select(v, idx, s_v, s_i, ArgmaxMerge());
  if (threadIdx.x != 0) return;
  const long long i0 = idx / m, j0 = idx % m;
  for (int pass = 0; pass < 2; ++pass) {
    long long i = i0, j = j0, count = 0, total = pass ? *len : 0;
    while (true) {
      if (j < -m) { *len = -1; return; }
      const signed char bt = ptr[i * m + (j < 0 ? j + m : j)];
      if (bt == -1) break;
      if (pass) {
        path[2 * (total - 1 - count)] = (unsigned long long)i;
        path[2 * (total - 1 - count) + 1] = (unsigned long long)j;
      }
      ++count;
      if (bt == -2) break;
      i -= bt == 2 ? 2 : 1;
      j -= bt == 1 ? 2 : 1;
    }
    if (!pass) *len = count;
  }
}

}  // namespace b2l_align
