// neighbors_kernels.cuh — nearest-neighbour graphs and filtering (neighbors_api.cu): librosa.segment.recurrence_matrix
// (librosa/segment.py:391-706, the bandwidths of 1332-1437) and librosa.decompose.nn_filter (decompose.py:409-592).
//
// recurrence_matrix runs as row blocks of one loop (nn_pack_kernel once, then nn_dist_kernel + nn_select_kernel per
// block of query rows, workspace rows * t doubles), followed by nn_graph_kernel over all rows and, in affinity mode,
// nn_median_kernel (med_k_scalar) and nn_affinity_kernel.  nn_filter is nn_agg_kernel over a neighbour table, which
// nn_compact_kernel builds from a dense device matrix.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"
#include "numerics.cuh"

namespace b2l {

constexpr int kNnTile = 64;            // rows and columns of one Gram tile
constexpr int kNnKc = 16;              // features staged per step of the Gram loop
constexpr int kNnMaxM = 4096;          // candidates per row of the selection (B2L_NN_MAX_CANDIDATES)
constexpr int kNnSelectThreads = 512;
constexpr int kNnNone = 0x7fffffff;    // index of an empty slot: sorts after every frame
constexpr int kNnStatsMax = 256;       // values per row of the affinity bandwidth statistics (B2L_NN_MAX_STATS)

// --------------------------------------------------------------------------------------------- packing
// X[i][f] = (double) src[lead * lead_stride + g * feat_stride + i * frame_stride] for feature f = lead * n_feat + g, and
// the squared norm of each frame.  A non-finite value sets `bad` (the reference's check_array refuses it).
template <class T>
__global__ void nn_pack_kernel(const T* __restrict__ src, long long n_lead, long long n_feat, long long lead_stride,
                               long long feat_stride, long long frame_stride, long long t, double* __restrict__ X,
                               double* __restrict__ norms, int* bad) {
  const long long D = n_lead * n_feat;
  const int lane = threadIdx.x & 31;
  for (long long i = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5; i < t;
       i += ((long long)gridDim.x * blockDim.x) >> 5) {
    double s = 0.0;
    bool ok = true;
    for (long long f = lane; f < D; f += 32) {
      const long long l = f / n_feat, g = f - l * n_feat;
      const double v = (double)src[l * lead_stride + g * feat_stride + i * frame_stride];
      ok &= finite_(v);
      X[i * D + f] = v;
      s = fma(v, v, s);
    }
    s = warp_reduce(s, [](double a, double b) { return a + b; });
    if (__any_sync(0xffffffffu, !ok) && lane == 0) atomicOr(bad, 1);
    if (lane == 0) norms[i] = s;
  }
}

// --------------------------------------------------------------------------------------------- distances
// m8n8k4 FP64 tensor-core product: acc += A (8x4, one element per lane: row lane/4, column lane%4) * B (4x8, one
// element per lane: row lane%4, column lane/4); acc holds row lane/4, columns 2*(lane%4) + {0, 1}.
__device__ __forceinline__ void dmma(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};\n"
               : "+d"(c0), "+d"(c1)
               : "d"(a), "d"(b));
}

struct NnDistArgs {
  const double* X;       // [t][D]
  const double* norms;   // [t] squared norms
  long long t, D;
  long long r0;          // first query row of the block (a multiple of kNnTile)
  int rows;              // query rows of the block
  int cosine;
  double* W;             // [rows][t] distances of the block
};

// One CTA per (column tile, query row tile), 8 warps.  The Gram tile of the pair of tiles (P, Q) is always formed as
// the tile of rows min(P, Q) against columns max(P, Q), and on a diagonal tile (i, j) is read from [min][max]: so
// d(i, j) and d(j, i) come out of the same operations, bit for bit, whichever row block asks for them.  The distance
// formulas combine the two norms with commutative operations only, for the same reason.
__global__ void __launch_bounds__(256) nn_dist_kernel(NnDistArgs a) {
  // the staged operands and, after the feature loop, the Gram tile share one buffer (static shared memory <= 48 KiB)
  __shared__ double s_buf[kNnTile * (kNnTile + 1)];
  double (*sA)[kNnKc + 1] = reinterpret_cast<double (*)[kNnKc + 1]>(s_buf);
  double (*sB)[kNnKc + 1] = reinterpret_cast<double (*)[kNnKc + 1]>(s_buf + kNnTile * (kNnKc + 1));
  double (*sG)[kNnTile + 1] = reinterpret_cast<double (*)[kNnTile + 1]>(s_buf);
  const long long qi = a.r0 / kNnTile + blockIdx.y;   // query row tile
  const long long cj = blockIdx.x;                    // column tile
  const long long P = qi < cj ? qi : cj, Q = qi < cj ? cj : qi;
  const long long p0 = P * kNnTile, q0 = Q * kNnTile;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = (warp >> 1) * 16, wn = (warp & 1) * 32;   // warp sub-tile: 16 rows x 32 columns, 2 x 4 mma tiles
  double acc[2][4][2];
#pragma unroll
  for (int m = 0; m < 2; ++m)
#pragma unroll
    for (int n = 0; n < 4; ++n) acc[m][n][0] = acc[m][n][1] = 0.0;
  for (long long k0 = 0; k0 < a.D; k0 += kNnKc) {
    for (int e = tid; e < kNnTile * kNnKc; e += 256) {
      const int r = e / kNnKc, k = e % kNnKc;
      const long long kk = k0 + k;
      sA[r][k] = (p0 + r < a.t && kk < a.D) ? a.X[(p0 + r) * a.D + kk] : 0.0;
      sB[r][k] = (q0 + r < a.t && kk < a.D) ? a.X[(q0 + r) * a.D + kk] : 0.0;
    }
    __syncthreads();
#pragma unroll
    for (int ks = 0; ks < kNnKc; ks += 4) {
      double fa[2], fb[4];
#pragma unroll
      for (int m = 0; m < 2; ++m) fa[m] = sA[wm + m * 8 + (lane >> 2)][ks + (lane & 3)];
#pragma unroll
      for (int n = 0; n < 4; ++n) fb[n] = sB[wn + n * 8 + (lane >> 2)][ks + (lane & 3)];
#pragma unroll
      for (int m = 0; m < 2; ++m)
#pragma unroll
        for (int n = 0; n < 4; ++n) dmma(acc[m][n][0], acc[m][n][1], fa[m], fb[n]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int m = 0; m < 2; ++m)
#pragma unroll
    for (int n = 0; n < 4; ++n) {
      const int r = wm + m * 8 + (lane >> 2), c = wn + n * 8 + 2 * (lane & 3);
      sG[r][c] = acc[m][n][0];
      sG[r][c + 1] = acc[m][n][1];
    }
  __syncthreads();
  const long long i0 = qi * kNnTile, j0 = cj * kNnTile;
  for (int e = tid; e < kNnTile * kNnTile; e += 256) {
    const int r = e / kNnTile, c = e % kNnTile;
    const long long i = i0 + r, j = j0 + c;
    if (i >= a.t || j >= a.t || i - a.r0 >= a.rows) continue;
    // (i, j) in the canonical tile: i's tile is P when qi <= cj
    int gr, gc;
    if (qi < cj) { gr = r; gc = c; }
    else if (qi > cj) { gr = c; gc = r; }
    else { gr = r < c ? r : c; gc = r < c ? c : r; }
    const double g = sG[gr][gc], ni = a.norms[i], nj = a.norms[j];
    double d;
    if (a.cosine) {
      if (ni == 0.0 || nj == 0.0) d = 1.0;   // a zero frame normalises to zero: 1 - 0
      else d = sub_rn(1.0, mul_rn(g, mul_rn(1.0 / sqrt_rn(ni), 1.0 / sqrt_rn(nj))));
      d = d < 0.0 ? 0.0 : (d > 2.0 ? 2.0 : d);
    } else {
      const double s = sub_rn(add_rn(ni, nj), mul_rn(2.0, g));
      d = s > 0.0 ? sqrt_rn(s) : 0.0;
    }
    a.W[(i - a.r0) * a.t + j] = d;
  }
}

// --------------------------------------------------------------------------------------------- block helpers
// Exclusive prefix sum of one int per thread over the block (blockDim.x <= 1024); *total gets the sum.  s holds 32
// ints.  Ends with a barrier, so s may be reused after it.
__device__ __forceinline__ int block_exclusive_scan(int v, int* s, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  __syncthreads();
  if (lane == 31) s[warp] = x;
  __syncthreads();
  int base = 0, tot = 0;
  for (int w = 0; w < nw; ++w) {
    if (w < warp) base += s[w];
    tot += s[w];
  }
  __syncthreads();
  *total = tot;
  return base + x - v;
}

// Ascending bitonic sort of n (a power of two) (key, index) pairs in shared memory by the whole block.
__device__ __forceinline__ void bitonic_sort(unsigned long long* key, int* idx, int n) {
  for (int size = 2; size <= n; size <<= 1)
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      __syncthreads();
      for (int e = threadIdx.x; e < n / 2; e += blockDim.x) {
        const int lo = 2 * e - (e & (stride - 1)), hi = lo + stride;
        const bool up = (lo & size) == 0;
        const unsigned long long ka = key[lo], kb = key[hi];
        const int ia = idx[lo], ib = idx[hi];
        const bool gt = ka > kb || (ka == kb && ia > ib);
        if (gt == up) { key[lo] = kb; key[hi] = ka; idx[lo] = ib; idx[hi] = ia; }
      }
    }
  __syncthreads();
}

// --------------------------------------------------------------------------------------------- selection
struct NnSelectArgs {
  const double* W;     // [rows][t] distances of the block
  long long t, r0;
  int rows;
  int M;               // candidates: sklearn's n_neighbors = min(t - 1, k + 2 width)
  int P;               // power of two >= M
  int k, width;
  int mode;            // 0 connectivity, 1 distance, 2 affinity
  int k_max;           // row stride of the tables
  int* out_idx;        // [t][k_max] kept links, ascending frame index
  double* out_val;     // [t][k_max] their distances
  int* out_count;      // [t]
};

// One CTA per query row: the M nearest other frames in (distance, index) order by an MSB radix select on the
// distance bits (a distance is >= 0, so its bits order like its value), then the row's links as the reference keeps
// them: |i - j| >= width; in connectivity mode the k lowest-indexed of those (every value is 1, segment.py:656-664),
// otherwise the k nearest with a non-zero distance (a zero is not a link: the CSR -> LIL round trip stores it but
// nonzero() skips it, and eliminate_zeros() drops it).
__global__ void __launch_bounds__(kNnSelectThreads) nn_select_kernel(NnSelectArgs a) {
  extern __shared__ unsigned long long s_key[];   // [P]
  int* s_idx = reinterpret_cast<int*>(s_key + a.P);
  __shared__ unsigned s_hist[256];
  __shared__ int s_scan[32];
  __shared__ unsigned long long s_prefix;
  __shared__ int s_need;
  const long long row = a.r0 + blockIdx.x;
  const double* w = a.W + (long long)blockIdx.x * a.t;
  const int tid = threadIdx.x;
  if (tid == 0) { s_prefix = 0; s_need = a.M; }
  // 1. the M-th smallest distance v: 8 passes of 8 bits
  unsigned long long mask = 0;
  for (int shift = 56; shift >= 0; shift -= 8) {
    for (int b = tid; b < 256; b += blockDim.x) s_hist[b] = 0;
    __syncthreads();
    const unsigned long long prefix = s_prefix;
    for (long long j = tid; j < a.t; j += blockDim.x) {
      if (j == row) continue;
      const unsigned long long kb = (unsigned long long)__double_as_longlong(w[j]);
      if ((kb & mask) == prefix) atomicAdd(&s_hist[(kb >> shift) & 255], 1u);
    }
    __syncthreads();
    if (tid == 0) {
      int need = s_need, b = 0;
      while ((int)s_hist[b] < need) need -= s_hist[b++];
      s_need = need;
      s_prefix = prefix | ((unsigned long long)b << shift);
    }
    mask |= 255ULL << shift;
    __syncthreads();
  }
  const unsigned long long vkey = s_prefix;
  const int n_eq = s_need;   // elements equal to v that belong to the top M (the lowest-indexed ones)
  // 2. gather: every distance below v, then the n_eq lowest-indexed ones equal to v, in index order
  int n_lt = 0, taken_eq = 0;
  for (long long j0 = 0; j0 < a.t; j0 += blockDim.x) {
    const long long j = j0 + tid;
    unsigned long long kb = ~0ULL;
    if (j < a.t && j != row) kb = (unsigned long long)__double_as_longlong(w[j]);
    int tot_lt, tot_eq;
    const int pos_lt = block_exclusive_scan(kb < vkey, s_scan, &tot_lt);
    const int pos_eq = block_exclusive_scan(kb == vkey, s_scan, &tot_eq);
    const int M_lt = a.M - n_eq;
    if (kb < vkey) { s_key[n_lt + pos_lt] = kb; s_idx[n_lt + pos_lt] = (int)j; }
    if (kb == vkey && taken_eq + pos_eq < n_eq) {
      s_key[M_lt + taken_eq + pos_eq] = kb;
      s_idx[M_lt + taken_eq + pos_eq] = (int)j;
    }
    n_lt += tot_lt;
    taken_eq += tot_eq;
  }
  for (int e = a.M + tid; e < a.P; e += blockDim.x) { s_key[e] = ~0ULL; s_idx[e] = kNnNone; }
  // 3. (distance, index) order
  bitonic_sort(s_key, s_idx, a.P);
  // 4. the links the reference keeps, re-keyed by index: kept -> frame index, dropped -> kNnNone
  const int per = (a.P + blockDim.x - 1) / blockDim.x;
  const int e0 = tid * per;
  int n_surv = 0;
  for (int e = e0; e < e0 + per && e < a.M; ++e) {
    const long long j = s_idx[e];
    const long long dij = j > row ? j - row : row - j;
    n_surv += dij >= a.width && (a.mode == 0 || s_key[e] != 0ULL);
  }
  int tot;
  int rank = block_exclusive_scan(n_surv, s_scan, &tot);
  for (int e = e0; e < e0 + per && e < a.P; ++e) {
    bool keep = false;
    if (e < a.M) {
      const long long j = s_idx[e];
      const long long dij = j > row ? j - row : row - j;
      const bool surv = dij >= a.width && (a.mode == 0 || s_key[e] != 0ULL);
      keep = surv && (a.mode == 0 || rank < a.k);
      rank += surv;
    }
    // connectivity keeps every survivor here: the k lowest indices are the first k after the re-sort
    if (!keep) s_idx[e] = kNnNone;
    s_key[e] = (unsigned long long)(unsigned)s_idx[e] << 32 | (unsigned long long)(unsigned)e;
  }
  // ascending frame index (the keys are distinct); the distances are read back from the row
  bitonic_sort(s_key, s_idx, a.P);
  int n_kept = 0;
  for (int e = 0; e < a.P && (int)(s_key[e] >> 32) != kNnNone; ++e) ++n_kept;   // uniform, all threads
  if (a.mode == 0 && n_kept > a.k) n_kept = a.k;
  for (int e = tid; e < n_kept; e += blockDim.x) {
    const int j = (int)(s_key[e] >> 32);
    a.out_idx[row * a.k_max + e] = j;
    a.out_val[row * a.k_max + e] = w[j];
  }
  if (tid == 0) a.out_count[row] = n_kept;
}

// --------------------------------------------------------------------------------------------- graph epilogue
struct NnGraphArgs {
  const int* in_idx;      // [t][k_in] from nn_select_kernel
  const double* in_val;
  const int* in_count;
  int k_in;
  long long t;
  int k;                  // the reference's k (bandwidth statistics use the k smallest of a row)
  int mode;               // 0 connectivity, 1 distance, 2 affinity
  int sym, self_link;
  int f64;                // distances rounded to float64 (else float32) before any statistic
  int k_out;              // row stride of the output table (k_in + 1)
  int* out_idx;
  double* out_val;        // distance in the output dtype (0 for an affinity self-link)
  int* out_count;
  double* kth;            // [t] distance to the k-th neighbour (NaN: no neighbour), affinity only
  double* avg;            // [t] mean distance to the first k neighbours, affinity only
};

__device__ __forceinline__ bool nn_contains(const int* idx, int n, int j) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int m = (lo + hi) >> 1;
    if (idx[m] < j) lo = m + 1; else hi = m;
  }
  return lo < n && idx[lo] == j;
}

// np.add.reduce of a contiguous 1-D array (NumPy's pairwise summation: blocks of 8 partial sums up to 128 elements,
// halves above that), for the row statistics.
template <class T, class Src>
__device__ T np_pairwise_sum(const Src* a, int n) {
  // iterative over the recursion tree: the halves of n > 128 are at most 12 levels deep for n <= 4097
  struct Frame { int off, n, state; T left; };
  Frame st[16];
  int sp = 0;
  st[0] = {0, n, 0, T(0)};
  T ret = T(0);
  for (;;) {
    Frame& f = st[sp];
    if (f.n <= 128) {
      T res;
      const Src* p = a + f.off;
      if (f.n < 8) {
        res = T(-0.0);
        for (int i = 0; i < f.n; ++i) res = add_rn(res, (T)p[i]);
      } else {
        T r[8];
        for (int j = 0; j < 8; ++j) r[j] = (T)p[j];
        int i = 8;
        for (; i < f.n - f.n % 8; i += 8)
          for (int j = 0; j < 8; ++j) r[j] = add_rn(r[j], (T)p[i + j]);
        res = add_rn(add_rn(add_rn(r[0], r[1]), add_rn(r[2], r[3])), add_rn(add_rn(r[4], r[5]), add_rn(r[6], r[7])));
        for (; i < f.n; ++i) res = add_rn(res, (T)p[i]);
      }
      ret = res;
    } else if (f.state == 0) {
      int n2 = f.n / 2;
      n2 -= n2 % 8;
      f.state = 1;
      st[++sp] = {f.off, n2, 0, T(0)};
      continue;
    } else if (f.state == 1) {
      int n2 = f.n / 2;
      n2 -= n2 % 8;
      f.left = ret;
      f.state = 2;
      st[++sp] = {f.off + n2, f.n - n2, 0, T(0)};
      continue;
    } else {
      ret = add_rn(f.left, ret);
    }
    if (sp == 0) return ret;
    --sp;
  }
}

// One thread per row.  sym keeps (i, j) when i is among j's links too (rec.minimum(rec.T): the two distances are
// equal bit for bit); self adds (i, i) in connectivity and affinity mode.  In affinity mode the row statistics of
// __affinity_bandwidth follow: the k-th smallest value of the row (its self-link counts as 0) and their mean.
template <class T>
__global__ void nn_graph_kernel(NnGraphArgs a) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < a.t; i += (long long)gridDim.x * blockDim.x) {
    const int n = a.in_count[i];
    const int* li = a.in_idx + i * a.k_in;
    const double* lv = a.in_val + i * a.k_in;
    int* oi = a.out_idx + i * a.k_out;
    double* ov = a.out_val + i * a.k_out;
    int c = 0;
    bool self_done = !(a.self_link && a.mode != 1);
    for (int e = 0; e < n; ++e) {
      const int j = li[e];
      if (a.sym && !nn_contains(a.in_idx + (long long)j * a.k_in, a.in_count[j], (int)i)) continue;
      if (!self_done && j > i) { oi[c] = (int)i; ov[c] = 0.0; ++c; self_done = true; }
      oi[c] = j;
      ov[c] = a.mode == 0 ? 1.0 : (double)(T)lv[e];
      ++c;
    }
    if (!self_done) { oi[c] = (int)i; ov[c] = 0.0; ++c; }
    if (a.mode == 0) for (int e = 0; e < c; ++e) if (oi[e] == (int)i) ov[e] = 1.0;
    a.out_count[i] = c;
    if (a.mode == 2 && a.kth) {
      // np.sort(row)[:k] by insertion into a local buffer: rows of at most kNnStatsMax values (checked on the host)
      T buf[kNnStatsMax];
      const int m = c < a.k ? c : a.k;
      if (c == 0) { a.kth[i] = __longlong_as_double(0x7ff8000000000000LL); a.avg[i] = a.kth[i]; continue; }
      for (int e = 0; e < c; ++e) {
        const T v = (T)ov[e];
        int p = e;
        while (p > 0 && buf[p - 1] > v) { buf[p] = buf[p - 1]; --p; }
        buf[p] = v;
      }
      a.kth[i] = (double)buf[m - 1];
      a.avg[i] = (double)div_rn(np_pairwise_sum<T>(buf, m), (T)m);
    }
  }
}

// np.nanmedian of the t row values of `kth` in T: one CTA, the two middle order statistics by radix select on the
// value bits (the values are >= 0).  out[0] = the median, NaN when every row is empty.
template <class T>
__global__ void nn_median_kernel(const double* kth, long long t, double* out) {
  using U = typename std::conditional<sizeof(T) == 4, unsigned, unsigned long long>::type;
  __shared__ unsigned s_hist[256];
  __shared__ int s_cnt;
  __shared__ U s_prefix;
  __shared__ int s_need;
  const int tid = threadIdx.x;
  if (tid == 0) s_cnt = 0;
  __syncthreads();
  int local = 0;
  for (long long i = tid; i < t; i += blockDim.x) local += kth[i] == kth[i];
  atomicAdd(&s_cnt, local);
  __syncthreads();
  const int n = s_cnt;
  if (n == 0) { if (tid == 0) out[0] = __longlong_as_double(0x7ff8000000000000LL); return; }
  T mid[2];
  const int ranks[2] = {(n - 1) / 2, n / 2};
  for (int q = 0; q < 2; ++q) {
    if (tid == 0) { s_prefix = 0; s_need = ranks[q] + 1; }
    U mask = 0;
    for (int shift = 8 * (int)sizeof(T) - 8; shift >= 0; shift -= 8) {
      for (int b = tid; b < 256; b += blockDim.x) s_hist[b] = 0;
      __syncthreads();
      const U prefix = s_prefix;
      for (long long i = tid; i < t; i += blockDim.x) {
        const double v = kth[i];
        if (v != v) continue;
        const T tv = (T)v;
        U kb;
        memcpy(&kb, &tv, sizeof(T));
        if ((kb & mask) == prefix) atomicAdd(&s_hist[(kb >> shift) & 255], 1u);
      }
      __syncthreads();
      if (tid == 0) {
        int need = s_need, b = 0;
        while ((int)s_hist[b] < need) need -= s_hist[b++];
        s_need = need;
        s_prefix = prefix | ((U)b << shift);
      }
      mask |= (U)255 << shift;
      __syncthreads();
    }
    U kb = s_prefix;
    memcpy(&mid[q], &kb, sizeof(T));
    __syncthreads();
  }
  if (tid == 0) out[0] = (double)(n & 1 ? mid[0] : div_rn(add_rn(mid[0], mid[1]), T(2)));
}

// rec.data = exp(rec.data / -bandwidth) in T.  bw_mode: 0 scalar (*scalar), 1 mean_k, 2 gmean_k, 3 mean_k_avg,
// 4 gmean_k_avg, 5 mean_k_avg_and_pair.  The graph rows are the reference's CSR rows (links of frame i).
template <class T>
__global__ void nn_affinity_kernel(const int* idx, double* val, const int* count, int k_out, long long t, int bw_mode,
                                   const double* scalar, const double* kth, const double* avg) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < t; i += (long long)gridDim.x * blockDim.x) {
    const int n = count[i];
    for (int e = 0; e < n; ++e) {
      const int j = idx[i * k_out + e];
      const T d = (T)val[i * k_out + e];
      T bw;
      if (bw_mode == 0) bw = (T)scalar[0];
      else {
        const T si = (T)(bw_mode <= 2 ? kth[i] : avg[i]), sj = (T)(bw_mode <= 2 ? kth[j] : avg[j]);
        if (bw_mode == 1 || bw_mode == 3) bw = div_rn(add_rn(si, sj), T(2));
        else if (bw_mode == 2 || bw_mode == 4) bw = sqrt_rn(mul_rn(si, sj));
        else bw = div_rn(add_rn(add_rn(si, sj), d), T(3));
      }
      val[i * k_out + e] = (double)(T)exp(div_rn(d, -bw));
    }
  }
}

// --------------------------------------------------------------------------------------------- aggregation
// a + b and a * b with x86's NaN rule: a NaN operand is the result (the first one), where the GPU would return its
// canonical NaN, so that a NaN in S reaches the output with the bits the reference gives it.
template <class T> __device__ __forceinline__ T add_x86(T a, T b) { return a != a ? a : (b != b ? b : add_rn(a, b)); }
template <class T> __device__ __forceinline__ T mul_x86(T a, T b) { return a != a ? a : (b != b ? b : mul_rn(a, b)); }

struct NnAggArgs {
  const void* S;          // [n_lead][t][F], "ft"
  void* out;              // same shape
  long long t, F, n_lead;
  const long long* start; // [t] first entry of frame i's neighbours (NULL: i * stride)
  long long stride;
  const int* count;       // [t]
  const int* idx;         // neighbour frame indices
  const double* w;        // weights (average only), values of R
  int agg;                // 0 mean, 1 median, 2 average
  int bins;               // bins per CTA
  int* zero_weight;       // set when a row's weights sum to zero (np.average raises)
};

// One CTA per (frame, chunk of `bins` bins, lead); S and out rows are contiguous in the bins, so every neighbour is
// one coalesced read.  mean: the neighbours summed in stored order in T, then one division by the count (np.mean along
// axis 0).  average: products with the weights in R, summed in order, divided by NumPy's pairwise sum of the weights,
// rounded to T.  median: each bin's values sorted in shared memory (bitonic, NaN last, padding +inf after it), the
// middle value or fl(fl(a + b) / 2) of the middle two; a NaN among them gives NaN (np.median's check).
template <class T, class R>
__global__ void nn_agg_kernel(NnAggArgs a) {
  extern __shared__ unsigned char s_raw[];
  const long long i = blockIdx.x;
  const long long lead = blockIdx.z;
  const long long b0 = (long long)blockIdx.y * a.bins;
  const T* S = (const T*)a.S + lead * a.t * a.F;
  T* out = (T*)a.out + lead * a.t * a.F + i * a.F;
  const int n = a.count[i];
  const long long st = a.start ? a.start[i] : i * a.stride;
  const int* nb = a.idx + st;
  const int tid = threadIdx.x;
  const long long nbins = a.F - b0 < a.bins ? a.F - b0 : a.bins;
  if (n == 0) {
    for (long long b = tid; b < nbins; b += blockDim.x) out[b0 + b] = S[i * a.F + b0 + b];
    return;
  }
  if (a.agg != 1) {
    const double* sw = a.w + st;
    R scl = R(1);
    if (a.agg == 2) {
      R* s_scl = reinterpret_cast<R*>(s_raw);
      if (tid == 0) *s_scl = np_pairwise_sum<R>(sw, n);
      __syncthreads();
      scl = *s_scl;
      if (scl == R(0)) {
        if (tid == 0) atomicOr(a.zero_weight, 1);
        return;
      }
    }
    for (long long b = tid; b < nbins; b += blockDim.x) {
      const long long col = b0 + b;
      if (a.agg == 0) {
        T acc = S[(long long)nb[0] * a.F + col];
        for (int e = 1; e < n; ++e) acc = add_x86(acc, S[(long long)nb[e] * a.F + col]);
        out[col] = acc != acc ? acc : (T)div_rn((double)acc, (double)n);
      } else {
        T first_nan = T(0);
        bool nan = false;
        R acc = mul_x86((R)S[(long long)nb[0] * a.F + col], (R)sw[0]);
        for (int e = 0; e < n; ++e) {
          const T v = S[(long long)nb[e] * a.F + col];
          if (!nan && v != v) { first_nan = v; nan = true; }
          if (e) acc = add_x86(acc, mul_x86((R)v, (R)sw[e]));
        }
        out[col] = nan ? first_nan : (T)div_rn(acc, scl);
      }
    }
    return;
  }
  // median: one warp per bin, P = next power of two >= n values per warp in shared memory
  int P = 1;
  while (P < n) P <<= 1;
  const int warp = tid >> 5, lane = tid & 31, nw = blockDim.x >> 5;
  T* sv = reinterpret_cast<T*>(s_raw) + (long long)warp * P;
  const T inf = T(INFINITY);
  for (long long b = warp; b < nbins; b += nw) {
    const long long col = b0 + b;
    bool any_nan = false;
    for (int e = lane; e < P; e += 32) {
      T v = e < n ? S[(long long)nb[e] * a.F + col] : inf;
      any_nan |= v != v;
      sv[e] = v;
    }
    any_nan = __any_sync(0xffffffffu, any_nan);
    if (any_nan) {   // np.median returns the NaN that its partition puts last: the first one in S's order
      if (lane == 0) {
        T v = T(0);
        for (int e = 0; e < n; ++e) { v = S[(long long)nb[e] * a.F + col]; if (v != v) break; }
        out[col] = v;
      }
      continue;
    }
    for (int size = 2; size <= P; size <<= 1)
      for (int stride = size >> 1; stride > 0; stride >>= 1) {
        __syncwarp();
        for (int e = lane; e < P / 2; e += 32) {
          const int lo = 2 * e - (e & (stride - 1)), hi = lo + stride;
          const bool up = (lo & size) == 0;
          const T x = sv[lo], y = sv[hi];
          if ((x > y) == up) { sv[lo] = y; sv[hi] = x; }
        }
      }
    __syncwarp();
    if (lane == 0) out[col] = n & 1 ? sv[n / 2] : div_rn(add_rn(sv[n / 2 - 1], sv[n / 2]), T(2));
    __syncwarp();
  }
}

// The dense matrix of a neighbour table: rec[j, i] = val of link (i, j), C-ordered t x t of T (the output is zeroed
// first).  One thread per table slot.
template <class T>
__global__ void nn_dense_kernel(const int* idx, const double* val, const int* count, long long t, int k_out, T* rec) {
  for (long long s = blockIdx.x * (long long)blockDim.x + threadIdx.x; s < t * k_out; s += (long long)gridDim.x * blockDim.x) {
    const long long i = s / k_out;
    const int e = (int)(s - i * k_out);
    if (e < count[i]) rec[(long long)idx[s] * t + i] = (T)val[s];
  }
}

// --------------------------------------------------------------------------------------------- compaction
// Column i of a dense C-ordered t x t matrix (scipy.sparse.csc_array(rec)): the rows j with rec[j, i] != 0, ascending,
// written to idx / w at start[i]; pass 0 counts them (count[i]), pass 1 writes them.  One thread per column walks the
// rows in order, so a warp reads 32 consecutive elements of a row at a time (coalesced).
template <class T>
__global__ void nn_compact_kernel(const T* rec, long long t, int pass, int* count, const long long* start, int* idx,
                                  double* w) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < t; i += (long long)gridDim.x * blockDim.x) {
    int c = 0;
    const long long s0 = pass == 1 ? start[i] : 0;
    for (long long j = 0; j < t; ++j) {
      const T v = rec[j * t + i];
      if (!(v == T(0))) {
        if (pass == 1) {
          idx[s0 + c] = (int)j;
          w[s0 + c] = (double)v;
        }
        ++c;
      }
    }
    if (pass == 0) count[i] = c;
  }
}

}  // namespace b2l
