// sequence_kernels.cuh — librosa.sequence.viterbi, viterbi_discriminative and viterbi_binary
// (librosa/sequence.py:1175-1876).
//
//   viterbi_logobs_kernel<T, MODE>   prob -> float64 log-likelihoods [problem][state][frame] and the verdict flags
//   viterbi_small_kernel<W>          decode, up to 32 states: W lanes per problem, 32 / W problems per warp
//   viterbi_cta_kernel<G>            decode, more states: one CTA per problem (G = 1), value rows in shared memory
//
// A problem is one (clip) of viterbi / viterbi_discriminative, one (clip, label) of viterbi_binary.  A model is the
// transition matrix and initial distribution a problem is decoded with: one for viterbi / viterbi_discriminative,
// one per label for viterbi_binary (problem p uses model p % n_models).
#pragma once
#include <float.h>

#include "numerics.cuh"

namespace b2l_seq {
using namespace b2l;

enum LogMode { kLogPlain = 0, kLogDisc = 1, kLogBinary = 2 };

struct LogObsArgs {
  const void* prob;               // [clip][n_states][n_steps], C order
  long long n_clips, n_steps;
  int n_states;
  long long t_blocks;             // ceil(n_steps / blockDim.x): grid.x = n_clips * t_blocks
  double eps;                     // tiny of prob's dtype (plain, disc); tiny(float64) (binary)
  const double* log_marginal;     // disc: [n_states]; binary: [n_states][2]
  double* out;                    // plain / disc [clip][n_states][n_steps]; binary [clip][label][2][n_steps]; NULL:
                                  // verdict only
  int* flags;                     // [0] bit 0: the first data check failed; binary: [1 + label] = 1 when that
                                  // label's (1 - p) + p fails np.allclose(., 1)
};

// np.allclose(x, 1) for one element, in x's dtype (NumPy 2 casts the Python-float tolerance to float32 for float32 x):
// |x - 1| <= atol + rtol, or x == 1; NaN and +-inf fail.
__device__ __forceinline__ bool close_to_one(float x) { return fabsf(x - 1.0f) <= (float)(1e-08 + 1e-05) || x == 1.0f; }
__device__ __forceinline__ bool close_to_one(double x) { return fabs(x - 1.0) <= 1e-08 + 1e-05 || x == 1.0; }

// log in x's dtype.  float32: the float64 log rounded once to float32 — the correctly rounded value except in
// double-rounding cases far rarer than the ulp NumPy's own float32 log may be off by, so the two differ by at most
// 1 ulp (CUDA's logf is itself only within 1 ulp, and the two errors can add up to 2).
__device__ __forceinline__ double log_in(float x) { return (double)(float)log((double)x); }
__device__ __forceinline__ double log_in(double x) { return log(x); }

// One thread per (clip, frame); the states are walked in order, so the column sum of viterbi_discriminative is
// NumPy's sequential reduction over a non-last axis, in prob's dtype.
//   plain:  log(p + eps) in prob's dtype; check 0 <= p <= 1 (NaN passes).
//   disc:   log(p + eps) in prob's dtype, minus log_marginal in float64; check p >= 0 and allclose(sum_s p, 1).
//   binary: rows (1 - p) in prob's dtype and p, both as float64, log(. + eps) - log_marginal in float64; check
//           0 <= p <= 1 and, per label, allclose((1 - p) + p, 1) in float64.
template <class T, int MODE>
__global__ void __launch_bounds__(256) viterbi_logobs_kernel(const LogObsArgs a) {
  const long long clip = blockIdx.x / a.t_blocks;
  const long long t = (blockIdx.x % a.t_blocks) * blockDim.x + threadIdx.x;
  if (t >= a.n_steps) return;
  const int S = a.n_states;
  const long long T_ = a.n_steps;
  const T* x = static_cast<const T*>(a.prob) + clip * S * T_ + t;
  const T eps = (T)a.eps;
  bool bad = false;
  T sum = 0;
  for (int s = 0; s < S; ++s) {
    const T p = x[(long long)s * T_];
    if (MODE == kLogPlain) {
      bad |= p < (T)0 || p > (T)1;
      if (a.out) a.out[(clip * S + s) * T_ + t] = log_in(p + eps);
    } else if (MODE == kLogDisc) {
      bad |= p < (T)0;
      sum = s == 0 ? p : sum + p;
      if (a.out) a.out[(clip * S + s) * T_ + t] = log_in(p + eps) - a.log_marginal[s];
    } else {
      bad |= p < (T)0 || p > (T)1;
      const double q = (double)((T)1 - p), pd = (double)p;
      if (!close_to_one(q + pd)) a.flags[1 + s] = 1;
      if (a.out) {
        double* o = a.out + ((clip * S + s) * 2) * T_ + t;
        o[0] = log(q + a.eps) - a.log_marginal[2 * s];
        o[T_] = log(pd + a.eps) - a.log_marginal[2 * s + 1];
      }
    }
  }
  if (MODE == kLogDisc && !close_to_one(sum)) bad = true;
  if (bad) atomicOr(a.flags, 1);
}

struct DecodeArgs {
  const double* lp;               // [problem][n_states][n_steps]
  long long n_problems, n_steps;
  int n_states, n_models;
  // Predecessors of state j, ascending, as an ELL table of `deg` entries per state: entry m of j is state
  // idx[m][j] with log_trans[idx, j] = lt[m][j]; shorter lists are padded with (0, -inf), which never beats a
  // candidate.  dense: deg = n_states and entry m is state m (idx unused).
  int deg, dense;
  const double* lt;               // [model][deg][n_states]
  const unsigned short* idx;      // [model][deg][n_states]
  const double* log_p_init;       // [model][n_states]
  int tables_in_smem;             // stage lt / idx / log_p_init in shared memory
  unsigned short* ptr;            // [problem][n_steps][n_states] back-pointers (step 0 unused)
  unsigned short* states;         // [problem][n_steps]
  double* logp;                   // [problem]
};

// Shared memory of the staged model tables, in bytes (host mirror in sequence_api.cu).
__host__ __device__ inline size_t seq_table_bytes(int n_states, int n_models, int deg, int dense) {
  const size_t e = (size_t)n_models * deg * n_states;
  return e * 8 + (size_t)n_models * n_states * 8 + (dense ? 0 : (e * 2 + 7) / 8 * 8);
}

// Copies the model tables into shared memory (when they fit) and returns the base pointers every thread reads.
__device__ __forceinline__ void stage_tables(const DecodeArgs& a, unsigned char* smem, const double*& lt,
                                             const unsigned short*& idx, const double*& pi) {
  lt = a.lt;
  idx = a.idx;
  pi = a.log_p_init;
  if (!a.tables_in_smem) return;
  const size_t e = (size_t)a.n_models * a.deg * a.n_states, ns = (size_t)a.n_models * a.n_states;
  double* s_lt = reinterpret_cast<double*>(smem);
  double* s_pi = s_lt + e;
  unsigned short* s_idx = reinterpret_cast<unsigned short*>(s_pi + ns);
  for (size_t i = threadIdx.x; i < e; i += blockDim.x) s_lt[i] = a.lt[i];
  for (size_t i = threadIdx.x; i < ns; i += blockDim.x) s_pi[i] = a.log_p_init[i];
  if (!a.dense)
    for (size_t i = threadIdx.x; i < e; i += blockDim.x) s_idx[i] = a.idx[i];
  __syncthreads();
  lt = s_lt;
  idx = s_idx;
  pi = s_pi;
}

// Walks the back-pointers of one problem from its last state `s` (librosa/sequence.py:1250-1257).
__device__ __forceinline__ void backtrace(const DecodeArgs& a, long long p, int s) {
  const long long T_ = a.n_steps, S = a.n_states;
  const unsigned short* pt = a.ptr + p * T_ * S;
  unsigned short* st = a.states + p * T_;
  for (long long t = T_ - 1; t >= 0; --t) {
    st[t] = (unsigned short)s;
    if (t > 0) s = pt[t * S + s];
  }
}

// ------------------------------------------------------------------ up to 32 states
// W lanes per problem (W = the next power of two >= n_states, at least 2), 32 / W problems per warp, 128 threads.
// Lane j owns state j: value[t-1][k] comes from lane k by shuffle, and each lane scans its predecessors in
// ascending order and keeps a candidate only when cost > best (the reference's first-maximum rule: a NaN cost never
// wins, and with no candidate above -inf the pointer stays 0).  Every lane of the warp runs the same `deg` steps, so
// the shuffles always see the whole warp.  The last row's argmax is a butterfly over the group; lane 0 of the group
// walks the back-pointers, which its own warp wrote.
template <int W>
__global__ void __launch_bounds__(128) viterbi_small_kernel(const DecodeArgs a) {
  extern __shared__ __align__(16) unsigned char smem[];
  const double* lt_b;
  const unsigned short* idx_b;
  const double* pi_b;
  stage_tables(a, smem, lt_b, idx_b, pi_b);
  const int S = a.n_states, D = a.deg;
  const long long T_ = a.n_steps;
  const int j = threadIdx.x & (W - 1);
  const long long gp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) / W;
  const bool live = gp < a.n_problems && j < S;
  const long long p = gp < a.n_problems ? gp : a.n_problems - 1;
  const int jj = j < S ? j : S - 1;
  const int model = (int)(p % a.n_models);
  const double* lt = lt_b + (size_t)model * D * S + jj;
  const unsigned short* idx = idx_b + (size_t)model * D * S + jj;
  const double* lp = a.lp + (p * S + jj) * T_;
  unsigned short* pt = a.ptr + p * T_ * S + jj;
  double v = lp[0] + pi_b[(size_t)model * S + jj];
  for (long long t = 1; t < T_; ++t) {
    const double obs = lp[t];
    double best = -INFINITY;
    int arg = 0;
    for (int m = 0; m < D; ++m) {
      const int k = a.dense ? m : idx[(size_t)m * S];
      const double cost = __shfl_sync(0xffffffffu, v, k, W) + lt[(size_t)m * S];
      if (cost > best) { best = cost; arg = k; }
    }
    v = obs + best;
    if (live) pt[t * S] = (unsigned short)arg;
  }
  double bv = v;
  int bi = j < S ? j : kArgNone;
  warp_select<W>(bv, bi, ArgmaxMerge());
  __syncwarp();   // the group's back-pointer stores are visible to its lane 0
  if (live && j == 0) {
    a.logp[p] = bv;
    backtrace(a, p, bi);
  }
}

// ------------------------------------------------------------------ more states
// G problems per CTA of 256 threads; value[t-1] / value[t] of each problem live in shared memory (16 G bytes per
// state), the model tables in shared memory too when they fit (medium models) and otherwise are read through L2
// (large models).  A thread owns states j = tid, tid + 256, ...; each predecessor entry (k, log_trans[k, j]) is
// fetched once and used for all G problems, in ascending k with the first-maximum rule.  One block argmax per
// problem; warp g's lane 0 walks problem g's back-pointers.  Only G = 1 is launched: a tile of G = 4 clips per CTA,
// which reuses each log_trans fetch four times, took 502 ms against 395 ms for G = 1 on a dense 1024-state model over
// 64 clips x 1 000 frames (H100 80GB HBM3, 400 W limit) — a quarter of the CTAs on 132 SMs costs more than the L2
// traffic it saves.
template <int G>
__global__ void __launch_bounds__(256) viterbi_cta_kernel(const DecodeArgs a) {
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ double s_rv[32];
  __shared__ int s_ri[32];
  __shared__ int s_last[G];
  __shared__ double s_logp[G];
  const int S = a.n_states, D = a.deg, tid = threadIdx.x, nt = blockDim.x;
  const long long T_ = a.n_steps;
  double* val = reinterpret_cast<double*>(smem);                 // [2][G][S]
  const double* lt;
  const unsigned short* idx;
  const double* pi;
  stage_tables(a, smem + (size_t)2 * G * S * 8, lt, idx, pi);    // a single model (n_models == 1)
  const long long p0 = (long long)blockIdx.x * G;
  const double* lp[G];
#pragma unroll
  for (int g = 0; g < G; ++g) lp[g] = a.lp + (p0 + g < a.n_problems ? p0 + g : a.n_problems - 1) * S * T_;
  for (int j = tid; j < S; j += nt)
#pragma unroll
    for (int g = 0; g < G; ++g) val[g * S + j] = lp[g][(long long)j * T_] + pi[j];
  for (long long t = 1; t < T_; ++t) {
    __syncthreads();
    const double* prev = val + ((t - 1) & 1) * G * S;
    double* cur = val + (t & 1) * G * S;
    for (int j = tid; j < S; j += nt) {
      double best[G];
      int arg[G];
#pragma unroll
      for (int g = 0; g < G; ++g) { best[g] = -INFINITY; arg[g] = 0; }
#pragma unroll 4
      for (int m = 0; m < D; ++m) {
        const int k = a.dense ? m : idx[(size_t)m * S + j];
        const double l = lt[(size_t)m * S + j];
#pragma unroll
        for (int g = 0; g < G; ++g) {
          const double cost = prev[g * S + k] + l;
          if (cost > best[g]) { best[g] = cost; arg[g] = k; }
        }
      }
#pragma unroll
      for (int g = 0; g < G; ++g) {
        cur[g * S + j] = lp[g][(long long)j * T_ + t] + best[g];
        if (p0 + g < a.n_problems) a.ptr[((p0 + g) * T_ + t) * S + j] = (unsigned short)arg[g];
      }
    }
  }
  __syncthreads();
  const double* last = val + ((T_ - 1) & 1) * G * S;
  for (int g = 0; g < G; ++g) {
    double bv = -INFINITY;
    int bi = kArgNone;
    for (int j = tid; j < S; j += nt) ArgmaxMerge()(bv, bi, last[g * S + j], j);
    block_select(bv, bi, s_rv, s_ri, ArgmaxMerge());
    if (tid == 0) { s_last[g] = bi; s_logp[g] = bv; }
    __syncthreads();
  }
  const int w = tid >> 5;
  if (w < G && (tid & 31) == 0 && p0 + w < a.n_problems) {
    a.logp[p0 + w] = s_logp[w];
    backtrace(a, p0 + w, s_last[w]);
  }
}

}  // namespace b2l_seq
