// pitch_kernels.cuh — librosa.yin / librosa.pyin (librosa/core/pitch.py:369-931, sequence.py:1174-1259), librosa.piptrack
// and librosa.pitch_tuning (core/pitch.py:112-366).
//
//   yin_cmnd_kernel   frames -> cumulative mean normalised difference (CMND), float32 [row][lag]
//   yin_pick_kernel   CMND -> f0 of yin (first threshold trough, else the global minimum, + parabolic shift)
//   pyin_obs_kernel   CMND -> the voiced observation candidates of pyin (compact) and voiced_prob
//   viterbi_kernel    candidates -> decoded state path, f0 and voiced flag of pyin (one CTA per clip, float64)
//   piptrack_kernel   spectrogram rows -> the dense (pitches, mags) of librosa.piptrack (one warp per frame row)
//   sign_scan_kernel  the S.min() < 0 verdict of a device spectrogram, for piptrack_kernel
//   tuning_hist_kernel  frequencies -> the residual histogram of librosa.pitch_tuning
//
// A row is one (clip, frame) pair.  n_lags = max_period - min_period + 1 lags per row.
#pragma once
#include <float.h>

#include "common.cuh"
#include "fft_engine.cuh"
#include "numerics.cuh"

namespace b2l {

struct YinCmndArgs {
  const float* y;
  long long clip_stride;
  int n, n_clips, n_frames;
  int frame_length, hop, pad, pad_mode;
  int min_period, max_period;
  const float2* tw;    // FftCfg full twiddle table of the transform size
  float* cmnd;         // [row][n_lags]
  int* status;         // bit 0: a non-finite sample was read
};

// ------------------------------------------------------------------ stage 1: CMND
// One frame per group of TPF threads (the register FFT of fft_engine.cuh), 256 threads per CTA.  The frame is
// zero-padded to N = 2M >= frame_length + max_period + 1, so the circular autocorrelation equals the linear one
// on lags 0 .. max_period:
//   z = pack(x) -> Z = FFT_M(z) -> 2X (r2c un-mix) -> P = |2X|^2 -> c2r rebuild -> swapped FFT_M -> 4N r.
// Then, as the reference does in float32 (:394-406): E(m) = sum_{i<=m} x_i^2 except E(0) = 0,
// d(k) = 2 (r_0 - r_k) - E(k-1); and in float64 (the running mean divides by the int64 lag range, :411-417):
// cmnd(k) = d(k) / (mean_{1..k} d + tiny).
template <int LOG2M>
struct CmndCfg {
  static constexpr int M = 1 << LOG2M;
  static constexpr int TPF = M >= 32 ? M / 32 : 1;
  using Fft = FftCfg<LOG2M, TPF>;
  static constexpr int NT = 256;
  static constexpr int G = NT / TPF;    // frames per CTA round
  static constexpr int GS = TPF < 32 ? TPF : 32;   // threads of a group that run the scans
};

template <int LOG2M>
__global__ void __launch_bounds__(256) yin_cmnd_kernel(const YinCmndArgs a) {
  using K = CmndCfg<LOG2M>;
  using Cfg = typename K::Fft;
  constexpr int M = Cfg::M, N = 2 * M, PPT = Cfg::PPT, TPF = K::TPF, G = K::G, GS = K::GS;
  extern __shared__ __align__(128) unsigned char smem[];
  float2* s_tw = reinterpret_cast<float2*>(smem);
  const int tid = threadIdx.x, grp = tid / TPF, t = tid % TPF;
  float2* xbuf = s_tw + Cfg::TW_COUNT + grp * Cfg::XBUF_F2;
  float* r = reinterpret_cast<float*>(xbuf);    // autocorrelation r[0 .. N) after the inverse transform
  const int gbar = 1 + grp;
  for (int i = tid; i < Cfg::TW_COUNT; i += blockDim.x) s_tw[i] = a.tw[i];
  __syncthreads();

  const int n_lags = a.max_period - a.min_period + 1;
  const long long rows = (long long)a.n_clips * a.n_frames;
  const float inv4n = 1.0f / (4.0f * (float)N);
  // every group runs every round (groups past the end redo the last row and store nothing): sub-warp groups share
  // a warp, whose __syncwarp / shuffles need all of its lanes
  for (long long base = (long long)blockIdx.x * G; base < rows; base += (long long)gridDim.x * G) {
    const long long row = min(base + grp, rows - 1);
    const bool store = base + grp < rows;
    const int clip = (int)(row / a.n_frames);
    const float* yc = a.y + (long long)clip * a.clip_stride;
    const long long s0 = (row % a.n_frames) * (long long)a.hop - a.pad;
    bool bad = false;
    auto sample = [&](int i) -> float {
      if (i >= a.frame_length) return 0.0f;
      const float v = load_padded(yc, a.n, s0 + i, a.pad_mode, a.pad);
      bad |= !(fabsf(v) <= FLT_MAX);
      return v;
    };
    // ---- forward: z[e] = x[2e] + i x[2e+1]
    float2 v[PPT];
    load_pass0<Cfg>(v, t, [&](int e) { return make_float2(sample(2 * e), sample(2 * e + 1)); });
    fft_forward<Cfg>(v, t, gbar, xbuf, s_tw);
    if constexpr (Cfg::NPASS > 1) group_sync<TPF>(gbar);
    static_for<0, PPT>([&](auto S) {
      constexpr int slot = decltype(S)::value;
      xbuf[xphys(spectrum_index<Cfg>(t, slot))] = v[slot];
    });
    group_sync<TPF>(gbar);
    // ---- power spectrum and c2r rebuild, straight into the operands of the inverse transform's first pass
    static_for<0, PPT>([&](auto S) {
      constexpr int slot = decltype(S)::value;
      const int e = t + pass0_offset<Cfg>(slot);
      float sn, cs;
      sincospif((float)e * (2.0f / (float)N), &sn, &cs);
      const float2 w = make_float2(cs, -sn);                 // exp(-2 pi i e / N)
      float2 xa, xb;
      r2c_pair(xbuf[xphys(e)], xbuf[xphys((M - e) & (M - 1))], w, xa, xb);
      const float pa = sqmag(xa), pb = sqmag(xb);
      float2 A, B;
      c2r_pair(make_float2(pa, 0.0f), make_float2(pb, 0.0f), w, A, B);
      v[slot] = make_float2(A.y, A.x);                       // re/im swapped: the forward FFT then inverts
    });
    group_sync<TPF>(gbar);
    fft_forward<Cfg>(v, t, gbar, xbuf, s_tw);
    if constexpr (Cfg::NPASS > 1) group_sync<TPF>(gbar);
    static_for<0, PPT>([&](auto S) {
      constexpr int slot = decltype(S)::value;
      const int e = spectrum_index<Cfg>(t, slot);
      if (2 * e <= a.max_period) {
        r[2 * e] = v[slot].y * inv4n;
        r[2 * e + 1] = v[slot].x * inv4n;
      }
    });
    group_sync<TPF>(gbar);
    // ---- d(k), running mean and CMND: the first GS threads of the group walk the lags 32 (GS) at a time
    if (t < GS) {
      const float r0 = r[0];
      float e_prev = 0.0f;      // E(k-1) for the first lag of the chunk
      float dsum = 0.0f;        // sum of d(1 .. k-1)
      float* out = a.cmnd + row * n_lags;
      for (int k0 = 1; k0 <= a.max_period; k0 += GS) {
        const int k = k0 + t;
        const float xs = k - 1 < a.frame_length && k <= a.max_period ? sample(k - 1) : 0.0f;
        float ek = xs * xs;     // inclusive scan of x_{k-1}^2 -> E(k-1)
#pragma unroll
        for (int o = 1; o < GS; o <<= 1) {
          const float u = __shfl_up_sync(0xffffffffu, ek, o, GS);
          if (t >= o) ek += u;
        }
        ek += e_prev;
        // the reference zeroes its energy row 0 before it reads E(k-1), so d(1) = 2 (r_0 - r_1) (:402-406)
        const float d = k <= a.max_period ? 2.0f * (r0 - r[k]) - (k == 1 ? 0.0f : ek) : 0.0f;
        float ds = d;
#pragma unroll
        for (int o = 1; o < GS; o <<= 1) {
          const float u = __shfl_up_sync(0xffffffffu, ds, o, GS);
          if (t >= o) ds += u;
        }
        ds += dsum;
        if (k <= a.max_period && k >= a.min_period && store) {
          const double mean = (double)ds / (double)k;
          out[k - a.min_period] = (float)((double)d / (mean + DBL_MIN));
        }
        e_prev = __shfl_sync(0xffffffffu, ek, GS - 1, GS);
        dsum = __shfl_sync(0xffffffffu, ds, GS - 1, GS);
      }
    }
    if (store && bad && a.status) atomicOr(a.status, B2L_STATUS_NOT_FINITE_SAMPLE);
    group_sync<TPF>(gbar);    // r[] is read before the next round overwrites the exchange area
  }
}

// ------------------------------------------------------------------ decisions: shared helpers
// util.localmin with the pitch overrides: index 0 is x[0] < x[1], the last index x[-1] < x[-2] (:596-597, :872-874).
__device__ __forceinline__ bool pitch_trough(const float* x, int i, int n) {
  if (i == 0) return x[0] < x[1];
  if (i == n - 1) return x[n - 1] < x[n - 2];
  return x[i] < x[i - 1] && x[i] <= x[i + 1];
}
// _parabolic_interpolation at lag i, float64 (:421-477): 0 at both ends and where |b| >= |a|.
__device__ __forceinline__ double pitch_shift(const float* x, int i, int n) {
  if (i == 0 || i == n - 1) return 0.0;
  const double xm = x[i - 1], x0 = x[i], xp = x[i + 1];
  const double a = xp + xm - 2.0 * x0;
  const double b = (xp - xm) / 2.0;
  return fabs(b) >= fabs(a) ? 0.0 : -b / a;
}
// np.argmin order: the first NaN wins, else the first minimum.
struct ArgminMerge {
  __device__ __forceinline__ void operator()(float& v, int& i, float ov, int oi) const {
    if (before(ov, oi, v, i)) { v = ov; i = oi; }
  }
  static __device__ __forceinline__ bool before(float va, int ia, float vb, int ib) {
    const bool na = isnan(va), nb = isnan(vb);
    if (na != nb) return na;
    if (na) return ia < ib;
    return va < vb || (va == vb && ia < ib);
  }
};

// Copies one CMND row into the warp's shared slice.
__device__ __forceinline__ void load_row(float* dst, const float* src, int n, int lane) {
  for (int i = lane; i < n; i += 32) dst[i] = __ldg(src + i);
  __syncwarp();
}

// ------------------------------------------------------------------ stage 2: yin decision
// One warp per row: the first lag (ascending) that is a trough below the threshold, else the first global minimum;
// f0 = sr / (min_period + lag + shift(lag)) (:599-627).
__global__ void __launch_bounds__(256) yin_pick_kernel(const float* __restrict__ cmnd, long long rows, int n_lags,
                                                       int min_period, double sr, double threshold,
                                                       double* __restrict__ f0) {
  extern __shared__ __align__(16) float s_rows[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  float* x = s_rows + (size_t)warp * n_lags;
  for (long long row = (long long)blockIdx.x * nw + warp; row < rows; row += (long long)gridDim.x * nw) {
    load_row(x, cmnd + row * n_lags, n_lags, lane);
    int pick = -1;
    for (int base = 0; base < n_lags && pick < 0; base += 32) {
      const int i = base + lane;
      const bool hit = i < n_lags && pitch_trough(x, i, n_lags) && (double)x[i] < threshold;
      const unsigned m = __ballot_sync(0xffffffffu, hit);
      if (m) pick = base + __ffs(m) - 1;
    }
    if (pick < 0) {
      float bv = x[0];
      int bi = 0;
      for (int i = lane; i < n_lags; i += 32)
        if (ArgminMerge::before(x[i], i, bv, bi)) { bv = x[i]; bi = i; }   // the merge functor changes the code
      warp_select(bv, bi, ArgminMerge());
      pick = bi;
    }
    if (lane == 0) f0[row] = sr / ((double)(min_period + pick) + pitch_shift(x, pick, n_lags));
    __syncwarp();
  }
}

// ------------------------------------------------------------------ stage 3: pyin observations
struct PyinObsArgs {
  const float* cmnd;
  long long rows;
  int n_lags, min_period, max_cand;
  int n_thresholds, n_pitch_bins, n_bins_per_semitone;
  double sr, fmin, no_trough_prob;
  const double* thresholds;   // [n_thresholds + 1] np.linspace(0, 1, n_thresholds + 1)
  const double* beta;         // [n_thresholds]     np.diff(beta.cdf(thresholds))
  const double* beta_cum;     // [n_thresholds + 1] np.sum(beta[:c])
  const double* pmf;          // boltzmann.pmf(pos, lambda, n) at n (n - 1) / 2 + pos, n = 1 .. max_cand
  int* count;                 // [row] voiced candidates kept
  int* cand_bin;              // [row][max_cand] pitch bins, ascending
  double* cand_prob;          // [row][max_cand]
  double* voiced_prob;        // [row]
};

// Per-warp shared slice of pyin_obs_kernel, in bytes (host mirror in pitch_api.cu).
__host__ __device__ inline size_t pyin_obs_slice(int n_lags, int max_cand, int n_thresholds) {
  size_t b = (size_t)max_cand * 8;                   // probability of each trough
  b += ((size_t)n_lags * 4 + 7) / 8 * 8;             // the CMND row
  b += (size_t)max_cand * 8;                         // trough lag, threshold class
  b += (size_t)n_thresholds * 8;                     // running position and count per threshold
  return b;
}

// One warp per row, restating __pyin_helper (:868-931):
//   troughs in ascending lag; class c = number of thresholds[1:] that do not exceed the height (so the trough is
//   below thresholds j >= c); n_j = troughs below threshold j; a trough's prior at threshold j is
//   pmf(position among those troughs, lambda, n_j); prob = sum_j prior * beta_j; the global minimum among the troughs
//   gets no_trough_prob * sum(beta[:c]) more.  Troughs with prob == 0 are dropped (np.nonzero).  A candidate's bin is
//   rint(12 bins_per_semitone log2(f0 / fmin)) clipped to [0, n_pitch_bins]; the last write per bin wins (ascending
//   lag), and bin n_pitch_bins is an unvoiced state that is overwritten afterwards.  voiced_prob sums the voiced bins in
//   ascending order, clipped to [0, 1].  Consecutive troughs are >= 2 lags apart and |shift| < 1, so the periods rise
//   and the bins never increase along the trough list: equal bins are neighbours, and the list read backwards is in
//   ascending bin order.
__global__ void __launch_bounds__(128) pyin_obs_kernel(const PyinObsArgs a) {
  extern __shared__ __align__(128) unsigned char smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  unsigned char* base_ptr = smem + (size_t)warp * pyin_obs_slice(a.n_lags, a.max_cand, a.n_thresholds);
  double* s_p = reinterpret_cast<double*>(base_ptr);
  float* x = reinterpret_cast<float*>(s_p + a.max_cand);
  int* s_lag = reinterpret_cast<int*>(base_ptr + a.max_cand * 8 + ((size_t)a.n_lags * 4 + 7) / 8 * 8);
  int* s_cls = s_lag + a.max_cand;
  int* s_pos = s_cls + a.max_cand;
  int* s_nj = s_pos + a.n_thresholds;
  const int T = a.n_thresholds;
  const double bins_per_octave = (double)(12 * a.n_bins_per_semitone);
  for (long long row = (long long)blockIdx.x * nw + warp; row < a.rows; row += (long long)gridDim.x * nw) {
    load_row(x, a.cmnd + row * a.n_lags, a.n_lags, lane);
    // ---- troughs, ascending
    int n_tr = 0;
    for (int base = 0; base < a.n_lags; base += 32) {
      const int i = base + lane;
      const bool tr = i < a.n_lags && pitch_trough(x, i, a.n_lags);
      const unsigned m = __ballot_sync(0xffffffffu, tr);
      if (tr) s_lag[n_tr + __popc(m & ((1u << lane) - 1u))] = i;
      n_tr += __popc(m);
    }
    __syncwarp();
    // ---- threshold class of every trough, and the global minimum among the troughs
    float gv = 0.0f;
    int gi = 0x7fffffff;
    for (int q = lane; q < n_tr; q += 32) {
      const float h = x[s_lag[q]];
      int lo = 1, hi = T + 1;                 // first j in [1, T] with h < thresholds[j], else T + 1
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if ((double)h < a.thresholds[mid]) hi = mid;
        else lo = mid + 1;
      }
      s_cls[q] = lo - 1;
      if (gi == 0x7fffffff || ArgminMerge::before(h, q, gv, gi)) { gv = h; gi = q; }
    }
    if (gi == 0x7fffffff) gv = __int_as_float(0x7f800000);   // lanes without a trough: +inf, index past the end
    warp_select(gv, gi, ArgminMerge());
    for (int j = lane; j < T; j += 32) {
      int c = 0;
      for (int q = 0; q < n_tr; ++q) c += s_cls[q] <= j;
      s_nj[j] = c;
      s_pos[j] = 0;
    }
    __syncwarp();
    // ---- probability of every trough: prior at each threshold it is below, weighted by beta
    for (int q = 0; q < n_tr; ++q) {
      const int c = s_cls[q];
      double acc = 0.0;
      if (c < T) {
        for (int j = lane; j < T; j += 32) {
          if (c <= j) {
            const int pos = s_pos[j]++;
            const int nj = s_nj[j];
            acc += a.pmf[(size_t)nj * (nj - 1) / 2 + pos] * a.beta[j];
          }
        }
      }
      acc = warp_reduce(acc, [](double u, double v) { return u + v; });
      if (lane == 0) s_p[q] = acc;
    }
    __syncwarp();
    if (lane == 0 && n_tr > 0) s_p[gi] += a.no_trough_prob * a.beta_cum[s_cls[gi]];
    __syncwarp();
    // ---- candidates -> pitch bins (s_cls is reused for the bin of each trough; -1: dropped)
    for (int q = lane; q < n_tr; q += 32) {
      int bin = -1;
      if (s_p[q] != 0.0) {
        const int lag = s_lag[q];
        const double period = (double)(a.min_period + lag) + pitch_shift(x, lag, a.n_lags);
        const double f0 = a.sr / period;
        const double b = rint(bins_per_octave * log2(f0 / a.fmin));
        bin = (int)fmin(fmax(b, 0.0), (double)a.n_pitch_bins);
      }
      s_cls[q] = bin;
    }
    __syncwarp();
    if (lane == 0) {
      int* ob = a.cand_bin + row * a.max_cand;
      double* op = a.cand_prob + row * a.max_cand;
      int n_out = 0, prev_bin = -1;
      double vp = 0.0;
      for (int q = n_tr - 1; q >= 0; --q) {           // ascending bins; the first seen per bin is the last written
        const int bin = s_cls[q];
        if (bin < 0 || bin == prev_bin) continue;
        prev_bin = bin;
        if (bin >= a.n_pitch_bins) continue;
        ob[n_out] = bin;
        op[n_out] = s_p[q];
        vp += s_p[q];
        ++n_out;
      }
      a.count[row] = n_out;
      a.voiced_prob[row] = vp < 0.0 ? 0.0 : (vp > 1.0 ? 1.0 : vp);
    }
    __syncwarp();
  }
}

// ------------------------------------------------------------------ stage 4: Viterbi
struct ViterbiArgs {
  const int* count;           // stage 3 output, [clip][frame]
  const int* cand_bin;
  const double* cand_prob;
  const double* voiced_prob;
  int n_frames, max_cand, n_pitch_bins, n_states;
  double log_p_init;          // log(1 / n_states + tiny)
  double tiny;                // tiny(float64)
  // log_trans[k, j] of pyin's transition matrix kron(loop(2, 1 - switch_prob), local(n_pitch_bins, width)), exactly
  // as NumPy forms it: for source k = (a, p) and target j = (b, q), local[p, q] = window(q - p) / rowsum[p] and the
  // value depends only on the class of rowsum[p], on d = q - p and on a == b:
  //   ltab[(cls[p] * 2 + (a != b)) * (2 hw + 1) + d + hw]  for |d| <= hw,  log(tiny) outside the band.
  // Predecessors of j: every k with log_trans[k, j] >= log_thr, ascending (every k when `full`).
  const int* cls;             // [n_pitch_bins]
  const double* ltab;
  int half_width, full;
  double log_thr;
  const double* freqs;        // [n_pitch_bins] fmin * 2^(bin / (12 bins_per_semitone))
  int fill;                   // unvoiced f0 = fill_na when set
  double fill_na;
  unsigned short* ptr;        // [clip][frame][state] back-pointers (frame 0 unused)
  unsigned short* states;     // [clip][frame]
  double* f0;                 // [clip][frame] (may be NULL)
  unsigned char* voiced;      // [clip][frame] (may be NULL)
};

// One CTA per clip, frames in order (librosa/sequence.py:1206-1259).  value[t-1] / value[t] live in shared memory; a
// thread owns states j = tid, tid + blockDim, ...; for each it scans the predecessors (the band |q - p| <= hw of each
// voicing half, or every state for a full search) in ascending k and keeps a candidate only when cost > best — the
// reference's first-maximum rule.  log P(obs | state) = log(p + tiny): the candidate probability for voiced bins
// that have one, 0 for the other voiced bins, (1 - voiced_prob) / n_pitch_bins for the unvoiced half.
// Shared memory: 18 bytes per state (two value rows, one mark).  The log-transition table is read through L1.
__host__ __device__ inline size_t viterbi_smem(int n_states) { return (size_t)n_states * 18; }

__global__ void __launch_bounds__(256) viterbi_kernel(const ViterbiArgs a) {
  extern __shared__ __align__(128) unsigned char smem[];
  const int S = a.n_states, tid = threadIdx.x, nt = blockDim.x;
  double* val0 = reinterpret_cast<double*>(smem);
  double* val1 = val0 + S;
  unsigned short* s_mark = reinterpret_cast<unsigned short*>(val1 + S);   // candidate index + 1 of a voiced bin, else 0
  __shared__ double s_red_v[32];
  __shared__ int s_red_i[32];
  for (int j = tid; j < S; j += nt) s_mark[j] = 0;
  const int clip = blockIdx.x;
  const long long row0 = (long long)clip * a.n_frames;
  const double log_zero = log(a.tiny);
  const int npb = a.n_pitch_bins, hw = a.half_width, wn = 2 * a.half_width + 1;
  auto mark = [&](long long row) {
    const int cnt = a.count[row];
    for (int c = tid; c < cnt; c += nt) s_mark[a.cand_bin[row * a.max_cand + c]] = (unsigned short)(c + 1);
  };
  // log-observation of state j at `row` (clears j's mark)
  auto log_obs = [&](long long row, int j, double log_unvoiced) -> double {
    if (j >= npb) return log_unvoiced;
    const int m = s_mark[j];
    if (!m) return log_zero;
    s_mark[j] = 0;
    return log(a.cand_prob[row * a.max_cand + (m - 1)] + a.tiny);
  };
  auto unvoiced = [&](long long row) { return log((1.0 - a.voiced_prob[row]) / (double)npb + a.tiny); };
  __syncthreads();
  mark(row0);
  __syncthreads();
  {
    const double lu = unvoiced(row0);
    for (int j = tid; j < S; j += nt) val0[j] = log_obs(row0, j, lu) + a.log_p_init;
  }
  double* prev = val0;
  double* cur = val1;
  for (int t = 1; t < a.n_frames; ++t) {
    const long long row = row0 + t;
    __syncthreads();     // the previous row is complete and its marks are cleared
    mark(row);
    __syncthreads();
    const double lu = unvoiced(row);
    unsigned short* pt = a.ptr + row * S;
    for (int j = tid; j < S; j += nt) {
      double best = -INFINITY;
      int arg = 0;
      const int q = j % npb, b = j >= npb;
      const int p_lo = a.full ? 0 : max(0, q - hw), p_hi = a.full ? npb - 1 : min(npb - 1, q + hw);
      for (int h = 0; h < 2; ++h) {
        const double* lt_h = a.ltab + (h != b) * wn + hw + q;   // + cls * 2 wn - p
        for (int p = p_lo; p <= p_hi; ++p) {
          const int d = q - p;
          const double lt = (d >= -hw && d <= hw) ? __ldg(lt_h + 2 * wn * __ldg(a.cls + p) - p) : log_zero;
          if (!a.full && !(lt >= a.log_thr)) continue;
          const int k = h * npb + p;
          const double cost = prev[k] + lt;
          if (cost > best) { best = cost; arg = k; }
        }
      }
      pt[j] = (unsigned short)arg;
      cur[j] = log_obs(row, j, lu) + best;
    }
    double* tmp = prev; prev = cur; cur = tmp;
  }
  __syncthreads();
  // ---- first argmax of the last row (np.argmax: the first NaN, else the first maximum)
  double bv = -INFINITY;
  int bi = kArgNone;
  for (int j = tid; j < S; j += nt) ArgmaxMerge()(bv, bi, prev[j], j);
  block_select(bv, bi, s_red_v, s_red_i, ArgmaxMerge());
  if (tid == 0) {
    // ---- backtrace and the state -> (f0, voiced) map (:844-850)
    int s = bi;
    for (int t = a.n_frames - 1; t >= 0; --t) {
      const long long row = row0 + t;
      a.states[row] = (unsigned short)s;
      if (a.f0) {
        const bool v = s < npb;
        a.f0[row] = (!v && a.fill) ? a.fill_na : a.freqs[s % npb];
        a.voiced[row] = v;
      }
      if (t > 0) s = a.ptr[row * S + s];
    }
  }
}

// ------------------------------------------------------------------ piptrack / pitch_tuning
// librosa.piptrack (core/pitch.py:182-366) and librosa.pitch_tuning (:112-179) in the reference's roundings: every
// operation the reference does in the spectrogram's type T is one separately rounded operation here (no contracted
// FMA), and what it promotes to float64 is computed in float64 and rounded once.

// Bits of b2l_piptrack's sign word: what S.min() < 0 needs (a NaN makes the minimum NaN, which is not < 0).
constexpr unsigned kSignNegative = 1u, kSignNaN = 2u;

// One pass over n values: sets kSignNegative when one is < 0 and kSignNaN when one is NaN.
template <class T>
__global__ void __launch_bounds__(256) sign_scan_kernel(const T* __restrict__ x, long long n, unsigned* __restrict__ word) {
  unsigned bits = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const T v = __ldg(x + i);
    bits |= (v < T(0) ? kSignNegative : 0u) | (v != v ? kSignNaN : 0u);
  }
  bits = __reduce_or_sync(0xffffffffu, bits);
  if ((threadIdx.x & 31) == 0 && bits) atomicOr(word, bits);
}

template <class T>
struct PiptrackArgs {
  const T* S;                // [clip] x (F bins, n_frames frames); bin k of frame t at t * frame_stride + k * bin_stride
  long long n_rows;          // n_clips * n_frames
  long long n_frames;
  long long frame_stride, bin_stride;
  int F;
  int k_lo, k_hi;            // bins with fmin <= f < fmax
  int abs_mode;              // 0 S as it is, 1 |S|, 2 |S| when the sign word says S.min() < 0
  const unsigned* sign;      // abs_mode 2: the word sign_scan_kernel wrote
  int ref_frame;             // 1: ref = threshold * max over the frame (np.max: NaN propagates), 0: ref_abs
  int thr_wide;              // threshold * max in float64 (threshold a float64 scalar) rather than in T
  double threshold, ref_abs;
  double sr, n_fft;
  T* pitches;                // [row][F]: zero off the peaks
  T* mags;
};

// One warp per (clip, frame) row: the row goes through the warp's slot of shared memory (|.| applied), the frame
// reference is formed, and every bin of both output rows is written: the interpolated peak where freq_mask &
// localmax(S * (S > ref)) holds, zero elsewhere.  The product is formed literally, so inf * 0 is NaN.
template <class T>
__global__ void __launch_bounds__(256) piptrack_kernel(const PiptrackArgs<T> a) {
  extern __shared__ __align__(16) unsigned char pip_smem[];
  const int nw = blockDim.x >> 5, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int F = a.F;
  T* s_row = reinterpret_cast<T*>(pip_smem) + (size_t)warp * ((F + 3) & ~3);
  const bool use_abs = a.abs_mode == 1 || (a.abs_mode == 2 && (*a.sign & (kSignNegative | kSignNaN)) == kSignNegative);
  const T thr_t = narrow<T>(a.threshold);   // NumPy's threshold * max in T (a Python float is cast to T)
  for (long long r = (long long)blockIdx.x * nw + warp; r < a.n_rows; r += (long long)gridDim.x * nw) {
    const long long clip = r / a.n_frames, t = r - clip * a.n_frames;
    const T* src = a.S + clip * F * a.n_frames + t * a.frame_stride;
    T mx = T(-INFINITY);
    bool nan = false;
    for (int i = lane; i < F; i += 32) {
      T v = __ldg(src + i * a.bin_stride);
      if (use_abs) v = fabs(v);
      s_row[i] = v;
      nan |= v != v;
      mx = fmax(mx, v);
    }
    mx = warp_reduce(mx, [](T u, T v) { return fmax(u, v); });
    if (__any_sync(0xffffffffu, nan)) mx = T(NAN);
    __syncwarp();
    double ref = a.ref_abs;
    if (a.ref_frame) ref = a.thr_wide ? __dmul_rn(a.threshold, (double)mx) : (double)mul_rn(thr_t, mx);
    T* po = a.pitches + r * F;
    T* mo = a.mags + r * F;
    for (int k = lane; k < F; k += 32) {
      T pitch = T(0), mag = T(0);
      if (k >= a.k_lo && k < a.k_hi && k > 0) {
        const bool last = k == F - 1;
        const T l = s_row[k - 1], c = s_row[k], rr = last ? c : s_row[k + 1];
        auto thr = [&](T v) { return (double)v > ref ? v : mul_rn(v, T(0)); };   // S * (S > ref)
        if (local_extremum(true, k, F, thr(l), thr(c), thr(rr))) {
          T shift = T(0), avg;
          if (last) {
            avg = sub_rn(c, l);                                     // np.gradient: one-sided at the edge
          } else {
            avg = mul_rn(sub_rn(rr, l), T(0.5));                    // (S[k+1] - S[k-1]) / 2
            shift = parabolic_shift(l, c, rr);
          }
          mag = parabolic_mag(c, avg, shift);
          pitch = narrow<T>(__ddiv_rn(__dmul_rn(__dadd_rn((double)k, (double)shift), a.sr), a.n_fft));
        }
      }
      po[k] = pitch;
      mo[k] = mag;
    }
    __syncwarp();
  }
}

// pitch_tuning's residual histogram: over the n values of f, count those > 0 (counts[n_bins]) and bin the residual
// mod(bins_per_octave * log2(f / 27.5), 1), folded to [-0.5, 0.5), into n_bins <= 2048 bins with float64 edges and
// np.histogram's rule (edges[b] <= x < edges[b + 1], the last bin closed).  The residual is computed in T with
// np.mod's rounding (fmod, then + 1 when negative); log2 is the float64 log2 rounded to T.  A NaN residual (f = inf)
// is dropped, as np.histogram drops it.
template <class T>
__global__ void __launch_bounds__(256) tuning_hist_kernel(const T* __restrict__ f, long long n, T bins_per_octave,
                                                          int n_bins, const double* __restrict__ edges,
                                                          unsigned long long* __restrict__ counts) {
  __shared__ unsigned int s_cnt[2048];
  for (int i = threadIdx.x; i < n_bins; i += blockDim.x) s_cnt[i] = 0;
  __syncthreads();
  unsigned int positive = 0;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const T v = __ldg(f + e);
    if (!(v > T(0))) continue;
    ++positive;
    const T res = tuning_residual(v, bins_per_octave);
    if (res != res) continue;
    atomicAdd(&s_cnt[residual_bin(res, n_bins, edges)], 1u);
  }
  positive = __reduce_add_sync(0xffffffffu, positive);
  if ((threadIdx.x & 31) == 0 && positive) atomicAdd(&counts[n_bins], (unsigned long long)positive);
  __syncthreads();
  for (int i = threadIdx.x; i < n_bins; i += blockDim.x)
    if (s_cnt[i]) atomicAdd(&counts[i], (unsigned long long)s_cnt[i]);
}

}  // namespace b2l
