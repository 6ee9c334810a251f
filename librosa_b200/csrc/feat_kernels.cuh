// feat_kernels.cuh — frame-wise features that sit next to the FFT path: spectral statistics of a stored
// magnitude spectrogram (the S= form of librosa.feature.spectral_centroid / bandwidth / rolloff / flatness /
// rms; the y= form is fused into fwd_kernel, MODE_STATS) and the two time-domain framings that need no FFT
// (rms(y=...), zero_crossing_rate), then the plan-free kernels over spectrograms and signals: onset strength, pcen,
// spectral contrast, piptrack, HPSS, reassignment, phase vocoder, resampling, power_to_db, the Griffin-Lim update
// and a batched transpose used as a layout adapter.  Included by feature_api.cu only.
#pragma once
#include "common.cuh"
#include "numerics.cuh"
#include "stats.cuh"

namespace b2l {

// S [n_rows][F] (one row per (clip, frame), bins contiguous) -> out [clip][N_STATS][n_frames].
// One warp per row: coalesced copy into shared memory, then frame_stats.  Sets B2L_STATUS_NEGATIVE_ENTRY when a
// negative entry is seen (the reference raises "only defined with non-negative energies").
__global__ void stats_kernel(const float* __restrict__ S, long long n_rows, int n_frames, int F,
                             const float* __restrict__ freq, StatsParams sp, float* __restrict__ out, int* status) {
  extern __shared__ __align__(16) float s_dyn[];
  const int nw = blockDim.x >> 5, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int Fp = (F + 3) & ~3;
  float* s_freq = s_dyn;
  float* s_row = s_dyn + Fp + (size_t)warp * Fp;
  for (int i = threadIdx.x; i < F; i += blockDim.x) s_freq[i] = freq[i];
  __syncthreads();
  for (long long r = (long long)blockIdx.x * nw + warp; r < n_rows; r += (long long)gridDim.x * nw) {
    const float* src = S + r * F;
    for (int i = lane; i < F; i += 32) s_row[i] = __ldg(src + i);
    __syncwarp();
    bool negative;
    const float v = frame_stats(s_row, s_freq, F, lane, sp, &negative);
    if (negative && lane == 0) atomicOr(status, B2L_STATUS_NEGATIVE_ENTRY);
    const long long clip = r / n_frames, frame = r % n_frames;
    if (lane < N_STATS) out[(clip * N_STATS + lane) * n_frames + frame] = v;
    __syncwarp();
  }
}

// Time-domain framing features.  Frame t of a clip covers padded samples [t*hop - pad, t*hop - pad + L).
//   what == 0: rms       sqrt(mean(x^2))                      (librosa/feature/spectral.py:881-890)
//   what == 1: the number of zero crossings inside the frame  (librosa/feature/spectral.py:1115-1133,
//              librosa/core/audio.py:1588-1602): samples with |x| <= threshold count as +0, a crossing at
//              position i >= 1 is signbit(x[i]) != signbit(x[i-1]) (zero_pos) or sign(x[i]) != sign(x[i-1]);
//              position 0 contributes `pad_first`.  Written as count * out_scale: callers that need the
//              float64 mean of the reference pass 1 and divide on the host.
// One warp per frame; the 4x overlap between frames is served by L1 / L2.
__global__ void frame_td_kernel(const float* __restrict__ y, long long clip_stride, int n, long long n_clips,
                                int L, int hop, int pad, int pad_mode, int n_frames, int what, float threshold,
                                int zero_pos, int pad_first, float out_scale, float* __restrict__ out, int* status) {
  const int nw = blockDim.x >> 5, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long total = n_clips * n_frames;
  for (long long r = (long long)blockIdx.x * nw + warp; r < total; r += (long long)gridDim.x * nw) {
    const long long clip = r / n_frames;
    const int frame = (int)(r % n_frames);
    const float* yc = y + clip * clip_stride;
    const long long s0 = (long long)frame * hop - pad;
    if (what == 0) {
      float acc = 0.0f;
      for (int i = lane; i < L; i += 32) {
        const float x = load_padded(yc, n, s0 + i, pad_mode, pad);
        acc = fmaf(x, x, acc);
      }
      acc = warp_sum(acc);
      if (lane == 0) out[r] = sqrtf(acc / (float)L);
    } else {
      int count = 0;
      bool bad = false;
      // class of a sample: 0 = non-negative / zero, 1 = negative (zero_pos) or -1/0/+1 (sign form)
      auto cls = [&](float x) -> int {
        if (!(fabsf(x) <= 3.0e38f)) bad = true;
        if (fabsf(x) <= threshold) x = 0.0f;
        return zero_pos ? (int)(x < 0.0f) : (x > 0.0f) - (x < 0.0f);
      };
      for (int base = 0; base < L; base += 32) {
        const int i = base + lane;
        const int c = i < L ? cls(load_padded(yc, n, s0 + i, pad_mode, pad)) : 0;
        int prev = __shfl_up_sync(0xffffffffu, c, 1);
        if (lane == 0 && i > 0 && i < L) prev = cls(load_padded(yc, n, s0 + i - 1, pad_mode, pad));
        const bool cross = i < L && (i == 0 ? pad_first != 0 : c != prev);
        count += __popc(__ballot_sync(0xffffffffu, cross));
      }
      if (__any_sync(0xffffffffu, bad) && lane == 0) atomicOr(status, B2L_STATUS_NOT_FINITE_SAMPLE);
      if (lane == 0) out[r] = (float)count * out_scale;
    }
  }
}

// The same two features when frame_length is a multiple of hop_length (the usual 2048 / 512): every sample is
// read ONCE.  The padded signal is cut into blocks of hop samples; a CTA takes FRAMES consecutive frames of one
// clip, reduces the FRAMES + R - 1 blocks they cover (R = frame_length / hop) — one warp per block, 16-byte
// coalesced loads for blocks inside the clip, the np.pad index map for the few that touch the padding — and
// then every frame is the sum of R block values:
//   rms:  block value = sum of squares;
//   zero crossings:  block value = number of positions p in the block whose sample differs in sign class from
//         the sample at p - 1 (which may lie in the previous block); a frame counts the crossings at its
//         positions 1 .. L-1, i.e. the block sum minus the crossing AT its first position, plus `pad_first`.
// frame_td_kernel (one warp per frame) re-reads every sample frame_length / hop times through a 64-bit modulo
// index map: 1.96 ms / 3.5 ms for the 903 MB of cfg-2 shapes against a 0.14 ms traffic floor.
constexpr int TD_FRAMES = 64;
__global__ void __launch_bounds__(256) frame_td_block_kernel(const float* __restrict__ y, long long clip_stride, int n, int L,
                                                             int hop, int pad, int pad_mode, int n_frames, int what,
                                                             float threshold, int zero_pos, int pad_first, float out_scale,
                                                             float* __restrict__ out, int* status) {
  extern __shared__ __align__(16) unsigned char s_td[];
  const int R = L / hop;
  const int nblk = TD_FRAMES + R - 1;
  float* s_val = reinterpret_cast<float*>(s_td);             // per block: sum of squares / crossing count
  int* s_first = reinterpret_cast<int*>(s_val + nblk);       // per block: crossing at its first position
  const int clip = blockIdx.y, t0 = blockIdx.x * TD_FRAMES;
  const float* yc = y + (long long)clip * clip_stride;
  const int nw = blockDim.x >> 5, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool vec_ok = ((reinterpret_cast<uintptr_t>(yc) & 15) == 0) && (hop % 4 == 0) && (pad % 4 == 0);
  bool bad = false;
  auto cls = [&](float x) -> int {
    if (!(fabsf(x) <= 3.0e38f)) bad = true;
    if (fabsf(x) <= threshold) x = 0.0f;
    return zero_pos ? (int)(x < 0.0f) : (x > 0.0f) - (x < 0.0f);
  };
  for (int b = warp; b < nblk; b += nw) {
    const long long p0 = (long long)(t0 + b) * hop - pad;      // first position of the block
    const bool inside = p0 >= 1 && p0 + hop <= n;              // the sample before the block is in range too
    float acc = 0.0f;
    int cnt = 0, first = 0;
    if (what == 0) {
      if (inside && vec_ok) {
        const float4* src = reinterpret_cast<const float4*>(yc + p0);
        for (int i = lane; i < hop / 4; i += 32) {
          const float4 v = __ldg(src + i);
          acc = fmaf(v.x, v.x, acc);
          acc = fmaf(v.y, v.y, acc);
          acc = fmaf(v.z, v.z, acc);
          acc = fmaf(v.w, v.w, acc);
        }
      } else {
        for (int i = lane; i < hop; i += 32) {
          const float x = load_padded(yc, n, p0 + i, pad_mode, pad);
          acc = fmaf(x, x, acc);
        }
      }
      acc = warp_sum(acc);
      if (lane == 0) s_val[b] = acc;
    } else if (inside && vec_ok) {
      // four consecutive samples per lane: three comparisons inside the lane, one with the previous lane's last
      // sample (the lane before lane 0 of a 128-sample step is the previous step's lane 31, or the sample before
      // the block)
      const float4* src = reinterpret_cast<const float4*>(yc + p0);
      int carry = cls(__ldg(yc + p0 - 1));            // class of the sample before the current 128-sample step
      for (int base = 0; base < hop / 4; base += 32) {
        const int i = base + lane;
        const bool live = i < hop / 4;
        const float4 v = live ? __ldg(src + i) : make_float4(0.f, 0.f, 0.f, 0.f);
        const int c0 = cls(v.x), c1 = cls(v.y), c2 = cls(v.z), c3 = cls(v.w);
        int prev = __shfl_up_sync(0xffffffffu, c3, 1);
        if (lane == 0) prev = carry;
        const int x0 = live && c0 != prev;
        if (base == 0 && lane == 0) first = x0;
        cnt += live ? x0 + (c1 != c0) + (c2 != c1) + (c3 != c2) : 0;
        carry = __shfl_sync(0xffffffffu, c3, 31);
      }
      cnt = (int)warp_sum((float)cnt);                 // counts stay far below 2^24: exact in float
      first = __shfl_sync(0xffffffffu, first, 0);
      if (lane == 0) {
        s_val[b] = (float)cnt;
        s_first[b] = first;
      }
    } else {
      for (int base = 0; base < hop; base += 32) {
        const int i = base + lane;
        const int c = i < hop ? cls(inside ? __ldg(yc + p0 + i) : load_padded(yc, n, p0 + i, pad_mode, pad)) : 0;
        int prev = __shfl_up_sync(0xffffffffu, c, 1);
        if (lane == 0 && i < hop) prev = cls(inside ? __ldg(yc + p0 + i - 1) : load_padded(yc, n, p0 + i - 1, pad_mode, pad));
        const bool cross = i < hop && c != prev;
        const unsigned m = __ballot_sync(0xffffffffu, cross);
        cnt += __popc(m);
        if (base == 0) first = (int)(m & 1u);
      }
      if (lane == 0) {
        s_val[b] = (float)cnt;
        s_first[b] = first;
      }
    }
  }
  if (what != 0 && __any_sync(0xffffffffu, bad) && lane == 0) atomicOr(status, B2L_STATUS_NOT_FINITE_SAMPLE);
  __syncthreads();
  for (int f = threadIdx.x; f < TD_FRAMES; f += blockDim.x) {
    const int t = t0 + f;
    if (t >= n_frames) break;
    float acc = 0.0f;
    for (int r = 0; r < R; ++r) acc += s_val[f + r];
    float* o = out + (long long)clip * n_frames + t;
    if (what == 0) *o = sqrtf(acc / (float)L);
    else *o = (acc - (float)s_first[f] + (float)(pad_first != 0)) * out_scale;
  }
}

// Spectral-flux onset strength (librosa/onset.py:445-640, onset_strength_multi) from a dB-scaled spectrogram
// S [clip][rows][T]:  env[c][t'] = mean_{m in channel c} max(0, S[m][t' + lag] - ref[m][t']),  ref = S after a
// maximum filter of `max_size` rows (scipy.ndimage.maximum_filter1d, reflect boundary), then shifted right by
// pad_width = lag (+ n_fft // (2 hop) when centred) and cut to T frames.  One thread per output frame, so
// every row access is coalesced; n_ch == 0 writes the un-aggregated flux of every row (aggregate=False).
struct OnsetArgs {
  int bounds[33];
  int n_ch, lag, max_size, pad_width, n_rows, T;
};
// The flux of row m at lag frame tp: np.maximum(0, S[m][tp + lag] - ref[m][tp]), a NaN difference kept (as
// np.maximum keeps it).  The max filter lets a NaN in the window through as NaN (np.maximum's rule; scipy's
// running-max filter returns a NaN or skips it depending on where it sits in the window).
__device__ __forceinline__ float onset_flux(const float* __restrict__ Sc, const OnsetArgs& a, int m, int tp) {
  float ref;
  if (a.max_size == 1) {
    ref = Sc[(long long)m * a.T + tp];
  } else {
    ref = -INFINITY;
    const int lo = m - a.max_size / 2;
    for (int j = 0; j < a.max_size; ++j) {
      int mm = lo + j;
      while (mm < 0 || mm >= a.n_rows) mm = mm < 0 ? -mm - 1 : 2 * a.n_rows - mm - 1;
      ref = MaxNan()(ref, Sc[(long long)mm * a.T + tp]);
    }
  }
  const float d = sub_rn(Sc[(long long)m * a.T + tp + a.lag], ref);
  return d != d ? d : fmaxf(0.0f, d);
}
__global__ void onset_kernel(const float* __restrict__ S, OnsetArgs a, float* __restrict__ out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= a.T) return;
  const long long clip = blockIdx.y;   // the entry offsets S and out per slice of at most 65 535 clips
  const float* Sc = S + clip * (long long)a.n_rows * a.T;
  const int tp = t - a.pad_width;
  const bool live = tp >= 0 && tp + a.lag < a.T;
  const int n_out = a.n_ch > 0 ? a.n_ch : a.n_rows;
  float* oc = out + clip * (long long)n_out * a.T + t;
  if (a.n_ch == 0) {
    for (int m = 0; m < a.n_rows; ++m) oc[(long long)m * a.T] = live ? onset_flux(Sc, a, m, tp) : 0.0f;
    return;
  }
  for (int c = 0; c < a.n_ch; ++c) {
    float acc = 0.0f;
    const int m0 = a.bounds[c], m1 = a.bounds[c + 1];
    if (live)
      for (int m = m0; m < m1; ++m) acc = add_rn(acc, onset_flux(Sc, a, m, tp));
    oc[(long long)c * a.T] = live && m1 > m0 ? div_rn(acc, (float)(m1 - m0)) : (live ? __int_as_float(0x7fc00000) : 0.0f);
  }
}
// The same flux aggregated with np.median over each channel's rows (util.sync(..., aggregate=np.median)): for an
// even row count the float32 mean of the two middle values, NaN when any flux of the column is NaN (np.maximum
// keeps it).  A CTA takes kOnsetMedFrames frames of one clip and one channel at a time: the flux tile is staged
// [frame][row] in shared memory (rows read coalesced along time), then one warp per frame bitonic-sorts its
// column of P = next power of two >= rows (padded with +inf) and reads the middle.  Channels up to
// kOnsetMedMaxRows rows (the entry point refuses more).
constexpr int kOnsetMedFrames = 16;
constexpr int kOnsetMedMaxRows = 512;
__global__ void onset_median_kernel(const float* __restrict__ S, OnsetArgs a, int P, float* __restrict__ out) {
  extern __shared__ float s_col[];   // [kOnsetMedFrames][P + 1]
  const int t0 = blockIdx.x * kOnsetMedFrames;
  const long long clip = blockIdx.y;
  const float* Sc = S + clip * (long long)a.n_rows * a.T;
  float* oc = out + clip * (long long)a.n_ch * a.T;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
  const int f_ld = threadIdx.x % kOnsetMedFrames, r_ld = threadIdx.x / kOnsetMedFrames;
  const int r_step = blockDim.x / kOnsetMedFrames;
  for (int c = 0; c < a.n_ch; ++c) {
    const int m0 = a.bounds[c], R = a.bounds[c + 1] - m0;
    {
      const int t = t0 + f_ld, tp = t - a.pad_width;
      const bool live = t < a.T && tp >= 0 && tp + a.lag < a.T;
      for (int r = r_ld; r < P; r += r_step) {
        float v = INFINITY;
        if (r < R && live) v = onset_flux(Sc, a, m0 + r, tp);
        s_col[f_ld * (P + 1) + r] = v;
      }
    }
    __syncthreads();
    for (int f = warp; f < kOnsetMedFrames; f += n_warps) {
      const int t = t0 + f, tp = t - a.pad_width;
      if (t >= a.T) continue;
      float* col = s_col + f * (P + 1);
      bool nan = false;
      for (int r = lane; r < R; r += 32) nan |= col[r] != col[r];
      nan = __any_sync(0xffffffffu, nan);
      const bool live = tp >= 0 && tp + a.lag < a.T;
      if (live && R > 0 && !nan) {
        for (int k = 2; k <= P; k <<= 1)
          for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = lane; i < P; i += 32) {
              const int p = i ^ j;
              if (p > i) {
                const float x = col[i], y = col[p];
                if (((i & k) == 0) == (x > y)) { col[i] = y; col[p] = x; }
              }
            }
            __syncwarp();
          }
      }
      if (lane == 0) {
        float v = 0.0f;
        if (live)
          v = R == 0 || nan ? __int_as_float(0x7fc00000)
                            : (R & 1 ? col[R >> 1] : __fmul_rn(__fadd_rn(col[(R >> 1) - 1], col[R >> 1]), 0.5f));
        oc[(long long)c * a.T + t] = v;
      }
    }
    __syncthreads();
  }
}

// detrend: scipy.signal.lfilter([1, -1], [1, -0.99]) along time (direct form II transposed), one thread per row,
// in float32 with one rounding per operation (the error bound is derived in tests/test_gpu_feature_kernels_tail.py)
__global__ void detrend_kernel(float* __restrict__ x, long long n_rows, int T) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_rows) return;
  float* xr = x + r * T;
  float z = 0.0f;
  for (int t = 0; t < T; ++t) {
    const float in = xr[t];
    const float y = add_rn(in, z);
    z = sub_rn(mul_rn(0.99f, y), in);
    xr[t] = y;
  }
}

// Per-channel energy normalisation (librosa/core/spectrum.py:2396-2666, pcen) of S [n_rows][T] (time contiguous):
//   M[t] = b * ref[t] + (1 - b) * M[t-1]              scipy.signal.lfilter([b], [1, b-1], ref, zi)  (:2629)
//   smooth = exp(-gain * (log(eps) + log1p(M / eps)))                                             (:2633)
//   out = log1p(S*smooth) | exp(power*(log S + log smooth)) | bias^power * expm1(power*log1p(S*smooth/bias))
// The recurrence is sequential in time and independent per row: a warp takes 32 rows, stages 32 x 32 tiles
// through shared memory so that global accesses are coalesced along time while each lane walks its own row.
struct PcenArgs {
  float gain, bias, power, eps, b;
  int mode;            // 0: power == 0, 1: bias == 0, 2: general
};
__global__ void pcen_kernel(const float* __restrict__ S, const float* __restrict__ ref, long long n_rows, int T,
                            PcenArgs a, const float* __restrict__ zi, float* __restrict__ zf, float* __restrict__ out) {
  __shared__ float s_s[4][32][33], s_r[4][32][33];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long row0 = ((long long)blockIdx.x * 4 + warp) * 32;
  if (row0 >= n_rows) return;
  const long long my_row = row0 + lane;
  float z = (my_row < n_rows && zi) ? zi[my_row] : 1.0f - a.b;      // lfilter_zi([b], [1, b-1]) = 1 - b
  const float log_eps = logf(a.eps), inv_eps = 1.0f / a.eps, bias_pow = powf(a.bias, a.power);
  for (int t0 = 0; t0 < T; t0 += 32) {
    const int tn = min(32, T - t0);
    for (int r = 0; r < 32; ++r) {
      const long long row = row0 + r;
      if (row < n_rows && lane < tn) {
        s_s[warp][r][lane] = S[row * T + t0 + lane];
        s_r[warp][r][lane] = ref[row * T + t0 + lane];
      }
    }
    __syncwarp();
    if (my_row < n_rows) {
      for (int i = 0; i < tn; ++i) {
        const float x = s_s[warp][lane][i];
        const float m = fmaf(a.b, s_r[warp][lane][i], z);
        z = (1.0f - a.b) * m;
        const float log_smooth = -a.gain * (log_eps + log1pf(m * inv_eps));
        float o;
        if (a.mode == 0) o = log1pf(x * expf(log_smooth));
        else if (a.mode == 1) o = expf(a.power * (logf(x) + log_smooth));
        else o = bias_pow * expm1f(a.power * log1pf(x * expf(log_smooth) / a.bias));
        s_s[warp][lane][i] = o;
      }
    }
    __syncwarp();
    for (int r = 0; r < 32; ++r) {
      const long long row = row0 + r;
      if (row < n_rows && lane < tn) out[row * T + t0 + lane] = s_s[warp][r][lane];
    }
    __syncwarp();
  }
  if (zf && my_row < n_rows) zf[my_row] = z;
}
// scipy.ndimage.maximum_filter1d along the row axis of [clip][rows][T] blocks (reflect boundary); grid.y covers
// rows m0 .. m0 + gridDim.y - 1
__global__ void maxfilter_rows_kernel(const float* __restrict__ S, int rows, int T, int size, int m0,
                                      float* __restrict__ out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  const int m = m0 + blockIdx.y;
  const float* Sc = S + (long long)blockIdx.z * rows * T;
  float v = -INFINITY;
  const int lo = m - size / 2;
  for (int j = 0; j < size; ++j) {
    int mm = lo + j;
    while (mm < 0 || mm >= rows) mm = mm < 0 ? -mm - 1 : 2 * rows - mm - 1;
    v = fmaxf(v, Sc[(long long)mm * T + t]);
  }
  out[((long long)blockIdx.z * rows + m) * T + t] = v;
}

// Spectral contrast (librosa/feature/spectral.py:355-532): for every frame and octave band, the mean of the
// `k` smallest (valley) and `k` largest (peak) magnitudes of the band's bins.  S [n_rows][F] (one row per frame,
// bins contiguous); peak / valley [clip][n_bands][n_frames].  One warp per frame: the row is copied to shared
// memory once, each band is copied into a power-of-two scratch (padded with +inf), sorted with a bitonic
// network by the warp, and the two tails are averaged.
struct ContrastArgs {
  int lo[16], count[16], k[16];   // first bin, bins in the sub-band, tail length (>= 1)
  int n_bands;
};
// Bitonic network on the first N entries of a register array of order-preserving keys (ascending), fully unrolled.
template <int N>
__device__ __forceinline__ void sort_keys(unsigned int (&v)[16]) {
#pragma unroll
  for (int k = 2; k <= N; k <<= 1) {
#pragma unroll
    for (int j = k >> 1; j > 0; j >>= 1) {
#pragma unroll
      for (int i = 0; i < N; ++i) {
        const int p = i ^ j;
        if (p > i) {
          const unsigned int x = v[i], y = v[p];
          const unsigned int lo = min(x, y), hi = max(x, y);
          const bool up = (i & k) == 0;
          v[i] = up ? lo : hi;
          v[p] = up ? hi : lo;
        }
      }
    }
  }
}

__global__ void contrast_kernel(const float* __restrict__ S, long long n_rows, int n_frames, int F, int sort_cap,
                                ContrastArgs a, float* __restrict__ peak, float* __restrict__ valley) {
  extern __shared__ __align__(16) float s_dyn[];
  const int nw = blockDim.x >> 5, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int Fp = (F + 3) & ~3;
  float* s_row = s_dyn + (size_t)warp * (Fp + sort_cap);
  float* s_sort = s_row + Fp;
  for (long long r = (long long)blockIdx.x * nw + warp; r < n_rows; r += (long long)gridDim.x * nw) {
    const float* src = S + r * F;
    for (int i = lane; i < F; i += 32) s_row[i] = __ldg(src + i);
    __syncwarp();
    const long long clip = r / n_frames, frame = r % n_frames;
    for (int b = 0; b < a.n_bands; ++b) {
      const int n = a.count[b];
      const int kk = min(a.k[b], n);
      float lo_sum = 0.0f, hi_sum = 0.0f;
      if (kk <= 16 && n <= 512) {
        // short tails of a band of at most 512 bins (the default quantile 0.02 gives k <= 9 for n_fft = 2048): lane l
        // owns the bins l, l + 32, ... of the band, sorts its (at most 16) order-preserving keys once in registers and
        // parks the sorted run in shared memory; the k smallest / largest of the band then come off the heads / tails
        // of the 32 runs — one warp reduction per extreme, and only the owning lane advances its pointer and
        // reloads.  (Round 1 rescanned the lane's elements for every extreme: 4 x as many instructions.)
        unsigned int v[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int i = lane + 32 * j;
          v[j] = i < n ? float_to_key(s_row[a.lo[b] + i]) : 0xffffffffu;   // padding sorts last
        }
        const int per = (n + 31) >> 5;                 // warp-uniform: entries per lane (the last ones may be padding)
        if (per > 8) sort_keys<16>(v);
        else if (per > 4) sort_keys<8>(v);
        else if (per > 2) sort_keys<4>(v);
        else if (per > 1) sort_keys<2>(v);
        unsigned int* s_keys = reinterpret_cast<unsigned int*>(s_sort);
#pragma unroll
        for (int j = 0; j < 16; ++j)
          if (j < per) s_keys[lane + 32 * j] = v[j];
        const int mine = lane < n ? (n - lane + 31) >> 5 : 0;   // valid entries of this lane
        __syncwarp();
        {
          int h = 0;
          unsigned int cand = mine > 0 ? v[0] : 0xffffffffu;
          float acc = 0.0f;
          for (int e = 0; e < kk; ++e) {
            const unsigned int win = __reduce_min_sync(0xffffffffu, cand);
            const unsigned int owners = __ballot_sync(0xffffffffu, cand == win && h < mine);
            if (owners == 0u) break;                              // fewer than k candidates left
            if (lane == __ffs(owners) - 1) {
              ++h;
              cand = h < mine ? s_keys[lane + 32 * h] : 0xffffffffu;
            }
            acc += key_to_float(win);
          }
          lo_sum = acc;
        }
        {
          // the largest come off the tails of the runs: `used` entries of this lane are gone, the next one sits at
          // s_top[-32 * used]  (an index form that counts up: ptxas 12.9 mis-addressed the count-down form by one entry)
          const unsigned int* s_top = s_keys + lane + 32 * (mine > 0 ? mine - 1 : 0);
          int used = 0;
          unsigned int cand = mine > 0 ? s_top[0] : 0u;
          float acc = 0.0f;
          for (int e = 0; e < kk; ++e) {
            const unsigned int win = __reduce_max_sync(0xffffffffu, cand);
            const unsigned int owners = __ballot_sync(0xffffffffu, cand == win && used < mine);
            if (owners == 0u) break;
            if (lane == __ffs(owners) - 1) {
              ++used;
              cand = used < mine ? s_top[-32 * used] : 0u;
            }
            acc += key_to_float(win);
          }
          hi_sum = acc;
        }
      } else if (kk <= 16) {
        // short tails of a longer band: extract the k extremes one at a time — lane-local scan of the lane's strided
        // elements, one warp reduction on the order-preserving keys, the owning lane knocks its element out
        for (int pass = 0; pass < 2; ++pass) {                  // 0: valley (minima), 1: peak (maxima)
          for (int i = lane; i < n; i += 32) s_sort[i] = s_row[a.lo[b] + i];
          __syncwarp();
          float acc = 0.0f;
          for (int e = 0; e < kk; ++e) {
            unsigned int best = pass == 0 ? 0xffffffffu : 0u;
            int best_i = -1;
            for (int i = lane; i < n; i += 32) {
              const unsigned int key = float_to_key(s_sort[i]);
              if (pass == 0 ? key < best : key > best) { best = key; best_i = i; }
              else if (best_i < 0 && key == best) best_i = i;
            }
            const unsigned int win = pass == 0 ? __reduce_min_sync(0xffffffffu, best) : __reduce_max_sync(0xffffffffu, best);
            const unsigned int owners = __ballot_sync(0xffffffffu, best == win && best_i >= 0);
            if (owners == 0u) break;                              // fewer than k finite candidates left
            if (lane == __ffs(owners) - 1) s_sort[best_i] = pass == 0 ? INFINITY : -INFINITY;
            acc += key_to_float(win);
            __syncwarp();
          }
          if (pass == 0) lo_sum = acc; else hi_sum = acc;
        }
      } else {
        int N = 1;
        while (N < n) N <<= 1;
        for (int i = lane; i < N; i += 32) s_sort[i] = i < n ? s_row[a.lo[b] + i] : INFINITY;
        __syncwarp();
        for (int k = 2; k <= N; k <<= 1)
          for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = lane; i < N; i += 32) {
              const int p = i ^ j;
              if (p > i) {
                const float x = s_sort[i], y = s_sort[p];
                if ((x > y) == ((i & k) == 0)) {
                  s_sort[i] = y;
                  s_sort[p] = x;
                }
              }
            }
            __syncwarp();
          }
        for (int i = lane; i < kk; i += 32) {
          lo_sum += s_sort[i];
          hi_sum += s_sort[n - 1 - i];
        }
        lo_sum = warp_sum(lo_sum);
        hi_sum = warp_sum(hi_sum);
      }
      if (lane == 0) {
        const long long o = (clip * a.n_bands + b) * n_frames + frame;
        valley[o] = lo_sum / (float)kk;       // n == 0: 0/0 = NaN, like the mean of an empty slice
        peak[o] = hi_sum / (float)kk;
      }
      __syncwarp();
    }
  }
}
__global__ void sub_kernel(const float* __restrict__ x, const float* __restrict__ y, long long n, float* __restrict__ out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = x[i] - y[i];
}

// Tuning estimation (librosa/core/pitch.py:28-109 estimate_tuning -> :182-366 piptrack -> :112-179 pitch_tuning).
// piptrack marks the bins k in [k_lo, k_hi) of a frame where the thresholded spectrum S * (S > ref) has a local
// maximum, refines them by parabolic interpolation (pitch = (k + shift) * sr / n_fft, mag = S[k] + skew) and
// estimate_tuning keeps the peaks whose mag reaches the MEDIAN mag of all peaks, then histograms the pitch
// residuals modulo one chroma bin.  The peak list is never materialised: every pass re-detects the peaks from
// the spectrogram (one warp per frame row) and accumulates one histogram —
//   mode 0/1/2: radix-select digits (11 + 11 + 10 bits) of the order-preserving key of mag -> exact median
//   mode 3:     residual histogram of the peaks with mag >= mag_threshold.
// The peaks, their pitch and mag and the residual follow piptrack_kernel / tuning_hist_kernel's rules
// (numerics.cuh), so a pass counts exactly what pitch_tuning would over the public piptrack's output.
struct PipArgs {
  int k_lo, k_hi;
  double threshold;         // relative to the frame maximum when ref_abs < 0, else unused
  double ref_abs;           // >= 0: absolute reference value (piptrack(ref=number)), compared in float64
  int thr_wide;             // threshold * max in float64 rather than float32
  double sr, n_fft;
  int mode;
  unsigned int prefix;      // digits selected so far (mode 1: top 11 bits, mode 2: top 22 bits)
  float mag_threshold;
  float bins_per_octave;
  int n_res_bins;
};
__global__ void pip_pass_kernel(const float* __restrict__ S, long long n_rows, int F, PipArgs a,
                                const double* __restrict__ edges, unsigned long long* __restrict__ hist) {
  extern __shared__ __align__(16) float s_dyn[];
  __shared__ unsigned int s_hist[2048];
  const int nw = blockDim.x >> 5, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* s_row = s_dyn + (size_t)warp * ((F + 3) & ~3);
  const int n_hist = a.mode == 3 ? a.n_res_bins : (a.mode == 2 ? 1024 : 2048);
  const float thr_t = narrow<float>(a.threshold);   // a Python float threshold is cast to float32
  for (int i = threadIdx.x; i < n_hist; i += blockDim.x) s_hist[i] = 0;
  __syncthreads();
  for (long long r = (long long)blockIdx.x * nw + warp; r < n_rows; r += (long long)gridDim.x * nw) {
    const float* src = S + r * F;
    float mx = -INFINITY;
    for (int i = lane; i < F; i += 32) {
      const float v = __ldg(src + i);
      s_row[i] = v;
      mx = MaxNan()(mx, v);
    }
    mx = warp_reduce(mx, MaxNan());                     // np.max: a NaN in the frame makes ref NaN (no peaks)
    __syncwarp();
    double ref = a.ref_abs;
    if (ref < 0.0) ref = a.thr_wide ? __dmul_rn(a.threshold, (double)mx) : (double)mul_rn(thr_t, mx);
    auto thr = [&](float v) { return (double)v > ref ? v : mul_rn(v, 0.0f); };   // S * (S > ref)
    for (int k = max(a.k_lo, 1) + lane; k < a.k_hi; k += 32) {
      const bool last = k == F - 1;
      const float c = s_row[k], l = s_row[k - 1], rr = last ? c : s_row[k + 1];
      if (!local_extremum(true, k, F, thr(l), thr(c), thr(rr))) continue;
      float shift = 0.0f, avg;
      if (last) {
        avg = sub_rn(c, l);                              // np.gradient, one-sided at the edge
      } else {
        avg = mul_rn(sub_rn(rr, l), 0.5f);
        shift = parabolic_shift(l, c, rr);
      }
      const float pitch = narrow<float>(__ddiv_rn(__dmul_rn(__dadd_rn((double)k, (double)shift), a.sr), a.n_fft));
      if (!(pitch > 0.0f)) continue;
      const float mag = parabolic_mag(c, avg, shift);
      const unsigned int key = float_to_key(mag);
      if (a.mode == 0) {
        atomicAdd(&s_hist[key >> 21], 1u);
      } else if (a.mode == 1) {
        if ((key >> 21) == a.prefix) atomicAdd(&s_hist[(key >> 10) & 0x7ffu], 1u);
      } else if (a.mode == 2) {
        if ((key >> 10) == a.prefix) atomicAdd(&s_hist[key & 0x3ffu], 1u);
      } else if (mag >= a.mag_threshold) {
        const float res = tuning_residual(pitch, a.bins_per_octave);
        if (res == res) atomicAdd(&s_hist[residual_bin(res, a.n_res_bins, edges)], 1u);
      }
    }
    __syncwarp();
  }
  __syncthreads();
  for (int i = threadIdx.x; i < n_hist; i += blockDim.x)
    if (s_hist[i]) atomicAdd(&hist[i], (unsigned long long)s_hist[i]);
}

// util.normalize(S, norm, axis=-2) of [clip][rows][T] blocks with the default threshold / fill
// (librosa/util/utils.py:797-1026): mag = |S| in float64, the column length summed over rows in order as NumPy sums
// a non-last axis, columns whose length is below tiny(float32) left unscaled, and S / length formed in float64 and
// rounded once to float32.  NumPy's mag**p and length**(1/p) take exact shortcuts for p = 1, 2 and 1/2 (copy,
// square, square root); other p go through pow.
// norm_kind: 0 = inf (max |x|), 1 = -inf (min |x|), 2 = count of non-zeros, 3 = p-norm with p = norm_p.
__global__ void normalize_rows_kernel(const float* __restrict__ x, int rows, int T, int norm_kind, double norm_p,
                                      float* __restrict__ out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  const float* xc = x + (long long)blockIdx.y * rows * T + t;
  float* oc = out + (long long)blockIdx.y * rows * T + t;
  double len = norm_kind == 1 ? INFINITY : 0.0;
  for (int r = 0; r < rows; ++r) {
    const double v = fabs((double)xc[(long long)r * T]);
    if (norm_kind == 0) len = MaxNan()(len, v);
    else if (norm_kind == 1) len = MinNan()(len, v);
    else if (norm_kind == 2) len += v > 0.0 ? 1.0 : 0.0;
    else len = add_rn(len, norm_p == 1.0 ? v : norm_p == 2.0 ? mul_rn(v, v) : norm_p == 0.5 ? sqrt_rn(v) : pow(v, norm_p));
  }
  if (norm_kind == 3 && norm_p != 1.0)
    len = norm_p == 2.0 ? sqrt_rn(len) : norm_p == 0.5 ? mul_rn(len, len) : pow(len, div_rn(1.0, norm_p));
  if (len < (double)tiny_of<float>()) len = 1.0;
  for (int r = 0; r < rows; ++r) oc[(long long)r * T] = narrow<float>(div_rn((double)xc[(long long)r * T], len));
}

// Median-filtering harmonic / percussive separation (librosa/decompose.py:241-389, hpss) on a magnitude
// spectrogram M [clip][T][F] (bins contiguous):
//   harm = median over `win_h` frames (scipy.ndimage.median_filter, reflect boundary, rank size // 2),
//   perc = median over `win_p` bins,
//   mask_h = softmask(harm, perc * margin_h), mask_p = softmask(perc, harm * margin_p)   (util/utils.py: softmask)
// One thread per element: the window goes into a register array padded with +inf to NS = 8 / 16 / 32 / 64
// entries and through a compile-time bitonic network (fminf / fmaxf pairs, no branches).  Neighbouring threads
// share all but one of their inputs, so the loads are served by L1.
template <int NS>
__device__ __forceinline__ float median_of(float (&v)[NS], int rank) {
#pragma unroll
  for (int k = 2; k <= NS; k <<= 1) {
#pragma unroll
    for (int j = k >> 1; j > 0; j >>= 1) {
#pragma unroll
      for (int i = 0; i < NS; ++i) {
        const int p = i ^ j;
        if (p > i) {
          const float x = v[i], y = v[p];
          const float lo = fminf(x, y), hi = fmaxf(x, y);
          const bool asc = (i & k) == 0;
          v[i] = asc ? lo : hi;
          v[p] = asc ? hi : lo;
        }
      }
    }
  }
  float m = v[0];
#pragma unroll
  for (int i = 1; i < NS; ++i)
    if (i == rank) m = v[i];
  return m;
}
__device__ __forceinline__ int reflect_index(int i, int n) {
  while (i < 0 || i >= n) i = i < 0 ? -i - 1 : 2 * n - i - 1;
  return i;
}
// util.softmask: an infinite power is the hard mask X > X_ref everywhere, also where both lie below tiny(float32)
// (the reference splits or zeroes those cells only for a finite power)
__device__ __forceinline__ float soft_mask(float x, float x_ref, float power, int split_zeros) {
  if (isinf(power)) return x > x_ref ? 1.0f : 0.0f;
  float z = fmaxf(x, x_ref);
  const bool bad = z < 1.17549435e-38f;
  if (bad) return split_zeros ? 0.5f : 0.0f;
  const float a = x / z, b = x_ref / z;
  const float pa = power == 2.0f ? a * a : (power == 1.0f ? a : powf(a, power));
  const float pb = power == 2.0f ? b * b : (power == 1.0f ? b : powf(b, power));
  return pa / (pa + pb);
}
struct HpssArgs {
  int T, F, win_h, win_p;
  int t0;                    // frame of grid.y == 0 (launches of at most 65 535 frames)
  float margin_h, margin_p, power;
  int split_zeros, mode;     // mode 0: masked components, 1: the masks
};
template <int NS>
__global__ void hpss_kernel(const float* __restrict__ M, const float2* __restrict__ Sc, HpssArgs a,
                            float* __restrict__ out_h, float* __restrict__ out_p) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  const int t = a.t0 + blockIdx.y;
  if (f >= a.F) return;
  const long long base = (long long)blockIdx.z * a.T * a.F;
  const float* Mc = M + base;
  float v[NS];
  const int t0 = t - a.win_h / 2;
#pragma unroll
  for (int j = 0; j < NS; ++j) v[j] = j < a.win_h ? __ldg(Mc + (long long)reflect_index(t0 + j, a.T) * a.F + f) : INFINITY;
  const float harm = median_of<NS>(v, a.win_h / 2);
  const int f0 = f - a.win_p / 2;
  const float* row = Mc + (long long)t * a.F;
#pragma unroll
  for (int j = 0; j < NS; ++j) v[j] = j < a.win_p ? __ldg(row + reflect_index(f0 + j, a.F)) : INFINITY;
  const float perc = median_of<NS>(v, a.win_p / 2);
  const float mh = soft_mask(harm, perc * a.margin_h, a.power, a.split_zeros);
  const float mp = soft_mask(perc, harm * a.margin_p, a.power, a.split_zeros);
  const long long o = base + (long long)t * a.F + f;
  if (a.mode == 1) {
    out_h[o] = mh;
    out_p[o] = mp;
  } else if (Sc) {
    const float2 s = Sc[o];
    reinterpret_cast<float2*>(out_h)[o] = make_float2(s.x * mh, s.y * mh);
    reinterpret_cast<float2*>(out_p)[o] = make_float2(s.x * mp, s.y * mp);
  } else {
    const float m = Mc[(long long)t * a.F + f];
    out_h[o] = m * mh;
    out_p[o] = m * mp;
  }
}
__global__ void cabs_kernel(const float2* __restrict__ x, long long n, float* __restrict__ out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float2 v = x[i];
    out[i] = hypotf(v.x, v.y);
  }
}

// Time-frequency reassignment (librosa/core/spectrum.py:646-1293, reassigned_spectrogram): elementwise over three
// STFTs of the same signal taken with the window h, its cyclic derivative dh and the time-weighted window th
// (all [clip][T][F], bins contiguous):
//   freq = f_k - Im(S_dh / S_h) * sr / (2 pi)         (eq. 5.20, :847-853)
//   time = t_frame + Re(S_th / S_h) / sr              (eq. 5.23, :1001-1016)
//   mag  = |S_h|; cells with mag < sqrt(ref_power) become NaN, optionally refilled with the bin frequency /
//   frame time, optionally clipped to [0, sr/2] / [0, duration]                         (:1240-1290)
struct ReassignArgs {
  int T, F;
  float freq_scale;      // sr / (2 pi)
  float inv_sr, mag_threshold, max_freq, max_time;
  int do_freq, do_time, apply_threshold, fill_nan, clip;
};
__global__ void reassign_kernel(const float2* __restrict__ Sh, const float2* __restrict__ Sdh,
                                const float2* __restrict__ Sth, const float* __restrict__ bin_freqs,
                                const float* __restrict__ frame_times, ReassignArgs a, long long n,
                                float* __restrict__ freqs, float* __restrict__ times, float* __restrict__ mags) {
  const float nan = __int_as_float(0x7fc00000);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int f = (int)(i % a.F);
    const int t = (int)((i / a.F) % a.T);
    const float2 h = Sh[i];
    const float den = fmaf(h.x, h.x, h.y * h.y);
    const float mag = hypotf(h.x, h.y);
    const bool low = a.apply_threshold && mag < a.mag_threshold;
    mags[i] = mag;
    const float bf = bin_freqs[f], ft = frame_times[t];
    float fr = bf, tm = ft;
    if (a.do_freq) {
      const float2 d = Sdh[i];
      fr = den > 0.0f ? bf - (d.y * h.x - d.x * h.y) / den * a.freq_scale : nan;
      if (low) fr = nan;
      if (a.fill_nan && isnan(fr)) fr = bf;
      if (a.clip && !isnan(fr)) fr = fminf(fmaxf(fr, 0.0f), a.max_freq);
    }
    if (a.do_time) {
      const float2 d = Sth[i];
      tm = den > 0.0f ? ft + (d.x * h.x + d.y * h.y) / den * a.inv_sr : nan;
      if (low) tm = nan;
      if (a.fill_nan && isnan(tm)) tm = ft;
      if (a.clip && !isnan(tm)) tm = fminf(fmaxf(tm, 0.0f), a.max_time);
    }
    freqs[i] = fr;
    times[i] = tm;
  }
}

// Phase vocoder (librosa/core/spectrum.py:1364-1530): output frame t takes its magnitude by linear interpolation
// of |D| at time t_out[t] and its phase as  angle(D[i0[0]]) + sum_{s<t} (angle(D[i1[s]]) - angle(D[i0[s]]))  —
// a float32 running sum along time (np.cumsum), so one thread walks the output frames of one (clip, bin).
// D [clip][T][F] complex64 (bins contiguous: neighbouring threads read neighbouring bins of the same frame).
__global__ void phase_vocoder_kernel(const float2* __restrict__ D, int T, int F, long long n_clips, int n_out,
                                     const int* __restrict__ i0, const int* __restrict__ i1,
                                     const int* __restrict__ lo, const double* __restrict__ dx,
                                     float2* __restrict__ out) {
  const long long id = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= n_clips * F) return;
  const long long clip = id / F;
  const int f = (int)(id % F);
  const float2* Dc = D + clip * (long long)T * F + f;
  float2* oc = out + clip * (long long)n_out * F + f;
  float phase = 0.0f;
  for (int t = 0; t < n_out; ++t) {
    const float2 a = Dc[(long long)i0[t] * F];
    if (t == 0) {
      phase = atan2f(a.y, a.x);
    }
    const float2 m0 = Dc[(long long)lo[t] * F], m1 = Dc[(long long)(lo[t] + 1) * F];
    const double y0 = (double)hypotf(m0.x, m0.y), y1 = (double)hypotf(m1.x, m1.y);
    const double mag = (y1 - y0) * dx[t] + y0;
    float sn, cs;
    sincosf(phase, &sn, &cs);
    oc[(long long)t * F] = make_float2((float)((double)cs * mag), (float)((double)sn * mag));
    const float2 b = Dc[(long long)i1[t] * F];
    phase += atan2f(b.y, b.x) - atan2f(a.y, a.x);
  }
}

// Elementwise helpers of the dB conversions (librosa/core/spectrum.py):
//   UNARY_SQUARE           x*x                        amplitude_to_db squares |S| before power_to_db (:2032-2037)
//   UNARY_DB_TO_POWER      ref * 10^(0.1 x)           db_to_power (:1899-1925)
//   UNARY_DB_TO_AMPLITUDE  sqrt(ref^2 * 10^(0.1 x))   db_to_amplitude (:2054-2081), param = ref^2
enum UnaryOp : int { UNARY_SQUARE = 0, UNARY_DB_TO_POWER = 1, UNARY_DB_TO_AMPLITUDE = 2 };
__global__ void unary_kernel(const float* __restrict__ in, long long n, int op, float param, float* __restrict__ out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float x = in[i];
    float r;
    if (op == UNARY_SQUARE) r = x * x;
    else {
      r = param * powf(10.0f, x * 0.1f);
      if (op == UNARY_DB_TO_AMPLITUDE) r = sqrtf(r);
    }
    out[i] = r;
  }
}

// ------------------------------------------------------------------ polyphase resampling
// librosa.resample(res_type="polyphase") = scipy.signal.resample_poly(y, up, down) (librosa/core/audio.py:1129-1145):
// upfirdn(h, x, up, down) cropped to [n_pre_remove, n_pre_remove + n_out) with the zero-padded low-pass h the host
// designs exactly as SciPy does (firwin(2 * 10 * max(up, down) + 1, 1 / max(up, down), window=("kaiser", 5.0)) * up,
// float32 for float32 data).  Output sample j is
//     y[j] = sum_m x[m] * h[(n_pre_remove + j) * down - m * up],
// accumulated over increasing m like SciPy's upfirdn loop; one thread per output sample (about 20 * max(1, down / up)
// taps each).  Samples j >= n_keep of a row are the zeros of util.fix_length; out_scale carries 1 / sqrt(ratio).
__global__ void resample_poly_kernel(const float* __restrict__ x, long long x_stride, int n_in, const float* __restrict__ h,
                                     int n_h, int up, int down, long long n_pre_remove, int n_keep, int n_total,
                                     long long n_clips, float out_scale, float* __restrict__ out) {
  const long long total = n_clips * n_total;
  for (long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x; o < total; o += (long long)gridDim.x * blockDim.x) {
    const long long clip = o / n_total;
    const int j = (int)(o - clip * n_total);
    float acc = 0.0f;
    if (j < n_keep) {
      const long long t = (n_pre_remove + j) * (long long)down;          // position in the up-sampled stream
      long long m_hi = t / up;
      if (m_hi > n_in - 1) m_hi = n_in - 1;
      long long m_lo = t - (n_h - 1);                                    // smallest m with t - m * up <= n_h - 1
      m_lo = m_lo <= 0 ? 0 : (m_lo + up - 1) / up;
      const float* xc = x + clip * x_stride;
      long long k = t - m_lo * up;
      for (long long m = m_lo; m <= m_hi; ++m, k -= up) acc = fmaf(__ldg(h + k), __ldg(xc + m), acc);
      acc *= out_scale;
    }
    out[o] = acc;
  }
}

// ------------------------------------------------------------------ power_to_db
// 10 log10(np.maximum(amin, S)) - db_sub, then np.maximum(log_spec, log_spec.max(per clip) - top_db)
// (librosa/core/spectrum.py:1866-1881).  np.maximum keeps a NaN cell, and a NaN clip maximum makes the whole clip NaN
// under top_db: a NaN maximum is stored as the all-ones key, which no finite key exceeds and key_to_float reads as NaN.
__global__ void db_kernel(const float* __restrict__ in, long long per_clip, float amin, float db_sub,
                          unsigned int* __restrict__ clip_max, float* __restrict__ out) {
  const int clip = blockIdx.y;
  const float* ic = in + (long long)clip * per_clip;
  float* oc = out + (long long)clip * per_clip;
  float mx = -INFINITY;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < per_clip;
       i += (long long)gridDim.x * blockDim.x) {
    const float v = 10.0f * log10f(MaxNan()(amin, ic[i])) - db_sub;
    oc[i] = v;
    mx = MaxNan()(mx, v);
  }
  mx = warp_reduce(mx, MaxNan());
  if ((threadIdx.x & 31) == 0 && !(mx == -INFINITY)) atomicMax(clip_max + clip, mx != mx ? 0xffffffffu : float_to_key(mx));
}

__global__ void db_clamp_kernel(float* __restrict__ x, long long per_clip, const unsigned int* __restrict__ clip_max,
                                float top_db) {
  const int clip = blockIdx.y;
  float* xc = x + (long long)clip * per_clip;
  const float floor_v = key_to_float(clip_max[clip]) - top_db;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < per_clip;
       i += (long long)gridDim.x * blockDim.x)
    xc[i] = MaxNan()(xc[i], floor_v);
}

// ------------------------------------------------------------------ Griffin-Lim phase update
// angles <- rebuilt - scale * tprev ;  angles <- angles / (|angles| + eps) * S      (elementwise)
// librosa/core/spectrum.py:2898-2903 (scale = momentum / (1 + momentum), eps = tiny(complex64)).
__global__ void gl_update_kernel(const float2* __restrict__ rebuilt, const float2* __restrict__ tprev,
                                 const float* __restrict__ S, float scale, float eps, float2* __restrict__ out,
                                 long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float2 a = rebuilt[i];
    if (tprev != nullptr) {
      const float2 p = tprev[i];
      a.x = fmaf(-scale, p.x, a.x);
      a.y = fmaf(-scale, p.y, a.y);
    }
    const float mag = hypotf(a.x, a.y) + eps;
    const float s = S[i];
    out[i] = make_float2(a.x / mag * s, a.y / mag * s);
  }
}

// ------------------------------------------------------------------ batched transpose
template <typename T>
__global__ void transpose_kernel(const T* __restrict__ in, int rows, int cols, T* __restrict__ out) {
  __shared__ T tile[32][33];
  const long long base = (long long)blockIdx.z * rows * cols;
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    int r = r0 + j, c = c0 + threadIdx.x;
    if (r < rows && c < cols) tile[j][threadIdx.x] = in[base + (long long)r * cols + c];
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    int c = c0 + j, r = r0 + threadIdx.x;
    if (r < rows && c < cols) out[base + (long long)c * rows + r] = tile[threadIdx.x][j];
  }
}

}  // namespace b2l
