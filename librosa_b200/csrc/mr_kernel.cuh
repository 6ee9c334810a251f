// mr_kernel.cuh — mixed-radix real FFT frames for even n_fft whose half is 5-smooth (2^a 3^b 5^c): the 400 / 320 /
// 480 / 800 / 960 / 1200-sample frames of speech front ends (25 ms at 16 kHz = 400 samples, ...).
//
// librosa.stft hands such frames to scipy.fft.rfft, whose ducc plans are mixed-radix Cooley-Tukey as well
// (librosa/core/spectrum.py:388); round 1 ran them through Bluestein's chirp-z transform on a power-of-two engine
// (czt_kernel.cuh: two 1024-point complex transforms per pair of 400-sample frames — five times the work of the
// n_fft = 512 kernel).  Here ONE WARP owns a frame:
//     z[e] = (x[2e] w[2e], x[2e+1] w[2e+1]),  e < M = n_fft / 2      packed real input, window folded in
//     Stockham passes of radix 5 / 3 / 8 / 4 / 2 between two shared-memory buffers of the warp (autosort, natural
//     order in and out; butterflies dealt to the lanes; pass twiddles from a shared table built in double precision)
//     X[k], X[M-k] from Z[k], Z[M-k]                                  real-FFT un-mix (r2c_pair)
// and the epilogues of the chirp-z kernel it replaces (complex STFT rows, |X|^power rows) plus a fused band-sparse
// mel projection (librosa/feature/spectral.py:2160) with the optional dB conversion and per-clip maximum that mfcc
// needs (librosa/core/spectrum.py:1866-1881).  Frames are read straight from global memory through the np.pad index
// map — consecutive warps take consecutive frames, so the n_fft / hop overlap is served by L1 / L2 and HBM sees
// every sample once.  Odd radices run first: with sub-length p = 1 a lane writes R consecutive values, and an odd
// R keeps the 64-bit stores of a half warp in distinct banks.
#pragma once
#include "common.cuh"
#include "fft_engine.cuh"
#include "fwd_kernel.cuh"   // load_padded, power_from_sq, sqmag, db10, sqrt_approx

namespace b2l {

struct MrArgs {
  const float* y;
  long long clip_stride;
  int n, n_clips;
  int L, M, hop, pad, pad_mode, n_frames, n_bins;   // L = n_fft, M = L / 2, n_bins = M + 1
  int n_pass;
  int radix[kMrMaxPass];
  int tw_off[kMrMaxPass];   // pass s (sub-length p_s > 1): tw[tw_off[s] + (r-1) p_s + k] = exp(-2 pi i r k / (p_s R_s))
  int tw_count;
  const float* win;         // [L] window * 1/2
  const float2* tw;
  const float2* twn;        // [M/2 + 1] exp(-2 pi i k / L)
  float2* out_c;            // mode 0: complex64 [clip][frame][bin]
  float* out_r;             // mode 1: |X|^power [clip][frame][bin];  mode 2: mel [clip][mel][frame]
  int mode, power_mode;
  float power;
  int* status;
  // mode 2
  const MelBand* band;
  const float* mel_w;
  int n_mels, mel_w_count;
  int log_mode;
  float amin, db_sub;
  unsigned int* clip_max;
};

// ---- radix-R DFTs in registers, natural order in and out (forward sign)
__device__ __forceinline__ void mr_dft3(float2 (&u)[3]) {
  constexpr float hs3 = 0.86602540378443864676f;   // sin(2 pi / 3)
  const float2 t1 = add2(u[1], u[2]);
  const float2 m1 = fma2(bc2(-0.5f), t1, u[0]);
  const float2 d = sub2(u[1], u[2]);
  const float2 m2 = mul2(mulni2(d), bc2(hs3));      // -i sin(2 pi/3) (u1 - u2)
  u[0] = add2(u[0], t1);
  u[1] = add2(m1, m2);
  u[2] = sub2(m1, m2);
}
__device__ __forceinline__ void mr_dft5(float2 (&u)[5]) {
  constexpr float c1 = 0.30901699437494742410f, c2 = -0.80901699437494742410f;   // cos(2 pi/5), cos(4 pi/5)
  constexpr float s1 = 0.95105651629515357212f, s2 = 0.58778525229247312917f;    // sin(2 pi/5), sin(4 pi/5)
  const float2 t1 = add2(u[1], u[4]), t2 = add2(u[2], u[3]);
  const float2 t3 = sub2(u[1], u[4]), t4 = sub2(u[2], u[3]);
  const float2 a1 = fma2(bc2(c2), t2, fma2(bc2(c1), t1, u[0]));
  const float2 a2 = fma2(bc2(c1), t2, fma2(bc2(c2), t1, u[0]));
  const float2 b1 = fma2(bc2(s2), t4, mul2(bc2(s1), t3));
  const float2 b2 = fma2(bc2(-s1), t4, mul2(bc2(s2), t3));
  u[0] = add2(u[0], add2(t1, t2));
  u[1] = add2(a1, mulni2(b1));   // a1 - i b1
  u[4] = add2(a1, muli2(b1));
  u[2] = add2(a2, mulni2(b2));
  u[3] = add2(a2, muli2(b2));
}

// One Stockham pass of radix R over M points: butterflies i = lane, lane + 32, ... < T = M / R.  FIRST: sub-length
// p == 1 (no twiddles, R consecutive outputs per butterfly).  Operand, twiddle and result addresses advance by
// constant strides (one add per access instead of a multiply-add and a scale).
template <int R, bool FIRST, int G>
__device__ __forceinline__ void mr_pass(const float2* __restrict__ src, float2* __restrict__ dst,
                                        const float2* __restrict__ tw, int p, int T, int lane) {
  constexpr bool POW2 = (R & (R - 1)) == 0;
  constexpr int LOGR = ilog2c(R);
  int k = FIRST ? 0 : lane % p;
  const int kstep = FIRST ? 0 : G % p;
  for (int i = lane; i < T; i += G) {
    float2 u[R];
    const float2* sp = src + i;
    const float2* tp = tw + k;
#pragma unroll
    for (int r = 0; r < R; ++r) {
      float2 x = *sp;
      sp += T;
      if (!FIRST && r > 0) {
        x = cmul(x, *tp);
        tp += p;
      }
      u[POW2 ? bitrevc(r, LOGR) : r] = x;
    }
    if constexpr (R == 3) mr_dft3(u);
    else if constexpr (R == 5) mr_dft5(u);
    else dft_reg<R, 0>(u);
    if constexpr (FIRST) {
      float2* dp = dst + i * R;
#pragma unroll
      for (int q = 0; q < R; ++q) dp[q] = u[q];
    } else {
      float2* dp = dst + (i - k) * R + k;
#pragma unroll
      for (int q = 0; q < R; ++q) {
        *dp = u[q];
        dp += p;
      }
      k += kstep;
      if (k >= p) k -= p;
    }
  }
}
template <bool FIRST, int G>
__device__ __forceinline__ void mr_pass_any(int R, const float2* src, float2* dst, const float2* tw, int p, int T, int lane) {
  switch (R) {
    case 5: mr_pass<5, FIRST, G>(src, dst, tw, p, T, lane); break;
    case 3: mr_pass<3, FIRST, G>(src, dst, tw, p, T, lane); break;
    case 8: mr_pass<8, FIRST, G>(src, dst, tw, p, T, lane); break;
    case 4: mr_pass<4, FIRST, G>(src, dst, tw, p, T, lane); break;
    default: mr_pass<2, FIRST, G>(src, dst, tw, p, T, lane); break;
  }
}

// Dynamic shared memory: window [L] | pass twiddles [tw_count] | un-mix twiddles [M/2+1] | mel bands | mel weights |
// per warp: two exchange buffers of M complex values.
__host__ __device__ inline size_t mr_table_bytes(int L, int tw_count, int n_mels, int mel_w_count) {
  size_t b = (size_t)((L + 3) & ~3) * 4 + (size_t)((tw_count + 1) & ~1) * 8 + (size_t)((L / 4 + 2) & ~1) * 8;
  b += (size_t)n_mels * sizeof(MelBand) + (size_t)((mel_w_count + 3) & ~3) * 4;
  return (b + 15) & ~(size_t)15;
}

// MODE 0: complex STFT rows, 1: |X|^power rows, 2: band-sparse mel projection (optionally in dB with the per-clip maximum)
// G: lanes per frame.  32 = a warp owns a frame; 16 = a warp carries two frames side by side (short frames: 40 radix-5
// butterflies fill 3 rounds of 16 lanes to 83 % where 2 rounds of 32 lanes reach 62 %).  The lane groups of a warp run
// in lockstep (__syncwarp); a group past the end of the batch repeats the last frame (identical stores).
template <int MODE, int G>
__global__ void __launch_bounds__(512, 2) mr_kernel(const MrArgs a) {
  extern __shared__ __align__(128) unsigned char smem[];
  constexpr int NG = 32 / G;                      // frames per warp
  const int tid = threadIdx.x, lane = tid & (G - 1), grp = tid / G, ngroups = blockDim.x / G;
  const int L = a.L, M = a.M;
  float* s_win = reinterpret_cast<float*>(smem);
  float2* s_tw = reinterpret_cast<float2*>(s_win + ((L + 3) & ~3));
  float2* s_twn = s_tw + ((a.tw_count + 1) & ~1);
  MelBand* s_band = reinterpret_cast<MelBand*>(s_twn + ((L / 4 + 2) & ~1));
  float* s_melw = reinterpret_cast<float*>(s_band + a.n_mels);
  float2* s_x = reinterpret_cast<float2*>(smem + mr_table_bytes(L, a.tw_count, a.n_mels, a.mel_w_count));
  for (int i = tid; i < L; i += blockDim.x) s_win[i] = a.win[i];
  for (int i = tid; i < a.tw_count; i += blockDim.x) s_tw[i] = a.tw[i];
  for (int i = tid; i <= M / 2; i += blockDim.x) s_twn[i] = a.twn[i];
  if constexpr (MODE == 2) {
    for (int i = tid; i < a.n_mels; i += blockDim.x) s_band[i] = a.band[i];
    for (int i = tid; i < a.mel_w_count; i += blockDim.x) s_melw[i] = a.mel_w[i];
  }
  __syncthreads();
  float2* buf0 = s_x + (size_t)grp * 2 * M;
  float2* buf1 = buf0 + M;

  const long long total = (long long)a.n_clips * a.n_frames;
  const long long stride = (long long)gridDim.x * ngroups;
  const bool vec_ok = ((a.clip_stride & 1) == 0) && ((reinterpret_cast<uintptr_t>(a.y) & 7) == 0);
  float wmax = -INFINITY;
  int wmax_clip = -1;
  // the lanes of this group (the groups of a warp may sit in different clips, so they reduce separately)
  const unsigned gmask = G == 32 ? 0xffffffffu : (((1u << (G & 31)) - 1u) << ((threadIdx.x & 31) & ~(G - 1)));
  auto flush_max = [&]() {   // per-clip maximum of the dB values this lane group produced (log_mode)
    if (wmax_clip >= 0) {
#pragma unroll
      for (int o = G / 2; o > 0; o >>= 1) wmax = fmaxf(wmax, __shfl_xor_sync(gmask, wmax, o));
      if (lane == 0 && wmax > -INFINITY) atomicMax(a.clip_max + wmax_clip, float_to_key(wmax));
    }
    wmax = -INFINITY;
  };
  // (clip, frame) of this group's frames without a division per frame: advanced by the constant group stride.  The
  // loop runs while the FIRST group of the warp has work, so that the warp stays convergent.
  const long long fw = (long long)blockIdx.x * ngroups + (grp & ~(NG - 1));     // first group of this warp
  const long long f0 = fw + (grp & (NG - 1));
  int clip, frame;
  {
    const long long fc = f0 < total ? f0 : total - 1;
    clip = (int)(fc / a.n_frames);
    frame = (int)(fc - (long long)clip * a.n_frames);
  }
  const int step_c = (int)(stride / a.n_frames), step_f = (int)(stride - (long long)step_c * a.n_frames);
  for (long long f = fw; f < total; f += stride) {
    const float* yc = a.y + (long long)clip * a.clip_stride;
    const long long s0 = (long long)frame * a.hop - a.pad;
    // ---- packed, windowed input
    if (s0 >= 0 && s0 + L <= a.n && vec_ok && (s0 & 1) == 0) {
      const float2* y2 = reinterpret_cast<const float2*>(yc + s0);
      const float2* w2 = reinterpret_cast<const float2*>(s_win);
      for (int e = lane; e < M; e += G) buf0[e] = mul2(__ldg(y2 + e), w2[e]);
    } else {
      for (int e = lane; e < M; e += G) {
        const float x0 = load_padded(yc, a.n, s0 + 2 * e, a.pad_mode, a.pad);
        const float x1 = load_padded(yc, a.n, s0 + 2 * e + 1, a.pad_mode, a.pad);
        buf0[e] = make_float2(x0 * s_win[2 * e], x1 * s_win[2 * e + 1]);
      }
    }
    __syncwarp();
    // ---- Stockham passes
    float2* src = buf0;
    float2* dst = buf1;
    mr_pass_any<true, G>(a.radix[0], src, dst, s_tw, 1, M / a.radix[0], lane);
    __syncwarp();
    int p = a.radix[0];
    for (int s = 1; s < a.n_pass; ++s) {
      float2* tmp = src;
      src = dst;
      dst = tmp;
      const int R = a.radix[s];
      mr_pass_any<false, G>(R, src, dst, s_tw + a.tw_off[s], p, M / R, lane);
      __syncwarp();
      p *= R;
    }
    {
      float2* tmp = src;
      src = dst;
      dst = tmp;
    }
    // ---- real-FFT un-mix and epilogue: src holds Z[0 .. M), dst is free
    const long long orow = ((long long)clip * a.n_frames + frame) * a.n_bins;
    float* prow = reinterpret_cast<float*>(dst);
    bool bad = false;
    auto unmix = [&](auto power_of) {
      for (int k = lane; k <= M / 2; k += G) {
        const float2 A = src[k], B = src[k == 0 ? 0 : M - k];
        bad = bad || !(fabsf(A.x) + fabsf(A.y) <= 3.0e38f);
        float2 xa, xb;
        r2c_pair(A, B, s_twn[k], xa, xb);
        const bool two = (M - k) != k;
        if constexpr (MODE == 0) {
          a.out_c[orow + k] = xa;
          if (two) a.out_c[orow + M - k] = xb;
        } else {
          const float pa = power_of(sqmag(xa)), pb = power_of(sqmag(xb));
          if constexpr (MODE == 1) {
            a.out_r[orow + k] = pa;
            if (two) a.out_r[orow + M - k] = pb;
          } else {
            prow[k] = pa;
            prow[M - k] = pb;   // k == M - k writes the same value twice: xa == xb there up to the sign of zero
          }
        }
      }
    };
    if (MODE == 0 || a.power_mode == 2) unmix([](float p2) { return p2; });
    else if (a.power_mode == 1) unmix([](float p2) { return sqrt_approx(p2); });
    else unmix([&](float p2) { return power_from_sq(p2, a.power_mode, a.power); });
    if (bad) *a.status = 1;   // util.valid_audio (librosa/util/utils.py:303-306): a non-finite sample poisons every bin
    if constexpr (MODE == 2) {
      __syncwarp();
      if (a.log_mode && clip != wmax_clip) {
        flush_max();
        wmax_clip = clip;
      }
      float* o = a.out_r + (long long)clip * a.n_mels * a.n_frames + frame;
      for (int m = lane; m < a.n_mels; m += G) {
        const MelBand b = s_band[m];
        const float* w = s_melw + b.off;
        const float* x = prow + b.lo;
        float acc0 = 0.0f, acc1 = 0.0f;
        int i = 0;
        for (; i + 1 < b.len; i += 2) {
          acc0 = fmaf(w[i], x[i], acc0);
          acc1 = fmaf(w[i + 1], x[i + 1], acc1);
        }
        if (i < b.len) acc0 = fmaf(w[i], x[i], acc0);
        float v = acc0 + acc1;
        if (a.log_mode) {
          v = db10(fmaxf(a.amin, v)) - a.db_sub;
          wmax = fmaxf(wmax, v);
        }
        o[(long long)m * a.n_frames] = v;
      }
    }
    __syncwarp();   // the rows are consumed before the next frame overwrites the buffers
    // advance; a group that runs past the end keeps its last frame
    if (f + (grp & (NG - 1)) + stride < total) {
      clip += step_c;
      frame += step_f;
      if (frame >= a.n_frames) {
        frame -= a.n_frames;
        ++clip;
      }
    }
  }
  if (MODE == 2 && a.log_mode) flush_max();
}

// ------------------------------------------------------------------ inverse: irfft of length L per frame
// scipy.fft.irfft(D, n=L) semantics (Im of the DC and Nyquist bins ignored, 1/L scale; librosa/core/spectrum.py:598):
// the packed spectrum Z[k] is rebuilt from X[k], X[M-k] (c2r_pair), the inverse transform is the forward engine on
// re/im-swapped data, and the windowed samples (window / L folded into `win`) go to the scratch array
// [clip][frame][L] that ola_kernel overlap-adds and normalises — the same contract as czt_inv_kernel, which this
// replaces for the mixed-radix sizes.
struct MrInvArgs {
  const float2* D;          // [clip][frames_stored][n_bins]
  long long d_clip_stride;
  int n_clips, n_frames, L, M, n_bins;
  int n_pass;
  int radix[kMrMaxPass];
  int tw_off[kMrMaxPass];
  int tw_count;
  const float* win;         // [L] window / L
  const float2* tw;
  const float2* twn;
  float* ytmp;              // [clip][n_frames][L]
};

__global__ void __launch_bounds__(512, 2) mr_inv_kernel(const MrInvArgs a) {
  extern __shared__ __align__(128) unsigned char smem[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
  const int L = a.L, M = a.M;
  float* s_win = reinterpret_cast<float*>(smem);
  float2* s_tw = reinterpret_cast<float2*>(s_win + ((L + 3) & ~3));
  float2* s_twn = s_tw + ((a.tw_count + 1) & ~1);
  float2* s_x = reinterpret_cast<float2*>(smem + mr_table_bytes(L, a.tw_count, 0, 0));
  for (int i = tid; i < L; i += blockDim.x) s_win[i] = a.win[i];
  for (int i = tid; i < a.tw_count; i += blockDim.x) s_tw[i] = a.tw[i];
  for (int i = tid; i <= M / 2; i += blockDim.x) s_twn[i] = a.twn[i];
  __syncthreads();
  float2* buf0 = s_x + (size_t)warp * 2 * M;
  float2* buf1 = buf0 + M;
  const long long total = (long long)a.n_clips * a.n_frames;
  const long long stride = (long long)gridDim.x * nwarps;
  const long long f0 = (long long)blockIdx.x * nwarps + warp;
  int clip = (int)(f0 / a.n_frames), frame = (int)(f0 - (long long)clip * a.n_frames);
  const int step_c = (int)(stride / a.n_frames), step_f = (int)(stride - (long long)step_c * a.n_frames);
  for (long long f = f0; f < total; f += stride, clip += step_c, frame += step_f) {
    if (frame >= a.n_frames) {
      frame -= a.n_frames;
      ++clip;
    }
    const float2* row = a.D + (long long)clip * a.d_clip_stride + (long long)frame * a.n_bins;
    for (int k = lane; k <= M / 2; k += 32) {
      float2 xa = __ldg(row + k), xb = __ldg(row + M - k);
      if (k == 0) xa.y = xb.y = 0.0f;                       // DC and Nyquist: imaginary parts ignored
      float2 A, B;
      c2r_pair(xa, xb, s_twn[k], A, B);
      buf0[k] = make_float2(A.y, A.x);                      // swapped: the inverse runs as a forward transform
      if (k != 0 && M - k != k) buf0[M - k] = make_float2(B.y, B.x);
    }
    __syncwarp();
    float2* src = buf0;
    float2* dst = buf1;
    mr_pass_any<true, 32>(a.radix[0], src, dst, s_tw, 1, M / a.radix[0], lane);
    __syncwarp();
    int p = a.radix[0];
    for (int s = 1; s < a.n_pass; ++s) {
      float2* tmp = src;
      src = dst;
      dst = tmp;
      const int R = a.radix[s];
      mr_pass_any<false, 32>(R, src, dst, s_tw + a.tw_off[s], p, M / R, lane);
      __syncwarp();
      p *= R;
    }
    float2* out = reinterpret_cast<float2*>(a.ytmp + ((long long)clip * a.n_frames + frame) * L);
    const float2* w2 = reinterpret_cast<const float2*>(s_win);
    for (int n = lane; n < M; n += 32) {
      const float2 r = dst[n];                              // z[n] = (r.y, r.x) = x[2n] + i x[2n+1]
      out[n] = mul2(make_float2(r.y, r.x), w2[n]);
    }
    __syncwarp();
  }
}

}  // namespace b2l
