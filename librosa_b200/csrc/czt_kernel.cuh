// czt_kernel.cuh — STFT frames of arbitrary length L (not a power of two) by Bluestein's chirp-z
// transform on top of the register FFT engine.
//
// librosa.stft accepts any n_fft (the reference's own tests use 501 / 1023 / 1025, speech front ends use
// 400); scipy.fft.rfft handles them with mixed-radix / Bluestein plans (librosa/core/spectrum.py:388).
// With b[n] = exp(-i*pi*n^2/L):
//     X[k] = b[k] * sum_n (x[n] w[n] b[n]) * conj(b[k-n])  =  b[k] * IFFT_P( FFT_P(a) . FFT_P(h) )[k]
// a[n] = x[n] w[n] b[n] zero-padded to P >= 2L-1 (a power of two), h[m] = conj(b[|m|]) wrapped to length P.
// FFT_P(h)/P, w*b and b are precomputed on the host in double precision.
//
// One group of TPF = P/32 threads per PAIR of frames (same engine configuration as an n_fft = 2P real frame; the
// two real frames are the real and imaginary part of one complex input);
// frames are read straight from global memory through the np.pad index map (the 2-4x frame overlap is
// served by L2), the product with FFT_P(h) is applied in registers, and the inverse transform reuses the
// forward one with re/im swapped.
#pragma once
#include "common.cuh"
#include "fft_engine.cuh"

namespace b2l {

struct CztArgs {
  const float* y;
  long long clip_stride;
  int n, n_clips;
  int L, hop, pad, pad_mode, n_frames, n_bins;   // n_bins = 1 + L/2
  const float2* wb;      // [L]  window[n] * b[n]
  const float2* bk;      // [n_bins] b[k]
  const float2* hf;      // [P]  FFT_P(h) / P
  float2* out_c;         // complex64 [clip][frame][bin]   (mode 0)
  float* out_r;          // |X|^power [clip][frame][bin]   (mode 1)
  int mode, power_mode;
  float power;
  int* status;
};

template <int LOG2P, int TPF, int NW>
__global__ void __launch_bounds__(NW * 32, 1) czt_kernel(const CztArgs a) {
  using Cfg = FftCfg<LOG2P, TPF>;
  constexpr int P = Cfg::M, PPT = Cfg::PPT;
  constexpr int NT = NW * 32;
  constexpr int G = NT / TPF;                  // frames per CTA step
  static_assert(TPF <= 32 || 1 + NT / TPF <= 15, "named barriers");
  extern __shared__ __align__(128) unsigned char smem[];
  float2* s_tw = reinterpret_cast<float2*>(smem);
  float2* s_xall = s_tw + ((Cfg::TW_COUNT + 15) & ~15);
  // the three per-plan tables (FFT_P(h)/P, window * chirp, output chirp) live in shared memory: every frame
  // reads all of them, and as global loads they competed with the sample gather for the LSU
  float2* s_hf = s_xall + G * Cfg::XBUF_F2;
  float2* s_wb = s_hf + P;
  float2* s_bk = s_wb + ((a.L + 1) & ~1);
  const int tid = threadIdx.x, grp = tid / TPF, t = tid % TPF;
  const int gbar = 2 + grp;
  float2* xbuf = s_xall + grp * Cfg::XBUF_F2;
  // inter-pass twiddles of the engine (the host appends them to the FFT_P(h)/P table)
  for (int i = tid; i < Cfg::TW_COUNT; i += NT) s_tw[i] = a.hf[P + i];   // appended after FFT_P(h)/P
  for (int i = tid; i < P; i += NT) s_hf[i] = a.hf[i];
  for (int i = tid; i < a.L; i += NT) s_wb[i] = a.wb[i];
  for (int i = tid; i < a.n_bins; i += NT) s_bk[i] = a.bk[i];
  __syncthreads();

  // Two real frames ride through one complex chirp-z transform: z = xA + i xB gives Z = XA + i XB, and since
  // XA, XB are spectra of real signals, XA[k] = (Z[k] + conj Z[L-k]) / 2 and XB[k] = (Z[k] - conj Z[L-k]) / 2i.
  // Z[L-k] = c[L-k] * b[L-k] with b[L-k] = (-1)^L b[k], so the chirp table still only covers k <= L/2.
  // Frames are paired INSIDE a clip (frames 2j, 2j+1; the odd last frame of a clip rides alone with a zero
  // partner): a non-finite or much louder neighbouring clip can then never leak into this one through the
  // un-mix (Z[k] +- conj Z[L-k]) / 2, whose round-off scales with the louder partner.
  const int ppc = (a.n_frames + 1) / 2;                       // pairs per clip
  const long long pairs = (long long)a.n_clips * ppc;
  const float sgn = (a.L & 1) ? -1.0f : 1.0f;
  for (long long p0 = (long long)blockIdx.x * G; p0 < pairs; p0 += (long long)gridDim.x * G) {
    // groups past the end redo the last pair (their stores are masked): sub-warp groups share a warp
    const long long pidx = min(p0 + grp, pairs - 1);
    const bool live_a = p0 + grp < pairs;
    const int clip_a = (int)(pidx / ppc), frame_a = 2 * (int)(pidx % ppc);
    const int clip_b = clip_a, frame_b = min(frame_a + 1, a.n_frames - 1);
    const bool live_b = live_a && frame_a + 1 < a.n_frames;
    const float* ya = a.y + (long long)clip_a * a.clip_stride;
    const float* yb = ya;
    const long long sa = (long long)frame_a * a.hop - a.pad, sb = (long long)frame_b * a.hop - a.pad;
    float2 v[PPT];
    load_pass0<Cfg>(v, t, [&](int e) {
      if (e >= a.L) return make_float2(0.0f, 0.0f);
      const float xa = load_padded(ya, a.n, sa + e, a.pad_mode, a.pad);
      const float xb = live_b ? load_padded(yb, a.n, sb + e, a.pad_mode, a.pad) : 0.0f;
      const float2 w = s_wb[e];
      return make_float2(fmaf(xa, w.x, -xb * w.y), fmaf(xa, w.y, xb * w.x));      // (xa + i xb) * w
    });
    fft_forward<Cfg>(v, t, gbar, xbuf, s_tw);
    if (live_a && !(fabsf(v[0].x) + fabsf(v[0].y) <= 3.0e38f)) *a.status = B2L_STATUS_NOT_FINITE_SAMPLE;   // util.valid_audio
    // C = A . FFT(h)/P in registers, published (re/im swapped) for the inverse transform's first pass
    if constexpr (Cfg::NPASS > 1) group_sync<TPF>(gbar);
    static_for<0, PPT>([&](auto S) {
      constexpr int slot = decltype(S)::value;
      const int idx = t + spectrum_offset<Cfg>(slot);
      const float2 c = cmul(v[slot], s_hf[idx]);
      xbuf[xphys(idx)] = make_float2(c.y, c.x);
    });
    group_sync<TPF>(gbar);
    load_pass0<Cfg>(v, t, [&](int e) { return xbuf[xphys(e)]; });
    group_sync<TPF>(gbar);
    fft_forward<Cfg>(v, t, gbar, xbuf, s_tw);
    // publish c[idx] (un-swapped) for idx < L so that every bin can reach its mirror L - k
    if constexpr (Cfg::NPASS > 1) group_sync<TPF>(gbar);
    static_for<0, PPT>([&](auto S) {
      constexpr int slot = decltype(S)::value;
      const int idx = t + spectrum_offset<Cfg>(slot);
      if (idx < a.L) xbuf[xphys(idx)] = make_float2(v[slot].y, v[slot].x);
    });
    group_sync<TPF>(gbar);
    // k <= L/2:  Z[k] = c[k] b[k],  conj Z[L-k] = sgn * conj(c[L-k]) conj(b[k])
    static_for<0, PPT>([&](auto S) {
      constexpr int slot = decltype(S)::value;
      const int k = t + spectrum_offset<Cfg>(slot);
      if (k < a.n_bins) {
        const float2 b = s_bk[k];
        const float2 zk = cmul(make_float2(v[slot].y, v[slot].x), b);
        const float2 cm = xbuf[xphys(k == 0 ? 0 : a.L - k)];
        const float sk = k == 0 ? 1.0f : sgn;                                                  // Z[L] is Z[0] itself
        const float2 zm = cmul(make_float2(cm.x, -cm.y), make_float2(sk * b.x, -sk * b.y));     // conj Z[L-k]
        const float2 XA = make_float2(0.5f * (zk.x + zm.x), 0.5f * (zk.y + zm.y));
        const float2 XB = make_float2(0.5f * (zk.y - zm.y), -0.5f * (zk.x - zm.x));             // (zk - zm) / 2i
        auto emit = [&](float2 X, int clip, int frame) {
          const long long o = ((long long)clip * a.n_frames + frame) * a.n_bins + k;
          if (a.mode == 0) {
            a.out_c[o] = X;
          } else {
            const float p2 = sqmag(X);
            a.out_r[o] = a.power_mode == 2 ? p2 : (a.power_mode == 1 ? sqrt_approx(p2) : power_from_sq(p2, a.power_mode, a.power));
          }
        };
        if (live_a) emit(XA, clip_a, frame_a);
        if (live_b) emit(XB, clip_b, frame_b);
      }
    });
    group_sync<TPF>(gbar);   // mirror reads done before the next pair's exchange writes
  }
}


// ------------------------------------------------------------------ inverse: irfft of length L per frame
// y[n] = (1/L) sum_k Xfull[k] e^{+2 pi i k n / L} with Xfull the Hermitian extension of the L/2+1 stored bins
// (scipy.fft.irfft(D, n=L): Im of DC — and of the Nyquist bin for even L — is ignored).  Same chirp-z
// structure with conjugated chirps:  y[n] = Re( conj(b[n]) * IFFT_P( FFT_P(Xfull conj(b)) . conj(FFT_P(h)) )[n] ) / L.
// The windowed frames (window * 1/L folded into `wbi`) go to a scratch array [clip][frame][L]; ola_kernel
// overlap-adds and normalises them (librosa/core/spectrum.py:598-624).
struct CztInvArgs {
  const float2* D;       // [clip][frames_stored][n_bins]
  long long d_clip_stride;
  int n_clips, n_frames, L, n_bins;
  const float2* bfull;   // [L] b[k]
  const float2* wbi;     // [L] conj(b[n]) * window[n] / L
  const float2* hf;      // [P] FFT_P(h)/P, then the engine twiddles
  float* ytmp;           // [clip][n_frames][L]
};

template <int LOG2P, int TPF, int NW>
__global__ void __launch_bounds__(NW * 32, 1) czt_inv_kernel(const CztInvArgs a) {
  using Cfg = FftCfg<LOG2P, TPF>;
  constexpr int P = Cfg::M, PPT = Cfg::PPT;
  constexpr int NT = NW * 32;
  constexpr int G = NT / TPF;
  extern __shared__ __align__(128) unsigned char smem[];
  float2* s_tw = reinterpret_cast<float2*>(smem);
  float2* s_xall = s_tw + ((Cfg::TW_COUNT + 15) & ~15);
  float2* s_hf = s_xall + G * Cfg::XBUF_F2;               // plan tables in shared memory, as in czt_kernel
  float2* s_wbi = s_hf + P;                               // (the input chirp stays in global memory: with it the
                                                          //  P = 4096 configuration would not fit)
  const int tid = threadIdx.x, grp = tid / TPF, t = tid % TPF;
  const int gbar = 2 + grp;
  float2* xbuf = s_xall + grp * Cfg::XBUF_F2;
  for (int i = tid; i < Cfg::TW_COUNT; i += NT) s_tw[i] = a.hf[P + i];
  for (int i = tid; i < P; i += NT) s_hf[i] = a.hf[i];
  for (int i = tid; i < a.L; i += NT) s_wbi[i] = a.wbi[i];
  __syncthreads();
  // As in czt_kernel, two frames share one complex transform: U = X_A + i X_B (Hermitian extensions) inverts to
  // u = y_A + i y_B because both signals are real.
  const int ppc = (a.n_frames + 1) / 2;                       // pairs stay inside a clip (see czt_kernel)
  const long long pairs = (long long)a.n_clips * ppc;
  for (long long p0 = (long long)blockIdx.x * G; p0 < pairs; p0 += (long long)gridDim.x * G) {
    const long long pidx = min(p0 + grp, pairs - 1);
    const bool live_a = p0 + grp < pairs;
    const int clip_a = (int)(pidx / ppc), frame_a = 2 * (int)(pidx % ppc);
    const int clip_b = clip_a, frame_b = min(frame_a + 1, a.n_frames - 1);
    const bool live_b = live_a && frame_a + 1 < a.n_frames;
    const float2* Da = a.D + (long long)clip_a * a.d_clip_stride + (long long)frame_a * a.n_bins;
    const float2* Db = a.D + (long long)clip_b * a.d_clip_stride + (long long)frame_b * a.n_bins;
    float2 v[PPT];
    load_pass0<Cfg>(v, t, [&](int e) {
      if (e >= a.L) return make_float2(0.0f, 0.0f);
      float2 xa, xb;
      if (e < a.n_bins) {
        xa = __ldg(Da + e);
        xb = __ldg(Db + e);
        if (e == 0 || 2 * e == a.L) xa.y = xb.y = 0.0f;  // DC, and Nyquist when L is even
      } else {
        xa = __ldg(Da + (a.L - e));
        xb = __ldg(Db + (a.L - e));
        xa.y = -xa.y;                                    // Hermitian extension
        xb.y = -xb.y;
      }
      if (!live_b) xb = make_float2(0.0f, 0.0f);         // odd last frame of a clip: no partner
      const float2 x = make_float2(xa.x - xb.y, xa.y + xb.x);     // X_A + i X_B
      const float2 b = __ldg(a.bfull + e);
      return cmul(x, make_float2(b.x, -b.y));            // U[e] * conj(b[e])
    });
    fft_forward<Cfg>(v, t, gbar, xbuf, s_tw);
    if constexpr (Cfg::NPASS > 1) group_sync<TPF>(gbar);
    static_for<0, PPT>([&](auto S) {
      constexpr int slot = decltype(S)::value;
      const int idx = t + spectrum_offset<Cfg>(slot);
      const float2 h = s_hf[idx];
      const float2 c = cmul(v[slot], make_float2(h.x, -h.y));     // conj(FFT_P(h)) = FFT_P(conj h), h symmetric
      xbuf[xphys(idx)] = make_float2(c.y, c.x);
    });
    group_sync<TPF>(gbar);
    load_pass0<Cfg>(v, t, [&](int e) { return xbuf[xphys(e)]; });
    group_sync<TPF>(gbar);
    fft_forward<Cfg>(v, t, gbar, xbuf, s_tw);
    static_for<0, PPT>([&](auto S) {
      constexpr int slot = decltype(S)::value;
      const int nn = t + spectrum_offset<Cfg>(slot);
      if (nn < a.L) {
        const float2 w = s_wbi[nn];
        // u = c * w with c un-swapped (c.re = v.y, c.im = v.x): frame A is its real part, frame B its imaginary part
        if (live_a) a.ytmp[((long long)clip_a * a.n_frames + frame_a) * a.L + nn] = fmaf(v[slot].y, w.x, -v[slot].x * w.y);
        if (live_b) a.ytmp[((long long)clip_b * a.n_frames + frame_b) * a.L + nn] = fmaf(v[slot].y, w.y, v[slot].x * w.x);
      }
    });
    if constexpr (Cfg::NPASS > 1) group_sync<TPF>(gbar);
  }
}

}  // namespace b2l
