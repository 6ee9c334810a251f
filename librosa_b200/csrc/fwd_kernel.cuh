// fwd_kernel.cuh — fused frame + pad + window + real FFT kernel with three epilogues
// (complex STFT / power spectrogram / band-sparse mel projection with optional dB + per-clip max).
//
// Replaces, per frame, the reference's  util.frame -> float64 window product -> scipy.fft.rfft
// (librosa/core/spectrum.py:341-390),  np.abs(.)**power (:3000-3013) and the mel einsum
// (librosa/feature/spectral.py:2160).
//
// Work decomposition: a persistent CTA walks tiles of FT consecutive frames of one clip.  The
// contiguous sample span of a tile, (FT-1)*hop + n_fft floats, is staged once into shared memory
// (frames overlap *inside* shared memory) — by a single 1-D TMA bulk copy (cp.async.bulk + mbarrier)
// for interior tiles, prefetched one tile ahead, or by a cooperative gather with the pad-mode index
// map for tiles that touch the clip edges.  Each group of TPF threads then transforms one frame in
// registers (fft_engine.cuh).
#pragma once
#include "common.cuh"
#include "fft_engine.cuh"
#include "stats.cuh"


namespace b2l {

// ------------------------------------------------------------------ mbarrier / TMA (PTX)
// smem_u32(): fft_engine.cuh
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t phase) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t"
      "}" ::"r"(smem_u32(bar)), "r"(phase)
      : "memory");
}
// 1-D bulk copy global -> shared, completion signalled on an mbarrier (SASS: UBLKCP).
__device__ __forceinline__ void tma_load_1d(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          smem_u32(dst_smem)),
      "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

// ------------------------------------------------------------------ padded sample fetch
// Virtual sample j of a clip of n samples under np.pad semantics (librosa/core/spectrum.py:252-328,
// equivalence to np.pad(y, n_fft//2, mode) per SURVEY Appendix A.2).
__device__ __forceinline__ float load_padded(const float* __restrict__ y, int n, long long j, int mode, int pad) {
  if (j >= 0 && j < n) return __ldg(y + j);
  switch (mode) {
    case PAD_EDGE:
      return __ldg(y + (j < 0 ? 0 : n - 1));
    case PAD_REFLECT: {
      if (n == 1) return __ldg(y);
      long long P = 2LL * (n - 1);
      long long m = j % P;
      if (m < 0) m += P;
      if (m >= n) m = P - m;
      return __ldg(y + m);
    }
    case PAD_SYMMETRIC: {
      long long P = 2LL * n;
      long long m = j % P;
      if (m < 0) m += P;
      if (m >= n) m = P - 1 - m;
      return __ldg(y + m);
    }
    case PAD_LINEAR_RAMP: {
      long long d = j < 0 ? -j : j - (n - 1);          // distance from the edge sample, 1..pad
      float edge = __ldg(y + (j < 0 ? 0 : n - 1));
      long long i = pad - d;                           // np.linspace(0, edge, pad, endpoint=False)[i]
      if (i <= 0) return 0.0f;
      return (float)((double)i * ((double)edge / (double)pad));
    }
    default:
      return 0.0f;
  }
}

// |X|^power from |X|^2 for power != 2 (kept out of line: the default power-2 path never executes it)
static __device__ __noinline__ float power_from_sq(float p2, int power_mode, float power) {
  float mag = sqrtf(p2);
  return power_mode == 1 ? mag : powf(mag, power);
}
__device__ __forceinline__ float sqmag(float2 x) { return fmaf(x.x, x.x, x.y * x.y); }
// 10 * log10(x) through the hardware base-2 logarithm (MUFU.LG2: 2 ulp, i.e. below 1e-6 dB anywhere in the float32
// range, sub-normal inputs included): the library log10f is 28 instructions per value, and the dB epilogue runs once
// per mel row and frame — for the short rows of n_fft = 1024 it was a third of the projection phase.
__device__ __forceinline__ float db10(float x) { return 3.0102999566398120f * __log2f(x); }
__device__ __forceinline__ float sqrt_approx(float x) {
  float r;
  asm("sqrt.approx.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}

// Exchange-buffer slot of Z[M - k] for k = t + TPF*c (the partner of bin k in the real-FFT un-mix).
// For warp-multiple groups the padded index is affine in the lane with a compile-time offset.
template <int M, int TPF, int C>
__device__ __forceinline__ int partner_slot(int t) {
  if constexpr (TPF % 32 == 0) {
    constexpr int WPG = TPF / 32;                 // warps per group
    const int tl = t & 31, tw = t >> 5;
    const int row = tw + WPG * C;                 // k = tl + 32*row
    const int rows = M / 32;
    // tl != 0: M-k = 32*(rows-1-row) + (32-tl);  tl == 0: M-k = 32*((rows-row) mod rows)
    const int a = 33 * (rows - 1 - row) + 32 - tl;
    const int b = 33 * ((rows - row) & (rows - 1));
    return tl == 0 ? b : a;
  } else {
    const int k = t + TPF * C;
    return xphys((M - k) & (M - 1));
  }
}

// ------------------------------------------------------------------ the kernel
// NW warps per CTA.  With NSPLIT > 1 the CTA is NSPLIT independent parts of NW/NSPLIT warps ("virtual CTAs",
// called halves below): each has
// its own staging buffer, exchange area, mbarrier, named barrier and tile sequence, and only the constant
// tables are shared.  The halves drift apart, so the shared-memory-bound phases of one (operand fetch,
// exchange, mel gather) overlap the FP32-bound butterflies of the other instead of all warps of the SM
// hitting the same pipe at once.
template <int LOG2M, int TPF, int NW, int MODE, int NSPLIT>
__global__ void __launch_bounds__(NW * 32, 1) fwd_kernel(const FwdArgs a) {
  using Cfg = FftCfg<LOG2M, TPF>;
  constexpr int M = Cfg::M, N = 2 * M, PPT = Cfg::PPT;
  constexpr int NT = NW * 32;
  constexpr int NH = NSPLIT;                   // independent parts ("halves" when 2)
  constexpr bool DUAL = NSPLIT > 1;
  constexpr int HT = NT / NH;                  // threads per half
  constexpr int HW = NW / NH;                  // warps per half
  constexpr int FT = HT / TPF;                 // frames per tile == frame groups per half
  static_assert(NW % NSPLIT == 0, "the warps are split evenly");
  static_assert(TPF <= 32 || NH + NT / TPF <= 15, "named barriers: 1..NH for the halves, then one per frame group");
  static_assert(FT >= 1 && FT <= 32, "tile must hold 1..32 frames");
  using ML = MelLayout<M, FT>;
  constexpr int H = ML::H;                     // mel rows handled concurrently by one warp (common.cuh)
  constexpr int NPAIR = PPT / 2;               // bin pairs (k, M-k) per thread

  extern __shared__ __align__(128) unsigned char smem[];
  const int tid = threadIdx.x;
  const int half = DUAL ? tid / HT : 0;
  const int htid = tid - half * HT;
  float* s_win = reinterpret_cast<float*>(smem + a.off_win);
  float2* s_tw = reinterpret_cast<float2*>(smem + a.off_tw);
  float* s_melw = reinterpret_cast<float*>(smem + a.off_melw);
  MelRow* s_row = reinterpret_cast<MelRow*>(smem + a.off_melband);
  float* s_in = reinterpret_cast<float*>(smem + a.off_in + half * a.in_stride);
  float2* s_xall = reinterpret_cast<float2*>(smem + a.off_xbuf + half * a.xbuf_stride);
  float* s_p = reinterpret_cast<float*>(s_xall);               // P rows alias the exchange regions (MelLayout)
  uint64_t* s_bar = reinterpret_cast<uint64_t*>(smem + a.off_bar) + half;

  const int grp = htid / TPF;                  // frame group == local frame index
  const int t = htid % TPF;
  const int gbar = 1 + NH + half * FT + grp;   // named barrier of this frame group (used when TPF > 32)
  // stride between the exchange regions of consecutive groups: padded in the modes that park the power row there
  constexpr int GS = (MODE == MODE_MEL || MODE == MODE_STATS) ? ML::GS : Cfg::XBUF_F2;
  float2* xbuf = s_xall + grp * GS;
  float2* xb_t = xbuf + xphys(t);                                   // &xbuf[xphys(t)]: base of the affine accesses
  const float2* xb_neg = xbuf - xphys(t) + ((t & 31) == 0 ? 1 : 0);  // base of the mirror (partner) accesses

  auto half_sync = [&]() {
    if constexpr (DUAL) asm volatile("bar.sync %0, %1;" ::"r"(half + 1), "n"(HT) : "memory");   // ids 1 .. NH
    else __syncthreads();
  };

  // ---- one-time table staging (whole CTA)
  for (int i = tid; i < N; i += NT) s_win[i] = a.window[i];
  for (int i = tid; i < Cfg::TW_COUNT_SPLIT; i += NT) s_tw[i] = a.tw[i];   // split layout (fft_forward SPLIT_TW)
  if constexpr (MODE == MODE_MEL) {
    for (int i = tid; i < a.mel_w_count; i += NT) s_melw[i] = a.mel_w[i];
    for (int i = tid; i < a.n_mel_rows; i += NT) s_row[i] = a.mel_rows[i];
  }
  if constexpr (MODE == MODE_STATS) {
    for (int i = tid; i < a.mel_w_count; i += NT) s_melw[i] = a.mel_w[i];   // bin frequencies
  }
  if (htid == 0) {
    mbar_init(s_bar, 1);
    fence_mbar_init();
  }
  __syncthreads();

  const int span = a.in_floats;
  const bool hop_even = (a.hop & 1) == 0;
  // un-mix twiddle of bin k = t + TPF*c:  W_N^k = W_N^t * W_(2*PPT)^c  (register x compile-time constant)
  const float2 wt = __ldg(a.twn + t);
  auto unmix_tw = [&](auto C) -> float2 {
    constexpr int c = decltype(C)::value;
    if constexpr (c == 0) return wt;
    else return cmul(wt, make_float2(TwC<c, 2 * PPT>::re, TwC<c, 2 * PPT>::im));
  };

  // Tile walk without divisions in the loop: tile = clip * tiles_per_clip + tix, advanced by the constant
  // stride (step_c clips, step_t tiles) of this half.
  // How a tile's span gets into shared memory:
  //   TILE_TMA      entirely inside the clip and 16-byte aligned -> one bulk copy
  //   TILE_TMA_ZERO zero ("constant") padding, aligned: bulk-copy the in-range part, threads zero the rest
  //   TILE_GATHER   anything else (reflect / edge / ... padding, unaligned clips): per-sample gather
  enum { TILE_GATHER = 0, TILE_TMA = 1, TILE_TMA_ZERO = 2 };
  struct TileInfo { int clip, tix, kind, lead, valid; };
  auto describe = [&](int clip, int tix) -> TileInfo {
    TileInfo ti;
    ti.clip = clip;
    ti.tix = tix;
    const long long s0 = (long long)tix * FT * a.hop - a.pad;
    ti.lead = s0 < 0 ? (int)(-s0) : 0;                                      // floats before the clip starts
    const long long end = s0 + span;
    ti.valid = (int)((end > a.n ? (long long)a.n : end) - (s0 + ti.lead));  // in-range floats
    if (!a.tma_ok || ((s0 + ti.lead) & 3) != 0) ti.kind = TILE_GATHER;
    else if (ti.lead == 0 && ti.valid == span) ti.kind = TILE_TMA;
    else if (a.pad_mode == PAD_CONSTANT && ti.valid > 0 && (ti.lead & 3) == 0 && (ti.valid & 3) == 0) ti.kind = TILE_TMA_ZERO;
    else ti.kind = TILE_GATHER;
    return ti;
  };
  // Called by the whole half after the staging buffer has been released (B0): one thread starts the bulk copy of
  // the tile's in-range part, every thread of the half writes the zero padding around it.
  auto prefetch = [&](const TileInfo& ti) {
    if (ti.clip < a.n_clips && ti.kind != TILE_GATHER && htid == 0) {
      const long long s0 = (long long)ti.tix * FT * a.hop - a.pad;
      fence_proxy_async();
      mbar_expect_tx(s_bar, (uint32_t)ti.valid * 4u);
      tma_load_1d(s_in + ti.lead, a.y + (long long)ti.clip * a.clip_stride + s0 + ti.lead, (uint32_t)ti.valid * 4u, s_bar);
    }
    if (ti.clip < a.n_clips && ti.kind == TILE_TMA_ZERO) {
      for (int i = htid; i < ti.lead; i += HT) s_in[i] = 0.0f;
      for (int i = ti.lead + ti.valid + htid; i < span; i += HT) s_in[i] = 0.0f;
    }
  };

  const int tile_step = (int)gridDim.x * NH;
  const int step_c = tile_step / a.tiles_per_clip, step_t = tile_step - step_c * a.tiles_per_clip;
  TileInfo cur;
  {
    const int first = (int)blockIdx.x * NH + half;
    cur = describe(first / a.tiles_per_clip, first % a.tiles_per_clip);
  }
  uint32_t phase = 0;
  prefetch(cur);

  constexpr bool ROWS = (MODE == MODE_MEL || MODE == MODE_STATS);
  float2 v[PPT];
  // ---------------- stage a tile's sample span and turn it into windowed pass-0 operands (first stage fused in)
  auto stage_and_fetch = [&](const TileInfo& ti) {
    if (ti.kind == TILE_GATHER) {
      const float* yc = a.y + (long long)ti.clip * a.clip_stride;
      const long long s0 = (long long)ti.tix * FT * a.hop - a.pad;
      for (int i = htid; i < span; i += HT) s_in[i] = load_padded(yc, a.n, s0 + i, a.pad_mode, a.pad);
      half_sync();
    } else {
      mbar_wait(s_bar, phase);
      phase ^= 1;
      if (ti.kind == TILE_TMA_ZERO) half_sync();   // zeros written by other threads
    }
    const float* fr = s_in + grp * a.hop;
    auto win = [&](auto S) {   // window pair of the element that lands in slot S
      constexpr int off = pass0_offset<Cfg>(decltype(S)::value);
      return *reinterpret_cast<const float2*>(s_win + 2 * (t + off));
    };
    if (hop_even) {
      load_pass0_windowed<Cfg>(v, t, [&](int e) { return *reinterpret_cast<const float2*>(fr + 2 * e); }, win);
    } else {
      load_pass0_windowed<Cfg>(v, t, [&](int e) { return make_float2(fr[2 * e], fr[2 * e + 1]); }, win);
    }
  };
  auto advance = [&](const TileInfo& ti) -> TileInfo {   // next tile of this half
    int nc = ti.clip + step_c, nt = ti.tix + step_t;
    if (nt >= a.tiles_per_clip) { nt -= a.tiles_per_clip; ++nc; }
    return describe(nc, nt);
  };

  for (; cur.clip < a.n_clips;) {
    const int clip = cur.clip, t0 = cur.tix * FT;
    stage_and_fetch(cur);
    const TileInfo nxt = advance(cur);
    // B0: staging buffer consumed -> prefetch the next tile behind the math.
    half_sync();
    prefetch(nxt);
    // In the modes whose power rows share the exchange regions (MEL / STATS), every warp has to be done with the
    // rows of the previous tile before the first exchange write.  That barrier ("rows consumed") sits right
    // there, in the pre-store hook, and not together with B0: the operand fetch and the register-only
    // butterflies of pass 0 of the fast warps overlap the tail of the slow warps' mel items.  (One merged
    // barrier before the first exchange write delays the prefetch: measured 2 % slower.)
    auto rows_consumed = [&]() {
      if constexpr (ROWS) half_sync();
    };

    // ---------------- M-point complex FFT
    fft_forward<Cfg, true, true>(v, t, gbar, xbuf, s_tw, rows_consumed);
    if constexpr (Cfg::NPASS == 1) rows_consumed();
    // Bin pair (k, M-k), k = t + TPF*c < M/2: Z[k] is already in one of this thread's registers; only the
    // upper half of the spectrum (indices >= M/2) has to reach its partner thread.
    // One-warp groups in the row modes (n_fft 2048): v[q] = Z[t + 32q], so the partner Z[M-k] of k = t + 32c is
    // register 31-c of lane 32-t (lane 0: its own register (32-c) mod 32, since Z[M] == Z[0]) and comes by warp
    // shuffle, which keeps 16 stores and 16 loads per thread off the shared-memory pipe.  Everything else goes
    // through shared memory.
    constexpr bool SHFL_UNMIX = TPF == 32 && (MODE == MODE_MEL || MODE == MODE_STATS);
    static_assert(!SHFL_UNMIX || (PPT == 32 && spectrum_offset<Cfg>(1) == 32), "v[q] = Z[t + 32q]");
    // un-mix addresses as one pointer per thread plus constants: measured -1.4 % (mel), -1.9 % (statistics) for
    // one-warp groups in the row modes and -0.5 % for the two-warp groups of n_fft 4096, but +6 % for the plain
    // STFT of n_fft 2048 (register allocation), which therefore keeps the index form
    constexpr bool AFFINE_UNMIX = (TPF % 32 == 0) && (TPF > 32 || MODE == MODE_MEL || MODE == MODE_STATS);
    if constexpr (!SHFL_UNMIX) {
      if constexpr (Cfg::NPASS > 1) group_sync<TPF>(gbar);
      static_for<0, PPT>([&](auto S) {
        constexpr int slot = decltype(S)::value;
        constexpr int D = spectrum_offset<Cfg>(slot);
        if constexpr (D >= M / 2) {
          if constexpr (AFFINE_UNMIX && D % 32 == 0) sts_c64(smem_u32(xb_t) + 8u * (D + D / 32), v[slot]);   // xphys(t + D), D a multiple of 32
          else sts_c64(smem_u32(xbuf) + 8u * xphys(t + D), v[slot]);
        }
      });
      group_sync<TPF>(gbar);
    }
    auto pair_operands = [&](auto C, float2& A, float2& B) {
      constexpr int c = decltype(C)::value;
      constexpr int sa = slot_of_pair<Cfg>(c);
      static_assert(sa >= 0, "pair operand must be register resident");
      A = v[sa];
      if constexpr (SHFL_UNMIX) {
        const float2 send = t == 0 ? v[(32 - c) & 31] : v[31 - c];
        B.x = __shfl_sync(0xffffffffu, send.x, (32 - t) & 31);
        B.y = __shfl_sync(0xffffffffu, send.y, (32 - t) & 31);
      } else if constexpr (AFFINE_UNMIX) {
        // padded slot of Z[M - k], k = t + TPF*c:  K_c - xphys(t) (+ 1 in lane 0 of a warp), K_c a constant —
        // see partner_slot; folded into one pointer per thread
        constexpr int K = 33 * (M / 32 - 1 - (TPF / 32) * c) + 32;
        if constexpr (c == 0) B = t == 0 ? A : xb_neg[K];   // k = 0 pairs with itself (Z[M] == Z[0])
        else B = xb_neg[K];
      } else {
        B = xbuf[partner_slot<M, TPF, c>(t)];
        if constexpr (c == 0) {
          if (t == 0) B = A;   // k = 0 pairs with itself (Z[M] == Z[0])
        }
      }
    };
    auto middle_bin = [&]() -> float2 {   // Z[M/2], read by t == 0 only
      if constexpr (SHFL_UNMIX) return v[PPT / 2];
      else return xbuf[xphys(M / 2)];
    };

    const int frame = t0 + grp;
    const bool frame_ok = frame < a.n_frames;
    // util.valid_audio (librosa/util/utils.py:303-306) on the device: one NaN / Inf sample makes every
    // bin of every frame that reads it non-finite, so testing one spectrum value per thread and frame
    // catches it without a separate pass over the input.
    if (frame_ok && !(fabsf(v[0].x) + fabsf(v[0].y) <= 3.0e38f)) *a.status = 1;

    if constexpr (MODE == MODE_STFT) {
      float2* orow = a.out_c + ((long long)clip * a.n_frames + frame) * (M + 1);
      static_for<0, NPAIR>([&](auto C) {
        const int k = t + TPF * decltype(C)::value;
        float2 A, B, xa, xb;
        pair_operands(C, A, B);
        r2c_pair(A, B, unmix_tw(C), xa, xb);
        stg_c64_if(orow + k, xa, frame_ok);
        stg_c64_if(orow + (M - k), xb, frame_ok);
      });
      if (t == 0) {
        float2 xa, xb;
        float2 zc = middle_bin();
        r2c_pair(zc, zc, make_float2(0.0f, -1.0f), xa, xb);   // W_N^(M/2) = -i
        stg_c64_if(orow + M / 2, xa, frame_ok);
      }
      group_sync<TPF>(gbar);   // pair reads done before the next tile's exchange writes
    } else {
      float pw[PPT + 1];
      static_for<0, NPAIR>([&](auto C) {
        constexpr int c = decltype(C)::value;
        float2 A, B, xa, xb;
        pair_operands(C, A, B);
        r2c_pair(A, B, unmix_tw(C), xa, xb);
        pw[2 * c] = sqmag(xa);
        pw[2 * c + 1] = sqmag(xb);
      });
      pw[PPT] = 0.0f;
      if (t == 0) {
        float2 xa, xb;
        float2 zc = middle_bin();
        r2c_pair(zc, zc, make_float2(0.0f, -1.0f), xa, xb);
        pw[PPT] = sqmag(xa);
      }
      if (MODE == MODE_STATS || a.power_mode == 1) {
        // |X| (power = 1; the statistics of MODE_STATS are defined on it): MUFU-based square root, inline.
        // sqrt.approx.f32 is accurate to 2^-23 relative; 33 calls of an out-of-line IEEE square root per
        // thread and frame would cost as much as half the FFT.
        static_for<0, PPT + 1>([&](auto S) { pw[decltype(S)::value] = sqrt_approx(pw[decltype(S)::value]); });
      } else if (a.power_mode != 2) {   // warp-uniform, cold: general exponent through powf
        static_for<0, PPT + 1>([&](auto S) {
          pw[decltype(S)::value] = power_from_sq(pw[decltype(S)::value], a.power_mode, a.power);
        });
      }
      if constexpr (MODE == MODE_SPEC) {
        float* orow = a.out_r + ((long long)clip * a.n_frames + frame) * (M + 1);
        if (frame_ok) {
          static_for<0, NPAIR>([&](auto C) {
            constexpr int c = decltype(C)::value;
            const int k = t + TPF * c;
            orow[k] = pw[2 * c];
            orow[M - k] = pw[2 * c + 1];
          });
          if (t == 0) orow[M / 2] = pw[PPT];
        }
        group_sync<TPF>(gbar);
      } else {
        // ---------------- band-sparse mel projection over the tile
        // The power row of frame f goes to the exchange region of its own group (P[f][k] at word f*RS + k,
        // MelLayout): only the group itself has to be done with its Z before the row is written.  Bins
        // M+1 .. M+3 of every row are kept at zero so that 4-bin groups may run past the Nyquist bin.
        constexpr int RS = ML::RS;
        group_sync<TPF>(gbar);   // every thread of the group is done reading the exchange region (last pass, pairs)
        float* prow = reinterpret_cast<float*>(xbuf);
        static_for<0, NPAIR>([&](auto C) {
          constexpr int c = decltype(C)::value;
          const int k = t + TPF * c;
          prow[k] = pw[2 * c];
          prow[M - k] = pw[2 * c + 1];
        });
        if (t == 0) {
          prow[M / 2] = pw[PPT];
          prow[M + 1] = 0.0f;
          prow[M + 2] = 0.0f;
          prow[M + 3] = 0.0f;
        }
        half_sync();   // B2: the tile's rows are complete
        if constexpr (MODE == MODE_STATS) {
          // one warp per frame of the tile: statistics of the magnitude row (stats.cuh)
          const int hwarp = htid >> 5, lane = htid & 31;
          for (int f = hwarp; f < FT; f += HW) {
            bool negative;
            const float r = frame_stats(s_p + f * RS, s_melw, M + 1, lane, a.stats, &negative);
            if (lane < N_STATS && t0 + f < a.n_frames)
              a.out_r[((long long)clip * N_STATS + lane) * a.n_frames + t0 + f] = r;
          }
        } else {
          // Work item = H adjacent mel rows; lane (fp, j) accumulates row item*H + j for the frame pair
          // (fp, fp + FP) over that row's padded band (host-built MelRow table: the rows of an item share
          // one trip count, start bins follow the bank rule of MelLayout, weights are zero padded and 16-byte
          // aligned).  One 16-byte weight fetch and one 16-byte power fetch per frame feed eight FMAs; no
          // cross-lane reduction.  Warp w of a half takes items w, w + HW, w + 2 HW, ...: round-robin in natural
          // order keeps neighbouring rows, whose bands overlap in shared memory, on warps that run at the same time
          // (a longest-first deal, against item lengths that differ tenfold from the lowest to the highest rows,
          // measured no faster).
          constexpr int FP = ML::FP;
          constexpr bool PAIR = ML::PAIR;
          const int hwarp = htid >> 5, lane = htid & 31;
          const int fp = lane & (FP - 1), j = lane / FP;
          const bool ok_a = (t0 + fp) < a.n_frames;
          const bool ok_b = PAIR && (t0 + fp + FP) < a.n_frames;
          float wmax = -INFINITY;
          const float* pbase = s_p + fp * RS;
          // output row stride / base: the public [clip][mel][frame] layout, or the tiled mfcc scratch whose
          // 64-frame tiles are contiguous 32 KB blocks for dct_clamp4_kernel (t0 + fp and t0 + fp + FP share a tile)
          const long long orow = a.out_tiled ? 64 : a.n_frames;
          float* obase = a.out_tiled
                             ? a.out_r + ((long long)clip * ((a.n_frames + 63) >> 6) + (t0 >> 6)) * a.n_mels * 64 + (t0 & 63) + fp
                             : a.out_r + (long long)clip * a.n_mels * a.n_frames + t0 + fp;
          // the row record is fetched one item ahead: a shared-memory load that would otherwise sit in front of
          // every (short) row with four warps per scheduler to hide it
          const int n_items = a.n_mel_rows / H;
          MelRow row_nx = s_row[(hwarp < n_items ? hwarp * H : 0) + j];
          for (int item = hwarp; item < n_items; item += HW) {
            const int m = item * H + j;
            const MelRow row = row_nx;
            const int item_nx = item + HW;
            row_nx = s_row[(item_nx < n_items ? item_nx * H : 0) + j];
            const float4* wp = reinterpret_cast<const float4*>(s_melw + row.off);
            const float4* pa = reinterpret_cast<const float4*>(pbase + row.lo);
            const float4* wend = wp + row.quads;
            float a0 = 0.0f, a1 = 0.0f, b0 = 0.0f, b1 = 0.0f;
            if constexpr (PAIR) {
              const float4* pb = pa + (FP * RS) / 4;
#pragma unroll 2
              for (; wp != wend; ++wp, ++pa, ++pb) {
                const float4 w = *wp, x = *pa, y = *pb;
                a0 = fmaf(w.x, x.x, a0);
                b0 = fmaf(w.x, y.x, b0);
                a1 = fmaf(w.y, x.y, a1);
                b1 = fmaf(w.y, y.y, b1);
                a0 = fmaf(w.z, x.z, a0);
                b0 = fmaf(w.z, y.z, b0);
                a1 = fmaf(w.w, x.w, a1);
                b1 = fmaf(w.w, y.w, b1);
              }
            } else {
#pragma unroll 2
              for (; wp != wend; ++wp, ++pa) {
                const float4 w = *wp, x = *pa;
                a0 = fmaf(w.x, x.x, a0);
                a1 = fmaf(w.y, x.y, a1);
                a0 = fmaf(w.z, x.z, a0);
                a1 = fmaf(w.w, x.w, a1);
              }
            }
            float va = a0 + a1, vb = b0 + b1;
            if (m < a.n_mels) {
              if (a.log_mode) {
                va = db10(fmaxf(a.amin, va)) - a.db_sub;
                if (ok_a) wmax = fmaxf(wmax, va);
                if constexpr (PAIR) {
                  vb = db10(fmaxf(a.amin, vb)) - a.db_sub;
                  if (ok_b) wmax = fmaxf(wmax, vb);
                }
              }
              float* o = obase + (long long)m * orow;
              if (ok_a) o[0] = va;
              if (ok_b) o[FP] = vb;
            }
          }
          if (a.log_mode) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) wmax = fmaxf(wmax, __shfl_xor_sync(0xffffffffu, wmax, o));
            if (lane == 0 && wmax > -INFINITY) atomicMax(a.clip_max + clip, float_to_key(wmax));
          }
        }
        // (the P reads are ordered before the next tile's exchange writes by its "rows consumed" barrier)
      }
    }
    cur = nxt;
  }
}

}  // namespace b2l
