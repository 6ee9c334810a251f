// fft_engine.cuh — register-resident Stockham complex FFT for sm_90a.
//
// One "frame group" of TPF threads transforms M = 2^LOG2M complex points; every thread keeps
// PPT = M / TPF points (32 for all production sizes) in registers.  Each pass is a radix-R DFT done
// entirely in registers (decimation-in-time, compile-time twiddles folded into FFMA immediates);
// passes exchange data through a padded shared-memory buffer that belongs to the group alone,
// so a warp-sized group synchronises with __syncwarp only.
//
// Stockham pass (radix R, sub-transform length p, T = M / R butterflies, butterfly i):
//     k = i mod p ;  u[r] = x[i + r*T] * exp(-2*pi*i * r*k / (p*R)) ;  v = DFT_R(u)
//     y[(i - k)*R + k + q*p] = v[q]
// After the last pass y is the DFT in natural order.
//
// The real-input transform of length N = 2M packs even/odd samples as re/im (z[n] = x[2n] + i x[2n+1])
// and un-mixes the result with one twiddled butterfly per bin pair (k, M-k); see r2c_pair().
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <type_traits>
#include <utility>

namespace b2l {

// ------------------------------------------------------------------ compile-time helpers
template <int I, int N, class F>
__device__ __forceinline__ void static_for(F&& f) {
  if constexpr (I < N) {
    f(std::integral_constant<int, I>{});
    static_for<I + 1, N>(static_cast<F&&>(f));
  }
}

__host__ __device__ constexpr int ilog2c(int x) { return x <= 1 ? 0 : 1 + ilog2c(x >> 1); }
__host__ __device__ constexpr int bitrevc(int x, int bits) {
  int r = 0;
  for (int i = 0; i < bits; ++i) r |= ((x >> i) & 1) << (bits - 1 - i);
  return r;
}

// cos / sin of 2*pi*j/n evaluated by the host compiler (octant reduction keeps 0, +-1, sqrt(1/2) exact)
constexpr double kPi = 3.14159265358979323846264338327950288;
constexpr double taylor_sin(double x) {
  double x2 = x * x, term = x, sum = x;
  for (int i = 1; i < 14; ++i) { term *= -x2 / double((2 * i) * (2 * i + 1)); sum += term; }
  return sum;
}
constexpr double taylor_cos(double x) {
  double x2 = x * x, term = 1.0, sum = 1.0;
  for (int i = 1; i < 14; ++i) { term *= -x2 / double((2 * i - 1) * (2 * i)); sum += term; }
  return sum;
}
struct cpair { double c, s; };
constexpr cpair cossin2pi(long j, long n) {   // (cos, sin) of 2*pi*j/n
  long t = ((j % n) + n) % n;
  long o = (8 * t) / n;          // octant
  long r = 8 * t - o * n;        // position inside the octant, in units of 2*pi/(8n)
  bool odd = (o & 1) != 0;
  long rr = odd ? (n - r) : r;
  double a = kPi * double(rr) / (4.0 * double(n));
  double c = taylor_cos(a), s = taylor_sin(a);
  switch (o) {
    case 0: return {c, s};
    case 1: return {s, c};
    case 2: return {-s, c};
    case 3: return {-c, s};
    case 4: return {-c, -s};
    case 5: return {-s, -c};
    case 6: return {s, -c};
    default: return {c, -s};
  }
}
template <int J, int N>
struct TwC {   // W_N^J = exp(-2*pi*i*J/N)
  static constexpr float re = float(cossin2pi(J, N).c);
  static constexpr float im = float(-cossin2pi(J, N).s);
};

// ------------------------------------------------------------------ complex helpers
// Component-wise FP32 operations on a complex value (re, im).  Every butterfly below is written with them, so the
// operation order inside each component is fixed by the source (FFMA / FADD / FMUL per component on sm_90).
__device__ __forceinline__ float2 bc2(float a) { return make_float2(a, a); }
__device__ __forceinline__ float2 neg2(float2 a) { return make_float2(-a.x, -a.y); }
__device__ __forceinline__ float2 muli2(float2 a) { return make_float2(-a.y, a.x); }    //  i * a
__device__ __forceinline__ float2 mulni2(float2 a) { return make_float2(a.y, -a.x); }   // -i * a
__device__ __forceinline__ float2 add2(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 sub2(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }
__device__ __forceinline__ float2 mul2(float2 a, float2 b) { return make_float2(a.x * b.x, a.y * b.y); }
__device__ __forceinline__ float2 fma2(float2 a, float2 b, float2 c) {
  return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
}

// a * b = b.x * a + b.y * (i a)
__device__ __forceinline__ float2 cmul(float2 a, float2 b) {
  return fma2(muli2(a), bc2(b.y), mul2(a, bc2(b.x)));
}
// Shared-memory store of a complex value as one v2.f32 store written in PTX.  saddr: 32-bit shared-window address.
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void sts_c64(uint32_t saddr, float2 v) {
  // no "memory" clobber: the statement stays ordered against the barriers (volatile asm, and they do clobber), and
  // the compiler remains free to move independent loads across it
  asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(saddr), "f"(v.x), "f"(v.y));
}
// Predicated global store of a complex value: one @p STG.64, never a branch (a branch per bin pair serialises the
// un-mix loop: ptxas stops interleaving the pairs).
__device__ __forceinline__ void stg_c64_if(float2* p, float2 v, bool ok) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %3, 0;\n\t@p st.global.v2.f32 [%0], {%1, %2};\n\t}" ::"l"(p), "f"(v.x), "f"(v.y),
      "r"((int)ok));
}

// DIT butterfly  (a, b) <- (a + w b, a - w b)  with a compile-time twiddle.
template <int J, int N>
__device__ __forceinline__ void bfly(float2& a, float2& b) {
  constexpr int j = ((J % N) + N) % N;
  if constexpr (j == 0) {
    float2 s = add2(a, b);
    b = sub2(a, b);
    a = s;
  } else if constexpr (4 * j == N) {            // w = -i
    float2 s = add2(a, mulni2(b));
    b = add2(a, muli2(b));
    a = s;
  } else {
    constexpr float wr = TwC<j, N>::re, wi = TwC<j, N>::im;
    float2 s = fma2(bc2(wr), b, a);              // a + wr * b
    s = fma2(bc2(wi), muli2(b), s);              //   + wi * (i b)
    b = fma2(bc2(2.0f), a, neg2(s));             // a - w b = 2 a - (a + w b)
    a = s;
  }
}

// In-register radix-R DFT on v[BASE .. BASE+R): input in bit-reversed slots, output natural.  S0 = 1 skips
// the first (twiddle-free) stage: the caller already formed the sums / differences of the slot pairs
// (2j, 2j+1) — see load_pass0_windowed, which fuses them with the window product.
template <int R, int BASE, int S0 = 0, int N>
__device__ __forceinline__ void dft_reg(float2 (&v)[N]) {
  constexpr int LOGR = ilog2c(R);
  static_for<S0, LOGR>([&](auto S) {
    constexpr int h = 1 << decltype(S)::value;
    static_for<0, R / 2>([&](auto I) {
      constexpr int i = decltype(I)::value;
      constexpr int blk = i / h, j = i % h;
      constexpr int ia = BASE + blk * 2 * h + j;
      bfly<j, 2 * h>(v[ia], v[ia + h]);
    });
  });
}

// ------------------------------------------------------------------ schedule
// Split twiddle table of a radix-32 pass: r = kTwSplitLo*a + b.  Row j holds W^(e k) with e = tw_row_exponent(j):
// the kTwSplitLo - 1 "low" factors (e = b), then the 32/kTwSplitLo - 1 "high" ones (e = kTwSplitLo*a).
constexpr int kTwSplitLo = 8;
constexpr int kTwSplitRows = (kTwSplitLo - 1) + (32 / kTwSplitLo - 1);
__host__ __device__ constexpr int tw_row_exponent(int row, bool split_pass) {
  return !split_pass || row < kTwSplitLo - 1 ? row + 1 : kTwSplitLo * (row - kTwSplitLo + 2);
}
// Passes of 2^log2m points that take the split table: radix-32 passes after the first, up to n_fft 4096 (the n_fft
// 8192 STFT kernel spills 16 instead of 8 bytes with it).
__host__ __device__ constexpr bool tw_split_pass(int log2m, int s, int radix) {
  return s > 0 && radix == 32 && log2m <= 11;
}

template <int LOG2M_, int TPF_>
struct FftCfg {
  static constexpr int LOG2M = LOG2M_;
  static constexpr int M = 1 << LOG2M_;
  static constexpr int TPF = TPF_;
  static constexpr int PPT = M / TPF_;
  static_assert(PPT >= 1 && PPT <= 32, "points per thread must be 1..32");
  static constexpr int LOGP = ilog2c(PPT);
  static constexpr int NPASS = PPT == 1 ? 1 : (LOG2M_ + LOGP - 1) / LOGP;
  // greedy: every pass uses radix PPT except the last, which takes what is left
  __host__ __device__ static constexpr int log_radix(int s) {
    int left = LOG2M_ - s * LOGP;
    return left >= LOGP ? LOGP : left;
  }
  __host__ __device__ static constexpr int radix(int s) { return 1 << log_radix(s); }
  __host__ __device__ static constexpr int sublen(int s) { return 1 << (s * LOGP); }   // p before pass s
  // twiddle table: pass s >= 1 stores tw_rows(s) rows of p_s entries, row j at tw[tw_offset(s) + j*p + k].
  // Full table: row r-1 = W_(pR)^(r k).  Split table: a pass of tw_split_pass stores the factors of r = 8a + b,
  // rows W^(b k) for b = 1..7 and then W^(8a k) for a = 1..3 (see tw_row_exponent); other passes as the full table.
  __host__ __device__ static constexpr int tw_rows(int s, bool split) {
    return split && tw_split_pass(LOG2M_, s, radix(s)) ? kTwSplitRows : radix(s) - 1;
  }
  __host__ __device__ static constexpr int tw_offset(int s, bool split = false) {
    int off = 0;
    for (int q = 1; q < s; ++q) off += tw_rows(q, split) * sublen(q);
    return off;
  }
  static constexpr int TW_COUNT = tw_offset(NPASS);
  static constexpr int TW_COUNT_SPLIT = tw_offset(NPASS, true);
  // exchange buffer: M complex values, one pad slot per 32
  static constexpr int XBUF_F2 = M + M / 32;
};

__device__ __forceinline__ int xphys(int e) { return e + (e >> 5); }

// Group barrier: warp-sized (or smaller) groups use __syncwarp, larger ones the named barrier whose id the
// caller assigns to the group (unique within the CTA, 1..15).
template <int TPF>
__device__ __forceinline__ void group_sync(int barrier_id) {
  if constexpr (TPF <= 32) {
    __syncwarp();
  } else {
    asm volatile("bar.sync %0, %1;" ::"r"(barrier_id), "n"(TPF) : "memory");   // ids 1..15, caller-assigned
  }
}

// ------------------------------------------------------------------ the transform
// Pass-0 operand fetch: v[slot] = load_in(e) for the elements thread t owns in the first pass
// (bit-reversed slots, as dft_reg expects).  Kept separate from fft_forward so callers can pick an
// aligned / unaligned / global-memory loader without duplicating the transform body.
template <class Cfg, class LoadIn>
__device__ __forceinline__ void load_pass0(float2 (&v)[Cfg::PPT], int t, LoadIn&& load_in) {
  constexpr int R = Cfg::radix(0), LOGR = Cfg::log_radix(0), T = Cfg::M / R, NB = Cfg::PPT / R;
  static_for<0, NB>([&](auto B) {
    constexpr int b = decltype(B)::value;
    const int i = t + Cfg::TPF * b;
    static_for<0, R>([&](auto Rr) {
      constexpr int r = decltype(Rr)::value;
      v[b * R + bitrevc(r, LOGR)] = load_in(i + r * T);
    });
  });
}

// Pass-0 operand fetch fused with the window product and the first butterfly stage of dft_reg: the slots
// (2j, 2j+1) of a radix-R block hold elements r and r + R/2, whose first-stage butterfly is twiddle free, so
//     v[2j] = xa*wa + xb*wb ,  v[2j+1] = xa*wa - xb*wb        (1 FMUL + 2 FFMA per component instead of
// 2 FMUL + 2 FADD).  load_x(e) returns the sample pair (x[2e], x[2e+1]); win(SLOT) the window pair of the
// element that lands in that slot (a compile-time slot index: the window source may be a register chunk).
// Requires radix(0) >= 2; run dft_reg<R, BASE, 1> afterwards.
template <class Cfg, class LoadX, class Win>
__device__ __forceinline__ void load_pass0_windowed(float2 (&v)[Cfg::PPT], int t, LoadX&& load_x, Win&& win) {
  constexpr int R = Cfg::radix(0), LOGR = Cfg::log_radix(0), T = Cfg::M / R, NB = Cfg::PPT / R;
  static_assert(R >= 2, "fused first stage needs a radix of at least 2");
  static_for<0, NB>([&](auto B) {
    constexpr int b = decltype(B)::value;
    const int i = t + Cfg::TPF * b;
    static_for<0, R / 2>([&](auto J) {
      constexpr int j = decltype(J)::value;
      constexpr int sa = b * R + 2 * j, sb = sa + 1;
      constexpr int ra = bitrevc(2 * j, LOGR), rb = bitrevc(2 * j + 1, LOGR);   // rb == ra + R/2
      const float2 xa = load_x(i + ra * T), xb = load_x(i + rb * T);
      const float2 wa = win(std::integral_constant<int, sa>{}), wb = win(std::integral_constant<int, sb>{});
      const float2 pw = mul2(xa, wa);
      v[sa] = fma2(xb, wb, pw);
      v[sb] = fma2(neg2(xb), wb, pw);
    });
  });
}

// Element offset (index minus t) that load_pass0 puts in v[slot], and the slot that receives element
// t + TPF*c — used by the inverse path, whose rebuilt spectrum values are born in registers.
template <class Cfg>
__host__ __device__ constexpr int pass0_offset(int slot) {
  constexpr int R = Cfg::radix(0), LOGR = Cfg::log_radix(0), T = Cfg::M / R;
  return Cfg::TPF * (slot / R) + bitrevc(slot % R, LOGR) * T;   // bitrevc is an involution
}
template <class Cfg>
__host__ __device__ constexpr int pass0_slot_of_pair(int c) {
  for (int s = 0; s < Cfg::PPT; ++s)
    if (pass0_offset<Cfg>(s) == Cfg::TPF * c) return s;
  return -1;
}

// v[] must hold the pass-0 operands (see load_pass0) and receives the spectrum:
//   v[b*RL + q] = Z[t + TPF*b + q*pL]   (RL, pL = radix / sub-length of the last pass, b = 0 .. PPT/RL-1).
// tw: the inter-pass twiddles in shared memory (FftCfg::tw_offset layout: per-thread constants, since thread t of a
// frame group always touches the same elements).
// FUSED0: the first butterfly stage of pass 0 was already done by load_pass0_windowed.
// SPLIT_TW: tw is the split table (FftCfg::tw_offset(s, true)): a pass of tw_split_pass loads 10 factors per thread
// instead of 31 twiddles and forms W^((8a + b) k) = W^(8a k) * W^(b k) right before use (one more float32 rounding).
// pre_store() runs once, right before the first write to xbuf (multi-pass schedules only): callers that share
// the exchange area with something else (the power rows of the previous tile) synchronise there instead of
// before the transform, so that the register-only part of pass 0 overlaps the wait.
struct NoHook { __device__ __forceinline__ void operator()() const {} };
template <class Cfg, bool FUSED0 = false, bool SPLIT_TW = false, class Pre = NoHook>
__device__ __forceinline__ void fft_forward(float2 (&v)[Cfg::PPT], int t, int barrier_id, float2* __restrict__ xbuf,
                                            const float2* __restrict__ tw, Pre&& pre_store = Pre()) {
  constexpr int M = Cfg::M, TPF = Cfg::TPF, PPT = Cfg::PPT;
  static_for<0, Cfg::NPASS>([&](auto S) {
    constexpr int s = decltype(S)::value;
    constexpr int R = Cfg::radix(s);
    constexpr int LOGR = Cfg::log_radix(s);
    constexpr int p = Cfg::sublen(s);
    constexpr int T = M / R;
    constexpr int NB = PPT / R;
    constexpr bool SPLIT = SPLIT_TW && tw_split_pass(Cfg::LOG2M, s, R);
    const float2* tws = tw + Cfg::tw_offset(s, SPLIT_TW);
    // ---- load (+ inter-pass twiddle)
    // Padded addresses: xphys(A + D) == xphys(A) + D + D/32 whenever the low five bits of A and D do not carry.
    // For groups of whole warps every offset below is a multiple of 32, so one run-time base per pass and
    // compile-time displacements replace an OR + shift-add + scale per access (a tenth of the instructions of the
    // n_fft = 4096 kernel, whose t spans two warps and keeps the compiler from folding the padding itself).
    constexpr bool AFFINE_LD = s > 0 && (TPF % 32 == 0) && (T % 32 == 0);
    const float2* ld_base = xbuf + xphys(t);
    static_for<0, NB>([&](auto B) {
      constexpr int b = decltype(B)::value;
      const int i = t + TPF * b;
      const float2* twk = tws + (i & (p - 1));
      float2 wlo[kTwSplitLo];   // SPLIT: wlo[b] = W^(b k), b >= 1
      if constexpr (SPLIT) {
        static_for<1, kTwSplitLo>([&](auto L) {
          constexpr int lo = decltype(L)::value;
          wlo[lo] = twk[(lo - 1) * p];
        });
      }
      static_for<0, R>([&](auto Rr) {
        constexpr int r = decltype(Rr)::value;
        constexpr int slot = b * R + bitrevc(r, LOGR);
        if constexpr (s > 0) {
          float2 x;
          if constexpr (AFFINE_LD) {
            constexpr int D = TPF * b + r * T;
            x = ld_base[D + D / 32];
          } else {
            x = xbuf[xphys(i + r * T)];
          }
          if constexpr (r > 0) {
            constexpr int lo = r % kTwSplitLo, hi = r / kTwSplitLo;
            if constexpr (!SPLIT) {
              x = cmul(x, twk[(r - 1) * p]);
            } else if constexpr (hi == 0) {
              x = cmul(x, wlo[lo]);
            } else if constexpr (lo == 0) {
              x = cmul(x, twk[(kTwSplitLo - 2 + hi) * p]);                     // W^(8a k), a = hi
            } else {
              x = cmul(x, cmul(twk[(kTwSplitLo - 2 + hi) * p], wlo[lo]));
            }
          }
          v[slot] = x;
        }
      });
    });
    // ---- radix-R DFTs in registers
    static_for<0, NB>([&](auto B) { dft_reg<R, decltype(B)::value * R, (FUSED0 && s == 0) ? 1 : 0>(v); });
    // ---- store for the next pass
    if constexpr (s + 1 < Cfg::NPASS) {
      if constexpr (s > 0) group_sync<TPF>(barrier_id);   // everyone finished reading pass s-1 data
      else pre_store();
      // butterfly i = t + TPF*b writes j(b) + q*p with j(b) = (i - k)*R + k, k = i mod p.  When TPF*b is a multiple
      // of p, k does not depend on b and j(b) = j(0) + TPF*b*R: displacement D = TPF*b*R + q*p from j(0).  It is
      // carry-free when j(0) is a multiple of 32 (pass 0: j(0) = 32 t) or D is (later passes: p >= 32).
      constexpr bool AFFINE_ST = (TPF % 32 == 0) && (R == 32 ? true : false) && (p == 1 || p % 32 == 0) && ((TPF * R) % 32 == 0) &&
                                 (p == 1 ? (R % 32 == 0) : true) && (TPF % p == 0 || p == 1);
      if constexpr (AFFINE_ST) {
        const int k0 = t & (p - 1);
        const uint32_t st_base = smem_u32(xbuf + xphys((t - k0) * R + k0));
        static_for<0, NB>([&](auto B) {
          constexpr int b = decltype(B)::value;
          static_for<0, R>([&](auto Q) {
            constexpr int q = decltype(Q)::value;
            constexpr int D = TPF * b * R + q * p;
            sts_c64(st_base + 8u * (D + D / 32), v[b * R + q]);
          });
        });
      } else {
        static_for<0, NB>([&](auto B) {
          constexpr int b = decltype(B)::value;
          const int i = t + TPF * b;
          const int k = i & (p - 1);
          const int j = (i - k) * R + k;
          const uint32_t xbuf_s = smem_u32(xbuf);
          static_for<0, R>([&](auto Q) {
            constexpr int q = decltype(Q)::value;
            sts_c64(xbuf_s + 8u * xphys(j + q * p), v[b * R + q]);
          });
        });
      }
      group_sync<TPF>(barrier_id);
    }
  });
}

// Offset (index minus t) of the spectrum element held in v[slot] after fft_forward, and the inverse map
// for bin pairs: the slot that holds Z[t + TPF*c].  Both are compile-time functions of the schedule.
template <class Cfg>
__host__ __device__ constexpr int spectrum_offset(int slot) {
  constexpr int RL = Cfg::radix(Cfg::NPASS - 1);
  constexpr int pL = Cfg::sublen(Cfg::NPASS - 1);
  return Cfg::TPF * (slot / RL) + (slot % RL) * pL;
}
template <class Cfg>
__host__ __device__ constexpr int slot_of_pair(int c) {
  for (int s = 0; s < Cfg::PPT; ++s)
    if (spectrum_offset<Cfg>(s) == Cfg::TPF * c) return s;
  return -1;
}

// Index of the spectrum element held in v[slot] after fft_forward.
template <class Cfg>
__device__ __forceinline__ int spectrum_index(int t, int slot) {
  constexpr int RL = Cfg::radix(Cfg::NPASS - 1);
  constexpr int pL = Cfg::sublen(Cfg::NPASS - 1);
  int b = slot / RL, q = slot % RL;
  return t + Cfg::TPF * b + q * pL;
}

// One bin pair of the real-input un-mix.  A = Z[k], B = Z[M-k] (Z computed from a window that already
// carries the factor 1/2), w = exp(-2*pi*i*k/N).  Returns X[k] in xa and X[M-k] in xb.
__device__ __forceinline__ void r2c_pair(float2 A, float2 B, float2 w, float2& xa, float2& xb) {
  // E = A + conj(B), O = -i (A - conj(B)), P = w O;  X[k] = E + P, X[M-k] = conj(E - P)
  const float2 cb = make_float2(B.x, -B.y);
  const float2 e = add2(A, cb);
  const float2 o = mulni2(sub2(A, cb));          // (A.y + B.y, B.x - A.x)
  const float2 pp = fma2(muli2(o), bc2(w.y), mul2(o, bc2(w.x)));
  xa = add2(e, pp);
  xb = make_float2(e.x - pp.x, pp.y - e.y);      // conj(E - P): scalar, the sign flip of one half has no packed form
}

// Inverse of r2c_pair: from X[k], X[M-k] rebuild Z[k], Z[M-k] (scaled by 2; caller folds 1/2 into its
// window).  w = exp(-2*pi*i*k/N) as above.
__device__ __forceinline__ void c2r_pair(float2 xa, float2 xb, float2 w, float2& A, float2& B) {
  // E = (Xa + conj(Xb)), P = (Xa - conj(Xb)) = w*O  ->  O = conj(w) * P
  const float2 cb = make_float2(xb.x, -xb.y);
  const float2 e = add2(xa, cb);
  const float2 pq = sub2(xa, cb);                // (xa.x - xb.x, xa.y + xb.y)
  const float2 o = fma2(mulni2(pq), bc2(w.y), mul2(pq, bc2(w.x)));   // conj(w) * P
  // Z[k] = E + i*O ; Z[M-k] = conj(E) + i*conj(O) = conj(E - i*O)
  A = add2(e, muli2(o));
  const float2 d = sub2(e, muli2(o));
  B = make_float2(d.x, -d.y);
}

}  // namespace b2l
