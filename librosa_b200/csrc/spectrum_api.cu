// spectrum_api.cu — C ABI of the plan-bound transforms (include/b2l.h): the forward (stft / spectrogram /
// melspectrogram / mfcc / spectral statistics) and inverse (istft) transforms, their S= pieces (mel and DCT
// projections) and the finite scan of the samples no frame reads.  The only unit that includes aux_kernels.cuh and
// mr_kernel.cuh: they define non-template kernels, whose host stubs a second including unit would define again.
#include <cuda_runtime.h>
#include <math.h>
#include <string.h>

#include <algorithm>

#include "aux_kernels.cuh"
#include "czt_kernel.cuh"
#include "internal.h"
#include "mr_kernel.cuh"

using namespace b2l;

// ------------------------------------------------------------------ per-size kernels (fwd_inst.cu, inv_inst.cu, czt_inst.cu)
#define B2L_CASE(L) case L: return fwd_kernel_##L(variant, mode);
static FwdKernel fwd_kernel_for(int log2m, int variant, int mode) {
  switch (log2m) { B2L_FFT_SIZES(B2L_CASE) }
  return nullptr;
}
#undef B2L_CASE
#define B2L_CASE(L) case L: return inv_kernel_##L(variant);
static InvKernel inv_kernel_for(int log2m, int variant) {
  switch (log2m) { B2L_FFT_SIZES(B2L_CASE) }
  return nullptr;
}
#undef B2L_CASE
#define B2L_CASE(L) case L: return czt_kernel_##L();
static CztKernel czt_kernel_for(int log2p) {
  switch (log2p) { B2L_CZT_SIZES(B2L_CASE) }
  return nullptr;
}
#undef B2L_CASE
#define B2L_CASE(L) case L: return czt_inv_kernel_##L();
static CztInvKernel czt_inv_kernel_for(int log2p) {
  switch (log2p) { B2L_CZT_SIZES(B2L_CASE) }
  return nullptr;
}
#undef B2L_CASE

// CTA variants of the forward and inverse kernels, tried in order (first that fits shared memory wins):
// 116 = 16 warps as two independent 8-warp halves, 16 / 8 = plain CTAs.
static int cta_variants(const HostFftCfg& cfg, int out[3]) {
  int n = 0;
  if (cfg.log2m >= 9 && cfg.log2m <= 11) out[n++] = 116;
  int nws[2];
  const int k = cfg.nw_options(nws);
  for (int i = 0; i < k; ++i) out[n++] = nws[i];
  return n;
}
static int variant_threads(int variant) { return variant == 116 ? 512 : variant * 32; }

// ------------------------------------------------------------------ forward launches
// The checks the forward paths share, in order: plan ownership, clip geometry, signal length, then the device
// pointers of a non-empty batch.  *T: frames per clip, 0 for an empty batch (nothing to launch).
static int frame_count(b2l_ctx* c, const b2l_plan* p, int64_t n_clips, int64_t n, int64_t y_stride, const float* d_y,
                       const void* d_out, long long* T) {
  if (p->ctx != c) return fail(B2L_ERR_INVALID, "plan belongs to another context");
  if (n_clips < 0 || n < 0 || y_stride < n) return fail(B2L_ERR_INVALID, "bad clip geometry");
  if (n > 0x7fffffffLL) return fail(B2L_ERR_UNSUPPORTED, "clips longer than 2^31-1 samples are not supported");
  *T = plan_frames(p, n);
  if (*T <= 0)
    return fail(B2L_ERR_INVALID, "n_fft=%d is too large for input signal of length=%lld", p->n_fft, (long long)n);
  if (n_clips == 0) *T = 0;
  else if (!d_y || !d_out) return fail(B2L_ERR_INVALID, "NULL device pointer");
  return B2L_OK;
}

struct StatsCall { StatsParams sp; const float* d_freq; };

static int run_forward(b2l_ctx* c, const b2l_plan* p, int mode, int log_mode, const float* d_y, int64_t n_clips,
                       int64_t n, int64_t y_stride, float2* out_c, float* out_r, const StatsCall* stats = nullptr) {
  long long T = 0;
  int rc = frame_count(c, p, n_clips, n, y_stride, d_y, mode == MODE_STFT ? (void*)out_c : (void*)out_r, &T);
  if (rc || T == 0) return rc;
  if (mode == MODE_MEL && p->n_mels == 0) return fail(B2L_ERR_INVALID, "plan has no mel stage");
  DeviceGuard g(c->device);

  HostFftCfg cfg(p->log2m);
  const int N = p->n_fft, M = N / 2;
  int variants[3];
  const int n_opt = cta_variants(cfg, variants);
  FwdArgs a;
  memset(&a, 0, sizeof(a));
  int variant = 0, ft = 0, halves = 1;
  size_t smem = 0;
  const b2l_plan::RowTable* rt = nullptr;
  for (int i = 0; i < n_opt && !variant; ++i) {
    const int v = variants[i];
    const int nh = v == 116 ? 2 : 1;
    const int nw = nh > 1 ? 16 : v;
    if (nw * 32 % (cfg.tpf * nh) != 0) continue;
    const int f = nw * 32 / nh / cfg.tpf;
    if (f < 1 || f > 32) continue;
    const long long span = (long long)(f - 1) * p->hop + N;
    if (span > 0x3fffffff) continue;
    const b2l_plan::RowTable* t = nullptr;
    if (mode == MODE_MEL) {
      rc = get_row_table(p, mel_rows_per_warp(f), &t);
      if (rc) return rc;
    }
    size_t off = 0;
    a.off_win = (int)off; off = align_up(off + (size_t)N * 4, 16);
    a.off_tw = (int)off; off = align_up(off + (size_t)cfg.tw_count(true) * 8, 16);
    a.off_bar = (int)off; off = align_up(off + 8 * nh, 16);   // "tile landed" mbarrier per half
    if (t) {
      a.off_melw = (int)off; off = align_up(off + (size_t)t->w_count * 4, 16);
      a.off_melband = (int)off; off = align_up(off + (size_t)t->n_rows * sizeof(MelRow), 16);
    }
    if (mode == MODE_STATS) {   // bin frequencies take the place of the mel weights
      a.off_melw = (int)off; off = align_up(off + (size_t)(M + 1) * 4, 16);
    }
    a.off_in = (int)(off = align_up(off, 128));
    a.in_stride = (int)align_up((size_t)span * 4, 128);
    off += (size_t)a.in_stride * nh;
    a.off_xbuf = (int)(off = align_up(off, 128));
    size_t xbytes = (size_t)f * cfg.xbuf_f2() * 8;
    if (mode == MODE_MEL || mode == MODE_STATS) {
      // the power row of a frame lives in the (padded) exchange region of its group: MelLayout (common.cuh);
      // slack after the last row: a short row of a work item may read up to one band length past bin M + 3
      // (only possible when 2 * GS < 2 * M + 8, i.e. M < 128)
      xbytes = (size_t)f * mel_group_stride(M, f) * 8 + (M < 128 ? (size_t)(M + 16) * 4 : 0);
    }
    a.xbuf_stride = (int)align_up(xbytes, 128);
    off += (size_t)a.xbuf_stride * nh;
    if (off > c->smem_optin) continue;
    variant = v;
    ft = f;
    halves = nh;
    smem = off;
    rt = t;
    a.in_floats = (int)span;
  }
  if (!variant)
    return fail(B2L_ERR_UNSUPPORTED, "hop_length=%d with n_fft=%d needs more shared memory than one SM has", p->hop,
                p->n_fft);

  a.y = d_y;
  a.clip_stride = y_stride;
  a.n = (int)n;
  a.n_clips = (int)n_clips;
  a.n_fft = N;
  a.hop = p->hop;
  a.pad = p->center ? N / 2 : 0;
  a.pad_mode = p->pad_mode;
  a.n_frames = (int)T;
  a.tiles_per_clip = (int)((T + ft - 1) / ft);
  a.total_tiles = (long long)a.tiles_per_clip * n_clips;
  a.tma_ok = (((uintptr_t)d_y & 15) == 0) && (y_stride % 4 == 0) && (a.in_floats % 4 == 0);
  a.window = p->d_win_fwd;
  a.tw = p->d_tw_fwd;
  a.twn = p->d_twn;
  a.out_c = out_c;
  a.out_r = out_r;
  a.power_mode = p->power_mode;
  a.power = p->power;
  a.n_mels = p->n_mels;
  if (mode == MODE_STATS) {
    if (!stats || !stats->d_freq) return fail(B2L_ERR_INVALID, "NULL frequency table");
    a.power_mode = 1;          // the statistics are defined on the magnitude |X|
    a.power = 1.0f;
    a.stats = stats->sp;
    a.mel_w = stats->d_freq;
    a.mel_w_count = M + 1;
  }
  if (rt) {
    a.mel_w_count = rt->w_count;
    a.mel_w = rt->d_w;
    a.mel_rows = rt->d_rows;
    a.n_mel_rows = rt->n_rows;
  }
  a.log_mode = log_mode ? 1 : 0;
  a.out_tiled = log_mode == 2 ? 1 : 0;   // b2l_mfcc: log-mel goes to the tiled scratch
  a.amin = p->amin;
  a.db_sub = 10.0f * log10f(fmaxf(p->amin, fabsf(p->ref_value)));
  a.clip_max = c->d_clip_max;
  a.status = c->d_status;

  const FwdKernel fn = fwd_kernel_for(p->log2m, variant, mode);
  if (!fn) return fail(B2L_ERR_CUDA, "no forward kernel variant %d for n_fft=%d", variant, N);
  const int threads = variant_threads(variant);
  long long grid = 0;
  if ((rc = resident_grid(c, fn, threads, smem, (a.total_tiles + halves - 1) / halves, &grid))) return rc;
  if (!grid) return fail(B2L_ERR_CUDA, "forward kernel does not fit on an SM (smem %zu)", smem);
  return launch(c, fn, (unsigned)grid, threads, smem, a);
}

// ------------------------------------------------------------------ chirp-z launch (n_fft not a power of two)
// Shared memory of czt_kernel / czt_inv_kernel with G frame groups: engine twiddles, exchange buffers, FFT_P(h)/P,
// the window * chirp table (even length) and, forward only, the chirp of the n_fft/2 + 1 output bins.
static size_t czt_smem(const b2l_plan* p, const HostFftCfg& cfg, int G, bool forward) {
  const size_t bins = forward ? (size_t)(1 + p->n_fft / 2) : 0;
  return (size_t)((cfg.tw_count() + 15) & ~15) * 8 + (size_t)G * cfg.xbuf_f2() * 8 +
         ((size_t)(1 << p->log2p) + (size_t)((p->n_fft + 1) & ~1) + bins) * 8;
}

static int run_czt(b2l_ctx* c, const b2l_plan* p, int mode, const float* d_y, int64_t n_clips, int64_t n,
                   int64_t y_stride, float2* out_c, float* out_r) {
  long long T = 0;
  int rc = frame_count(c, p, n_clips, n, y_stride, d_y, mode == 0 ? (void*)out_c : (void*)out_r, &T);
  if (rc || T == 0) return rc;
  DeviceGuard g(c->device);
  HostFftCfg cfg(p->log2p);
  const int nw = cfg.czt_nw();
  const int G = nw * 32 / cfg.tpf;
  CztArgs a;
  memset(&a, 0, sizeof(a));
  a.y = d_y;
  a.clip_stride = y_stride;
  a.n = (int)n;
  a.n_clips = (int)n_clips;
  a.L = p->n_fft;
  a.hop = p->hop;
  a.pad = p->center ? p->n_fft / 2 : 0;
  a.pad_mode = p->pad_mode;
  a.n_frames = (int)T;
  a.n_bins = 1 + p->n_fft / 2;
  a.wb = p->d_czt_wb;
  a.bk = p->d_czt_bk;
  a.hf = p->d_czt_hf;
  a.out_c = out_c;
  a.out_r = out_r;
  a.mode = mode;
  a.power_mode = p->power_mode;
  a.power = p->power;
  a.status = c->d_status;
  const size_t smem = czt_smem(p, cfg, G, true);
  const CztKernel fn = czt_kernel_for(p->log2p);
  // the table part of the shared memory depends on n_fft, not only on P: size the grid for the largest case (the
  // kernels run one block per SM anyway)
  const long long steps = ((long long)n_clips * ((T + 1) / 2) + G - 1) / G;   // frames go in pairs inside a clip
  long long grid = 0;
  if ((rc = resident_grid(c, fn, nw * 32, c->smem_optin / 2 + 1, steps, &grid))) return rc;
  if (smem > c->smem_optin) return fail(B2L_ERR_UNSUPPORTED, "n_fft=%d needs more shared memory than one SM has", p->n_fft);
  if (!grid) return fail(B2L_ERR_CUDA, "chirp-z kernel does not fit on an SM (smem %zu)", smem);
  return launch(c, fn, (unsigned)grid, nw * 32, smem, a);
}

// ------------------------------------------------------------------ mixed-radix launch (even n_fft, 5-smooth half)
// Warps per block (*nw) and shared memory (*smem) of mr_kernel / mr_inv_kernel: the tables (with n_mels mel rows of
// mel_w_count weights) plus two M-point buffers per frame, fpw frames per warp.  Two resident blocks per SM when
// they fit: at most half of the SM's shared memory each.
static int mr_block(const b2l_ctx* c, const b2l_plan* p, int n_mels, int mel_w_count, int fpw, int* nw, size_t* smem) {
  const size_t tables = mr_table_bytes(p->n_fft, p->mr_tw_count, n_mels, mel_w_count);
  const size_t per_warp = (size_t)2 * (p->n_fft / 2) * sizeof(float2) * (size_t)fpw;
  const size_t budget = (c->smem_optin + 1024) / 2 - 1024;
  int w = 16;
  while (w > 1 && tables + w * per_warp > budget) --w;
  if (tables + w * per_warp > c->smem_optin)
    return fail(B2L_ERR_UNSUPPORTED, "n_fft=%d needs more shared memory than one SM has", p->n_fft);
  *nw = w;
  *smem = tables + w * per_warp;
  return B2L_OK;
}

// mode 0: complex STFT, 1: |X|^power, 2: mel (log_mode 1: dB values + per-clip maximum for mfcc)
static int run_mr(b2l_ctx* c, const b2l_plan* p, int mode, int log_mode, const float* d_y, int64_t n_clips, int64_t n,
                  int64_t y_stride, float2* out_c, float* out_r) {
  long long T = 0;
  int rc = frame_count(c, p, n_clips, n, y_stride, d_y, mode == 0 ? (void*)out_c : (void*)out_r, &T);
  if (rc || T == 0) return rc;
  if (mode == 2 && p->n_mels == 0) return fail(B2L_ERR_INVALID, "plan has no mel stage");
  if (n_clips > 0x7fffffffLL || T > 0x7fffffffLL) return fail(B2L_ERR_UNSUPPORTED, "batch too large");
  DeviceGuard g(c->device);
  MrArgs a;
  memset(&a, 0, sizeof(a));
  a.y = d_y;
  a.clip_stride = y_stride;
  a.n = (int)n;
  a.n_clips = (int)n_clips;
  a.L = p->n_fft;
  a.M = p->n_fft / 2;
  a.hop = p->hop;
  a.pad = p->center ? p->n_fft / 2 : 0;
  a.pad_mode = p->pad_mode;
  a.n_frames = (int)T;
  a.n_bins = 1 + p->n_fft / 2;
  a.n_pass = p->mr_n_pass;
  for (int s = 0; s < p->mr_n_pass; ++s) {
    a.radix[s] = p->mr_radix[s];
    a.tw_off[s] = p->mr_tw_off[s];
  }
  a.tw_count = p->mr_tw_count;
  a.win = p->d_mr_win;
  a.tw = p->d_mr_tw;
  a.twn = p->d_mr_twn;
  a.out_c = out_c;
  a.out_r = out_r;
  a.mode = mode;
  a.power_mode = p->power_mode;
  a.power = p->power;
  a.status = c->d_status;
  if (mode == 2) {
    a.band = p->d_band;
    a.mel_w = p->d_mel_w;
    a.n_mels = p->n_mels;
    a.mel_w_count = p->mel_w_count;
    a.log_mode = log_mode ? 1 : 0;
    a.amin = p->amin;
    a.db_sub = 10.0f * log10f(fmaxf(p->amin, fabsf(p->ref_value)));
    a.clip_max = c->d_clip_max;
  }
  // frames per warp: short frames ride two to a warp (their butterfly rounds fill 16 lanes better than 32)
  const int fpw = a.M <= 512 ? 2 : 1;
  int nw = 0;
  size_t smem = 0;
  if ((rc = mr_block(c, p, a.n_mels, a.mel_w_count, fpw, &nw, &smem))) return rc;
  auto kern = fpw == 2 ? (mode == 0 ? mr_kernel<0, 16> : (mode == 1 ? mr_kernel<1, 16> : mr_kernel<2, 16>))
                       : (mode == 0 ? mr_kernel<0, 32> : (mode == 1 ? mr_kernel<1, 32> : mr_kernel<2, 32>));
  const long long total = (long long)n_clips * T;
  long long grid = 0;
  if ((rc = resident_grid(c, kern, nw * 32, smem, (total + (long long)nw * fpw - 1) / ((long long)nw * fpw), &grid)))
    return rc;
  if (!grid) return fail(B2L_ERR_CUDA, "mixed-radix kernel does not fit on an SM (smem %zu)", smem);
  return launch(c, kern, (unsigned)grid, nw * 32, smem, a);
}

extern "C" int b2l_stft(b2l_ctx* c, const b2l_plan* p, const float* d_y, int64_t n_clips, int64_t n, int64_t y_stride,
                        void* d_D) {
  if (!c || !p) return fail(B2L_ERR_INVALID, "NULL ctx / plan");
  switch (p->path) {
    case PATH_MR: return run_mr(c, p, 0, 0, d_y, n_clips, n, y_stride, (float2*)d_D, nullptr);
    case PATH_CZT: return run_czt(c, p, 0, d_y, n_clips, n, y_stride, (float2*)d_D, nullptr);
    default: return run_forward(c, p, MODE_STFT, 0, d_y, n_clips, n, y_stride, (float2*)d_D, nullptr);
  }
}
extern "C" int b2l_spectrogram(b2l_ctx* c, const b2l_plan* p, const float* d_y, int64_t n_clips, int64_t n,
                               int64_t y_stride, float* d_S) {
  if (!c || !p) return fail(B2L_ERR_INVALID, "NULL ctx / plan");
  switch (p->path) {
    case PATH_MR: return run_mr(c, p, 1, 0, d_y, n_clips, n, y_stride, nullptr, d_S);
    case PATH_CZT: return run_czt(c, p, 1, d_y, n_clips, n, y_stride, nullptr, d_S);
    default: return run_forward(c, p, MODE_SPEC, 0, d_y, n_clips, n, y_stride, nullptr, d_S);
  }
}

// ------------------------------------------------------------------ device-side input validation
template <typename T, typename Kernel>
static int scan_finite(b2l_ctx* c, Kernel kernel, const T* d_y, int64_t n_clips, int64_t n, int64_t y_stride,
                       int64_t begin) {
  if (!c || !d_y) return fail(B2L_ERR_INVALID, "NULL argument");
  if (n_clips <= 0 || begin >= n) return B2L_OK;
  if (n > 0x7fffffffLL) return fail(B2L_ERR_UNSUPPORTED, "scan_finite: clips longer than 2^31-1 samples");
  DeviceGuard g(c->device);
  long long bx = ((n - begin) + 1023) / 1024;
  if (bx > 64) bx = 64;
  const dim3 grid((unsigned)bx, (unsigned)std::min(n_clips, kMaxGridY));
  return launch(c, kernel, grid, 256, 0, d_y, y_stride, (int)n, (int)(begin < 0 ? 0 : begin), n_clips, c->d_status);
}
extern "C" int b2l_scan_finite(b2l_ctx* c, const float* d_y, int64_t n_clips, int64_t n, int64_t y_stride,
                               int64_t begin) {
  return scan_finite(c, finite_scan_kernel, d_y, n_clips, n, y_stride, begin);
}
extern "C" int b2l_scan_finite_f64(b2l_ctx* c, const double* d_y, int64_t n_clips, int64_t n, int64_t y_stride,
                                   int64_t begin) {
  return scan_finite(c, finite_scan64_kernel, d_y, n_clips, n, y_stride, begin);
}
// ------------------------------------------------------------------ frame-wise spectral statistics
extern "C" int b2l_spectral_stats(b2l_ctx* c, const b2l_plan* p, const b2l_stats_desc* d, const float* d_y,
                                  int64_t n_clips, int64_t n, int64_t y_stride, const float* d_freq, float* d_out) {
  if (!c || !p) return fail(B2L_ERR_INVALID, "NULL ctx / plan");
  if (p->path != PATH_POW2)
    return fail(B2L_ERR_UNSUPPORTED,
                "n_fft=%d: compose b2l_spectrogram + b2l_spectral_stats_from_spec for non-power-of-two sizes", p->n_fft);
  StatsCall sc;
  int rc = check_stats_desc(d, &sc.sp);
  if (rc) return rc;
  sc.d_freq = d_freq;
  return run_forward(c, p, MODE_STATS, 0, d_y, n_clips, n, y_stride, nullptr, d_out, &sc);
}

extern "C" int b2l_melspectrogram(b2l_ctx* c, const b2l_plan* p, const float* d_y, int64_t n_clips, int64_t n,
                                  int64_t y_stride, float* d_mel) {
  if (!c || !p) return fail(B2L_ERR_INVALID, "NULL ctx / plan");
  switch (p->path) {
    case PATH_MR: return run_mr(c, p, 2, 0, d_y, n_clips, n, y_stride, nullptr, d_mel);
    case PATH_CZT:
      return fail(B2L_ERR_UNSUPPORTED, "n_fft=%d: compose b2l_spectrogram + b2l_mel_project for non-power-of-two sizes",
                  p->n_fft);
    default: return run_forward(c, p, MODE_MEL, 0, d_y, n_clips, n, y_stride, nullptr, d_mel);
  }
}

static int launch_dct(b2l_ctx* c, const b2l_plan* p, const float* d_L, int64_t n_clips, int64_t T, int clamp,
                      float* d_out, int tiled = 0) {
  const int KG = (p->n_mfcc + 7) / 8;
  if (KG > 16) return fail(B2L_ERR_UNSUPPORTED, "n_mfcc=%d > 128 is not supported", p->n_mfcc);
  // DCT rows plus one tile buffer of two 64-frame blocks (dct_clamp4_kernel)
  const size_t smem = ((size_t)p->n_mels * 8 * KG + 2 * (size_t)p->n_mels * 64) * 4;
  if (smem > c->smem_optin) {
    // too many input rows for the shared-memory tile (e.g. mfcc(S=...) of a 1025-bin spectrogram): generic kernel
    if (tiled) return fail(B2L_ERR_UNSUPPORTED, "n_mels=%d is too large for the fused mfcc path", p->n_mels);
    if (n_clips > kMaxGridY) return fail(B2L_ERR_UNSUPPORTED, "dct: more than 65535 leading indices");
    return launch(c, dct_generic_kernel, dim3((unsigned)((T + 127) / 128), (unsigned)n_clips), 128, 0, d_L, p->d_dct,
                  clamp ? c->d_clip_max : nullptr, clamp ? p->top_db : -1.0f, p->n_mels, p->n_mfcc, 8 * KG, (int)T, d_out);
  }
  // two warp sets over the mel rows when the partial sums fit in the tile buffer
  const int ks = KG <= 10 && p->n_mels >= 8 * KG ? 2 : 1;   // 640 threads at most; 32*KG*32 partial sums <= 2*n_mels*64 tile words
  auto kern = ks == 2 ? dct_clamp4_kernel<2> : dct_clamp4_kernel<1>;
  const int threads = KG * 32 * ks;
  const int tiles = (int)((T + DCT4_TILE - 1) / DCT4_TILE);
  const long long total = (long long)tiles * n_clips;
  long long grid = 0;
  if (int rc = resident_grid(c, kern, threads, smem, total, &grid)) return rc;
  if (!grid) return fail(B2L_ERR_CUDA, "DCT kernel does not fit on an SM");
  return launch(c, kern, (unsigned)grid, threads, smem, d_L, p->d_dct, clamp ? c->d_clip_max : nullptr,
                clamp ? p->top_db : -1.0f, p->n_mels, p->n_mfcc, (int)T, tiles, total, tiled, d_out);
}

extern "C" int b2l_mfcc(b2l_ctx* c, const b2l_plan* p, const float* d_y, int64_t n_clips, int64_t n, int64_t y_stride,
                        float* d_mfcc, float* d_logmel) {
  if (!c || !p) return fail(B2L_ERR_INVALID, "NULL ctx / plan");
  if (p->n_mfcc == 0) return fail(B2L_ERR_INVALID, "plan has no mfcc stage");
  if (p->path == PATH_CZT)
    return fail(B2L_ERR_UNSUPPORTED, "n_fft=%d: compose spectrogram, mel_project, power_to_db and dct_project for "
                "non-power-of-two sizes", p->n_fft);
  if (n_clips <= 0) return n_clips == 0 ? B2L_OK : fail(B2L_ERR_INVALID, "negative n_clips");
  DeviceGuard g(c->device);
  const long long T = plan_frames(p, n);
  if (T <= 0) return fail(B2L_ERR_INVALID, "n_fft=%d is too large for input signal of length=%lld", p->n_fft, (long long)n);
  int rc = ensure_clip_max(c, (size_t)n_clips);
  if (rc) return rc;
  CUDA_TRY(cudaMemsetAsync(c->d_clip_max, 0, (size_t)n_clips * sizeof(unsigned int), c->stream));
  Temp own(c->stream);
  float* scratch = d_logmel;
  // the log-mel scratch is tiled: [clip][ceil(T/64)][n_mels][64] (see dct_clamp4_kernel)
  if (!scratch) {
    CUDA_TRY(own.alloc((size_t)n_clips * p->n_mels * ((T + 63) / 64 * 64) * sizeof(float)));
    scratch = (float*)own.p;
  }
  // mixed-radix frames (mr_kernel): the dB rows go to the scratch in the plain [clip][mel][frame] layout
  const int tiled = p->path == PATH_POW2 ? 1 : 0;
  rc = p->path == PATH_MR ? run_mr(c, p, 2, 1, d_y, n_clips, n, y_stride, nullptr, scratch)
                       : run_forward(c, p, MODE_MEL, 2, d_y, n_clips, n, y_stride, nullptr, scratch);
  return rc ? rc : launch_dct(c, p, scratch, n_clips, T, 1, d_mfcc, tiled);
}

// ------------------------------------------------------------------ inverse launches
// n_fft a power of two: inv_kernel (irFFT, window and overlap-add in one pass)
static int run_inverse(b2l_ctx* c, const b2l_plan* p, const void* d_D, int64_t n_clips, int64_t n_frames_stored,
                       int64_t n_frames_used, const float* d_inv_wss, int64_t out_len, float* d_y, int64_t y_stride) {
  if (out_len > 0x7fffffffLL || n_frames_stored > 0x7fffffffLL)
    return fail(B2L_ERR_UNSUPPORTED, "istft output longer than 2^31-1 samples is not supported");
  DeviceGuard g(c->device);
  HostFftCfg cfg(p->log2m);
  const int N = p->n_fft, M = N / 2;
  int variants[3];
  const int n_opt = cta_variants(cfg, variants);
  InvArgs a;
  memset(&a, 0, sizeof(a));
  int variant = 0, G = 0, halves = 1;
  size_t smem = 0;
  const int clen = N > p->hop ? N - p->hop : 0;
  for (int i = 0; i < n_opt && !variant; ++i) {
    const int v = variants[i];
    const bool dual = v == 116;
    const int nw = dual ? 16 : v;
    const int nh = dual ? 2 : 1;
    if (nw * 32 % (cfg.tpf * nh) != 0) continue;
    const int gg = nw * 32 / nh / cfg.tpf;
    if (gg < 1) continue;
    size_t off = 0;
    a.off_win = (int)off; off = align_up(off + (size_t)N * 4, 16);
    a.off_tw = (int)off; off = align_up(off + (size_t)cfg.tw_count() * 8, 16);
    a.off_acc = (int)off;
    a.acc_stride = (int)align_up((size_t)2 * clen * 4, 16);
    off += (size_t)a.acc_stride * nh;
    a.off_xbuf = (int)(off = align_up(off, 128));
    a.xbuf_stride = (int)align_up((size_t)gg * cfg.xbuf_f2() * 8, 128);
    off += (size_t)a.xbuf_stride * nh;
    if (off > c->smem_optin) continue;
    variant = v;
    G = gg;
    halves = nh;
    smem = off;
  }
  if (!variant) return fail(B2L_ERR_UNSUPPORTED, "istft configuration does not fit in shared memory");
  a.acc_floats = 2 * clen;
  a.D = (const float2*)d_D;
  a.d_clip_stride = (long long)n_frames_stored * (M + 1);
  a.n_clips = (int)n_clips;
  a.n_frames = (int)n_frames_used;
  a.n_fft = N;
  a.hop = p->hop;
  a.start = p->center ? N / 2 : 0;
  a.out_len = (int)out_len;
  a.y_clip_stride = y_stride;
  a.y = d_y;
  a.window = p->d_win_inv;
  a.inv_wss = d_inv_wss;
  a.tw = p->d_tw;
  a.twn = p->d_twn;
  a.vec4 = (p->hop % 4 == 0) && (clen % 4 == 0) && (a.start % 4 == 0) && (y_stride % 4 == 0) &&
           (cfg.xbuf_f2() % 2 == 0) &&   // frame buffers 16-byte aligned inside the exchange area
           (((uintptr_t)d_y & 15) == 0) && (((uintptr_t)d_inv_wss & 15) == 0);
  // one slot of consecutive (clip, frame) pairs per resident half-CTA (1 CTA per SM): equal work everywhere,
  // no partial last wave; slots are whole rounds of G frames, and at least 4 rounds long so that the halo
  // frames recomputed at the start of a slot stay a small fraction
  const long long total_frames = (long long)n_clips * n_frames_used;
  long long fps = (total_frames + (long long)c->sm_count * halves - 1) / ((long long)c->sm_count * halves);
  if (fps < 4LL * G) fps = 4LL * G;
  fps = (fps + G - 1) / G * G;
  if (fps > 0x7fffffffLL) return fail(B2L_ERR_UNSUPPORTED, "istft batch too large");
  a.frames_per_slot = (int)fps;
  const long long items = (total_frames + fps - 1) / fps;
  const long long grid = (items + halves - 1) / halves;
  const InvKernel fn = inv_kernel_for(p->log2m, variant);
  if (!fn) return fail(B2L_ERR_CUDA, "no inverse kernel variant %d for n_fft=%d", variant, N);
  const int threads = variant_threads(variant);
  int rc = blocks_per_sm(c, fn, threads, smem, nullptr);
  return rc ? rc : launch(c, fn, (unsigned)grid, threads, smem, a);
}

// mixed-radix inverse frames (mr_inv_kernel) into the scratch array
static int run_mr_inverse(b2l_ctx* c, const b2l_plan* p, const void* d_D, int64_t n_clips, int64_t n_frames_stored,
                          int64_t n_frames_used) {
  const int L = p->n_fft;
  MrInvArgs a;
  memset(&a, 0, sizeof(a));
  a.D = (const float2*)d_D;
  a.d_clip_stride = (long long)n_frames_stored * (L / 2 + 1);
  a.n_clips = (int)n_clips;
  a.n_frames = (int)n_frames_used;
  a.L = L;
  a.M = L / 2;
  a.n_bins = L / 2 + 1;
  a.n_pass = p->mr_n_pass;
  for (int s = 0; s < p->mr_n_pass; ++s) {
    a.radix[s] = p->mr_radix[s];
    a.tw_off[s] = p->mr_tw_off[s];
  }
  a.tw_count = p->mr_tw_count;
  a.win = p->d_mr_win_inv;
  a.tw = p->d_mr_tw;
  a.twn = p->d_mr_twn;
  a.ytmp = c->d_scratch;
  int nw = 0;
  size_t smem = 0;
  long long grid = 0;
  const long long total = (long long)n_clips * n_frames_used;
  int rc = mr_block(c, p, 0, 0, 1, &nw, &smem);
  if (rc || (rc = resident_grid(c, mr_inv_kernel, nw * 32, smem, (total + nw - 1) / nw, &grid))) return rc;
  if (!grid) return fail(B2L_ERR_CUDA, "mixed-radix inverse kernel does not fit on an SM (smem %zu)", smem);
  return launch(c, mr_inv_kernel, (unsigned)grid, nw * 32, smem, a);
}

// chirp-z inverse frames (czt_inv_kernel) into the scratch array
static int run_czt_inverse(b2l_ctx* c, const b2l_plan* p, const void* d_D, int64_t n_clips, int64_t n_frames_stored,
                           int64_t n_frames_used) {
  const int L = p->n_fft;
  HostFftCfg cfg(p->log2p);
  const int nw = cfg.czt_nw();
  const int G = nw * 32 / cfg.tpf;
  CztInvArgs a;
  memset(&a, 0, sizeof(a));
  a.D = (const float2*)d_D;
  a.d_clip_stride = (long long)n_frames_stored * (L / 2 + 1);
  a.n_clips = (int)n_clips;
  a.n_frames = (int)n_frames_used;
  a.L = L;
  a.n_bins = L / 2 + 1;
  a.bfull = p->d_czt_bfull;
  a.wbi = p->d_czt_wbi;
  a.hf = p->d_czt_hf;
  a.ytmp = c->d_scratch;
  const size_t smem = czt_smem(p, cfg, G, false);
  if (smem > c->smem_optin) return fail(B2L_ERR_UNSUPPORTED, "n_fft=%d needs more shared memory than one SM has", L);
  const CztInvKernel fn = czt_inv_kernel_for(p->log2p);
  const long long steps = ((long long)n_clips * ((n_frames_used + 1) / 2) + G - 1) / G;   // frames go in pairs inside a clip
  long long grid = 0;
  // sized like the forward (run_czt)
  if (int rc = resident_grid(c, fn, nw * 32, c->smem_optin / 2 + 1, steps, &grid)) return rc;
  if (!grid) return fail(B2L_ERR_CUDA, "chirp-z inverse kernel does not fit on an SM");
  return launch(c, fn, (unsigned)grid, nw * 32, smem, a);
}

extern "C" int b2l_istft(b2l_ctx* c, const b2l_plan* p, const void* d_D, int64_t n_clips, int64_t n_frames_stored,
                         int64_t n_frames_used, const float* d_inv_wss, int64_t out_len, float* d_y,
                         int64_t y_stride) {
  if (!c || !p) return fail(B2L_ERR_INVALID, "NULL ctx / plan");
  if (p->ctx != c) return fail(B2L_ERR_INVALID, "plan belongs to another context");
  if (n_clips < 0 || n_frames_used < 1 || n_frames_used > n_frames_stored || out_len < 0 || y_stride < out_len)
    return fail(B2L_ERR_INVALID, "bad istft geometry");
  if (n_clips == 0 || out_len == 0) return B2L_OK;
  if (!d_D || !d_inv_wss || !d_y) return fail(B2L_ERR_INVALID, "NULL device pointer");
  if (p->path == PATH_POW2)
    return run_inverse(c, p, d_D, n_clips, n_frames_stored, n_frames_used, d_inv_wss, out_len, d_y, y_stride);
  // mixed-radix or chirp-z frames into the scratch array, then a gather overlap-add
  if (out_len > 0x7fffffffLL || n_clips > kMaxGridY) return fail(B2L_ERR_UNSUPPORTED, "istft batch too large");
  DeviceGuard g(c->device);
  const int L = p->n_fft;
  int rc = ensure_scratch(c, (size_t)n_clips * (size_t)n_frames_used * L * sizeof(float));
  if (rc == B2L_OK)
    rc = p->path == PATH_MR ? run_mr_inverse(c, p, d_D, n_clips, n_frames_stored, n_frames_used)
                         : run_czt_inverse(c, p, d_D, n_clips, n_frames_stored, n_frames_used);
  if (rc) return rc;
  const dim3 og((unsigned)row_blocks(out_len, 256, 8LL * c->sm_count, n_clips), (unsigned)n_clips);
  return launch(c, ola_kernel, og, 256, 0, c->d_scratch, (int)n_frames_used, L, p->hop, p->center ? L / 2 : 0,
                (int)out_len, y_stride, d_inv_wss, d_y);
}

// ------------------------------------------------------------------ S= pieces
extern "C" int b2l_mel_project(b2l_ctx* c, const b2l_plan* p, const float* d_S, int64_t n_clips, int64_t n_frames,
                               float* d_mel) {
  if (!c || !p || !d_S || !d_mel) return fail(B2L_ERR_INVALID, "NULL argument");
  if (p->n_mels == 0) return fail(B2L_ERR_INVALID, "plan has no mel stage");
  if (n_clips <= 0 || n_frames <= 0) return B2L_OK;
  DeviceGuard g(c->device);
  const int F = p->n_fft / 2 + 1;
  {
    // a few rows whose bands cover most of the spectrum (chroma): dense_project_kernel
    const size_t dsmem = ((((size_t)F * 33 + 3) & ~(size_t)3) + (size_t)F * 16 + 8 * 16 * 32) * 4;
    if (p->d_mel_wT && (long long)p->mel_w_count * 4 >= (long long)p->n_mels * F && dsmem <= c->smem_optin) {
      const int r4 = (p->n_mels + 3) / 4;
      auto kern = r4 == 1 ? dense_project_kernel<1> : r4 == 2 ? dense_project_kernel<2> : r4 == 3 ? dense_project_kernel<3> : dense_project_kernel<4>;
      const int rc = blocks_per_sm(c, kern, 256, dsmem, nullptr);
      if (rc) return rc;
      const int tiles_d = (int)((n_frames + 31) / 32);
      const long long total = (long long)tiles_d * n_clips;
      long long grid_d = c->sm_count;
      if (grid_d > total) grid_d = total;
      return launch(c, kern, (unsigned)grid_d, 256, dsmem, d_S, p->d_mel_wT, p->n_mels, F, (int)n_frames, tiles_d, total,
                    d_mel);
    }
  }
  size_t smem = (size_t)F * 33 * 4;
  if (smem > c->smem_optin) return fail(B2L_ERR_UNSUPPORTED, "n_fft too large for mel_project");
  const int rc = blocks_per_sm(c, mel_project_kernel, 256, smem, nullptr);
  if (rc) return rc;
  const int tiles = (int)((n_frames + 31) / 32);
  const long long grid = (long long)tiles * n_clips;
  if (grid > 0x7fffffffLL) return fail(B2L_ERR_UNSUPPORTED, "too many tiles");
  return launch(c, mel_project_kernel, (unsigned)grid, 256, smem, d_S, p->d_mel_w, p->d_band, p->n_mels, F, (int)n_frames,
                tiles, d_mel);
}

extern "C" int b2l_dct_project(b2l_ctx* c, const b2l_plan* p, const float* d_S, int64_t n_clips, int64_t n_frames,
                               float* d_mfcc) {
  if (!c || !p || !d_S || !d_mfcc) return fail(B2L_ERR_INVALID, "NULL argument");
  if (p->n_mfcc == 0) return fail(B2L_ERR_INVALID, "plan has no mfcc stage");
  if (n_clips <= 0 || n_frames <= 0) return B2L_OK;
  DeviceGuard g(c->device);
  return launch_dct(c, p, d_S, n_clips, n_frames, 0, d_mfcc);
}
