// api.cu — C ABI of libb2l.so (see include/b2l.h): every entry point that launches a kernel — the forward
// (stft / spectrogram / melspectrogram / mfcc / spectral statistics) and inverse (istft) transforms and the
// feature kernels and the pitch trackers.  The only unit that includes aux_kernels.cuh, mr_kernel.cuh,
// feat_kernels.cuh and pitch_kernels.cuh: they define non-template kernels, whose host stubs a second including
// unit would define again.
#include <cuda_runtime.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>

#include "aux_kernels.cuh"
#include "czt_kernel.cuh"
#include "feat_kernels.cuh"
#include "internal.h"
#include "mr_kernel.cuh"
#include "pitch_kernels.cuh"

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

// ------------------------------------------------------------------ which kernels serve a plan
enum Path { PATH_POW2, PATH_MR, PATH_CZT, PATH_NONE };
enum Entry {
  ENTRY_SPECTRUM,   // stft, spectrogram, istft
  ENTRY_MEL,        // melspectrogram, mfcc
  ENTRY_STATS,      // spectral_stats
};
// B2L_MR=0 sends the spectrum entry points of the mixed-radix sizes back to the chirp-z kernels where those exist
// (n_fft <= 2047).  Read on every call: a plan outlives changes of the environment.
static bool mr_enabled(const b2l_plan* p) {
  if (p->log2p == 0) return true;   // no chirp-z tables for this size
  const char* e = getenv("B2L_MR");
  return !(e && *e) || atoi(e) != 0;
}
static Path route(const b2l_plan* p, Entry entry) {
  if (!p->czt) return PATH_POW2;
  switch (entry) {
    case ENTRY_SPECTRUM: return p->mr && mr_enabled(p) ? PATH_MR : PATH_CZT;
    case ENTRY_MEL: return p->mr ? PATH_MR : PATH_NONE;   // B2L_MR does not apply here
    default: return PATH_NONE;
  }
}

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
  switch (route(p, ENTRY_SPECTRUM)) {
    case PATH_MR: return run_mr(c, p, 0, 0, d_y, n_clips, n, y_stride, (float2*)d_D, nullptr);
    case PATH_CZT: return run_czt(c, p, 0, d_y, n_clips, n, y_stride, (float2*)d_D, nullptr);
    default: return run_forward(c, p, MODE_STFT, 0, d_y, n_clips, n, y_stride, (float2*)d_D, nullptr);
  }
}
extern "C" int b2l_spectrogram(b2l_ctx* c, const b2l_plan* p, const float* d_y, int64_t n_clips, int64_t n,
                               int64_t y_stride, float* d_S) {
  if (!c || !p) return fail(B2L_ERR_INVALID, "NULL ctx / plan");
  switch (route(p, ENTRY_SPECTRUM)) {
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
// ------------------------------------------------------------------ frame-wise spectral statistics / framings
static int check_stats_desc(const b2l_stats_desc* d, StatsParams* sp) {
  if (!d) return fail(B2L_ERR_INVALID, "NULL stats descriptor");
  if (!(d->roll_percent > 0.0f && d->roll_percent < 1.0f))
    return fail(B2L_ERR_INVALID, "roll_percent must lie in the range (0, 1)");
  if (!(d->flat_amin > 0.0f)) return fail(B2L_ERR_INVALID, "amin must be strictly positive");
  if (!(d->bw_p > 0.0f)) return fail(B2L_ERR_INVALID, "p must be strictly positive");
  if (d->frame_length < 1) return fail(B2L_ERR_INVALID, "frame_length must be positive");
  sp->roll_percent = d->roll_percent;
  sp->flat_amin = d->flat_amin;
  sp->flat_power = d->flat_power;
  sp->bw_p = d->bw_p;
  sp->bw_norm = d->bw_norm ? 1 : 0;
  sp->frame_length = d->frame_length;
  sp->want = d->want ? (d->want & ((1 << N_STATS) - 1)) : (1 << N_STATS) - 1;
  return B2L_OK;
}

extern "C" int b2l_spectral_stats_from_spec(b2l_ctx* c, const b2l_stats_desc* d, const float* d_S, int64_t n_clips,
                                            int64_t n_frames, int32_t n_bins, const float* d_freq, float* d_out) {
  if (!c || !d_S || !d_freq || !d_out) return fail(B2L_ERR_INVALID, "NULL argument");
  StatsCall sc;
  int rc = check_stats_desc(d, &sc.sp);
  if (rc) return rc;
  if (n_bins < 2) return fail(B2L_ERR_INVALID, "a spectrum needs at least two bins");
  if (n_clips <= 0 || n_frames <= 0) return B2L_OK;
  if (n_frames > 0x7fffffffLL) return fail(B2L_ERR_UNSUPPORTED, "too many frames");
  DeviceGuard g(c->device);
  const int Fp = (n_bins + 3) & ~3;
  int nw = 8;
  while (nw > 1 && (size_t)(nw + 1) * Fp * 4 > c->smem_optin) nw >>= 1;
  const size_t smem = (size_t)(nw + 1) * Fp * 4;
  if (smem > c->smem_optin) return fail(B2L_ERR_UNSUPPORTED, "n_bins=%d rows do not fit in shared memory", n_bins);
  rc = blocks_per_sm(c, stats_kernel, nw * 32, smem, nullptr);
  if (rc) return rc;
  const long long rows = (long long)n_clips * n_frames;
  const long long grid = grid_stride_blocks(rows, nw, 8LL * c->sm_count);
  return launch(c, stats_kernel, (unsigned)grid, nw * 32, smem, d_S, rows, (int)n_frames, n_bins, d_freq, sc.sp, d_out,
                c->d_status);
}

extern "C" int b2l_spectral_stats(b2l_ctx* c, const b2l_plan* p, const b2l_stats_desc* d, const float* d_y,
                                  int64_t n_clips, int64_t n, int64_t y_stride, const float* d_freq, float* d_out) {
  if (!c || !p) return fail(B2L_ERR_INVALID, "NULL ctx / plan");
  if (route(p, ENTRY_STATS) == PATH_NONE)
    return fail(B2L_ERR_UNSUPPORTED,
                "n_fft=%d: compose b2l_spectrogram + b2l_spectral_stats_from_spec for non-power-of-two sizes", p->n_fft);
  StatsCall sc;
  int rc = check_stats_desc(d, &sc.sp);
  if (rc) return rc;
  sc.d_freq = d_freq;
  return run_forward(c, p, MODE_STATS, 0, d_y, n_clips, n, y_stride, nullptr, d_out, &sc);
}

extern "C" int b2l_frame_feature(b2l_ctx* c, int32_t what, const float* d_y, int64_t n_clips, int64_t n,
                                 int64_t y_stride, int32_t frame_length, int32_t hop_length, int32_t center,
                                 int32_t pad_mode, float threshold, int32_t zero_pos, int32_t pad_first, float out_scale,
                                 float* d_out) {
  if (!c) return fail(B2L_ERR_INVALID, "NULL ctx");
  if (what != B2L_FRAME_RMS && what != B2L_FRAME_ZERO_CROSSINGS) return fail(B2L_ERR_INVALID, "bad feature id %d", what);
  if (frame_length < 1) return fail(B2L_ERR_INVALID, "frame_length=%d must be positive", frame_length);
  if (hop_length < 1) return fail(B2L_ERR_INVALID, "hop_length=%d must be a positive integer", hop_length);
  if (pad_mode < 0 || pad_mode > B2L_PAD_EMPTY) return fail(B2L_ERR_INVALID, "bad pad_mode %d", pad_mode);
  if (n_clips < 0 || n < 0 || y_stride < n) return fail(B2L_ERR_INVALID, "bad clip geometry");
  if (n > 0x7fffffffLL) return fail(B2L_ERR_UNSUPPORTED, "clips longer than 2^31-1 samples are not supported");
  const int pad = center ? frame_length / 2 : 0;
  const long long padded = n + 2LL * pad;
  if (padded < frame_length)
    return fail(B2L_ERR_INVALID, "Input is too short (n=%lld) for frame_length=%d", (long long)padded, frame_length);
  const long long T = 1 + (padded - frame_length) / hop_length;
  if (n_clips == 0) return B2L_OK;
  if (!d_y || !d_out) return fail(B2L_ERR_INVALID, "NULL device pointer");
  if (T > 0x7fffffffLL) return fail(B2L_ERR_UNSUPPORTED, "too many frames");
  DeviceGuard g(c->device);
  // frame_length a multiple of hop_length: block form, every sample read once (feat_kernels.cuh)
  {
    const long long tiles = (T + TD_FRAMES - 1) / TD_FRAMES;
    if (frame_length % hop_length == 0 && frame_length / hop_length <= 64 && n_clips <= kMaxGridY && tiles <= 0x7fffffffLL) {
      const int R = frame_length / hop_length;
      const size_t smem = (size_t)(TD_FRAMES + R - 1) * 8;
      return launch(c, frame_td_block_kernel, dim3((unsigned)tiles, (unsigned)n_clips), 256, smem, d_y, y_stride, (int)n,
                    frame_length, hop_length, pad, pad_mode, (int)T, what, threshold, zero_pos, pad_first, out_scale, d_out,
                    c->d_status);
    }
  }
  const long long rows = (long long)n_clips * T;
  const long long grid = grid_stride_blocks(rows, 8, 8LL * c->sm_count);
  return launch(c, frame_td_kernel, (unsigned)grid, 256, 0, d_y, y_stride, (int)n, n_clips, frame_length, hop_length, pad,
                pad_mode, (int)T, what, threshold, zero_pos, pad_first, out_scale, d_out, c->d_status);
}

extern "C" int b2l_melspectrogram(b2l_ctx* c, const b2l_plan* p, const float* d_y, int64_t n_clips, int64_t n,
                                  int64_t y_stride, float* d_mel) {
  if (!c || !p) return fail(B2L_ERR_INVALID, "NULL ctx / plan");
  switch (route(p, ENTRY_MEL)) {
    case PATH_MR: return run_mr(c, p, 2, 0, d_y, n_clips, n, y_stride, nullptr, d_mel);
    case PATH_NONE:
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
  const Path path = route(p, ENTRY_MEL);
  if (path == PATH_NONE)
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
  const int tiled = path == PATH_POW2 ? 1 : 0;
  rc = path == PATH_MR ? run_mr(c, p, 2, 1, d_y, n_clips, n, y_stride, nullptr, scratch)
                       : run_forward(c, p, MODE_MEL, 2, d_y, n_clips, n, y_stride, nullptr, scratch);
  return rc ? rc : launch_dct(c, p, scratch, n_clips, T, 1, d_mfcc, tiled);
}

// ------------------------------------------------------------------ inverse launches
// Grows the context's scratch array to at least `bytes` (the contents are not kept).
static int ensure_scratch(b2l_ctx* c, size_t bytes) {
  if (c->scratch_bytes >= bytes) return B2L_OK;
  if (c->d_scratch) {
    CUDA_TRY(cudaStreamSynchronize(c->stream));
    CUDA_TRY(cudaFree(c->d_scratch));
    c->d_scratch = nullptr;
    c->scratch_bytes = 0;
  }
  CUDA_TRY(cudaMalloc((void**)&c->d_scratch, bytes));
  c->scratch_bytes = bytes;
  return B2L_OK;
}

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
  const Path path = route(p, ENTRY_SPECTRUM);
  if (path == PATH_POW2)
    return run_inverse(c, p, d_D, n_clips, n_frames_stored, n_frames_used, d_inv_wss, out_len, d_y, y_stride);
  // mixed-radix or chirp-z frames into the scratch array, then a gather overlap-add
  if (out_len > 0x7fffffffLL || n_clips > kMaxGridY) return fail(B2L_ERR_UNSUPPORTED, "istft batch too large");
  DeviceGuard g(c->device);
  const int L = p->n_fft;
  int rc = ensure_scratch(c, (size_t)n_clips * (size_t)n_frames_used * L * sizeof(float));
  if (rc == B2L_OK)
    rc = path == PATH_MR ? run_mr_inverse(c, p, d_D, n_clips, n_frames_stored, n_frames_used)
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

// ------------------------------------------------------------------ polyphase resampling
extern "C" int b2l_resample_poly(b2l_ctx* c, const float* d_x, int64_t n_clips, int64_t n_in, int64_t x_stride,
                                 const float* d_h, int32_t n_h, int32_t up, int32_t down, int64_t n_pre_remove,
                                 int64_t n_keep, int64_t n_total, float out_scale, float* d_out) {
  if (!c || !d_x || !d_h || !d_out) return fail(B2L_ERR_INVALID, "NULL argument");
  if (up < 1 || down < 1 || n_h < 1 || n_pre_remove < 0 || n_keep < 0 || n_total < n_keep || x_stride < n_in)
    return fail(B2L_ERR_INVALID, "bad resampling geometry");
  if (n_clips <= 0 || n_total <= 0) return B2L_OK;
  if (n_in > 0x7fffffffLL || n_total > 0x7fffffffLL) return fail(B2L_ERR_UNSUPPORTED, "signals longer than 2^31-1 samples");
  DeviceGuard g(c->device);
  const long long grid = grid_stride_blocks((long long)n_clips * n_total, 256, 32LL * c->sm_count);
  return launch(c, resample_poly_kernel, (unsigned)grid, 256, 0, d_x, x_stride, (int)n_in, d_h, n_h, up, down,
                n_pre_remove, (int)n_keep, (int)n_total, n_clips, out_scale, d_out);
}

extern "C" int b2l_power_to_db(b2l_ctx* c, const float* d_in, int64_t n_clips, int64_t per_clip, float amin,
                               float ref_value, float top_db, float* d_out) {
  if (!c || !d_in || !d_out) return fail(B2L_ERR_INVALID, "NULL argument");
  if (!(amin > 0.0f)) return fail(B2L_ERR_INVALID, "amin must be strictly positive");
  if (n_clips <= 0 || per_clip <= 0) return B2L_OK;
  DeviceGuard g(c->device);
  int rc = ensure_clip_max(c, (size_t)n_clips);
  if (rc) return rc;
  CUDA_TRY(cudaMemsetAsync(c->d_clip_max, 0, (size_t)n_clips * sizeof(unsigned int), c->stream));
  const float db_sub = 10.0f * log10f(fmaxf(amin, fabsf(ref_value)));
  return for_clip_slices(n_clips, [&](int64_t c0, int64_t m) {
    const dim3 grid((unsigned)row_blocks(per_clip, 256 * 8, 4LL * c->sm_count, m), (unsigned)m);
    int rc = launch(c, db_kernel, grid, 256, 0, d_in + c0 * per_clip, per_clip, amin, db_sub, c->d_clip_max + c0,
                    d_out + c0 * per_clip);
    if (rc == B2L_OK && top_db >= 0.0f)
      rc = launch(c, db_clamp_kernel, grid, 256, 0, d_out + c0 * per_clip, per_clip, c->d_clip_max + c0, top_db);
    return rc;
  });
}

extern "C" int b2l_onset_from_spec(b2l_ctx* c, const b2l_onset_desc* d, const float* d_S, int64_t n_clips,
                                   int64_t n_rows, int64_t n_frames, float* d_out) {
  if (!c || !d || !d_S || !d_out) return fail(B2L_ERR_INVALID, "NULL argument");
  if (d->lag < 1) return fail(B2L_ERR_INVALID, "lag=%d must be a positive integer", d->lag);
  if (d->max_size < 1) return fail(B2L_ERR_INVALID, "max_size=%d must be a positive integer", d->max_size);
  if (d->pad_width < 0) return fail(B2L_ERR_INVALID, "negative pad_width");
  if (d->n_channels < 0 || d->n_channels > 32) return fail(B2L_ERR_UNSUPPORTED, "at most 32 onset channels");
  if (n_clips <= 0 || n_rows <= 0 || n_frames <= 0) return B2L_OK;
  if (n_clips > kMaxGridY || n_rows > 0x7fffffffLL || n_frames > 0x7fffffffLL)
    return fail(B2L_ERR_UNSUPPORTED, "onset: batch too large");
  OnsetArgs a;
  memset(&a, 0, sizeof(a));
  for (int i = 0; i <= d->n_channels; ++i) {
    a.bounds[i] = d->bounds[i];
    if (a.bounds[i] < 0 || a.bounds[i] > n_rows || (i > 0 && a.bounds[i] < a.bounds[i - 1]))
      return fail(B2L_ERR_INVALID, "channel boundaries must be non-decreasing row indices");
  }
  a.n_ch = d->n_channels;
  a.lag = d->lag;
  a.max_size = d->max_size;
  a.pad_width = d->pad_width;
  a.n_rows = (int)n_rows;
  a.T = (int)n_frames;
  DeviceGuard g(c->device);
  int rc = launch(c, onset_kernel, dim3((unsigned)((n_frames + 127) / 128), (unsigned)n_clips), 128, 0, d_S, a, d_out);
  if (rc || !d->detrend) return rc;
  const long long rows = (long long)n_clips * (a.n_ch > 0 ? a.n_ch : a.n_rows);
  return launch(c, detrend_kernel, (unsigned)((rows + 127) / 128), 128, 0, d_out, rows, a.T);
}

extern "C" int b2l_onset_median_from_spec(b2l_ctx* c, const b2l_onset_desc* d, const float* d_S, int64_t n_clips,
                                          int64_t n_rows, int64_t n_frames, float* d_out) {
  if (!c || !d || !d_S || !d_out) return fail(B2L_ERR_INVALID, "NULL argument");
  if (d->lag < 1) return fail(B2L_ERR_INVALID, "lag=%d must be a positive integer", d->lag);
  if (d->max_size < 1) return fail(B2L_ERR_INVALID, "max_size=%d must be a positive integer", d->max_size);
  if (d->pad_width < 0) return fail(B2L_ERR_INVALID, "negative pad_width");
  if (d->n_channels < 1 || d->n_channels > 32) return fail(B2L_ERR_UNSUPPORTED, "1 to 32 onset channels");
  if (n_clips <= 0 || n_rows <= 0 || n_frames <= 0) return B2L_OK;
  if (n_clips > kMaxGridY || n_rows > 0x7fffffffLL || n_frames > 0x7fffffffLL)
    return fail(B2L_ERR_UNSUPPORTED, "onset: batch too large");
  OnsetArgs a;
  memset(&a, 0, sizeof(a));
  int widest = 0;
  for (int i = 0; i <= d->n_channels; ++i) {
    a.bounds[i] = d->bounds[i];
    if (a.bounds[i] < 0 || a.bounds[i] > n_rows || (i > 0 && a.bounds[i] < a.bounds[i - 1]))
      return fail(B2L_ERR_INVALID, "channel boundaries must be non-decreasing row indices");
    if (i > 0) widest = std::max(widest, a.bounds[i] - a.bounds[i - 1]);
  }
  if (widest > kOnsetMedMaxRows)
    return fail(B2L_ERR_UNSUPPORTED, "onset: median aggregation over a channel of %d rows; the GPU kernel takes up to %d",
                widest, kOnsetMedMaxRows);
  a.n_ch = d->n_channels;
  a.lag = d->lag;
  a.max_size = d->max_size;
  a.pad_width = d->pad_width;
  a.n_rows = (int)n_rows;
  a.T = (int)n_frames;
  int P = 32;
  while (P < widest) P <<= 1;
  const size_t smem = (size_t)kOnsetMedFrames * (P + 1) * sizeof(float);
  DeviceGuard g(c->device);
  const dim3 grid((unsigned)((n_frames + kOnsetMedFrames - 1) / kOnsetMedFrames), (unsigned)n_clips);
  int rc = launch(c, onset_median_kernel, grid, 256, smem, d_S, a, P, d_out);
  if (rc || !d->detrend) return rc;
  const long long rows = (long long)n_clips * a.n_ch;
  return launch(c, detrend_kernel, (unsigned)((rows + 127) / 128), 128, 0, d_out, rows, a.T);
}

extern "C" int b2l_pcen(b2l_ctx* c, const b2l_pcen_desc* d, const float* d_S, int64_t n_clips, int64_t n_rows,
                        int64_t n_frames, const float* d_zi, float* d_zf, float* d_scratch, float* d_out) {
  if (!c || !d || !d_S || !d_out) return fail(B2L_ERR_INVALID, "NULL argument");
  if (d->power < 0.0f) return fail(B2L_ERR_INVALID, "power=%g must be nonnegative", d->power);
  if (d->gain < 0.0f) return fail(B2L_ERR_INVALID, "gain=%g must be non-negative", d->gain);
  if (d->bias < 0.0f) return fail(B2L_ERR_INVALID, "bias=%g must be non-negative", d->bias);
  if (!(d->eps > 0.0f)) return fail(B2L_ERR_INVALID, "eps=%g must be strictly positive", d->eps);
  if (!(d->b >= 0.0f && d->b <= 1.0f)) return fail(B2L_ERR_INVALID, "b=%g must be between 0 and 1", d->b);
  if (d->max_size < 1) return fail(B2L_ERR_INVALID, "max_size=%d must be a positive integer", d->max_size);
  if (n_clips <= 0 || n_rows <= 0 || n_frames <= 0) return B2L_OK;
  if (n_frames > 0x7fffffffLL || n_rows > kMaxGridY || n_clips > kMaxGridY)
    return fail(B2L_ERR_UNSUPPORTED, "pcen: batch too large");
  DeviceGuard g(c->device);
  const float* ref = d_S;
  if (d->max_size > 1) {
    if (!d_scratch) return fail(B2L_ERR_INVALID, "max_size > 1 needs a scratch buffer of the size of S");
    const dim3 grid((unsigned)((n_frames + 127) / 128), (unsigned)n_rows, (unsigned)n_clips);
    if (int rc = launch(c, maxfilter_rows_kernel, grid, 128, 0, d_S, (int)n_rows, (int)n_frames, d->max_size, d_scratch))
      return rc;
    ref = d_scratch;
  }
  PcenArgs a;
  a.gain = d->gain;
  a.bias = d->bias;
  a.power = d->power;
  a.eps = d->eps;
  a.b = d->b;
  a.mode = d->power == 0.0f ? 0 : (d->bias == 0.0f ? 1 : 2);
  const long long rows = (long long)n_clips * n_rows;
  return launch(c, pcen_kernel, (unsigned)((rows + 127) / 128), 128, 0, d_S, ref, rows, (int)n_frames, a, d_zi, d_zf,
                d_out);
}

extern "C" int b2l_spectral_contrast(b2l_ctx* c, const b2l_contrast_desc* d, const float* d_S, int64_t n_clips,
                                     int64_t n_frames, int32_t n_bins, float* d_peak, float* d_valley) {
  if (!c || !d || !d_S || !d_peak || !d_valley) return fail(B2L_ERR_INVALID, "NULL argument");
  if (d->n_bands < 1 || d->n_bands > 16) return fail(B2L_ERR_UNSUPPORTED, "1 to 16 bands (n_bands + 1) are supported");
  if (n_clips <= 0 || n_frames <= 0) return B2L_OK;
  ContrastArgs a;
  memset(&a, 0, sizeof(a));
  a.n_bands = d->n_bands;
  int max_count = 1;
  for (int b = 0; b < d->n_bands; ++b) {
    if (d->lo[b] < 0 || d->count[b] < 0 || d->lo[b] + d->count[b] > n_bins || d->k[b] < 1)
      return fail(B2L_ERR_INVALID, "band %d: bad bin range / tail length", b);
    a.lo[b] = d->lo[b];
    a.count[b] = d->count[b];
    a.k[b] = d->k[b];
    max_count = std::max(max_count, d->count[b]);
  }
  int cap = 32;   // at least one entry per lane: the short-tail path parks 32 sorted runs in the scratch
  while (cap < max_count) cap <<= 1;
  DeviceGuard g(c->device);
  const size_t per_warp = ((size_t)((n_bins + 3) & ~3) + cap) * 4;
  int nw = 8;
  while (nw > 1 && per_warp * nw > c->smem_optin) nw >>= 1;
  const size_t smem = per_warp * nw;
  if (smem > c->smem_optin) return fail(B2L_ERR_UNSUPPORTED, "n_bins=%d rows do not fit in shared memory", n_bins);
  const int rc = blocks_per_sm(c, contrast_kernel, nw * 32, smem, nullptr);
  if (rc) return rc;
  const long long rows = (long long)n_clips * n_frames;
  const long long grid = grid_stride_blocks(rows, nw, 8LL * c->sm_count);
  return launch(c, contrast_kernel, (unsigned)grid, nw * 32, smem, d_S, rows, (int)n_frames, n_bins, cap, a, d_peak,
                d_valley);
}

extern "C" int b2l_sub(b2l_ctx* c, const float* d_x, const float* d_y, int64_t n, float* d_out) {
  if (!c || !d_x || !d_y || !d_out) return fail(B2L_ERR_INVALID, "NULL argument");
  if (n <= 0) return B2L_OK;
  DeviceGuard g(c->device);
  return launch(c, sub_kernel, (unsigned)grid_stride_blocks(n, 256 * 8, 8LL * c->sm_count), 256, 0, d_x, d_y, n, d_out);
}

extern "C" int b2l_pip_pass(b2l_ctx* c, const b2l_pip_desc* d, const float* d_S, int64_t n_rows, int32_t n_bins,
                            const double* h_edges, uint64_t* h_hist) {
  if (!c || !d || !d_S || !h_hist) return fail(B2L_ERR_INVALID, "NULL argument");
  if (d->mode < 0 || d->mode > 3) return fail(B2L_ERR_INVALID, "bad pass mode %d", d->mode);
  if (d->mode == 3 && (!h_edges || d->n_res_bins < 1 || d->n_res_bins > 2048))
    return fail(B2L_ERR_INVALID, "residual histogram needs 1..2048 bins and their edges");
  if (d->k_lo < 0 || d->k_hi > n_bins) return fail(B2L_ERR_INVALID, "bad bin range");
  const int n_hist = d->mode == 3 ? d->n_res_bins : (d->mode == 2 ? 1024 : 2048);
  for (int i = 0; i < n_hist; ++i) h_hist[i] = 0;
  if (n_rows <= 0 || d->k_hi <= d->k_lo) return B2L_OK;
  DeviceGuard g(c->device);
  int rc = ensure_scratch(c, 2048 * sizeof(unsigned long long) + 2049 * sizeof(double));
  if (rc) return rc;
  unsigned long long* d_hist = reinterpret_cast<unsigned long long*>(c->d_scratch);
  double* d_edges = reinterpret_cast<double*>(d_hist + 2048);
  CUDA_TRY(cudaMemsetAsync(d_hist, 0, 2048 * sizeof(unsigned long long), c->stream));
  if (d->mode == 3)
    CUDA_TRY(cudaMemcpyAsync(d_edges, h_edges, (size_t)(d->n_res_bins + 1) * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  PipArgs a;
  a.k_lo = d->k_lo;
  a.k_hi = d->k_hi;
  a.threshold = d->threshold;
  a.ref_abs = d->ref_abs;
  a.hz_per_bin = d->hz_per_bin;
  a.mode = d->mode;
  a.prefix = d->prefix;
  a.mag_threshold = d->mag_threshold;
  a.bins_per_octave = d->bins_per_octave;
  a.n_res_bins = d->n_res_bins;
  const size_t per_warp = (size_t)((n_bins + 3) & ~3) * 4;
  int nw = 8;
  while (nw > 1 && per_warp * nw + 8192 + 1024 > c->smem_optin) nw >>= 1;
  const size_t smem = per_warp * nw;
  if (smem + 8192 + 1024 > c->smem_optin) return fail(B2L_ERR_UNSUPPORTED, "n_bins=%d rows do not fit in shared memory", n_bins);
  // 8 KB of static shared memory (the block's histogram) and 1 KB reserved by the system
  if ((rc = blocks_per_sm(c, pip_pass_kernel, nw * 32, smem, nullptr, c->smem_optin - 8192 - 1024))) return rc;
  const long long grid = grid_stride_blocks(n_rows, nw, 4LL * c->sm_count);
  if ((rc = launch(c, pip_pass_kernel, (unsigned)grid, nw * 32, smem, d_S, n_rows, n_bins, a, d_edges, d_hist))) return rc;
  CUDA_TRY(cudaMemcpyAsync(h_hist, d_hist, (size_t)n_hist * sizeof(unsigned long long), cudaMemcpyDeviceToHost, c->stream));
  CUDA_TRY(cudaStreamSynchronize(c->stream));
  return B2L_OK;
}

extern "C" int b2l_normalize_rows(b2l_ctx* c, const float* d_in, int64_t n_clips, int64_t n_rows, int64_t n_frames,
                                  int32_t norm_kind, float norm_p, float* d_out) {
  if (!c || !d_in || !d_out) return fail(B2L_ERR_INVALID, "NULL argument");
  if (norm_kind < 0 || norm_kind > 3) return fail(B2L_ERR_INVALID, "bad norm kind %d", norm_kind);
  if (norm_kind == 3 && !(norm_p > 0.0f)) return fail(B2L_ERR_INVALID, "Unsupported norm: %g", norm_p);
  if (n_clips <= 0 || n_rows <= 0 || n_frames <= 0) return B2L_OK;
  if (n_clips > kMaxGridY || n_rows > 0x7fffffffLL || n_frames > 0x7fffffffLL) return fail(B2L_ERR_UNSUPPORTED, "normalize: batch too large");
  DeviceGuard g(c->device);
  return launch(c, normalize_rows_kernel, dim3((unsigned)((n_frames + 127) / 128), (unsigned)n_clips), 128, 0, d_in,
                (int)n_rows, (int)n_frames, norm_kind, norm_p, d_out);
}

extern "C" int b2l_cabs(b2l_ctx* c, const void* d_complex, int64_t n, float* d_out) {
  if (!c || !d_complex || !d_out) return fail(B2L_ERR_INVALID, "NULL argument");
  if (n <= 0) return B2L_OK;
  DeviceGuard g(c->device);
  return launch(c, cabs_kernel, (unsigned)grid_stride_blocks(n, 256 * 8, 8LL * c->sm_count), 256, 0,
                (const float2*)d_complex, n, d_out);
}

extern "C" int b2l_hpss(b2l_ctx* c, const b2l_hpss_desc* d, const float* d_mag, const void* d_S_complex,
                        int64_t n_clips, int64_t n_frames, int64_t n_bins, void* d_out_harm, void* d_out_perc) {
  if (!c || !d || !d_mag || !d_out_harm || !d_out_perc) return fail(B2L_ERR_INVALID, "NULL argument");
  if (d->win_harm < 1 || d->win_perc < 1) return fail(B2L_ERR_INVALID, "kernel sizes must be positive");
  if (d->win_harm > 64 || d->win_perc > 64) return fail(B2L_ERR_UNSUPPORTED, "median filters longer than 64 are not supported");
  if (d->margin_harm < 1.0f || d->margin_perc < 1.0f)
    return fail(B2L_ERR_INVALID, "Margins must be >= 1.0. A typical range is between 1 and 10.");
  if (!(d->power > 0.0f)) return fail(B2L_ERR_INVALID, "power must be strictly positive");
  if (n_clips <= 0 || n_frames <= 0 || n_bins <= 0) return B2L_OK;
  if (n_frames > kMaxGridY || n_clips > kMaxGridY || n_bins > 0x7fffffffLL)
    return fail(B2L_ERR_UNSUPPORTED, "hpss: batch too large");
  HpssArgs a;
  a.T = (int)n_frames;
  a.F = (int)n_bins;
  a.win_h = d->win_harm;
  a.win_p = d->win_perc;
  a.margin_h = d->margin_harm;
  a.margin_p = d->margin_perc;
  a.power = d->power;
  a.split_zeros = (d->margin_harm == 1.0f && d->margin_perc == 1.0f) ? 1 : 0;
  a.mode = d->mask_only ? 1 : 0;
  DeviceGuard g(c->device);
  const int w = std::max(d->win_harm, d->win_perc);
  auto kern = w <= 8 ? hpss_kernel<8> : w <= 16 ? hpss_kernel<16> : w <= 32 ? hpss_kernel<32> : hpss_kernel<64>;
  const dim3 grid((unsigned)((n_bins + 127) / 128), (unsigned)n_frames, (unsigned)n_clips);
  const float2* sc = d->mask_only ? nullptr : (const float2*)d_S_complex;
  return launch(c, kern, grid, 128, 0, d_mag, sc, a, (float*)d_out_harm, (float*)d_out_perc);
}

extern "C" int b2l_reassign(b2l_ctx* c, const b2l_reassign_desc* d, const void* d_Sh, const void* d_Sdh,
                            const void* d_Sth, int64_t n_clips, int64_t n_frames, int64_t n_bins,
                            const float* d_bin_freqs, const float* d_frame_times, float* d_freqs, float* d_times,
                            float* d_mags) {
  if (!c || !d || !d_Sh || !d_bin_freqs || !d_frame_times || !d_freqs || !d_times || !d_mags)
    return fail(B2L_ERR_INVALID, "NULL argument");
  if ((d->reassign_frequencies && !d_Sdh) || (d->reassign_times && !d_Sth))
    return fail(B2L_ERR_INVALID, "missing derivative / time-weighted STFT");
  if (n_clips <= 0 || n_frames <= 0 || n_bins <= 0) return B2L_OK;
  if (n_frames > 0x7fffffffLL || n_bins > 0x7fffffffLL) return fail(B2L_ERR_UNSUPPORTED, "reassign: too large");
  ReassignArgs a;
  a.T = (int)n_frames;
  a.F = (int)n_bins;
  a.freq_scale = (float)(0.5 * (double)d->sr / 3.14159265358979323846);
  a.inv_sr = (float)(1.0 / (double)d->sr);
  a.mag_threshold = d->mag_threshold;
  a.max_freq = (float)(0.5 * (double)d->sr);
  a.max_time = d->max_time;
  a.do_freq = d->reassign_frequencies ? 1 : 0;
  a.do_time = d->reassign_times ? 1 : 0;
  a.apply_threshold = d->apply_threshold ? 1 : 0;
  a.fill_nan = d->fill_nan ? 1 : 0;
  a.clip = d->clip ? 1 : 0;
  DeviceGuard g(c->device);
  const long long n = (long long)n_clips * n_frames * n_bins;
  return launch(c, reassign_kernel, (unsigned)grid_stride_blocks(n, 256 * 4, 16LL * c->sm_count), 256, 0,
                (const float2*)d_Sh, (const float2*)d_Sdh, (const float2*)d_Sth, d_bin_freqs, d_frame_times, a, n, d_freqs,
                d_times, d_mags);
}

extern "C" int b2l_phase_vocoder(b2l_ctx* c, const void* d_D, int64_t n_clips, int64_t n_frames, int64_t n_bins,
                                 int64_t n_out, const int32_t* d_i0, const int32_t* d_i1, const int32_t* d_lo,
                                 const double* d_dx, void* d_out) {
  if (!c || !d_D || !d_i0 || !d_i1 || !d_lo || !d_dx || !d_out) return fail(B2L_ERR_INVALID, "NULL argument");
  if (n_clips <= 0 || n_bins <= 0 || n_out <= 0) return B2L_OK;
  if (n_frames < 2) return fail(B2L_ERR_UNSUPPORTED, "phase_vocoder needs at least two input frames");
  if (n_frames > 0x7fffffffLL || n_bins > 0x7fffffffLL || n_out > 0x7fffffffLL)
    return fail(B2L_ERR_UNSUPPORTED, "phase_vocoder: too large");
  DeviceGuard g(c->device);
  const long long threads = (long long)n_clips * n_bins;
  return launch(c, phase_vocoder_kernel, (unsigned)((threads + 127) / 128), 128, 0, (const float2*)d_D, (int)n_frames,
                (int)n_bins, n_clips, (int)n_out, d_i0, d_i1, d_lo, d_dx, (float2*)d_out);
}

extern "C" int b2l_unary(b2l_ctx* c, int32_t op, const float* d_in, int64_t n, float param, float* d_out) {
  if (!c || !d_in || !d_out) return fail(B2L_ERR_INVALID, "NULL argument");
  if (op < 0 || op > B2L_UNARY_DB_TO_AMPLITUDE) return fail(B2L_ERR_INVALID, "bad unary op %d", op);
  if (n <= 0) return B2L_OK;
  DeviceGuard g(c->device);
  return launch(c, unary_kernel, (unsigned)grid_stride_blocks(n, 256 * 8, 8LL * c->sm_count), 256, 0, d_in, n, op, param,
                d_out);
}

extern "C" int b2l_dct_project(b2l_ctx* c, const b2l_plan* p, const float* d_S, int64_t n_clips, int64_t n_frames,
                               float* d_mfcc) {
  if (!c || !p || !d_S || !d_mfcc) return fail(B2L_ERR_INVALID, "NULL argument");
  if (p->n_mfcc == 0) return fail(B2L_ERR_INVALID, "plan has no mfcc stage");
  if (n_clips <= 0 || n_frames <= 0) return B2L_OK;
  DeviceGuard g(c->device);
  return launch_dct(c, p, d_S, n_clips, n_frames, 0, d_mfcc);
}

extern "C" int b2l_gl_update(b2l_ctx* c, const void* d_rebuilt, const void* d_tprev, const float* d_S, float scale,
                             float eps, void* d_angles, int64_t n) {
  if (!c || !d_rebuilt || !d_S || !d_angles) return fail(B2L_ERR_INVALID, "NULL argument");
  if (n <= 0) return B2L_OK;
  DeviceGuard g(c->device);
  return launch(c, gl_update_kernel, (unsigned)grid_stride_blocks(n, 256, 8LL * c->sm_count), 256, 0,
                (const float2*)d_rebuilt, (const float2*)d_tprev, d_S, scale, eps, (float2*)d_angles, n);
}

extern "C" int b2l_transpose(b2l_ctx* c, const void* d_in, int64_t n_clips, int64_t rows, int64_t cols,
                             int32_t elem_bytes, void* d_out) {
  if (!c || !d_in || !d_out) return fail(B2L_ERR_INVALID, "NULL argument");
  if (n_clips <= 0 || rows <= 0 || cols <= 0) return B2L_OK;
  if (elem_bytes != 4 && elem_bytes != 8) return fail(B2L_ERR_INVALID, "elem_bytes must be 4 or 8");
  DeviceGuard g(c->device);
  return for_clip_slices(n_clips, [&](int64_t c0, int64_t m) {
    const dim3 grid((unsigned)((cols + 31) / 32), (unsigned)((rows + 31) / 32), (unsigned)m), block(32, 8);
    const size_t off = (size_t)c0 * (size_t)rows * (size_t)cols;
    return elem_bytes == 4 ? launch(c, transpose_kernel<float>, grid, block, 0, (const float*)d_in + off, (int)rows,
                                    (int)cols, (float*)d_out + off)
                           : launch(c, transpose_kernel<float2>, grid, block, 0, (const float2*)d_in + off, (int)rows,
                                    (int)cols, (float2*)d_out + off);
  });
}

// ------------------------------------------------------------------ pitch tracking (pitch_kernels.cuh)
static int check_periods(int min_period, int max_period, int frame_length) {
  if (min_period < 0 || max_period <= min_period || max_period >= frame_length)
    return fail(B2L_ERR_INVALID, "periods %d .. %d do not fit frame_length=%d", min_period, max_period, frame_length);
  return B2L_OK;
}

#define B2L_CASE(L) case L: return yin_cmnd_kernel<L>;
static void (*yin_cmnd_kernel_for(int log2m))(YinCmndArgs) {
  switch (log2m) { B2L_FFT_SIZES(B2L_CASE) }
  return nullptr;
}
#undef B2L_CASE

extern "C" int b2l_yin_cmnd(b2l_ctx* c, const b2l_yin_desc* d, const float* d_y, int64_t n_clips, int64_t n,
                            int64_t y_stride, float* d_cmnd) {
  if (!c || !d) return fail(B2L_ERR_INVALID, "NULL argument");
  const int L = d->frame_length;
  if (L < 1) return fail(B2L_ERR_INVALID, "frame_length=%d must be positive", L);
  if (d->hop_length < 1) return fail(B2L_ERR_INVALID, "hop_length=%d must be a positive integer", d->hop_length);
  if (d->pad_mode < 0 || d->pad_mode > B2L_PAD_EMPTY) return fail(B2L_ERR_INVALID, "bad pad_mode %d", d->pad_mode);
  if (int rc = check_periods(d->min_period, d->max_period, L)) return rc;
  if (n_clips < 0 || n < 0 || y_stride < n) return fail(B2L_ERR_INVALID, "bad clip geometry");
  if (n > 0x7fffffffLL) return fail(B2L_ERR_UNSUPPORTED, "clips longer than 2^31-1 samples are not supported");
  const int pad = d->center ? L / 2 : 0;
  const long long padded = n + 2LL * pad;
  if (padded < L) return fail(B2L_ERR_INVALID, "Input is too short (n=%lld) for frame_length=%d", padded, L);
  // zero padding to N >= frame_length + max_period + 1 keeps lags 0 .. max_period free of circular wrap-around
  const long long need = (long long)L + d->max_period + 1;
  int log2n = 0;
  while ((1LL << log2n) < need) ++log2n;
  const int log2m = std::max(kMinLog2M, log2n - 1);
  if (log2m > kMaxLog2M)
    return fail(B2L_ERR_UNSUPPORTED, "yin: the zero-padded frame needs %lld points (frame_length %d + max_period %d + 1); "
                "the GPU FFT goes up to %d", 1LL << log2n, L, d->max_period, 2 << kMaxLog2M);
  const long long T = 1 + (padded - L) / d->hop_length;
  if (T > 0x7fffffffLL) return fail(B2L_ERR_UNSUPPORTED, "too many frames");
  if (n_clips == 0) return B2L_OK;
  if (!d_y || !d_cmnd) return fail(B2L_ERR_INVALID, "NULL device pointer");
  DeviceGuard g(c->device);
  const HostFftCfg cfg(log2m);
  const std::vector<float2> tw = engine_twiddles(cfg);
  Temp d_tw(c->stream);
  CUDA_TRY(upload(d_tw, tw.data(), tw.size()));
  const int G = 256 / cfg.tpf;
  const size_t smem = (size_t)cfg.tw_count() * 8 + (size_t)G * cfg.xbuf_f2() * 8;
  auto fn = yin_cmnd_kernel_for(log2m);
  long long grid = 0;
  if (int rc = resident_grid(c, fn, 256, smem, (n_clips * T + G - 1) / G, &grid)) return rc;
  if (!grid) return fail(B2L_ERR_CUDA, "yin_cmnd_kernel does not fit on an SM (smem %zu)", smem);
  YinCmndArgs a;
  a.y = d_y;
  a.clip_stride = y_stride;
  a.n = (int)n;
  a.n_clips = (int)n_clips;
  a.n_frames = (int)T;
  a.frame_length = L;
  a.hop = d->hop_length;
  a.pad = pad;
  a.pad_mode = d->pad_mode;
  a.min_period = d->min_period;
  a.max_period = d->max_period;
  a.tw = (const float2*)d_tw.p;
  a.cmnd = d_cmnd;
  a.status = c->d_status;
  return launch(c, fn, (unsigned)grid, 256, smem, a);
}

extern "C" int b2l_yin_pick(b2l_ctx* c, const b2l_yin_desc* d, const float* d_cmnd, int64_t n_rows, double* d_f0) {
  if (!c || !d) return fail(B2L_ERR_INVALID, "NULL argument");
  if (int rc = check_periods(d->min_period, d->max_period, d->max_period + 1)) return rc;
  if (n_rows < 0) return fail(B2L_ERR_INVALID, "bad row count");
  if (n_rows == 0) return B2L_OK;
  if (!d_cmnd || !d_f0) return fail(B2L_ERR_INVALID, "NULL device pointer");
  DeviceGuard g(c->device);
  const int n_lags = d->max_period - d->min_period + 1;
  const size_t smem = (size_t)8 * n_lags * 4;
  long long grid = 0;
  if (int rc = resident_grid(c, yin_pick_kernel, 256, smem, (n_rows + 7) / 8, &grid)) return rc;
  if (!grid) return fail(B2L_ERR_UNSUPPORTED, "yin: %d lags do not fit in shared memory", n_lags);
  return launch(c, yin_pick_kernel, (unsigned)grid, 256, smem, d_cmnd, (long long)n_rows, n_lags, d->min_period, d->sr,
                d->trough_threshold, d_f0);
}

static int check_pyin_desc(const b2l_pyin_desc* d) {
  if (int rc = check_periods(d->min_period, d->max_period, d->max_period + 1)) return rc;
  if (d->n_thresholds < 1) return fail(B2L_ERR_INVALID, "n_thresholds=%d must be positive", d->n_thresholds);
  if (d->n_pitch_bins < 1 || d->n_bins_per_semitone < 1) return fail(B2L_ERR_INVALID, "bad pitch bins");
  return B2L_OK;
}

extern "C" int b2l_pyin_obs(b2l_ctx* c, const b2l_pyin_desc* d, const float* d_cmnd, int64_t n_rows, int32_t* d_count,
                            int32_t* d_cand_bin, double* d_cand_prob, double* d_voiced_prob) {
  if (!c || !d) return fail(B2L_ERR_INVALID, "NULL argument");
  if (int rc = check_pyin_desc(d)) return rc;
  if (n_rows < 0) return fail(B2L_ERR_INVALID, "bad row count");
  if (n_rows == 0) return B2L_OK;
  if (!d_cmnd || !d_count || !d_cand_bin || !d_cand_prob || !d_voiced_prob || !d->d_thresholds || !d->d_beta ||
      !d->d_beta_cum || !d->d_pmf)
    return fail(B2L_ERR_INVALID, "NULL device pointer");
  DeviceGuard g(c->device);
  PyinObsArgs a;
  a.cmnd = d_cmnd;
  a.rows = n_rows;
  a.n_lags = d->max_period - d->min_period + 1;
  a.min_period = d->min_period;
  a.max_cand = (a.n_lags + 1) / 2;
  a.n_thresholds = d->n_thresholds;
  a.n_pitch_bins = d->n_pitch_bins;
  a.n_bins_per_semitone = d->n_bins_per_semitone;
  a.sr = d->sr;
  a.fmin = d->fmin;
  a.no_trough_prob = d->no_trough_prob;
  a.thresholds = d->d_thresholds;
  a.beta = d->d_beta;
  a.beta_cum = d->d_beta_cum;
  a.pmf = d->d_pmf;
  a.count = d_count;
  a.cand_bin = d_cand_bin;
  a.cand_prob = d_cand_prob;
  a.voiced_prob = d_voiced_prob;
  const size_t smem = 4 * pyin_obs_slice(a.n_lags, a.max_cand, a.n_thresholds);
  if (smem > c->smem_optin) return fail(B2L_ERR_UNSUPPORTED, "pyin: %d lags do not fit in shared memory", a.n_lags);
  long long grid = 0;
  if (int rc = resident_grid(c, pyin_obs_kernel, 128, smem, (n_rows + 3) / 4, &grid)) return rc;
  if (!grid) return fail(B2L_ERR_UNSUPPORTED, "pyin: %d lags do not fit in shared memory", a.n_lags);
  return launch(c, pyin_obs_kernel, (unsigned)grid, 128, smem, a);
}

extern "C" int b2l_viterbi(b2l_ctx* c, const b2l_pyin_desc* d, const int32_t* d_count, const int32_t* d_cand_bin,
                           const double* d_cand_prob, const double* d_voiced_prob, int64_t n_clips, int64_t n_frames,
                           uint16_t* d_states, double* d_f0, uint8_t* d_voiced) {
  if (!c || !d) return fail(B2L_ERR_INVALID, "NULL argument");
  if (int rc = check_pyin_desc(d)) return rc;
  if (n_clips < 0 || n_frames < 0) return fail(B2L_ERR_INVALID, "bad batch geometry");
  if (d->half_width < 0) return fail(B2L_ERR_INVALID, "half_width=%d must be non-negative", d->half_width);
  const long long S = 2LL * d->n_pitch_bins;
  if (S > 65536) return fail(B2L_ERR_UNSUPPORTED, "viterbi: %lld states do not fit 16-bit back-pointers", S);
  cudaFuncAttributes fa;
  CUDA_TRY(cudaFuncGetAttributes(&fa, viterbi_kernel));
  const size_t smem = viterbi_smem((int)S), smem_limit = c->smem_optin - fa.sharedSizeBytes;
  if (smem > smem_limit)
    return fail(B2L_ERR_UNSUPPORTED, "viterbi: %lld states need %zu bytes of shared memory, the device has %zu", S, smem,
                smem_limit);
  if (n_clips == 0 || n_frames == 0) return B2L_OK;
  if (n_clips > 0x7fffffffLL) return fail(B2L_ERR_UNSUPPORTED, "too many clips");
  if (!d_count || !d_cand_bin || !d_cand_prob || !d_voiced_prob || !d_states || (d_f0 && !d_voiced) ||
      !d->d_cls || !d->d_ltab || !d->d_freqs)
    return fail(B2L_ERR_INVALID, "NULL device pointer");
  DeviceGuard g(c->device);
  Temp ptr(c->stream);
  CUDA_TRY(ptr.alloc((size_t)n_clips * n_frames * S * sizeof(uint16_t)));
  ViterbiArgs a;
  a.count = d_count;
  a.cand_bin = d_cand_bin;
  a.cand_prob = d_cand_prob;
  a.voiced_prob = d_voiced_prob;
  a.n_frames = (int)n_frames;
  a.max_cand = (d->max_period - d->min_period + 2) / 2;
  a.n_pitch_bins = d->n_pitch_bins;
  a.n_states = (int)S;
  a.log_p_init = d->log_p_init;
  a.tiny = DBL_MIN;
  a.cls = d->d_cls;
  a.ltab = d->d_ltab;
  a.half_width = d->half_width;
  a.full = d->full;
  a.log_thr = d->log_thr;
  a.freqs = d->d_freqs;
  a.fill = d->fill;
  a.fill_na = d->fill_na;
  a.ptr = (unsigned short*)ptr.p;
  a.states = d_states;
  a.f0 = d_f0;
  a.voiced = d_voiced;
  int occ = 0, rc;
  if ((rc = blocks_per_sm(c, viterbi_kernel, 256, smem, &occ, smem_limit))) return rc;
  if (occ < 1) return fail(B2L_ERR_UNSUPPORTED, "viterbi: %lld states do not fit on an SM", S);
  return launch(c, viterbi_kernel, (unsigned)n_clips, 256, smem, a);
}
