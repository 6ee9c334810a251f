// f64_api.cu — C ABI of the double-precision path (f64_kernels.cuh): what the reference computes for float64
// audio / complex128 spectra (librosa/core/spectrum.py:341, :388, :598; feature/spectral.py:2005, 2160).
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "f64_kernels.cuh"
#include "internal.h"

using namespace b2l;

std::vector<double2> b2l::f64_twiddles(int n, int count) {
  std::vector<double2> tw((size_t)count);
  const long double two_pi = 6.283185307179586476925286766559005768L;
  for (int j = 0; j < count; ++j) {
    const long double a = two_pi * (long double)j / (long double)n;
    tw[(size_t)j] = make_double2((double)cosl(a), (double)(-sinl(a)));
  }
  return tw;
}

namespace {

const int kMaxFft64 = 1 << 20;   // power-of-two n_fft (work area in shared memory up to 16384, else in global memory)
const int kMaxDft64 = 1 << 16;   // any other n_fft: direct O(n_fft^2) DFT

}  // namespace

extern "C" int b2l_stft_f64(b2l_ctx* c, const double* d_y, int64_t n_clips, int64_t n, int64_t y_stride, int32_t n_fft,
                            int32_t hop, int32_t center, int32_t pad_mode, const double* h_window, void* d_out) {
  if (!c || !h_window) return fail(B2L_ERR_INVALID, "NULL argument");
  if (n_fft < 2 || hop < 1 || n_clips < 0 || n < 0 || y_stride < n) return fail(B2L_ERR_INVALID, "bad geometry");
  if (n > 0x7fffffffLL) return fail(B2L_ERR_UNSUPPORTED, "clips longer than 2^31-1 samples are not supported");
  const long long padded = n + (center ? 2LL * (n_fft / 2) : 0);
  if (padded < n_fft) return fail(B2L_ERR_INVALID, "n_fft=%d is too large for input signal of length=%lld", n_fft, (long long)n);
  const long long T = 1 + (padded - n_fft) / hop;
  if (n_clips == 0) return B2L_OK;
  if (!d_y || !d_out) return fail(B2L_ERR_INVALID, "NULL device pointer");
  if (n_clips * T > 0x7fffffffLL) return fail(B2L_ERR_UNSUPPORTED, "float64 stft: more than 2^31-1 frames in one call");
  DeviceGuard g(c->device);
  cudaStream_t st = c->stream;
  const int l2 = ilog2_exact(n_fft);
  const bool fft = l2 >= 2 && n_fft <= kMaxFft64;
  if (!fft && n_fft > kMaxDft64) return fail(B2L_ERR_UNSUPPORTED, "float64 stft: n_fft=%d (direct DFT path is limited to %d)", n_fft, kMaxDft64);
  std::vector<double2> tw = f64_twiddles(n_fft, fft ? n_fft / 2 + 1 : n_fft);
  Temp d_tw(st), d_win(st), d_z(st);
  CUDA_TRY(upload(d_tw, tw.data(), tw.size()));
  CUDA_TRY(upload(d_win, h_window, (size_t)n_fft));
  F64FwdArgs a;
  memset(&a, 0, sizeof(a));
  a.y = d_y;
  a.y_stride = y_stride;
  a.n = (int)n;
  a.n_clips = (int)n_clips;
  a.n_fft = n_fft;
  a.hop = hop;
  a.pad = center ? n_fft / 2 : 0;
  a.pad_mode = pad_mode;
  a.n_frames = (int)T;
  a.log2m = fft ? l2 - 1 : 0;
  a.window = (const double*)d_win.p;
  a.tw = (const double2*)d_tw.p;
  a.out = (double2*)d_out;
  a.status = c->d_status;
  size_t smem = fft ? (size_t)(n_fft / 2) * sizeof(double2) : (size_t)n_fft * sizeof(double);
  if (smem > 128 * 1024) {   // work area in global memory (L2 resident), one slice per frame
    CUDA_TRY(d_z.alloc((size_t)n_clips * (size_t)T * smem));
    a.zscratch = (double2*)d_z.p;
    smem = 0;
  }
  int rc = blocks_per_sm(c, stft64_kernel, 256, smem, nullptr);
  return rc ? rc : launch(c, stft64_kernel, (unsigned)(n_clips * T), 256, smem, a);
}

extern "C" int b2l_istft_f64(b2l_ctx* c, const void* d_D, int64_t n_clips, int64_t n_frames_stored, int64_t n_frames_used,
                             int32_t n_fft, int32_t hop, int32_t center, const double* h_window, const double* h_inv_wss,
                             int64_t out_len, double* d_y, int64_t y_stride) {
  if (!c || !h_window || !h_inv_wss) return fail(B2L_ERR_INVALID, "NULL argument");
  if (n_fft < 2 || hop < 1 || n_clips < 0 || n_frames_used < 1 || n_frames_used > n_frames_stored || out_len < 0 || y_stride < out_len)
    return fail(B2L_ERR_INVALID, "bad istft geometry");
  if (n_clips == 0 || out_len == 0) return B2L_OK;
  if (!d_D || !d_y) return fail(B2L_ERR_INVALID, "NULL device pointer");
  if (n_clips * n_frames_used > 0x7fffffffLL || out_len > 0x7fffffffLL)
    return fail(B2L_ERR_UNSUPPORTED, "float64 istft: batch too large for one call");
  DeviceGuard g(c->device);
  cudaStream_t st = c->stream;
  const int l2 = ilog2_exact(n_fft);
  const bool fft = l2 >= 2 && n_fft <= kMaxFft64;
  if (!fft && n_fft > kMaxDft64) return fail(B2L_ERR_UNSUPPORTED, "float64 istft: n_fft=%d (direct DFT path is limited to %d)", n_fft, kMaxDft64);
  const int F = n_fft / 2 + 1;
  std::vector<double2> tw = f64_twiddles(n_fft, fft ? n_fft / 2 + 1 : n_fft);
  Temp d_tw(st), d_win(st), d_wss(st), d_frames(st), d_z(st);
  CUDA_TRY(upload(d_tw, tw.data(), tw.size()));
  CUDA_TRY(upload(d_win, h_window, (size_t)n_fft));
  CUDA_TRY(upload(d_wss, h_inv_wss, (size_t)out_len));
  CUDA_TRY(d_frames.alloc((size_t)n_clips * (size_t)n_frames_used * (size_t)n_fft * sizeof(double)));
  F64InvArgs a;
  memset(&a, 0, sizeof(a));
  a.D = (const double2*)d_D;
  a.d_clip_stride = (long long)n_frames_stored * F;
  a.n_clips = (int)n_clips;
  a.n_frames = (int)n_frames_used;
  a.n_fft = n_fft;
  a.hop = hop;
  a.start = center ? n_fft / 2 : 0;
  a.out_len = (int)out_len;
  a.log2m = fft ? l2 - 1 : 0;
  a.window = (const double*)d_win.p;
  a.tw = (const double2*)d_tw.p;
  a.frames = (double*)d_frames.p;
  a.inv_wss = (const double*)d_wss.p;
  a.y = d_y;
  a.y_stride = y_stride;
  size_t smem = fft ? (size_t)(n_fft / 2) * sizeof(double2) : (size_t)F * sizeof(double2);
  if (smem > 128 * 1024) {
    CUDA_TRY(d_z.alloc((size_t)n_clips * (size_t)n_frames_used * smem));
    a.zscratch = (double2*)d_z.p;
    smem = 0;
  }
  int rc = blocks_per_sm(c, istft64_frames_kernel, 256, smem, nullptr);
  if (rc || (rc = launch(c, istft64_frames_kernel, (unsigned)(n_clips * n_frames_used), 256, smem, a))) return rc;
  return for_clip_slices(n_clips, [&](int64_t c0, int64_t m) {
    F64InvArgs s = a;
    s.frames += c0 * n_frames_used * n_fft;
    s.y += c0 * y_stride;
    const dim3 grid((unsigned)row_blocks(out_len, 256, 8LL * c->sm_count, m), (unsigned)m);
    return launch(c, ola64_kernel, grid, 256, 0, s);
  });
}

extern "C" int b2l_f64_abs_pow(b2l_ctx* c, const void* d_D, int64_t n, double power, double* d_S) {
  if (!c || !d_D || !d_S) return fail(B2L_ERR_INVALID, "NULL argument");
  if (n <= 0) return B2L_OK;
  DeviceGuard g(c->device);
  return launch(c, abs_pow64_kernel, (unsigned)grid_stride_blocks(n, 256, 16LL * c->sm_count), 256, 0,
                (const double2*)d_D, n, power, d_S);
}

extern "C" int b2l_f64_mel(b2l_ctx* c, const double* d_S, int64_t n_clips, int64_t n_frames, int32_t n_bins,
                           const float* h_mel, int32_t n_mels, double* d_out) {
  if (!c || !d_S || !h_mel || !d_out) return fail(B2L_ERR_INVALID, "NULL argument");
  if (n_clips <= 0 || n_frames <= 0 || n_mels <= 0) return B2L_OK;
  DeviceGuard g(c->device);
  cudaStream_t st = c->stream;
  std::vector<MelBand> bands((size_t)n_mels);
  std::vector<float> w;
  for (int m = 0; m < n_mels; ++m) {
    const float* row = h_mel + (size_t)m * n_bins;
    int lo = 0, hi = n_bins - 1;
    while (lo < n_bins && row[lo] == 0.0f) ++lo;
    while (hi >= lo && row[hi] == 0.0f) --hi;
    MelBand b;
    b.off = (int)w.size();
    b.pad = 0;
    if (lo > hi) {
      b.lo = 0;
      b.len = 0;
    } else {
      b.lo = lo;
      b.len = hi - lo + 1;
      w.insert(w.end(), row + lo, row + hi + 1);
    }
    bands[(size_t)m] = b;
  }
  if (w.empty()) w.push_back(0.0f);
  Temp d_w(st), d_b(st);
  CUDA_TRY(upload(d_w, w.data(), w.size()));
  CUDA_TRY(upload(d_b, bands.data(), bands.size()));
  const long long rows = n_clips * n_frames;
  const long long blocks = (rows * 32 + 255) / 256;
  if (blocks > 0x7fffffffLL) return fail(B2L_ERR_UNSUPPORTED, "float64 mel: too many frames in one call");
  return launch(c, mel64_kernel, (unsigned)blocks, 256, 0, d_S, (const float*)d_w.p, (const MelBand*)d_b.p, n_mels, n_bins,
                (int)n_frames, rows, d_out);
}

extern "C" int b2l_f64_db(b2l_ctx* c, const double* d_in, int64_t n_clips, int64_t per_clip, double amin, double ref_value,
                          double top_db, double* d_out) {
  if (!c || !d_in || !d_out) return fail(B2L_ERR_INVALID, "NULL argument");
  if (!(amin > 0.0)) return fail(B2L_ERR_INVALID, "amin must be strictly positive");
  if (n_clips <= 0 || per_clip <= 0) return B2L_OK;
  DeviceGuard g(c->device);
  cudaStream_t st = c->stream;
  Temp d_max(st);   // one maximum per clip of the whole batch
  CUDA_TRY(d_max.alloc((size_t)n_clips * sizeof(unsigned long long)));
  CUDA_TRY(cudaMemsetAsync(d_max.p, 0, (size_t)n_clips * sizeof(unsigned long long), st));
  unsigned long long* clip_max = (unsigned long long*)d_max.p;
  const double db_sub = 10.0 * log10(fmax(amin, fabs(ref_value)));
  return for_clip_slices(n_clips, [&](int64_t c0, int64_t m) {
    const dim3 grid((unsigned)row_blocks(per_clip, 256, 8LL * c->sm_count, m), (unsigned)m);
    int rc = launch(c, db64_kernel, grid, 256, 0, d_in + c0 * per_clip, per_clip, amin, db_sub, d_out + c0 * per_clip,
                    clip_max + c0);
    if (rc == B2L_OK && top_db >= 0.0)
      rc = launch(c, db64_clamp_kernel, grid, 256, 0, d_out + c0 * per_clip, per_clip, top_db, clip_max + c0);
    return rc;
  });
}

extern "C" int b2l_f64_dct(b2l_ctx* c, const double* d_L, int64_t n_clips, int32_t n_mels, int64_t n_frames,
                           const double* h_dct, int32_t n_mfcc, double* d_out) {
  if (!c || !d_L || !h_dct || !d_out) return fail(B2L_ERR_INVALID, "NULL argument");
  if (n_clips <= 0 || n_frames <= 0 || n_mfcc <= 0) return B2L_OK;
  DeviceGuard g(c->device);
  cudaStream_t st = c->stream;
  const size_t smem = (size_t)n_mfcc * n_mels * sizeof(double);
  if (smem > c->smem_optin) return fail(B2L_ERR_UNSUPPORTED, "float64 dct: matrix does not fit in shared memory");
  Temp d_dct(st);
  CUDA_TRY(upload(d_dct, h_dct, (size_t)n_mfcc * n_mels));
  if (int rc = blocks_per_sm(c, dct64_kernel, 128, smem, nullptr)) return rc;
  return for_clip_slices(n_clips, [&](int64_t c0, int64_t m) {
    return launch(c, dct64_kernel, dim3((unsigned)((n_frames + 127) / 128), (unsigned)m), 128, smem,
                  d_L + c0 * n_mels * n_frames, (const double*)d_dct.p, n_mels, n_mfcc, (int)n_frames,
                  d_out + c0 * n_mfcc * n_frames);
  });
}
