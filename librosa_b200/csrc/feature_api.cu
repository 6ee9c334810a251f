// feature_api.cu — C ABI of the plan-free kernels over spectrograms and signals (feat_kernels.cuh, include/b2l.h):
// spectral statistics of a stored spectrogram, time-domain framings, resampling, power_to_db, onset strength, pcen,
// spectral contrast, piptrack, normalisation, HPSS, reassignment, phase vocoder, Griffin-Lim update and transpose.
#include <cuda_runtime.h>
#include <math.h>
#include <string.h>

#include <algorithm>

#include "feat_kernels.cuh"
#include "internal.h"

using namespace b2l;

// ------------------------------------------------------------------ frame-wise spectral statistics / framings
int b2l::check_stats_desc(const b2l_stats_desc* d, StatsParams* sp) {
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
  StatsParams sp;
  int rc = check_stats_desc(d, &sp);
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
  return launch(c, stats_kernel, (unsigned)grid, nw * 32, smem, d_S, rows, (int)n_frames, n_bins, d_freq, sp, d_out,
                c->d_status);
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

// The checks the two onset entry points share, in order: lag, max_size, pad_width, the channel count
// (min_channels .. 32, else `channels_msg`), the batch extents, then the channel boundaries.  *a comes back filled, or
// with a->T == 0 for an empty batch (nothing to launch).
static int onset_args(const b2l_onset_desc* d, int min_channels, const char* channels_msg, int64_t n_clips,
                      int64_t n_rows, int64_t n_frames, OnsetArgs* a) {
  memset(a, 0, sizeof(*a));
  if (d->lag < 1) return fail(B2L_ERR_INVALID, "lag=%d must be a positive integer", d->lag);
  if (d->max_size < 1) return fail(B2L_ERR_INVALID, "max_size=%d must be a positive integer", d->max_size);
  if (d->pad_width < 0) return fail(B2L_ERR_INVALID, "negative pad_width");
  if (d->n_channels < min_channels || d->n_channels > 32) return fail(B2L_ERR_UNSUPPORTED, "%s", channels_msg);
  if (n_clips <= 0 || n_rows <= 0 || n_frames <= 0) return B2L_OK;
  if (n_clips > kMaxGridY || n_rows > 0x7fffffffLL || n_frames > 0x7fffffffLL)
    return fail(B2L_ERR_UNSUPPORTED, "onset: batch too large");
  for (int i = 0; i <= d->n_channels; ++i) {
    a->bounds[i] = d->bounds[i];
    if (a->bounds[i] < 0 || a->bounds[i] > n_rows || (i > 0 && a->bounds[i] < a->bounds[i - 1]))
      return fail(B2L_ERR_INVALID, "channel boundaries must be non-decreasing row indices");
  }
  a->n_ch = d->n_channels;
  a->lag = d->lag;
  a->max_size = d->max_size;
  a->pad_width = d->pad_width;
  a->n_rows = (int)n_rows;
  a->T = (int)n_frames;
  return B2L_OK;
}

extern "C" int b2l_onset_from_spec(b2l_ctx* c, const b2l_onset_desc* d, const float* d_S, int64_t n_clips,
                                   int64_t n_rows, int64_t n_frames, float* d_out) {
  if (!c || !d || !d_S || !d_out) return fail(B2L_ERR_INVALID, "NULL argument");
  OnsetArgs a;
  int rc = onset_args(d, 0, "at most 32 onset channels", n_clips, n_rows, n_frames, &a);
  if (rc || a.T == 0) return rc;
  DeviceGuard g(c->device);
  rc = launch(c, onset_kernel, dim3((unsigned)((n_frames + 127) / 128), (unsigned)n_clips), 128, 0, d_S, a, d_out);
  if (rc || !d->detrend) return rc;
  const long long rows = (long long)n_clips * (a.n_ch > 0 ? a.n_ch : a.n_rows);
  return launch(c, detrend_kernel, (unsigned)((rows + 127) / 128), 128, 0, d_out, rows, a.T);
}

extern "C" int b2l_onset_median_from_spec(b2l_ctx* c, const b2l_onset_desc* d, const float* d_S, int64_t n_clips,
                                          int64_t n_rows, int64_t n_frames, float* d_out) {
  if (!c || !d || !d_S || !d_out) return fail(B2L_ERR_INVALID, "NULL argument");
  OnsetArgs a;
  int rc = onset_args(d, 1, "1 to 32 onset channels", n_clips, n_rows, n_frames, &a);
  if (rc || a.T == 0) return rc;
  int widest = 0;
  for (int i = 1; i <= a.n_ch; ++i) widest = std::max(widest, a.bounds[i] - a.bounds[i - 1]);
  if (widest > kOnsetMedMaxRows)
    return fail(B2L_ERR_UNSUPPORTED, "onset: median aggregation over a channel of %d rows; the GPU kernel takes up to %d",
                widest, kOnsetMedMaxRows);
  int P = 32;
  while (P < widest) P <<= 1;
  const size_t smem = (size_t)kOnsetMedFrames * (P + 1) * sizeof(float);
  DeviceGuard g(c->device);
  const dim3 grid((unsigned)((n_frames + kOnsetMedFrames - 1) / kOnsetMedFrames), (unsigned)n_clips);
  rc = launch(c, onset_median_kernel, grid, 256, smem, d_S, a, P, d_out);
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
  const long long rows = (long long)n_clips * n_rows;
  if (n_frames > 0x7fffffffLL || n_rows > 0x7fffffffLL || (rows + 127) / 128 > 0x7fffffffLL)
    return fail(B2L_ERR_UNSUPPORTED, "pcen: batch too large");
  DeviceGuard g(c->device);
  const float* ref = d_S;
  if (d->max_size > 1) {
    if (!d_scratch) return fail(B2L_ERR_INVALID, "max_size > 1 needs a scratch buffer of the size of S");
    // rows on grid.y and clips on grid.z: slices of at most 65 535 of each
    const int rc = for_clip_slices(n_clips, [&](int64_t c0, int64_t m) {
      const size_t off = (size_t)c0 * (size_t)n_rows * (size_t)n_frames;
      for (int64_t r0 = 0; r0 < n_rows; r0 += kMaxGridY) {
        const dim3 grid((unsigned)((n_frames + 127) / 128), (unsigned)std::min(kMaxGridY, n_rows - r0), (unsigned)m);
        if (int rc = launch(c, maxfilter_rows_kernel, grid, 128, 0, d_S + off, (int)n_rows, (int)n_frames, d->max_size,
                            (int)r0, d_scratch + off))
          return rc;
      }
      return (int)B2L_OK;
    });
    if (rc) return rc;
    ref = d_scratch;
  }
  PcenArgs a;
  a.gain = d->gain;
  a.bias = d->bias;
  a.power = d->power;
  a.eps = d->eps;
  a.b = d->b;
  a.mode = d->power == 0.0f ? 0 : (d->bias == 0.0f ? 1 : 2);
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
  if (n_frames > 0x7fffffffLL || n_bins > 0x7fffffffLL) return fail(B2L_ERR_UNSUPPORTED, "hpss: batch too large");
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
  const float2* sc = d->mask_only ? nullptr : (const float2*)d_S_complex;
  // complex masked components are float2 elements, masks and real components float
  const size_t out_words = sc ? 2 : 1;
  // frames on grid.y and clips on grid.z: slices of at most 65 535 of each, the frame slice passed as a.t0
  return for_clip_slices(n_clips, [&](int64_t c0, int64_t m) {
    const size_t off = (size_t)c0 * (size_t)n_frames * (size_t)n_bins;
    for (int64_t t0 = 0; t0 < n_frames; t0 += kMaxGridY) {
      a.t0 = (int)t0;
      const dim3 grid((unsigned)((n_bins + 127) / 128), (unsigned)std::min(kMaxGridY, n_frames - t0), (unsigned)m);
      if (int rc = launch(c, kern, grid, 128, 0, d_mag + off, sc ? sc + off : nullptr, a,
                          (float*)d_out_harm + out_words * off, (float*)d_out_perc + out_words * off))
        return rc;
    }
    return (int)B2L_OK;
  });
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
