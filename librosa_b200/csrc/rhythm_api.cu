// rhythm_api.cu — C ABI of the rhythm features (rhythm_kernels.cuh): librosa.feature.tempogram and the tempo
// estimate on top of it (librosa/feature/rhythm.py:38-470), and librosa.beat.beat_track's tracker
// (beat_kernels.cuh, librosa/beat.py:510-742), and librosa.onset.onset_detect's normaliser, peak picker and backtracker
// (onset_kernels.cuh).  The only unit that includes rhythm_kernels.cuh, beat_kernels.cuh and onset_kernels.cuh.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "internal.h"
#include "rhythm_kernels.cuh"
#include "beat_kernels.cuh"
#include "onset_kernels.cuh"

using namespace b2l;

namespace {
const int kMaxTempogramWin = 4096;   // N = 8192 points: 64 KB of packed transform in shared memory
}

extern "C" int b2l_tempogram(b2l_ctx* c, const b2l_tempogram_desc* d, const void* d_env, int64_t n_rows, int64_t n,
                             const double* d_window, double* d_out) {
  if (!c || !d) return fail(B2L_ERR_INVALID, "NULL argument");
  const int W = d->win_length;
  if (W < 1) return fail(B2L_ERR_INVALID, "win_length must be a positive integer");
  if (W > kMaxTempogramWin)
    return fail(B2L_ERR_UNSUPPORTED, "tempogram: win_length=%d; the GPU kernel supports windows up to %d onset frames",
                W, kMaxTempogramWin);
  if (d->norm < B2L_TG_NORM_NONE || d->norm > B2L_TG_NORM_P) return fail(B2L_ERR_INVALID, "Unsupported norm: %d", d->norm);
  if (d->norm == B2L_TG_NORM_P && !(d->norm_p > 0.0)) return fail(B2L_ERR_INVALID, "norm exponent must be positive");
  if (n_rows < 0 || n < 0) return fail(B2L_ERR_INVALID, "bad envelope geometry");
  if (n > 0x7fffffffLL) return fail(B2L_ERR_UNSUPPORTED, "envelopes longer than 2^31-1 frames are not supported");
  const int pad = d->center ? W / 2 : 0;
  if (n + 2LL * pad < W) return fail(B2L_ERR_INVALID, "Input is too short (n=%lld) for frame_length=%d", n + 2LL * pad, W);
  const long long T = d->center ? n : n - W + 1;
  if (n_rows == 0 || T == 0) return B2L_OK;
  if (n_rows * T > 0x7fffffffLL) return fail(B2L_ERR_UNSUPPORTED, "tempogram: more than 2^31-1 frames in one call");
  if (!d_env || !d_window || !d_out) return fail(B2L_ERR_INVALID, "NULL device pointer");
  DeviceGuard g(c->device);
  int log2n = 2;                                      // N >= 4 keeps the packed transform at least 2 points long
  while ((1 << log2n) < 2 * W - 1) ++log2n;
  const int N = 1 << log2n, M = N / 2;
  const std::vector<double2> tw = f64_twiddles(N, M + 1);
  Temp d_tw(c->stream);
  CUDA_TRY(upload(d_tw, tw.data(), tw.size()));
  TempogramArgs a;
  memset(&a, 0, sizeof(a));
  a.x = d_env;
  a.n = (int)n;
  a.win = W;
  a.pad = pad;
  a.n_frames = (int)T;
  a.log2m = log2n - 1;
  a.window = d_window;
  a.tw = (const double2*)d_tw.p;
  a.norm = d->norm;
  a.norm_p = d->norm_p;
  a.out = d_out;
  a.status = c->d_status;
  const int threads = std::min(1024, std::max(32, M / 2));
  const size_t smem = tempogram_smem_doubles(a.log2m, W) * sizeof(double);
  auto fn = d->env_f64 ? tempogram_kernel<double> : tempogram_kernel<float>;
  int occ = 0, rc;
  if ((rc = blocks_per_sm(c, fn, threads, smem, &occ))) return rc;
  if (occ < 1) return fail(B2L_ERR_UNSUPPORTED, "tempogram: win_length=%d does not fit on an SM (smem %zu)", W, smem);
  return launch(c, fn, (unsigned)(n_rows * T), threads, smem, a);
}

extern "C" int b2l_tempo(b2l_ctx* c, const b2l_tempo_desc* d, const void* d_tg, int64_t n_rows,
                         const double* d_logprior, const double* d_bpms, double* d_out) {
  if (!c || !d) return fail(B2L_ERR_INVALID, "NULL argument");
  if (d->n_lags < 1) return fail(B2L_ERR_INVALID, "n_lags=%d must be positive", d->n_lags);
  if (n_rows < 0 || d->n_frames < 0) return fail(B2L_ERR_INVALID, "bad tempogram geometry");
  if (n_rows == 0 || (!d->mean && d->n_frames == 0)) return B2L_OK;
  if (d->n_frames > 0x7fffffffLL) return fail(B2L_ERR_UNSUPPORTED, "tempo: more than 2^31-1 frames per row");
  if (!d_tg || !d_logprior || !d_bpms || !d_out) return fail(B2L_ERR_INVALID, "NULL device pointer");
  DeviceGuard g(c->device);
  TempoArgs a;
  a.tg = d_tg;
  a.rows = n_rows;
  a.n_lags = d->n_lags;
  a.n_frames = (int)d->n_frames;
  a.row_stride = d->row_stride;
  a.lag_stride = d->lag_stride;
  a.frame_stride = d->frame_stride;
  a.logprior = d_logprior;
  a.bpms = d_bpms;
  a.out = d_out;
  if (d->mean) {
    if (n_rows > 0x7fffffffLL) return fail(B2L_ERR_UNSUPPORTED, "tempo: more than 2^31-1 rows in one call");
    auto fn = d->tg_f64 ? tempo_mean_kernel<double> : tempo_mean_kernel<float>;
    return launch(c, fn, (unsigned)n_rows, 256, 0, a);
  }
  const long long blocks = (n_rows * d->n_frames + 7) / 8;   // 8 warps per CTA, one per (row, frame)
  if (blocks > 0x7fffffffLL) return fail(B2L_ERR_UNSUPPORTED, "tempo: too many frames in one call");
  auto fn = d->tg_f64 ? tempo_frames_kernel<double> : tempo_frames_kernel<float>;
  return launch(c, fn, (unsigned)blocks, 256, 0, a);
}

extern "C" int b2l_beat_track(b2l_ctx* c, const b2l_beat_desc* d, const void* d_env, int64_t n_clips, int64_t n,
                              void* d_localscore, void* d_cumscore, int32_t* d_backlink, uint8_t* d_beats,
                              void* d_sparse, int64_t* d_count) {
  if (!c || !d) return fail(B2L_ERR_INVALID, "NULL argument");
  if (n_clips < 0 || n < 0) return fail(B2L_ERR_INVALID, "bad envelope geometry");
  if (d->n_fpb != 1 && d->n_fpb != n) return fail(B2L_ERR_INVALID, "n_fpb=%d must be 1 or n=%lld", d->n_fpb, (long long)n);
  if (d->units < B2L_BEAT_FRAMES || d->units > B2L_BEAT_TIME) return fail(B2L_ERR_INVALID, "unknown units %d", d->units);
  if (d_sparse && (n_clips != 1 || !d_count)) return fail(B2L_ERR_INVALID, "a sparse beat list needs one clip and a count");
  if (n_clips == 0 || n == 0) {
    if (d_count) CUDA_TRY(cudaMemsetAsync(d_count, 0, sizeof(int64_t), c->stream));
    return B2L_OK;
  }
  if (n > 0x7fffffffLL) return fail(B2L_ERR_UNSUPPORTED, "beat_track: envelopes longer than 2^31-1 frames");
  if (n_clips > 0x7fffffffLL) return fail(B2L_ERR_UNSUPPORTED, "beat_track: more than 2^31-1 clips in one call");
  if (!d_env || !d_beats || !d->d_fpb || !d->d_logfpb || !d->d_woff || !d->d_wtab || !d->d_logd)
    return fail(B2L_ERR_INVALID, "NULL device pointer");
  DeviceGuard g(c->device);
  const size_t elem = d->env_f64 ? sizeof(double) : sizeof(float);
  const size_t row = (size_t)n_clips * (size_t)n;
  Temp t_ls(c->stream), t_cum(c->stream), t_back(c->stream), t_scratch(c->stream);
  if (!d_localscore) { CUDA_TRY(t_ls.alloc(row * elem)); d_localscore = t_ls.p; }
  if (!d_cumscore) { CUDA_TRY(t_cum.alloc(row * (d->dp_f64 ? sizeof(double) : sizeof(float)))); d_cumscore = t_cum.p; }
  if (!d_backlink) { CUDA_TRY(t_back.alloc(row * sizeof(int32_t))); d_backlink = (int32_t*)t_back.p; }
  CUDA_TRY(t_scratch.alloc(row * sizeof(double)));
  b2l_beat::BeatArgs a;
  memset(&a, 0, sizeof(a));
  a.env = d_env;
  a.n = (int)n;
  a.tv = d->n_fpb != 1;
  a.fpb = d->d_fpb;
  a.logfpb = d->d_logfpb;
  a.woff = d->d_woff;
  a.wtab = d->d_wtab;
  a.logd = d->d_logd;
  a.tightness = (double)d->tightness;
  a.trim = d->trim;
  a.localscore = d_localscore;
  a.cumscore = d_cumscore;
  a.backlink = d_backlink;
  a.scratch = t_scratch.p;
  a.beats = d_beats;
  a.units = d->units;
  a.sparse = d_sparse;
  a.count = (long long*)d_count;
  a.hop_length = d->hop_length;
  a.sr = d->sr;
  if (d->env_f64 && !d->dp_f64) return fail(B2L_ERR_INVALID, "a float64 envelope needs the float64 DP");
  auto fn = d->env_f64 ? b2l_beat::beat_track_kernel<double, double>
                       : d->dp_f64 ? b2l_beat::beat_track_kernel<float, double> : b2l_beat::beat_track_kernel<float, float>;
  return launch(c, fn, (unsigned)n_clips, 256, 0, a);
}

extern "C" int b2l_any_nonzero(b2l_ctx* c, const void* d_x, int64_t n, int32_t f64, int32_t* d_flag) {
  if (!c || !d_flag) return fail(B2L_ERR_INVALID, "NULL argument");
  if (n < 0) return fail(B2L_ERR_INVALID, "negative length");
  DeviceGuard g(c->device);
  CUDA_TRY(cudaMemsetAsync(d_flag, 0, sizeof(int32_t), c->stream));
  if (n == 0) return B2L_OK;
  if (!d_x) return fail(B2L_ERR_INVALID, "NULL device pointer");
  const unsigned blocks = (unsigned)grid_stride_blocks(n, 256, 4LL * c->sm_count);
  if (f64) return launch(c, b2l_beat::any_nonzero_kernel<double>, blocks, 256, 0, (const double*)d_x, (long long)n, d_flag);
  return launch(c, b2l_beat::any_nonzero_kernel<float>, blocks, 256, 0, (const float*)d_x, (long long)n, d_flag);
}

extern "C" int b2l_plp_select(b2l_ctx* c, const b2l_plp_desc* d, void* d_ftgram, int64_t n_frames) {
  if (!c || !d) return fail(B2L_ERR_INVALID, "NULL argument");
  if (d->n_bins < 1 || n_frames < 0) return fail(B2L_ERR_INVALID, "bad Fourier tempogram geometry");
  if (n_frames == 0) return B2L_OK;
  if (!d_ftgram || !d->d_keep) return fail(B2L_ERR_INVALID, "NULL device pointer");
  const long long blocks = (n_frames + 7) / 8;   // 8 warps per CTA, one per frame
  if (blocks > 0x7fffffffLL) return fail(B2L_ERR_UNSUPPORTED, "plp: too many frames in one call");
  DeviceGuard g(c->device);
  if (d->c128)
    return launch(c, b2l_beat::plp_select_kernel<double2>, (unsigned)blocks, 256, 0, (double2*)d_ftgram,
                  (long long)n_frames, d->n_bins, d->d_keep, d->d_logprior, d->sqrt_tiny);
  return launch(c, b2l_beat::plp_select_kernel<float2>, (unsigned)blocks, 256, 0, (float2*)d_ftgram,
                (long long)n_frames, d->n_bins, d->d_keep, d->d_logprior, d->sqrt_tiny);
}

extern "C" int b2l_plp_finish(b2l_ctx* c, void* d_pulse, int64_t n_rows, int64_t n, int32_t f64) {
  if (!c) return fail(B2L_ERR_INVALID, "NULL argument");
  if (n_rows < 0 || n < 0) return fail(B2L_ERR_INVALID, "bad pulse geometry");
  if (n_rows == 0 || n == 0) return B2L_OK;
  if (n_rows > 0x7fffffffLL || n > 0x7fffffffLL) return fail(B2L_ERR_UNSUPPORTED, "plp: batch too large");
  if (!d_pulse) return fail(B2L_ERR_INVALID, "NULL device pointer");
  DeviceGuard g(c->device);
  if (f64) return launch(c, b2l_beat::plp_finish_kernel<double>, (unsigned)n_rows, 256, 0, (double*)d_pulse, (int)n,
                         c->d_status);
  return launch(c, b2l_beat::plp_finish_kernel<float>, (unsigned)n_rows, 256, 0, (float*)d_pulse, (int)n,
                c->d_status);
}

extern "C" int b2l_onset_normalize(b2l_ctx* c, const void* d_x, int64_t n_rows, int64_t n, int32_t f64, double tiny,
                                   void* d_out, int64_t* d_flags) {
  if (!c || !d_flags) return fail(B2L_ERR_INVALID, "NULL argument");
  if (n_rows < 0 || n < 0) return fail(B2L_ERR_INVALID, "bad envelope geometry");
  if (n > 0x7fffffffLL) return fail(B2L_ERR_UNSUPPORTED, "onset_detect: envelopes of 2^31 frames or more");
  if (n_rows > 0x7fffffffLL) return fail(B2L_ERR_UNSUPPORTED, "onset_detect: more than 2^31-1 rows in one call");
  DeviceGuard g(c->device);
  CUDA_TRY(cudaMemsetAsync(d_flags, 0, 2 * sizeof(int64_t), c->stream));
  if (n_rows == 0 || n == 0) return B2L_OK;
  if (!d_x) return fail(B2L_ERR_INVALID, "NULL device pointer");
  long long* flags = (long long*)d_flags;
  if (f64)
    return launch(c, b2l_onset::onset_normalize_kernel<double>, (unsigned)n_rows, 256, 0, (const double*)d_x, (int)n,
                  tiny, (double*)d_out, flags);
  return launch(c, b2l_onset::onset_normalize_kernel<float>, (unsigned)n_rows, 256, 0, (const float*)d_x, (int)n,
                (float)tiny, (float*)d_out, flags);
}

extern "C" int b2l_peak_pick(b2l_ctx* c, const b2l_peak_desc* d, const void* d_x, int64_t n_rows, int64_t n,
                             const int64_t* d_flags, uint8_t* d_dense, void* d_sparse, int64_t* d_count) {
  if (!c || !d) return fail(B2L_ERR_INVALID, "NULL argument");
  if (n_rows < 0 || n < 0) return fail(B2L_ERR_INVALID, "bad envelope geometry");
  if (d->pre_max < 0 || d->pre_avg < 0 || d->wait < 0 || d->post_max < 1 || d->post_avg < 1)
    return fail(B2L_ERR_INVALID, "peak_pick: window lengths out of range");
  if (d->method < B2L_PEAK_GREEDY || d->method > B2L_PEAK_DP_VALUE) return fail(B2L_ERR_INVALID, "unknown method %d", d->method);
  if (d->units < B2L_BEAT_FRAMES || d->units > B2L_BEAT_TIME) return fail(B2L_ERR_INVALID, "unknown units %d", d->units);
  if (d_sparse && (n_rows != 1 || !d_count)) return fail(B2L_ERR_INVALID, "a sparse peak list needs one row and a count");
  if (n > 0x7fffffffLL) return fail(B2L_ERR_UNSUPPORTED, "peak_pick: rows of 2^31 frames or more");
  if (n_rows > 0x7fffffffLL) return fail(B2L_ERR_UNSUPPORTED, "peak_pick: more than 2^31-1 rows in one call");
  DeviceGuard g(c->device);
  if (n_rows == 0 || n == 0) {
    if (d_count) CUDA_TRY(cudaMemsetAsync(d_count, 0, sizeof(int64_t), c->stream));
    return B2L_OK;
  }
  if (!d_x) return fail(B2L_ERR_INVALID, "NULL device pointer");
  b2l_onset::PeakArgs a;
  memset(&a, 0, sizeof(a));
  auto clamp = [n](int64_t v) { return (long long)std::min<int64_t>(v, n); };   // longer windows clip the same way
  a.x = d_x;
  a.n = (int)n;
  a.pre_max = clamp(d->pre_max);
  a.post_max = clamp(d->post_max);
  a.pre_avg = clamp(d->pre_avg);
  a.post_avg = clamp(d->post_avg);
  a.wait = clamp(d->wait);
  a.delta = d->delta;
  a.flags = (const long long*)d_flags;
  a.dense = d_dense;
  a.sparse = d_sparse;
  a.count = (long long*)d_count;
  a.units = d->units;
  a.hop_length = d->hop_length;
  a.sr = d->sr;
  Temp t_scratch(c->stream), t_marks(c->stream);
  if (d->method != B2L_PEAK_GREEDY) {
    CUDA_TRY(t_scratch.alloc((size_t)n_rows * 2 * (size_t)(n + 1) * sizeof(double)));
    CUDA_TRY(t_marks.alloc((size_t)n_rows * (size_t)n));
    a.scratch = (double*)t_scratch.p;
    a.marks = (uint8_t*)t_marks.p;
  }
  using namespace b2l_onset;
  void (*fn)(PeakArgs);
  if (d->method == B2L_PEAK_GREEDY) fn = d->f64 ? peak_pick_kernel<double, kGreedy> : peak_pick_kernel<float, kGreedy>;
  else if (d->method == B2L_PEAK_DP_COUNT) fn = d->f64 ? peak_pick_kernel<double, kDpCount> : peak_pick_kernel<float, kDpCount>;
  else fn = d->f64 ? peak_pick_kernel<double, kDpValue> : peak_pick_kernel<float, kDpValue>;
  return launch(c, fn, (unsigned)n_rows, 256, 0, a);
}

extern "C" int b2l_onset_backtrack(b2l_ctx* c, const void* d_energy, int64_t n, int32_t f64, const int64_t* d_events,
                                   int64_t n_events, const int64_t* d_count, int32_t units, int32_t hop_length,
                                   double sr, void* d_out) {
  if (!c) return fail(B2L_ERR_INVALID, "NULL argument");
  if (n < 0 || n_events < 0) return fail(B2L_ERR_INVALID, "bad geometry");
  if (units < B2L_BEAT_FRAMES || units > B2L_BEAT_TIME) return fail(B2L_ERR_INVALID, "unknown units %d", units);
  if (n > 0x7fffffffLL) return fail(B2L_ERR_UNSUPPORTED, "onset_backtrack: energy of 2^31 frames or more");
  if (n_events == 0) return B2L_OK;
  if ((n && !d_energy) || !d_events || !d_out) return fail(B2L_ERR_INVALID, "NULL device pointer");
  DeviceGuard g(c->device);
  Temp t_last(c->stream);
  CUDA_TRY(t_last.alloc((size_t)n * sizeof(int)));
  const long long* ev = (const long long*)d_events;
  const long long* cnt = (const long long*)d_count;
  if (f64)
    return launch(c, b2l_onset::onset_backtrack_kernel<double>, 1u, 1024, 0, (const double*)d_energy, (int)n, ev,
                  (long long)n_events, cnt, (int*)t_last.p, (int)units, (int)hop_length, sr, d_out, c->d_status);
  return launch(c, b2l_onset::onset_backtrack_kernel<float>, 1u, 1024, 0, (const float*)d_energy, (int)n, ev,
                (long long)n_events, cnt, (int*)t_last.p, (int)units, (int)hop_length, sr, d_out, c->d_status);
}
