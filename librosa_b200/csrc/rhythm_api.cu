// rhythm_api.cu — C ABI of the rhythm features (rhythm_kernels.cuh): librosa.feature.tempogram and the tempo
// estimate on top of it (librosa/feature/rhythm.py:38-470).  The only unit that includes rhythm_kernels.cuh.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "internal.h"
#include "rhythm_kernels.cuh"

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
