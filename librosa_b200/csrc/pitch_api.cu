// pitch_api.cu — C ABI of the pitch trackers (pitch_kernels.cuh, include/b2l.h): librosa.yin and librosa.pyin as the
// CMND, yin decision, pyin observation and Viterbi decoding launches; librosa.piptrack and librosa.pitch_tuning.
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <vector>

#include "internal.h"
#include "pitch_kernels.cuh"

using namespace b2l;

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

template <class T>
static int launch_piptrack(b2l_ctx* c, const b2l_piptrack_desc* d, const void* d_S, int64_t n_clips, int32_t F,
                           int64_t n_frames, void* d_pitches, void* d_mags) {
  const size_t per_warp = (size_t)((F + 3) & ~3) * sizeof(T);
  if (per_warp > B2L_PIPTRACK_MAX_ROW_BYTES || per_warp > c->smem_optin)
    return fail(B2L_ERR_UNSUPPORTED, "piptrack: a row of %d bins does not fit in shared memory", F);
  int nw = 8;
  while (nw > 1 && per_warp * nw > c->smem_optin) nw >>= 1;
  const size_t smem = per_warp * nw;
  PiptrackArgs<T> a;
  a.S = (const T*)d_S;
  a.n_rows = n_clips * n_frames;
  a.n_frames = n_frames;
  a.frame_stride = d->layout_c ? 1 : F;
  a.bin_stride = d->layout_c ? n_frames : 1;
  a.F = F;
  a.k_lo = d->k_lo;
  a.k_hi = d->k_hi;
  a.abs_mode = d->abs_mode;
  a.sign = nullptr;
  a.ref_frame = d->ref_frame;
  a.thr_wide = d->thr_wide;
  a.threshold = d->threshold;
  a.ref_abs = d->ref_abs;
  a.sr = d->sr;
  a.n_fft = d->n_fft;
  a.pitches = (T*)d_pitches;
  a.mags = (T*)d_mags;
  if (d->abs_mode == 2) {   // S.min() < 0, decided on the device: one pass sets the sign word the main kernel reads
    if (int rc = ensure_scratch(c, sizeof(unsigned))) return rc;
    unsigned* word = reinterpret_cast<unsigned*>(c->d_scratch);
    CUDA_TRY(cudaMemsetAsync(word, 0, sizeof(unsigned), c->stream));
    const long long n = a.n_rows * F;
    if (int rc = launch(c, sign_scan_kernel<T>, (unsigned)grid_stride_blocks(n, 256, 32LL * c->sm_count), 256, 0,
                        a.S, n, word))
      return rc;
    a.sign = word;
  }
  long long grid = 0;
  if (int rc = resident_grid(c, piptrack_kernel<T>, nw * 32, smem, (a.n_rows + nw - 1) / nw, &grid)) return rc;
  if (!grid) return fail(B2L_ERR_UNSUPPORTED, "piptrack: a row of %d bins does not fit on an SM", F);
  return launch(c, piptrack_kernel<T>, (unsigned)grid, nw * 32, smem, a);
}

extern "C" int b2l_piptrack(b2l_ctx* c, const b2l_piptrack_desc* d, const void* d_S, int64_t n_clips, int32_t n_bins,
                            int64_t n_frames, void* d_pitches, void* d_mags) {
  if (!c || !d) return fail(B2L_ERR_INVALID, "NULL argument");
  if (n_clips < 0 || n_frames < 0 || n_bins < 2) return fail(B2L_ERR_INVALID, "piptrack: bad geometry");
  if (d->k_lo < 0 || d->k_hi > n_bins) return fail(B2L_ERR_INVALID, "piptrack: bad bin range");
  if (d->abs_mode < 0 || d->abs_mode > 2) return fail(B2L_ERR_INVALID, "piptrack: bad abs_mode %d", d->abs_mode);
  if (n_clips == 0 || n_frames == 0) return B2L_OK;
  if (!d_S || !d_pitches || !d_mags) return fail(B2L_ERR_INVALID, "NULL device pointer");
  DeviceGuard g(c->device);
  return d->f64 ? launch_piptrack<double>(c, d, d_S, n_clips, n_bins, n_frames, d_pitches, d_mags)
                : launch_piptrack<float>(c, d, d_S, n_clips, n_bins, n_frames, d_pitches, d_mags);
}

extern "C" int b2l_pitch_tuning(b2l_ctx* c, const void* d_f, int64_t n, int32_t f64, double bins_per_octave,
                                int32_t n_bins, const double* h_edges, uint64_t* h_counts) {
  if (!c || !h_edges || !h_counts) return fail(B2L_ERR_INVALID, "NULL argument");
  if (n_bins < 1 || n_bins > 2048) return fail(B2L_ERR_INVALID, "pitch_tuning: %d bins; 1 .. 2048 are supported", n_bins);
  if (n < 0) return fail(B2L_ERR_INVALID, "pitch_tuning: bad length");
  for (int i = 0; i <= n_bins; ++i) h_counts[i] = 0;
  if (n == 0) return B2L_OK;
  if (!d_f) return fail(B2L_ERR_INVALID, "NULL device pointer");
  DeviceGuard g(c->device);
  if (int rc = ensure_scratch(c, 2049 * sizeof(unsigned long long) + 2049 * sizeof(double))) return rc;
  unsigned long long* d_counts = reinterpret_cast<unsigned long long*>(c->d_scratch);
  double* d_edges = reinterpret_cast<double*>(d_counts + 2049);
  CUDA_TRY(cudaMemsetAsync(d_counts, 0, (size_t)(n_bins + 1) * sizeof(unsigned long long), c->stream));
  CUDA_TRY(cudaMemcpyAsync(d_edges, h_edges, (size_t)(n_bins + 1) * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  const unsigned grid = (unsigned)grid_stride_blocks(n, 256, 16LL * c->sm_count);
  int rc = f64 ? launch(c, tuning_hist_kernel<double>, grid, 256, 0, (const double*)d_f, (long long)n, bins_per_octave,
                        (int)n_bins, (const double*)d_edges, d_counts)
               : launch(c, tuning_hist_kernel<float>, grid, 256, 0, (const float*)d_f, (long long)n,
                        (float)bins_per_octave, (int)n_bins, (const double*)d_edges, d_counts);
  if (rc) return rc;
  CUDA_TRY(cudaMemcpyAsync(h_counts, d_counts, (size_t)(n_bins + 1) * sizeof(unsigned long long), cudaMemcpyDeviceToHost,
                           c->stream));
  CUDA_TRY(cudaStreamSynchronize(c->stream));
  return B2L_OK;
}
