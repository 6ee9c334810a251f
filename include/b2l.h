/* b2l.h — C ABI of libb2l.so, the H100 (sm_90a) replacement for librosa's FFT time-frequency path.
 *
 * librosa has no FFI: its boundary for this path is the public Python API.  The Python package
 * `librosa_b200` mirrors those signatures and makes one call into this library per public function;
 * INTEGRATION.md shows the ctypes binding.  Each entry point names the reference code it replaces
 * (paths relative to the librosa checkout, commit b7e7bf4).
 *
 * Conventions
 *   - every function returns an int status (B2L_OK == 0); b2l_last_error() gives the message of the
 *     last failure on the calling thread;
 *   - plain pointers and sizes only; device pointers are marked d_, host pointers h_;
 *   - all work is enqueued on the context's stream; b2l_ctx_sync() waits for it;
 *   - a context is bound to one CUDA device and is not thread-safe; use one context per thread / GPU;
 *   - there is no CPU fallback: without a usable sm_90 device b2l_ctx_create fails.
 */
#ifndef B2L_H_
#define B2L_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2L_VERSION 100 /* 0.1.0 */

enum b2l_status {
  B2L_OK = 0,
  B2L_ERR_INVALID = 1,     /* bad argument (the Python layer raises ParameterError before calling) */
  B2L_ERR_CUDA = 2,        /* CUDA runtime / launch failure */
  B2L_ERR_UNSUPPORTED = 3, /* valid for librosa, not built for the GPU yet (never a silent fallback) */
  B2L_ERR_OOM = 4,
  B2L_ERR_NCCL = 5
};

/* np.pad modes accepted by librosa.stft (librosa/_typing.py:60-71, core/spectrum.py:252-265). */
enum b2l_pad_mode {
  B2L_PAD_CONSTANT = 0,
  B2L_PAD_EDGE = 1,
  B2L_PAD_REFLECT = 2,
  B2L_PAD_SYMMETRIC = 3,
  B2L_PAD_LINEAR_RAMP = 4,
  B2L_PAD_EMPTY = 5
};

typedef struct b2l_ctx b2l_ctx;
typedef struct b2l_plan b2l_plan;
typedef struct b2l_event b2l_event;

/* Constants of one transform configuration.  Built on the host by the Python layer with the same
 * float64 expressions as the reference (filters.get_window + util.pad_center, filters.mel, the
 * scipy.fft.dct matrix), uploaded once per plan. */
typedef struct b2l_plan_desc {
  int32_t n_fft;             /* 2^k in 8..8192; even <= 4096 with a 5-smooth half (mixed radix); any 3..2047 (chirp-z)  core/spectrum.py:58-69 */
  int32_t hop_length;        /* >= 1                                        core/spectrum.py:235-237 */
  int32_t center;            /* 0 / 1                                       core/spectrum.py:252     */
  int32_t pad_mode;          /* enum b2l_pad_mode                           core/spectrum.py:287     */
  const double* h_window;    /* [n_fft] window after pad_center             core/spectrum.py:243-249 */
  int32_t n_mels;            /* 0: no mel stage                             feature/spectral.py:2158 */
  const float* h_mel_basis;  /* [n_mels][1 + n_fft/2] float32 (filters.mel) filters.py:117-251       */
  float power;               /* exponent of |STFT|                          core/spectrum.py:3000    */
  int32_t n_mfcc;            /* 0: no mfcc stage                            feature/spectral.py:2005 */
  const float* h_dct_basis;  /* [n_mfcc][n_mels] DCT rows (lifter folded in) feature/spectral.py:2005-2015 */
  float amin;                /* power_to_db amin                            core/spectrum.py:1875    */
  float ref_value;           /* power_to_db |ref|                           core/spectrum.py:1876    */
  float top_db;              /* < 0 means None                              core/spectrum.py:1878-1881 */
} b2l_plan_desc;

/* ---- library / device ---------------------------------------------------------------------- */
int b2l_version(void);
const char* b2l_last_error(void);
int b2l_device_count(int* count);

int b2l_ctx_create(int device, b2l_ctx** ctx);
int b2l_ctx_destroy(b2l_ctx* ctx);
int b2l_ctx_sync(b2l_ctx* ctx);
int b2l_ctx_device(const b2l_ctx* ctx, int* device);
int b2l_ctx_sm_count(const b2l_ctx* ctx, int* sms);
/* kernels launched by this context since creation (bench.py reports it as gpu_launches) */
int b2l_ctx_launch_count(const b2l_ctx* ctx, uint64_t* launches);

/* ---- util.valid_audio on the device (librosa/util/utils.py:246-308) ----------------------------
 * The forward kernels set B2L_STATUS_NOT_FINITE_SAMPLE in a per-context status word when a non-finite sample
 * reaches a frame;
 * b2l_scan_finite covers samples [begin, n) that no frame reads (tail / hop > n_fft gaps);
 * b2l_scan_finite_f64 does the same for the float64 signals of the FP64 path and flags exactly the samples
 * np.isfinite rejects.  The Python layer resets the word before a call on host data, reads it with the
 * results and raises ParameterError("Audio buffer is not finite everywhere") exactly as the reference does. */
int b2l_status_reset(b2l_ctx* ctx);
int b2l_status_read(b2l_ctx* ctx, int* status); /* synchronises the ctx stream */

/* Bits of the status word.  The forward transforms and b2l_scan_finite* set B2L_STATUS_NOT_FINITE_SAMPLE with a
 * plain store of that bit, which clears any other bit already set; every other setter uses atomicOr.  So within one
 * reset epoch nothing may set bits 1-3 before a forward kernel or a finite scan runs: each caller that reads bits
 * 1-3 either resets the word right before the kernels that set them, or runs them after its last forward kernel. */
enum b2l_status_bit {
  B2L_STATUS_NOT_FINITE_SAMPLE = 1, /* a kernel read a non-finite input sample (util.valid_audio)      */
  B2L_STATUS_NEGATIVE_ENTRY = 2,    /* b2l_spectral_stats_from_spec read a negative spectrogram entry */
  B2L_STATUS_NOT_FINITE_VALUE = 4,  /* b2l_tempogram or b2l_plp_finish met a non-finite value         */
  B2L_STATUS_NEGATIVE_EVENT = 8     /* b2l_onset_backtrack was given a negative event frame          */
};
int b2l_scan_finite(b2l_ctx* ctx, const float* d_y, int64_t n_clips, int64_t n, int64_t y_stride,
                    int64_t begin);
int b2l_scan_finite_f64(b2l_ctx* ctx, const double* d_y, int64_t n_clips, int64_t n, int64_t y_stride,
                        int64_t begin);

/* ---- memory --------------------------------------------------------------------------------- */
int b2l_alloc(b2l_ctx* ctx, size_t bytes, void** d_ptr);
int b2l_free(b2l_ctx* ctx, void* d_ptr);
int b2l_memset(b2l_ctx* ctx, void* d_ptr, int value, size_t bytes);
int b2l_h2d(b2l_ctx* ctx, void* d_dst, const void* h_src, size_t bytes); /* async on the ctx stream */
int b2l_d2h(b2l_ctx* ctx, void* h_dst, const void* d_src, size_t bytes); /* async on the ctx stream */
int b2l_d2d(b2l_ctx* ctx, void* d_dst, const void* d_src, size_t bytes);
/* strided device-to-device copy of `rows` rows of `width_bytes` (cudaMemcpy2DAsync on the context stream) */
int b2l_copy2d(b2l_ctx* ctx, void* d_dst, size_t dst_pitch, const void* d_src, size_t src_pitch, size_t width_bytes,
               size_t rows);
int b2l_host_alloc(size_t bytes, void** h_ptr);                          /* pinned host memory */
int b2l_host_free(void* h_ptr);
int b2l_mem_info(b2l_ctx* ctx, size_t* free_bytes, size_t* total_bytes);

/* ---- timing (CUDA events on the ctx stream) -------------------------------------------------- */
int b2l_event_create(b2l_ctx* ctx, b2l_event** ev);
int b2l_event_record(b2l_ctx* ctx, b2l_event* ev);
int b2l_event_elapsed_ms(b2l_event* start, b2l_event* stop, float* ms); /* syncs on stop */
int b2l_event_destroy(b2l_event* ev);

/* ---- plans ------------------------------------------------------------------------------------ */
int b2l_plan_create(b2l_ctx* ctx, const b2l_plan_desc* desc, b2l_plan** plan);
int b2l_plan_destroy(b2l_plan* plan);
/* frame count for a clip of n samples: 1 + (n + 2*pad - n_fft) / hop   (core/spectrum.py:277-355) */
int b2l_plan_n_frames(const b2l_plan* plan, int64_t n, int64_t* n_frames);

/* ---- the hot path ------------------------------------------------------------------------------
 * Layouts (device memory, float32 / complex64):
 *   y      [n_clips][y_stride]               first n samples of each row are the clip
 *   D      [n_clips][n_frames][1 + n_fft/2]  bins contiguous; viewed by NumPy as (..., bin, frame),
 *                                            which for a single clip is exactly the reference's
 *                                            Fortran-ordered stft matrix (core/spectrum.py:356)
 *   mel    [n_clips][n_mels][n_frames]       C order, like the reference einsum output
 *   mfcc   [n_clips][n_mfcc][n_frames]
 */

/* librosa.stft — core/spectrum.py:58-391 (frame, window, rfft). */
int b2l_stft(b2l_ctx* ctx, const b2l_plan* plan, const float* d_y, int64_t n_clips, int64_t n,
             int64_t y_stride, void* d_D /* complex64 */);

/* np.abs(stft)**power — core/spectrum.py:2920-3015 (_spectrogram); out [n_clips][n_frames][bins]. */
int b2l_spectrogram(b2l_ctx* ctx, const b2l_plan* plan, const float* d_y, int64_t n_clips, int64_t n,
                    int64_t y_stride, float* d_S);

/* librosa.feature.melspectrogram(y=...) — feature/spectral.py:2022-2161, fused with stft. */
int b2l_melspectrogram(b2l_ctx* ctx, const b2l_plan* plan, const float* d_y, int64_t n_clips, int64_t n,
                       int64_t y_stride, float* d_mel);

/* librosa.feature.mfcc(y=...) — feature/spectral.py:1843-2019 incl. power_to_db
 * (core/spectrum.py:1735-1883, per-clip top_db reference max).  d_logmel is scratch of
 * n_clips * n_mels * (n_frames rounded up to a multiple of 64) floats (internal tiled layout; NULL: allocated
 * and freed internally); like d_y and d_mfcc it needs only the 4-byte alignment of a float. */
int b2l_mfcc(b2l_ctx* ctx, const b2l_plan* plan, const float* d_y, int64_t n_clips, int64_t n,
             int64_t y_stride, float* d_mfcc, float* d_logmel);

/* librosa.istft — core/spectrum.py:395-626 (+ __overlap_add :629-643).  n_frames_stored is the frame
 * count of D; n_frames_used <= stored is what the reference would use for `length` (:523-531).
 * d_inv_wss: [out_len] reciprocal of the trimmed window-sum-square where > tiny, else 1
 * (filters.window_sumsquare, filters.py:1268-1339; core/spectrum.py:606-624). */
int b2l_istft(b2l_ctx* ctx, const b2l_plan* plan, const void* d_D, int64_t n_clips, int64_t n_frames_stored,
              int64_t n_frames_used, const float* d_inv_wss, int64_t out_len, float* d_y, int64_t y_stride);

/* ---- pieces of the path for S= inputs (device arrays in the layouts above) -------------------- */
/* mel_basis . S for a given spectrogram S [n_clips][n_frames][bins] (feature/spectral.py:2160). */
int b2l_mel_project(b2l_ctx* ctx, const b2l_plan* plan, const float* d_S, int64_t n_clips,
                    int64_t n_frames, float* d_mel);
/* power_to_db over [n_clips][rows][cols] blocks, top_db reference max per clip
 * (core/spectrum.py:1839-1883); in place when d_out == d_in. */
int b2l_power_to_db(b2l_ctx* ctx, const float* d_in, int64_t n_clips, int64_t per_clip, float amin,
                    float ref_value, float top_db, float* d_out);
/* Spectral-flux onset strength envelope of a dB-scaled spectrogram d_S [n_clips][n_rows][n_frames]
 * (librosa/onset.py:445-640 onset_strength_multi; :217-367 onset_strength is channel 0 of the default call):
 *   out [n_clips][n_channels][n_frames], channel c = mean over rows bounds[c] .. bounds[c+1]-1 of
 *   max(0, S[m][t + lag] - maxfilter_rows(S, max_size)[m][t]), shifted right by pad_width frames
 *   (lag, plus n_fft // (2 hop) when centred), optionally detrended (lfilter([1,-1],[1,-0.99])).
 *   n_channels == 0: no aggregation, out [n_clips][n_rows][n_frames]. */
typedef struct b2l_onset_desc {
  int32_t lag, max_size, pad_width, detrend, n_channels;
  int32_t bounds[33];
} b2l_onset_desc;
int b2l_onset_from_spec(b2l_ctx* ctx, const b2l_onset_desc* desc, const float* d_S, int64_t n_clips, int64_t n_rows,
                        int64_t n_frames, float* d_out);
/* The same envelope aggregated with np.median over each channel's rows (util.sync(..., aggregate=np.median)): the
 * float32 mean of the two middle values for an even row count, NaN when a flux of the column is NaN.  1 to 32
 * channels of at most 512 rows each (else B2L_ERR_UNSUPPORTED). */
int b2l_onset_median_from_spec(b2l_ctx* ctx, const b2l_onset_desc* desc, const float* d_S, int64_t n_clips,
                               int64_t n_rows, int64_t n_frames, float* d_out);
/* Per-channel energy normalisation, librosa.pcen (core/spectrum.py:2396-2666), of d_S [n_clips][n_rows][n_frames]
 * along time: first-order IIR smoother with coefficient b (lfilter([b], [1, b-1])), adaptive gain and root
 * compression.  d_zi / d_zf: optional initial / final filter state, one float per (clip, row) (NULL: the
 * lfilter_zi steady state 1 - b / not returned).  max_size > 1 max-filters the smoother's input over rows
 * (scipy.ndimage.maximum_filter1d) into d_scratch (same size as S).  In place when d_out == d_S and max_size == 1. */
typedef struct b2l_pcen_desc {
  float gain, bias, power, eps, b;
  int32_t max_size;
} b2l_pcen_desc;
int b2l_pcen(b2l_ctx* ctx, const b2l_pcen_desc* desc, const float* d_S, int64_t n_clips, int64_t n_rows,
             int64_t n_frames, const float* d_zi, float* d_zf, float* d_scratch, float* d_out);
/* Spectral contrast, librosa.feature.spectral_contrast (feature/spectral.py:355-532): per frame and octave band
 * the mean of the k[b] largest (peak) and k[b] smallest (valley) magnitudes among bins lo[b] .. lo[b]+count[b]-1
 * of d_S [n_clips][n_frames][n_bins]; peak / valley [n_clips][n_bands][n_frames].  The caller derives the bands
 * from the bin frequencies (:483-499) and finishes with power_to_db(peak) - power_to_db(valley) (b2l_power_to_db,
 * b2l_sub) or peak - valley (linear=True). */
typedef struct b2l_contrast_desc {
  int32_t n_bands;   /* reference's n_bands + 1, at most 16 */
  int32_t lo[16], count[16], k[16];
} b2l_contrast_desc;
int b2l_spectral_contrast(b2l_ctx* ctx, const b2l_contrast_desc* desc, const float* d_S, int64_t n_clips,
                          int64_t n_frames, int32_t n_bins, float* d_peak, float* d_valley);
/* librosa.resample(res_type="polyphase") (core/audio.py:1129-1145 -> scipy.signal.resample_poly): d_x [n_clips][x_stride]
 * (n_in valid samples per row) -> d_out [n_clips][n_total].  d_h: the zero-padded float32 low-pass * up (n_h taps, device),
 * designed on the host as SciPy does; output sample j < n_keep is sum_m x[m] h[(n_pre_remove + j) * down - m * up],
 * samples n_keep .. n_total-1 are the zeros of util.fix_length (:1172-1173); out_scale = 1 / sqrt(ratio) for scale=True. */
int b2l_resample_poly(b2l_ctx* ctx, const float* d_x, int64_t n_clips, int64_t n_in, int64_t x_stride, const float* d_h,
                      int32_t n_h, int32_t up, int32_t down, int64_t n_pre_remove, int64_t n_keep, int64_t n_total,
                      float out_scale, float* d_out);
/* librosa.cqt / vqt (core/constantq.py:820-1266): the filter-bank projection of every octave, stacked as __trim_stack
 * does (:1169-1194), in one launch per 65 535 clips.  Octave o's STFT d_D [n_clips][n_frames][n_fft_bins] (complex64,
 * n_frames >= the output's) meets rows indptr_off .. indptr_off + n_rows - 1 of the concatenated complex64 CSR basis
 * (d_indptr holds absolute positions into d_indices / d_data; nnz: the octave's nonzeros) and fills output rows
 * row0 .. row0 + n_rows - 1 of d_out [n_clips][n_frames][n_bins].  Each element is SciPy's `csr @ D` for complex64
 * bit for bit (ascending columns, unfused multiply and add); d_rscale [n_bins] (1 / sqrt(lengths), or NULL when
 * scale=False) multiplies in double with one rounding, as numpy's complex64 /= float64 does.  Sets no status bit.
 *
 * kind: B2L_CQT_FULL for such an octave.  B2L_CQT_PSEUDO (pseudo_cqt, :474-590) marks an octave whose table holds the
 * float32 |basis| in the real parts (imaginary parts 0) and whose rows project |D| (np.abs of complex64 as NumPy's
 * vectorised x86 loop computes it: larger part * sqrtf(fmaf(r, r, 1)), r = smaller / larger): SciPy's float32
 * `csr @ np.abs(D)` bit for bit.  B2L_CQT_DIVIDE, or'd in, makes the octave's rows divide
 * by d_rscale in double (one rounding) instead of multiplying.  b2l_cqt_project refuses pseudo octaves
 * (B2L_ERR_INVALID); b2l_cqt_project_abs takes both kinds and writes float32 into d_out [n_clips][n_frames][n_bins]:
 * a pseudo row its scaled sum, a full row the np.abs of the complex64 value b2l_cqt_project would store. */
#define B2L_CQT_MAX_OCTAVES 32
#define B2L_CQT_FULL 0
#define B2L_CQT_PSEUDO 1
#define B2L_CQT_DIVIDE 0x10
typedef struct b2l_cqt_octave {
  const void* d_D;
  int64_t n_frames;
  int32_t n_fft_bins;
  int32_t row0;
  int32_t n_rows;
  int32_t indptr_off;
  int32_t nnz;
  int32_t kind;
} b2l_cqt_octave;   /* 40 bytes */
int b2l_cqt_project(b2l_ctx* ctx, const b2l_cqt_octave* h_oct, int32_t n_oct, const int32_t* d_indptr,
                    const int32_t* d_indices, const void* d_data, const double* d_rscale, int64_t n_clips,
                    int64_t n_frames, int32_t n_bins, void* d_out);
int b2l_cqt_project_abs(b2l_ctx* ctx, const b2l_cqt_octave* h_oct, int32_t n_oct, const int32_t* d_indptr,
                        const int32_t* d_indices, const void* d_data, const double* d_rscale, int64_t n_clips,
                        int64_t n_frames, int32_t n_bins, float* d_out);
/* librosa.iirt (core/spectrum.py:1522-1713).  b2l_pad_center: np.pad(y, pad, mode) of each clip of d_x [n_clips][n]
 * into d_out [n_clips][n + 2 pad] (enum b2l_pad_mode; an empty signal takes only "constant" / "empty").
 * b2l_iirt_filter: scipy.signal.sosfiltfilt (padtype "odd", SciPy's default padlen) of every (clip, band) chain,
 * one thread per chain, bit for bit in float64: the odd extension formed in float32, then SciPy's _sosfilt loop with
 * unfused multiplies and adds.  Chain (clip, j) of rate r reads d_x + clip * x_stride (n samples; n must exceed the
 * band's padlen) and band d_bands[j]; its scratch column is d_scratch + clip * n_bands + j, with rows scratch_stride
 * doubles apart, n + padlen rows of which are written; rows 0 .. n-1 hold the filtered signal afterwards.
 * d_coef [bands][B2L_IIRT_MAX_SECTIONS][8] holds per section b0 b1 b2 a1 a2 and sosfilt_zi's two entries (a0 == 1);
 * sections 0 .. max_sections - 1 run for every band, so a band with fewer fills the rest with pass-through sections
 * (b0 = 1, all else 0).  d_info [bands][2] holds the section count and padlen.
 * b2l_iirt_stmsp: d_out [n_clips][n_bands][n_frames] float32, element (clip, d_bands[j], t) of rate r =
 * factor * sum_{i < w} x[d_starts[t] + i]^2 over the filtered signal in the scratch (rows at or past n read as the
 * zeros of util.fix_length), summed in NumPy's pairwise order as given by the leaf program d_leaves [n_leaves][4]
 * (row offset, length <= 128, partial sums combined after it, 0), rounded once to float32.  Both set no status bit. */
#define B2L_IIRT_MAX_SECTIONS 10
#define B2L_IIRT_MAX_RATES 16
#define B2L_IIRT_MAX_DEPTH 32 /* partial sums held at once by a leaf program */
typedef struct b2l_iirt_rate {
  const float* d_x;
  int64_t x_stride;
  int64_t n;
  double* d_scratch;
  int64_t scratch_stride;
  const int32_t* d_bands;
  int32_t n_bands;
  int32_t n_leaves;
  const int32_t* d_starts;
  const int32_t* d_leaves;
  double factor;
} b2l_iirt_rate;
int b2l_pad_center(b2l_ctx* ctx, const float* d_x, int64_t n_clips, int64_t n, int32_t pad, int32_t pad_mode,
                   float* d_out);
int b2l_iirt_filter(b2l_ctx* ctx, const b2l_iirt_rate* h_rates, int32_t n_rates, const double* d_coef,
                    const int32_t* d_info, int32_t max_sections, int64_t n_clips);
int b2l_iirt_stmsp(b2l_ctx* ctx, const b2l_iirt_rate* h_rates, int32_t n_rates, int64_t n_clips, int64_t n_frames,
                   int32_t n_bands, float* d_out);
/* librosa.feature.delta (feature/utils.py:20-130): scipy.signal.savgol_filter along the middle axis of
 * d_x [outer][n][inner] (float32, or float64 with f64) into d_y of the same geometry and type, in one launch.
 * Bit for bit scipy.ndimage.convolve1d: d_taps [width] are the reversed coefficients (savgol_coeffs(...)[::-1]),
 * `sym` ndimage's classification of them (1 symmetric, -1 antisymmetric, 0 neither), the sum runs in double in
 * ndimage's order with unfused operations and is rounded once.  d_pad [width - 1] is the padded-index table of the
 * line: the source sample of positions -h .. -1 and n .. n + h - 1 (h = width / 2), -1 for cval.  interp: outputs
 * 0 .. h-1 and n-h .. n-1 of each line are d_edge [width - 1][width] (rows 0 .. h-1 over samples 0 .. width-1, rows
 * h .. width-2 over samples n-width .. n-1) applied in ascending order; a non-finite sample in those windows sets
 * B2L_STATUS_NOT_FINITE_VALUE.  Widths above B2L_DELTA_MAX_WIDTH return B2L_ERR_UNSUPPORTED. */
#define B2L_DELTA_MAX_WIDTH 255
typedef struct b2l_delta_desc {
  int32_t width;
  int32_t sym;
  int32_t interp;
  int32_t f64;
  double cval;
  const double* d_taps;
  const double* d_edge;
  const int64_t* d_pad;
} b2l_delta_desc;
int b2l_delta(b2l_ctx* ctx, const b2l_delta_desc* desc, const void* d_x, int64_t outer, int64_t n, int64_t inner,
              void* d_y);
/* librosa.feature.stack_memory (feature/utils.py:133-315): d_out [n_clips][n_steps * d][t], C order, element
 * (c, s * d + r, i) = input (c, r, i - s * delay), where element (c, r, i) of d_x is at c * clip_stride + r * row_stride
 * + i * col_stride (elements of elem_size bytes: 1, 2, 4, 8 or 16).  Columns outside [0, t) are np.pad's padded
 * positions: d_pad [(n_steps - 1) * |delay|] holds the source column of positions -len .. -1 (delay > 0) or
 * t .. t + len - 1 (delay < 0), -1 for the constant, whose bytes are fill.  One launch; no status bit. */
typedef struct b2l_stack_desc {
  int32_t elem_size;
  int32_t n_steps;
  int64_t delay;
  int64_t clip_stride;
  int64_t row_stride;
  int64_t col_stride;
  uint8_t fill[16];
} b2l_stack_desc;
int b2l_stack_memory(b2l_ctx* ctx, const b2l_stack_desc* desc, const void* d_x, int64_t n_clips, int64_t d, int64_t t,
                     const int64_t* d_pad, void* d_out);
/* librosa.util.localmax / localmin (util/utils.py:1029-1178) along the middle axis of d_x [outer][n][inner], n >= 2,
 * elements of `type` (enum b2l_elem_type), into d_out of the same geometry, one byte (0 / 1) per element: never at
 * position 0; x[i] > x[i-1] and x[i] >= x[i+1] inside the line (mirrored when !is_max); x[n-1] > x[n-2] at its end.
 * NaN compares false.  One launch. */
enum b2l_elem_type {
  B2L_ELEM_I8 = 0, B2L_ELEM_U8 = 1, B2L_ELEM_I16 = 2, B2L_ELEM_U16 = 3, B2L_ELEM_I32 = 4, B2L_ELEM_U32 = 5,
  B2L_ELEM_I64 = 6, B2L_ELEM_U64 = 7, B2L_ELEM_F32 = 8, B2L_ELEM_F64 = 9, B2L_ELEM_BOOL = 10
};
int b2l_localext(b2l_ctx* ctx, const void* d_x, int32_t type, int32_t is_max, int64_t outer, int64_t n, int64_t inner,
                 uint8_t* d_out);
/* The constant-Q chroma features (feature/spectral.py:1296-1839): chroma_cqt / chroma_vqt (:1296-1423, :1576-1706),
 * the CENS steps of chroma_cens (:1426-1573) and tonnetz (:1709-1839), in one launch per 65 535 clips.
 * b2l_chroma_fold reads d_in [n_clips] x (n_bins, n_frames) in the form `input` names (complex64 input is taken as
 * |x|, correctly rounded) and, per frame, applies the cq_to_chroma map (CSR d_row_ptr [n_chroma + 1], d_cols, d_weights
 * float64: filters.cq_to_chroma, filters.py:737-861; an identity for tonnetz(chroma=...)), zeroes values below
 * `threshold` (when has_threshold) and normalises with `norm` (util.normalize, util/utils.py:958-1024: the length in
 * float64, lengths below tiny(dtype) replaced by 1), all in the chroma precision (out_f64).  The epilogue then:
 *   PLAIN    writes the chroma to d_out [n_clips][n_chroma][n_frames];
 *   CENS     L1-normalises, quantises to multiples of 0.25 at the steps 0.4 / 0.2 / 0.1 / 0.05, normalises with
 *            post_norm (NONE: the quantised values, for b2l_chroma_smooth) and writes as PLAIN;
 *   TONNETZ  L1-normalises and writes the float64 projection d_phi [6][n_chroma] of it to d_out [n_clips][6][n_frames].
 * A non-finite value met by a normalisation sets B2L_STATUS_NOT_FINITE_VALUE (normalize's "Input must be finite").
 * b2l_chroma_smooth is chroma_cens's scipy.ndimage.convolve(x, w, mode="constant") along frames of d_in
 * [n_clips][n_chroma][n_frames] followed by util.normalize(norm): out[t] = sum_k d_tap_w[k] * x[t - reach +
 * d_tap_off[k]] in double, ascending k, zero outside the clip, rounded once, with reach = win_len - 1 - win_len / 2;
 * the taps are the positions of the reversed window whose weight exceeds DBL_EPSILON in magnitude, as ndimage keeps. */
enum b2l_chroma_input {
  B2L_CHROMA_IN_C64_FT = 0, /* complex64 [n_frames][n_bins] per clip */
  B2L_CHROMA_IN_F32_FT = 1,
  B2L_CHROMA_IN_F32_C = 2,  /* float32 [n_bins][n_frames] per clip */
  B2L_CHROMA_IN_F64_FT = 3,
  B2L_CHROMA_IN_F64_C = 4
};
enum b2l_chroma_norm { B2L_CHROMA_NORM_NONE = 0, B2L_CHROMA_NORM_INF = 1, B2L_CHROMA_NORM_NEG_INF = 2,
                       B2L_CHROMA_NORM_ZERO = 3, B2L_CHROMA_NORM_P = 4 };
enum b2l_chroma_epilogue { B2L_CHROMA_PLAIN = 0, B2L_CHROMA_CENS = 1, B2L_CHROMA_TONNETZ = 2 };
typedef struct b2l_chroma_desc {
  int32_t input;          /* enum b2l_chroma_input */
  int32_t out_f64;        /* chroma precision: float64 (1) or float32 (0) */
  int32_t n_bins;
  int32_t n_chroma;
  int32_t nnz;            /* nonzeros of the map */
  int32_t norm;           /* enum b2l_chroma_norm */
  double norm_p;          /* the p of B2L_CHROMA_NORM_P */
  int32_t has_threshold;
  int32_t epilogue;       /* enum b2l_chroma_epilogue */
  double threshold;
  int32_t post_norm;      /* CENS: enum b2l_chroma_norm after the quantisation */
  int32_t pad_;
  double post_p;
  const int32_t* d_row_ptr;
  const int32_t* d_cols;
  const double* d_weights;
  const double* d_phi;    /* TONNETZ only */
} b2l_chroma_desc;
int b2l_chroma_fold(b2l_ctx* ctx, const b2l_chroma_desc* desc, const void* d_in, int64_t n_clips, int64_t n_frames,
                    void* d_out);
int b2l_chroma_smooth(b2l_ctx* ctx, const void* d_in, int64_t n_clips, int32_t n_chroma, int64_t n_frames,
                      int32_t f64, const int32_t* d_tap_off, const double* d_tap_w, int32_t n_taps, int32_t win_len,
                      int32_t norm, double norm_p, void* d_out);
/* out = x - y over n floats */
int b2l_sub(b2l_ctx* ctx, const float* d_x, const float* d_y, int64_t n, float* d_out);
/* Tuning estimation for chroma_stft (feature/spectral.py:1137-1293): librosa.estimate_tuning
 * (core/pitch.py:28-109) = piptrack peaks (:182-366) whose interpolated magnitude reaches the median of all
 * peaks, histogrammed by pitch residual (pitch_tuning, :112-179).  One call = one pass over the magnitude /
 * power spectrogram d_S [n_rows][n_bins] that re-detects the peaks among bins k_lo .. k_hi-1 and returns ONE
 * histogram in h_hist (the call synchronises):
 *   mode 0 / 1 / 2  digits 31..21 / 20..10 / 9..0 of the order-preserving key of the peak magnitudes (restricted
 *                   to keys whose higher digits equal `prefix`): radix selection of the exact median on the host
 *                   from three 2048 / 2048 / 1024-entry histograms;
 *   mode 3          n_res_bins-bin histogram (edges h_edges[n_res_bins + 1], np.histogram semantics) of
 *                   mod(bins_per_octave * log2(pitch / 27.5), 1) folded to [-0.5, 0.5) over peaks with
 *                   mag >= mag_threshold. */
typedef struct b2l_pip_desc {
  int32_t k_lo, k_hi;      /* bins with fmin <= f < fmax */
  float threshold;         /* peaks must exceed threshold * max over the frame ... */
  float ref_abs;           /* ... or this absolute value when >= 0 (piptrack(ref=number)) */
  double hz_per_bin;       /* sr / n_fft */
  int32_t mode;
  uint32_t prefix;
  float mag_threshold;
  float bins_per_octave;
  int32_t n_res_bins;
} b2l_pip_desc;
int b2l_pip_pass(b2l_ctx* ctx, const b2l_pip_desc* desc, const float* d_S, int64_t n_rows, int32_t n_bins,
                 const double* h_edges, uint64_t* h_hist);
/* util.normalize(x, norm, axis=-2) of [n_clips][n_rows][n_frames] (util/utils.py:797-1026, default threshold and
 * fill): norm_kind 0 = inf, 1 = -inf, 2 = number of non-zeros, 3 = p-norm (norm_p > 0). */
int b2l_normalize_rows(b2l_ctx* ctx, const float* d_in, int64_t n_clips, int64_t n_rows, int64_t n_frames,
                       int32_t norm_kind, float norm_p, float* d_out);
/* ---- SURVEY 8f rank 3: harmonic / percussive separation, librosa.decompose.hpss (decompose.py:241-389) --------
 * d_mag [n_clips][n_frames][n_bins] magnitudes.  harm / perc = running medians over win_harm frames / win_perc
 * bins (scipy.ndimage.median_filter, reflect boundary), turned into soft masks (util.softmask, `power`, margins).
 * mask_only: d_out_* receive the float32 masks.  Otherwise the masked spectrogram: complex64 S * mask when
 * d_S_complex is given (the reference's (|S| * mask) * phase), else float32 d_mag * mask.  Windows up to 64. */
typedef struct b2l_hpss_desc {
  int32_t win_harm, win_perc;
  float margin_harm, margin_perc, power;   /* power may be +inf (hard mask) */
  int32_t mask_only;
} b2l_hpss_desc;
int b2l_hpss(b2l_ctx* ctx, const b2l_hpss_desc* desc, const float* d_mag, const void* d_S_complex, int64_t n_clips,
             int64_t n_frames, int64_t n_bins, void* d_out_harm, void* d_out_perc);
/* |z| of n complex64 values */
int b2l_cabs(b2l_ctx* ctx, const void* d_complex, int64_t n, float* d_out);
/* Time-frequency reassignment, librosa.reassigned_spectrogram (core/spectrum.py:1019-1293 with
 * __reassign_frequencies :646-856 and __reassign_times :859-1016): elementwise over the STFTs taken with the
 * window (d_Sh), its cyclic derivative (d_Sdh) and the time-weighted window (d_Sth), all complex64
 * [n_clips][n_frames][n_bins]; d_bin_freqs [n_bins] (Hz), d_frame_times [n_frames] (s).  Outputs float32 in the
 * same layout.  mag_threshold = sqrt(ref_power); apply_threshold = ref_power > 0. */
typedef struct b2l_reassign_desc {
  float sr, mag_threshold, max_time;
  int32_t reassign_frequencies, reassign_times, apply_threshold, fill_nan, clip;
} b2l_reassign_desc;
int b2l_reassign(b2l_ctx* ctx, const b2l_reassign_desc* desc, const void* d_Sh, const void* d_Sdh, const void* d_Sth,
                 int64_t n_clips, int64_t n_frames, int64_t n_bins, const float* d_bin_freqs,
                 const float* d_frame_times, float* d_freqs, float* d_times, float* d_mags);
/* librosa.phase_vocoder (core/spectrum.py:1364-1530) on d_D [n_clips][n_frames][n_bins] complex64 ->
 * d_out [n_clips][n_out][n_bins].  Per output frame t (device arrays of length n_out, built by the caller from
 * `rate` / `t_out`): i0 = floor(t_out), i1 = min(i0 + 1, n_frames - 1) for the phase increments (:1498-1512);
 * lo, dx = the segment and offset scipy.interpolate.interp1d(kind="linear", fill_value="extrapolate") uses for
 * the magnitudes (:1517-1527). */
int b2l_phase_vocoder(b2l_ctx* ctx, const void* d_D, int64_t n_clips, int64_t n_frames, int64_t n_bins,
                      int64_t n_out, const int32_t* d_i0, const int32_t* d_i1, const int32_t* d_lo,
                      const double* d_dx, void* d_out);
/* Elementwise pieces of the dB conversions over n floats (in place when d_out == d_in):
 *   B2L_UNARY_SQUARE           x*x                       amplitude_to_db (core/spectrum.py:1946-2038) = power_to_db
 *                                                        of the squared magnitudes with ref^2 / amin^2
 *   B2L_UNARY_DB_TO_POWER      param * 10^(0.1 x)        db_to_power (core/spectrum.py:1899-1925), param = ref
 *   B2L_UNARY_DB_TO_AMPLITUDE  sqrt(param * 10^(0.1 x))  db_to_amplitude (:2054-2081), param = ref^2 */
enum { B2L_UNARY_SQUARE = 0, B2L_UNARY_DB_TO_POWER = 1, B2L_UNARY_DB_TO_AMPLITUDE = 2 };
int b2l_unary(b2l_ctx* ctx, int32_t op, const float* d_in, int64_t n, float param, float* d_out);
/* DCT rows applied along the mel axis of S [n_clips][n_mels][n_frames] (feature/spectral.py:2005). */
int b2l_dct_project(b2l_ctx* ctx, const b2l_plan* plan, const float* d_S, int64_t n_clips,
                    int64_t n_frames, float* d_mfcc);
/* [n_clips][rows][cols] -> [n_clips][cols][rows], elem_bytes 4 or 8 (layout adapter for NumPy
 * arrays that arrive as C-ordered (..., bin, frame)). */
int b2l_transpose(b2l_ctx* ctx, const void* d_in, int64_t n_clips, int64_t rows, int64_t cols,
                  int32_t elem_bytes, void* d_out);

/* ---- first "next" row of SURVEY 8f: Griffin-Lim (core/spectrum.py:2669-2917) -----------------------
 * Phase update between the istft and stft of one iteration, elementwise over n complex values:
 *   angles = rebuilt - scale * tprev (tprev may be NULL);  angles = angles / (|angles| + eps) * S
 * (core/spectrum.py:2898-2903; scale = momentum / (1 + momentum)).  All arrays in the D / S layouts. */
int b2l_gl_update(b2l_ctx* ctx, const void* d_rebuilt, const void* d_tprev, const float* d_S, float scale, float eps,
                  void* d_angles, int64_t n);

/* ---- second "next" row of SURVEY 8f: the frame-wise consumers of _spectrogram -----------------------
 * Statistics of the magnitude spectrum |X| of every frame, out [n_clips][B2L_N_STATS][n_frames]:
 *   row 0 spectral_centroid  (feature/spectral.py:46-191)   sum f S / sum S  (util.normalize, norm=1)
 *   row 1 spectral_bandwidth (:194-352)  (sum S |f - centroid|^p)^(1/p), S normalised when bw_norm
 *   row 2 spectral_rolloff   (:535-684)  lowest f whose running sum reaches roll_percent * total
 *   row 3 spectral_flatness  (:687-803)  geometric / arithmetic mean of max(amin, S^power)
 *   row 4 rms(S=...)         (:806-916)  with frame_length = n_fft
 *   row 5 sum S
 * d_freq: [bins] bin frequencies in Hz (core/convert.py:1369 fft_frequencies, or the caller's `freq`). */
#define B2L_N_STATS 6
typedef struct b2l_stats_desc {
  float roll_percent;  /* (0, 1) */
  float flat_amin;     /* > 0 */
  float flat_power;
  float bw_p;          /* > 0 */
  int32_t bw_norm;
  int32_t frame_length;
  int32_t want;        /* bit r set: row r is needed (0 = all rows); rows not asked for are unspecified */
} b2l_stats_desc;
/* y= form: fused with the stft (no spectrogram is written); power-of-two n_fft plans. */
int b2l_spectral_stats(b2l_ctx* ctx, const b2l_plan* plan, const b2l_stats_desc* desc, const float* d_y,
                       int64_t n_clips, int64_t n, int64_t y_stride, const float* d_freq, float* d_out);
/* S= form: d_S [n_clips][n_frames][n_bins] magnitudes.  B2L_STATUS_NEGATIVE_ENTRY is set in the status word
 * (b2l_status_read) when S holds a negative entry (the reference raises ParameterError). */
int b2l_spectral_stats_from_spec(b2l_ctx* ctx, const b2l_stats_desc* desc, const float* d_S, int64_t n_clips,
                                 int64_t n_frames, int32_t n_bins, const float* d_freq, float* d_out);
/* Time-domain framings, out [n_clips][n_frames] with n_frames = 1 + (n + 2*pad - frame_length) / hop:
 *   B2L_FRAME_RMS            rms(y=...)          feature/spectral.py:881-890
 *   B2L_FRAME_ZERO_CROSSINGS zero_crossing_rate  feature/spectral.py:1062-1133 + core/audio.py:1588-1728;
 *                            writes count * out_scale per frame (out_scale = 1: the caller divides by
 *                            frame_length in float64, like np.mean over booleans); threshold / zero_pos / pad_first as in
 *                            zero_crossings(threshold=, zero_pos=, pad=). */
enum { B2L_FRAME_RMS = 0, B2L_FRAME_ZERO_CROSSINGS = 1 };
int b2l_frame_feature(b2l_ctx* ctx, int32_t what, const float* d_y, int64_t n_clips, int64_t n, int64_t y_stride,
                      int32_t frame_length, int32_t hop_length, int32_t center, int32_t pad_mode, float threshold,
                      int32_t zero_pos, int32_t pad_first, float out_scale, float* d_out);

/* ---- pitch tracking: librosa.yin / librosa.pyin (core/pitch.py:369-931, sequence.py:1174-1259) ---------------
 * A row is one (clip, frame) pair; n_lags = max_period - min_period + 1; max_cand = (n_lags + 1) / 2.
 * b2l_yin_cmnd: frames (frame_length, hop_length, center / pad_mode as librosa.util.frame after np.pad) -> the
 *   cumulative mean normalised difference, float32 d_cmnd [n_clips][n_frames][n_lags]; the autocorrelation comes
 *   from the register FFT at N = the smallest power of two >= frame_length + max_period + 1 (up to 8192, else
 *   B2L_ERR_UNSUPPORTED).  Sets B2L_STATUS_NOT_FINITE_SAMPLE when a frame reads a non-finite sample.
 * b2l_yin_pick: CMND rows -> f0 of yin, float64 [n_rows]. */
typedef struct b2l_yin_desc {
  int32_t frame_length, hop_length, center, pad_mode;
  int32_t min_period, max_period;
  double sr, trough_threshold;
} b2l_yin_desc;
int b2l_yin_cmnd(b2l_ctx* ctx, const b2l_yin_desc* desc, const float* d_y, int64_t n_clips, int64_t n,
                 int64_t y_stride, float* d_cmnd);
int b2l_yin_pick(b2l_ctx* ctx, const b2l_yin_desc* desc, const float* d_cmnd, int64_t n_rows, double* d_f0);
/* pyin's decision stages.  Tables are device arrays built by the caller:
 *   d_thresholds [n_thresholds + 1] np.linspace(0, 1, n_thresholds + 1); d_beta [n_thresholds] the beta weights;
 *   d_beta_cum [n_thresholds + 1] np.sum(beta[:c]); d_pmf: scipy.stats.boltzmann.pmf(pos, lambda, n) at
 *   n (n - 1) / 2 + pos for n = 1 .. max_cand;
 *   the Viterbi's log(T + tiny) of T = kron(transition_loop(2, 1 - switch_prob), transition_local(n_pitch_bins,
 *   2 half_width + 1)) for source state (a, p) and target (b, q): d_ltab[(d_cls[p] * 2 + (a != b)) * (2 half_width
 *   + 1) + q - p + half_width] for |q - p| <= half_width (d_cls[p]: class of the row sum of transition_local's row p),
 *   log(tiny) elsewhere; a transition is searched when its value is >= log_thr, or always when full;
 *   d_freqs [n_pitch_bins] the bin frequencies.
 * b2l_pyin_obs: CMND rows -> per row the voiced candidates (count, pitch bins ascending, probabilities; at most
 *   max_cand) and voiced_prob.
 * b2l_viterbi: candidates of [n_clips][n_frames] rows -> decoded states (uint16) and, when d_f0 is given, f0 and the
 *   voiced flag (d_voiced, one byte per frame; unvoiced f0 = fill_na when fill).  2 * n_pitch_bins states, at most
 *   what fits in shared memory at 18 bytes per state. */
typedef struct b2l_pyin_desc {
  int32_t min_period, max_period;
  int32_t n_thresholds, n_pitch_bins, n_bins_per_semitone;
  double sr, fmin, no_trough_prob;
  const double* d_thresholds;
  const double* d_beta;
  const double* d_beta_cum;
  const double* d_pmf;
  double log_p_init, fill_na;
  int32_t fill;
  int32_t half_width, full;
  double log_thr;
  const int32_t* d_cls;
  const double* d_ltab;
  const double* d_freqs;
} b2l_pyin_desc;
int b2l_pyin_obs(b2l_ctx* ctx, const b2l_pyin_desc* desc, const float* d_cmnd, int64_t n_rows, int32_t* d_count,
                 int32_t* d_cand_bin, double* d_cand_prob, double* d_voiced_prob);
int b2l_viterbi(b2l_ctx* ctx, const b2l_pyin_desc* desc, const int32_t* d_count, const int32_t* d_cand_bin,
                const double* d_cand_prob, const double* d_voiced_prob, int64_t n_clips, int64_t n_frames,
                uint16_t* d_states, double* d_f0, uint8_t* d_voiced);
/* librosa.piptrack (core/pitch.py:182-366) over d_S [n_clips] x (n_bins, n_frames), float32 or float64 (f64), in
 * memory [clip][frame][bin] ("ft") or, with layout_c, [clip][bin][frame], into d_pitches / d_mags [n_clips][n_frames]
 * [n_bins] of the same type (every bin written, zero off the peaks).  abs_mode: 0 takes S as it is, 1 takes |S|, 2
 * takes |S| when S holds a value < 0 and no NaN (the reference's S.min() < 0), which one extra launch decides on the
 * device.  The frame reference is threshold * max over the frame's bins (ref_frame; in float64 when thr_wide, else
 * in the data type; a NaN bin makes it NaN) or ref_abs; peaks are the bins k_lo <= k < k_hi where
 * localmax(S * (S > ref)) holds along the bins.  Interpolation in the reference's precision: the parabolic shift in
 * float64 from sums in the data type, pitch = (k + shift) * sr / n_fft in float64, mag = S + 0.5 * avg * shift in the
 * data type, unfused.  A row of more than B2L_PIPTRACK_MAX_ROW_BYTES (bins rounded up to 4, times the element size)
 * returns B2L_ERR_UNSUPPORTED. */
#define B2L_PIPTRACK_MAX_ROW_BYTES (200 * 1024)
typedef struct b2l_piptrack_desc {
  int32_t f64, layout_c;
  int32_t k_lo, k_hi;
  int32_t abs_mode, ref_frame, thr_wide, pad_;
  double threshold, ref_abs, sr, n_fft;
} b2l_piptrack_desc;
int b2l_piptrack(b2l_ctx* ctx, const b2l_piptrack_desc* desc, const void* d_S, int64_t n_clips, int32_t n_bins,
                 int64_t n_frames, void* d_pitches, void* d_mags);
/* librosa.pitch_tuning's histogram (core/pitch.py:112-179) over the n values of d_f (float32, or float64 with f64), in
 * one launch: h_counts[b] for b < n_bins counts the residuals mod(bins_per_octave * log2(f / 27.5), 1) folded to
 * [-0.5, 0.5) of the values f > 0 that fall in [h_edges[b], h_edges[b + 1]) (np.histogram; the last bin closed), and
 * h_counts[n_bins] counts the values > 0.  1 <= n_bins <= 2048.  Synchronises. */
int b2l_pitch_tuning(b2l_ctx* ctx, const void* d_f, int64_t n, int32_t f64, double bins_per_octave, int32_t n_bins,
                     const double* h_edges, uint64_t* h_counts);

/* ---- rhythm: librosa.feature.tempogram / tempo (feature/rhythm.py:38-470) ---------------------------------------
 * b2l_tempogram: onset envelopes d_env [n_rows][n] (float32, or float64 when env_f64) -> the normalised local
 *   autocorrelation, float64 d_out [n_rows][n_frames][win_length] (lags contiguous); n_frames = n when centred
 *   (np.pad mode "linear_ramp", then the first n frames), n - win_length + 1 otherwise.  d_window [win_length] is
 *   the float64 window.  The arithmetic is FP64 for both envelope types.  win_length up to 4096
 *   (else B2L_ERR_UNSUPPORTED).  util.normalize along the lags with `norm` (B2L_TG_NORM_*; norm_p the exponent of
 *   B2L_TG_NORM_P) and threshold tiny(float64); sets B2L_STATUS_NOT_FINITE_VALUE when an autocorrelation value is not
 *   finite (normalize's "Input must be finite").
 * b2l_tempo: tempograms -> the BPM d_bpms[k] of the first lag k maximising log1p(1e6 tg) + d_logprior[k]
 *   (NaN counts as the maximum), float64.  Element (row, lag, frame) of d_tg (float32, or float64 when tg_f64)
 *   is at row * row_stride + lag * lag_stride + frame * frame_stride.  With mean != 0 the tempogram is first
 *   averaged over the frames (d_out [n_rows]), else every frame is scored (d_out [n_rows][n_frames]). */
enum b2l_tempogram_norm {
  B2L_TG_NORM_NONE = 0,
  B2L_TG_NORM_MAX = 1,     /* np.inf */
  B2L_TG_NORM_MIN = 2,     /* -np.inf */
  B2L_TG_NORM_COUNT = 3,   /* 0 */
  B2L_TG_NORM_P = 4        /* p > 0 */
};
typedef struct b2l_tempogram_desc {
  int32_t win_length, center, norm, env_f64;
  double norm_p;
} b2l_tempogram_desc;
int b2l_tempogram(b2l_ctx* ctx, const b2l_tempogram_desc* desc, const void* d_env, int64_t n_rows, int64_t n,
                  const double* d_window, double* d_out);
typedef struct b2l_tempo_desc {
  int32_t n_lags, mean, tg_f64;
  int64_t n_frames, row_stride, lag_stride, frame_stride;
} b2l_tempo_desc;
int b2l_tempo(b2l_ctx* ctx, const b2l_tempo_desc* desc, const void* d_tg, int64_t n_rows, const double* d_logprior,
              const double* d_bpms, double* d_out);

/* ---- beat tracking: librosa.beat.beat_track's tracker (beat.py:510-742) and plp -----------------------------------------
 * b2l_beat_track: onset envelopes d_env [n_clips][n] (float32, or float64 when env_f64) and frames per beat ->
 *   d_beats [n_clips][n] (1 at a beat), one launch.  The stages restate the reference's arithmetic: normalisation
 *   by std(ddof=1) (NumPy pairwise sums), the Gaussian local score, the DP with float32 `tightness`, the last
 *   beat (median of the cumulative score's local maxima), the backtrack and the trim.  Frames per beat come per
 *   clip (n_fpb == 1) or per frame (n_fpb == n) as device float64 tables [n_clips][n_fpb] built by the caller with
 *   libm: d_fpb (integers >= 1), d_logfpb (log, or logf for the float32 DP), d_woff (index into d_wtab of the
 *   window's centre; d_wtab[woff + d] = exp(-0.5 x x), x = d * 32.0 / fpb, for |d| <= min(fpb, n - 1)), and
 *   d_logd [n_logd] = log(d) for 1 <= d <= min(2 max fpb, n - 1).  The DP and d_cumscore are float64 when dp_f64
 *   (numba's choice whenever the envelope or the frames per beat are float64), else float32; d_localscore has the
 *   envelope's type.  d_localscore, d_cumscore ([n_clips][n]) and d_backlink may be NULL (a work area is used).  With d_sparse (one clip only) the beat
 *   frames surviving the trim are also written in ascending order, converted to `units` (int64 frames or
 *   samples = frame * hop_length, float64 seconds = samples / sr), and their number to d_count.
 * b2l_any_nonzero: *d_flag = 1 when an element of d_x [n] (float32, or float64 when f64) is not zero, else 0. */
enum b2l_beat_units { B2L_BEAT_FRAMES = 0, B2L_BEAT_SAMPLES = 1, B2L_BEAT_TIME = 2 };
typedef struct b2l_beat_desc {
  int32_t n_fpb, env_f64, dp_f64, trim, units;
  float tightness;
  int32_t hop_length;
  double sr;
  const double* d_fpb;
  const double* d_logfpb;
  const double* d_woff;
  const double* d_wtab;
  const double* d_logd;
} b2l_beat_desc;
int b2l_beat_track(b2l_ctx* ctx, const b2l_beat_desc* desc, const void* d_env, int64_t n_clips, int64_t n,
                   void* d_localscore, void* d_cumscore, int32_t* d_backlink, uint8_t* d_beats, void* d_sparse,
                   int64_t* d_count);
int b2l_any_nonzero(b2l_ctx* ctx, const void* d_x, int64_t n, int32_t f64, int32_t* d_flag);
/* librosa.beat.plp (beat.py:320-507) around the stft / istft entry points:
 * b2l_plp_select: in place on a Fourier tempogram d_ftgram [n_frames][n_bins] (complex64, or complex128 when c128;
 *   n_frames counts every (row, frame)): zero the bins whose d_keep entry is 0 (the tempo range), zero every bin
 *   whose log1p(1e6 |X|) (+ d_logprior[bin] in float64 when d_logprior != NULL) is below the frame's maximum, then
 *   divide by sqrt_tiny + |max(X)| under NumPy's lexicographic complex max.  d_keep / d_logprior: float64 [n_bins].
 * b2l_plp_finish: in place on the pulse d_pulse [n_rows][n] (float32, or float64 when f64): clip below at 0, then
 *   divide each row by its maximum (1 when below tiny); a non-finite value sets B2L_STATUS_NOT_FINITE_VALUE. */
typedef struct b2l_plp_desc {
  int32_t n_bins, c128;
  double sqrt_tiny;
  const double* d_keep;
  const double* d_logprior;
} b2l_plp_desc;
int b2l_plp_select(b2l_ctx* ctx, const b2l_plp_desc* desc, void* d_ftgram, int64_t n_frames);
int b2l_plp_finish(b2l_ctx* ctx, void* d_pulse, int64_t n_rows, int64_t n, int32_t f64);

/* ---- onset detection: librosa.onset.onset_detect, util.peak_pick and onset.onset_backtrack (onset.py:31-214,
 *      :370-441, util/utils.py:1188-1496) ----------------------------------------------------------------------------
 * b2l_onset_normalize: one launch over d_x [n_rows][n] (float32, or float64 when f64).  With d_out != NULL each row
 *   is written there as (x - min x) / (max(x - min x) + tiny), NaN propagating, every step in the envelope's type.
 *   d_flags [2] is cleared first; bit 0 of d_flags[0] is set when an element of the (normalised) batch is not zero,
 *   bit 1 when one is not finite — onset_detect's verdict over the whole call.
 * b2l_peak_pick: one launch, one CTA per row of d_x.  The picks of util.peak_pick(method) with integer windows
 *   (pre_* >= 0, post_* >= 1, wait >= 0) and float64 delta: the greedy picker takes a frame when it equals the
 *   maximum of its window (NaN: never) and is >= the window mean + delta (a left-to-right sum in the data's type,
 *   divided by the count in float64), then skips `wait` frames; the dynamic-programming pickers run numba's
 *   sequential cumsum and backward DP (dp_count maximises the number of picks, dp_value their sum).  With d_flags
 *   (from b2l_onset_normalize) every row is all-False unless the verdict is "nonzero and finite".  Writes d_dense
 *   [n_rows][n] (1 at a pick) when not NULL and, with d_sparse (one row only), the picks in ascending order
 *   converted to `units` (as b2l_beat_track) and their number to d_count.
 * b2l_onset_backtrack: one launch.  Each of the first *d_count (NULL: n_events) int64 frames of d_events is replaced
 *   by the last local minimum of d_energy [n] at or before it (e[i] <= e[i-1] and e[i] < e[i+1]; frame 0 always
 *   counts; frames past n - 1 take the last), converted to `units`, in d_out.  A negative event sets
 *   B2L_STATUS_NEGATIVE_EVENT and writes nothing. */
enum b2l_peak_method { B2L_PEAK_GREEDY = 0, B2L_PEAK_DP_COUNT = 1, B2L_PEAK_DP_VALUE = 2 };
typedef struct b2l_peak_desc {
  int64_t pre_max, post_max, pre_avg, post_avg, wait;
  double delta;
  int32_t method, f64, units, hop_length;
  double sr;
} b2l_peak_desc;
int b2l_onset_normalize(b2l_ctx* ctx, const void* d_x, int64_t n_rows, int64_t n, int32_t f64, double tiny,
                        void* d_out, int64_t* d_flags);
int b2l_peak_pick(b2l_ctx* ctx, const b2l_peak_desc* desc, const void* d_x, int64_t n_rows, int64_t n,
                  const int64_t* d_flags, uint8_t* d_dense, void* d_sparse, int64_t* d_count);
int b2l_onset_backtrack(b2l_ctx* ctx, const void* d_energy, int64_t n, int32_t f64, const int64_t* d_events,
                        int64_t n_events, const int64_t* d_count, int32_t units, int32_t hop_length, double sr,
                        void* d_out);

/* ---- HMM decoding: librosa.sequence.viterbi, viterbi_discriminative, viterbi_binary (sequence.py:1175-1876) -------
 * b2l_seq_logobs: one launch over d_prob [n_clips][n_states][n_steps] (float32, or float64 when f64), one thread
 *   per (clip, frame).  With d_out != NULL writes the float64 log-likelihoods the decoder reads:
 *     B2L_SEQ_PLAIN   log(p + eps) in prob's dtype                                   -> [clip][state][frame]
 *     B2L_SEQ_DISC    log(p + eps) in prob's dtype, minus d_log_marginal[state]      -> [clip][state][frame]
 *     B2L_SEQ_BINARY  rows (1 - p) (prob's dtype) and p as float64, log(. + eps) minus d_log_marginal[label][2]
 *                                                                                    -> [clip][label][2][frame]
 *   and ORs the verdict into d_flags (never cleared here): d_flags[0] bit 0 when a p is outside [0, 1] (PLAIN,
 *   BINARY; NaN passes) or, for DISC, negative or in a column whose sum over the states (in order, in prob's dtype)
 *   fails np.allclose(., 1); BINARY sets d_flags[1 + label] when (1 - p) + p fails np.allclose(., 1) in float64.
 * b2l_seq_decode: one launch.  Decodes n_problems problems of d_lp [problem][n_states][n_steps] (n_steps >= 1)
 *   with model problem % n_models: value[0] = lp[0] + log_p_init; value[t, j] = lp[t, j] + max over the
 *   predecessors k of j (ascending, first maximum, a NaN cost never taken, pointer 0 when none beats -inf) of
 *   value[t-1, k] + log_trans[k, j]; the last state is np.argmax(value[-1]) (the first NaN, else the first maximum).
 *   Writes d_states [problem][n_steps] and d_logp [problem] = value[-1, state[-1]].  Back-pointers take
 *   2 n_states n_steps bytes per problem of stream-ordered scratch.  Size classes (B2L_SEQ_*): up to 32 states W
 *   lanes per problem; otherwise one CTA per problem with the two value rows in shared memory and
 *   the model tables there too when they fit (MEDIUM) or read through L2 (LARGE); more states than two float64 rows
 *   of the shared memory hold -> B2L_ERR_UNSUPPORTED.  Several models need at most 32 states.
 * b2l_seq_route: the class (out[0]) and lanes per problem (out[1], small class) b2l_seq_decode would use. */
enum b2l_seq_mode { B2L_SEQ_PLAIN = 0, B2L_SEQ_DISC = 1, B2L_SEQ_BINARY = 2 };
enum b2l_seq_class { B2L_SEQ_SMALL = 0, B2L_SEQ_MEDIUM = 1, B2L_SEQ_LARGE = 2 };
typedef struct b2l_seq_logobs_desc {
  int32_t mode, f64;
  int64_t n_clips, n_states, n_steps;
  double eps;                        /* tiny(prob) for PLAIN / DISC, tiny(float64) for BINARY */
  const double* d_log_marginal;      /* DISC: [n_states]; BINARY: [n_states][2]; device */
} b2l_seq_logobs_desc;
typedef struct b2l_seq_model {
  int32_t n_states, n_models;
  int32_t deg, dense;                /* predecessor entries per state; dense: deg = n_states, entry m is state m */
  const double* d_lt;                /* [model][deg][n_states] log_trans[pred, j], padded with -inf */
  const uint16_t* d_idx;             /* [model][deg][n_states] pred, ascending, padded with 0 (NULL when dense) */
  const double* d_log_p_init;        /* [model][n_states] */
} b2l_seq_model;
int b2l_seq_logobs(b2l_ctx* ctx, const b2l_seq_logobs_desc* desc, const void* d_prob, double* d_out,
                   int32_t* d_flags);
int b2l_seq_decode(b2l_ctx* ctx, const b2l_seq_model* model, const double* d_lp, int64_t n_problems,
                   int64_t n_steps, uint16_t* d_states, double* d_logp);
int b2l_seq_route(b2l_ctx* ctx, const b2l_seq_model* model, int64_t n_problems, int32_t* out);

/* ---- alignment: librosa.sequence.dtw, dtw_backtracking, rqa (sequence.py:185-1075) ------------------------------
 * b2l_dtw_cost: one launch, one thread per cell.  C = scipy's cdist(X, Y, metric) in float64 (float32 features are
 *   widened), written [N][M], or [M][N] (C.T) with transpose.  Feature f of frame n of X is d_x[h_x_off[f] + n]
 *   (float32, or float64 when f64), likewise Y; the K features are summed in table order, unfused.  Sets bit 0 of
 *   d_flags[0] when a cost is NaN.
 * b2l_nan_flag: one launch; sets bit 0 of d_flags[0] when one of the n elements of d_x is NaN.
 * b2l_dtw_accumulate: one launch per anti-diagonal of 32 x 32 tiles.  D [n][m] float64 and steps [n][m] int32 of
 *   C [n][m] (float32, or float64 when c_f64): D = min over the steps k in table order (strictly better only) of
 *   D[i - a_k][j - b_k] + (w_mul[k] C[i][j] + w_add[k]), predecessors outside the matrix +inf; D[0][0] = C[0][0]
 *   (subseq: D[0][j] = C[0][j]) and +inf elsewhere before the scan.  With band, C counts as +inf unless
 *   band_lo < j - i < band_hi.
 * b2l_dtw_backtrack: one launch.  Walks d_steps from row n - 1 at column `start` (< 0: the last column, or with d_D
 *   and subseq the first argmin of D's last row) until row 0 (subseq) or (0, 0), or an index below 0, writing
 *   (row, column) pairs (flip: (column, row)) to d_wp [n + m][2] int64 in walk order and the count to *d_len.  A
 *   failure writes -status instead: 1 an all-inf last row and 2 an inf end cell (both with check_end and d_D), 3 a
 *   path that misses (0, 0) (check_end, not subseq), 4 a (0, 0) step, 5 a step index outside the table, 6 bit 0 of
 *   d_flags[0] (d_flags may be NULL).
 * b2l_rqa: one launch per anti-diagonal of 32 x 32 tiles.  librosa's RQA score (sim's dtype: float32, or float64
 *   when f64) and int8 pointers of sim [n][m].
 * b2l_rqa_path: two launches.  The path from the first np.argmax of score (64-bit index) along the pointers, start
 *   to end, as uint64 pairs in d_path [n][2], and its length in *d_len (-1: a column index below -m). */
enum b2l_dtw_metric { B2L_DTW_EUCLIDEAN = 0, B2L_DTW_SQEUCLIDEAN = 1, B2L_DTW_CITYBLOCK = 2, B2L_DTW_CHEBYSHEV = 3,
                      B2L_DTW_COSINE = 4 };
typedef struct b2l_dtw_cost_desc {
  int32_t f64, metric, transpose;
  int64_t K, N, M;
  const int64_t* h_x_off;            /* [K] host */
  const int64_t* h_y_off;            /* [K] host */
} b2l_dtw_cost_desc;
typedef struct b2l_dtw_desc {
  int64_t n, m;
  int32_t c_f64, n_steps, subseq, band;
  int64_t band_lo, band_hi;
  const int64_t* h_steps;            /* [n_steps][2] host */
  const double* h_w_add;             /* [n_steps] host */
  const double* h_w_mul;             /* [n_steps] host */
} b2l_dtw_desc;
int b2l_dtw_cost(b2l_ctx* ctx, const b2l_dtw_cost_desc* desc, const void* d_x, const void* d_y, double* d_C,
                 int32_t* d_flags);
int b2l_nan_flag(b2l_ctx* ctx, const void* d_x, int64_t n, int32_t f64, int32_t* d_flags);
int b2l_dtw_accumulate(b2l_ctx* ctx, const b2l_dtw_desc* desc, const void* d_C, double* d_D, int32_t* d_steps);
int b2l_dtw_backtrack(b2l_ctx* ctx, const b2l_dtw_desc* desc, const int32_t* d_steps, const double* d_D,
                      int64_t start, int32_t check_end, int32_t flip, const int32_t* d_flags, int64_t* d_wp,
                      int64_t* d_len);
int b2l_rqa(b2l_ctx* ctx, const void* d_sim, int64_t n, int64_t m, int32_t f64, double gap_onset, double gap_extend,
            int32_t knight, void* d_score, int8_t* d_ptr);
int b2l_rqa_path(b2l_ctx* ctx, const void* d_score, const int8_t* d_ptr, int64_t n, int64_t m, int32_t f64,
                 uint64_t* d_path, int64_t* d_len);

/* ---- double-precision path: float64 audio / complex128 spectra ---------------------------------
 * librosa computes a float64 signal in float64 (dtype_r2c, core/spectrum.py:341; the window product :388 and the
 * irfft :598 follow the input's precision; the mel einsum feature/spectral.py:2160 and scipy.fft.dct :2005
 * too).  These entry points do the same on the device in FP64 (f64_kernels.cuh): a correctness path next to
 * the float32 hot path.  Device arrays are double / double2 in the layouts of the float32 functions; constants
 * come as HOST pointers and are uploaded stream-ordered. */
/* librosa.stft for float64 y — core/spectrum.py:58-391; h_window: [n_fft] (get_window + pad_center);
 * d_out: [n_clips][n_frames][1 + n_fft/2] complex128; power-of-two n_fft up to 2^20 (in-place FFT, work area in
 * shared memory up to 16384 and in global memory above), any other n_fft up to 65536 (direct DFT). */
int b2l_stft_f64(b2l_ctx* ctx, const double* d_y, int64_t n_clips, int64_t n, int64_t y_stride, int32_t n_fft,
                 int32_t hop_length, int32_t center, int32_t pad_mode, const double* h_window, void* d_out);
/* librosa.istft for complex128 D — core/spectrum.py:395-643; h_inv_wss: [out_len] reciprocal trimmed
 * window-sum-square in float64 (filters.py:1268-1339), 1 where wss <= tiny. */
int b2l_istft_f64(b2l_ctx* ctx, const void* d_D, int64_t n_clips, int64_t n_frames_stored, int64_t n_frames_used,
                  int32_t n_fft, int32_t hop_length, int32_t center, const double* h_window,
                  const double* h_inv_wss, int64_t out_len, double* d_y, int64_t y_stride);
/* np.abs(D)**power — core/spectrum.py:3000-3013; n complex128 elements in, n float64 out. */
int b2l_f64_abs_pow(b2l_ctx* ctx, const void* d_D, int64_t n, double power, double* d_S);
/* einsum("...ft,mf->...mt", S, mel_basis) — feature/spectral.py:2160; d_S [n_clips][n_frames][n_bins] float64,
 * h_mel [n_mels][n_bins] float32 (filters.mel), d_out [n_clips][n_mels][n_frames] float64. */
int b2l_f64_mel(b2l_ctx* ctx, const double* d_S, int64_t n_clips, int64_t n_frames, int32_t n_bins,
                const float* h_mel, int32_t n_mels, double* d_out);
/* power_to_db on float64 — core/spectrum.py:1866-1881; the top_db reference maximum is per clip
 * (per_clip elements); top_db < 0: no floor. */
int b2l_f64_db(b2l_ctx* ctx, const double* d_in, int64_t n_clips, int64_t per_clip, double amin, double ref_value,
               double top_db, double* d_out);
/* scipy.fft.dct(S, axis=-2, type, norm)[:n_mfcc] (* lifter) as the explicit matrix h_dct [n_mfcc][n_mels] —
 * feature/spectral.py:2005-2015; d_L [n_clips][n_mels][n_frames] -> d_out [n_clips][n_mfcc][n_frames]. */
int b2l_f64_dct(b2l_ctx* ctx, const double* d_L, int64_t n_clips, int32_t n_mels, int64_t n_frames,
                const double* h_dct, int32_t n_mfcc, double* d_out);

/* ---- feature.inverse ------------------------------------------------------------------------- */
/* librosa.feature.inverse.mel_to_stft — feature/inverse.py:28-114 (util.nnls, util/_nnls.py:22-175):
 * min |A X - B|^2 over X >= 0 per frame, A = h_basis [n_mels][n_bins] (triangular: every bin in <= 2 rows),
 * started from max(0, pinv(A) B) (h_pinv [n_bins][n_mels]) and refined by n_iter accelerated projected-gradient
 * steps of size `step` (1 / sigma_max(A)^2); the result is raised to inv_power = 1 / power.
 * d_mel [n_clips][n_mels][n_frames] -> d_out [n_clips][n_bins][n_frames]. */
int b2l_nnls_mel(b2l_ctx* ctx, const float* d_mel, int64_t n_clips, int64_t n_frames, int32_t n_mels, int32_t n_bins,
                 const float* h_basis, const float* h_pinv, float step, int32_t n_iter, float inv_power, float* d_out);

/* ---- nearest neighbours (segment.recurrence_matrix, decompose.nn_filter) ------------------------ */
#define B2L_NN_MAX_FRAMES 65536       /* frames of one recurrence matrix */
#define B2L_NN_MAX_CANDIDATES 4096    /* sklearn's n_neighbors = min(t - 1, k + 2 width) */
#define B2L_NN_MAX_STATS 256          /* links per frame of the affinity bandwidth statistics (k + 1) */
enum b2l_nn_metric { B2L_NN_EUCLIDEAN = 0, B2L_NN_COSINE = 1 };
enum b2l_nn_bandwidth {
  B2L_NN_BW_SCALAR = 0, B2L_NN_BW_MEAN_K = 1, B2L_NN_BW_GMEAN_K = 2, B2L_NN_BW_MEAN_K_AVG = 3,
  B2L_NN_BW_GMEAN_K_AVG = 4, B2L_NN_BW_MEAN_K_AVG_AND_PAIR = 5, B2L_NN_BW_MED_K_SCALAR = 6
};
enum b2l_nn_aggregate { B2L_NN_MEAN = 0, B2L_NN_MEDIAN = 1, B2L_NN_AVERAGE = 2 };
typedef struct b2l_nn_desc {
  int32_t metric;        /* enum b2l_nn_metric */
  int32_t mode;          /* 0 connectivity, 1 distance, 2 affinity */
  int32_t k, width;
  int32_t n_cand;        /* min(t - 1, k + 2 width) */
  int32_t sym, self_link;
  int32_t f64;           /* distances are rounded to float64 (else float32) before any statistic or output */
  int32_t bw_mode;       /* enum b2l_nn_bandwidth (affinity mode) */
  int32_t src_f64;       /* the source data is float64 (else float32) */
  double bandwidth;      /* B2L_NN_BW_SCALAR */
  /* feature f = lead * n_feat + g of frame i is src[lead * lead_stride + g * feat_stride + i * frame_stride] */
  int64_t n_lead, n_feat, lead_stride, feat_stride, frame_stride;
} b2l_nn_desc;
/* librosa.segment.recurrence_matrix (segment.py:391-706) of t frames as a neighbour table: row i of d_idx / d_val
 * [t][k_out] (k_out >= min(k, n_cand) + 1) holds the links of frame i (column i of the reference's csc_array),
 * ascending frame index, d_count[i] of them; d_val is 1 (connectivity), the distance rounded to the output dtype
 * (distance) or exp(-distance / bandwidth) in that dtype (affinity).  Float64 distances (FP64 tensor cores), d(i, j)
 * == d(j, i) bit for bit; candidates in (distance, index) order.  Synchronises (finite check, bandwidth errors).
 * Data with a NaN or an infinity sets *h_not_finite = 1 and computes nothing. */
int b2l_nn_graph(b2l_ctx* ctx, const b2l_nn_desc* desc, const void* d_src, int64_t t, int32_t k_out, int32_t* d_idx,
                 double* d_val, int32_t* d_count, int32_t* h_not_finite);
typedef struct b2l_nn_filter_desc {
  int32_t agg;           /* enum b2l_nn_aggregate */
  int32_t s_f64;         /* S is float64 (else float32) */
  int32_t r_f64;         /* np.average computes in float64 (np.result_type(S, weights)) */
  int32_t max_count;     /* the largest neighbour count (median) */
  int64_t stride;        /* entries of frame i start at i * stride when d_start is NULL */
} b2l_nn_filter_desc;
/* decompose.nn_filter's aggregation (decompose.py:550-592): d_S [n_lead][t][n_bins] ("ft"), frame i's neighbours
 * d_idx[start_i .. start_i + d_count[i]) with weights d_w (values of the compute dtype; average only), out like S.
 * *h_zero_weight = 1 when some frame's weights sum to zero (np.average raises; synchronises for average). */
int b2l_nn_filter(b2l_ctx* ctx, const b2l_nn_filter_desc* desc, const void* d_S, int64_t n_lead, int64_t t,
                  int64_t n_bins, const int64_t* d_start, const int32_t* d_count, const int32_t* d_idx,
                  const double* d_w, void* d_out, int32_t* h_zero_weight);
/* The dense C-ordered t x t matrix (B2L_ELEM_F32 / F64 / BOOL) of a b2l_nn_graph table: rec[j, i] = d_val of link
 * (i, j), zero elsewhere. */
int b2l_nn_dense(b2l_ctx* ctx, const int32_t* d_idx, const double* d_val, const int32_t* d_count, int64_t t,
                 int32_t k_out, int32_t elem, void* d_rec);
/* scipy.sparse.csc_array of a dense C-ordered t x t matrix (B2L_ELEM_F32 / F64 / BOOL): pass 0 writes the non-zero
 * count of every column, pass 1 the rows (ascending) and values of column i at d_start[i]. */
int b2l_nn_compact(b2l_ctx* ctx, const void* d_rec, int32_t elem, int64_t t, int32_t pass, int32_t* d_count,
                   const int64_t* d_start, int32_t* d_idx, double* d_w);

/* ---- multi-GPU split / join (one process per GPU; NCCL over NVLink) --------------------------- */
/* 128-byte NCCL unique id, created on rank 0 and handed to the other ranks by the launcher. */
int b2l_comm_unique_id(void* id128);
int b2l_comm_init(b2l_ctx* ctx, const void* id128, int rank, int world);
int b2l_comm_destroy(b2l_ctx* ctx);
/* broadcast `bytes` from root's d_buf into every rank's d_buf (plan constants, small) */
int b2l_comm_broadcast(b2l_ctx* ctx, void* d_buf, size_t bytes, int root);
/* root holds world*shard_bytes at d_full; every rank receives its shard into d_shard */
int b2l_comm_scatter(b2l_ctx* ctx, const void* d_full, void* d_shard, size_t shard_bytes, int root);
/* inverse of scatter */
int b2l_comm_gather(b2l_ctx* ctx, const void* d_shard, void* d_full, size_t shard_bytes, int root);
int b2l_comm_barrier(b2l_ctx* ctx);

#ifdef __cplusplus
}
#endif
#endif /* B2L_H_ */
