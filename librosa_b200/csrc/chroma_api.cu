// chroma_api.cu — C ABI of the constant-Q chroma features (chroma_kernels.cuh): librosa.feature.chroma_cqt /
// chroma_vqt / chroma_cens / tonnetz (librosa/feature/spectral.py:1296-1839).  The only unit that includes
// chroma_kernels.cuh.
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>

#include "internal.h"
// after internal.h: the kernels use the status bits of b2l.h
#include "chroma_kernels.cuh"

using namespace b2l;

namespace {

using b2l_chroma::kThreads;

constexpr int kFoldFrames = 32;     // frames per fold block
constexpr int kSmoothFrames = 128;  // frames per smoothing block
// Largest map (nonzeros and row offsets) staged in shared memory; a larger one is read through L1.
constexpr size_t kMapCap = 16 * 1024;
// The fold kernel's static shared memory (its not-finite flag), kept out of the dynamic limit.
constexpr size_t kStaticSmem = 64;

size_t even(size_t n) { return (n + 1) / 2 * 2; }

// Mirror of the fold kernel's shared-memory layout.
size_t fold_smem_bytes(int tf, int nb, int nc, int nnz, bool staged, size_t out_size, size_t mag_size) {
  return tf * 8 + (staged ? (size_t)nnz * 8 : 0) + even((size_t)tf * nc) * out_size + even((size_t)tf * nb) * mag_size +
         (staged ? (size_t)(nc + 1 + nnz) * 4 : 0);
}

bool valid_norm(int kind, double p) {
  return kind >= B2L_CHROMA_NORM_NONE && kind <= B2L_CHROMA_NORM_P && (kind != B2L_CHROMA_NORM_P || p > 0);
}

template <class In, class Out>
int fold(b2l_ctx* c, b2l_chroma::FoldArgs a, int64_t n_clips) {
  auto fn = b2l_chroma::chroma_fold_kernel<In, Out>;
  const size_t mag = sizeof(typename b2l_chroma::Mag<In>::R);
  const size_t map_bytes = (size_t)a.nnz * 12 + (a.n_chroma + 1) * 4;
  a.staged_map = map_bytes <= kMapCap;
  DeviceGuard g(c->device);
  // frames per block: kFoldFrames, fewer when a tall input (thousands of bins) would not fit the opt-in limit
  const size_t limit = c->smem_optin - kStaticSmem;
  int tf = kFoldFrames;
  while (tf > 1 && fold_smem_bytes(tf, a.n_bins, a.n_chroma, a.nnz, a.staged_map, sizeof(Out), mag) > limit) tf /= 2;
  const size_t smem = fold_smem_bytes(tf, a.n_bins, a.n_chroma, a.nnz, a.staged_map, sizeof(Out), mag);
  if (smem > limit) return fail(B2L_ERR_UNSUPPORTED, "chroma: %d input bins do not fit shared memory", a.n_bins);
  a.tf = tf;
  const long long tiles = (a.T + tf - 1) / tf;
  if (tiles > 0x7fffffffLL) return fail(B2L_ERR_UNSUPPORTED, "chroma: too many frames");
  if (int rc = blocks_per_sm(c, fn, kThreads, smem, nullptr, limit)) return rc;
  return for_clip_slices(n_clips, [&](int64_t c0, int64_t m) {
    a.clip0 = c0;
    return launch(c, fn, dim3((unsigned)tiles, (unsigned)m), kThreads, smem, a);
  });
}

template <class T>
int smooth(b2l_ctx* c, b2l_chroma::SmoothArgs a, int64_t n_clips, int win_len) {
  auto fn = b2l_chroma::chroma_smooth_kernel<T>;
  const int ts = kSmoothFrames;
  const size_t base = ts * 8 + (size_t)ts * a.n_chroma * sizeof(T);
  size_t smem = base + (size_t)a.n_chroma * (ts + win_len - 1) * sizeof(T);
  a.span = ts + win_len - 1;
  if (smem > c->smem_optin || smem > 96 * 1024) {   // a long window with many rows: read the rows through L1
    smem = base;
    a.span = 0;
  }
  a.ts = ts;
  const long long tiles = (a.T + ts - 1) / ts;
  DeviceGuard g(c->device);
  if (int rc = blocks_per_sm(c, fn, kThreads, smem, nullptr)) return rc;
  return for_clip_slices(n_clips, [&](int64_t c0, int64_t m) {
    a.clip0 = c0;
    return launch(c, fn, dim3((unsigned)tiles, (unsigned)m), kThreads, smem, a);
  });
}

}  // namespace

extern "C" int b2l_chroma_fold(b2l_ctx* c, const b2l_chroma_desc* d, const void* d_in, int64_t n_clips,
                               int64_t n_frames, void* d_out) {
  if (!c || !d || !d_in || !d_out || !d->d_row_ptr || !d->d_cols || !d->d_weights) return fail(B2L_ERR_INVALID, "NULL argument");
  if (d->input < B2L_CHROMA_IN_C64_FT || d->input > B2L_CHROMA_IN_F64_C || d->n_bins < 1 || d->n_chroma < 1 ||
      d->nnz < 0 || n_clips < 0 || n_frames < 0 || !valid_norm(d->norm, d->norm_p) ||
      d->epilogue < B2L_CHROMA_PLAIN || d->epilogue > B2L_CHROMA_TONNETZ || (d->epilogue == B2L_CHROMA_TONNETZ && !d->d_phi) ||
      (d->epilogue == B2L_CHROMA_CENS && !valid_norm(d->post_norm, d->post_p)))
    return fail(B2L_ERR_INVALID, "chroma: bad descriptor");
  if (n_clips == 0 || n_frames == 0) return B2L_OK;
  b2l_chroma::FoldArgs a{};
  a.in = d_in;
  a.ft = d->input == B2L_CHROMA_IN_C64_FT || d->input == B2L_CHROMA_IN_F32_FT || d->input == B2L_CHROMA_IN_F64_FT;
  a.n_bins = d->n_bins;
  a.n_chroma = d->n_chroma;
  a.T = n_frames;
  a.row_ptr = d->d_row_ptr;
  a.cols = d->d_cols;
  a.weights = d->d_weights;
  a.nnz = d->nnz;
  a.norm = d->norm;
  a.norm_p = d->norm_p;
  a.has_threshold = d->has_threshold;
  a.threshold = d->threshold;
  a.epilogue = d->epilogue;
  a.post_norm = d->epilogue == B2L_CHROMA_CENS ? d->post_norm : B2L_CHROMA_NORM_NONE;
  a.post_p = d->post_p;
  a.phi = d->d_phi;
  a.out = d_out;
  a.status = c->d_status;
  const bool f64 = d->out_f64 != 0;
  switch (d->input) {
    case B2L_CHROMA_IN_C64_FT: return f64 ? fold<float2, double>(c, a, n_clips) : fold<float2, float>(c, a, n_clips);
    case B2L_CHROMA_IN_F32_FT:
    case B2L_CHROMA_IN_F32_C: return f64 ? fold<float, double>(c, a, n_clips) : fold<float, float>(c, a, n_clips);
    default: return f64 ? fold<double, double>(c, a, n_clips) : fold<double, float>(c, a, n_clips);
  }
}

extern "C" int b2l_chroma_smooth(b2l_ctx* c, const void* d_in, int64_t n_clips, int32_t n_chroma, int64_t n_frames,
                                 int32_t f64, const int32_t* d_tap_off, const double* d_tap_w, int32_t n_taps,
                                 int32_t win_len, int32_t norm, double norm_p, void* d_out) {
  if (!c || !d_in || !d_out || (n_taps > 0 && (!d_tap_off || !d_tap_w))) return fail(B2L_ERR_INVALID, "NULL argument");
  if (n_chroma < 1 || n_clips < 0 || n_frames < 0 || n_taps < 0 || win_len < 1 || n_taps > win_len ||
      !valid_norm(norm, norm_p))
    return fail(B2L_ERR_INVALID, "chroma_smooth: bad arguments");
  if (n_clips == 0 || n_frames == 0) return B2L_OK;
  b2l_chroma::SmoothArgs a{};
  a.in = d_in;
  a.n_chroma = n_chroma;
  a.T = n_frames;
  a.reach = win_len - 1 - win_len / 2;
  a.tap_off = d_tap_off;
  a.tap_w = d_tap_w;
  a.n_taps = n_taps;
  a.norm = norm;
  a.norm_p = norm_p;
  a.out = d_out;
  return f64 ? smooth<double>(c, a, n_clips, win_len) : smooth<float>(c, a, n_clips, win_len);
}
