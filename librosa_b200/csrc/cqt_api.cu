// cqt_api.cu — C ABI of the constant-Q filter-bank projection (cqt_kernels.cuh): librosa.cqt / vqt / pseudo_cqt /
// hybrid_cqt (librosa/core/constantq.py:209-590, 820-1266).  The only unit that includes cqt_kernels.cuh.
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>

#include "cqt_kernels.cuh"
#include "internal.h"

using namespace b2l;

namespace {

// Largest octave table (nonzeros and row offsets) staged in shared memory; a denser basis (sparsity=0 at a large
// n_fft) is read from global memory through L1 instead.
const size_t kStageCap = 48 * 1024;

size_t table_bytes(const b2l_cqt_octave& o) { return (size_t)o.nnz * (sizeof(float2) + sizeof(int)) + (o.n_rows + 1) * 4; }


// b2l_cqt_project (complex64 out, complex octaves only) and b2l_cqt_project_abs (float32 magnitudes out).
int project(b2l_ctx* c, const b2l_cqt_octave* h_oct, int32_t n_oct, const int32_t* d_indptr, const int32_t* d_indices,
            const void* d_data, const double* d_rscale, int64_t n_clips, int64_t n_frames, int32_t n_bins, void* d_out,
            bool mag) {
  if (!c || !h_oct || !d_indptr || !d_indices || !d_data || !d_out) return fail(B2L_ERR_INVALID, "NULL argument");
  if (n_oct < 1 || n_oct > B2L_CQT_MAX_OCTAVES)
    return fail(B2L_ERR_UNSUPPORTED, "cqt: %d octaves; the projection takes 1 to %d", n_oct, B2L_CQT_MAX_OCTAVES);
  if (n_clips < 0 || n_frames < 0 || n_bins < 1) return fail(B2L_ERR_INVALID, "cqt: bad output geometry");
  b2l_cqt::ProjectArgs a;
  size_t smem = 0;
  long long tiles = 0;
  for (int o = 0; o < n_oct; ++o) {
    const b2l_cqt_octave& h = h_oct[o];
    if (!h.d_D || h.n_rows < 1 || h.row0 < 0 || h.row0 + h.n_rows > n_bins || h.nnz < 0 || h.indptr_off < 0 ||
        h.n_fft_bins < 1 || h.n_frames < n_frames || (h.kind & ~(B2L_CQT_PSEUDO | B2L_CQT_DIVIDE)) != 0)
      return fail(B2L_ERR_INVALID, "cqt: bad descriptor of octave %d", o);
    if ((h.kind & B2L_CQT_PSEUDO) && !mag)
      return fail(B2L_ERR_INVALID, "cqt: octave %d is a pseudo (magnitude) octave; use b2l_cqt_project_abs", o);
    b2l_cqt::Octave& d = a.oct[o];
    d.D = (const float2*)h.d_D;
    d.T_o = h.n_frames;
    d.F = h.n_fft_bins;
    d.row0 = h.row0;
    d.n_rows = h.n_rows;
    d.indptr_off = h.indptr_off;
    d.nnz = h.nnz;
    d.kind = h.kind;
    d.tile0 = tiles;
    tiles += (n_frames * h.n_rows + b2l_cqt::kThreads - 1) / b2l_cqt::kThreads;
    smem = std::max(smem, table_bytes(h));
  }
  if (n_clips == 0 || n_frames == 0) return B2L_OK;
  if (tiles > 0x7fffffffLL) return fail(B2L_ERR_UNSUPPORTED, "cqt: too many frames");
  a.n_oct = n_oct;
  a.indptr = d_indptr;
  a.indices = d_indices;
  a.data = (const float2*)d_data;
  a.rscale = d_rscale;
  a.T = n_frames;
  a.n_bins = n_bins;
  a.mag = mag;
  a.out = d_out;
  a.staged = smem <= kStageCap;
  if (!a.staged) smem = 0;
  DeviceGuard g(c->device);
  if (int rc = blocks_per_sm(c, b2l_cqt::cqt_project_kernel, b2l_cqt::kThreads, smem, nullptr)) return rc;
  return for_clip_slices(n_clips, [&](int64_t c0, int64_t m) {
    a.clip0 = c0;
    return launch(c, b2l_cqt::cqt_project_kernel, dim3((unsigned)tiles, (unsigned)m), b2l_cqt::kThreads, smem, a);
  });
}

}  // namespace

static_assert(sizeof(b2l_cqt_octave) == 40, "b2l_cqt_octave is part of the C ABI");
static_assert(b2l_cqt::kPseudo == B2L_CQT_PSEUDO && b2l_cqt::kDivide == B2L_CQT_DIVIDE, "octave kind bits");

extern "C" int b2l_cqt_project(b2l_ctx* c, const b2l_cqt_octave* h_oct, int32_t n_oct, const int32_t* d_indptr,
                               const int32_t* d_indices, const void* d_data, const double* d_rscale, int64_t n_clips,
                               int64_t n_frames, int32_t n_bins, void* d_out) {
  return project(c, h_oct, n_oct, d_indptr, d_indices, d_data, d_rscale, n_clips, n_frames, n_bins, d_out, false);
}

extern "C" int b2l_cqt_project_abs(b2l_ctx* c, const b2l_cqt_octave* h_oct, int32_t n_oct, const int32_t* d_indptr,
                                   const int32_t* d_indices, const void* d_data, const double* d_rscale,
                                   int64_t n_clips, int64_t n_frames, int32_t n_bins, float* d_out) {
  return project(c, h_oct, n_oct, d_indptr, d_indices, d_data, d_rscale, n_clips, n_frames, n_bins, d_out, true);
}
