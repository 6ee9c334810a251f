// iirt_api.cu — C ABI of the semitone filter-bank spectrogram (iirt_kernels.cuh): librosa.iirt
// (librosa/core/spectrum.py:1522-1713).  The only unit that includes iirt_kernels.cuh.
#include <cuda_runtime.h>
#include <stdint.h>

#include "iirt_kernels.cuh"
#include "internal.h"

using namespace b2l;

namespace {

int fill_rates(const b2l_iirt_rate* h, int32_t n_rates, int64_t n_clips, b2l_iirt::Args& a) {
  if (!h) return fail(B2L_ERR_INVALID, "NULL argument");
  if (n_rates < 1 || n_rates > B2L_IIRT_MAX_RATES)
    return fail(B2L_ERR_UNSUPPORTED, "iirt: %d sampling rates; the kernels take 1 to %d", n_rates, B2L_IIRT_MAX_RATES);
  if (n_clips < 0) return fail(B2L_ERR_INVALID, "iirt: bad clip count");
  for (int r = 0; r < n_rates; ++r) {
    const b2l_iirt_rate& s = h[r];
    if (!s.d_x || !s.d_scratch || !s.d_bands || s.n_bands < 1 || s.n < 1 || s.x_stride < s.n ||
        s.scratch_stride < n_clips * s.n_bands)
      return fail(B2L_ERR_INVALID, "iirt: bad descriptor of rate %d", r);
    b2l_iirt::Rate& d = a.rate[r];
    d.x = s.d_x;
    d.x_stride = s.x_stride;
    d.n = s.n;
    d.scr = s.d_scratch;
    d.stride = s.scratch_stride;
    d.bands = s.d_bands;
    d.n_bands = s.n_bands;
    d.starts = s.d_starts;
    d.leaves = (const int4*)s.d_leaves;
    d.n_leaves = s.n_leaves;
    d.factor = s.factor;
  }
  a.n_rates = n_rates;
  a.n_clips = n_clips;
  return B2L_OK;
}

template <int NS>
int launch_filter(b2l_ctx* c, const b2l_iirt::Args& a, long long blocks) {
  return launch(c, b2l_iirt::sosfiltfilt_kernel<NS>, dim3((unsigned)blocks), b2l_iirt::kFilterThreads, 0, a);
}

}  // namespace

extern "C" int b2l_pad_center(b2l_ctx* c, const float* d_x, int64_t n_clips, int64_t n, int32_t pad, int32_t pad_mode,
                              float* d_out) {
  if (!c || !d_x || !d_out) return fail(B2L_ERR_INVALID, "NULL argument");
  if (n_clips < 0 || n < 0 || pad < 0 || pad_mode < B2L_PAD_CONSTANT || pad_mode > B2L_PAD_EMPTY)
    return fail(B2L_ERR_INVALID, "pad: bad geometry");
  if (n == 0 && pad > 0 && pad_mode != B2L_PAD_CONSTANT && pad_mode != B2L_PAD_EMPTY)
    return fail(B2L_ERR_INVALID, "pad: an empty signal can only be padded with zeros");
  if (n + 2LL * pad > 0x7fffffffLL) return fail(B2L_ERR_UNSUPPORTED, "signals longer than 2^31-1 samples");
  if (n_clips == 0 || n + 2LL * pad == 0) return B2L_OK;
  DeviceGuard g(c->device);
  const long long grid = grid_stride_blocks(n_clips * (n + 2LL * pad), 256, 32LL * c->sm_count);
  return launch(c, b2l_iirt::pad_center_kernel, dim3((unsigned)grid), 256, 0, d_x, (long long)n_clips, (int)n,
                (int)pad, (int)pad_mode, d_out);
}

extern "C" int b2l_iirt_filter(b2l_ctx* c, const b2l_iirt_rate* h_rates, int32_t n_rates, const double* d_coef,
                               const int32_t* d_info, int32_t max_sections, int64_t n_clips) {
  if (!c || !d_coef || !d_info) return fail(B2L_ERR_INVALID, "NULL argument");
  if (max_sections < 1 || max_sections > B2L_IIRT_MAX_SECTIONS)
    return fail(B2L_ERR_UNSUPPORTED, "iirt: %d second-order sections; the filter kernel takes 1 to %d", max_sections,
                B2L_IIRT_MAX_SECTIONS);
  b2l_iirt::Args a = {};
  if (int rc = fill_rates(h_rates, n_rates, n_clips, a)) return rc;
  a.coef = d_coef;
  a.info = d_info;
  long long blocks = 0;
  for (int r = 0; r < n_rates; ++r) {
    a.rate[r].block0 = blocks;
    blocks += (n_clips * a.rate[r].n_bands + b2l_iirt::kFilterThreads - 1) / b2l_iirt::kFilterThreads;
  }
  if (blocks == 0) return B2L_OK;
  if (blocks > 0x7fffffffLL) return fail(B2L_ERR_UNSUPPORTED, "iirt: too many chains");
  DeviceGuard g(c->device);
  switch (max_sections) {   // the kernel runs exactly the largest cascade of the launch
    case 1: return launch_filter<1>(c, a, blocks);
    case 2: return launch_filter<2>(c, a, blocks);
    case 3: return launch_filter<3>(c, a, blocks);
    case 4: return launch_filter<4>(c, a, blocks);
    case 5: return launch_filter<5>(c, a, blocks);
    case 6: return launch_filter<6>(c, a, blocks);
    case 7: return launch_filter<7>(c, a, blocks);
    case 8: return launch_filter<8>(c, a, blocks);
    case 9: return launch_filter<9>(c, a, blocks);
    default: return launch_filter<10>(c, a, blocks);
  }
}

extern "C" int b2l_iirt_stmsp(b2l_ctx* c, const b2l_iirt_rate* h_rates, int32_t n_rates, int64_t n_clips,
                              int64_t n_frames, int32_t n_bands, float* d_out) {
  if (!c || !d_out) return fail(B2L_ERR_INVALID, "NULL argument");
  if (n_frames < 0 || n_bands < 1) return fail(B2L_ERR_INVALID, "iirt: bad output geometry");
  b2l_iirt::Args a = {};
  if (int rc = fill_rates(h_rates, n_rates, n_clips, a)) return rc;
  a.T = n_frames;
  a.n_out_bands = n_bands;
  a.out = d_out;
  long long blocks = 0;
  for (int r = 0; r < n_rates; ++r) {
    const b2l_iirt_rate& s = h_rates[r];
    if (!s.d_starts || !s.d_leaves || s.n_leaves < 1) return fail(B2L_ERR_INVALID, "iirt: rate %d has no frame table", r);
    a.rate[r].sblock0 = blocks;
    blocks += (s.scratch_stride * n_frames + b2l_iirt::kStmspThreads - 1) / b2l_iirt::kStmspThreads;
  }
  if (blocks == 0) return B2L_OK;
  if (blocks > 0x7fffffffLL) return fail(B2L_ERR_UNSUPPORTED, "iirt: too many frames");
  DeviceGuard g(c->device);
  return launch(c, b2l_iirt::stmsp_kernel, dim3((unsigned)blocks), b2l_iirt::kStmspThreads, 0, a);
}
