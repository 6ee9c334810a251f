// align_api.cu — C ABI of the alignment kernels (align_kernels.cuh): librosa.sequence.dtw, dtw_backtracking and rqa
// (librosa/sequence.py:185-1075).  The only unit that includes align_kernels.cuh.
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>

#include "align_kernels.cuh"
#include "internal.h"

using namespace b2l;

namespace {

using b2l_align::kTile;

// One launch per anti-diagonal of kTile x kTile tiles, in order.
template <class Rule>
int run_waves(b2l_ctx* c, const Rule& rule, int64_t n, int64_t m) {
  const long long tn = (n + kTile - 1) / kTile, tm = (m + kTile - 1) / kTile;
  for (long long w = 0; w < tn + tm - 1; ++w) {
    const long long lo = std::max(0LL, w - (tm - 1)), hi = std::min(w, tn - 1);
    if (int rc = launch(c, b2l_align::wave_kernel<kTile, Rule>, dim3((unsigned)(hi - lo + 1)), dim3(kTile), 0, rule, w,
                        lo))
      return rc;
  }
  return B2L_OK;
}

int check_geometry(int64_t n, int64_t m) {
  if (n < 1 || m < 1) return fail(B2L_ERR_INVALID, "alignment: empty %lld x %lld matrix", (long long)n, (long long)m);
  if ((n + kTile - 1) / kTile > 0x7fffffffLL) return fail(B2L_ERR_UNSUPPORTED, "alignment: too many rows");
  return B2L_OK;
}

int check_steps(const b2l_dtw_desc* d) {
  if (d->n_steps < 1 || !d->h_steps || !d->h_w_add || !d->h_w_mul) return fail(B2L_ERR_INVALID, "dtw: no step table");
  for (int k = 0; k < d->n_steps; ++k)
    if (d->h_steps[2 * k] < 0 || d->h_steps[2 * k + 1] < 0) return fail(B2L_ERR_INVALID, "dtw: negative step");
  return B2L_OK;
}

// The step table as two device columns (rows, columns) in one stream-ordered temporary.
int upload_steps(Temp& t, const b2l_dtw_desc* d, const long long** sa, const long long** sb) {
  std::vector<long long> h(2 * (size_t)d->n_steps);
  for (int k = 0; k < d->n_steps; ++k) {
    h[k] = d->h_steps[2 * k];
    h[d->n_steps + k] = d->h_steps[2 * k + 1];
  }
  CUDA_TRY(upload(t, h.data(), h.size()));
  *sa = (const long long*)t.p;
  *sb = *sa + d->n_steps;
  return B2L_OK;
}

}  // namespace

extern "C" int b2l_dtw_cost(b2l_ctx* c, const b2l_dtw_cost_desc* d, const void* d_x, const void* d_y, double* d_C,
                            int32_t* d_flags) {
  if (!c || !d) return fail(B2L_ERR_INVALID, "NULL argument");
  if (d->K < 1 || d->N < 1 || d->M < 1) return fail(B2L_ERR_INVALID, "dtw: bad cost geometry");
  if (d->metric < B2L_DTW_EUCLIDEAN || d->metric > B2L_DTW_COSINE)
    return fail(B2L_ERR_INVALID, "dtw: unknown metric %d", d->metric);
  if (!d_x || !d_y || !d_C || !d_flags || !d->h_x_off || !d->h_y_off) return fail(B2L_ERR_INVALID, "NULL pointer");
  if ((d->M + 255) / 256 > 0x7fffffffLL) return fail(B2L_ERR_UNSUPPORTED, "dtw: too many columns");
  DeviceGuard g(c->device);
  Temp off(c->stream);
  std::vector<long long> h(2 * (size_t)d->K);
  std::copy(d->h_x_off, d->h_x_off + d->K, h.begin());
  std::copy(d->h_y_off, d->h_y_off + d->K, h.begin() + d->K);
  CUDA_TRY(upload(off, h.data(), h.size()));
  b2l_align::CostArgs a;
  a.x = d_x;
  a.y = d_y;
  a.x_off = (const long long*)off.p;
  a.y_off = a.x_off + d->K;
  a.K = d->K;
  a.N = d->N;
  a.M = d->M;
  a.transpose = d->transpose;
  a.C = d_C;
  a.flags = d_flags;
  using namespace b2l_align;
  void (*fn)(CostArgs);
#define B2L_COST(M) fn = d->f64 ? dtw_cost_kernel<double, M> : dtw_cost_kernel<float, M>; break;
  switch (d->metric) {
    case B2L_DTW_EUCLIDEAN: B2L_COST(kEuclidean)
    case B2L_DTW_SQEUCLIDEAN: B2L_COST(kSqEuclidean)
    case B2L_DTW_CITYBLOCK: B2L_COST(kCityblock)
    case B2L_DTW_CHEBYSHEV: B2L_COST(kChebyshev)
    default: B2L_COST(kCosine)
  }
#undef B2L_COST
  const dim3 grid((unsigned)((d->M + 255) / 256), (unsigned)std::min<int64_t>(d->N, kMaxGridY));
  return launch(c, fn, grid, dim3(256), 0, a);
}

extern "C" int b2l_nan_flag(b2l_ctx* c, const void* d_x, int64_t n, int32_t f64, int32_t* d_flags) {
  if (!c || n < 0) return fail(B2L_ERR_INVALID, "bad argument");
  if (n == 0) return B2L_OK;
  if (!d_x || !d_flags) return fail(B2L_ERR_INVALID, "NULL device pointer");
  DeviceGuard g(c->device);
  const long long blocks = grid_stride_blocks(n, 256 * 8, (long long)c->sm_count * 8);
  if (f64) return launch(c, b2l_align::nan_flag_kernel<double>, dim3((unsigned)blocks), dim3(256), 0,
                         (const double*)d_x, (long long)n, (int*)d_flags);
  return launch(c, b2l_align::nan_flag_kernel<float>, dim3((unsigned)blocks), dim3(256), 0, (const float*)d_x,
                (long long)n, (int*)d_flags);
}

extern "C" int b2l_dtw_accumulate(b2l_ctx* c, const b2l_dtw_desc* d, const void* d_C, double* d_D, int32_t* d_steps) {
  if (!c || !d) return fail(B2L_ERR_INVALID, "NULL argument");
  if (int rc = check_geometry(d->n, d->m)) return rc;
  if (int rc = check_steps(d)) return rc;
  if (!d_C || !d_D || !d_steps) return fail(B2L_ERR_INVALID, "NULL device pointer");
  DeviceGuard g(c->device);
  Temp steps(c->stream), w(c->stream);
  const long long *sa, *sb;
  if (int rc = upload_steps(steps, d, &sa, &sb)) return rc;
  std::vector<double> hw(2 * (size_t)d->n_steps);
  bool skip = true;
  for (int k = 0; k < d->n_steps; ++k) {
    hw[k] = d->h_w_add[k];
    hw[d->n_steps + k] = d->h_w_mul[k];
    skip &= d->h_w_mul[k] > 0;
  }
  CUDA_TRY(upload(w, hw.data(), hw.size()));
  auto fill = [&](auto& r) {
    r.D = d_D;
    r.steps = d_steps;
    r.sa = sa;
    r.sb = sb;
    r.w_add = (const double*)w.p;
    r.w_mul = r.w_add + d->n_steps;
    r.n = d->n;
    r.m = d->m;
    r.n_steps = d->n_steps;
    r.subseq = d->subseq;
    r.band = d->band;
    r.skip_outside = skip;
    r.band_lo = d->band_lo;
    r.band_hi = d->band_hi;
  };
  if (d->c_f64) {
    b2l_align::DtwRule<double> r;
    fill(r);
    r.C = (const double*)d_C;
    return run_waves(c, r, d->n, d->m);
  }
  b2l_align::DtwRule<float> r;
  fill(r);
  r.C = (const float*)d_C;
  return run_waves(c, r, d->n, d->m);
}

extern "C" int b2l_dtw_backtrack(b2l_ctx* c, const b2l_dtw_desc* d, const int32_t* d_steps, const double* d_D,
                                 int64_t start, int32_t check_end, int32_t flip, const int32_t* d_flags,
                                 int64_t* d_wp, int64_t* d_len) {
  if (!c || !d) return fail(B2L_ERR_INVALID, "NULL argument");
  if (int rc = check_geometry(d->n, d->m)) return rc;
  if (int rc = check_steps(d)) return rc;
  if (start >= d->m) return fail(B2L_ERR_INVALID, "dtw: start column %lld past %lld", (long long)start, (long long)d->m);
  if (!d_steps || !d_wp || !d_len) return fail(B2L_ERR_INVALID, "NULL device pointer");
  DeviceGuard g(c->device);
  Temp steps(c->stream);
  b2l_align::WalkArgs a;
  if (int rc = upload_steps(steps, d, &a.sa, &a.sb)) return rc;
  a.steps = d_steps;
  a.D = d_D;
  a.n_steps = d->n_steps;
  a.n = d->n;
  a.m = d->m;
  a.subseq = d->subseq;
  a.start = start;
  a.check_end = check_end;
  a.flip = flip;
  a.flags = d_flags;
  a.wp = (long long*)d_wp;
  a.len = (long long*)d_len;
  return launch(c, b2l_align::dtw_walk_kernel, dim3(1), dim3(32), 0, a);
}

extern "C" int b2l_rqa(b2l_ctx* c, const void* d_sim, int64_t n, int64_t m, int32_t f64, double gap_onset,
                       double gap_extend, int32_t knight, void* d_score, int8_t* d_ptr) {
  if (!c) return fail(B2L_ERR_INVALID, "NULL argument");
  if (int rc = check_geometry(n, m)) return rc;
  if (!d_sim || !d_score || !d_ptr) return fail(B2L_ERR_INVALID, "NULL device pointer");
  DeviceGuard g(c->device);
  auto fill = [&](auto& r, auto* sim, auto* score) {
    r.sim = sim;
    r.score = score;
    r.ptr = (signed char*)d_ptr;
    r.n = n;
    r.m = m;
    r.gap_onset = gap_onset;
    r.gap_extend = gap_extend;
    r.knight = knight;
  };
  if (f64) {
    b2l_align::RqaRule<double> r;
    fill(r, (const double*)d_sim, (double*)d_score);
    return run_waves(c, r, n, m);
  }
  b2l_align::RqaRule<float> r;
  fill(r, (const float*)d_sim, (float*)d_score);
  return run_waves(c, r, n, m);
}

extern "C" int b2l_rqa_path(b2l_ctx* c, const void* d_score, const int8_t* d_ptr, int64_t n, int64_t m, int32_t f64,
                            uint64_t* d_path, int64_t* d_len) {
  if (!c) return fail(B2L_ERR_INVALID, "NULL argument");
  if (int rc = check_geometry(n, m)) return rc;
  if (!d_score || !d_ptr || !d_path || !d_len) return fail(B2L_ERR_INVALID, "NULL device pointer");
  DeviceGuard g(c->device);
  using namespace b2l_align;
  const long long total = (long long)n * m;
  const int parts = (int)std::min<long long>((total + 4095) / 4096, (long long)c->sm_count * 16);
  const long long per = (total + parts - 1) / parts;
  Temp part(c->stream);
  CUDA_TRY(part.alloc((size_t)parts * (sizeof(double) + sizeof(long long))));
  double* pv = (double*)part.p;
  long long* pi = (long long*)(pv + parts);
  int rc = f64 ? launch(c, rqa_argmax_kernel<double>, dim3(parts), dim3(kArgThreads), 0, (const double*)d_score, total,
                        per, pv, pi)
               : launch(c, rqa_argmax_kernel<float>, dim3(parts), dim3(kArgThreads), 0, (const float*)d_score, total,
                        per, pv, pi);
  if (rc) return rc;
  return launch(c, rqa_walk_kernel, dim3(1), dim3(kArgThreads), 0,
                (const signed char*)d_ptr, (long long)n, (long long)m, (const double*)pv, (const long long*)pi, parts,
                (unsigned long long*)d_path, (long long*)d_len);
}
