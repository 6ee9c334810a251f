// neighbors_api.cu — C ABI of the nearest-neighbour kernels (neighbors_kernels.cuh, include/b2l.h):
// librosa.segment.recurrence_matrix as a neighbour table and librosa.decompose.nn_filter's aggregation.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <algorithm>
#include <vector>

#include "internal.h"
#include "neighbors_kernels.cuh"

using namespace b2l;

static_assert(kNnMaxM == B2L_NN_MAX_CANDIDATES, "candidate limit");
static_assert(kNnStatsMax == B2L_NN_MAX_STATS, "statistics limit");

// Workspace of one row block: at most this many distances (256 MiB).
static constexpr long long kNnBlockElems = 32LL << 20;

extern "C" int b2l_nn_graph(b2l_ctx* c, const b2l_nn_desc* d, const void* d_src, int64_t t, int32_t k_out,
                            int32_t* d_idx, double* d_val, int32_t* d_count, int32_t* h_not_finite) {
  if (!c || !d || !h_not_finite) return fail(B2L_ERR_INVALID, "NULL argument");
  *h_not_finite = 0;
  if (t < 2 || t > B2L_NN_MAX_FRAMES) return fail(B2L_ERR_UNSUPPORTED, "recurrence_matrix: %lld frames; 2 .. %d are supported",
                                                  (long long)t, B2L_NN_MAX_FRAMES);
  if (d->n_cand < 1 || d->n_cand > kNnMaxM || d->n_cand > t - 1)
    return fail(B2L_ERR_UNSUPPORTED, "recurrence_matrix: %d candidates per frame; 1 .. %d are supported", d->n_cand, kNnMaxM);
  if (d->k < 1 || d->width < 1 || d->mode < 0 || d->mode > 2 || d->metric < 0 || d->metric > 1)
    return fail(B2L_ERR_INVALID, "recurrence_matrix: bad descriptor");
  const int k_sel = std::min(d->k, d->n_cand);
  if (k_out < k_sel + 1) return fail(B2L_ERR_INVALID, "recurrence_matrix: the table needs %d columns", k_sel + 1);
  const bool stats = d->mode == 2 && d->bw_mode != B2L_NN_BW_SCALAR;
  if (stats && k_sel + 1 > kNnStatsMax)
    return fail(B2L_ERR_UNSUPPORTED, "recurrence_matrix: bandwidth statistics over %d links per frame; up to %d are "
                "supported", k_sel + 1, kNnStatsMax);
  if (d->n_lead < 1 || d->n_feat < 1) return fail(B2L_ERR_INVALID, "recurrence_matrix: no features");
  if (!d_src || !d_idx || !d_val || !d_count) return fail(B2L_ERR_INVALID, "NULL device pointer");
  DeviceGuard g(c->device);
  const long long D = d->n_lead * d->n_feat;
  Temp X(c->stream), norms(c->stream), bad(c->stream);
  CUDA_TRY(X.alloc((size_t)t * D * sizeof(double)));
  CUDA_TRY(norms.alloc((size_t)t * sizeof(double)));
  CUDA_TRY(bad.alloc(sizeof(int)));
  CUDA_TRY(cudaMemsetAsync(bad.p, 0, sizeof(int), c->stream));
  {
    const unsigned grid = (unsigned)grid_stride_blocks(t, 8, 16LL * c->sm_count);
    int rc = d->src_f64
                 ? launch(c, nn_pack_kernel<double>, grid, 256, 0, (const double*)d_src, (long long)d->n_lead,
                          (long long)d->n_feat, (long long)d->lead_stride, (long long)d->feat_stride,
                          (long long)d->frame_stride, (long long)t, (double*)X.p, (double*)norms.p, (int*)bad.p)
                 : launch(c, nn_pack_kernel<float>, grid, 256, 0, (const float*)d_src, (long long)d->n_lead,
                          (long long)d->n_feat, (long long)d->lead_stride, (long long)d->feat_stride,
                          (long long)d->frame_stride, (long long)t, (double*)X.p, (double*)norms.p, (int*)bad.p);
    if (rc) return rc;
  }
  int h_bad = 0;
  CUDA_TRY(cudaMemcpyAsync(&h_bad, bad.p, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  CUDA_TRY(cudaStreamSynchronize(c->stream));
  if (h_bad) {   // sklearn's check_array refuses the data: nothing is computed
    *h_not_finite = 1;
    return B2L_OK;
  }
  // row blocks: distances of `rows` query frames against all t, then their selection
  const long long tiles = (t + kNnTile - 1) / kNnTile;
  long long R = std::max(1LL, kNnBlockElems / t / kNnTile) * kNnTile;
  R = std::min(R, tiles * kNnTile);
  Temp W(c->stream), sidx(c->stream), sval(c->stream), scnt(c->stream);
  CUDA_TRY(W.alloc((size_t)R * t * sizeof(double)));
  CUDA_TRY(sidx.alloc((size_t)t * k_sel * sizeof(int)));
  CUDA_TRY(sval.alloc((size_t)t * k_sel * sizeof(double)));
  CUDA_TRY(scnt.alloc((size_t)t * sizeof(int)));
  int P = 1;
  while (P < d->n_cand) P <<= 1;
  const size_t sel_smem = (size_t)P * (sizeof(unsigned long long) + sizeof(int));
  cudaFuncAttributes fa;
  CUDA_TRY(cudaFuncGetAttributes(&fa, nn_select_kernel));   // its static shared memory comes off the opt-in limit
  int occ = 0;
  if (int rc = blocks_per_sm(c, nn_select_kernel, kNnSelectThreads, sel_smem, &occ, c->smem_optin - fa.sharedSizeBytes))
    return rc;
  if (occ < 1) return fail(B2L_ERR_UNSUPPORTED, "recurrence_matrix: %d candidates do not fit on an SM", d->n_cand);
  for (long long r0 = 0; r0 < t; r0 += R) {
    const int rows = (int)std::min(R, t - r0);
    NnDistArgs da;
    da.X = (const double*)X.p;
    da.norms = (const double*)norms.p;
    da.t = t;
    da.D = D;
    da.r0 = r0;
    da.rows = rows;
    da.cosine = d->metric == B2L_NN_COSINE;
    da.W = (double*)W.p;
    if (int rc = launch(c, nn_dist_kernel, dim3((unsigned)tiles, (unsigned)((rows + kNnTile - 1) / kNnTile)), 256, 0, da))
      return rc;
    NnSelectArgs sa;
    sa.W = (const double*)W.p;
    sa.t = t;
    sa.r0 = r0;
    sa.rows = rows;
    sa.M = d->n_cand;
    sa.P = P;
    sa.k = k_sel;
    sa.width = d->width;
    sa.mode = d->mode;
    sa.k_max = k_sel;
    sa.out_idx = (int*)sidx.p;
    sa.out_val = (double*)sval.p;
    sa.out_count = (int*)scnt.p;
    if (int rc = launch(c, nn_select_kernel, (unsigned)rows, kNnSelectThreads, sel_smem, sa)) return rc;
  }
  // the graph: sym, self links, and the bandwidth statistics of affinity mode
  Temp kth(c->stream), avg(c->stream), bw(c->stream);
  if (stats) {
    CUDA_TRY(kth.alloc((size_t)t * sizeof(double)));
    CUDA_TRY(avg.alloc((size_t)t * sizeof(double)));
  }
  CUDA_TRY(bw.alloc(sizeof(double)));
  NnGraphArgs ga;
  ga.in_idx = (const int*)sidx.p;
  ga.in_val = (const double*)sval.p;
  ga.in_count = (const int*)scnt.p;
  ga.k_in = k_sel;
  ga.t = t;
  ga.k = d->k;
  ga.mode = d->mode;
  ga.sym = d->sym;
  ga.self_link = d->self_link;
  ga.k_out = k_out;
  ga.out_idx = d_idx;
  ga.out_val = d_val;
  ga.out_count = d_count;
  ga.kth = stats ? (double*)kth.p : nullptr;
  ga.avg = stats ? (double*)avg.p : nullptr;
  const unsigned gg = (unsigned)grid_stride_blocks(t, 128, 8LL * c->sm_count);
  if (int rc = d->f64 ? launch(c, nn_graph_kernel<double>, gg, 128, 0, ga) : launch(c, nn_graph_kernel<float>, gg, 128, 0, ga))
    return rc;
  if (d->mode != 2) return B2L_OK;
  int bw_mode = 0;
  if (d->bw_mode == B2L_NN_BW_SCALAR) {
    CUDA_TRY(cudaMemcpyAsync(bw.p, &d->bandwidth, sizeof(double), cudaMemcpyHostToDevice, c->stream));
  } else if (d->bw_mode == B2L_NN_BW_MED_K_SCALAR) {
    if (int rc = d->f64 ? launch(c, nn_median_kernel<double>, 1, 1024, 0, (const double*)kth.p, (long long)t, (double*)bw.p)
                        : launch(c, nn_median_kernel<float>, 1, 1024, 0, (const double*)kth.p, (long long)t, (double*)bw.p))
      return rc;
    double h = 0;
    CUDA_TRY(cudaMemcpyAsync(&h, bw.p, sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(cudaStreamSynchronize(c->stream));
    if (isnan(h)) return fail(B2L_ERR_INVALID, "Cannot estimate bandwidth from an empty graph");
  } else {
    bw_mode = d->bw_mode;
    std::vector<int> cnt((size_t)t);
    CUDA_TRY(cudaMemcpyAsync(cnt.data(), d_count, (size_t)t * sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(cudaStreamSynchronize(c->stream));
    for (long long i = 0; i < t; ++i)
      if (cnt[i] == 0) return fail(B2L_ERR_INVALID, "The sample at time point %lld has no neighbors", i);
  }
  return d->f64 ? launch(c, nn_affinity_kernel<double>, gg, 128, 0, (const int*)d_idx, d_val, (const int*)d_count, (int)k_out,
                         (long long)t, bw_mode, (const double*)bw.p, (const double*)kth.p, (const double*)avg.p)
                : launch(c, nn_affinity_kernel<float>, gg, 128, 0, (const int*)d_idx, d_val, (const int*)d_count, (int)k_out,
                         (long long)t, bw_mode, (const double*)bw.p, (const double*)kth.p, (const double*)avg.p);
}

template <class T, class R>
static int launch_agg(b2l_ctx* c, const NnAggArgs& a, int max_n) {
  if (a.agg != B2L_NN_MEDIAN) {
    const unsigned by = (unsigned)((a.F + a.bins - 1) / a.bins);
    return launch(c, nn_agg_kernel<T, R>, dim3((unsigned)a.t, by, (unsigned)a.n_lead), 128, sizeof(R), a);
  }
  int P = 1;
  while (P < max_n) P <<= 1;
  const size_t per_warp = (size_t)P * sizeof(T);
  int nw = 8;
  while (nw > 1 && per_warp * nw > c->smem_optin) nw >>= 1;
  if (per_warp * nw > c->smem_optin)
    return fail(B2L_ERR_UNSUPPORTED, "nn_filter: the median of %d neighbours does not fit in shared memory", max_n);
  NnAggArgs b = a;
  b.bins = nw * 4;
  int occ = 0;
  if (int rc = blocks_per_sm(c, nn_agg_kernel<T, R>, nw * 32, per_warp * nw, &occ)) return rc;
  if (occ < 1) return fail(B2L_ERR_UNSUPPORTED, "nn_filter: the median of %d neighbours does not fit on an SM", max_n);
  const unsigned by = (unsigned)((b.F + b.bins - 1) / b.bins);
  return launch(c, nn_agg_kernel<T, R>, dim3((unsigned)b.t, by, (unsigned)b.n_lead), nw * 32, per_warp * nw, b);
}

extern "C" int b2l_nn_filter(b2l_ctx* c, const b2l_nn_filter_desc* d, const void* d_S, int64_t n_lead, int64_t t,
                             int64_t n_bins, const int64_t* d_start, const int32_t* d_count, const int32_t* d_idx,
                             const double* d_w, void* d_out, int32_t* h_zero_weight) {
  if (!c || !d) return fail(B2L_ERR_INVALID, "NULL argument");
  if (n_lead < 0 || t < 0 || n_bins < 0 || d->stride < 0) return fail(B2L_ERR_INVALID, "nn_filter: bad geometry");
  if (d->agg < B2L_NN_MEAN || d->agg > B2L_NN_AVERAGE) return fail(B2L_ERR_INVALID, "nn_filter: bad aggregate");
  if (t > 0x7fffffffLL || n_lead > 65535) return fail(B2L_ERR_UNSUPPORTED, "nn_filter: too many frames or channels");
  if (h_zero_weight) *h_zero_weight = 0;
  if (n_lead == 0 || t == 0 || n_bins == 0) return B2L_OK;
  if (!d_S || !d_count || !d_idx || !d_out || (d->agg == B2L_NN_AVERAGE && !d_w) || (!d_start && d->stride == 0))
    return fail(B2L_ERR_INVALID, "NULL device pointer");
  DeviceGuard g(c->device);
  Temp zero(c->stream);
  CUDA_TRY(zero.alloc(sizeof(int)));
  CUDA_TRY(cudaMemsetAsync(zero.p, 0, sizeof(int), c->stream));
  NnAggArgs a;
  a.S = d_S;
  a.out = d_out;
  a.t = t;
  a.F = n_bins;
  a.n_lead = n_lead;
  a.start = (const long long*)d_start;
  a.stride = d->stride;
  a.count = d_count;
  a.idx = d_idx;
  a.w = d_w;
  a.agg = d->agg;
  a.bins = 512;
  a.zero_weight = (int*)zero.p;
  int rc;
  if (d->s_f64) rc = launch_agg<double, double>(c, a, d->max_count);
  else if (d->r_f64) rc = launch_agg<float, double>(c, a, d->max_count);
  else rc = launch_agg<float, float>(c, a, d->max_count);
  if (rc) return rc;
  if (d->agg == B2L_NN_AVERAGE && h_zero_weight) {
    CUDA_TRY(cudaMemcpyAsync(h_zero_weight, zero.p, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(cudaStreamSynchronize(c->stream));
  }
  return B2L_OK;
}

extern "C" int b2l_nn_compact(b2l_ctx* c, const void* d_rec, int32_t elem, int64_t t, int32_t pass, int32_t* d_count,
                              const int64_t* d_start, int32_t* d_idx, double* d_w) {
  if (!c) return fail(B2L_ERR_INVALID, "NULL argument");
  if (t < 0 || t > 0x7fffffffLL || pass < 0 || pass > 1) return fail(B2L_ERR_INVALID, "nn_compact: bad arguments");
  if (t == 0) return B2L_OK;
  if (!d_rec || !d_count || (pass == 1 && (!d_start || !d_idx || !d_w))) return fail(B2L_ERR_INVALID, "NULL device pointer");
  DeviceGuard g(c->device);
  const unsigned grid = (unsigned)grid_stride_blocks(t, 128, 16LL * c->sm_count);
  switch (elem) {
    case B2L_ELEM_F32:
      return launch(c, nn_compact_kernel<float>, grid, 128, 0, (const float*)d_rec, (long long)t, (int)pass, d_count,
                    (const long long*)d_start, d_idx, d_w);
    case B2L_ELEM_F64:
      return launch(c, nn_compact_kernel<double>, grid, 128, 0, (const double*)d_rec, (long long)t, (int)pass, d_count,
                    (const long long*)d_start, d_idx, d_w);
    case B2L_ELEM_BOOL:
      return launch(c, nn_compact_kernel<bool>, grid, 128, 0, (const bool*)d_rec, (long long)t, (int)pass, d_count,
                    (const long long*)d_start, d_idx, d_w);
    default:
      return fail(B2L_ERR_UNSUPPORTED, "nn_compact: element type %d is not supported", elem);
  }
}

extern "C" int b2l_nn_dense(b2l_ctx* c, const int32_t* d_idx, const double* d_val, const int32_t* d_count, int64_t t,
                            int32_t k_out, int32_t elem, void* d_rec) {
  if (!c) return fail(B2L_ERR_INVALID, "NULL argument");
  if (t < 0 || k_out < 1) return fail(B2L_ERR_INVALID, "nn_dense: bad geometry");
  if (t == 0) return B2L_OK;
  if (!d_idx || !d_val || !d_count || !d_rec) return fail(B2L_ERR_INVALID, "NULL device pointer");
  DeviceGuard g(c->device);
  const size_t esize = elem == B2L_ELEM_F64 ? 8 : elem == B2L_ELEM_F32 ? 4 : 1;
  CUDA_TRY(cudaMemsetAsync(d_rec, 0, (size_t)t * t * esize, c->stream));
  const unsigned grid = (unsigned)grid_stride_blocks(t * k_out, 256, 16LL * c->sm_count);
  switch (elem) {
    case B2L_ELEM_F32:
      return launch(c, nn_dense_kernel<float>, grid, 256, 0, (const int*)d_idx, d_val, (const int*)d_count, (long long)t,
                    (int)k_out, (float*)d_rec);
    case B2L_ELEM_F64:
      return launch(c, nn_dense_kernel<double>, grid, 256, 0, (const int*)d_idx, d_val, (const int*)d_count, (long long)t,
                    (int)k_out, (double*)d_rec);
    case B2L_ELEM_BOOL:
      return launch(c, nn_dense_kernel<bool>, grid, 256, 0, (const int*)d_idx, d_val, (const int*)d_count, (long long)t,
                    (int)k_out, (bool*)d_rec);
    default:
      return fail(B2L_ERR_UNSUPPORTED, "nn_dense: element type %d is not supported", elem);
  }
}
