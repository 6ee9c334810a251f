// inverse_api.cu — feature.inverse on the device: mel spectrogram -> STFT magnitude by non-negative least squares
// (librosa/feature/inverse.py:28-114 -> librosa/util/_nnls.py:22-175).
//
// The reference minimises |A X - B|^2 over X >= 0 (A = mel basis, B = mel spectrogram, one independent problem
// per frame) with SciPy's L-BFGS-B started from the clipped pseudo-inverse solution; the problem is
// under-determined (1025 unknowns, 128 equations), so its result is one of many minimisers and the reference's
// own test only bounds the residual (tests/test_features.py:897-921: dtype, X >= 0, shape, RMSE <= 5e-2).
// Here: the same start X0 = max(0, pinv(A) B), then a fixed number of accelerated projected-gradient (FISTA)
// steps with step 1/sigma_max(A)^2 on the band-sparse basis — one warp per frame, iterate and residual in
// shared memory.  Measured against the live reference: the residual after 100 steps is at or below L-BFGS-B's.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <vector>

#include "common.cuh"
#include "internal.h"

using namespace b2l;

namespace {

struct BinRows { unsigned short ra, rb; float wa, wb; };   // the (at most two) mel rows a bin feeds

constexpr int NNLS_WARPS = 8;

// One warp per (clip, frame).  Dynamic shared memory: band table, weights, bin table, then per warp x, y, r, b.
__global__ void nnls_fista_kernel(const float* __restrict__ Mel, long long n_cols, int T, int n_mels, int F,
                                  const MelBand* __restrict__ band, const float* __restrict__ w, int w_count,
                                  const BinRows* __restrict__ bins, const float* __restrict__ pinv,
                                  const float* __restrict__ beta, int n_iter, float step, float inv_power,
                                  float* __restrict__ out) {
  extern __shared__ __align__(16) unsigned char sm[];
  MelBand* s_band = reinterpret_cast<MelBand*>(sm);
  float* s_w = reinterpret_cast<float*>(s_band + n_mels);
  BinRows* s_bins = reinterpret_cast<BinRows*>(s_w + ((w_count + 3) & ~3));
  float* s_work = reinterpret_cast<float*>(s_bins + F);
  for (int i = threadIdx.x; i < n_mels; i += blockDim.x) s_band[i] = band[i];
  for (int i = threadIdx.x; i < w_count; i += blockDim.x) s_w[i] = w[i];
  for (int i = threadIdx.x; i < F; i += blockDim.x) s_bins[i] = bins[i];
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int per_warp = 2 * F + 2 * n_mels;
  float* x = s_work + warp * per_warp;
  float* y = x + F;
  float* r = y + F;
  float* b = r + n_mels;
  for (long long col = (long long)blockIdx.x * NNLS_WARPS + warp; col < n_cols; col += (long long)gridDim.x * NNLS_WARPS) {
    const long long clip = col / T;
    const int t = (int)(col - clip * T);
    const float* mcol = Mel + clip * n_mels * T + t;
    for (int m = lane; m < n_mels; m += 32) b[m] = mcol[(long long)m * T];
    __syncwarp();
    // start: the projected least-squares solution max(0, pinv(A) b)   (_nnls.py:60-64)
    for (int k = lane; k < F; k += 32) {
      const float* prow = pinv + (long long)k * n_mels;
      float acc = 0.0f;
      for (int m = 0; m < n_mels; ++m) acc = fmaf(prow[m], b[m], acc);
      acc = fmaxf(acc, 0.0f);
      x[k] = acc;
      y[k] = acc;
    }
    __syncwarp();
    for (int it = 0; it < n_iter; ++it) {
      for (int m = lane; m < n_mels; m += 32) {          // r = A y - b on the band-sparse rows
        const MelBand bd = s_band[m];
        const float* wp = s_w + bd.off;
        const float* yp = y + bd.lo;
        float acc = -b[m];
        for (int i = 0; i < bd.len; ++i) acc = fmaf(wp[i], yp[i], acc);
        r[m] = acc;
      }
      __syncwarp();
      const float bt = beta[it];
      for (int k = lane; k < F; k += 32) {               // projected gradient step + momentum
        const BinRows br = s_bins[k];
        const float g = fmaf(br.wa, r[br.ra], br.wb * r[br.rb]);
        const float xn = fmaxf(0.0f, fmaf(-step, g, y[k]));
        y[k] = fmaf(bt, xn - x[k], xn);
        x[k] = xn;
      }
      __syncwarp();
    }
    float* ocol = out + clip * F * T + t;
    for (int k = lane; k < F; k += 32) {
      const float v = x[k];
      ocol[(long long)k * T] = inv_power == 1.0f ? v : (inv_power == 0.5f ? sqrtf(v) : powf(v, inv_power));
    }
    __syncwarp();
  }
}

}  // namespace

extern "C" int b2l_nnls_mel(b2l_ctx* c, const float* d_mel, int64_t n_clips, int64_t n_frames, int32_t n_mels,
                            int32_t n_bins, const float* h_basis, const float* h_pinv, float step, int32_t n_iter,
                            float inv_power, float* d_out) {
  if (!c || !d_mel || !h_basis || !h_pinv || !d_out) return fail(B2L_ERR_INVALID, "NULL argument");
  if (n_clips <= 0 || n_frames <= 0) return B2L_OK;
  if (n_mels < 1 || n_mels > 65535 || n_bins < 1 || n_iter < 0 || !(step > 0.0f))
    return fail(B2L_ERR_INVALID, "bad nnls geometry");
  DeviceGuard g(c->device);
  cudaStream_t st = c->stream;
  // band form of the rows and the transposed (bin -> rows) form
  std::vector<MelBand> bands((size_t)n_mels);
  std::vector<float> w;
  std::vector<BinRows> bins((size_t)n_bins, BinRows{0, 0, 0.0f, 0.0f});
  std::vector<int> used((size_t)n_bins, 0);
  bool too_dense = false;
  for (int m = 0; m < n_mels; ++m) {
    const float* row = h_basis + (size_t)m * n_bins;
    int lo = 0, hi = n_bins - 1;
    while (lo < n_bins && row[lo] == 0.0f) ++lo;
    while (hi >= lo && row[hi] == 0.0f) --hi;
    MelBand b;
    b.off = (int)w.size();
    b.pad = 0;
    b.lo = lo > hi ? 0 : lo;
    b.len = lo > hi ? 0 : hi - lo + 1;
    for (int k = b.lo; k < b.lo + b.len; ++k) {
      w.push_back(row[k]);
      if (row[k] != 0.0f) {
        BinRows& e = bins[(size_t)k];
        if (used[(size_t)k] == 0) { e.ra = (unsigned short)m; e.wa = row[k]; }
        else if (used[(size_t)k] == 1) { e.rb = (unsigned short)m; e.wb = row[k]; }
        else too_dense = true;
        ++used[(size_t)k];
      }
    }
    bands[(size_t)m] = b;
  }
  if (too_dense)
    return fail(B2L_ERR_UNSUPPORTED, "nnls: a frequency bin feeds more than two filters (not a triangular mel basis)");
  if (w.empty()) w.push_back(0.0f);
  // FISTA momentum coefficients (the same for every column)
  std::vector<float> beta((size_t)(n_iter > 0 ? n_iter : 1));
  double tk = 1.0;
  for (int i = 0; i < n_iter; ++i) {
    const double tn = 0.5 * (1.0 + sqrt(1.0 + 4.0 * tk * tk));
    beta[(size_t)i] = (float)((tk - 1.0) / tn);
    tk = tn;
  }
  Temp d_band(st), d_w(st), d_bins(st), d_pinv(st), d_beta(st);
  CUDA_TRY(upload(d_band, bands.data(), bands.size()));
  CUDA_TRY(upload(d_w, w.data(), w.size()));
  CUDA_TRY(upload(d_bins, bins.data(), bins.size()));
  CUDA_TRY(upload(d_pinv, h_pinv, (size_t)n_bins * n_mels));
  CUDA_TRY(upload(d_beta, beta.data(), beta.size()));
  const size_t smem = (size_t)n_mels * sizeof(MelBand) + ((w.size() + 3) & ~(size_t)3) * 4 + (size_t)n_bins * sizeof(BinRows) +
                      (size_t)NNLS_WARPS * (2 * (size_t)n_bins + 2 * (size_t)n_mels) * 4;
  if (smem > c->smem_optin) return fail(B2L_ERR_UNSUPPORTED, "nnls: n_fft too large for the shared-memory iterate");
  int rc = blocks_per_sm(c, nnls_fista_kernel, NNLS_WARPS * 32, smem, nullptr);
  if (rc) return rc;
  const long long cols = n_clips * n_frames;
  const long long grid = grid_stride_blocks(cols, NNLS_WARPS, 2LL * c->sm_count);
  return launch(c, nnls_fista_kernel, (unsigned)grid, NNLS_WARPS * 32, smem, d_mel, cols, (int)n_frames, n_mels, n_bins,
                (const MelBand*)d_band.p, (const float*)d_w.p, (int)w.size(), (const BinRows*)d_bins.p,
                (const float*)d_pinv.p, (const float*)d_beta.p, n_iter, step, inv_power, d_out);
}
