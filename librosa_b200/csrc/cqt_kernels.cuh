// cqt_kernels.cuh — the filter-bank projection of librosa.cqt / vqt (librosa/core/constantq.py:1197-1223 and the
// stacking of __trim_stack, :1169-1194).
//
//   cqt_project_kernel   every octave's fft_basis.dot(D) into one [clip][T][n_bins] output, scale included
//
// The octaves' complex64 CSR bases are concatenated: row r of octave o spans nonzeros
// indptr[o.indptr_off + r] .. indptr[o.indptr_off + r + 1] of indices / data (absolute positions).  A block serves one
// clip and 256 consecutive (frame, row) elements of one octave, rows fastest, so its writes run along the bin axis of
// the "ft" output and each thread writes one element exactly once.  The block first copies its octave's nonzeros to
// shared memory (when the largest octave table fits), then every thread sums its row's nonzeros in ascending column
// order, starting from zero, with unfused single-precision multiplies and adds: the order and the rounding of
// SciPy's csr_matvecs for complex64, so the result equals `csr @ D` bit for bit.  A frame's D row is read through
// L1: the threads on the same frame read overlapping bands of it, and at most two blocks share a frame.
#pragma once
#include <stdint.h>

namespace b2l_cqt {

constexpr int kMaxOctaves = 32;   // B2L_CQT_MAX_OCTAVES
constexpr int kThreads = 256;

struct Octave {
  const float2* D;     // [n_clips][T_o][F]
  long long T_o;
  long long tile0;     // first block (x) of this octave
  int F, row0, n_rows, indptr_off, nnz;
};

struct ProjectArgs {
  Octave oct[kMaxOctaves];
  int n_oct;
  const int* indptr;
  const int* indices;
  const float2* data;
  const double* rscale;   // [n_bins] 1 / sqrt(lengths), or nullptr (scale=False)
  long long T;            // frames written: min over the octaves
  int n_bins;
  int staged;             // nonzeros copied to shared memory
  long long clip0;        // first clip of this launch (blockIdx.y = clip - clip0)
  float2* out;            // [n_clips][T][n_bins]
};

__global__ void __launch_bounds__(kThreads) cqt_project_kernel(const ProjectArgs a) {
  extern __shared__ __align__(16) unsigned char smem[];
  int o = 0;
  while (o + 1 < a.n_oct && (long long)blockIdx.x >= a.oct[o + 1].tile0) ++o;
  const Octave& d = a.oct[o];
  const int* ip = a.indptr + d.indptr_off;
  const int* ptr = ip;
  const int* idx = a.indices;
  const float2* val = a.data;
  int sub = 0;
  if (a.staged) {
    const int base = __ldg(ip);
    float2* s_val = reinterpret_cast<float2*>(smem);
    int* s_idx = reinterpret_cast<int*>(s_val + d.nnz);
    int* s_ptr = s_idx + d.nnz;
    for (int i = threadIdx.x; i < d.nnz; i += kThreads) {
      s_val[i] = __ldg(a.data + base + i);
      s_idx[i] = __ldg(a.indices + base + i);
    }
    for (int i = threadIdx.x; i <= d.n_rows; i += kThreads) s_ptr[i] = __ldg(ip + i);
    __syncthreads();
    ptr = s_ptr;
    idx = s_idx;
    val = s_val;
    sub = base;
  }
  const long long clip = a.clip0 + blockIdx.y;
  const long long flat = ((long long)blockIdx.x - d.tile0) * kThreads + threadIdx.x;
  const long long t = flat / d.n_rows;
  const int r = (int)(flat - t * d.n_rows);
  if (t >= a.T) return;
  const float2* Dt = d.D + (clip * d.T_o + t) * d.F;
  float re = 0.0f, im = 0.0f;
  const int k1 = ptr[r + 1] - sub;
  for (int k = ptr[r] - sub; k < k1; ++k) {
    const float2 v = val[k];
    const float2 x = __ldg(Dt + idx[k]);
    re = __fadd_rn(re, __fsub_rn(__fmul_rn(v.x, x.x), __fmul_rn(v.y, x.y)));
    im = __fadd_rn(im, __fadd_rn(__fmul_rn(v.x, x.y), __fmul_rn(v.y, x.x)));
  }
  const int row = d.row0 + r;
  if (a.rscale) {   // numpy's complex64 /= float64: complex128 division by (s + 0j) = multiply by 1 / s, one rounding
    const double s = __ldg(a.rscale + row);
    re = __double2float_rn(__dmul_rn((double)re, s));
    im = __double2float_rn(__dmul_rn((double)im, s));
  }
  a.out[(clip * a.T + t) * a.n_bins + row] = make_float2(re, im);
}

}  // namespace b2l_cqt
