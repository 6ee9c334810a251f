// cqt_kernels.cuh — the filter-bank projection of librosa.cqt / vqt / pseudo_cqt / hybrid_cqt
// (librosa/core/constantq.py:1197-1223, 474-590 and the stacking of __trim_stack, :1169-1194).
//
//   cqt_project_kernel   every octave's fft_basis.dot(D) into one [clip][T][n_bins] output, scale included; complex64
//                        out (cqt / vqt), or float32 |.| out (pseudo_cqt / hybrid_cqt)
//
// The octaves' complex64 CSR bases are concatenated: row r of octave o spans nonzeros
// indptr[o.indptr_off + r] .. indptr[o.indptr_off + r + 1] of indices / data (absolute positions).  A block serves one
// clip and 256 consecutive (frame, row) elements of one octave, rows fastest, so its writes run along the bin axis of
// the "ft" output and each thread writes one element exactly once.  The block first copies its octave's nonzeros to
// shared memory (when the largest octave table fits), then every thread sums its row's nonzeros in ascending column
// order, starting from zero, with unfused single-precision multiplies and adds: the order and the rounding of
// SciPy's csr_matvecs for complex64, so the result equals `csr @ D` bit for bit.  A frame's D row is read through
// L1: the threads on the same frame read overlapping bands of it, and at most two blocks share a frame.
//
// A pseudo octave (kPseudo) holds the real |basis| in the real parts of the same table and projects |D|: each row
// sums w * np_abs(D[t][col]) in the same order with unfused float32 operations, SciPy's float32 csr_matvecs on
// np.abs(D).  The row scale is one double operation rounded once, as numpy's float32 (*= or /=) float64 array does:
// a multiply, or with kDivide a divide (pseudo_cqt's C /= sqrt(n_fft)).  With `mag`, a complex row stores np_abs of
// the complex64 value it would otherwise store (np.abs(cqt(...))) and a pseudo row its real sum.
#pragma once
#include <math.h>
#include <stdint.h>

namespace b2l_cqt {

constexpr int kMaxOctaves = 32;   // B2L_CQT_MAX_OCTAVES
constexpr int kThreads = 256;
constexpr int kPseudo = 1;      // B2L_CQT_PSEUDO
constexpr int kDivide = 0x10;   // B2L_CQT_DIVIDE

// np.abs of complex64 as NumPy's vectorised loop computes it on x86 (AVX2 / AVX-512 with FMA): the larger part
// times sqrt(fma(r, r, 1)), r the smaller part over the larger, in float32.  It is not always the correctly rounded
// |z| (about a third of random inputs differ from it by one ulp), so the projection does not use the chroma fold's
// correctly rounded Mag, nor plp's cabs_ (hypotf, numerics.cuh).
__device__ __forceinline__ float np_abs(float2 v) {
  const float re = fabsf(v.x), im = fabsf(v.y);
  if (isinf(re) || isinf(im)) return INFINITY;
  if (isnan(re) || isnan(im)) return NAN;
  const float big = fmaxf(re, im), small = fminf(re, im);
  if (big == 0.0f) return 0.0f;
  const float r = __fdiv_rn(small, big);
  return __fmul_rn(__fsqrt_rn(__fmaf_rn(r, r, 1.0f)), big);
}

struct Octave {
  const float2* D;     // [n_clips][T_o][F]
  long long T_o;
  long long tile0;     // first block (x) of this octave
  int F, row0, n_rows, indptr_off, nnz;
  int kind;            // kPseudo and / or kDivide bits
};

struct ProjectArgs {
  Octave oct[kMaxOctaves];
  int n_oct;
  const int* indptr;
  const int* indices;
  const float2* data;
  const double* rscale;   // [n_bins] per-row scale (multiplier, divisor for kDivide octaves), or nullptr: none
  long long T;            // frames written: min over the octaves
  int n_bins;
  int staged;             // nonzeros copied to shared memory
  long long clip0;        // first clip of this launch (blockIdx.y = clip - clip0)
  int mag;                // out holds float32 magnitudes, else complex64
  void* out;              // [n_clips][T][n_bins]
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
  if (d.kind & kPseudo) {
    for (int k = ptr[r] - sub; k < k1; ++k)
      re = __fadd_rn(re, __fmul_rn(val[k].x, np_abs(__ldg(Dt + idx[k]))));
  } else {
    for (int k = ptr[r] - sub; k < k1; ++k) {
      const float2 v = val[k];
      const float2 x = __ldg(Dt + idx[k]);
      re = __fadd_rn(re, __fsub_rn(__fmul_rn(v.x, x.x), __fmul_rn(v.y, x.y)));
      im = __fadd_rn(im, __fadd_rn(__fmul_rn(v.x, x.y), __fmul_rn(v.y, x.x)));
    }
  }
  const int row = d.row0 + r;
  if (a.rscale) {   // one double operation per part, one rounding; numpy's complex64 /= float64 divides by (s + 0j),
    const double s = __ldg(a.rscale + row);   // which is a multiply by the table's 1 / s
    if (d.kind & kDivide) {
      re = __double2float_rn(__ddiv_rn((double)re, s));
      im = __double2float_rn(__ddiv_rn((double)im, s));
    } else {
      re = __double2float_rn(__dmul_rn((double)re, s));
      im = __double2float_rn(__dmul_rn((double)im, s));
    }
  }
  const long long at = (clip * a.T + t) * a.n_bins + row;
  if (a.mag)
    static_cast<float*>(a.out)[at] = (d.kind & kPseudo) ? re : np_abs(make_float2(re, im));
  else
    static_cast<float2*>(a.out)[at] = make_float2(re, im);
}

}  // namespace b2l_cqt
