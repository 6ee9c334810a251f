// internal.h — host-side state and helpers shared by the C ABI units (runtime.cu, plan.cu and the *_api.cu units:
// spectrum, feature, pitch, f64, inverse, ...) and the per-size kernel instantiations (fwd_inst.cu, inv_inst.cu, czt_inst.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <map>
#include <set>
#include <tuple>
#include <vector>

#include "../../include/b2l.h"
#include "common.cuh"
#include "fft_engine.cuh"

namespace b2l {

// Transform sizes with an instantiation unit: fwd_inst.cu / inv_inst.cu for LOG2M (n_fft = 2^(LOG2M+1): 8 .. 8192),
// czt_inst.cu for LOG2P (chirp-z transform size P = 2^LOG2P).  SIZES / CZT_SIZES in the Makefile list the same values.
#define B2L_FFT_SIZES(X) X(2) X(3) X(4) X(5) X(6) X(7) X(8) X(9) X(10) X(11) X(12)
#define B2L_CZT_SIZES(X) X(5) X(6) X(7) X(8) X(9) X(10) X(11) X(12)
constexpr int kMinLog2M = 2, kMaxLog2M = 12;

// The transform that serves a plan's n_fft, decided once by plan_path (plan.cu): fwd_kernel / inv_kernel for the
// powers of two, mr_kernel / mr_inv_kernel for the even sizes with a 5-smooth half, czt_kernel / czt_inv_kernel for
// the rest of 3 .. 2047.
enum Path { PATH_POW2, PATH_MR, PATH_CZT };

struct CztArgs;
struct CztInvArgs;
typedef void (*FwdKernel)(FwdArgs);
typedef void (*InvKernel)(InvArgs);
typedef void (*CztKernel)(CztArgs);
typedef void (*CztInvKernel)(CztInvArgs);

// The kernel of one CTA variant (16 or 8 warps; 116 = 16 warps as two independent 8-warp halves), or nullptr when
// that variant is not built for the size.
#define B2L_DECL_FFT(L) FwdKernel fwd_kernel_##L(int variant, int mode); InvKernel inv_kernel_##L(int variant);
#define B2L_DECL_CZT(L) CztKernel czt_kernel_##L(); CztInvKernel czt_inv_kernel_##L();
B2L_FFT_SIZES(B2L_DECL_FFT)
B2L_CZT_SIZES(B2L_DECL_CZT)
#undef B2L_DECL_FFT
#undef B2L_DECL_CZT

// Host mirror of FftCfg<LOG2M, TPF> (fft_engine.cuh): same schedule, evaluated at run time.
struct HostFftCfg {
  int log2m, M, tpf, ppt, logp, npass;
  explicit HostFftCfg(int l2m) {
    log2m = l2m;
    M = 1 << l2m;
    tpf = M >= 32 ? M / 32 : 1;
    ppt = M / tpf;
    logp = 0;
    while ((1 << logp) < ppt) ++logp;
    npass = ppt == 1 ? 1 : (log2m + logp - 1) / logp;
  }
  int log_radix(int s) const { int left = log2m - s * logp; return left >= logp ? logp : left; }
  int radix(int s) const { return 1 << log_radix(s); }
  int sublen(int s) const { return 1 << (s * logp); }
  bool split_pass(int s, bool split) const { return split && tw_split_pass(log2m, s, radix(s)); }
  int tw_rows(int s, bool split) const { return split_pass(s, split) ? kTwSplitRows : radix(s) - 1; }
  int tw_offset(int s, bool split = false) const {
    int off = 0;
    for (int q = 1; q < s; ++q) off += tw_rows(q, split) * sublen(q);
    return off;
  }
  int tw_count(bool split = false) const { return tw_offset(npass, split); }
  int xbuf_f2() const { return M + M / 32; }
  // warps per CTA of czt_kernel for P = 2^log2p (mirror of czt_inst.cu)
  int czt_nw() const { return log2m >= 10 ? 16 : (tpf > 16 ? 16 : tpf); }
  // warps per CTA tried in order (first that fits shared memory wins)
  int nw_options(int out[2]) const {
    if (log2m >= 10) { out[0] = 16; out[1] = 8; return 2; }
    out[0] = tpf >= 1 ? (tpf > 16 ? 16 : tpf) : 1;
    return 1;
  }
};

// Formats the message returned by b2l_last_error (per thread) and returns `code`.
int fail(int code, const char* fmt, ...);

#define CUDA_TRY(expr)                                                                        \
  do {                                                                                        \
    cudaError_t _e = (expr);                                                                  \
    if (_e != cudaSuccess) {                                                                  \
      cudaGetLastError();                                                                     \
      return fail(_e == cudaErrorMemoryAllocation ? B2L_ERR_OOM : B2L_ERR_CUDA, "%s: %s (%s:%d)", #expr, \
                  cudaGetErrorString(_e), __FILE__, __LINE__);                                \
    }                                                                                         \
  } while (0)

}  // namespace b2l

// ------------------------------------------------------------------ objects
struct b2l_ctx {
  int device = 0;
  int sm_count = 0;
  size_t smem_optin = 0;
  cudaStream_t stream = nullptr;
  uint64_t launches = 0;
  struct ncclComm* comm = nullptr;
  int rank = 0, world = 1;
  unsigned int* d_clip_max = nullptr;   // scratch for per-clip maxima
  int* d_status = nullptr;              // enum b2l_status_bit flags set since the last reset
  float* d_scratch = nullptr;           // grow-only scratch (istft frames, pip_pass histograms)
  size_t scratch_bytes = 0;
  size_t clip_max_cap = 0;
  // cudaFuncSetAttribute and the occupancy query cost tens of microseconds: blocks_per_sm
  std::set<const void*> smem_limit_set;                          // kernels whose shared-memory limit is raised
  std::map<std::tuple<const void*, int, size_t>, int> occupancy;   // (kernel, threads, smem) -> blocks / SM
  // pinned staging ring for uploads from pageable host memory (staged_h2d)
  std::vector<void*> stage_bufs;
  std::vector<cudaEvent_t> stage_evs;
};

struct b2l_plan {
  b2l_ctx* ctx = nullptr;
  int n_fft = 0, hop = 0, center = 0, pad_mode = 0, log2m = 0;
  b2l::Path path = b2l::PATH_POW2;   // only this path's tables below are built
  // every device allocation of the plan (b2l_plan_destroy frees them); the row tables below add theirs lazily
  mutable std::vector<void*> allocs;
  float* d_win_fwd = nullptr;   // window * 1/2
  float* d_win_inv = nullptr;   // window * 1/n_fft
  float2* d_tw = nullptr;       // inter-pass twiddles, full table (inv_kernel)
  float2* d_tw_fwd = nullptr;   // inter-pass twiddles, split table (fwd_kernel)
  float2* d_twn = nullptr;
  int tw_count = 0;
  // mel: band-sparse rows (bins [lo, lo+len) of each mel row); d_mel_w / d_band feed mel_project, the
  // fused kernel uses a MelRow table built per tile geometry (H rows per warp step), cached here
  int n_mels = 0, mel_w_count = 0;
  float* d_mel_w = nullptr;
  b2l::MelBand* d_band = nullptr;
  float* d_mel_wT = nullptr;     // n_mels <= 16: dense transposed weights [bin][16] (dense_project_kernel)
  std::vector<b2l::MelBand> h_band;
  std::vector<float> h_mel_w;
  struct RowTable { b2l::MelRow* d_rows = nullptr; float* d_w = nullptr; int n_rows = 0, w_count = 0; };
  mutable std::map<int, RowTable> row_tables;
  int power_mode = 2;
  float power = 2.0f;
  // chirp-z path (czt_kernel.cuh): transform size P = 2^log2p
  int log2p = 0;
  float2* d_czt_wb = nullptr;   // [n_fft] window * b
  float2* d_czt_bk = nullptr;   // [1 + n_fft/2] b
  float2* d_czt_hf = nullptr;   // [P] FFT_P(h)/P followed by the engine's inter-pass twiddles
  float2* d_czt_bfull = nullptr;   // [n_fft] b (inverse)
  float2* d_czt_wbi = nullptr;     // [n_fft] conj(b) * window / n_fft (inverse)
  // mixed-radix path (mr_kernel.cuh)
  int mr_n_pass = 0, mr_tw_count = 0;
  int mr_radix[b2l::kMrMaxPass] = {0}, mr_tw_off[b2l::kMrMaxPass] = {0};
  float* d_mr_win = nullptr;       // [n_fft] window * 1/2
  float* d_mr_win_inv = nullptr;   // [n_fft] window / n_fft (inverse)
  float2* d_mr_tw = nullptr;       // pass twiddles
  float2* d_mr_twn = nullptr;      // [n_fft/4 + 1] exp(-2 pi i k / n_fft)
  // mfcc
  int n_mfcc = 0;
  float* d_dct = nullptr;
  float amin = 1e-10f, ref_value = 1.0f, top_db = 80.0f;
};

namespace b2l {

struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(int dev) {
    cudaGetDevice(&prev);
    if (prev != dev) cudaSetDevice(dev);
    else prev = -1;
  }
  ~DeviceGuard() {
    if (prev >= 0) cudaSetDevice(prev);
  }
};

// ------------------------------------------------------------------ host helpers
inline int ilog2_exact(int x) {
  int l = 0;
  while ((1 << l) < x) ++l;
  return (1 << l) == x ? l : -1;
}

inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// stream-ordered temporary: freed behind the work that uses it, no host synchronisation
struct Temp {
  void* p = nullptr;
  cudaStream_t st;
  explicit Temp(cudaStream_t s) : st(s) {}
  cudaError_t alloc(size_t bytes) { return cudaMallocAsync(&p, bytes ? bytes : 16, st); }
  ~Temp() {
    if (p) cudaFreeAsync(p, st);
  }
};

template <class T>
cudaError_t upload(Temp& t, const T* h, size_t count) {
  cudaError_t e = t.alloc(count * sizeof(T));
  if (e != cudaSuccess) return e;
  return cudaMemcpyAsync(t.p, h, count * sizeof(T), cudaMemcpyHostToDevice, t.st);   // pageable source: returns after the copy is staged
}

// exp(-2*pi*i*j/n) for j < count, in long double rounded to double (the FP64 transforms' twiddles; f64_api.cu)
std::vector<double2> f64_twiddles(int n, int count);

// Grows the context's per-clip maximum scratch to at least n_clips entries.
int ensure_clip_max(b2l_ctx* c, size_t n_clips);
// Grows the context's scratch array to at least `bytes` (the contents are not kept).
int ensure_scratch(b2l_ctx* c, size_t bytes);

// Checks a spectral-statistics descriptor and converts it to the kernels' StatsParams (feature_api.cu).
int check_stats_desc(const b2l_stats_desc* d, StatsParams* sp);

// ------------------------------------------------------------------ launches
// Resident blocks per SM of kernel `fn` with `threads` threads and `smem` bytes of dynamic shared memory, cached per
// (fn, threads, smem); with occ == NULL (a grid sized otherwise) nothing is queried.  The first time `fn` is seen its
// dynamic shared-memory limit is raised to `smem_limit` (0: the device's opt-in maximum; a kernel with static shared
// memory passes what is left of it).
int blocks_per_sm(b2l_ctx* c, const void* fn, int threads, size_t smem, int* occ, size_t smem_limit = 0);
template <class... P>
int blocks_per_sm(b2l_ctx* c, void (*fn)(P...), int threads, size_t smem, int* occ, size_t smem_limit = 0) {
  return blocks_per_sm(c, (const void*)fn, threads, smem, occ, smem_limit);
}

// Launches `fn` on the context's stream, checks the launch and counts it: the only place that does any of the three.
template <class... P, class... A>
int launch(b2l_ctx* c, void (*fn)(P...), dim3 grid, dim3 block, size_t smem, const A&... args) {
  fn<<<grid, block, smem, c->stream>>>(args...);
  CUDA_TRY(cudaGetLastError());
  c->launches++;
  return B2L_OK;
}

// Grid of a kernel that keeps every block resident: sm_count * (blocks per SM with `query_smem` bytes of dynamic
// shared memory), at most `need`; 0 when not even one block fits (each caller reports that in its own words).
template <class... P>
int resident_grid(b2l_ctx* c, void (*fn)(P...), int threads, size_t query_smem, long long need, long long* grid) {
  int occ = 0;
  if (int rc = blocks_per_sm(c, fn, threads, query_smem, &occ)) return rc;
  *grid = occ < 1 ? 0 : std::min((long long)c->sm_count * occ, need);
  return B2L_OK;
}

// Blocks of a grid-stride loop over `work` items, `per_block` items per block per pass, at most `cap` blocks.
inline long long grid_stride_blocks(long long work, long long per_block, long long cap) {
  return std::min((work + per_block - 1) / per_block, cap);
}

// x-extent of an (x, clips) grid over m clips of `per_row` items: one block per `per_block` items, but about
// `budget` blocks in all, and at least one per clip.
inline long long row_blocks(long long per_row, long long per_block, long long budget, long long m) {
  return std::max(1LL, std::min((per_row + per_block - 1) / per_block, (budget + m - 1) / m));
}

// Largest grid.y / grid.z extent.  Kernels that carry the clip index there run larger batches in slices.
constexpr int64_t kMaxGridY = 65535;

// Calls body(c0, m) for consecutive slices [c0, c0 + m) of at most kMaxGridY clips; returns the first non-zero status.
template <class F>
int for_clip_slices(int64_t n_clips, F body) {
  for (int64_t c0 = 0; c0 < n_clips; c0 += kMaxGridY)
    if (int rc = body(c0, std::min(kMaxGridY, n_clips - c0))) return rc;
  return B2L_OK;
}

// ------------------------------------------------------------------ plans (plan.cu)
long long plan_frames(const b2l_plan* p, long long n);
// Inter-pass twiddles of the register FFT of complex size 2^cfg.log2m (FftCfg::tw_offset layout; split: fwd_kernel's table).
std::vector<float2> engine_twiddles(const HostFftCfg& cfg, bool split = false);
// MelRow table for warps that process H mel rows at a time (see MelRow / MelLayout in common.cuh), built on first use.
int get_row_table(const b2l_plan* p, int H, const b2l_plan::RowTable** out);

}  // namespace b2l
