// plan.cu — C ABI of libb2l.so (see include/b2l.h): transform plans.  The host builds every table a plan's kernels
// read (windows, twiddles, chirp-z and mixed-radix tables, mel rows, the DCT) in double precision and uploads it
// once.  Launches no kernel.
#include <cuda_runtime.h>
#include <math.h>

#include <algorithm>
#include <complex>
#include <vector>

#include "internal.h"

using namespace b2l;

// Uploads a host table to a new device allocation owned by the plan (b2l_plan_destroy frees it).
template <class T>
static int upload(const b2l_plan* p, const std::vector<T>& h, T** d) {
  *d = nullptr;
  const size_t bytes = h.size() * sizeof(T);
  CUDA_TRY(cudaMalloc((void**)d, bytes ? bytes : 16));
  p->allocs.push_back(*d);
  if (bytes) CUDA_TRY(cudaMemcpy(*d, h.data(), bytes, cudaMemcpyHostToDevice));
  return B2L_OK;
}

// inter-pass twiddles of the register FFT for a complex size 2^log2m (FftCfg::tw_offset layout): the full table, or
// the split one of fwd_kernel (radix-32 passes as the factors of tw_row_exponent)
std::vector<float2> b2l::engine_twiddles(const HostFftCfg& cfg, bool split) {
  const double two_pi = 6.283185307179586476925286766559;
  std::vector<float2> tw((size_t)cfg.tw_count(split));
  for (int s = 1; s < cfg.npass; ++s) {
    const int R = cfg.radix(s), pl = cfg.sublen(s), off = cfg.tw_offset(s, split);
    for (int j = 0; j < cfg.tw_rows(s, split); ++j) {
      const int e = tw_row_exponent(j, cfg.split_pass(s, split));
      for (int k = 0; k < pl; ++k) {
        // exp(-2*pi*i * e*k / (p*R)); reduce the integer phase first to keep the argument small
        long long num = ((long long)e * k) % ((long long)pl * R);
        double ang = -two_pi * (double)num / (double)((long long)pl * R);
        tw[(size_t)off + (size_t)j * pl + k] = make_float2((float)cos(ang), (float)sin(ang));
      }
    }
  }
  return tw;
}

// in-place radix-2 FFT in double precision (host, plan construction only)
static void host_fft(std::vector<std::complex<double>>& x) {
  const size_t n = x.size();
  for (size_t i = 1, j = 0; i < n; ++i) {
    size_t bit = n >> 1;
    for (; j & bit; bit >>= 1) j ^= bit;
    j ^= bit;
    if (i < j) std::swap(x[i], x[j]);
  }
  for (size_t len = 2; len <= n; len <<= 1) {
    for (size_t i = 0; i < n; i += len)
      for (size_t k = 0; k < len / 2; ++k) {
        const double ang = -2.0 * kPi * (double)k / (double)len;
        const std::complex<double> w(cos(ang), sin(ang));
        const std::complex<double> u = x[i + k], v = x[i + k + len / 2] * w;
        x[i + k] = u + v;
        x[i + k + len / 2] = u - v;
      }
  }
}

// exp(-2 pi i k / n_fft), k = 0 .. n_fft / 4: the real-FFT un-mix twiddles of the forward and inverse kernels
static std::vector<float2> unmix_twiddles(int N) {
  std::vector<float2> twn((size_t)N / 4 + 1);
  for (int k = 0; k <= N / 4; ++k) {
    const double ang = -2.0 * kPi * (double)k / (double)N;
    twn[k] = make_float2((float)cos(ang), (float)sin(ang));
  }
  return twn;
}

// Radix schedule of the mixed-radix kernel for n_fft = 2 M: M = 5^c 3^b 2^a as c fives, b threes, then eights and a
// four / two.  False when n_fft is odd, M has another prime factor, or the schedule / buffers would not fit.
static bool mr_factor(int n_fft, std::vector<int>& radices) {
  radices.clear();
  if (n_fft < 12 || (n_fft & 1) || n_fft > 4096) return false;
  int m = n_fft / 2;
  while (m % 5 == 0) { radices.push_back(5); m /= 5; }
  while (m % 3 == 0) { radices.push_back(3); m /= 3; }
  while (m % 8 == 0) { radices.push_back(8); m /= 8; }
  if (m % 4 == 0) { radices.push_back(4); m /= 4; }
  if (m % 2 == 0) { radices.push_back(2); m /= 2; }
  return m == 1 && (int)radices.size() <= kMrMaxPass && !radices.empty();
}

// Which transform serves n_fft >= 1 (host mirror: _pipeline.transform_path), with what that path needs: *log2m for a
// power of two, the radix schedule for the mixed-radix kernels, *log2p (chirp-z size P = 2^log2p >= 2 n_fft - 1, at
// least one warp of the engine) for the chirp-z kernels, which are built up to P = 4096.
static int plan_path(int n_fft, Path* path, int* log2m, int* log2p, std::vector<int>& radices) {
  const int l2n = ilog2_exact(n_fft);
  if (l2n >= 0) {
    if (l2n - 1 < kMinLog2M || l2n - 1 > kMaxLog2M)
      return fail(B2L_ERR_UNSUPPORTED,
                  "n_fft=%d: the sm_90a kernels are built for powers of two from %d to %d (no CPU fallback)", n_fft,
                  2 << kMinLog2M, 2 << kMaxLog2M);
    *path = PATH_POW2;
    *log2m = l2n - 1;
    return B2L_OK;
  }
  if (mr_factor(n_fft, radices)) {
    *path = PATH_MR;
    return B2L_OK;
  }
  if (n_fft > 2047)
    return fail(B2L_ERR_UNSUPPORTED,
                "n_fft=%d: non-power-of-two sizes are supported from 3 to 2047, and even sizes up to 4096 whose half "
                "has no prime factor above 5 (no CPU fallback)", n_fft);
  *path = PATH_CZT;
  for (*log2p = 5; (1 << *log2p) < 2 * n_fft - 1;) ++*log2p;
  return B2L_OK;
}

// ------------------------------------------------------------------ table builders
// windows and twiddles of fwd_kernel / inv_kernel (n_fft a power of two)
static int build_pow2(b2l_plan* p, const double* window) {
  const int N = p->n_fft;
  HostFftCfg cfg(p->log2m);
  std::vector<float> wf(N), wi(N);
  for (int i = 0; i < N; ++i) {
    wf[i] = (float)(window[i] * 0.5);
    wi[i] = (float)(window[i] / (double)N);
  }
  p->tw_count = cfg.tw_count();
  int rc;
  if ((rc = upload(p, wf, &p->d_win_fwd)) || (rc = upload(p, wi, &p->d_win_inv)) ||
      (rc = upload(p, engine_twiddles(cfg), &p->d_tw)) || (rc = upload(p, engine_twiddles(cfg, true), &p->d_tw_fwd)) ||
      (rc = upload(p, unmix_twiddles(N), &p->d_twn)))
    return rc;
  return B2L_OK;
}

// chirp-z tables (czt_kernel.cuh) for transform size P = 2^p->log2p
static int build_czt(b2l_plan* p, const double* window) {
  const int L = p->n_fft, P = 1 << p->log2p;
  std::vector<std::complex<double>> b(L);
  for (int n = 0; n < L; ++n) {
    const long long q = ((long long)n * n) % (2LL * L);          // n^2 mod 2L keeps the phase exact
    const double ang = -kPi * (double)q / (double)L;
    b[n] = std::complex<double>(cos(ang), sin(ang));
  }
  std::vector<float2> wb(L), bk(L / 2 + 1);
  for (int n = 0; n < L; ++n) {
    const std::complex<double> z = window[n] * b[n];
    wb[n] = make_float2((float)z.real(), (float)z.imag());
  }
  for (int k = 0; k <= L / 2; ++k) bk[k] = make_float2((float)b[k].real(), (float)b[k].imag());
  std::vector<std::complex<double>> h(P, std::complex<double>(0.0, 0.0));
  h[0] = std::conj(b[0]);
  for (int m = 1; m < L; ++m) h[m] = h[P - m] = std::conj(b[m]);
  host_fft(h);
  std::vector<float2> hf((size_t)P);
  for (int i = 0; i < P; ++i) hf[i] = make_float2((float)(h[i].real() / P), (float)(h[i].imag() / P));
  std::vector<float2> tw = engine_twiddles(HostFftCfg(p->log2p));
  hf.insert(hf.end(), tw.begin(), tw.end());
  std::vector<float2> bfull(L), wbi(L);
  for (int n = 0; n < L; ++n) {
    bfull[n] = make_float2((float)b[n].real(), (float)b[n].imag());
    const std::complex<double> z = std::conj(b[n]) * (window[n] / (double)L);
    wbi[n] = make_float2((float)z.real(), (float)z.imag());
  }
  int rc;
  if ((rc = upload(p, wb, &p->d_czt_wb)) || (rc = upload(p, bk, &p->d_czt_bk)) || (rc = upload(p, hf, &p->d_czt_hf)) ||
      (rc = upload(p, bfull, &p->d_czt_bfull)) || (rc = upload(p, wbi, &p->d_czt_wbi)))
    return rc;
  return B2L_OK;
}

// mixed-radix tables (odd radices first, see mr_kernel.cuh) for the radix schedule of mr_factor
static int build_mr(b2l_plan* p, const std::vector<int>& radices, const double* window) {
  const int N = p->n_fft;
  p->mr_n_pass = (int)radices.size();
  std::vector<float2> tw;
  int sub = 1;
  for (int s = 0; s < p->mr_n_pass; ++s) {
    const int R = radices[s];
    p->mr_radix[s] = R;
    p->mr_tw_off[s] = (int)tw.size();
    if (sub > 1)
      for (int r = 1; r < R; ++r)
        for (int k = 0; k < sub; ++k) {
          const long long num = ((long long)r * k) % ((long long)sub * R);
          const double ang = -2.0 * kPi * (double)num / (double)((long long)sub * R);
          tw.push_back(make_float2((float)cos(ang), (float)sin(ang)));
        }
    sub *= R;
  }
  if (tw.empty()) tw.push_back(make_float2(1.0f, 0.0f));
  p->mr_tw_count = (int)tw.size();
  std::vector<float> wf(N), wi(N);
  for (int i = 0; i < N; ++i) {
    wf[i] = (float)(window[i] * 0.5);
    wi[i] = (float)(window[i] / (double)N);
  }
  int rc;
  if ((rc = upload(p, wf, &p->d_mr_win)) || (rc = upload(p, wi, &p->d_mr_win_inv)) || (rc = upload(p, tw, &p->d_mr_tw)) ||
      (rc = upload(p, unmix_twiddles(N), &p->d_mr_twn)))
    return rc;
  return B2L_OK;
}

// band-sparse mel rows: bins [lo, lo + len) of each row of the [n_mels][n_fft/2 + 1] basis
static int build_mel(b2l_plan* p, const float* basis, int n_mels) {
  const int F = p->n_fft / 2 + 1;
  std::vector<MelBand> bands(n_mels);
  std::vector<float> w;
  for (int m = 0; m < n_mels; ++m) {
    const float* row = basis + (size_t)m * F;
    int lo = -1, hi = -1;
    for (int k = 0; k < F; ++k)
      if (row[k] != 0.0f) {
        if (lo < 0) lo = k;
        hi = k;
      }
    MelBand b;
    b.off = (int)w.size();
    b.pad = 0;
    if (lo < 0) {
      b.lo = 0;
      b.len = 0;
    } else {
      b.lo = lo;
      b.len = hi - lo + 1;
      w.insert(w.end(), row + lo, row + hi + 1);
    }
    bands[m] = b;
  }
  p->n_mels = n_mels;
  p->mel_w_count = (int)w.size();
  p->h_band = bands;
  p->h_mel_w = w;
  int rc;
  if ((rc = upload(p, w, &p->d_mel_w)) || (rc = upload(p, bands, &p->d_band))) return rc;
  return B2L_OK;
}

// n_mels <= 16: the basis transposed and zero padded to [bin][16] (dense_project_kernel)
static int build_dense_mel(b2l_plan* p, const float* basis) {
  const int F = p->n_fft / 2 + 1;
  std::vector<float> wT((size_t)F * 16, 0.0f);
  for (int m = 0; m < p->n_mels; ++m)
    for (int k = 0; k < F; ++k) wT[(size_t)k * 16 + m] = basis[(size_t)m * F + k];
  return upload(p, wT, &p->d_mel_wT);
}

// DCT rows transposed and zero padded to 8-coefficient groups: dctT[m][8*KG] (dct_clamp4_kernel)
static int build_dct(b2l_plan* p, const float* basis, int n_mfcc) {
  const int KP = (n_mfcc + 7) / 8 * 8;
  std::vector<float> dct((size_t)p->n_mels * KP, 0.0f);
  for (int k = 0; k < n_mfcc; ++k)
    for (int m = 0; m < p->n_mels; ++m) dct[(size_t)m * KP + k] = basis[(size_t)k * p->n_mels + m];
  p->n_mfcc = n_mfcc;
  return upload(p, dct, &p->d_dct);
}

// ------------------------------------------------------------------ plans
extern "C" int b2l_plan_destroy(b2l_plan* p) {
  if (!p) return B2L_OK;
  DeviceGuard g(p->ctx->device);
  cudaStreamSynchronize(p->ctx->stream);
  for (void* d : p->allocs) cudaFree(d);
  delete p;
  return B2L_OK;
}

extern "C" int b2l_plan_create(b2l_ctx* c, const b2l_plan_desc* d, b2l_plan** out) {
  if (!c || !d || !out) return fail(B2L_ERR_INVALID, "NULL argument");
  if (d->n_fft < 1) return fail(B2L_ERR_INVALID, "n_fft=%d must be positive", d->n_fft);
  if (d->hop_length < 1) return fail(B2L_ERR_INVALID, "hop_length=%d must be a positive integer", d->hop_length);
  Path path = PATH_POW2;
  int log2m = -1, log2p = 0;
  std::vector<int> radices;
  if (int rc = plan_path(d->n_fft, &path, &log2m, &log2p, radices)) return rc;
  if (!d->h_window) return fail(B2L_ERR_INVALID, "window is NULL");
  if (d->pad_mode < 0 || d->pad_mode > B2L_PAD_EMPTY) return fail(B2L_ERR_INVALID, "bad pad_mode %d", d->pad_mode);
  if (d->n_mels < 0 || d->n_mfcc < 0) return fail(B2L_ERR_INVALID, "negative n_mels / n_mfcc");
  if (d->n_mels > 0 && !d->h_mel_basis) return fail(B2L_ERR_INVALID, "mel basis is NULL");
  if (d->n_mfcc > 0 && (!d->h_dct_basis || d->n_mels == 0))
    return fail(B2L_ERR_INVALID, "mfcc stage needs a mel stage and a DCT basis");
  if (d->n_mfcc > 0 && !(d->amin > 0.0f)) return fail(B2L_ERR_INVALID, "amin must be strictly positive");

  DeviceGuard g(c->device);
  b2l_plan* p = new b2l_plan();
  p->ctx = c;
  p->n_fft = d->n_fft;
  p->hop = d->hop_length;
  p->center = d->center ? 1 : 0;
  p->pad_mode = d->pad_mode;
  p->path = path;
  p->log2m = log2m;
  p->log2p = log2p;
  p->power = d->power;
  p->power_mode = d->power == 2.0f ? 2 : (d->power == 1.0f ? 1 : 0);
  p->amin = d->amin;
  p->ref_value = d->ref_value;
  p->top_db = d->top_db;
  int rc = path == PATH_POW2 ? build_pow2(p, d->h_window)
           : path == PATH_MR ? build_mr(p, radices, d->h_window)
                             : build_czt(p, d->h_window);
  if (rc == B2L_OK && d->n_mels > 0) rc = build_mel(p, d->h_mel_basis, d->n_mels);
  if (rc == B2L_OK && d->n_mels > 0 && d->n_mels <= 16) rc = build_dense_mel(p, d->h_mel_basis);
  if (rc == B2L_OK && d->n_mfcc > 0) rc = build_dct(p, d->h_dct_basis, d->n_mfcc);
  if (rc) {
    b2l_plan_destroy(p);
    return rc;
  }
  *out = p;
  return B2L_OK;
}

long long b2l::plan_frames(const b2l_plan* p, long long n) {
  long long padded = n + (p->center ? 2LL * (p->n_fft / 2) : 0);
  if (padded < p->n_fft) return 0;
  return 1 + (padded - p->n_fft) / p->hop;
}

extern "C" int b2l_plan_n_frames(const b2l_plan* p, int64_t n, int64_t* n_frames) {
  if (!p || !n_frames) return fail(B2L_ERR_INVALID, "NULL argument");
  *n_frames = plan_frames(p, n);
  return B2L_OK;
}

int b2l::get_row_table(const b2l_plan* p, int H, const b2l_plan::RowTable** out) {
  auto it = p->row_tables.find(H);
  if (it != p->row_tables.end()) {
    *out = &it->second;
    return B2L_OK;
  }
  const int rsm = H < 4 ? 4 : H, G = rsm / 4;   // row starts: lo_j == 4*(j mod G) (mod rsm)
  const int n_rows = (p->n_mels + H - 1) / H * H;
  const int n_items = n_rows / H;
  std::vector<MelRow> rows(n_rows);
  std::vector<float> w;
  for (int item = 0; item < n_items; ++item) {
    std::vector<int> start(H), lenp(H);
    int quads = 0;
    for (int j = 0; j < H; ++j) {
      const int m = item * H + j;
      if (m < p->n_mels && p->h_band[m].len > 0) {
        const MelBand& b = p->h_band[m];
        const int want = 4 * (j % G);
        int st = b.lo - ((((b.lo - want) % rsm) + rsm) % rsm);   // largest bin <= lo congruent to `want` mod rsm
        if (st < 0) st = b.lo - (b.lo % 4);                       // lowest rows: keep the 16-byte alignment only
        start[j] = st;
        lenp[j] = b.lo + b.len - st;
      } else {
        start[j] = 4 * (j % G);
        lenp[j] = 0;
      }
      quads = std::max(quads, (lenp[j] + 3) / 4);
    }
    for (int j = 0; j < H; ++j) {
      const int m = item * H + j;
      MelRow r;
      r.lo = (unsigned short)start[j];
      r.quads = (unsigned short)quads;
      r.off = (unsigned int)w.size();
      size_t base = w.size();
      w.resize(base + (size_t)4 * quads, 0.0f);
      if (lenp[j] > 0) {
        const MelBand& b = p->h_band[m];
        for (int i = 0; i < b.len; ++i) w[base + (b.lo - start[j]) + i] = p->h_mel_w[b.off + i];
      }
      rows[m] = r;
    }
  }
  b2l_plan::RowTable t;
  t.n_rows = n_rows;
  t.w_count = (int)w.size();
  int rc;
  if ((rc = upload(p, rows, &t.d_rows)) || (rc = upload(p, w, &t.d_w))) return rc;
  *out = &p->row_tables.emplace(H, t).first->second;
  return B2L_OK;
}
