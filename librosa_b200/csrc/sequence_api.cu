// sequence_api.cu — C ABI of the HMM decoder (sequence_kernels.cuh): librosa.sequence.viterbi,
// viterbi_discriminative and viterbi_binary (librosa/sequence.py:1175-1876).  The only unit that includes
// sequence_kernels.cuh.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>

#include "internal.h"
#include "sequence_kernels.cuh"

using namespace b2l;

namespace {

// Static shared memory of viterbi_cta_kernel (reduction scratch and per-problem results), kept out of the dynamic
// budget.
const size_t kCtaStatic = 1024;

struct Route {
  int cls;        // B2L_SEQ_SMALL / MEDIUM / LARGE
  int W, G;       // lanes per problem (small), problems per CTA (medium, large)
  int in_smem;    // model tables staged in shared memory
  size_t smem;    // dynamic shared memory per block
};

int route(const b2l_ctx* c, const b2l_seq_model* m, int64_t n_problems, Route* r) {
  const size_t budget = c->smem_optin - kCtaStatic;
  const int S = m->n_states;
  const size_t tables = b2l_seq::seq_table_bytes(S, m->n_models, m->deg, m->dense);
  memset(r, 0, sizeof(*r));
  if (S <= 32) {
    r->cls = B2L_SEQ_SMALL;
    r->W = 2;
    while (r->W < S) r->W *= 2;
    r->in_smem = tables <= 48 * 1024;
    r->smem = r->in_smem ? tables : 0;
    return B2L_OK;
  }
  if (m->n_models != 1) return fail(B2L_ERR_INVALID, "viterbi: several models need at most 32 states");
  r->G = 1;
  if ((size_t)2 * S * sizeof(double) > budget)
    return fail(B2L_ERR_UNSUPPORTED, "viterbi: %d states; the GPU decoder holds at most %zu (two float64 value rows "
                "in shared memory)", S, budget / 16);
  const size_t rows1 = (size_t)2 * r->G * S * sizeof(double);
  r->in_smem = rows1 + tables <= budget;
  r->cls = r->in_smem ? B2L_SEQ_MEDIUM : B2L_SEQ_LARGE;
  r->smem = rows1 + (r->in_smem ? tables : 0);
  (void)n_problems;
  return B2L_OK;
}

template <class K>
int launch_decode(b2l_ctx* c, K fn, long long blocks, int threads, size_t smem, const b2l_seq::DecodeArgs& a) {
  if (int rc = blocks_per_sm(c, fn, threads, smem, nullptr, c->smem_optin - kCtaStatic)) return rc;
  return launch(c, fn, dim3((unsigned)blocks), dim3(threads), smem, a);
}

}  // namespace

extern "C" int b2l_seq_logobs(b2l_ctx* c, const b2l_seq_logobs_desc* d, const void* d_prob, double* d_out,
                              int32_t* d_flags) {
  if (!c || !d) return fail(B2L_ERR_INVALID, "NULL argument");
  if (d->n_clips < 0 || d->n_states < 0 || d->n_steps < 0) return fail(B2L_ERR_INVALID, "bad batch geometry");
  if (d->mode < B2L_SEQ_PLAIN || d->mode > B2L_SEQ_BINARY) return fail(B2L_ERR_INVALID, "unknown mode %d", d->mode);
  if (d->n_states > 65535) return fail(B2L_ERR_UNSUPPORTED, "viterbi: %lld states do not fit 16-bit states",
                                       (long long)d->n_states);
  if (d->n_clips == 0 || d->n_states == 0 || d->n_steps == 0) return B2L_OK;
  if (!d_prob || !d_flags || (d_out && d->mode != B2L_SEQ_PLAIN && !d->d_log_marginal))
    return fail(B2L_ERR_INVALID, "NULL device pointer");
  const int threads = 256;
  const long long t_blocks = (d->n_steps + threads - 1) / threads;
  if (d->n_clips > 0x7fffffffLL / t_blocks) return fail(B2L_ERR_UNSUPPORTED, "viterbi: too many clips x frames");
  DeviceGuard g(c->device);
  b2l_seq::LogObsArgs a;
  a.prob = d_prob;
  a.n_clips = d->n_clips;
  a.n_steps = d->n_steps;
  a.n_states = (int)d->n_states;
  a.t_blocks = t_blocks;
  a.eps = d->eps;
  a.log_marginal = d->d_log_marginal;
  a.out = d_out;
  a.flags = d_flags;
  using namespace b2l_seq;
  void (*fn)(LogObsArgs);
  if (d->mode == B2L_SEQ_PLAIN) fn = d->f64 ? viterbi_logobs_kernel<double, kLogPlain> : viterbi_logobs_kernel<float, kLogPlain>;
  else if (d->mode == B2L_SEQ_DISC) fn = d->f64 ? viterbi_logobs_kernel<double, kLogDisc> : viterbi_logobs_kernel<float, kLogDisc>;
  else fn = d->f64 ? viterbi_logobs_kernel<double, kLogBinary> : viterbi_logobs_kernel<float, kLogBinary>;
  return launch(c, fn, dim3((unsigned)(d->n_clips * t_blocks)), dim3(threads), 0, a);
}

extern "C" int b2l_seq_route(b2l_ctx* c, const b2l_seq_model* m, int64_t n_problems, int32_t* out) {
  if (!c || !m || !out) return fail(B2L_ERR_INVALID, "NULL argument");
  if (m->n_states < 1 || m->n_models < 1 || m->deg < 1 || m->deg > m->n_states)
    return fail(B2L_ERR_INVALID, "bad model geometry");
  Route r;
  if (int rc = route(c, m, n_problems, &r)) return rc;
  out[0] = r.cls;
  out[1] = r.cls == B2L_SEQ_SMALL ? r.W : r.G;
  return B2L_OK;
}

extern "C" int b2l_seq_decode(b2l_ctx* c, const b2l_seq_model* m, const double* d_lp, int64_t n_problems,
                              int64_t n_steps, uint16_t* d_states, double* d_logp) {
  if (!c || !m) return fail(B2L_ERR_INVALID, "NULL argument");
  if (n_problems < 0 || n_steps < 0) return fail(B2L_ERR_INVALID, "bad batch geometry");
  if (m->n_states < 1 || m->n_models < 1 || m->deg < 1 || m->deg > m->n_states)
    return fail(B2L_ERR_INVALID, "bad model geometry");
  if (m->n_states > 65535) return fail(B2L_ERR_UNSUPPORTED, "viterbi: %d states do not fit 16-bit back-pointers",
                                       m->n_states);
  if (m->dense && m->deg != m->n_states) return fail(B2L_ERR_INVALID, "a dense model lists every state");
  Route r;
  if (int rc = route(c, m, n_problems, &r)) return rc;
  if (n_problems == 0 || n_steps == 0) return B2L_OK;
  if (!d_lp || !d_states || !d_logp || !m->d_lt || !m->d_log_p_init || (!m->dense && !m->d_idx))
    return fail(B2L_ERR_INVALID, "NULL device pointer");
  DeviceGuard g(c->device);
  Temp ptr(c->stream);
  CUDA_TRY(ptr.alloc((size_t)n_problems * n_steps * m->n_states * sizeof(uint16_t)));
  b2l_seq::DecodeArgs a;
  a.lp = d_lp;
  a.n_problems = n_problems;
  a.n_steps = n_steps;
  a.n_states = m->n_states;
  a.n_models = m->n_models;
  a.deg = m->deg;
  a.dense = m->dense;
  a.lt = m->d_lt;
  a.idx = m->d_idx;
  a.log_p_init = m->d_log_p_init;
  a.tables_in_smem = r.in_smem;
  a.ptr = (unsigned short*)ptr.p;
  a.states = d_states;
  a.logp = d_logp;
  using namespace b2l_seq;
  if (r.cls == B2L_SEQ_SMALL) {
    const long long blocks = (n_problems + 128 / r.W - 1) / (128 / r.W);
    if (blocks > 0x7fffffffLL) return fail(B2L_ERR_UNSUPPORTED, "viterbi: too many problems in one call");
    switch (r.W) {
      case 2: return launch_decode(c, viterbi_small_kernel<2>, blocks, 128, r.smem, a);
      case 4: return launch_decode(c, viterbi_small_kernel<4>, blocks, 128, r.smem, a);
      case 8: return launch_decode(c, viterbi_small_kernel<8>, blocks, 128, r.smem, a);
      case 16: return launch_decode(c, viterbi_small_kernel<16>, blocks, 128, r.smem, a);
      default: return launch_decode(c, viterbi_small_kernel<32>, blocks, 128, r.smem, a);
    }
  }
  const long long blocks = (n_problems + r.G - 1) / r.G;
  if (blocks > 0x7fffffffLL) return fail(B2L_ERR_UNSUPPORTED, "viterbi: too many problems in one call");
  return launch_decode(c, viterbi_cta_kernel<1>, blocks, 256, r.smem, a);
}
