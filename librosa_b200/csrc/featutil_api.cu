// featutil_api.cu — C ABI of the feature-stacking utilities (featutil_kernels.cuh): librosa.feature.delta and
// librosa.feature.stack_memory (librosa/feature/utils.py), and the peak test librosa.util.localmax / localmin.  The
// only unit that includes featutil_kernels.cuh.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include "featutil_kernels.cuh"
#include "internal.h"

using namespace b2l;

namespace {

template <class T>
int launch_delta(b2l_ctx* c, b2l_featutil::DeltaArgs& a) {
  namespace F = b2l_featutil;
  const size_t taps = (2 * a.h + 1) * sizeof(double);
  if (a.inner == 1) {
    a.tiles = (a.n + F::kTile - 1) / F::kTile;
    const long long grid = grid_stride_blocks(a.outer * a.tiles, F::kWarps, 32LL * c->sm_count);
    return launch(c, F::delta_rows_kernel<T>, dim3((unsigned)grid), F::kThreads, F::rows_smem_bytes(a.h), a);
  }
  const long long grid = grid_stride_blocks(a.outer * a.n * a.inner, F::kThreads, 32LL * c->sm_count);
  return launch(c, F::delta_strided_kernel<T>, dim3((unsigned)grid), F::kThreads, taps, a);
}

template <int S>
int launch_stack(b2l_ctx* c, const b2l_featutil::StackArgs& a) {
  namespace F = b2l_featutil;
  const long long grid = grid_stride_blocks(a.rows * a.chunks, F::kWarps, 32LL * c->sm_count);
  return launch(c, F::stack_memory_kernel<S>, dim3((unsigned)grid), F::kThreads, 0, a);
}

template <class T>
int launch_localext(b2l_ctx* c, const void* d_x, bool is_max, long long outer, long long n, long long inner,
                    uint8_t* d_out) {
  namespace F = b2l_featutil;
  const long long total = outer * n * inner;
  const unsigned grid = (unsigned)grid_stride_blocks(total, F::kThreads * 4, 32LL * c->sm_count);
  if (inner == 1)
    return launch(c, F::localext_kernel<T, true>, dim3(grid), F::kThreads, 0, (const T*)d_x, total, n, inner, is_max, d_out);
  return launch(c, F::localext_kernel<T, false>, dim3(grid), F::kThreads, 0, (const T*)d_x, total, n, inner, is_max, d_out);
}

}  // namespace

extern "C" int b2l_delta(b2l_ctx* c, const b2l_delta_desc* desc, const void* d_x, int64_t outer, int64_t n,
                         int64_t inner, void* d_y) {
  if (!c || !desc || !d_x || !d_y || !desc->d_taps || !desc->d_pad) return fail(B2L_ERR_INVALID, "NULL argument");
  const int w = desc->width;
  if (w < 3 || w % 2 != 1) return fail(B2L_ERR_INVALID, "delta: width must be an odd integer >= 3");
  if (w > B2L_DELTA_MAX_WIDTH)
    return fail(B2L_ERR_UNSUPPORTED, "delta: width=%d exceeds the %d taps the GPU kernels hold in shared memory", w,
                B2L_DELTA_MAX_WIDTH);
  if (outer < 0 || n < 0 || inner < 1 || desc->sym < -1 || desc->sym > 1) return fail(B2L_ERR_INVALID, "delta: bad geometry");
  if (desc->interp && (n < w || !desc->d_edge)) return fail(B2L_ERR_INVALID, "delta: interp needs width <= n and an edge map");
  if (outer == 0 || n == 0) return B2L_OK;
  b2l_featutil::DeltaArgs a = {};
  a.x = d_x;
  a.y = d_y;
  a.outer = outer;
  a.n = n;
  a.inner = inner;
  a.h = w / 2;
  a.sym = desc->sym;
  a.interp = desc->interp;
  a.cval = desc->cval;
  a.fw = desc->d_taps;
  a.edge = desc->d_edge;
  a.pad = (const long long*)desc->d_pad;
  a.status = c->d_status;
  DeviceGuard g(c->device);
  return desc->f64 ? launch_delta<double>(c, a) : launch_delta<float>(c, a);
}

extern "C" int b2l_stack_memory(b2l_ctx* c, const b2l_stack_desc* desc, const void* d_x, int64_t n_clips, int64_t d,
                                int64_t t, const int64_t* d_pad, void* d_out) {
  if (!c || !desc || !d_x || !d_out) return fail(B2L_ERR_INVALID, "NULL argument");
  const int S = desc->elem_size;
  if (S != 1 && S != 2 && S != 4 && S != 8 && S != 16)
    return fail(B2L_ERR_UNSUPPORTED, "stack_memory: %d-byte elements; the gather takes 1, 2, 4, 8 or 16", S);
  if (n_clips < 0 || d < 0 || t < 1 || desc->n_steps < 1 || desc->delay == 0)
    return fail(B2L_ERR_INVALID, "stack_memory: bad geometry");
  b2l_featutil::StackArgs a = {};
  a.n_pad = (int64_t)(desc->n_steps - 1) * (desc->delay < 0 ? -desc->delay : desc->delay);
  if (a.n_pad > 0 && !d_pad) return fail(B2L_ERR_INVALID, "stack_memory: no padded-index table");
  a.rows = n_clips * desc->n_steps * d;
  if (a.rows == 0) return B2L_OK;
  a.x = d_x;
  a.clip_stride = desc->clip_stride;
  a.row_stride = desc->row_stride;
  a.col_stride = desc->col_stride;
  a.out = d_out;
  a.n_clips = n_clips;
  a.d = d;
  a.t = t;
  a.delay = desc->delay;
  a.n_steps = desc->n_steps;
  a.pad = (const long long*)d_pad;
  memcpy(&a.fill, desc->fill, sizeof(a.fill));
  a.chunks = (t + b2l_featutil::kChunk - 1) / b2l_featutil::kChunk;
  DeviceGuard g(c->device);
  switch (S) {
    case 1: return launch_stack<1>(c, a);
    case 2: return launch_stack<2>(c, a);
    case 4: return launch_stack<4>(c, a);
    case 8: return launch_stack<8>(c, a);
    default: return launch_stack<16>(c, a);
  }
}

extern "C" int b2l_localext(b2l_ctx* c, const void* d_x, int32_t type, int32_t is_max, int64_t outer, int64_t n,
                            int64_t inner, uint8_t* d_out) {
  if (!c) return fail(B2L_ERR_INVALID, "NULL argument");
  if (outer < 0 || n < 2 || inner < 0) return fail(B2L_ERR_INVALID, "localext: bad geometry (the axis needs 2 or more values)");
  if (outer == 0 || inner == 0) return B2L_OK;
  if (!d_x || !d_out) return fail(B2L_ERR_INVALID, "NULL device pointer");
  DeviceGuard g(c->device);
  const bool mx = is_max != 0;
  switch (type) {
    case B2L_ELEM_I8: return launch_localext<int8_t>(c, d_x, mx, outer, n, inner, d_out);
    case B2L_ELEM_U8: return launch_localext<uint8_t>(c, d_x, mx, outer, n, inner, d_out);
    case B2L_ELEM_I16: return launch_localext<int16_t>(c, d_x, mx, outer, n, inner, d_out);
    case B2L_ELEM_U16: return launch_localext<uint16_t>(c, d_x, mx, outer, n, inner, d_out);
    case B2L_ELEM_I32: return launch_localext<int32_t>(c, d_x, mx, outer, n, inner, d_out);
    case B2L_ELEM_U32: return launch_localext<uint32_t>(c, d_x, mx, outer, n, inner, d_out);
    case B2L_ELEM_I64: return launch_localext<long long>(c, d_x, mx, outer, n, inner, d_out);
    case B2L_ELEM_U64: return launch_localext<unsigned long long>(c, d_x, mx, outer, n, inner, d_out);
    case B2L_ELEM_F32: return launch_localext<float>(c, d_x, mx, outer, n, inner, d_out);
    case B2L_ELEM_F64: return launch_localext<double>(c, d_x, mx, outer, n, inner, d_out);
    case B2L_ELEM_BOOL: return launch_localext<bool>(c, d_x, mx, outer, n, inner, d_out);
    default: return fail(B2L_ERR_UNSUPPORTED, "localext: element type %d", type);
  }
}
