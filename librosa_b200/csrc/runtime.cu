// runtime.cu — C ABI of libb2l.so (see include/b2l.h): errors, contexts, the input status word, memory, events
// and the multi-GPU split / join.  Launches no kernel.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <string>
#include <thread>
#include <vector>

#include "internal.h"

using namespace b2l;

// ------------------------------------------------------------------ errors
static thread_local std::string g_last_error;

int b2l::fail(int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_last_error = buf;
  return code;
}

extern "C" int b2l_version(void) { return B2L_VERSION; }
extern "C" const char* b2l_last_error(void) { return g_last_error.c_str(); }

// ------------------------------------------------------------------ launch configuration
int b2l::blocks_per_sm(b2l_ctx* c, const void* fn, int threads, size_t smem, int* occ, size_t smem_limit) {
  if (c->smem_limit_set.count(fn) == 0) {
    CUDA_TRY(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  (int)(smem_limit ? smem_limit : c->smem_optin)));
    c->smem_limit_set.insert(fn);
  }
  if (!occ) return B2L_OK;
  const auto key = std::make_tuple(fn, threads, smem);
  auto hit = c->occupancy.find(key);
  if (hit == c->occupancy.end()) {
    int n = 0;
    CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, fn, threads, smem));
    hit = c->occupancy.emplace(key, n).first;
  }
  *occ = hit->second;
  return B2L_OK;
}

// ------------------------------------------------------------------ NCCL (loaded on demand)
// Only the handful of entry points needed for the batch split / join; resolved from libnccl.so.2 with
// dlopen so that single-GPU use has no NCCL dependency.
typedef struct ncclComm* ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
typedef int ncclResult_t;
enum { ncclChar = 0 };
struct NcclApi {
  void* handle = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*Broadcast)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Send)(const void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Recv)(void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
};
static NcclApi g_nccl;

static int nccl_load() {
  if (g_nccl.handle) return B2L_OK;
  const char* names[] = {"libnccl.so.2", "libnccl.so"};
  void* h = nullptr;
  for (const char* n : names) {
    h = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
    if (h) break;
  }
  if (!h) return fail(B2L_ERR_NCCL, "cannot dlopen libnccl.so.2: %s", dlerror());
#define SYM(field, name)                                                       \
  *(void**)(&g_nccl.field) = dlsym(h, name);                                   \
  if (!g_nccl.field) return fail(B2L_ERR_NCCL, "libnccl is missing %s", name);
  SYM(GetUniqueId, "ncclGetUniqueId")
  SYM(CommInitRank, "ncclCommInitRank")
  SYM(CommDestroy, "ncclCommDestroy")
  SYM(Broadcast, "ncclBroadcast")
  SYM(Send, "ncclSend")
  SYM(Recv, "ncclRecv")
  SYM(GroupStart, "ncclGroupStart")
  SYM(GroupEnd, "ncclGroupEnd")
  SYM(AllReduce, "ncclAllReduce")
  SYM(GetErrorString, "ncclGetErrorString")
#undef SYM
  g_nccl.handle = h;
  return B2L_OK;
}
#define NCCL_TRY(expr)                                                                            \
  do {                                                                                            \
    ncclResult_t _r = (expr);                                                                     \
    if (_r != 0) return fail(B2L_ERR_NCCL, "%s: %s", #expr, g_nccl.GetErrorString ? g_nccl.GetErrorString(_r) : "?"); \
  } while (0)

// ------------------------------------------------------------------ objects
struct b2l_event {
  cudaEvent_t ev;
  int device;
};

// ------------------------------------------------------------------ library / device
extern "C" int b2l_device_count(int* count) {
  if (!count) return fail(B2L_ERR_INVALID, "count is NULL");
  CUDA_TRY(cudaGetDeviceCount(count));
  return B2L_OK;
}

extern "C" int b2l_ctx_create(int device, b2l_ctx** out) {
  if (!out) return fail(B2L_ERR_INVALID, "ctx out pointer is NULL");
  int n = 0;
  CUDA_TRY(cudaGetDeviceCount(&n));
  if (device < 0 || device >= n) return fail(B2L_ERR_INVALID, "device %d out of range (have %d)", device, n);
  cudaDeviceProp prop;
  CUDA_TRY(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0)
    return fail(B2L_ERR_UNSUPPORTED, "device %d is sm_%d%d; libb2l is built for sm_90a only (no fallback path)",
                device, prop.major, prop.minor);
  DeviceGuard g(device);
  b2l_ctx* c = new b2l_ctx();
  c->device = device;
  c->sm_count = prop.multiProcessorCount;
  c->smem_optin = prop.sharedMemPerBlockOptin;
  cudaError_t e = cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaMalloc((void**)&c->d_status, 256);
  if (e == cudaSuccess) e = cudaMemset(c->d_status, 0, 256);
  if (e != cudaSuccess) {
    if (c->stream) cudaStreamDestroy(c->stream);
    delete c;
    return fail(B2L_ERR_CUDA, "context setup: %s", cudaGetErrorString(e));
  }
  *out = c;
  return B2L_OK;
}

extern "C" int b2l_ctx_destroy(b2l_ctx* c) {
  if (!c) return B2L_OK;
  DeviceGuard g(c->device);
  if (c->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(c->comm);
  if (c->d_clip_max) cudaFree(c->d_clip_max);
  if (c->d_status) cudaFree(c->d_status);
  if (c->d_scratch) cudaFree(c->d_scratch);
  if (c->stream) cudaStreamSynchronize(c->stream);
  for (void* b : c->stage_bufs) cudaFreeHost(b);
  for (cudaEvent_t e : c->stage_evs) cudaEventDestroy(e);
  if (c->stream) cudaStreamDestroy(c->stream);
  delete c;
  return B2L_OK;
}

extern "C" int b2l_ctx_sync(b2l_ctx* c) {
  if (!c) return fail(B2L_ERR_INVALID, "ctx is NULL");
  DeviceGuard g(c->device);
  CUDA_TRY(cudaStreamSynchronize(c->stream));
  return B2L_OK;
}
extern "C" int b2l_ctx_device(const b2l_ctx* c, int* device) {
  if (!c || !device) return fail(B2L_ERR_INVALID, "NULL argument");
  *device = c->device;
  return B2L_OK;
}
extern "C" int b2l_ctx_sm_count(const b2l_ctx* c, int* sms) {
  if (!c || !sms) return fail(B2L_ERR_INVALID, "NULL argument");
  *sms = c->sm_count;
  return B2L_OK;
}
extern "C" int b2l_ctx_launch_count(const b2l_ctx* c, uint64_t* launches) {
  if (!c || !launches) return fail(B2L_ERR_INVALID, "NULL argument");
  *launches = c->launches;
  return B2L_OK;
}

// ------------------------------------------------------------------ device-side input validation
extern "C" int b2l_status_reset(b2l_ctx* c) {
  if (!c) return fail(B2L_ERR_INVALID, "ctx is NULL");
  DeviceGuard g(c->device);
  CUDA_TRY(cudaMemsetAsync(c->d_status, 0, sizeof(int), c->stream));
  return B2L_OK;
}
extern "C" int b2l_status_read(b2l_ctx* c, int* status) {
  if (!c || !status) return fail(B2L_ERR_INVALID, "NULL argument");
  DeviceGuard g(c->device);
  CUDA_TRY(cudaMemcpyAsync(status, c->d_status, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  CUDA_TRY(cudaStreamSynchronize(c->stream));
  return B2L_OK;
}

// ------------------------------------------------------------------ memory
int b2l::ensure_clip_max(b2l_ctx* c, size_t n_clips) {
  if (c->clip_max_cap < n_clips) {
    if (c->d_clip_max) {
      CUDA_TRY(cudaStreamSynchronize(c->stream));
      CUDA_TRY(cudaFree(c->d_clip_max));
      c->d_clip_max = nullptr;
      c->clip_max_cap = 0;
    }
    size_t cap = n_clips < 1024 ? 1024 : n_clips;
    CUDA_TRY(cudaMalloc((void**)&c->d_clip_max, cap * sizeof(unsigned int)));
    c->clip_max_cap = cap;
  }
  return B2L_OK;
}

extern "C" int b2l_alloc(b2l_ctx* c, size_t bytes, void** d_ptr) {
  if (!c || !d_ptr) return fail(B2L_ERR_INVALID, "NULL argument");
  DeviceGuard g(c->device);
  *d_ptr = nullptr;
  if (bytes == 0) bytes = 16;
  CUDA_TRY(cudaMalloc(d_ptr, bytes));
  return B2L_OK;
}
extern "C" int b2l_free(b2l_ctx* c, void* d_ptr) {
  if (!c) return fail(B2L_ERR_INVALID, "ctx is NULL");
  if (!d_ptr) return B2L_OK;
  DeviceGuard g(c->device);
  CUDA_TRY(cudaStreamSynchronize(c->stream));
  CUDA_TRY(cudaFree(d_ptr));
  return B2L_OK;
}
extern "C" int b2l_memset(b2l_ctx* c, void* d_ptr, int value, size_t bytes) {
  if (!c) return fail(B2L_ERR_INVALID, "ctx is NULL");
  DeviceGuard g(c->device);
  CUDA_TRY(cudaMemsetAsync(d_ptr, value, bytes, c->stream));
  return B2L_OK;
}
// Upload from PAGEABLE host memory (what a drop-in caller's ndarray is): cudaMemcpyAsync would stage it through
// the driver's single bounce buffer on the calling thread (10-20 GB/s).  Instead `nthreads` host threads copy
// 4 MB pieces into a ring of pinned buffers (two per thread) and enqueue the DMA of each piece on the context's
// stream as soon as it is staged, so the host-side copies run in parallel and overlap the PCIe transfer.
// Piece order on the stream is arbitrary (the pieces are disjoint); work enqueued after the call returns is
// ordered behind all of them.
static const size_t kStagePiece = 4u << 20;
static int staged_h2d(b2l_ctx* c, char* d_dst, const char* h_src, size_t bytes, int nthreads) {
  const size_t want = 2 * (size_t)nthreads;
  while (c->stage_bufs.size() < want) {
    void* b = nullptr;
    CUDA_TRY(cudaHostAlloc(&b, kStagePiece, cudaHostAllocPortable));
    c->stage_bufs.push_back(b);
    cudaEvent_t e;
    CUDA_TRY(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    c->stage_evs.push_back(e);
  }
  std::atomic<size_t> next(0);
  std::atomic<int> err(0);
  auto worker = [&](int w) {
    cudaSetDevice(c->device);
    for (int k = 0;; ++k) {
      const size_t off = next.fetch_add(1) * kStagePiece;
      if (off >= bytes || err.load()) break;
      const size_t len = std::min(kStagePiece, bytes - off);
      const int b = 2 * w + (k & 1);
      cudaError_t e = cudaEventSynchronize(c->stage_evs[b]);   // the DMA that last used this buffer is done
      if (e == cudaSuccess) {
        memcpy(c->stage_bufs[b], h_src + off, len);
        e = cudaMemcpyAsync(d_dst + off, c->stage_bufs[b], len, cudaMemcpyHostToDevice, c->stream);
      }
      if (e == cudaSuccess) e = cudaEventRecord(c->stage_evs[b], c->stream);
      if (e != cudaSuccess) err.store((int)e);
    }
  };
  std::vector<std::thread> pool;
  for (int w = 1; w < nthreads; ++w) pool.emplace_back(worker, w);
  worker(0);
  for (auto& t : pool) t.join();
  if (err.load()) {
    cudaGetLastError();
    return fail(B2L_ERR_CUDA, "staged upload: %s", cudaGetErrorString((cudaError_t)err.load()));
  }
  return B2L_OK;
}

extern "C" int b2l_h2d(b2l_ctx* c, void* d_dst, const void* h_src, size_t bytes) {
  if (!c) return fail(B2L_ERR_INVALID, "ctx is NULL");
  DeviceGuard g(c->device);
  if (bytes >= (16u << 20)) {
    static int threads = -1;   // B2L_H2D_THREADS: staging threads for pageable sources (0 = plain cudaMemcpyAsync)
    if (threads < 0) {
      const char* e = getenv("B2L_H2D_THREADS");
      threads = e && *e ? atoi(e) : 6;
      if (threads > 32) threads = 32;
    }
    cudaPointerAttributes attr;
    if (threads > 0 && cudaPointerGetAttributes(&attr, h_src) == cudaSuccess && attr.type == cudaMemoryTypeUnregistered)
      return staged_h2d(c, (char*)d_dst, (const char*)h_src, bytes, threads);
    cudaGetLastError();
  }
  CUDA_TRY(cudaMemcpyAsync(d_dst, h_src, bytes, cudaMemcpyHostToDevice, c->stream));
  return B2L_OK;
}
extern "C" int b2l_d2h(b2l_ctx* c, void* h_dst, const void* d_src, size_t bytes) {
  if (!c) return fail(B2L_ERR_INVALID, "ctx is NULL");
  DeviceGuard g(c->device);
  CUDA_TRY(cudaMemcpyAsync(h_dst, d_src, bytes, cudaMemcpyDeviceToHost, c->stream));
  return B2L_OK;
}
extern "C" int b2l_d2d(b2l_ctx* c, void* d_dst, const void* d_src, size_t bytes) {
  if (!c) return fail(B2L_ERR_INVALID, "ctx is NULL");
  DeviceGuard g(c->device);
  CUDA_TRY(cudaMemcpyAsync(d_dst, d_src, bytes, cudaMemcpyDeviceToDevice, c->stream));
  return B2L_OK;
}
extern "C" int b2l_copy2d(b2l_ctx* c, void* d_dst, size_t dst_pitch, const void* d_src, size_t src_pitch,
                          size_t width_bytes, size_t rows) {
  if (!c || !d_dst || !d_src) return fail(B2L_ERR_INVALID, "NULL argument");
  if (width_bytes == 0 || rows == 0) return B2L_OK;
  if (dst_pitch < width_bytes || src_pitch < width_bytes) return fail(B2L_ERR_INVALID, "pitch smaller than the row width");
  DeviceGuard g(c->device);
  CUDA_TRY(cudaMemcpy2DAsync(d_dst, dst_pitch, d_src, src_pitch, width_bytes, rows, cudaMemcpyDeviceToDevice, c->stream));
  return B2L_OK;
}
extern "C" int b2l_host_alloc(size_t bytes, void** h_ptr) {
  if (!h_ptr) return fail(B2L_ERR_INVALID, "NULL argument");
  if (bytes == 0) bytes = 16;
  CUDA_TRY(cudaHostAlloc(h_ptr, bytes, cudaHostAllocPortable));
  return B2L_OK;
}
extern "C" int b2l_host_free(void* h_ptr) {
  if (!h_ptr) return B2L_OK;
  CUDA_TRY(cudaFreeHost(h_ptr));
  return B2L_OK;
}
extern "C" int b2l_mem_info(b2l_ctx* c, size_t* free_bytes, size_t* total_bytes) {
  if (!c || !free_bytes || !total_bytes) return fail(B2L_ERR_INVALID, "NULL argument");
  DeviceGuard g(c->device);
  CUDA_TRY(cudaMemGetInfo(free_bytes, total_bytes));
  return B2L_OK;
}

// ------------------------------------------------------------------ events
extern "C" int b2l_event_create(b2l_ctx* c, b2l_event** ev) {
  if (!c || !ev) return fail(B2L_ERR_INVALID, "NULL argument");
  DeviceGuard g(c->device);
  b2l_event* e = new b2l_event();
  e->device = c->device;
  cudaError_t r = cudaEventCreate(&e->ev);
  if (r != cudaSuccess) {
    delete e;
    return fail(B2L_ERR_CUDA, "cudaEventCreate: %s", cudaGetErrorString(r));
  }
  *ev = e;
  return B2L_OK;
}
extern "C" int b2l_event_record(b2l_ctx* c, b2l_event* ev) {
  if (!c || !ev) return fail(B2L_ERR_INVALID, "NULL argument");
  DeviceGuard g(c->device);
  CUDA_TRY(cudaEventRecord(ev->ev, c->stream));
  return B2L_OK;
}
extern "C" int b2l_event_elapsed_ms(b2l_event* start, b2l_event* stop, float* ms) {
  if (!start || !stop || !ms) return fail(B2L_ERR_INVALID, "NULL argument");
  DeviceGuard g(stop->device);
  CUDA_TRY(cudaEventSynchronize(stop->ev));
  CUDA_TRY(cudaEventElapsedTime(ms, start->ev, stop->ev));
  return B2L_OK;
}
extern "C" int b2l_event_destroy(b2l_event* ev) {
  if (!ev) return B2L_OK;
  DeviceGuard g(ev->device);
  cudaEventDestroy(ev->ev);
  delete ev;
  return B2L_OK;
}

// ------------------------------------------------------------------ multi-GPU split / join
extern "C" int b2l_comm_unique_id(void* id128) {
  if (!id128) return fail(B2L_ERR_INVALID, "NULL argument");
  int rc = nccl_load();
  if (rc) return rc;
  ncclUniqueId id;
  NCCL_TRY(g_nccl.GetUniqueId(&id));
  memcpy(id128, &id, sizeof(id));
  return B2L_OK;
}
extern "C" int b2l_comm_init(b2l_ctx* c, const void* id128, int rank, int world) {
  if (!c || !id128) return fail(B2L_ERR_INVALID, "NULL argument");
  if (world < 1 || rank < 0 || rank >= world) return fail(B2L_ERR_INVALID, "bad rank %d / world %d", rank, world);
  int rc = nccl_load();
  if (rc) return rc;
  DeviceGuard g(c->device);
  ncclUniqueId id;
  memcpy(&id, id128, sizeof(id));
  NCCL_TRY(g_nccl.CommInitRank(&c->comm, world, id, rank));
  c->rank = rank;
  c->world = world;
  return B2L_OK;
}
extern "C" int b2l_comm_destroy(b2l_ctx* c) {
  if (!c || !c->comm) return B2L_OK;
  DeviceGuard g(c->device);
  cudaStreamSynchronize(c->stream);
  NCCL_TRY(g_nccl.CommDestroy(c->comm));
  c->comm = nullptr;
  c->world = 1;
  c->rank = 0;
  return B2L_OK;
}
extern "C" int b2l_comm_broadcast(b2l_ctx* c, void* d_buf, size_t bytes, int root) {
  if (!c || !c->comm) return fail(B2L_ERR_INVALID, "communicator not initialised");
  DeviceGuard g(c->device);
  NCCL_TRY(g_nccl.Broadcast(d_buf, d_buf, bytes, ncclChar, root, c->comm, c->stream));
  return B2L_OK;
}
extern "C" int b2l_comm_scatter(b2l_ctx* c, const void* d_full, void* d_shard, size_t shard_bytes, int root) {
  if (!c || !c->comm) return fail(B2L_ERR_INVALID, "communicator not initialised");
  DeviceGuard g(c->device);
  NCCL_TRY(g_nccl.GroupStart());
  if (c->rank == root)
    for (int r = 0; r < c->world; ++r)
      NCCL_TRY(g_nccl.Send((const char*)d_full + (size_t)r * shard_bytes, shard_bytes, ncclChar, r, c->comm, c->stream));
  NCCL_TRY(g_nccl.Recv(d_shard, shard_bytes, ncclChar, root, c->comm, c->stream));
  NCCL_TRY(g_nccl.GroupEnd());
  return B2L_OK;
}
extern "C" int b2l_comm_gather(b2l_ctx* c, const void* d_shard, void* d_full, size_t shard_bytes, int root) {
  if (!c || !c->comm) return fail(B2L_ERR_INVALID, "communicator not initialised");
  DeviceGuard g(c->device);
  NCCL_TRY(g_nccl.GroupStart());
  if (c->rank == root)
    for (int r = 0; r < c->world; ++r)
      NCCL_TRY(g_nccl.Recv((char*)d_full + (size_t)r * shard_bytes, shard_bytes, ncclChar, r, c->comm, c->stream));
  NCCL_TRY(g_nccl.Send(d_shard, shard_bytes, ncclChar, root, c->comm, c->stream));
  NCCL_TRY(g_nccl.GroupEnd());
  return B2L_OK;
}
extern "C" int b2l_comm_barrier(b2l_ctx* c) {
  if (!c || !c->comm) return fail(B2L_ERR_INVALID, "communicator not initialised");
  DeviceGuard g(c->device);
  int rc = ensure_clip_max(c, 1);
  if (rc) return rc;
  NCCL_TRY(g_nccl.AllReduce(c->d_clip_max, c->d_clip_max, 1, ncclChar, 0 /* ncclSum */, c->comm, c->stream));
  CUDA_TRY(cudaStreamSynchronize(c->stream));
  return B2L_OK;
}
