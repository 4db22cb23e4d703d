// runtime.cu -- device selection, the library stream, memory and error plumbing.
// One process drives one GPU (LOCAL_RANK, overridable with SCS_B200_DEVICE).
#include "../common.cuh"
#include "../dev_api.h"
#include <mutex>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

static int g_init = 0;  // 0 = not tried, 1 = ok, -1 = failed
static int g_dev = 0;
static int g_num_sms = B200_NUM_SMS_FALLBACK;
static cudaStream_t g_stream = nullptr;
static cudaEvent_t g_ev0 = nullptr, g_ev1 = nullptr;
static char g_err[512] = "";
static long long g_launches = 0;
static void *g_stage = nullptr;  // pinned staging buffer for pageable host copies
static size_t g_stage_bytes = 0;
// Threading (ADVICE r01): the library drives ONE device through ONE stream. Calls may come from any host
// thread -- every entry point that touches the device first binds the calling thread to that device
// (cudaSetDevice is thread-local state) -- but they are serialised where they share state: the init, and the
// pinned bounce buffer of the pageable-memory copies. Concurrent solves on the same stream are ordered by the
// stream; include/scs_b200.h documents that one process = one GPU = one solve at a time.
static std::mutex g_init_mu, g_stage_mu;
static inline void bind_thread() {
  if (g_init == 1) cudaSetDevice(g_dev);
}

extern "C" void b200_set_error(const char *what, cudaError_t e, const char *file, int line) {
  snprintf(g_err, sizeof(g_err), "%s:%d: %s -> %s", file, line, what, cudaGetErrorString(e));
  if (getenv("SCS_B200_VERBOSE")) fprintf(stderr, "scs_b200: %s\n", g_err);
}
extern "C" void b200_count_launch(int n) { g_launches += n; }
extern "C" long long b200_launches(void) { return g_launches; }
extern "C" const char *b200_last_error(void) { return g_err; }

extern "C" int b200_runtime_init(void) {
  if (g_init == 1) {
    bind_thread();
    return 0;
  }
  std::lock_guard<std::mutex> lk(g_init_mu);
  if (g_init == 1) {
    bind_thread();
    return 0;
  }
  if (g_init == -1) return -1;
  g_init = -1;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) {
    snprintf(g_err, sizeof(g_err), "no CUDA device visible");
    return -1;
  }
  const char *e = getenv("SCS_B200_DEVICE");
  if (!e) e = getenv("LOCAL_RANK");
  g_dev = e ? atoi(e) % ndev : 0;
  CUDA_OK(cudaSetDevice(g_dev));
  cudaDeviceProp prop;
  CUDA_OK(cudaGetDeviceProperties(&prop, g_dev));
  if (prop.major != 9 || prop.minor != 0) {
    snprintf(g_err, sizeof(g_err), "device %d is sm_%d%d; this library is built for sm_90a only",
             g_dev, prop.major, prop.minor);
    return -1;
  }
  g_num_sms = prop.multiProcessorCount;
  CUDA_OK(cudaStreamCreateWithFlags(&g_stream, cudaStreamNonBlocking));
  CUDA_OK(cudaEventCreate(&g_ev0));
  CUDA_OK(cudaEventCreate(&g_ev1));
  g_stage_bytes = (size_t)64 << 20;
  CUDA_OK(cudaMallocHost(&g_stage, g_stage_bytes));
  g_init = 1;
  return 0;
}
extern "C" int b200_device_ok(void) { return b200_runtime_init() == 0; }
extern "C" int b200_num_sms(void) { return g_num_sms; }
extern "C" void *b200_stream(void) { return (void *)g_stream; }

// ---------------------------------------------------------------------------------------------
// Device memory: a small caching allocator. cudaMalloc / cudaFree cost milliseconds per call for the large buffers of
// a workspace (and cudaFree synchronises the device); a process that solves one problem after another -- the common
// production pattern, and bench.py's end-to-end call -- gets the blocks of the previous workspace back instead.
// Freed blocks are kept in a size-keyed list (exact size match on reuse: workspaces of one problem shape reuse each
// other's blocks) up to B200_POOL_MAX_BYTES; beyond that, and under memory pressure (a failed cudaMalloc trims the
// pool and retries), blocks go back to the driver. SCS_B200_POOL=0 disables caching; scs_b200_release_memory() trims.
// Reused blocks are NOT zeroed -- like fresh cudaMalloc memory, whose contents are unspecified too.
#include <map>
#include <vector>
static std::mutex g_pool_mu;
static std::multimap<size_t, void *> g_pool_free;  // size -> block
static std::map<void *, size_t> g_pool_size;       // every live or cached block we handed out -> its size
static size_t g_pool_cached = 0;
// pinned host blocks, cached the same way (see b200_host_alloc)
static std::multimap<size_t, void *> g_hpool_free;
static std::map<void *, size_t> g_hpool_size;
static size_t g_hpool_cached = 0;
#define B200_HPOOL_MAX_BYTES ((size_t)64 << 20)
static int g_pool_on = -1;
#define B200_POOL_MAX_BYTES ((size_t)24 << 30)
static bool pool_enabled() {
  if (g_pool_on < 0) {
    const char *e = getenv("SCS_B200_POOL");
    g_pool_on = (e && atoi(e) == 0) ? 0 : 1;
  }
  return g_pool_on == 1;
}
static void pool_trim_locked() {
  for (auto &kv : g_pool_free) {
    cudaFree(kv.second);
    g_pool_size.erase(kv.second);
  }
  g_pool_free.clear();
  g_pool_cached = 0;
  for (auto &kv : g_hpool_free) {
    cudaFreeHost(kv.second);
    g_hpool_size.erase(kv.second);
  }
  g_hpool_free.clear();
  g_hpool_cached = 0;
}
extern "C" void scs_b200_release_memory(void) {
  if (g_init != 1) return;
  bind_thread();
  std::lock_guard<std::mutex> lk(g_pool_mu);
  cudaStreamSynchronize(g_stream);
  pool_trim_locked();
}

extern "C" void *b200_malloc(size_t bytes) {
  if (b200_runtime_init() != 0) return nullptr;
  void *p = nullptr;
  if (bytes == 0) bytes = 16;
  std::lock_guard<std::mutex> lk(g_pool_mu);
  if (pool_enabled()) {
    auto it = g_pool_free.find(bytes);
    if (it != g_pool_free.end()) {
      p = it->second;
      g_pool_free.erase(it);
      g_pool_cached -= bytes;
      return p;
    }
  }
  cudaError_t e = cudaMalloc(&p, bytes);
  if (e != cudaSuccess && g_pool_cached > 0) {  // memory pressure: give the cached blocks back and retry once
    cudaGetLastError();
    cudaStreamSynchronize(g_stream);
    pool_trim_locked();
    e = cudaMalloc(&p, bytes);
  }
  if (e != cudaSuccess) {
    b200_set_error("cudaMalloc", e, __FILE__, __LINE__);
    return nullptr;
  }
  g_pool_size[p] = bytes;
  return p;
}
extern "C" void b200_free(void *p) {
  if (!p) return;
  bind_thread();
  std::lock_guard<std::mutex> lk(g_pool_mu);
  auto it = g_pool_size.find(p);
  if (it == g_pool_size.end()) {  // not ours (cannot happen): hand it to the driver
    cudaFree(p);
    return;
  }
  const size_t bytes = it->second;
  if (pool_enabled() && g_pool_cached + bytes <= B200_POOL_MAX_BYTES) {
    // the block may still be in use by work enqueued on the library stream: every consumer of pooled memory is
    // ordered on that same stream, so handing it to the next b200_malloc is safe without a synchronisation
    g_pool_free.insert({bytes, p});
    g_pool_cached += bytes;
    return;
  }
  g_pool_size.erase(it);
  cudaFree(p);
}
// pinned host blocks (a few control words and the AA's small R factor per workspace) are cached the same way:
// cudaMallocHost / cudaFreeHost are device-wide synchronisations and cost far more than the blocks are worth
extern "C" void *b200_host_alloc(size_t bytes) {
  if (b200_runtime_init() != 0) return nullptr;
  void *p = nullptr;
  if (bytes == 0) bytes = 16;
  std::lock_guard<std::mutex> lk(g_pool_mu);
  if (pool_enabled()) {
    auto it = g_hpool_free.find(bytes);
    if (it != g_hpool_free.end()) {
      p = it->second;
      g_hpool_free.erase(it);
      g_hpool_cached -= bytes;
      return p;
    }
  }
  if (cudaMallocHost(&p, bytes) != cudaSuccess) return nullptr;
  g_hpool_size[p] = bytes;
  return p;
}
extern "C" void b200_host_free(void *p) {
  if (!p) return;
  std::lock_guard<std::mutex> lk(g_pool_mu);
  auto it = g_hpool_size.find(p);
  if (it != g_hpool_size.end() && pool_enabled() && g_hpool_cached + it->second <= B200_HPOOL_MAX_BYTES) {
    g_hpool_free.insert({it->second, p});
    g_hpool_cached += it->second;
    return;
  }
  if (it != g_hpool_size.end()) g_hpool_size.erase(it);
  cudaFreeHost(p);
}

// Host<->device copies. The caller's buffer may be pageable: stage through the
// pinned bounce buffer in chunks so that the copy is a true async DMA and the
// caller's memory can be reused as soon as the call returns.
extern "C" int b200_h2d(void *d_dst, const void *src, size_t bytes) {
  if (b200_runtime_init() != 0) return -1;
  cudaPointerAttributes at;
  bool pinned = (cudaPointerGetAttributes(&at, src) == cudaSuccess && at.type == cudaMemoryTypeHost);
  cudaGetLastError();
  if (pinned) {
    CUDA_OK(cudaMemcpyAsync(d_dst, src, bytes, cudaMemcpyHostToDevice, g_stream));
    return 0;
  }
  std::lock_guard<std::mutex> lk(g_stage_mu);
  size_t off = 0;
  while (off < bytes) {
    size_t c = bytes - off < g_stage_bytes ? bytes - off : g_stage_bytes;
    CUDA_OK(cudaStreamSynchronize(g_stream));  // staging buffer free
    memcpy(g_stage, (const char *)src + off, c);
    CUDA_OK(cudaMemcpyAsync((char *)d_dst + off, g_stage, c, cudaMemcpyHostToDevice, g_stream));
    off += c;
  }
  CUDA_OK(cudaStreamSynchronize(g_stream));
  return 0;
}
extern "C" int b200_d2h(void *dst, const void *d_src, size_t bytes) {
  if (b200_runtime_init() != 0) return -1;
  cudaPointerAttributes at;
  bool pinned = (cudaPointerGetAttributes(&at, dst) == cudaSuccess && at.type == cudaMemoryTypeHost);
  cudaGetLastError();
  if (pinned) {
    CUDA_OK(cudaMemcpyAsync(dst, d_src, bytes, cudaMemcpyDeviceToHost, g_stream));
    return 0;
  }
  std::lock_guard<std::mutex> lk(g_stage_mu);
  size_t off = 0;
  while (off < bytes) {
    size_t c = bytes - off < g_stage_bytes ? bytes - off : g_stage_bytes;
    CUDA_OK(cudaMemcpyAsync(g_stage, (const char *)d_src + off, c, cudaMemcpyDeviceToHost, g_stream));
    CUDA_OK(cudaStreamSynchronize(g_stream));
    memcpy((char *)dst + off, g_stage, c);
    off += c;
  }
  return 0;
}
extern "C" int b200_d2d(void *d_dst, const void *d_src, size_t bytes) {
  bind_thread();
  CUDA_OK(cudaMemcpyAsync(d_dst, d_src, bytes, cudaMemcpyDeviceToDevice, g_stream));
  return 0;
}
extern "C" int b200_memset0(void *d_dst, size_t bytes) {
  if (b200_runtime_init() != 0) return -1;
  CUDA_OK(cudaMemsetAsync(d_dst, 0, bytes, g_stream));
  return 0;
}
extern "C" int b200_sync(void) {
  if (b200_runtime_init() != 0) return -1;
  CUDA_OK(cudaStreamSynchronize(g_stream));
  return 0;
}
extern "C" int b200_timer_start(void) {
  CUDA_OK(cudaEventRecord(g_ev0, g_stream));
  return 0;
}
extern "C" double b200_timer_stop_ms(void) {
  if (cudaEventRecord(g_ev1, g_stream) != cudaSuccess) return -1.0;
  if (cudaEventSynchronize(g_ev1) != cudaSuccess) return -1.0;
  float ms = 0.f;
  if (cudaEventElapsedTime(&ms, g_ev0, g_ev1) != cudaSuccess) return -1.0;
  return (double)ms;
}

// ---------------------------------------------------------------------------------------------
// Section timers on the device (ScsInfo.lin_sys_time / cone_time / accel_time, reference semantics
// src/scs.c:1360-1393,1472-1475 -- there a host clock around synchronous CPU code; here the work is
// asynchronous, so the sections are bracketed by CUDA events ON THE LIBRARY STREAM and the elapsed device
// time between consecutive marks is billed to the section named by the later mark).
// b200_section_mark(s): "everything enqueued since the previous mark belongs to section s".
// The marks of up to SEC_RING intervals are kept; b200_section_flush() (after any stream sync, e.g. at the
// convergence check every 25 iterations) adds them up and recycles the events.
#define SEC_RING 1024
#define SEC_MAX 8
static cudaEvent_t g_sec_ev[SEC_RING + 1];
static int g_sec_tag[SEC_RING + 1];
static int g_sec_n = 0;       // marks recorded since the last flush (event 0 = the open mark)
static int g_sec_made = 0;
static double g_sec_ms[SEC_MAX];
extern "C" int b200_section_begin(void) {
  bind_thread();
  if (!g_sec_made) {
    for (int i = 0; i <= SEC_RING; ++i) CUDA_OK(cudaEventCreate(&g_sec_ev[i]));
    g_sec_made = 1;
  }
  for (int i = 0; i < SEC_MAX; ++i) g_sec_ms[i] = 0.0;
  g_sec_n = 0;
  CUDA_OK(cudaEventRecord(g_sec_ev[0], g_stream));
  return 0;
}
extern "C" int b200_section_flush(void) {
  if (!g_sec_made || g_sec_n == 0) return 0;
  CUDA_OK(cudaEventSynchronize(g_sec_ev[g_sec_n]));
  for (int i = 1; i <= g_sec_n; ++i) {
    float ms = 0.f;
    CUDA_OK(cudaEventElapsedTime(&ms, g_sec_ev[i - 1], g_sec_ev[i]));
    g_sec_ms[g_sec_tag[i]] += (double)ms;
  }
  // the last mark opens the next interval
  cudaEvent_t t = g_sec_ev[0];
  g_sec_ev[0] = g_sec_ev[g_sec_n];
  g_sec_ev[g_sec_n] = t;
  g_sec_n = 0;
  return 0;
}
extern "C" int b200_section_mark(int section) {
  if (!g_sec_made || section < 0 || section >= SEC_MAX) return -1;
  if (g_sec_n == SEC_RING && b200_section_flush() != 0) return -1;
  ++g_sec_n;
  g_sec_tag[g_sec_n] = section;
  CUDA_OK(cudaEventRecord(g_sec_ev[g_sec_n], g_stream));
  return 0;
}
extern "C" double b200_section_ms(int section) {
  return (section >= 0 && section < SEC_MAX) ? g_sec_ms[section] : 0.0;
}
