// runtime.cu -- device selection, execution contexts (stream, events, timers), memory and error plumbing.
// One process drives one GPU (LOCAL_RANK, overridable with SCS_B200_DEVICE).
#include "../common.cuh"
#include "../dev_api.h"
#include <atomic>
#include <map>
#include <mutex>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <vector>

static std::atomic<int> g_init{0};  // 0 = not tried, 1 = ok, -1 = failed
static int g_dev = 0;
static int g_num_sms = B200_NUM_SMS_FALLBACK;
static thread_local char t_err[512] = "";  // a refused call on one thread cannot overwrite another thread's message
static char g_init_err[512] = "";          // why the one runtime initialisation failed, for every thread
static std::atomic<long long> g_launches{0};
static void *g_stage = nullptr;  // pinned staging buffer for pageable host copies
static size_t g_stage_bytes = 0;

// ---------------------------------------------------------------------------------------------
// Execution contexts. Everything a solve enqueues goes to the stream of the context bound to the calling thread, and
// its timer events, section ring and launch counter are that context's. Each workspace owns a context (or shares its
// parent's) and every entry point binds it for the length of the call (b200_ctx_enter / b200_ctx_leave), so two
// threads solving two workspaces share no stream, event or counter. Calls bound to no workspace -- the dev-API
// tests, the timing helpers -- run on the process context g_default. Device memory blocks freed while a context is
// current park on that context's own list (see b200_free); include/scs_b200.h documents the threading rules.
#define SEC_RING 1024
#define SEC_MAX 8
struct B200Ctx {
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr, ev_join = nullptr;
  // section timers: see b200_section_mark
  cudaEvent_t sec_ev[SEC_RING + 1];
  int sec_tag[SEC_RING + 1];
  int sec_n = 0;  // marks recorded since the last flush (event 0 = the open mark)
  int sec_made = 0;
  double sec_ms[SEC_MAX];
  std::atomic<long long> launches{0};  // the process context is shared by the unbound calls of every thread
  // device and pinned host blocks freed while this context was current: reused by this context only (guarded by
  // g_pool_mu), merged into the shared pool when the context is released
  std::multimap<size_t, void *> free_dev, free_host;
  size_t cached_dev = 0, cached_host = 0;
};
static B200Ctx g_default;
static thread_local B200Ctx *t_ctx = nullptr;
static inline B200Ctx *cur() { return t_ctx ? t_ctx : &g_default; }
static std::mutex g_init_mu, g_stage_mu, g_ctx_mu;
static std::vector<B200Ctx *> g_ctx_parked;  // released contexts, stream and events kept for the next workspace
static std::vector<B200Ctx *> g_ctx_all;     // every context made, the process context included (under g_ctx_mu)
// every entry point that touches the device first binds the calling thread to it (cudaSetDevice is per thread)
static inline void bind_thread() {
  if (g_init == 1) cudaSetDevice(g_dev);
}

extern "C" void b200_set_error(const char *what, cudaError_t e, const char *file, int line) {
  snprintf(t_err, sizeof(t_err), "%s:%d: %s -> %s", file, line, what, cudaGetErrorString(e));
  if (getenv("SCS_B200_VERBOSE")) fprintf(stderr, "scs_b200: %s\n", t_err);
}
extern "C" void b200_count_launch(int n) {
  g_launches += n;
  cur()->launches += n;
}
extern "C" long long b200_launches(void) { return g_launches.load(); }
extern "C" long long b200_ctx_launches(void) { return cur()->launches.load(); }
extern "C" const char *b200_last_error(void) { return t_err; }

static int ctx_make(B200Ctx *c) {
  CUDA_OK(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
  CUDA_OK(cudaEventCreate(&c->ev0));
  CUDA_OK(cudaEventCreate(&c->ev1));
  CUDA_OK(cudaEventCreateWithFlags(&c->ev_join, cudaEventDisableTiming));
  return 0;
}
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
  if (g_init == -1) {
    snprintf(t_err, sizeof(t_err), "%s", g_init_err);
    return -1;
  }
  g_init = -1;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) {
    snprintf(t_err, sizeof(t_err), "no CUDA device visible");
    snprintf(g_init_err, sizeof(g_init_err), "%s", t_err);
    return -1;
  }
  const char *e = getenv("SCS_B200_DEVICE");
  if (!e) e = getenv("LOCAL_RANK");
  g_dev = e ? atoi(e) % ndev : 0;
  CUDA_OK(cudaSetDevice(g_dev));
  cudaDeviceProp prop;
  CUDA_OK(cudaGetDeviceProperties(&prop, g_dev));
  if (prop.major != 9 || prop.minor != 0) {
    snprintf(t_err, sizeof(t_err), "device %d is sm_%d%d; this library is built for sm_90a only",
             g_dev, prop.major, prop.minor);
    snprintf(g_init_err, sizeof(g_init_err), "%s", t_err);
    return -1;
  }
  g_num_sms = prop.multiProcessorCount;
  if (ctx_make(&g_default) != 0) return -1;
  {
    std::lock_guard<std::mutex> lk(g_ctx_mu);
    g_ctx_all.push_back(&g_default);
  }
  g_stage_bytes = (size_t)64 << 20;
  CUDA_OK(cudaMallocHost(&g_stage, g_stage_bytes));
  g_init = 1;
  return 0;
}
extern "C" int b200_device_ok(void) { return b200_runtime_init() == 0; }
extern "C" int b200_num_sms(void) { return g_num_sms; }
extern "C" void *b200_stream(void) { return (void *)cur()->stream; }

// A context from the parked ones, else a new one (a stream and three events; the 1 025 section events are made at the
// context's first solve). NULL when the runtime or a CUDA call fails.
extern "C" B200Ctx *b200_ctx_create(void) {
  if (b200_runtime_init() != 0) return nullptr;
  {
    std::lock_guard<std::mutex> lk(g_ctx_mu);
    if (!g_ctx_parked.empty()) {
      B200Ctx *c = g_ctx_parked.back();
      g_ctx_parked.pop_back();
      c->launches = 0;
      return c;
    }
  }
  B200Ctx *c = new B200Ctx();
  if (ctx_make(c) != 0) {
    if (c->stream) cudaStreamDestroy(c->stream);
    if (c->ev0) cudaEventDestroy(c->ev0);
    if (c->ev1) cudaEventDestroy(c->ev1);
    if (c->ev_join) cudaEventDestroy(c->ev_join);
    delete c;
    return nullptr;
  }
  std::lock_guard<std::mutex> lk(g_ctx_mu);
  g_ctx_all.push_back(c);
  return c;
}
extern "C" B200Ctx *b200_ctx_enter(B200Ctx *c) {
  B200Ctx *prev = t_ctx;
  t_ctx = c;
  bind_thread();
  return prev;
}
extern "C" void b200_ctx_leave(B200Ctx *prev) { t_ctx = prev; }
extern "C" B200Ctx *b200_ctx_bound(void) { return t_ctx; }

// ---------------------------------------------------------------------------------------------
// Device memory: a small caching allocator. cudaMalloc / cudaFree cost milliseconds per call for the large buffers of
// a workspace (and cudaFree synchronises the device); a process that solves one problem after another -- the common
// production pattern, and bench.py's end-to-end call -- gets the blocks of the previous workspace back instead.
// Freed blocks are kept in size-keyed lists (exact size match on reuse: workspaces of one problem shape reuse each
// other's blocks) up to B200_POOL_MAX_BYTES; beyond that, and under memory pressure (a failed cudaMalloc trims the
// pool and retries), blocks go back to the driver. SCS_B200_POOL=0 disables caching; scs_b200_release_memory() trims.
// Reused blocks are NOT zeroed -- like fresh cudaMalloc memory, whose contents are unspecified too.
// Streams: a block freed while a context is current may still be read or written by work enqueued on that context's
// stream, so it goes to the context's own list and only that context reuses it: stream order makes the reuse safe.
// b200_ctx_release synchronises the stream and then merges the list into the shared pool g_pool_free, so every block
// in the shared pool is idle and b200_malloc may hand it to any stream. A block in a context's list is idle once that
// context's stream has been synchronised after the block was freed: pool_drain_locked does so for every context, under
// the pool lock (which every free takes), to give every cached block back.
static std::mutex g_pool_mu;
static std::multimap<size_t, void *> g_pool_free;  // size -> idle block
static std::map<void *, size_t> g_pool_size;       // every live or cached block we handed out -> its size
static size_t g_pool_cached = 0;                   // bytes cached in the shared pool and every context's list
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
// a context's lists into the shared pool; its stream must have been synchronised
static void ctx_merge_locked(B200Ctx *c) {
  g_pool_free.insert(c->free_dev.begin(), c->free_dev.end());
  g_hpool_free.insert(c->free_host.begin(), c->free_host.end());
  c->free_dev.clear();
  c->free_host.clear();
  c->cached_dev = c->cached_host = 0;
}
// the shared pool back to the driver: its blocks are idle, no stream needs to be waited for
static void pool_trim_locked() {
  for (auto &kv : g_pool_free) {
    cudaFree(kv.second);
    g_pool_size.erase(kv.second);
    g_pool_cached -= kv.first;
  }
  g_pool_free.clear();
  for (auto &kv : g_hpool_free) {
    cudaFreeHost(kv.second);
    g_hpool_size.erase(kv.second);
    g_hpool_cached -= kv.first;
  }
  g_hpool_free.clear();
}
// Every context's lists into the shared pool and the pool back to the driver. A context's blocks were freed before the
// pool lock was taken, so the work that used them was enqueued before this synchronisation of its stream; a context in
// the middle of a call on another thread only waits for the lock to free or allocate.
static void pool_drain_locked() {
  std::vector<B200Ctx *> all;
  {
    std::lock_guard<std::mutex> lk(g_ctx_mu);
    all = g_ctx_all;
  }
  for (B200Ctx *c : all) {
    if (c->free_dev.empty() && c->free_host.empty()) continue;
    cudaStreamSynchronize(c->stream);
    ctx_merge_locked(c);
  }
  pool_trim_locked();
}
extern "C" void scs_b200_release_memory(void) {
  if (g_init != 1) return;
  bind_thread();
  std::lock_guard<std::mutex> lk(g_pool_mu);
  pool_drain_locked();
}
// Synchronises the context's stream, merges its lists into the shared pool and parks it for b200_ctx_create.
extern "C" void b200_ctx_release(B200Ctx *c) {
  if (!c || c == &g_default) return;
  bind_thread();
  cudaStreamSynchronize(c->stream);
  {
    std::lock_guard<std::mutex> lk(g_pool_mu);
    ctx_merge_locked(c);
  }
  std::lock_guard<std::mutex> lk(g_ctx_mu);
  g_ctx_parked.push_back(c);
}

// a cached block of `bytes`: the current context's own list first, then the shared pool; nullptr if neither has one
static void *pool_take_locked(std::multimap<size_t, void *> &own, size_t &own_cached,
                              std::multimap<size_t, void *> &shared, size_t &total, size_t bytes) {
  std::multimap<size_t, void *> *from = &own;
  auto it = own.find(bytes);
  if (it == own.end()) {
    from = &shared;
    it = shared.find(bytes);
    if (it == shared.end()) return nullptr;
  } else {
    own_cached -= bytes;
  }
  void *p = it->second;
  from->erase(it);
  total -= bytes;
  return p;
}

extern "C" void *b200_malloc(size_t bytes) {
  if (b200_runtime_init() != 0) return nullptr;
  void *p = nullptr;
  if (bytes == 0) bytes = 16;
  B200Ctx *c = cur();
  std::lock_guard<std::mutex> lk(g_pool_mu);
  if (pool_enabled()) {
    p = pool_take_locked(c->free_dev, c->cached_dev, g_pool_free, g_pool_cached, bytes);
    if (p) return p;
  }
  cudaError_t e = cudaMalloc(&p, bytes);
  if (e != cudaSuccess && g_pool_cached > 0) {
    // memory pressure: give every cached block back and retry once
    cudaGetLastError();
    pool_drain_locked();
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
  B200Ctx *c = cur();
  std::lock_guard<std::mutex> lk(g_pool_mu);
  auto it = g_pool_size.find(p);
  if (it == g_pool_size.end()) {  // not ours (cannot happen): hand it to the driver
    cudaFree(p);
    return;
  }
  const size_t bytes = it->second;
  if (pool_enabled() && g_pool_cached + bytes <= B200_POOL_MAX_BYTES) {
    // the block may still be in use by work enqueued on the current context's stream: only that context reuses it
    c->free_dev.insert({bytes, p});
    c->cached_dev += bytes;
    g_pool_cached += bytes;
    return;
  }
  g_pool_size.erase(it);
  cudaFree(p);
}
// pinned host blocks (a few control words and the AA's small R factor per workspace) are cached the same way, on the
// same per-context rule: cudaMallocHost / cudaFreeHost are device-wide synchronisations and cost far more than the
// blocks are worth
extern "C" void *b200_host_alloc(size_t bytes) {
  if (b200_runtime_init() != 0) return nullptr;
  void *p = nullptr;
  if (bytes == 0) bytes = 16;
  B200Ctx *c = cur();
  std::lock_guard<std::mutex> lk(g_pool_mu);
  if (pool_enabled()) {
    p = pool_take_locked(c->free_host, c->cached_host, g_hpool_free, g_hpool_cached, bytes);
    if (p) return p;
  }
  if (cudaMallocHost(&p, bytes) != cudaSuccess) return nullptr;
  g_hpool_size[p] = bytes;
  return p;
}
extern "C" void b200_host_free(void *p) {
  if (!p) return;
  B200Ctx *c = cur();
  std::lock_guard<std::mutex> lk(g_pool_mu);
  auto it = g_hpool_size.find(p);
  if (it != g_hpool_size.end() && pool_enabled() && g_hpool_cached + it->second <= B200_HPOOL_MAX_BYTES) {
    c->free_host.insert({it->second, p});
    c->cached_host += it->second;
    g_hpool_cached += it->second;
    return;
  }
  if (it != g_hpool_size.end()) g_hpool_size.erase(it);
  cudaFreeHost(p);
}

// Bytes and the largest single copy of b200_h2d and b200_d2h, per direction since the last reset (a copy staged in
// chunks counts as one): what lets a caller check that a device-resident problem never crosses PCIe.
static long long g_xfer[4];  // h2d bytes, h2d largest, d2h bytes, d2h largest
static void count_xfer(int dir, size_t bytes) {
  std::lock_guard<std::mutex> lk(g_stage_mu);
  g_xfer[2 * dir] += (long long)bytes;
  if ((long long)bytes > g_xfer[2 * dir + 1]) g_xfer[2 * dir + 1] = (long long)bytes;
}
extern "C" void scs_b200_transfer_stats(long long out[4]) {
  std::lock_guard<std::mutex> lk(g_stage_mu);
  for (int i = 0; i < 4; ++i) out[i] = g_xfer[i];
}
extern "C" void scs_b200_transfer_stats_reset(void) {
  std::lock_guard<std::mutex> lk(g_stage_mu);
  for (int i = 0; i < 4; ++i) g_xfer[i] = 0;
}

// 1 if p is device (or managed) memory of the library's device, else 0
extern "C" int b200_is_device_ptr(const void *p) {
  if (!p || b200_runtime_init() != 0) return 0;
  cudaPointerAttributes at;
  if (cudaPointerGetAttributes(&at, p) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return (at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged) && at.device == g_dev;
}
// Ordering with a caller's stream (NULL: the legacy default stream). The context's stream is non-blocking, so nothing
// orders it with the caller's work implicitly: an event recorded on one stream is waited for by the other. Neither
// call blocks the host.
static int join(cudaStream_t from, cudaStream_t to) {
  CUDA_OK(cudaEventRecord(cur()->ev_join, from));
  CUDA_OK(cudaStreamWaitEvent(to, cur()->ev_join, 0));
  return 0;
}
extern "C" int b200_wait_for_caller(void *caller_stream) {
  if (b200_runtime_init() != 0) return -1;
  return join((cudaStream_t)caller_stream, cur()->stream);
}
extern "C" int b200_caller_waits(void *caller_stream) {
  if (b200_runtime_init() != 0) return -1;
  return join(cur()->stream, (cudaStream_t)caller_stream);
}

// Host<->device copies. The caller's buffer may be pageable: stage through the
// pinned bounce buffer in chunks so that the copy is a true async DMA and the
// caller's memory can be reused as soon as the call returns. The bounce buffer is
// shared by every context behind g_stage_mu; each copy drains its own stream.
extern "C" int b200_h2d(void *d_dst, const void *src, size_t bytes) {
  if (b200_runtime_init() != 0) return -1;
  cudaStream_t st = cur()->stream;
  count_xfer(0, bytes);
  cudaPointerAttributes at;
  bool pinned = (cudaPointerGetAttributes(&at, src) == cudaSuccess && at.type == cudaMemoryTypeHost);
  cudaGetLastError();
  if (pinned) {
    CUDA_OK(cudaMemcpyAsync(d_dst, src, bytes, cudaMemcpyHostToDevice, st));
    return 0;
  }
  CUDA_OK(cudaStreamSynchronize(st));  // the stream's earlier work drains outside the shared buffer's lock
  std::lock_guard<std::mutex> lk(g_stage_mu);
  size_t off = 0;
  while (off < bytes) {
    size_t c = bytes - off < g_stage_bytes ? bytes - off : g_stage_bytes;
    CUDA_OK(cudaStreamSynchronize(st));  // staging buffer free
    memcpy(g_stage, (const char *)src + off, c);
    CUDA_OK(cudaMemcpyAsync((char *)d_dst + off, g_stage, c, cudaMemcpyHostToDevice, st));
    off += c;
  }
  CUDA_OK(cudaStreamSynchronize(st));
  return 0;
}
extern "C" int b200_d2h(void *dst, const void *d_src, size_t bytes) {
  if (b200_runtime_init() != 0) return -1;
  cudaStream_t st = cur()->stream;
  count_xfer(1, bytes);
  cudaPointerAttributes at;
  bool pinned = (cudaPointerGetAttributes(&at, dst) == cudaSuccess && at.type == cudaMemoryTypeHost);
  cudaGetLastError();
  if (pinned) {
    CUDA_OK(cudaMemcpyAsync(dst, d_src, bytes, cudaMemcpyDeviceToHost, st));
    return 0;
  }
  CUDA_OK(cudaStreamSynchronize(st));  // the stream's earlier work drains outside the shared buffer's lock
  std::lock_guard<std::mutex> lk(g_stage_mu);
  size_t off = 0;
  while (off < bytes) {
    size_t c = bytes - off < g_stage_bytes ? bytes - off : g_stage_bytes;
    CUDA_OK(cudaMemcpyAsync(g_stage, (const char *)d_src + off, c, cudaMemcpyDeviceToHost, st));
    CUDA_OK(cudaStreamSynchronize(st));
    memcpy((char *)dst + off, g_stage, c);
    off += c;
  }
  return 0;
}
extern "C" int b200_d2d(void *d_dst, const void *d_src, size_t bytes) {
  bind_thread();
  cudaStream_t st = cur()->stream;
  CUDA_OK(cudaMemcpyAsync(d_dst, d_src, bytes, cudaMemcpyDeviceToDevice, st));
  return 0;
}
extern "C" int b200_memset0(void *d_dst, size_t bytes) {
  if (b200_runtime_init() != 0) return -1;
  cudaStream_t st = cur()->stream;
  CUDA_OK(cudaMemsetAsync(d_dst, 0, bytes, st));
  return 0;
}
extern "C" int b200_sync(void) {
  if (b200_runtime_init() != 0) return -1;
  cudaStream_t st = cur()->stream;
  CUDA_OK(cudaStreamSynchronize(st));
  return 0;
}
extern "C" int b200_timer_start(void) {
  CUDA_OK(cudaEventRecord(cur()->ev0, cur()->stream));
  return 0;
}
extern "C" double b200_timer_stop_ms(void) {
  B200Ctx *c = cur();
  if (cudaEventRecord(c->ev1, c->stream) != cudaSuccess) return -1.0;
  if (cudaEventSynchronize(c->ev1) != cudaSuccess) return -1.0;
  float ms = 0.f;
  if (cudaEventElapsedTime(&ms, c->ev0, c->ev1) != cudaSuccess) return -1.0;
  return (double)ms;
}

// ---------------------------------------------------------------------------------------------
// Section timers on the device (ScsInfo.lin_sys_time / cone_time / accel_time, reference semantics
// src/scs.c:1360-1393,1472-1475 -- there a host clock around synchronous CPU code; here the work is
// asynchronous, so the sections are bracketed by CUDA events ON THE CONTEXT'S STREAM and the elapsed device
// time between consecutive marks is billed to the section named by the later mark).
// b200_section_mark(s): "everything enqueued since the previous mark belongs to section s".
// The marks of up to SEC_RING intervals are kept; b200_section_flush() (after any stream sync, e.g. at the
// convergence check every 25 iterations) adds them up and recycles the events. Ring and totals are the current
// context's.
extern "C" int b200_section_begin(void) {
  bind_thread();
  B200Ctx *c = cur();
  if (!c->sec_made) {
    for (int i = 0; i <= SEC_RING; ++i) CUDA_OK(cudaEventCreate(&c->sec_ev[i]));
    c->sec_made = 1;
  }
  for (int i = 0; i < SEC_MAX; ++i) c->sec_ms[i] = 0.0;
  c->sec_n = 0;
  CUDA_OK(cudaEventRecord(c->sec_ev[0], c->stream));
  return 0;
}
extern "C" int b200_section_flush(void) {
  B200Ctx *c = cur();
  if (!c->sec_made || c->sec_n == 0) return 0;
  CUDA_OK(cudaEventSynchronize(c->sec_ev[c->sec_n]));
  for (int i = 1; i <= c->sec_n; ++i) {
    float ms = 0.f;
    CUDA_OK(cudaEventElapsedTime(&ms, c->sec_ev[i - 1], c->sec_ev[i]));
    c->sec_ms[c->sec_tag[i]] += (double)ms;
  }
  // the last mark opens the next interval
  cudaEvent_t t = c->sec_ev[0];
  c->sec_ev[0] = c->sec_ev[c->sec_n];
  c->sec_ev[c->sec_n] = t;
  c->sec_n = 0;
  return 0;
}
extern "C" int b200_section_mark(int section) {
  B200Ctx *c = cur();
  if (!c->sec_made || section < 0 || section >= SEC_MAX) return -1;
  if (c->sec_n == SEC_RING && b200_section_flush() != 0) return -1;
  ++c->sec_n;
  c->sec_tag[c->sec_n] = section;
  CUDA_OK(cudaEventRecord(c->sec_ev[c->sec_n], c->stream));
  return 0;
}
extern "C" double b200_section_ms(int section) {
  return (section >= 0 && section < SEC_MAX) ? cur()->sec_ms[section] : 0.0;
}
