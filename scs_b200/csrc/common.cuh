// common.cuh -- device-side helpers shared by all kernels of the SCS hot path.
//
// * deterministic block reductions (fixed shuffle tree + fixed smem order)
// * "last block finishes" grid reductions: every block writes its partial to a
//   fixed slot, the last block to arrive sums the slots in index order, so a
//   launch with a fixed grid is bit-reproducible (no fp64 atomics anywhere)
// * the fp64 tensor-core mma (mma.sync m8n8k4 .f64 -> SASS DMMA)
// * sm_90a TMA 1-D bulk copy + mbarrier wrappers (cp.async.bulk -> SASS UBLKCP)
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define B200_NUM_SMS_FALLBACK 148
#define B200_RED_THREADS 512  // threads per block of every reduction-carrying vector kernel
#define B200_MAX_PARTIALS 2048
// stored column indices carry flags in bits 30/31 (kernels/spmv.cu, flagged stream); every reader masks
#define B200_FLAG_END 0x80000000u   // last stored entry of its (virtual) row
#define B200_FLAG_SKIP 0x40000000u  // explicit zero, not gathered: an empty row's one entry, or layout padding
#define B200_COLMASK 0x3fffffff

#define CUDA_OK(call)                                                        \
  do {                                                                       \
    cudaError_t e__ = (call);                                                \
    if (e__ != cudaSuccess) {                                                \
      b200_set_error(#call, e__, __FILE__, __LINE__);                        \
      return -1;                                                             \
    }                                                                        \
  } while (0)

extern "C" void b200_set_error(const char *what, cudaError_t e, const char *file, int line);
extern "C" void b200_count_launch(int n);

// ---------------------------------------------------------------- reductions
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Block-wide sum of NV values per thread; result valid in thread 0.
// smem must hold NV * 32 doubles. All threads must call.
template <int NV>
__device__ __forceinline__ void block_sum(double (&v)[NV], double *smem) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
#pragma unroll
  for (int i = 0; i < NV; ++i) v[i] = warp_sum(v[i]);
  __syncthreads();  // protect smem reuse across consecutive calls
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < NV; ++i) smem[i * 32 + wid] = v[i];
  }
  __syncthreads();
  if (wid == 0) {
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      double t = (lane < nw) ? smem[i * 32 + lane] : 0.0;
      v[i] = warp_sum(t);
    }
  }
}
template <int NV>
__device__ __forceinline__ void block_max(double (&v)[NV], double *smem) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
#pragma unroll
  for (int i = 0; i < NV; ++i) v[i] = warp_max(v[i]);
  __syncthreads();
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < NV; ++i) smem[i * 32 + wid] = v[i];
  }
  __syncthreads();
  if (wid == 0) {
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      double t = (lane < nw) ? smem[i * 32 + lane] : 0.0;  // all maxima here are of |.| >= 0
      v[i] = warp_max(t);
    }
  }
}

// Grid-level finish. Thread 0 of each block holds `mine[0..NV)`; it publishes
// them into partials[i * gridDim.x + blockIdx.x], then the last block to
// arrive (ticket counter) reduces the slots in index order with warp 0 and
// returns true in ALL threads of that block with the totals in thread 0's
// `mine`. `is_max[i]` selects max instead of sum for value i (bitmask).
// The counter is reset by the last block, so the buffer is reusable by the
// next kernel on the same stream.
// grid_finish_of: the same over `nblocks` participating blocks, this one being block `bid` (a kernel that runs the
// reduction of a smaller grid than its own).
template <int NV>
__device__ __forceinline__ bool grid_finish_of(double (&mine)[NV], double *partials, unsigned int *counter,
                                               unsigned max_mask, double *smem, unsigned nblocks, unsigned bid) {
  __shared__ int s_last;
  if (threadIdx.x == 0) {
#pragma unroll
    for (int i = 0; i < NV; ++i) partials[i * nblocks + bid] = mine[i];
    __threadfence();
    unsigned t = atomicAdd(counter, 1u);
    s_last = (t == nblocks - 1);
  }
  __syncthreads();
  if (!s_last) return false;
  __threadfence();
  // fixed-order reduction of gridDim.x slots: thread t accumulates slots t, t+B, ...
  double acc[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const bool mx = (max_mask >> i) & 1u;
    double a = 0.0;
    for (unsigned j = threadIdx.x; j < nblocks; j += blockDim.x) {
      double p = __ldcg(&partials[i * nblocks + j]);
      a = mx ? fmax(a, p) : a + p;
    }
    acc[i] = a;
  }
  // split by kind: run both reductions, pick per value
  double s[NV], m[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) { s[i] = acc[i]; m[i] = acc[i]; }
  block_sum<NV>(s, smem);
  block_max<NV>(m, smem);
  if (threadIdx.x == 0) {
#pragma unroll
    for (int i = 0; i < NV; ++i) mine[i] = ((max_mask >> i) & 1u) ? m[i] : s[i];
    *counter = 0u;
    __threadfence();
  }
  return true;
}
template <int NV>
__device__ __forceinline__ bool grid_finish(double (&mine)[NV], double *partials, unsigned int *counter,
                                            unsigned max_mask, double *smem) {
  return grid_finish_of<NV>(mine, partials, counter, max_mask, smem, gridDim.x, blockIdx.x);
}

// ---------------------------------------------------------------- Moreau post-scaling (cones)
// Every cone projection writes Pi(x) / r + s: the wrapper of reference cones.c:1583-1592, fused into its last pass.
// ry NULL => x + s; sv NULL => the bare projection (cone-operator tests).
__device__ __forceinline__ double moreau_post(double x, const double *ry, const double *sv, long long row) {
  return sv == nullptr ? x : ry ? x / ry[row] + sv[row] : x + sv[row];
}

// ---------------------------------------------------------------- fp64 tensor core (SASS DMMA)
// One m8n8k4 fp64 mma accumulated in place: {c0, c1} += A B over the warp, with this lane's A[g][t] in a, B[t][g]
// in b and C[g][2t], C[g][2t+1] in c0, c1 (g = lane >> 2, t = lane & 3).
__device__ __forceinline__ void dmma_m8n8k4(double &c0, double &c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
               : "+d"(c0), "+d"(c1)
               : "d"(a), "d"(b));
}

// ---------------------------------------------------------------- TMA / mbarrier (sm_90a)
__device__ __forceinline__ uint32_t smem_u32(const void *p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t *bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, unsigned parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t"
      "}" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
// 1-D bulk async copy global -> shared, completion on mbarrier (bytes multiple of 16,
// both addresses 16-byte aligned).
__device__ __forceinline__ void tma_load_1d(void *dst_smem, const void *src_gmem, unsigned bytes,
                                            uint64_t *bar, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint "
      "[%0], [%1], %2, [%3], %4;" ::"r"(smem_u32(dst_smem)),
      "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
      : "memory");
}
// ---------------------------------------------------------------- programmatic dependent launch (sm_90+)
// A kernel launched with cudaLaunchAttributeProgrammaticStreamSerialization may become resident while its
// predecessor in the stream is still running: everything before pdl_wait() (barrier init, descriptor and matrix
// prefetch -- data no predecessor writes) overlaps the predecessor's tail; pdl_wait() returns once the predecessor
// grid has completed and its writes are visible. pdl_launch_dependents() lets the SUCCESSOR's CTAs be scheduled
// as soon as every CTA of this grid has issued it (they then sit in their own pdl_wait()).
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

#ifdef __CUDACC__
// host: launch `kernel` on `st`, optionally as a programmatic dependent of the previous kernel in the stream
template <typename... KArgs, typename... Args>
static inline cudaError_t b200_launch(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                                      bool pdl, Args... args) {
  cudaLaunchConfig_t cfg;
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}
#endif

// ---------------------------------------------------------------- self-validating 16-byte messages (multi-GPU)
// A double travels as two 8-byte words, each carrying the 32-bit sequence number of the exchange in its upper half
// (NCCL's "LL" scheme): an 8-byte store is atomic, so a reader that sees the expected sequence number in BOTH words has
// the whole value -- no fence and no separate flag on either side.
__device__ __forceinline__ void ll_store(unsigned long long *dst2, double v, unsigned seq32) {
  const unsigned long long b = (unsigned long long)__double_as_longlong(v);
  const unsigned long long w0 = (b & 0xffffffffull) | ((unsigned long long)seq32 << 32);
  const unsigned long long w1 = (b >> 32) | ((unsigned long long)seq32 << 32);
  asm volatile("st.volatile.global.v2.u64 [%0], {%1, %2};" ::"l"(dst2), "l"(w0), "l"(w1) : "memory");
}
// raw 16-byte read; ll_valid / ll_value interpret it (lets a caller issue several reads before it looks at any)
__device__ __forceinline__ void ll_load_raw(const unsigned long long *src2, unsigned long long &w0,
                                            unsigned long long &w1) {
  asm volatile("ld.volatile.global.v2.u64 {%0, %1}, [%2];" : "=l"(w0), "=l"(w1) : "l"(src2));
}
__device__ __forceinline__ bool ll_valid(unsigned long long w0, unsigned long long w1, unsigned seq32) {
  return (unsigned)(w0 >> 32) == seq32 && (unsigned)(w1 >> 32) == seq32;
}
__device__ __forceinline__ double ll_value(unsigned long long w0, unsigned long long w1) {
  return __longlong_as_double((long long)((w0 & 0xffffffffull) | (w1 << 32)));
}
// returns true and the value once both halves carry seq32
__device__ __forceinline__ bool ll_try_load(const unsigned long long *src2, unsigned seq32, double &v) {
  unsigned long long w0, w1;
  asm volatile("ld.volatile.global.v2.u64 {%0, %1}, [%2];" : "=l"(w0), "=l"(w1) : "l"(src2) : "memory");
  if ((unsigned)(w0 >> 32) != seq32 || (unsigned)(w1 >> 32) != seq32) return false;
  v = __longlong_as_double((long long)((w0 & 0xffffffffull) | (w1 << 32)));
  return true;
}

__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
