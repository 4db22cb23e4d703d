// gather_bench.cu -- what does ONE random 8-byte gather cost on B200?  (measurement tool, not product)
//
// The SpMV of a uniformly random sparse matrix does exactly one random fp64 gather per nonzero,
// and that gather -- not the 12 B/nnz matrix stream -- is what bounds it (DESIGN.md section 3.1).
// This binary measures the ceiling: a kernel that does nothing but read a coalesced int32 index
// stream and gather x[idx] (no shared memory, no row logic), for several load flavours, loads in
// flight per thread, occupancies and gather-vector sizes. Output: one line per variant with the
// time for N gathers and the rate in gathers / clock / SM.
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o scripts/bin/gather_bench scripts/gather_bench.cu
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <vector>

#define CK(x)                                                                      \
  do {                                                                             \
    cudaError_t e = (x);                                                           \
    if (e != cudaSuccess) {                                                        \
      printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__); \
      exit(1);                                                                     \
    }                                                                              \
  } while (0)

enum { M_NC = 0, M_CA = 1, M_CG = 2, M_CS = 3, M_CV = 4, M_NC_NOALLOC = 5, M_HALF = 6, M_V2 = 7, NMODES = 8 };
static const char *mode_name[NMODES] = {"ld.global.nc", "ld.global.ca", "ld.global.cg", "ld.global.cs",
                                        "ld.volatile", "nc.L1::no_allocate", "nc,16-of-32-lanes",
                                        "nc.v2.f64 (16B)"};

template <int MODE>
__device__ __forceinline__ double gload(const double *p) {
  double r;
  if (MODE == M_NC || MODE == M_HALF) asm volatile("ld.global.nc.f64 %0, [%1];" : "=d"(r) : "l"(p));
  else if (MODE == M_CA) asm volatile("ld.global.ca.f64 %0, [%1];" : "=d"(r) : "l"(p));
  else if (MODE == M_CG) asm volatile("ld.global.cg.f64 %0, [%1];" : "=d"(r) : "l"(p));
  else if (MODE == M_CS) asm volatile("ld.global.cs.f64 %0, [%1];" : "=d"(r) : "l"(p));
  else if (MODE == M_CV) asm volatile("ld.volatile.global.f64 %0, [%1];" : "=d"(r) : "l"(p));
  else if (MODE == M_NC_NOALLOC) asm volatile("ld.global.nc.L1::no_allocate.f64 %0, [%1];" : "=d"(r) : "l"(p));
  else {
    double r2;
    const double *q = (const double *)((uintptr_t)p & ~(uintptr_t)15);
    asm volatile("ld.global.nc.v2.f64 {%0, %1}, [%2];" : "=d"(r), "=d"(r2) : "l"(q));
    r = ((uintptr_t)p & 8) ? r2 : r;
  }
  return r;
}

// every warp takes chunks of 32*U consecutive indices; U independent gathers in flight per thread
template <int MODE, int U>
__global__ void k_gather(const int *__restrict__ idx, const double *__restrict__ x, double *__restrict__ out,
                         long long total) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  double acc = 0.0;
  for (long long base = warp * 32 * U; base + 32 * U <= total; base += nwarps * 32 * U) {
    int c[U];
    double v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) c[u] = __ldcs(&idx[base + u * 32 + lane]);
    if (MODE == M_HALF) {
#pragma unroll
      for (int u = 0; u < U; ++u) v[u] = (lane & 1) ? 0.0 : gload<MODE>(&x[c[u]]);
    } else {
#pragma unroll
      for (int u = 0; u < U; ++u) v[u] = gload<MODE>(&x[c[u]]);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) acc += v[u];
  }
  out[(long long)blockIdx.x * blockDim.x + threadIdx.x] = acc;
}

// plain streaming read of the same index stream (what the kernel costs without any gather)
__global__ void k_stream(const int *__restrict__ idx, double *__restrict__ out, long long total) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x, nt = (long long)gridDim.x * blockDim.x;
  long long acc = 0;
  for (long long i = t; i < total; i += nt) acc += __ldcs(&idx[i]);
  out[t] = (double)acc;
}

template <int MODE, int U>
static float run(const int *d_idx, const double *d_x, double *d_out, long long total, int threads, int bps,
                 int nsm, int reps, const int *d_flush_idx, long long flush_total) {
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  float best = 1e30f, sum = 0.f;
  const int grid = nsm * bps;
  for (int r = 0; r < reps + 1; ++r) {
    // evict the index stream / vector from L2 the way the CG loop does: stream another 160 MB
    k_stream<<<nsm * 4, 512>>>(d_flush_idx, d_out, flush_total);
    CK(cudaEventRecord(e0));
    k_gather<MODE, U><<<grid, threads>>>(d_idx, d_x, d_out, total);
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    float ms;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    if (r > 0) { sum += ms; if (ms < best) best = ms; }
  }
  CK(cudaEventDestroy(e0));
  CK(cudaEventDestroy(e1));
  return sum / reps;
}

template <int MODE>
static void sweep(const int *d_idx, const double *d_x, double *d_out, long long total, int nsm, double ghz,
                  long long vec_len, const int *d_flush, long long flush_total) {
  static const int cfg[][2] = {{256, 4}, {512, 2}, {512, 4}, {1024, 2}};
  for (int c = 0; c < 4; ++c) {
    const int th = cfg[c][0], bps = cfg[c][1];
    float ms[3];
    ms[0] = run<MODE, 2>(d_idx, d_x, d_out, total, th, bps, nsm, 5, d_flush, flush_total);
    ms[1] = run<MODE, 4>(d_idx, d_x, d_out, total, th, bps, nsm, 5, d_flush, flush_total);
    ms[2] = run<MODE, 8>(d_idx, d_x, d_out, total, th, bps, nsm, 5, d_flush, flush_total);
    const int us[3] = {2, 4, 8};
    for (int k = 0; k < 3; ++k) {
      const double n_g = (MODE == M_HALF) ? total / 2.0 : (double)total;
      printf("GATHER vec=%lld mode=\"%s\" threads=%d blocks/SM=%d U=%d : %.1f us  %.3f gathers/clk/SM  "
             "(%.0f Ggather/s)\n",
             vec_len, mode_name[MODE], th, bps, us[k], ms[k] * 1e3, n_g / (ms[k] * 1e-3) / (nsm * ghz * 1e9),
             n_g / (ms[k] * 1e-3) / 1e9);
    }
  }
}

int main(int argc, char **argv) {
  const long long total = argc > 1 ? atoll(argv[1]) : 10000000LL;
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  const int nsm = prop.multiProcessorCount;
  int khz = 0;
  CK(cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0));
  const double ghz = khz / 1e6;
  printf("device %s, %d SMs, %.3f GHz (max), N = %lld gathers per launch\n", prop.name, nsm, ghz, total);
  const long long vec_lens[3] = {1000000LL, 3000000LL, 4096LL};
  const long long flush_total = 40000000LL;  // 160 MB of int32 > 50 MB L2
  int *d_idx, *d_flush;
  double *d_x, *d_out;
  CK(cudaMalloc(&d_idx, (size_t)total * 4));
  CK(cudaMalloc(&d_flush, (size_t)flush_total * 4));
  CK(cudaMemset(d_flush, 0, (size_t)flush_total * 4));
  CK(cudaMalloc(&d_x, (size_t)3000000 * 8 + 64));
  CK(cudaMalloc(&d_out, (size_t)nsm * 8 * 1024 * 8));
  {
    std::vector<double> hx(3000000);
    for (size_t i = 0; i < hx.size(); ++i) hx[i] = 1.0 + 1e-6 * (double)(i % 977);
    CK(cudaMemcpy(d_x, hx.data(), hx.size() * 8, cudaMemcpyHostToDevice));
  }
  // baseline: the index stream alone
  {
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    CK(cudaMemset(d_idx, 0, (size_t)total * 4));
    float acc = 0;
    for (int r = 0; r < 6; ++r) {
      k_stream<<<nsm * 4, 512>>>(d_flush, d_out, flush_total);
      CK(cudaEventRecord(e0));
      k_stream<<<nsm * 4, 512>>>(d_idx, d_out, total);
      CK(cudaEventRecord(e1));
      CK(cudaEventSynchronize(e1));
      float ms;
      CK(cudaEventElapsedTime(&ms, e0, e1));
      if (r > 0) acc += ms;
    }
    printf("STREAM idx only (%lld int32, cold L2): %.1f us  %.0f GB/s\n", total, acc / 5 * 1e3,
           total * 4.0 / (acc / 5 * 1e-3) / 1e9);
  }
  for (int v = 0; v < 3; ++v) {
    const long long L = vec_lens[v];
    std::vector<int> h(total);
    uint64_t s = 0x9E3779B97F4A7C15ull + (uint64_t)v;
    for (long long i = 0; i < total; ++i) {
      s ^= s << 13; s ^= s >> 7; s ^= s << 17;
      h[i] = (int)(s % (uint64_t)L);
    }
    CK(cudaMemcpy(d_idx, h.data(), (size_t)total * 4, cudaMemcpyHostToDevice));
    sweep<M_NC>(d_idx, d_x, d_out, total, nsm, ghz, L, d_flush, flush_total);
    if (v < 2) {
      sweep<M_CA>(d_idx, d_x, d_out, total, nsm, ghz, L, d_flush, flush_total);
      sweep<M_CG>(d_idx, d_x, d_out, total, nsm, ghz, L, d_flush, flush_total);
      sweep<M_NC_NOALLOC>(d_idx, d_x, d_out, total, nsm, ghz, L, d_flush, flush_total);
      sweep<M_HALF>(d_idx, d_x, d_out, total, nsm, ghz, L, d_flush, flush_total);
      sweep<M_V2>(d_idx, d_x, d_out, total, nsm, ghz, L, d_flush, flush_total);
    }
    if (v == 0) {
      sweep<M_CS>(d_idx, d_x, d_out, total, nsm, ghz, L, d_flush, flush_total);
      sweep<M_CV>(d_idx, d_x, d_out, total, nsm, ghz, L, d_flush, flush_total);
    }
  }
  return 0;
}
