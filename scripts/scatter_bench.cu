// scatter_bench.cu -- what does ONE random fp64 `red.global.add` cost on H100, alone and next to a gather?
// (measurement tool, not product; companion of gather_bench.cu)
//
// Question (VERDICT r01, next-round item 4-iv): the CG operator G p = R_x p + A' R_y^-1 A p is applied today as
// two gather SpMVs (24 B/nnz of matrix stream, 2 random 8-byte gathers per nonzero).  A ONE-PASS form walks the
// rows of A once: t_i = (sum_j A_ij p_j) / R_i  (gather), then Gp_j += A_ij t_i (scatter with red.global.add.f64):
// 12 B/nnz of stream, one gather + one reduction per nonzero.  Whether it wins is decided by the throughput of
// the L2 atomic units and by whether reductions (SM->L2 request path) overlap gathers (L2->SM response path).
//
// Kernels (N nonzeros as rows of exactly 4 entries, random columns in a vector of length L):
//   gather4   : per row 4 gathers, sum, store t          (= one SpMV of the two-pass form, minus row logic)
//   scatter4  : per row read t, 4 x red.add               (the scatter ceiling)
//   onepass4  : per row 4 gathers, t = sum/R, 4 x red.add (the fused candidate) + block-reduced dot
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o scripts/bin/scatter_bench scripts/scatter_bench.cu
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <vector>

#define CK(x)                                                                        \
  do {                                                                               \
    cudaError_t e = (x);                                                             \
    if (e != cudaSuccess) {                                                          \
      printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__); \
      exit(1);                                                                       \
    }                                                                                \
  } while (0)

__device__ __forceinline__ void red_add(double *p, double v) {
  asm volatile("red.global.add.f64 [%0], %1;" ::"l"(p), "d"(v) : "memory");
}
__device__ __forceinline__ int4 ld_stream_i4(const int4 *p) {
  int4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.s32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ double2 ld_stream_d2(const double2 *p) {
  double2 r;
  asm volatile("ld.global.nc.L1::no_allocate.v2.f64 {%0,%1}, [%2];" : "=d"(r.x), "=d"(r.y) : "l"(p));
  return r;
}

// MODE 0: gather only, 1: scatter only, 2: one pass
template <int MODE>
__global__ void k_rows4(const int4 *__restrict__ idx, const double2 *__restrict__ vals, const double *__restrict__ p,
                        const double *__restrict__ rinv, double *__restrict__ t, double *gp, long long nrows,
                        double *dot_out) {
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x, nt = (long long)gridDim.x * blockDim.x;
  double dot = 0.0;
  for (long long r = tid; r < nrows; r += nt) {
    const int4 c = ld_stream_i4(&idx[r]);
    const double2 a01 = ld_stream_d2(&vals[2 * r]), a23 = ld_stream_d2(&vals[2 * r + 1]);
    double s;
    if (MODE == 1) {
      s = t[r];
    } else {
      const double x0 = __ldg(&p[c.x]), x1 = __ldg(&p[c.y]), x2 = __ldg(&p[c.z]), x3 = __ldg(&p[c.w]);
      s = a01.x * x0 + a01.y * x1 + a23.x * x2 + a23.y * x3;
      s *= rinv[r];
    }
    if (MODE == 0) {
      t[r] = s;
    } else {
      red_add(&gp[c.x], a01.x * s);
      red_add(&gp[c.y], a01.y * s);
      red_add(&gp[c.z], a23.x * s);
      red_add(&gp[c.w], a23.y * s);
    }
    dot += s * s;
  }
  // cheap block reduce so the dot is not optimised away
  for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
  if ((threadIdx.x & 31) == 0 && dot == 123.456) dot_out[blockIdx.x] = dot;
}

__global__ void k_flush(const int *__restrict__ idx, double *__restrict__ out, long long total) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x, nt = (long long)gridDim.x * blockDim.x;
  long long acc = 0;
  for (long long i = t; i < total; i += nt) acc += __ldcs(&idx[i]);
  if (acc == 12345) out[t] = (double)acc;
}

template <int MODE>
static float run(const int4 *idx, const double2 *vals, const double *p, const double *rinv, double *t, double *gp,
                 long long nrows, double *dot, int threads, int grid, const int *flush, long long flush_total,
                 double *out, int nsm) {
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  float sum = 0.f;
  const int reps = 6;
  for (int r = 0; r < reps + 1; ++r) {
    k_flush<<<nsm * 4, 512>>>(flush, out, flush_total);
    CK(cudaEventRecord(e0));
    k_rows4<MODE><<<grid, threads>>>(idx, vals, p, rinv, t, gp, nrows, dot);
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    float ms;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    if (r > 0) sum += ms;
  }
  CK(cudaEventDestroy(e0));
  CK(cudaEventDestroy(e1));
  return sum / reps;
}

int main(int argc, char **argv) {
  const long long nnz = argc > 1 ? atoll(argv[1]) : 10000000LL;
  const long long nrows = nnz / 4;
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  const int nsm = prop.multiProcessorCount;
  printf("device %s, %d SMs; %lld nonzeros as %lld rows of 4\n", prop.name, nsm, nnz, nrows);
  const long long flush_total = 40000000LL;
  int *d_flush;
  int4 *d_idx;
  double2 *d_vals;
  double *d_p, *d_rinv, *d_t, *d_gp, *d_dot, *d_out;
  CK(cudaMalloc(&d_flush, flush_total * 4));
  CK(cudaMemset(d_flush, 0, flush_total * 4));
  CK(cudaMalloc(&d_idx, nrows * 16));
  CK(cudaMalloc(&d_vals, nrows * 32));
  CK(cudaMalloc(&d_p, 3000000 * 8));
  CK(cudaMalloc(&d_gp, 3000000 * 8));
  CK(cudaMalloc(&d_rinv, nrows * 8));
  CK(cudaMalloc(&d_t, nrows * 8));
  CK(cudaMalloc(&d_dot, 65536 * 8));
  CK(cudaMalloc(&d_out, (size_t)nsm * 4 * 512 * 8));
  {
    std::vector<double> h(3000000, 1.0);
    CK(cudaMemcpy(d_p, h.data(), h.size() * 8, cudaMemcpyHostToDevice));
    CK(cudaMemset(d_gp, 0, 3000000 * 8));
    std::vector<double> hr(nrows, 0.5), hv(nnz, 0.25);
    CK(cudaMemcpy(d_rinv, hr.data(), nrows * 8, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d_t, hr.data(), nrows * 8, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d_vals, hv.data(), nnz * 8, cudaMemcpyHostToDevice));
  }
  const long long Ls[2] = {1000000LL, 3000000LL};
  for (int v = 0; v < 2; ++v) {
    const long long L = Ls[v];
    std::vector<int> h(nnz);
    uint64_t s = 0x9E3779B97F4A7C15ull + (uint64_t)v;
    for (long long i = 0; i < nnz; ++i) {
      s ^= s << 13; s ^= s >> 7; s ^= s << 17;
      h[i] = (int)(s % (uint64_t)L);
    }
    CK(cudaMemcpy(d_idx, h.data(), nnz * 4, cudaMemcpyHostToDevice));
    static const int cfg[][2] = {{256, 4}, {256, 8}, {512, 4}, {1024, 2}};
    for (int c = 0; c < 4; ++c) {
      const int th = cfg[c][0], grid = nsm * cfg[c][1];
      const float g = run<0>(d_idx, d_vals, d_p, d_rinv, d_t, d_gp, nrows, d_dot, th, grid, d_flush, flush_total, d_out, nsm);
      const float sc = run<1>(d_idx, d_vals, d_p, d_rinv, d_t, d_gp, nrows, d_dot, th, grid, d_flush, flush_total, d_out, nsm);
      const float op = run<2>(d_idx, d_vals, d_p, d_rinv, d_t, d_gp, nrows, d_dot, th, grid, d_flush, flush_total, d_out, nsm);
      printf("vec=%lld threads=%d blocks/SM=%d : gather4 %.1f us | scatter4(red.add.f64) %.1f us | onepass4 %.1f us "
             "(two-pass equivalent = 2 x gather4 = %.1f us)\n",
             L, th, cfg[c][1], g * 1e3, sc * 1e3, op * 1e3, 2 * g * 1e3);
    }
  }
  return 0;
}
