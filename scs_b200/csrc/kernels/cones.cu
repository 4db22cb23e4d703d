// cones.cu -- projection onto the box / second-order / PSD rows of the cone
// product K under SCS's Moreau wrapper, on the device.
//
// Replaces reference src/cones.c: proj_box_cone :1182-1245, proj_soc :1250-1279,
// proj_semi_definite_cone :999-1067, the dispatch proj_cone :1340-1494 and the
// wrapper proj_dual_cone :1552-1596 (zero and LP rows are fused into
// admm.cu:k_cone_pre; here they are handled only by the operator-level entry
// b200_cones_proj_dual).
//
//  * SOC: "segmented norm + scale".  Small cones (q <= SOC_BIG) are batched:
//    one warp per cone, two passes (norm, scale) with the R-metric post-scaling
//    fused.  A big cone is cut into 4096-row chunks: pass 1 writes one partial
//    sum of squares per chunk, pass 2 adds the chunk partials of its cone in
//    index order (bit-reproducible, no atomics) and rescales its chunk.
//  * box: Newton on t, <= 25 steps; every step is one grid reduction whose last
//    block updates t and the stop flag in device memory; no host round trip.
//  * PSD: blocks grouped by order k; unpack (sqrt2-scaled diagonal, as the
//    reference) -> cusolverDnXsyevBatched -> X = V+ diag(lambda+) V+' as an fp64
//    shared-memory GEMM -> repack with the post-scaling fused.
#include "../common.cuh"
#include "../admm_api.h"
#include <cusolverDn.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <map>
#include <vector>

#define SOC_BIG 8192
#define SOC_CHUNK 4096
#define SOC_BATCH_ROWS 4096
#define BOX_MAX_ITERS 25
#define CT 256

struct PsdGroup {
  int k;            // matrix order
  int count;        // number of blocks
  int *d_off;       // offset of each block inside the m-vector (count)
  double *d_mats;   // count * k * k  (column-major, eigenvectors on exit)
  double *d_evals;  // count * k
  void *d_work;
  size_t work_bytes;
  void *h_work;
  size_t h_work_bytes;
  int *d_info;      // count
};

struct B200Cones {
  int m, nz, nl, bsize, qsize, ssize;
  int box_off, soc_off, psd_off;
  // box
  double *d_bl, *d_bu;
  double *d_box;  // [0]=t (warm start), [1]=gt, [2]=ht
  int *d_box_flag;  // [0]=done, [1]=iters
  double *d_part;
  unsigned int *d_cnt;
  // SOC
  int *d_q_off;        // qsize+1 prefix offsets relative to soc_off
  int n_small_items;
  int4 *d_small_items;  // (unused, unused, cone_first, ncones)
  int n_chunks;
  int4 *d_chunks;  // (big cone index, row_start rel. to soc_off, nrows, first?)
  int n_big;
  int4 *d_big;  // per big cone: (first_chunk, nchunks, off, q)
  double *d_chunk_part;
  double *d_head_a0;
  // PSD
  std::vector<PsdGroup> *groups;
  int *d_psd1_off;  // offsets of the order-1 blocks
  int n_psd1;
  cusolverDnHandle_t solver;
  cusolverDnParams_t solver_params;
  double *d_scratch;  // m
  // three-dimensional cones (kernels/cone_triples.cu): ep primal exp, ed dual exp, psize power
  int n_ep, n_ed, n_pow;
  long long tri_off;  // first row of the exponential triples
  double *d_pow;      // power cone parameters (sign = primal / dual), psize
  B200CpsdCones *cpsd;  // complex PSD blocks (kernels/cones_complex.cu), or NULL
  B200SpecCones *spec;  // nuclear / l1 / sum-of-largest cones (kernels/cones_spectral.cu), or NULL
  long long spec_rows;  // rows of the spectral cones: the last rows of the m-vector
  // sticky device flag: OR of every per-matrix `info` the batched eigen-solver has returned (reference
  // cones.c:1048-1052 propagates a failed syevr as "error in project_cones"); read by b200_cones_check
  int *d_err;
};

// OR the eigen-solver's per-matrix status words into the sticky flag (tiny; runs after every batched syevd)
__global__ void k_psd_info_or(int count, const int *__restrict__ info, int *err) {
  int bad = 0;
  for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < count; b += gridDim.x * blockDim.x)
    if (info[b] != 0) bad = 1;
  if (bad) atomicOr(err, 1);
}
extern "C" void b200_psd_info_or(int count, const int *d_info, int *d_err) {
  if (!d_err || count <= 0) return;
  k_psd_info_or<<<(count + 255) / 256 > 64 ? 64 : (count + 255) / 256, 256, 0, (cudaStream_t)b200_stream()>>>(
      count, d_info, d_err);
  b200_count_launch(1);
}

// ------------------------------------------------------------------ SOC kernels
__device__ __forceinline__ void soc_decide(double v1, double s, double &a0, double &scale) {
  // out[0] = a0 ; out[1:] = scale * x[1:]
  if (s <= v1) {
    a0 = v1;
    scale = 1.0;
  } else if (s <= -v1) {
    a0 = 0.0;
    scale = 0.0;
  } else {
    const double alpha = (s + v1) / 2.0;
    a0 = alpha;
    scale = alpha / s;
  }
}
__device__ __forceinline__ double post_scale(double xnew, const double *ry, const double *sv,
                                             long long row) {
  // x / r + s  (or x + s when r is NULL); sv NULL => plain projection output
  if (sv == nullptr) return xnew;
  return (ry != nullptr) ? xnew / ry[row] + sv[row] : xnew + sv[row];
}

__global__ void __launch_bounds__(CT)
k_soc_small(const int4 *__restrict__ items, const int *__restrict__ q_off, int soc_off,
            double *__restrict__ x, const double *sv, const double *ry) {
  const int4 it = items[blockIdx.x];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  for (int c = it.z + w; c < it.z + it.w; c += nw) {
    const int off = q_off[c], q = q_off[c + 1] - off;
    if (q <= 0) continue;
    const long long base = (long long)soc_off + off;
    if (q == 1) {
      if (lane == 0) x[base] = post_scale(fmax(x[base], 0.0), ry, sv, base);
      continue;
    }
    double acc = 0.0;
    for (int j = 1 + lane; j < q; j += 32) {
      const double xv = x[base + j];
      acc = fma(xv, xv, acc);
    }
    acc = warp_sum(acc);
    const double s = sqrt(acc);
    const double v1 = x[base];
    double a0, scale;
    soc_decide(v1, s, a0, scale);
    __syncwarp();
    for (int j = lane; j < q; j += 32) {
      const double xv = x[base + j];
      const double xn = (j == 0) ? a0 : (scale == 1.0 ? xv : (scale == 0.0 ? 0.0 : xv * scale));
      x[base + j] = post_scale(xn, ry, sv, base + j);
    }
  }
}

__global__ void __launch_bounds__(CT)
k_soc_big_partial(const int4 *__restrict__ chunks, int soc_off, const double *__restrict__ x,
                  double *__restrict__ chunk_part) {
  __shared__ double s_red[32];
  const int4 ch = chunks[blockIdx.x];
  const long long base = (long long)soc_off + ch.y;
  double acc[1] = {0.0};
  for (int j = threadIdx.x + (ch.w ? 1 : 0); j < ch.z; j += blockDim.x) {
    const double xv = x[base + j];
    acc[0] = fma(xv, xv, acc[0]);
  }
  block_sum<1>(acc, s_red);
  if (threadIdx.x == 0) chunk_part[blockIdx.x] = acc[0];
}

__global__ void __launch_bounds__(CT)
k_soc_big_apply(const int4 *__restrict__ chunks, const int4 *__restrict__ big, int soc_off,
                double *__restrict__ x, const double *__restrict__ chunk_part,
                double *__restrict__ head_a0, const double *sv, const double *ry) {
  __shared__ double s_scale;
  const int4 ch = chunks[blockIdx.x];
  const int4 bc = big[ch.x];
  if (threadIdx.x < 32) {
    // every chunk of a cone adds that cone's chunk partials in the same fixed order
    double acc = 0.0;
    for (int c = threadIdx.x; c < bc.y; c += 32) acc += chunk_part[bc.x + c];
    acc = warp_sum(acc);
    if (threadIdx.x == 0) {
      const double s = sqrt(acc);
      const double v1 = x[(long long)soc_off + bc.z];  // element 0 is not written by this kernel
      double a0, scale;
      soc_decide(v1, s, a0, scale);
      s_scale = scale;
      if (ch.w) head_a0[ch.x] = a0;  // consumed by k_soc_big_heads
    }
  }
  __syncthreads();
  const double scale = s_scale;
  const long long base = (long long)soc_off + ch.y;
  for (int j = threadIdx.x + (ch.w ? 1 : 0); j < ch.z; j += blockDim.x) {
    const double xv = x[base + j];
    const double xn = (scale == 1.0) ? xv : (scale == 0.0 ? 0.0 : xv * scale);
    x[base + j] = post_scale(xn, ry, sv, base + j);
  }
}
// element 0 of every big cone, written after all chunks have read it
__global__ void k_soc_big_heads(int n_big, const int4 *__restrict__ big, int soc_off,
                                double *__restrict__ x, const double *__restrict__ head_a0,
                                const double *sv, const double *ry) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= n_big) return;
  const long long row = (long long)soc_off + big[b].z;
  x[row] = post_scale(head_a0[b], ry, sv, row);
}

// ------------------------------------------------------------------ box kernels
__global__ void __launch_bounds__(B200_RED_THREADS)
k_box_newton(int bsize, int box_off, const double *__restrict__ x, const double *__restrict__ bl,
             const double *__restrict__ bu, const double *ry, double *box, int *flag,
             double *partials, unsigned int *counter) {
  if (flag[0]) return;
  __shared__ double s_red[64];
  const double t = box[0];
  double a[2] = {0.0, 0.0};
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < bsize - 1; j += gridDim.x * blockDim.x) {
    const long long row = (long long)box_off + 1 + j;
    const double xv = x[row];
    const double r = ry ? 1.0 / ry[row] : 1.0;
    const double u = bu[j], l = bl[j];
    if (xv > t * u) {
      a[0] += r * (t * u - xv) * u;
      a[1] += r * u * u;
    } else if (xv < t * l) {
      a[0] += r * (t * l - xv) * l;
      a[1] += r * l * l;
    }
  }
  block_sum<2>(a, s_red);
  if (grid_finish<2>(a, partials, counter, 0u, s_red)) {
    if (threadIdx.x == 0) {
      const double rho_t = ry ? 1.0 / ry[box_off] : 1.0;
      const double gt = rho_t * (t - x[box_off]) + a[0];
      const double ht = rho_t + a[1];
      const double tn = fmax(t - gt / fmax(ht, 1e-8), 0.0);
      box[0] = tn;
      flag[1] += 1;
      if (fabs(gt / fmax(ht, 1e-6)) < 1e-12 * fmax(tn, 1.0) ||
          fabs(tn - t) < 1e-11 * fmax(tn, 1.0))
        flag[0] = 1;
    }
  }
}
__global__ void k_box_apply(int bsize, int box_off, double *__restrict__ x,
                            const double *__restrict__ bl, const double *__restrict__ bu,
                            const double *sv, const double *ry, double *box) {
  const double t = (bsize == 1) ? fmax(x[box_off], 0.0) : box[0];
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < bsize; j += gridDim.x * blockDim.x) {
    const long long row = (long long)box_off + j;
    double xn;
    if (j == 0) {
      xn = t;
    } else {
      const double xv = x[row];
      const double u = bu[j - 1], l = bl[j - 1];
      xn = xv;
      if (xv > t * u) xn = t * u;
      else if (xv < t * l) xn = t * l;
    }
    x[row] = post_scale(xn, ry, sv, row);
  }
}

// ------------------------------------------------------------------ PSD kernels
// packed lower triangle, column-major: column j starts at j*k - j*(j-1)/2, holds rows j..k-1
__device__ __forceinline__ int packed_idx(int i, int j, int k) {  // i >= j
  return j * k - (j * (j - 1)) / 2 + (i - j);
}
__global__ void k_psd_unpack(int k, int count, const int *__restrict__ off,
                             const double *__restrict__ x, double *__restrict__ mats) {
  const int b = blockIdx.y;
  if (b >= count) return;
  const double *p = x + off[b];
  double *M = mats + (size_t)b * k * k;
  const double sqrt2 = sqrt(2.0);
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < k * k; e += gridDim.x * blockDim.x) {
    const int i = e % k, j = e / k;  // M[i + j*k]
    const double v = (i >= j) ? p[packed_idx(i, j, k)] : p[packed_idx(j, i, k)];
    M[e] = (i == j) ? v * sqrt2 : v;
  }
}
// X = sum_{lambda_c > 0} lambda_c v_c v_c', written as a packed lower triangle (diag / sqrt2) with post-scaling,
// on the fp64 TENSOR-CORE path: mma.sync.aligned.m8n8k4.row.col.f64 (DMMA; SASS "DMMA").
// wgmma has no fp64 kind, so this is the tensor pipe an fp64 contraction at 1e-13 parity can use on sm_90a
// (north_star: "tensor-core GEMM for the dense Z+ Z+' contraction", reference cones.c:1058-1062 dsyrk).
// CTA = 4 warps = one 32x32 output tile (ti >= tj) of one block; warp w owns the 16x16 quadrant (w >> 1, w & 1)
// = 2 x 2 mma tiles. Fragments (PTX ISA, m8n8k4 .f64): A[g][t], B[t][g], C[g][2t], C[g][2t+1] with g = lane >> 2,
// t = lane & 3. The shared tiles are padded to a row stride of 36 doubles: the 16 lanes of a half-warp then read 16
// distinct 8-byte banks. Eigenvalues arrive in ascending order (syevd): column chunks whose largest eigenvalue is
// <= 0 contribute nothing and are skipped.
//
// The spectral cones (kernels/cones_spectral.cu) run the same contraction with other weights and outputs:
//  REC_PSD     weights max(lambda, 0), packed lower triangle of V diag(w) V' (the PSD cone);
//  REC_SIGNED  weights of either sign, every column chunk contributes (sum-of-largest-eigenvalues cone);
//  REC_RECT    V of order ld = rows + cols, output the dense column-major rows x cols block
//              V[0:rows, :] diag(w) V[rows:ld, :]' (nuclear-norm cone, from the symmetric embedding); only the
//              last `cols` columns of V carry weight, so the chunk loop starts at the chunk holding column ld - cols.
#define PT 32
#define PTD 36
enum { REC_PSD = 0, REC_SIGNED = 1, REC_RECT = 2 };
template <int MODE>
__global__ void __launch_bounds__(128)
k_reconstruct_dmma(int ld, int rows, int cols, int count, const int *__restrict__ off,
                   const double *__restrict__ mats, const double *__restrict__ evals, double *__restrict__ x,
                   const double *sv, const double *ry) {
  __shared__ double sA[PT][PTD];  // V[i0+ii, c0+cc] * w_c
  __shared__ double sB[PT][PTD];  // V[bro+j0+jj, c0+cc]
  const int b = blockIdx.z;
  const int ti = blockIdx.y, tj = blockIdx.x;
  if (MODE != REC_RECT && tj > ti) return;
  const double *V = mats + (size_t)b * ld * ld;
  const double *lam = evals + (size_t)b * ld;
  const int bro = (MODE == REC_RECT) ? rows : 0;  // first row of the right factor inside V
  const int i0 = ti * PT, j0 = tj * PT;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int g = lane >> 2, t = lane & 3;
  const int wr = (w >> 1) * 16, wc = (w & 1) * 16;
  double acc[2][2][2];
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int c = 0; c < 2; ++c) acc[a][c][0] = acc[a][c][1] = 0.0;
  const int cstart = (MODE == REC_RECT) ? ((ld - cols) / PT) * PT : 0;
  for (int c0 = cstart; c0 < ld; c0 += PT) {
    if (MODE == REC_PSD) {
      const int clast = (c0 + PT - 1 < ld) ? c0 + PT - 1 : ld - 1;
      if (lam[clast] <= 0.0) continue;  // block-uniform: nothing positive in this chunk
    }
    for (int e = threadIdx.x; e < PT * PT; e += blockDim.x) {
      const int rr = e % PT, cc = e / PT;
      const int c = c0 + cc;
      double la = 0.0, va = 0.0, vb = 0.0;
      if (c < ld) {
        la = lam[c];
        if (MODE == REC_PSD) la = la > 0.0 ? la : 0.0;
        if (i0 + rr < rows) va = V[(size_t)(i0 + rr) + (size_t)c * ld];
        if (j0 + rr < cols) vb = V[(size_t)(bro + j0 + rr) + (size_t)c * ld];
      }
      sA[rr][cc] = va * la;
      sB[rr][cc] = vb;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < PT; kk += 4) {
      const double a0 = sA[wr + g][kk + t], a1 = sA[wr + 8 + g][kk + t];
      const double b0 = sB[wc + g][kk + t], b1 = sB[wc + 8 + g][kk + t];
      dmma_m8n8k4(acc[0][0][0], acc[0][0][1], a0, b0);
      dmma_m8n8k4(acc[0][1][0], acc[0][1][1], a0, b1);
      dmma_m8n8k4(acc[1][0][0], acc[1][0][1], a1, b0);
      dmma_m8n8k4(acc[1][1][0], acc[1][1][1], a1, b1);
    }
    __syncthreads();
  }
  const double inv_sqrt2 = 1.0 / sqrt(2.0);
  const long long base = off[b];
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int c = 0; c < 2; ++c)
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const int i = i0 + wr + 8 * a + g, j = j0 + wc + 8 * c + 2 * t + q;
        if (MODE == REC_RECT) {
          if (i < rows && j < cols) {
            const long long row = base + i + (long long)j * rows;
            x[row] = post_scale(acc[a][c][q], ry, sv, row);
          }
        } else if (i < rows && j < rows && i >= j) {
          const double val = (i == j) ? acc[a][c][q] * inv_sqrt2 : acc[a][c][q];
          const long long row = base + packed_idx(i, j, rows);
          x[row] = post_scale(val, ry, sv, row);
        }
      }
}
// Launchers for kernels/cones_spectral.cu (count blocks; off[b] = first row of block b's matrix)
// (blocks b0 .. b0 + nb - 1 of a sub-batch: offset pointers, the kernels index the sub-batch from 0)
extern "C" void b200_psd_unpack_launch(int k, int count, const int *d_off, const double *d_x, double *d_mats) {
  for (int b0 = 0; b0 < count; b0 += B200_EIG_BATCH) {
    const int nb = std::min(B200_EIG_BATCH, count - b0);
    dim3 ug((k * k + 255) / 256, nb);
    k_psd_unpack<<<ug, 256, 0, (cudaStream_t)b200_stream()>>>(k, nb, d_off + b0, d_x, d_mats + (size_t)b0 * k * k);
    b200_count_launch(1);
  }
}
extern "C" void b200_reconstruct_launch(int mode, int ld, int rows, int cols, int count, const int *d_off,
                                        const double *d_mats, const double *d_w, double *d_x, const double *d_s,
                                        const double *d_ry) {
  cudaStream_t st = (cudaStream_t)b200_stream();
  const int ntr = (rows + PT - 1) / PT, ntc = (cols + PT - 1) / PT;
  for (int b0 = 0; b0 < count; b0 += B200_EIG_BATCH) {
    const int nb = std::min(B200_EIG_BATCH, count - b0);
    const int *off = d_off + b0;
    const double *V = d_mats + (size_t)b0 * ld * ld, *w = d_w + (size_t)b0 * ld;
    dim3 rg(ntc, ntr, nb);
    if (mode == REC_PSD)
      k_reconstruct_dmma<REC_PSD><<<rg, 128, 0, st>>>(ld, rows, cols, nb, off, V, w, d_x, d_s, d_ry);
    else if (mode == REC_RECT)
      k_reconstruct_dmma<REC_RECT><<<rg, 128, 0, st>>>(ld, rows, cols, nb, off, V, w, d_x, d_s, d_ry);
    else
      k_reconstruct_dmma<REC_SIGNED><<<rg, 128, 0, st>>>(ld, rows, cols, nb, off, V, w, d_x, d_s, d_ry);
    b200_count_launch(1);
  }
}
extern "C" int b200_syevd_batched(void *solver, void *params, int n, double *d_mats, double *d_evals, void *d_work,
                                  size_t work_bytes, void *h_work, size_t h_work_bytes, int *d_info, int count,
                                  int *d_err, const char *what) {
  for (int b0 = 0; b0 < count; b0 += B200_EIG_BATCH) {
    const int nb = std::min(B200_EIG_BATCH, count - b0);
    const cusolverStatus_t cs = cusolverDnXsyevBatched(
        (cusolverDnHandle_t)solver, (cusolverDnParams_t)params, CUSOLVER_EIG_MODE_VECTOR, CUBLAS_FILL_MODE_LOWER, n,
        CUDA_R_64F, d_mats + (size_t)b0 * n * n, n, CUDA_R_64F, d_evals + (size_t)b0 * n, CUDA_R_64F, d_work,
        work_bytes, h_work, h_work_bytes, d_info + b0, nb);
    if (cs != CUSOLVER_STATUS_SUCCESS) {
      b200_set_error(what, cudaErrorUnknown, __FILE__, __LINE__);
      return -1;
    }
  }
  b200_psd_info_or(count, d_info, d_err);
  return 0;
}
__global__ void k_psd_order1(int count, const int *__restrict__ off, double *__restrict__ x,
                             const double *sv, const double *ry) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= count) return;
  const long long row = off[b];
  x[row] = post_scale(fmax(x[row], 0.0), ry, sv, row);
}

// ------------------------------------------------------------------ Moreau wrapper kernels (operator API)
__global__ void k_moreau_pre(int m, int nz, int nl, double *__restrict__ x, double *__restrict__ s,
                             const double *ry) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < m;
       i += (long long)gridDim.x * blockDim.x) {
    const double ui = x[i];
    s[i] = ui;
    const double r = ry ? ry[i] : 1.0;
    double out;
    if (i < nz) {
      out = ui;  // 0 / r + s
      if (ry) out = 0.0 / r + ui;
    } else if (i < (long long)nz + nl) {
      double xx = ry ? ui * -r : -ui;
      xx = fmax(xx, 0.0);
      out = ry ? xx / r + ui : xx + ui;
    } else {
      out = ry ? ui * -r : -ui;
    }
    x[i] = out;
  }
}

// ------------------------------------------------------------------ host side
// ---- cuSOLVER handle cache (per device, at most 4 parked): scs_init of a PSD problem no longer pays cusolverDnCreate
#include <mutex>
static std::mutex g_solver_mu;
static std::vector<std::pair<int, cusolverDnHandle_t>> g_solver_free;

extern "C" void *b200_solver_acquire(void) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return nullptr;
  cusolverDnHandle_t h = nullptr;
  {
    std::lock_guard<std::mutex> lk(g_solver_mu);
    for (size_t i = 0; i < g_solver_free.size(); ++i)
      if (g_solver_free[i].first == dev) {
        h = g_solver_free[i].second;
        g_solver_free.erase(g_solver_free.begin() + i);
        break;
      }
  }
  if (!h && cusolverDnCreate(&h) != CUSOLVER_STATUS_SUCCESS) return nullptr;
  if (cusolverDnSetStream(h, (cudaStream_t)b200_stream()) != CUSOLVER_STATUS_SUCCESS) {
    cusolverDnDestroy(h);
    return nullptr;
  }
  return (void *)h;
}

extern "C" void b200_solver_release(void *handle) {
  if (!handle) return;
  int dev = 0;
  if (cudaGetDevice(&dev) == cudaSuccess) {
    std::lock_guard<std::mutex> lk(g_solver_mu);
    if (g_solver_free.size() < 4) {
      g_solver_free.emplace_back(dev, (cusolverDnHandle_t)handle);
      return;
    }
  }
  cusolverDnDestroy((cusolverDnHandle_t)handle);
}

static int grid_for(long long n, int threads) {
  long long g = (n + threads - 1) / threads;
  long long cap = 8LL * b200_num_sms();
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

extern "C" B200Cones *b200_cones_create(int m, int nz, int nl, int bsize, const double *h_bl,
                                        const double *h_bu, int qsize, const int *h_q, int ssize,
                                        const int *h_s) {
  if (b200_runtime_init() != 0) return nullptr;
  B200Cones *c = (B200Cones *)calloc(1, sizeof(B200Cones));
  if (!c) return nullptr;
  c->m = m; c->nz = nz; c->nl = nl; c->bsize = bsize; c->qsize = qsize; c->ssize = ssize;
  c->box_off = nz + nl;
  c->soc_off = c->box_off + bsize;
  long long qtot = 0;
  for (int i = 0; i < qsize; ++i) qtot += h_q[i];
  c->psd_off = c->soc_off + (int)qtot;
  c->groups = new std::vector<PsdGroup>();
  int rc = 0;
  c->d_part = (double *)b200_malloc(8 * 2048 * 8);
  c->d_cnt = (unsigned int *)b200_malloc(64);
  c->d_scratch = (double *)b200_malloc((size_t)(m > 0 ? m : 1) * 8);
  if (!c->d_part || !c->d_cnt || !c->d_scratch) { b200_cones_destroy(c); return nullptr; }
  rc |= b200_memset0(c->d_cnt, 64);

  // ---- box
  if (bsize > 0) {
    c->d_box = (double *)b200_malloc(8 * 8);
    c->d_box_flag = (int *)b200_malloc(8 * 4);
    const int nb = bsize > 1 ? bsize - 1 : 1;
    c->d_bl = (double *)b200_malloc((size_t)nb * 8);
    c->d_bu = (double *)b200_malloc((size_t)nb * 8);
    if (!c->d_box || !c->d_box_flag || !c->d_bl || !c->d_bu) { b200_cones_destroy(c); return nullptr; }
    double init[8] = {1.0, 0, 0, 0, 0, 0, 0, 0};  // box_t_warm_start = 1 (cones.c:1562)
    rc |= b200_h2d(c->d_box, init, sizeof(init));
    rc |= b200_memset0(c->d_box_flag, 32);
    if (bsize > 1) {
      rc |= b200_h2d(c->d_bl, h_bl, (size_t)(bsize - 1) * 8);
      rc |= b200_h2d(c->d_bu, h_bu, (size_t)(bsize - 1) * 8);
    }
  }
  // ---- SOC tables
  if (qsize > 0) {
    std::vector<int> qoff(qsize + 1, 0);
    for (int i = 0; i < qsize; ++i) qoff[i + 1] = qoff[i] + h_q[i];
    std::vector<int4> items, chunks, big;
    int i = 0;
    while (i < qsize) {
      if (h_q[i] > SOC_BIG) {
        int4 bc;
        bc.x = (int)chunks.size();
        bc.z = qoff[i];
        bc.w = h_q[i];
        int done = 0, nch = 0;
        while (done < h_q[i]) {
          int len = std::min(SOC_CHUNK, h_q[i] - done);
          int4 ch;
          ch.x = (int)big.size();
          ch.y = qoff[i] + done;
          ch.z = len;
          ch.w = (done == 0) ? 1 : 0;
          chunks.push_back(ch);
          done += len;
          ++nch;
        }
        bc.y = nch;
        big.push_back(bc);
        ++i;
      } else {
        int first = i, rows = 0;
        while (i < qsize && h_q[i] <= SOC_BIG && (rows == 0 || rows + h_q[i] <= SOC_BATCH_ROWS) &&
               (i - first) < 4096) {
          rows += h_q[i];
          ++i;
        }
        int4 it;
        it.x = qoff[first]; it.y = rows; it.z = first; it.w = i - first;
        items.push_back(it);
      }
    }
    c->n_small_items = (int)items.size();
    c->n_chunks = (int)chunks.size();
    c->n_big = (int)big.size();
    c->d_q_off = (int *)b200_malloc((size_t)(qsize + 1) * 4);
    c->d_small_items = (int4 *)b200_malloc((items.size() + 1) * sizeof(int4));
    c->d_chunks = (int4 *)b200_malloc((chunks.size() + 1) * sizeof(int4));
    c->d_big = (int4 *)b200_malloc((big.size() + 1) * sizeof(int4));
    c->d_chunk_part = (double *)b200_malloc((chunks.size() + 1) * 8);
    c->d_head_a0 = (double *)b200_malloc((big.size() + 1) * 8);
    if (!c->d_q_off || !c->d_small_items || !c->d_chunks || !c->d_big || !c->d_chunk_part || !c->d_head_a0) {
      b200_cones_destroy(c);
      return nullptr;
    }
    rc |= b200_h2d(c->d_q_off, qoff.data(), (size_t)(qsize + 1) * 4);
    if (!items.empty()) rc |= b200_h2d(c->d_small_items, items.data(), items.size() * sizeof(int4));
    if (!chunks.empty()) rc |= b200_h2d(c->d_chunks, chunks.data(), chunks.size() * sizeof(int4));
    if (!big.empty()) rc |= b200_h2d(c->d_big, big.data(), big.size() * sizeof(int4));
    rc |= b200_sync();
  }
  // ---- PSD groups
  if (ssize > 0) {
    std::map<int, std::vector<int>> by_k;
    long long off = c->psd_off;
    for (int i = 0; i < ssize; ++i) {
      const int k = h_s[i];
      if (k > 0) by_k[k].push_back((int)off);
      off += (long long)k * (k + 1) / 2;
    }
    c->solver = (cusolverDnHandle_t)b200_solver_acquire();
    if (!c->solver || cusolverDnCreateParams(&c->solver_params) != CUSOLVER_STATUS_SUCCESS) {
      b200_cones_destroy(c);
      return nullptr;
    }
    c->d_err = (int *)b200_malloc(64);
    if (!c->d_err || b200_memset0(c->d_err, 64) != 0) { b200_cones_destroy(c); return nullptr; }
    for (auto &kv : by_k) {
      const int k = kv.first;
      const int count = (int)kv.second.size();
      if (k == 1) {
        c->n_psd1 = count;
        c->d_psd1_off = (int *)b200_malloc((size_t)count * 4);
        if (!c->d_psd1_off) { b200_cones_destroy(c); return nullptr; }
        rc |= b200_h2d(c->d_psd1_off, kv.second.data(), (size_t)count * 4);
        rc |= b200_sync();
        continue;
      }
      PsdGroup g;
      memset(&g, 0, sizeof(g));
      g.k = k; g.count = count;
      g.d_off = (int *)b200_malloc((size_t)count * 4);
      g.d_mats = (double *)b200_malloc((size_t)count * k * k * 8);
      g.d_evals = (double *)b200_malloc((size_t)count * k * 8);
      g.d_info = (int *)b200_malloc((size_t)count * 4);
      auto drop_group = [&]() {
        b200_free(g.d_off); b200_free(g.d_mats); b200_free(g.d_evals); b200_free(g.d_info);
        b200_free(g.d_work); free(g.h_work);
        b200_cones_destroy(c);
      };
      if (!g.d_off || !g.d_mats || !g.d_evals || !g.d_info) { drop_group(); return nullptr; }
      rc |= b200_h2d(g.d_off, kv.second.data(), (size_t)count * 4);
      rc |= b200_sync();
      size_t wd = 0, wh = 0;
      const cusolverStatus_t bs = cusolverDnXsyevBatched_bufferSize(
          c->solver, c->solver_params, CUSOLVER_EIG_MODE_VECTOR, CUBLAS_FILL_MODE_LOWER, k, CUDA_R_64F, g.d_mats, k,
          CUDA_R_64F, g.d_evals, CUDA_R_64F, &wd, &wh, std::min(count, B200_EIG_BATCH));
      if (bs != CUSOLVER_STATUS_SUCCESS) {
        char what[112];
        snprintf(what, sizeof(what), "cusolverDnXsyevBatched_bufferSize (order %d, %d blocks): status %d", k,
                 std::min(count, B200_EIG_BATCH), (int)bs);
        b200_set_error(what, cudaErrorUnknown, __FILE__, __LINE__);
        drop_group();
        return nullptr;
      }
      g.work_bytes = wd;
      g.h_work_bytes = wh;
      g.d_work = b200_malloc(wd ? wd : 16);
      g.h_work = wh ? malloc(wh) : nullptr;
      if (!g.d_work || (wh && !g.h_work)) { drop_group(); return nullptr; }
      c->groups->push_back(g);
    }
  }
  if (rc != 0 || b200_sync() != 0) { b200_cones_destroy(c); return nullptr; }
  return c;
}

// new (already scaled) box bounds, and the Newton warm start back to t = 1: the box state of b200_cones_create
extern "C" int b200_cones_set_box(B200Cones *c, const double *h_bl, const double *h_bu) {
  if (c->bsize <= 0) return 0;
  const double init[8] = {1.0, 0, 0, 0, 0, 0, 0, 0};
  int rc = b200_h2d(c->d_box, init, sizeof(init)) | b200_memset0(c->d_box_flag, 32);
  if (c->bsize > 1) {
    rc |= b200_h2d(c->d_bl, h_bl, (size_t)(c->bsize - 1) * 8);
    rc |= b200_h2d(c->d_bu, h_bu, (size_t)(c->bsize - 1) * 8);
  }
  return rc != 0 || b200_sync() != 0 ? -1 : 0;
}

extern "C" void b200_cones_destroy(B200Cones *c) {
  if (!c) return;
  b200_sync();
  b200_free(c->d_bl); b200_free(c->d_bu); b200_free(c->d_box); b200_free(c->d_box_flag);
  b200_free(c->d_part); b200_free(c->d_cnt);
  b200_free(c->d_q_off); b200_free(c->d_small_items); b200_free(c->d_chunks);
  b200_free(c->d_big); b200_free(c->d_chunk_part); b200_free(c->d_head_a0); b200_free(c->d_psd1_off);
  b200_free(c->d_scratch);
  b200_free(c->d_pow);
  b200_free(c->d_err);
  b200_cpsd_destroy(c->cpsd);
  b200_spec_destroy(c->spec);
  if (c->groups) {
    for (auto &g : *c->groups) {
      b200_free(g.d_off); b200_free(g.d_mats); b200_free(g.d_evals); b200_free(g.d_info);
      b200_free(g.d_work); free(g.h_work);
    }
    delete c->groups;
  }
  if (c->solver_params) cusolverDnDestroyParams(c->solver_params);
  b200_solver_release((void *)c->solver);
  free(c);
}

extern "C" double *b200_cones_scratch(B200Cones *c) { return c->d_scratch; }

// log-det, nuclear-norm, l1-norm and sum-of-largest-eigenvalues cones occupy the last rows, in that order (reference
// cones.c:1446-1490). Called before b200_cones_set_triples / _set_complex_psd, whose rows sit just before them.
extern "C" int b200_cones_set_spectral(B200Cones *c, int dsize, const int *h_d, int nucsize, const int *h_nuc_m,
                                       const int *h_nuc_n, int ell1_size, const int *h_ell1, int sl_size,
                                       const int *h_sl_n, const int *h_sl_k) {
  long long rows = 0;
  for (int i = 0; i < dsize; ++i) rows += 2 + (long long)h_d[i] * (h_d[i] + 1) / 2;
  for (int i = 0; i < nucsize; ++i) rows += 1 + (long long)h_nuc_m[i] * h_nuc_n[i];
  for (int i = 0; i < ell1_size; ++i) rows += 1 + (long long)h_ell1[i];
  for (int i = 0; i < sl_size; ++i) rows += 1 + (long long)h_sl_n[i] * (h_sl_n[i] + 1) / 2;
  if (rows == 0) return 0;
  if (rows > c->m) return -1;
  if (!c->d_err) {
    c->d_err = (int *)b200_malloc(64);
    if (!c->d_err || b200_memset0(c->d_err, 64) != 0) return -1;
  }
  c->spec_rows = rows;
  c->spec = b200_spec_create(dsize, h_d, nucsize, h_nuc_m, h_nuc_n, ell1_size, h_ell1, sl_size, h_sl_n, h_sl_k,
                             (long long)c->m - rows, c->d_err);
  return c->spec ? 0 : -1;
}

extern "C" int b200_cones_reset_spectral(B200Cones *c) { return c->spec ? b200_spec_reset(c->spec) : 0; }

extern "C" int b200_cones_logdet_stats(B200Cones *c, int *iter, int *newton_success, double res[3]) {
  return c->spec ? b200_spec_logdet_stats(c->spec, iter, newton_success, res) : -1;
}

// exponential / power cones occupy the 3 (ep + ed + psize) rows before the spectral cones, i.e. the LAST rows when
// there are none (scs.h cone order)
extern "C" int b200_cones_set_triples(B200Cones *c, int ep, int ed, int psize, const double *h_p) {
  c->n_ep = ep; c->n_ed = ed; c->n_pow = psize;
  c->tri_off = (long long)c->m - c->spec_rows - 3LL * ((long long)ep + ed + psize);
  if (c->tri_off < 0) return -1;
  if (psize > 0) {
    c->d_pow = (double *)b200_malloc((size_t)psize * 8);
    if (!c->d_pow || b200_h2d(c->d_pow, h_p, (size_t)psize * 8) != 0 || b200_sync() != 0) return -1;
  }
  return 0;
}

// complex PSD blocks sit between the real PSD blocks and the exponential triples (scs.h cone order)
extern "C" int b200_cones_set_complex_psd(B200Cones *c, int cssize, const int *h_cs, int n_triples) {
  long long rows = 0;
  for (int i = 0; i < cssize; ++i) rows += (long long)h_cs[i] * h_cs[i];
  if (rows == 0) return 0;
  const long long first = (long long)c->m - c->spec_rows - 3LL * n_triples - rows;
  if (first < 0) return -1;
  if (!c->d_err) {
    c->d_err = (int *)b200_malloc(64);
    if (!c->d_err || b200_memset0(c->d_err, 64) != 0) return -1;
  }
  c->cpsd = b200_cpsd_create(cssize, h_cs, first);
  if (c->cpsd) b200_cpsd_set_err(c->cpsd, c->d_err);
  return c->cpsd ? 0 : -1;
}

extern "C" int b200_cones_project_rest(B200Cones *c, double *d_x, const double *d_s,
                                       const double *d_ry) {
  cudaStream_t st = (cudaStream_t)b200_stream();
  // ---- box
  if (c->bsize > 0) {
    if (c->bsize > 1) {
      CUDA_OK(cudaMemsetAsync(c->d_box_flag, 0, 8, st));
      const int g = grid_for(c->bsize - 1, B200_RED_THREADS * 4);
      for (int it = 0; it < BOX_MAX_ITERS; ++it)
        k_box_newton<<<g, B200_RED_THREADS, 0, st>>>(c->bsize, c->box_off, d_x, c->d_bl, c->d_bu,
                                                     d_ry, c->d_box, c->d_box_flag, c->d_part,
                                                     c->d_cnt);
      b200_count_launch(BOX_MAX_ITERS);
    }
    k_box_apply<<<grid_for(c->bsize, 256), 256, 0, st>>>(c->bsize, c->box_off, d_x, c->d_bl, c->d_bu,
                                                          d_s, d_ry, c->d_box);
    b200_count_launch(1);
  }
  // ---- SOC
  if (c->n_small_items > 0) {
    k_soc_small<<<c->n_small_items, CT, 0, st>>>(c->d_small_items, c->d_q_off, c->soc_off, d_x, d_s,
                                                 d_ry);
    b200_count_launch(1);
  }
  if (c->n_chunks > 0) {
    k_soc_big_partial<<<c->n_chunks, CT, 0, st>>>(c->d_chunks, c->soc_off, d_x, c->d_chunk_part);
    k_soc_big_apply<<<c->n_chunks, CT, 0, st>>>(c->d_chunks, c->d_big, c->soc_off, d_x,
                                                c->d_chunk_part, c->d_head_a0, d_s, d_ry);
    k_soc_big_heads<<<(c->n_big + 63) / 64, 64, 0, st>>>(c->n_big, c->d_big, c->soc_off, d_x,
                                                        c->d_head_a0, d_s, d_ry);
    b200_count_launch(3);
  }
  // ---- PSD
  if (c->n_psd1 > 0) {
    k_psd_order1<<<(c->n_psd1 + 127) / 128, 128, 0, st>>>(c->n_psd1, c->d_psd1_off, d_x, d_s, d_ry);
    b200_count_launch(1);
  }
  if (c->groups) {
    for (auto &g : *c->groups) {
      const int k = g.k;
      b200_psd_unpack_launch(k, g.count, g.d_off, d_x, g.d_mats);
      if (b200_syevd_batched(c->solver, c->solver_params, k, g.d_mats, g.d_evals, g.d_work, g.work_bytes, g.h_work,
                             g.h_work_bytes, g.d_info, g.count, c->d_err, "cusolverDnXsyevBatched") != 0)
        return -1;
      b200_reconstruct_launch(REC_PSD, k, k, k, g.count, g.d_off, g.d_mats, g.d_evals, d_x, d_s, d_ry);
    }
  }
  // ---- complex PSD
  if (c->cpsd && b200_cpsd_project(c->cpsd, d_x, d_s, d_ry) != 0) return -1;
  // ---- exponential / power triples
  if (c->n_ep + c->n_ed + c->n_pow > 0) {
    if (b200_cone_triples_project(c->n_ep, c->n_ed, c->n_pow, c->tri_off, c->d_pow, d_x, d_s, d_ry) != 0)
      return -1;
  }
  // ---- nuclear / l1 / sum-of-largest
  if (c->spec && b200_spec_project(c->spec, d_x, d_s, d_ry) != 0) return -1;
  CUDA_OK(cudaGetLastError());
  return 0;
}

// 0: every eigen-decomposition so far reported success; -1: at least one did not (sticky). Syncs the stream.
extern "C" int b200_cones_check(B200Cones *c) {
  if (!c || !c->d_err) return 0;
  int h = 0;
  if (b200_d2h(&h, c->d_err, sizeof(int)) != 0 || b200_sync() != 0) return -1;
  if (h & 2) {  // LD_ERR_BIT of kernels/cones_spectral.cu
    b200_set_error("log-det cone projection failed: Newton and both interior-point variants missed the tolerances",
                   cudaErrorUnknown, __FILE__, __LINE__);
    return -1;
  }
  if (h != 0) {
    b200_set_error("batched syevd reported a failure (info != 0) in a PSD or spectral cone projection",
                   cudaErrorUnknown, __FILE__, __LINE__);
    return -1;
  }
  return 0;
}

extern "C" int b200_cones_proj_dual(B200Cones *c, double *d_x, const double *d_ry) {
  cudaStream_t st = (cudaStream_t)b200_stream();
  if (c->m <= 0) return 0;
  k_moreau_pre<<<grid_for(c->m, 256), 256, 0, st>>>(c->m, c->nz, c->nl, d_x, c->d_scratch, d_ry);
  b200_count_launch(1);
  CUDA_OK(cudaGetLastError());
  return b200_cones_project_rest(c, d_x, c->d_scratch, d_ry);
}
