// cones_complex.cu -- projection onto the complex (Hermitian) PSD cone, batched by order.
//
// Replaces reference src/cones.c:1072-1156 (proj_complex_semi_definite_cone: zheevr + zherk per block).
// Operator parity vs the reference's zheevr projection <= 5e-13 (tests/test_zz_reference_fixtures_gpu.py); enabled by
// default. The index arithmetic is also checked on the CPU against the reference
// (numpy restatement in tests/test_complex_psd_cpu.py, <= 3e-14).
//
// Vectorisation (docs/src/api/cones.rst, cones.c:1095-1103): a block of order k occupies k^2 doubles;
// column j of the lower triangle starts at j (2k - j): the real diagonal entry, then (re, im) pairs of
// rows j+1 .. k-1; off-diagonals carry the factor sqrt(2) (the code scales the diagonal by sqrt(2) before
// the eigen-decomposition and by 1/sqrt(2) after it, which is the same thing up to a global factor).
//
// Method: the real embedding. For H = A + iB (A symmetric, B antisymmetric) the real symmetric matrix
// M = [[A, -B], [B, A]] of order 2k has the eigenvalues of H twice, and the embedding commutes with the
// spectral projection: Pi_PSD(M) = [[A+, -B+], [B+, A+]] with H+ = A+ + iB+. So the block is unpacked
// into M, decomposed with the same batched cuSOLVER syevd the real cone uses (the north star names
// cuSOLVER for the eigen-decomposition), reconstructed as V+ diag(lambda+) V+' with an fp64 tiled GEMM,
// and A+ (top-left) and B+ (bottom-left) are packed back with the Moreau post-scaling fused.
#include "../common.cuh"
#include "../admm_api.h"
#include "../eigen.cuh"
#include <map>
#include <math.h>
#include <vector>

namespace {

// (re, im) of the sqrt(2)-scaled Hermitian matrix at (i, j), i >= j, from the packed block p
__device__ __forceinline__ void packed_entry(const double *p, int kc, int i, int j, double &re, double &im) {
  const int base = j * (2 * kc - j);
  if (i == j) {
    re = p[base] * 1.4142135623730951;  // sqrt(2)
    im = 0.0;
  } else {
    re = p[base + 1 + 2 * (i - j - 1)];
    im = p[base + 2 + 2 * (i - j - 1)];
  }
}

__global__ void k_cpsd_unpack(int kc, int count, const int *__restrict__ off, const double *__restrict__ x,
                              double *__restrict__ mats) {
  const int b = blockIdx.y;
  if (b >= count) return;
  const int K = 2 * kc;
  const double *p = x + off[b];
  double *M = mats + (size_t)b * K * K;
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < K * K; e += gridDim.x * blockDim.x) {
    const int I = e % K, J = e / K;  // M[I + J*K]
    const int i = I % kc, j = J % kc, bi = I / kc, bj = J / kc;
    double re, im;
    if (i >= j) {
      packed_entry(p, kc, i, j, re, im);
    } else {  // H(i,j) = conj(H(j,i))
      packed_entry(p, kc, j, i, re, im);
      im = -im;
    }
    // blocks: (0,0) = (1,1) = A ; (1,0) = B ; (0,1) = -B
    M[e] = (bi == bj) ? re : (bi == 1 ? im : -im);
  }
}

// X = sum_{lambda_c > 0} lambda_c v_c v_c' on 32x32 tiles of the lower triangle of the embedding; the
// top-left block gives Re(H+), the bottom-left block Im(H+); diag / sqrt(2); post-scaling fused.
#define CPT 32
__global__ void __launch_bounds__(CPT * 8)
k_cpsd_reconstruct(int kc, int count, const int *__restrict__ off, const double *__restrict__ mats,
                   const double *__restrict__ evals, double *__restrict__ x, const double *sv,
                   const double *ry) {
  __shared__ double sA[CPT][CPT + 1];
  __shared__ double sB[CPT][CPT + 1];
  const int K = 2 * kc;
  const int b = blockIdx.z;
  const int ti = blockIdx.y, tj = blockIdx.x;
  if (tj > ti) return;
  if (tj * CPT >= kc) return;  // columns J >= kc: the bottom-right copy of A+, not needed
  const double *V = mats + (size_t)b * K * K;
  const double *lam = evals + (size_t)b * K;
  const int i0 = ti * CPT, j0 = tj * CPT;
  const int tx = threadIdx.x % CPT, ty = threadIdx.x / CPT;  // ty in 0..7, 4 rows per thread
  double acc[4] = {0, 0, 0, 0};
  for (int c0 = 0; c0 < K; c0 += CPT) {
    for (int e = threadIdx.x; e < CPT * CPT; e += blockDim.x) {
      const int rr = e % CPT, cc = e / CPT;
      const int c = c0 + cc;
      double la = 0.0, va = 0.0, vb = 0.0;
      if (c < K) {
        la = lam[c];
        la = la > 0.0 ? la : 0.0;
        if (i0 + rr < K) va = V[(size_t)(i0 + rr) + (size_t)c * K];
        if (j0 + rr < K) vb = V[(size_t)(j0 + rr) + (size_t)c * K];
      }
      sA[rr][cc] = va * la;
      sB[rr][cc] = vb;
    }
    __syncthreads();
#pragma unroll 8
    for (int cc = 0; cc < CPT; ++cc) {
      const double bj = sB[tx][cc];
#pragma unroll
      for (int r = 0; r < 4; ++r) acc[r] = fma(sA[ty * 4 + r][cc], bj, acc[r]);
    }
    __syncthreads();
  }
  const long long base = off[b];
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int I = i0 + ty * 4 + r, J = j0 + tx;
    if (I >= K || J >= kc || I < J) continue;
    const long long col = base + (long long)J * (2 * kc - J);
    if (I < kc) {  // real part of H+(I, J)
      if (I == J) {
        x[col] = moreau_post(acc[r] * 0.7071067811865476, ry, sv, col);
      } else {
        const long long row = col + 1 + 2 * (I - J - 1);
        x[row] = moreau_post(acc[r], ry, sv, row);
      }
    } else {  // imaginary part of H+(I - kc, J), strictly lower triangle only
      const int i = I - kc;
      if (i > J) {
        const long long row = col + 2 + 2 * (i - J - 1);
        x[row] = moreau_post(acc[r], ry, sv, row);
      }
    }
  }
}

}  // namespace

struct B200CpsdCones {
  std::vector<B200EigGroup> groups;  // one per complex order kc, of embedding order N = 2 kc
  B200Eig *eig;                      // owned by B200Cones (kernels/cones.cu)
};

extern "C" void b200_cpsd_destroy(B200CpsdCones *c) {
  if (!c) return;
  b200_sync();
  for (auto &g : c->groups) eig_group_free(g);
  delete c;
}

// h_cs: complex PSD orders; first_row: row of the first complex block inside the m-vector
extern "C" B200CpsdCones *b200_cpsd_create(int cssize, const int *h_cs, long long first_row, B200Eig *eig) {
  if (b200_runtime_init() != 0) return nullptr;
  B200CpsdCones *c = new B200CpsdCones();
  c->eig = eig;
  std::map<int, std::vector<int>> by_k;
  long long off = first_row;
  for (int i = 0; i < cssize; ++i) {
    if (h_cs[i] > 0) by_k[h_cs[i]].push_back((int)off);
    off += (long long)h_cs[i] * h_cs[i];
  }
  for (auto &kv : by_k) {
    c->groups.push_back(B200EigGroup());  // pushed first so that destroy releases what was allocated
    if (eig_group_add(eig, c->groups.back(), 2 * kv.first, kv.second) != 0) {
      b200_cpsd_destroy(c);
      return nullptr;
    }
  }
  return c;
}

// d_x rows of the complex blocks hold -R x on entry and Pi(.) / R + s on exit (Moreau wrapper, cones.c:1583)
extern "C" int b200_cpsd_project(B200CpsdCones *c, double *d_x, const double *d_s, const double *d_ry) {
  cudaStream_t st = (cudaStream_t)b200_stream();
  for (auto &g : c->groups) {
    const int K = g.N, kc = K / 2;
    const size_t KK = (size_t)K * K;
    eig_sub_batches(g.count, [&](int b0, int nb) {
      dim3 ug((K * K + 255) / 256, nb);
      k_cpsd_unpack<<<ug, 256, 0, st>>>(kc, nb, g.d_off + b0, d_x, g.d_mats + b0 * KK);
      b200_count_launch(1);
    });
    if (eig_syevd(c->eig, g, "cusolverDnXsyevBatched (complex PSD embedding)") != 0) return -1;
    const int nt = (K + CPT - 1) / CPT;
    eig_sub_batches(g.count, [&](int b0, int nb) {
      dim3 rg(nt, nt, nb);
      k_cpsd_reconstruct<<<rg, CPT * 8, 0, st>>>(kc, nb, g.d_off + b0, g.d_mats + b0 * KK,
                                                 g.d_evals + (size_t)b0 * K, d_x, d_s, d_ry);
      b200_count_launch(1);
    });
  }
  CUDA_OK(cudaGetLastError());
  return 0;
}
