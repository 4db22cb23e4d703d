// eigen.cuh -- the batched eigensolver of the eigen-decomposition cones: real PSD (kernels/cones.cu), complex PSD
// (kernels/cones_complex.cu), log-det, nuclear norm and sum of largest eigenvalues (kernels/cones_spectral.cu).
// Host-side C++ included by those three files only; the C host layer sees none of it.
#pragma once
#include <cusolverDn.h>
#include <stddef.h>
#include <algorithm>
#include <vector>

/* Every launcher of the eigen-decomposition cones, and every batched eigensolver call, covers a group of one order in
 * sub-batches of at most B200_EIG_BATCH blocks, and the eigensolver workspace is sized for min(count, B200_EIG_BATCH).
 * The per-block kernels take the block index from gridDim.y or gridDim.z, which stop at 65535; and
 * cusolverDnXsyevBatched asks for about 0.5 MB of workspace per matrix whatever its order (measured on an H100 with
 * cuSOLVER 11.7.5: 35 GB for 65535 matrices of order 2), while cuSOLVER 11.7.3 (CUDA 12.8, the build PyTorch wheels
 * bundle) refuses the workspace query from 32767 matrices on (16384 pass). 4096 keeps the workspace near 2 GB. */
#define B200_EIG_BATCH 4096

// f(b0, nb) for the sub-batches [b0, b0 + nb) of a group of count blocks, in order
template <typename F>
inline void eig_sub_batches(int count, F f) {
  for (int b0 = 0; b0 < count; b0 += B200_EIG_BATCH) f(b0, std::min(B200_EIG_BATCH, count - b0));
}

// One eigensolver context per cone workspace (B200Cones), shared by every group of every family. The groups are
// decomposed one after another on the library stream, so one workspace of the largest queried size serves them all.
// All zero until the first group is added; freed by eig_destroy.
struct B200Eig {
  cusolverDnHandle_t solver;
  cusolverDnParams_t params;
  void *d_work, *h_work;
  size_t d_work_bytes, h_work_bytes;  // allocated: the largest query of any group
  int *d_info;                        // one status word per matrix of the largest group
  int info_count;
  // sticky device flag: OR of every status word the eigensolver has returned (reference cones.c:1048-1052 propagates
  // a failed syevr as "error in project_cones"), and LD_ERR_BIT of kernels/cones_spectral.cu; read by b200_cones_check
  int *d_err;
};

// the blocks of one order N of one family
struct B200EigGroup {
  int N, count;
  int *d_off;       // first row of each block's matrix in the m-vector
  double *d_mats;   // count * N * N, column-major; eigenvectors on exit
  double *d_evals;  // count * N, ascending
  size_t work_bytes, h_work_bytes;  // this group's own workspace query: every eigensolver call on it passes these
};

// Allocates g for the blocks whose matrices start at rows offs, of order N, creating the context on first use. For
// N > 1, queries the workspace of min(count, B200_EIG_BATCH) matrices and grows the context's to fit (order-1 groups
// need no eigensolver). 0, or -1 (a failed query is recorded); g is then safe to pass to eig_group_free.
int eig_group_add(B200Eig *e, B200EigGroup &g, int N, const std::vector<int> &offs);
void eig_group_free(B200EigGroup &g);
void eig_destroy(B200Eig *e);
// cusolverDnXsyevBatched (eigenvectors, lower triangle) on every matrix of g, sub-batch by sub-batch, then the status
// words ORed into e->d_err. 0, or -1 with the error recorded as `what`.
int eig_syevd(B200Eig *e, const B200EigGroup &g, const char *what);

extern "C" {
/* shared with kernels/cones_spectral.cu (kernels/cones.cu): the sqrt2-scaled unpack of packed lower triangles, and
 * the DMMA contraction V diag(w) V' with weights max(w, 0) (mode 0, packed lower output; w ascending), signed weights
 * (mode 1, packed lower output) or its rectangular block (mode 2, dense rows x cols output from V of order
 * ld = rows + cols) */
void b200_psd_unpack_launch(int k, int count, const int *d_off, const double *d_x, double *d_mats);
void b200_reconstruct_launch(int mode, int ld, int rows, int cols, int count, const int *d_off, const double *d_mats,
                             const double *d_w, double *d_x, const double *d_s, const double *d_ry);

/* complex PSD blocks (kernels/cones_complex.cu; reference cones.c:1072-1156) */
typedef struct B200CpsdCones B200CpsdCones;
B200CpsdCones *b200_cpsd_create(int cssize, const int *h_cs, long long first_row, B200Eig *eig);
int b200_cpsd_project(B200CpsdCones *c, double *d_x, const double *d_s, const double *d_ry);
void b200_cpsd_destroy(B200CpsdCones *c);

/* log-det, nuclear-norm, l1-norm and sum-of-largest-eigenvalues cones (kernels/cones_spectral.cu) */
typedef struct B200SpecCones B200SpecCones;
B200SpecCones *b200_spec_create(int dsize, const int *h_d, int nucsize, const int *h_nuc_m, const int *h_nuc_n,
                                int ell1_size, const int *h_ell1, int sl_size, const int *h_sl_n, const int *h_sl_k,
                                long long first_row, B200Eig *eig);
int b200_spec_project(B200SpecCones *c, double *d_x, const double *d_s, const double *d_ry);
int b200_spec_reset(B200SpecCones *c);
int b200_spec_logdet_stats(B200SpecCones *c, int *iter, int *newton_success, double res[3]);
void b200_spec_destroy(B200SpecCones *c);
}
