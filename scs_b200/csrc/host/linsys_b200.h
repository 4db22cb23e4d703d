/* linsys_b200.h -- private definition of struct SCS_LIN_SYS_WORK for this
 * backend (the reference keeps one such private.h per backend, e.g.
 * linsys/cpu/indirect/private.h:16-31). */
#ifndef LINSYS_B200_H
#define LINSYS_B200_H
#include "../../../include/scs_b200.h"
#include "../dev_api.h"
#include "../admm_api.h"

struct SCS_LIN_SYS_WORK {
  int n, m;
  long long nnz;
  B200Spmv *A;      /* CSR of A  (rows of A; built by transposing the CSC input) */
  B200Spmv *At;     /* CSR of A' (= the CSC arrays of A as given) */
  B200Spmv *P;      /* full symmetric P in CSR, or NULL */
  double *d_Pdiag;  /* diag(P) (n) or NULL */
  double *d_diag_r; /* device copy of [R_x; R_y] (n+m+1) */
  double *d_b;      /* staging for the host-pointer plugin call (n+m) */
  double *d_s;      /* staging for the warm start (n) */
  B200Cg cg;
  /* row-sharded mode: this rank owns rows [row0, row0+mloc); offsets has nranks+1 entries */
  int nranks, rank, row0, mloc;
  /* m-space-reordered pair for the CG operator (single GPU, flagged-stream operators; else NULL): A_cg = the
   * non-empty rows of A by smallest column index, each with A's lane split, At_cg = view of At with renumbered
   * columns, d_ry_cg = R_y in that order */
  B200Spmv *A_cg, *At_cg;
  double *d_ry_cg;
  int *d_perm, *d_inv;
  int p_in_exchange; /* cg.d_p points into the peer-mapped exchange allocation (sharded-x mode): not ours to free */
  int *offsets;
  int last_cg_its;
  long long tot_cg_its;
  long long n_solves;
};

/* device-pointer variants used by the ADMM driver */
int b200_linsys_solve_dev(ScsLinSysWork *w, double *d_b, const double *d_s, double tol,
                          const double *d_tol);
int b200_linsys_update_diag_r_dev(ScsLinSysWork *w, const double *d_diag_r);
int b200_linsys_full_equilibrate(const ScsMatrix *A, const int *bnd, int nbnd, double *d_D, double *d_E);
int b200_linsys_scale_local(ScsLinSysWork *w, const double *d_D, const double *d_E);
/* contiguous row blocks balanced by nonzeros; offsets[nranks+1] (also exported for the tests) */
void b200_row_partition(int m, int n, const scs_int *Ap, const scs_int *Ai, int nranks, int *offsets);
/* the limits of the operators checked in scs_int width (host/abi.c): dimensions below 2^30, nnz(A) and nnz(P) at most
 * B200_MAX_STORED; prints a message naming the limit and returns nonzero when one is exceeded */
int b200_over_dim(const char *what, long long index, scs_int v);
int b200_over_stored(const char *what, scs_int v);
int b200_matrix_over_limits(const ScsMatrix *A, const ScsMatrix *P);

#endif
