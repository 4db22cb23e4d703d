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
  int last_cg_its; /* the last solve of either kind */
  /* the first CG batch of a solve is sized from the last solve of its kind: warm-started (ADMM, d_s != NULL) solves
   * take a few dozen iterations, the cold tolerance-1e-12 solves of g a thousand or more */
  int last_admm_its, last_g_its;
  long long tot_cg_its;
  long long n_solves;
  /* the execution context: the parent ScsWork's when created inside scs_init (own_ctx = 0), else its own */
  B200Ctx *ctx;
  int own_ctx;
};

/* device-pointer variants used by the ADMM driver */
int b200_linsys_solve_dev(ScsLinSysWork *w, double *d_b, const double *d_s, double tol,
                          const double *d_tol);
int b200_linsys_update_diag_r_dev(ScsLinSysWork *w, const double *d_diag_r);
ScsLinSysWork *b200_linsys_from_ops(int m, int n, B200Spmv *A, B200Spmv *At, B200Spmv *P, double *d_Pdiag,
                                    const scs_float *diag_r);
/* one upload of a host CSC (p and i of 8 bytes with idx64, else 4) into the builder's validated int32 / fp64 device
 * arrays; refused (< 0, a message on stderr) when the CSC is malformed. upper: P's upper triangle, counted in *ndiag */
int b200_csc_upload(const char *what, int rows, int n, const void *p, const void *i, const double *x, int idx64,
                    int upper, int **d_p, int **d_i, double **d_x, long long *nnz, long long *ndiag);
int b200_linsys_full_equilibrate(const ScsMatrix *A, const int *bnd, int nbnd, double *d_D, double *d_E);
int b200_linsys_scale_local(ScsLinSysWork *w, const double *d_D, const double *d_E);
/* contiguous row blocks balanced by nonzeros; offsets[nranks+1] (also exported for the tests) */
void b200_row_partition(int m, int n, const scs_int *Ap, const scs_int *Ai, int nranks, int *offsets);
/* the limits of the operators checked in scs_int width (host/abi.c): dimensions below 2^30, nnz(A) and nnz(P) at most
 * B200_MAX_STORED; prints a message naming the limit and returns nonzero when one is exceeded */
int b200_over_dim(const char *what, long long index, scs_int v);
int b200_over_stored(const char *what, scs_int v);
int b200_matrix_over_limits(const ScsMatrix *A, const ScsMatrix *P);
/* the argument checks of the device-pointer entry points (host/abi.c), each printing a message when it fails:
 * b200_dev_ptr_ok: 1 when p is device or managed memory of the library's device; b200_single_gpu: 1 unless the
 * process is one of several ranks; b200_overlap: 1 when the byte ranges [a, a + a_bytes) and [b, b + b_bytes)
 * intersect (a NULL pointer overlaps nothing) */
int b200_dev_ptr_ok(const void *p, const char *what);
int b200_single_gpu(void);
int b200_overlap(const char *a_name, const void *a, size_t a_bytes, const char *b_name, const void *b,
                 size_t b_bytes);

/* The caller's device CSC arrays, validated and copied into the library's own int32 / fp64 blocks */
typedef struct {
  int *Ap, *Ai, *Pp, *Pi;
  double *Ax, *Px;
  long long nnzA, nnzP, fullP;
} B200DevMats;
void b200_dev_mats_free(B200DevMats *dm);
/* one scs_int of device memory, read back (syncs); -1 on failure */
scs_int b200_read_dev_int(const scs_int *d_v);
/* scs_init's validate_matrix on device arrays (the CSC index arrays in scs_int width): the same checks, in the same
 * order, with the same messages, run by the validating copy (kernels/setup.cu) into dm's blocks. 0, or -1 */
int b200_validate_matrix_dev(const ScsMatrix *A, const ScsMatrix *P, B200DevMats *dm);

#endif
