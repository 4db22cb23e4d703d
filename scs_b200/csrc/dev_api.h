/* dev_api.h -- INTERNAL thin C layer between the C host code (host/ *.c) and the
 * hand-written sm_90a kernels (kernels/ *.cu).  All pointers named d_* are
 * device pointers; everything is enqueued on the library stream and is
 * asynchronous unless stated otherwise.  Return value: 0 ok, <0 error
 * (message via b200_last_error()). */
#ifndef B200_DEV_API_H
#define B200_DEV_API_H
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------ runtime ---- */
int b200_runtime_init(void);           /* picks device (LOCAL_RANK / SCS_B200_DEVICE), creates stream */
int b200_device_ok(void);
const char *b200_last_error(void);
int b200_num_sms(void);
void *b200_stream(void);               /* cudaStream_t */
void *b200_malloc(size_t bytes);       /* cudaMalloc, NULL on failure */
void b200_free(void *d_p);
void *b200_host_alloc(size_t bytes);   /* pinned host memory */
void b200_host_free(void *p);
int b200_h2d(void *d_dst, const void *src, size_t bytes);  /* async on stream (pageable => staged) */
int b200_d2h(void *dst, const void *d_src, size_t bytes);  /* async on stream */
int b200_d2d(void *d_dst, const void *d_src, size_t bytes);
int b200_memset0(void *d_dst, size_t bytes);
int b200_sync(void);
long long b200_launches(void);
/* CUDA-event timing on the library stream */
int b200_timer_start(void);
double b200_timer_stop_ms(void);       /* syncs; <0 on error */
/* device-side section timers (ScsInfo.lin_sys_time / cone_time / accel_time): CUDA events on the library
 * stream; the device time between two consecutive marks is billed to the section of the later mark */
enum { B200_SEC_LINSYS = 0, B200_SEC_CONE = 1, B200_SEC_ACCEL = 2, B200_SEC_OTHER = 3 };
int b200_section_begin(void);
int b200_section_mark(int section);
int b200_section_flush(void);          /* syncs with the last mark */
double b200_section_ms(int section);

/* ------------------------------------------------------------ SpMV ------- */
/* A sparse operator stored row-major (CSR): row r has entries
 * [rowptr[r], rowptr[r+1]) with column indices colidx[] and values vals[].
 * For SCS both orientations are used: the CSC arrays of A *are* the CSR of A'
 * (reference linsys/scs_matrix.c:161-186 accum_by_atrans), and the explicit
 * transpose At gives the CSR of A (reference cpu/indirect/private.c:7-46). */
typedef struct B200Spmv B200Spmv;

/* Limits of every operator: row and column counts below 2^30 (bits 30 and 31 of a stored column index are flags), and
 * at most B200_MAX_STORED entries in the stream, nnz plus one per empty row (the kernel forms stream positions up to
 * stored + 128 in 32-bit int). The host layer checks user input against them before narrowing it to int. */
#define B200_MAX_DIM ((1LL << 30) - 1)
#define B200_MAX_STORED (2147483647LL - 128)

/* an operator from a host CSR: the arrays are uploaded and the operator is built on the device like every other
 * (b200_spmv_create_dev, kernels/spmv.cu); nrows and nnz may be 0. NULL on failure */
B200Spmv *b200_spmv_create(int nrows, int ncols, const int *h_rowptr, const int *h_colidx,
                           const double *h_vals);
void b200_spmv_destroy(B200Spmv *M);
/* both resident orientations built ON THE DEVICE from the host CSC of A (kernels/setup.cu); m, n or nnz may be 0:
 * 0 ok, < 0 error */
int b200_setup_ops_from_csc(int m, int n, const int *h_Ap, const int *h_Ai, const double *h_Ax, B200Spmv **A_out,
                            B200Spmv **At_out);
/* the same from a CSC with 64-bit column pointers and row indices (the DLONG ABI): they are uploaded and narrowed to
 * int on the device, and the build is refused (< 0) if a pointer decreases, leaves [0, nnz] or p[0] != 0, or a row
 * index leaves [0, m) -- checked before any kernel reads an index. nnz = h_Ap[n] must not exceed B200_MAX_STORED. */
int b200_setup_ops_from_csc64(int m, int n, const long long *h_Ap, const long long *h_Ai, const double *h_Ax,
                              B200Spmv **A_out, B200Spmv **At_out);
int b200_spmv_nrows(const B200Spmv *M);
int b200_spmv_ncols(const B200Spmv *M);
long long b200_spmv_nnz(const B200Spmv *M);
long long b200_spmv_stored(const B200Spmv *M);     /* entries in the stream: flagged streams add one per empty row */
const double *b200_spmv_vals(const B200Spmv *M);   /* device */
const int *b200_spmv_colidx(const B200Spmv *M);    /* device */
const int *b200_spmv_rowptr(const B200Spmv *M);    /* device */
/* algorithmic bytes of one launch: 12 nnz (11 nnz packed) + 4 (R+1) + 8 C + 8 R (+ 8 R per extra row vector) */
double b200_spmv_alg_bytes(const B200Spmv *M, int extra_row_vectors);

enum { B200_POST_NONE = 0, B200_POST_DIV = 1, B200_POST_FMA_DOT = 2, B200_POST_FMA = 3, B200_POST_MUL = 4 };
/* B200_POST_MUL: y = s * d[r] with d = R_y^-1 precomputed -- what the reference's own GPU backend does
 * (linsys/gpu/indirect/private.c:78,164: inv_r_y, scale_by_diag); used by K1 inside the CG loop, where the fp64
 * division chain of POST_DIV holds the warps out of the gather pipeline. */
/* The row operand d[r] of the epilogue: a vector (B200_D_VEC), one value d[0] for every row (B200_D_ONE), or a
 * two-value table d[0..1] indexed by bit r of d_dmask (B200_D_TWO). The table forms stream no row vector; the one-pass
 * flagged-stream kernel only (no virtual rows). */
enum { B200_D_VEC = 0, B200_D_ONE = 1, B200_D_TWO = 2 };
enum { B200_HOOK_NONE = 0, B200_HOOK_CG_ALPHA = 1, B200_HOOK_P2P_SIGNAL = 2, B200_HOOK_P2P_ROUTE = 3 };
/* B200_HOOK_P2P_SIGNAL: when the LAST block of the launch has stored its rows, it publishes
 * hook_val into slot `rank` of every peer's flag line (d_hook_arg -> B200P2pSignal). */
typedef struct {
  int nranks, rank;
  unsigned long long *flags[8]; /* flags[r]: flag line of rank r as mapped in this process */
} B200P2pSignal;

/* B200_HOOK_P2P_ROUTE (POST_NONE only, flagged-stream kernel): output row j is not stored to d_y but PUSHED over
 * NVLink into the inbox of the rank that owns slice [lo[o], lo[o+1]) of the output space, as a 16-byte SELF-VALIDATING
 * element: {low 32 bits of the double | seq << 32, high 32 bits | seq << 32} with seq = the low 32 bits of hook_val
 * (the scheme of NCCL's LL protocol: every 8-byte half carries its own flag, so the receiver needs no fence, no
 * separate "ready" flag and can start summing while rows are still arriving). dst[o] = this rank's lane of rank o's
 * inbox as mapped in this process (element j - lo[o]); lo[nranks] = nrows. The SpMV thereby IS the reduce-scatter
 * send of the sharded-x CG (kernels/cg.cu). */
typedef struct {
  int nranks, rank;
  int lo[9];
  unsigned long long *dst[8];
  unsigned long long *flags[8];
} B200P2pRoute;

typedef struct {
  const double *d_x;     /* gather vector, length ncols */
  double *d_y;           /* output, length nrows */
  const double *d_init;  /* NULL: chain starts at 0; else at init_sign * d_init[r] (may alias d_y) */
  double init_sign;
  int post;              /* B200_POST_*: y = s | s / d[r] | fma(d[r], v[r], s) with dot(v, y) | same, no dot | s * d[r] */
  const double *d_d;
  int dform;             /* B200_D_*: how d[r] is read (the post-operations other than NONE) */
  const unsigned *d_dmask; /* B200_D_TWO: bit r selects d_d[0] or d_d[1] for row r */
  const double *d_v;
  double *d_dot;         /* B200_POST_FMA_DOT: receives sum_r v[r]*y[r] */
  int hook;              /* B200_HOOK_*: run by the last block after the dot is final */
  void *d_hook_arg;      /* B200CgCtl* for B200_HOOK_CG_ALPHA, B200P2pSignal* / B200P2pRoute* for the P2P hooks */
  unsigned long long hook_val;
  const int *d_skip;     /* optional: kernel returns at once if *d_skip != 0 */
  int pdl;               /* 1: launch as a programmatic dependent of the previous kernel in the stream (the kernel's
                            prologue -- barrier init, first matrix stages -- overlaps that kernel's tail) */
} B200SpmvArgs;

/* reordered copies for the CG operator (kernels/spmv.cu, kernels/setup.cu): rows of A by smallest column index */
int b200_perm_rows_by_min_col(const B200Spmv *A, int *d_perm /* new -> old */);
/* d_perm: in sorted, out placed (its first nrows entries, the kept rows, move by less than 32 slots); d_inv: out,
 * old -> new for all of M's rows */
B200Spmv *b200_spmv_permuted_rows(const B200Spmv *M, int *d_perm, int *d_inv, int nrows /* kept: perm[0..nrows) */);
int b200_spmv_refresh_permuted(B200Spmv *Mp, const B200Spmv *M, const int *d_perm); /* values only */
B200Spmv *b200_spmv_renumbered_cols(const B200Spmv *M, const int *d_inv /* old -> new */); /* view: borrows M's arrays */
/* for the CG loop's operators: store the index stream at 3 bytes per entry when M has at most 2^22 columns (else
 * nothing changes); M then serves POST_MUL / POST_FMA_DOT / POST_FMA only and b200_spmv_colidx(M) is NULL */
int b200_spmv_pack_indices(B200Spmv *M);
int b200_spmv_entry_bytes(const B200Spmv *M); /* bytes per stored entry the kernel streams: 12, or 11 when packed */
/* host placement behind b200_spmv_permuted_rows (pure host code): returns the copy's stored count */
long long b200_spmv_place_rows(int nrows, const int *sp_old, int *perm, int *sp_new);
int b200_gather_vec(int n, const int *d_perm, const double *d_src, double *d_dst); /* dst[i] = src[perm[i]] */

int b200_spmv(const B200Spmv *M, const B200SpmvArgs *a);
int b200_spmv_can_route(const B200Spmv *M); /* 1: B200_HOOK_P2P_ROUTE is available for this operator */
/* per-launch CUDA-event timing of M0 and M1 launched alternately (cold L2), ms per launch */
int b200_spmv_time_pair(const B200Spmv *M0, const B200Spmv *M1, int reps, double *out_ms);

/* ------------------------------------------------------------ CG --------- */
/* Device-resident control block of one PCG solve (reference
 * linsys/cpu/indirect/private.c:133-217). Lives in device memory; the host
 * reads it back only to learn `done` / `iters`. */
typedef struct {
  double ztr, ztr_prev, alpha, beta, pGp, rnorm, tol, bnorm;
  int iters;    /* CG iterations completed */
  int done;     /* 1: converged / broke / hit max_its; kernels early-exit */
  int max_its;
  int skip;     /* 1: ||b||_inf <= 1e-12, whole solve is b := 0 */
  int pad[4];
} B200CgCtl;

typedef struct {
  int n, m;
  const B200Spmv *A;   /* CSR of A  (m x n): rows of A   -> used for z = A p      */
  const B200Spmv *At;  /* CSR of A' (n x m): cols of A   -> used for y = A' z     */
  const B200Spmv *P;   /* full symmetric P as CSR (n x n) or NULL                 */
  /* m-space-reordered pair used ONLY inside mat_vec when set (tmp lives in the permuted order): A_cg = the non-empty
   * rows of A sorted by smallest column, At_cg = A' with its column indices renumbered, d_ry_cg = R_y in that order */
  const B200Spmv *A_cg, *At_cg;
  const double *d_ry_cg;
  /* the same row operands as tables (b200_cg_classify_diag): d_diag_tab = {the two values of 1/R_y over the rows of
   * A_cg, R_x[0]}, bit r of d_ry_mask picks the value of row r of A_cg; ry_form = B200_D_TWO when 1/R_y takes at most
   * two values there, rx_form = B200_D_ONE when R_x is uniform, else B200_D_VEC (d_ry_cg, d_rx) */
  double *d_diag_tab;
  unsigned *d_diag_mixed;
  unsigned *d_ry_mask;
  int ry_form, rx_form;
  const double *d_rx;  /* R_x (n) */
  const double *d_ry;  /* R_y (m) */
  double *d_ry_inv;    /* 1 / R_y (m), refreshed by b200_cg_set_preconditioner */
  double *d_M;         /* Jacobi preconditioner (n) */
  double *d_p, *d_r, *d_Gp, *d_z, *d_tmp; /* n, n, n, n, m */
  B200CgCtl *d_ctl;
  double *d_partials;  /* reduction slots */
  unsigned int *d_counter;
  B200CgCtl *h_ctl;    /* pinned mirror */
  /* row-sharded mode (nranks > 1): A, At hold only rows [row0, row0+mloc) of the matrix */
  int nranks, row0, mloc;
  const int *offsets;  /* host: row block boundaries, nranks+1 */
  double *d_red;       /* n: partial A_g' z before the all-reduce */
  int use_p2p;         /* 1: fused peer-memory reduction instead of the NCCL all-reduce */
  B200P2pSignal *d_p2p_sig; /* device copy of the peer flag table */
  B200P2pRoute *d_p2p_route; /* device copy of the push-routing table (sharded-x mode); d_p then lives in the
                                peer-mapped exchange allocation */
} B200Cg;

/* M_j = 1 / (R_x,j + P_jj + sum_k A_kj^2 / R_y,k)   (private.c:50-82) */
int b200_cg_set_preconditioner(const B200Cg *cg, const double *d_Pdiag);
/* after b200_cg_set_preconditioner, with the reordered pair and d_perm (its rows) in place: fills d_diag_tab and
 * d_ry_mask and sets ry_form / rx_form (one 4-byte read-back) */
int b200_cg_classify_diag(B200Cg *cg, const int *d_perm);
/* Full device solve of [[R_x+P, A'],[A, -R_y]] [x;y] = b in place on d_b (n+m),
 * warm start d_s (n) or NULL; returns CG iterations (>=0) or <0 on error.
 * Synchronises with the host only to poll the done flag. (private.c:284-324) */
int b200_cg_solve(B200Cg *cg, double *d_b, const double *d_s, double tol, int max_its,
                  int its_hint, const double *d_tol /* optional device tol */);
/* one CG iteration (4 kernels), for timing */
int b200_cg_one_iteration(B200Cg *cg, double *d_x);
/* algorithmic bytes of one CG iteration; per_kernel (optional): K1, K2, K3, K4 (DESIGN.md section 3) */
double b200_cg_iter_alg_bytes(const B200Cg *cg, double *per_kernel);
/* per-kernel device times (ms per launch) of `reps` genuine CG iterations: K1, K2, K3, K4, whole iteration */
int b200_cg_time_kernels(B200Cg *cg, double *d_x, int reps, double *out_ms);

/* ------------------------------------------------------------ comm (kernels/comm.cu) */
int b200_comm_rank(void);
int b200_comm_nranks(void);
int b200_allreduce_sum(double *d_buf, size_t count);
int b200_allgatherv(double *d_buf, const int *offsets);
/* peer-memory (CUDA IPC over NVLink) exchange buffers for the fused CG reduction */
int b200_p2p_setup(int n);
int b200_p2p_ok(int n);
int b200_p2p_stride(void);
double *b200_p2p_base(int r);
unsigned long long *b200_p2p_flags(int r);
double *b200_p2p_pvec(int r);   /* rank r's p vector inside its exchange allocation (sharded-x mode) */
double *b200_p2p_inbox(int r);  /* rank r's inbox [G][ceil(n/G)] of 16-byte elements (2 doubles of storage each) */
double *b200_p2p_pbox(int r);   /* rank r's p-box: the peers' p slices arrive here as 16-byte elements, [n][2] */
int b200_p2p_claim_pvec(void);  /* the exchange p vector serves one workspace at a time; 0 = claimed */
void b200_p2p_release_pvec(void);
unsigned long long b200_p2p_next_seq(void);

/* ------------------------------------------------------------ vector ops - */
/* out = |a|_inf etc. are produced into device scalars; see admm.cu */

#ifdef __cplusplus
}
#endif
#endif
