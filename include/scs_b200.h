/*
 * scs_b200.h -- C ABI of the B200-native ADMM hot path for SCS (cvxgrp/scs 3.2.11).
 *
 * Everything here is `extern "C"`, plain pointers and sizes.  Three groups:
 *
 *  (1) the OUTER ABI -- scs_init / scs_update / scs_solve / scs_finish / scs /
 *      scs_set_default_settings / scs_version and the data structs.  The struct
 *      layouts are byte-for-byte those of the reference build with
 *      DLONG=0, SFLOAT=0 and no spectral cones (reference include/scs.h:47-244,
 *      include/aa_stats.h:21-42, include/scs_types.h:16-30), so a caller
 *      compiled against the reference headers can link this library instead.
 *      Compiled with USE_SPECTRAL_CONES, ScsCone gains the reference's spectral
 *      block; that layout is served by libscs_b200_spectral.so.
 *      Compiled with DLONG, scs_int is 64 bits wide as in the reference's DLONG
 *      build (scs_types.h:14-24 on LP64); those layouts are served by
 *      libscs_b200_long.so, libscs_b200_spectral_long.so and the plugin-only
 *      libscs_b200_linsys_long.so.  The kernels index with 32-bit integers: a
 *      64-bit count, size or index is checked and narrowed at the entry points,
 *      and a value that does not fit is refused, never truncated.
 *
 *  (2) the LINEAR-SYSTEM PLUGIN ABI -- the five link-time symbols every SCS
 *      backend defines (reference include/linsys.h:25-71).  Host pointers in and
 *      out, exactly as the stock src/scs.c calls them (scs.c:1092,1127,763,1220).
 *
 *  (3) OPERATOR-LEVEL entry points (scs_b200_*): the cone projection, Anderson
 *      acceleration and SpMV operators of the hot path callable one at a time
 *      with host buffers.  The reference keeps these internal
 *      (include/cones.h:80-90, include/aa.h:66-143, linsys/scs_matrix.h); they are
 *      exported here so the parity tests can compare operator by operator.
 *
 * All compute happens in hand-written sm_90a CUDA kernels; there is no CPU
 * fallback: every entry point fails (NULL / nonzero / SCS_FAILED) when no CUDA
 * device is usable.
 *
 * Threading: one process drives ONE GPU (SCS_B200_DEVICE / LOCAL_RANK) through ONE stream.  Entry points may be
 * called from any host thread (each binds the calling thread to the library's device; the pinned staging buffer of
 * pageable copies is mutex-protected), but work of different workspaces is ordered by that single stream and the
 * kernel-launch sequence of a solve is not re-entrant: run one scs_solve / scs_solve_lin_sys at a time per
 * process (the reference is re-entrant per ScsWork; this library is re-entrant per process).
 */
#ifndef SCS_B200_H
#define SCS_B200_H

#ifdef __cplusplus
extern "C" {
#endif

/* primitive types of the reference build this ABI matches: SFLOAT=0, and DLONG=0 unless compiled with DLONG
 * (include/scs_types.h) */
#ifdef DLONG
typedef long long scs_int;
#else
typedef int scs_int;
#endif
typedef double scs_float;
#define SCS_NULL 0

/* exit flags of scs_solve / scs (values of reference include/scs.h:33-42) */
enum {
  SCS_INFEASIBLE_INACCURATE = -7, SCS_UNBOUNDED_INACCURATE = -6, SCS_SIGINT = -5, SCS_FAILED = -4,
  SCS_INDETERMINATE = -3, SCS_INFEASIBLE = -2, SCS_UNBOUNDED = -1, SCS_UNFINISHED = 0, SCS_SOLVED = 1,
  SCS_SOLVED_INACCURATE = 2
};

/* opaque workspaces */
typedef struct SCS_WORK ScsWork;
typedef struct SCS_LIN_SYS_WORK ScsLinSysWork;
typedef struct SCS_B200_CONE_WORK ScsB200ConeWork;
typedef struct SCS_B200_AA_WORK ScsB200AaWork;

/* The data structs below declare their members in the reference's order and with the reference's types,
 * several per line: the LAYOUT (pinned by tests/test_abi_cpu.py: sizes and offsets) is what a caller compiled
 * against the reference's headers relies on. */

/* CSC sparse matrix, zero-based (layout of reference include/scs.h:47-58): values x[nnz], row indices i[nnz],
 * column pointers p[n+1], then the shape m x n */
typedef struct {
  scs_float *x;
  scs_int *i, *p;
  scs_int m, n;
} ScsMatrix;

/* solver settings (layout of reference include/scs.h:61-101; defaults glbopts.h:35-50) */
typedef struct {
  scs_int normalize;
  scs_float scale;
  scs_int adaptive_scale;
  scs_float rho_x;
  scs_int max_iters;
  scs_float eps_abs, eps_rel, eps_infeas, alpha, time_limit_secs;
  scs_int verbose, warm_start;
  scs_int acceleration_lookback, acceleration_interval, acceleration_type_1;
  scs_float acceleration_regularization, acceleration_relaxation;
  const char *write_data_filename, *log_csv_filename; /* the CSV log is accepted and ignored with a warning */
} ScsSettings;

/* problem data (layout of reference include/scs.h:104-119): A is m x n, P the n x n upper triangle or NULL */
typedef struct {
  scs_int m, n;
  ScsMatrix *A, *P;
  scs_float *b, *c; /* lengths m, n */
} ScsData;

/* cone product K; the rows of A follow this order (layout of reference include/scs.h:122-172) */
typedef struct {
  scs_int z, l;        /* zero-cone rows, nonnegative-orthant rows */
  scs_float *bu, *bl;  /* box cone bounds, bsize-1 each */
  scs_int bsize;       /* box cone length including t */
  scs_int *q;          /* second-order cone sizes [qsize] */
  scs_int qsize;
  scs_int *s;          /* PSD matrix orders [ssize] */
  scs_int ssize;
  scs_int *cs;         /* complex PSD orders [cssize]: NOT supported by the device path */
  scs_int cssize;
  scs_int ep, ed;      /* primal / dual exponential triples */
  scs_float *p;        /* power cone parameters in [-1, 1] [psize]; negative = dual cone */
  scs_int psize;
#ifdef USE_SPECTRAL_CONES
  /* spectral cones (layout of the reference's USE_SPECTRAL_CONES build, include/scs.h:154-171); only
   * libscs_b200_spectral.so is compiled with this block. Their rows follow the power cones in this order. */
  scs_int *d;          /* log-det cone orders [dsize]: accepted by the layout, refused by scs_init */
  scs_int dsize;
  scs_int *nuc_m, *nuc_n; /* nuclear-norm cones: m x n column-major, 1 <= n <= m, 1 + m n rows each */
  scs_int nucsize;
  scs_int *ell1;       /* l1-norm cones: 1 + ell1[i] rows each */
  scs_int ell1_size;
  scs_int *sl_n, *sl_k; /* sum-of-largest-eigenvalues cones: order n, 0 < k < n, 1 + n(n+1)/2 rows each */
  scs_int sl_size;
#endif
} ScsCone;

/* solution or certificate (layout of reference include/scs.h:180-187) */
typedef struct {
  scs_float *x, *y, *s;
} ScsSolution;

/* Anderson-acceleration lifetime counters (layout of reference include/aa_stats.h:21-42) */
typedef struct {
  scs_int iter, n_accept;
  scs_int n_reject_lapack, n_reject_rank0, n_reject_nonfinite, n_reject_weight_cap, n_safeguard_reject;
  scs_int last_rank;
  scs_float last_aa_norm, last_regularization;
} AaStats;

/* solve report; times in milliseconds (layout of reference include/scs.h:190-244) */
typedef struct {
  scs_int iter;
  char status[128], lin_sys_solver[128];
  scs_int status_val, scale_updates;
  scs_float pobj, dobj, res_pri, res_dual, gap;
  scs_float res_infeas, res_unbdd_a, res_unbdd_p;
  scs_float setup_time, solve_time, scale, comp_slack;
  scs_int rejected_accel_steps, accepted_accel_steps;
  AaStats aa_stats;
  scs_float lin_sys_time, cone_time, accel_time;
} ScsInfo;

/* ------------------------------------------------------------------ (1) --
 * Outer ABI.  Replaces reference include/scs.h:271-338 / src/scs.c:1245-1551.
 * The ADMM iteration (scs.c:1356-1455) runs with all iterates resident in HBM;
 * the host sees scalars only (every CONVERGED_INTERVAL=25 iterations) and the
 * solution at the end. */
ScsWork *scs_init(const ScsData *d, const ScsCone *k, const ScsSettings *stgs);
scs_int scs_update(ScsWork *w, scs_float *b, scs_float *c);
scs_int scs_solve(ScsWork *w, ScsSolution *sol, ScsInfo *info,
                  scs_int warm_start);
void scs_finish(ScsWork *w);
scs_int scs(const ScsData *d, const ScsCone *k, const ScsSettings *stgs,
            ScsSolution *sol, ScsInfo *info);
void scs_set_default_settings(ScsSettings *stgs);
const char *scs_version(void);

/* ------------------------------------------------------------------ (2) --
 * Linear-system plugin ABI.  Replaces reference linsys/cpu/indirect/private.c
 * :221-349 and linsys/gpu/indirect/private.c:204-527.  A, P, diag_r are HOST
 * pointers (borrowed only during the call; copied to the device).  `b` (n+m)
 * and `s` (n or NULL) are HOST pointers; `b` is overwritten with [x; y]. */
ScsLinSysWork *scs_init_lin_sys_work(const ScsMatrix *A, const ScsMatrix *P,
                                     const scs_float *diag_r);
void scs_free_lin_sys_work(ScsLinSysWork *w);
scs_int scs_solve_lin_sys(ScsLinSysWork *w, scs_float *b, const scs_float *s,
                          scs_float tol);
scs_int scs_update_lin_sys_diag_r(ScsLinSysWork *w,
                                  const scs_float *new_diag_r);
const char *scs_get_lin_sys_method(void);

/* ------------------------------------------------------------------ (3) --
 * Operator-level entry points (host buffers; used by tests/ and bench.py). */

/* CG iterations used by the most recent scs_solve_lin_sys, and the running
 * total (reference private.h:29 tot_cg_its). */
scs_int scs_b200_linsys_last_cg_its(const ScsLinSysWork *w);
long long scs_b200_linsys_total_cg_its(const ScsLinSysWork *w);

/* y (+)= A x  and  y (+)= A' x  through the device SpMV kernels
 * (reference linsys/scs_matrix.c:161-203 accum_by_atrans / accum_by_a).
 * x, y are HOST arrays; accumulate != 0 adds into the incoming y. */
scs_int scs_b200_accum_by_a(ScsLinSysWork *w, const scs_float *x, scs_float *y,
                            scs_int accumulate);
scs_int scs_b200_accum_by_atrans(ScsLinSysWork *w, const scs_float *x,
                                 scs_float *y, scs_int accumulate);

/* Time one device SpMV (op 0: A x via the row-major copy, op 1: A' x via the
 * CSC arrays) with per-launch CUDA events over `reps` launches; A x and A'x are
 * launched alternately so neither matrix stays in L2 (as in the CG loop).
 * Inputs resident in HBM.  Returns average milliseconds per launch, <0 on
 * error.  *alg_bytes receives the algorithmic bytes of one launch (DESIGN.md). */
double scs_b200_time_spmv(ScsLinSysWork *w, scs_int op, scs_int reps,
                          double *alg_bytes);
/* Time `reps` CG iterations (4 kernels each) the same way. */
double scs_b200_time_cg_iter(ScsLinSysWork *w, scs_int reps, double *alg_bytes);
/* The kernels of the CG loop AS THEY RUN INSIDE A SOLVE (the solver's own p / tmp / r after a genuine CG start
 * on the host right-hand side b, length n+m), each bracketed by CUDA events on the library stream:
 * out_ms[0..4] = ms per launch of K1 (tmp = R_y^-1 A p), K2 (Gp = R_x p + A' tmp, p'Gp, alpha), K3 (x, r, z update
 * + reductions), K4 (p update) and of the whole iteration; out_bytes[0..4] = algorithmic bytes of each
 * (reference path: linsys/cpu/indirect/private.c:106-119,174-214). P = NULL. 0 on success. out_ms must hold 12
 * doubles: on several GPUs (sharded-x push mode, all ranks call together) out_ms[0..2] = K1, K2 (with its NVLink
 * pushes), the slice kernel; [3] = 0; [4] = iteration; [5..11] = the phases inside the slice kernel (rank-local). */
scs_int scs_b200_time_cg_kernels(ScsLinSysWork *w, const scs_float *b, scs_int reps, double *out_ms,
                                 double *out_bytes);

/* Cone operator: replaces reference src/cones.c:1498-1596 (init_cone /
 * proj_dual_cone / finish_cone) for zero, LP, box, SOC, PSD, exponential and power cones,
 * and in the spectral library also nuclear-norm, l1-norm and sum-of-largest-eigenvalues cones.
 * D is the row scaling of the equilibrated problem (length m) or NULL
 * (reference normalize_box_cone, cones.c:1160-1177).  x (length m) and r_y
 * (length m or NULL) are HOST arrays; x is projected in place onto the dual
 * cone under the R-metric. Returns 0, or <0 on failure. */
ScsB200ConeWork *scs_b200_init_cone(const ScsCone *k, scs_int m,
                                    const scs_float *D);
scs_int scs_b200_proj_dual_cone(ScsB200ConeWork *c, scs_float *x,
                                const scs_float *r_y);
void scs_b200_finish_cone(ScsB200ConeWork *c);

/* Anderson acceleration operator: replaces reference src/aa.c:657-979
 * (aa_init / aa_apply / aa_safeguard / aa_reset / aa_finish / aa_get_stats).
 * f, x, f_new, x_new are HOST arrays of length dim. */
ScsB200AaWork *scs_b200_aa_init(scs_int dim, scs_int mem, scs_int min_len,
                                scs_int type1, scs_float regularization,
                                scs_float relaxation,
                                scs_float safeguard_factor,
                                scs_float max_weight_norm,
                                scs_int ir_max_steps, scs_int verbosity);
scs_float scs_b200_aa_apply(ScsB200AaWork *a, scs_float *f, const scs_float *x);
scs_int scs_b200_aa_safeguard(ScsB200AaWork *a, scs_float *f_new,
                              scs_float *x_new);
void scs_b200_aa_reset(ScsB200AaWork *a);
void scs_b200_aa_finish(ScsB200AaWork *a);
AaStats scs_b200_aa_get_stats(const ScsB200AaWork *a);

/* Per-solve device statistics of the last scs_solve on this workspace. */
typedef struct {
  long long cg_iters;        /* total CG iterations */
  long long lin_sys_solves;  /* scs_solve_lin_sys calls */
  long long kernel_launches; /* kernels of this library launched */
  double spmv_ms;            /* reserved */
  scs_int n_gpus;
} ScsB200Stats;
scs_int scs_b200_get_stats(const ScsWork *w, ScsB200Stats *out);
/* Change max_iters of a live workspace (the settings are deep-copied at
 * scs_init; used by bench.py to run W warm-up and then exactly K timed steps). */
scs_int scs_b200_set_max_iters(ScsWork *w, scs_int max_iters);

/* Multi-GPU (one process per GPU, row-sharded KKT solve; SURVEY 8e). Rank 0 creates the
 * 128-byte NCCL unique id, the launcher distributes it (bench.py: torch.distributed), every
 * rank calls scs_b200_comm_init BEFORE scs_init / scs_init_lin_sys_work. Every rank passes
 * the same (full) problem; each keeps only its row block of A on its GPU. */
scs_int scs_b200_comm_unique_id(char *out128);
scs_int scs_b200_comm_init(scs_int rank, scs_int nranks, const char *id128);
scs_int scs_b200_comm_finalize(void);
/* peer-memory reduction of the sharded CG: 0 automatic, 1 one pass, 2 reduce-scatter + all-gather (DESIGN.md 6) */
void scs_b200_set_p2p_mode(int mode);
/* "sharded-x" push mode of the multi-GPU CG (x, r, z, Gp owned by n-slices, one slice kernel per rank and iteration;
 * kernels/cg.cu k_cgx_iteration, DESIGN.md 6): the DEFAULT since round 2; 0 selects the replicated modes above.
 * Also SCS_B200_SHARD_X=0/1. */
void scs_b200_set_shard_x(int on);
/* contiguous row blocks of A balanced by nonzeros: offsets[nranks+1] (host logic, no GPU needed) */
scs_int scs_b200_row_partition(scs_int m, scs_int n, const scs_int *Ap, const scs_int *Ai,
                               scs_int nranks, scs_int *offsets);

/* The SCS problem-file format (replaces reference src/rw.c:574-684 SCS(write_data) / SCS(read_data)): files
 * written by either library are read by the other. scs_init honours ScsSettings.write_data_filename with it.
 * read: allocates *d, *k, *stgs (release with scs_b200_free_data); returns 0, or -1 with everything freed. */
scs_int scs_b200_write_data(const char *filename, const ScsData *d, const ScsCone *k,
                            const ScsSettings *stgs);
scs_int scs_b200_read_data(const char *filename, ScsData **d, ScsCone **k, ScsSettings **stgs);
void scs_b200_free_data(ScsData *d, ScsCone *k, ScsSettings *stgs);

/* Number of kernels this library has launched in this process. */
long long scs_b200_launch_count(void);
/* 1 if a CUDA device of compute capability 10.x is usable, else 0. */
scs_int scs_b200_device_ok(void);
/* Device memory is cached across workspaces (a freed block is handed to the next allocation of the same size instead of
 * going back to the driver: cudaMalloc / cudaFree cost milliseconds each and cudaFree synchronises the device). This
 * returns every cached block to the driver; SCS_B200_POOL=0 disables the caching altogether. */
void scs_b200_release_memory(void);

#ifdef __cplusplus
}
#endif
#endif /* SCS_B200_H */
