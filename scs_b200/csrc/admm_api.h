/* admm_api.h -- INTERNAL: device-resident ADMM state and the C launchers of
 * kernels/admm.cu, kernels/cones.cu, kernels/aa.cu (device pointers only). */
#ifndef B200_ADMM_API_H
#define B200_ADMM_API_H
#include "dev_api.h"

#ifdef __cplusplus
extern "C" {
#endif

/* slots of the device scalar board d_sc[] (doubles) */
enum {
  SC_VNORM2 = 0,  /* sum v_i^2                                   */
  SC_NM_WS,       /* ||u_x + tau g_x||_inf                        */
  SC_TOL,         /* CG tolerance of this iteration               */
  SC_TAU_T,       /* u_t[l-1] from root_plus                      */
  SC_NM_AXSB,     /* ||A x + s - b tau||_inf  (normalised)         */
  SC_NM_PXATYC,   /* ||P x + A'y + c tau||_inf (normalised)        */
  SC_O_AXSB,      /* un-normalised inf-norms ...                   */
  SC_O_AX,
  SC_O_AXS,
  SC_O_S,
  SC_O_PXATYC,
  SC_O_PX,
  SC_O_ATY,
  SC_BTY_TAU,     /* y'b   (normalised, tau not divided out)       */
  SC_CTX_TAU,     /* c'x                                           */
  SC_XPX_TAU,     /* x'Px                                          */
  SC_TAU,         /* |u_tau|                                       */
  SC_KAP,         /* |rsk_kappa|                                   */
  SC_TMP0, SC_TMP1, SC_TMP2, SC_TMP3, SC_TMP4, SC_TMP5, SC_TMP6, SC_TMP7,
  SC_COUNT = 32
};

typedef struct {
  int n, m;
  double *d_u, *d_u_t, *d_v, *d_v_prev, *d_rsk, *d_g, *d_R; /* l = n+m+1 each */
  double *d_ws;                                            /* n */
  double *d_sc;                                            /* SC_COUNT scalars */
  double *d_part;                                          /* reduction slots */
  unsigned int *d_cnt;
} B200Admm;

int b200_admm_sumsq(long long len, const double *d_v, double *d_out, double *d_part,
                    unsigned int *d_cnt);
int b200_admm_prep_linsys(const B200Admm *w, int iter, int store_prev, double pw);
int b200_admm_root_plus(const B200Admm *w, int iter);
int b200_admm_cone_pre(const B200Admm *w, int iter, int nz, int nl, double *d_cs);
int b200_admm_rsk_dual(const B200Admm *w, int do_dual, double alpha);
int b200_admm_dual_update(const B200Admm *w, double alpha);
int b200_admm_remap_v(const B200Admm *w);
int b200_admm_set_diag_r(const B200Admm *w, int nz, double rho_x, double scale);
int b200_admm_build_h(const B200Admm *w, const double *d_c, const double *d_b);
int b200_admm_warm_start(const B200Admm *w, const double *d_x, const double *d_y,
                         const double *d_s);
int b200_admm_cold_start(const B200Admm *w);
int b200_admm_resid_rows(const B200Admm *w, const double *d_ax, const double *d_b,
                         const double *d_D, double inv_ds, double dual_scale);
int b200_admm_resid_cols(const B200Admm *w, const double *d_aty, const double *d_px,
                         const double *d_c, const double *d_E, double inv_ps);
int b200_admm_unnormalize_sol(const B200Admm *w, const double *d_D, const double *d_E,
                              double primal_scale, double dual_scale, double *d_x, double *d_y,
                              double *d_s);
int b200_admm_normalize_sol(int n, int m, const double *d_D, const double *d_E,
                            double primal_scale, double dual_scale, double *d_x, double *d_y,
                            double *d_s);
int b200_vec_norms_dot(long long len, const double *d_a, const double *d_b, double *d_out3,
                       double *d_part, unsigned int *d_cnt);
int b200_vec_scale(long long len, double *d_a, double f);
int b200_vec_fill(long long len, double *d_a, double f);
int b200_vec_scale_by(long long len, double *d_a, const double *d_d, double f);

/* ---------------------------------------------------------------- equilibration (kernels/equil.cu) */
/* Ruiz + L2 equilibration in place on both resident orientations of A (P = 0). bnd[0] = z+l+bsize,
 * bnd[1..nbnd) = sizes of the cones sharing one D value. d_D (m), d_E (n) are outputs. */
int b200_equilibrate_dev(B200Spmv *A_rows, B200Spmv *A_cols, const int *bnd, int nbnd, double *d_D,
                         double *d_E);
/* the same with P != 0, bit for bit host/equilibrate.c: P scaled in place on its upper CSC (d_Pp, d_Pi, d_Px); d_Fp,
 * d_Fi, d_Fsrc: the structure of the full P (b200_sym_expand_structure) */
int b200_equilibrate_qp_dev(B200Spmv *A_rows, B200Spmv *A_cols, const int *d_Pp, const int *d_Pi, double *d_Px,
                            const int *d_Fp, const int *d_Fi, const int *d_Fsrc, const int *bnd, int nbnd,
                            double *d_D, double *d_E);
/* b = b_orig * D, c = c_orig * E (D, E NULL: plain copies); h_max (host, 4) receives max |b_orig|, max |b|,
 * max |c_orig|, max |c| (synchronises). b200_scale_b_c then multiplies both by sigma: together the device form of
 * host/equilibrate.c b200_normalize_b_c, bit for bit */
int b200_normalize_b_c_dev(int m, int n, const double *d_b_orig, const double *d_c_orig, const double *d_D,
                           const double *d_E, double *d_b, double *d_c, double *h_max);
int b200_scale_b_c(int m, int n, double *d_b, double *d_c, double sigma);
int b200_rescale_dev(B200Spmv *M, const double *d_rowscale, const double *d_colscale, int row_is_d);

/* ---------------------------------------------------------------- cones (kernels/cones.cu) */
typedef struct B200Cones B200Cones;
/* k_* arrays are HOST arrays; box bounds already scaled (normalize_box_cone). */
B200Cones *b200_cones_create(int m, int nz, int nl, int bsize, const double *h_bl,
                             const double *h_bu, int qsize, const int *h_q, int ssize,
                             const int *h_s);
/* exponential (ep primal, ed dual) and power (psize, parameters h_p, sign = primal/dual) triples: the
 * last 3 (ep + ed + psize) rows of the cone product (kernels/cone_triples.cu) */
int b200_cones_set_triples(B200Cones *c, int ep, int ed, int psize, const double *h_p);
int b200_cone_triples_project(int n_exp_primal, int n_exp_dual, int n_pow, long long exp_off,
                              const double *d_pow, double *d_x, const double *d_s, const double *d_ry);
/* complex PSD blocks (kernels/cones_complex.cu; reference cones.c:1072-1156). n_triples = ep + ed + psize. */
typedef struct B200CpsdCones B200CpsdCones;
B200CpsdCones *b200_cpsd_create(int cssize, const int *h_cs, long long first_row);
int b200_cpsd_project(B200CpsdCones *c, double *d_x, const double *d_s, const double *d_ry);
void b200_cpsd_destroy(B200CpsdCones *c);
void b200_cpsd_set_err(B200CpsdCones *c, int *d_err);
/* cuSOLVER handles are expensive to create (a cuBLAS handle + workspace each): workspaces borrow them from a small
 * per-device cache and hand them back at destroy (kernels/cones.cu). The pointer is a cusolverDnHandle_t. */
void *b200_solver_acquire(void);
void b200_solver_release(void *handle);
int b200_cones_set_complex_psd(B200Cones *c, int cssize, const int *h_cs, int n_triples);
/* log-det (d), nuclear-norm (nuc_m x nuc_n), l1-norm (ell1) and sum-of-largest-eigenvalues (sl_n, sl_k) cones of the
 * spectral build: the LAST rows of the cone product, in that order (kernels/cones_spectral.cu; reference
 * cones.c:1446-1490). Must be called before b200_cones_set_triples / b200_cones_set_complex_psd. 0 on success (also
 * when all are empty). */
int b200_cones_set_spectral(B200Cones *c, int dsize, const int *h_d, int nucsize, const int *h_nuc_m,
                            const int *h_nuc_n, int ell1_size, const int *h_ell1, int sl_size, const int *h_sl_n,
                            const int *h_sl_k);
/* the log-det cones' warm starts and saved projections back to zero, as at creation (0, or -1) */
int b200_cones_reset_spectral(B200Cones *c);
/* the Newton_stats record (iter, newton_success, residuals) of the last log-det cone projected; -1 when there are
 * no log-det cones. Syncs. */
int b200_cones_logdet_stats(B200Cones *c, int *iter, int *newton_success, double res[3]);
typedef struct B200SpecCones B200SpecCones;
B200SpecCones *b200_spec_create(int dsize, const int *h_d, int nucsize, const int *h_nuc_m, const int *h_nuc_n,
                                int ell1_size, const int *h_ell1, int sl_size, const int *h_sl_n, const int *h_sl_k,
                                long long first_row, int *d_err);
int b200_spec_project(B200SpecCones *c, double *d_x, const double *d_s, const double *d_ry);
int b200_spec_reset(B200SpecCones *c);
int b200_spec_logdet_stats(B200SpecCones *c, int *iter, int *newton_success, double res[3]);
void b200_spec_destroy(B200SpecCones *c);
/* shared with kernels/cones_spectral.cu (kernels/cones.cu): the sqrt2-scaled unpack of packed lower triangles, and
 * the DMMA contraction V diag(w) V' with weights max(w, 0) (mode 0, packed lower output; w ascending), signed weights
 * (mode 1, packed lower output) or its rectangular block (mode 2, dense rows x cols output from V of order
 * ld = rows + cols) */
void b200_psd_info_or(int count, const int *d_info, int *d_err);
void b200_psd_unpack_launch(int k, int count, const int *d_off, const double *d_x, double *d_mats);
void b200_reconstruct_launch(int mode, int ld, int rows, int cols, int count, const int *d_off, const double *d_mats,
                             const double *d_w, double *d_x, const double *d_s, const double *d_ry);
/* Every launcher of the eigen-decomposition cones, and every batched eigensolver call, covers a group of one order in
 * sub-batches of at most B200_EIG_BATCH blocks, and the eigensolver workspace is sized for min(count, B200_EIG_BATCH).
 * The per-block kernels take the block index from gridDim.y or gridDim.z, which stop at 65535; and
 * cusolverDnXsyevBatched asks for about 0.5 MB of workspace per matrix whatever its order (measured on an H100 with
 * cuSOLVER 11.7.5: 35 GB for 65535 matrices of order 2), while cuSOLVER 11.7.3 (CUDA 12.8, the build PyTorch wheels
 * bundle) refuses the workspace query from 32767 matrices on (16384 pass). 4096 keeps the workspace near 2 GB. */
#define B200_EIG_BATCH 4096
/* cusolverDnXsyevBatched (eigenvectors, lower triangle) on count matrices of order n, sub-batch by sub-batch, then
 * the status words ORed into d_err; solver / params: cusolverDnHandle_t / cusolverDnParams_t. 0, or -1 with the error
 * recorded as `what`. */
int b200_syevd_batched(void *solver, void *params, int n, double *d_mats, double *d_evals, void *d_work,
                       size_t work_bytes, void *h_work, size_t h_work_bytes, int *d_info, int count, int *d_err,
                       const char *what);
void b200_cones_destroy(B200Cones *c);
/* new box bounds (HOST arrays of bsize - 1, already scaled) and the box Newton warm start back to 1, as at creation */
int b200_cones_set_box(B200Cones *c, const double *h_bl, const double *h_bu);
/* Projects the box/SOC/PSD rows. On entry d_x (length m, the y block of u) holds
 * x = -r .* u on those rows and d_s holds the saved u (k_cone_pre); on exit
 * d_x = Pi(x) ./ r + s on those rows. d_ry: R_y (m). */
int b200_cones_project_rest(B200Cones *c, double *d_x, const double *d_s, const double *d_ry);
/* Full Moreau wrapper on a bare m-vector (operator-level tests): in place
 * x <- x + R^-1 Pi_K^{R^-1}(-R x); d_ry may be NULL (R = I). */
int b200_cones_proj_dual(B200Cones *c, double *d_x, const double *d_ry);
/* 0 unless a batched eigen-decomposition has reported info != 0 since creation (sticky); syncs */
int b200_cones_check(B200Cones *c);
double *b200_cones_scratch(B200Cones *c); /* m doubles (Moreau copy s) */

/* ---------------------------------------------------------------- AA (kernels/aa.cu) */
typedef struct B200Aa B200Aa;
B200Aa *b200_aa_create(int dim, int mem, int min_len, int type1, double regularization,
                       double relaxation, double safeguard_factor, double max_weight_norm,
                       int ir_max_steps, int verbosity);
void b200_aa_destroy(B200Aa *a);
double b200_aa_apply_dev(B200Aa *a, double *d_f, const double *d_x);
int b200_aa_safeguard_dev(B200Aa *a, double *d_f_new, double *d_x_new);
void b200_aa_reset_dev(B200Aa *a);
void b200_aa_restart_dev(B200Aa *a); /* the state of a new workspace: reset, and its statistics zeroed */
void b200_aa_stats(const B200Aa *a, int *out_ints8, double *out_dbl2);

#ifdef __cplusplus
}
#endif
#endif
