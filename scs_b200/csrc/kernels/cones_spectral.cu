// cones_spectral.cu -- projection onto the nuclear-norm, l1-norm and sum-of-largest-eigenvalues cones of SCS's
// spectral build, on the device. Only libscs_b200_spectral.so creates these cones; the kernels do not depend on the
// ScsCone layout and are linked into both libraries.
//
// Replaces reference src/spectral_cones/nuclear/{ell1_cone.c, nuclear_cone.c} and
// src/spectral_cones/sum-largest/{sum_largest_eval_cone.c, sum_largest_cone.c}. Each block of rows holds -R x on
// entry and Pi_K(.) / R + s on exit (the Moreau wrapper, as every cone of kernels/cones.cu).
//
//  * l1 cone (t, x), 1 + n rows: Pi = (t + mu, sign(x) max(|x| - mu, 0)) with the threshold mu >= 0 of
//    ell1_threshold (sort-free: Michelot's active-set iteration, one CTA per cone, fixed-order block sums). Cones of
//    up to ELL1_INLINE entries are finished by that CTA; the soft thresholding of bigger ones runs on 4096-row chunks.
//  * sum-of-largest cone (t, X), 1 + n(n+1)/2 rows, X packed like the PSD cone: groups by order n; sqrt2-scaled
//    unpack -> cusolverDnXsyevBatched -> the reference's sorted vector projection of (sqrt2 t, eigenvalues
//    descending), one thread per cone -> V diag(e') V' on the DMMA path with every eigenvalue (either sign) ->
//    repack with the diagonal / sqrt2, t' / sqrt2.
//  * nuclear-norm cone (t, X), 1 + m n rows, X m x n column-major with m >= n: groups by (m, n). The SVD comes from
//    the same batched symmetric eigensolver through the embedding E = [[0, X], [X', 0]] of order m + n: its
//    eigenvalues are +-sigma_i and m - n zeros, and an eigenvector of sigma_i > 0 is (u_i; v_i) / sqrt2 with
//    X v_i = sigma_i u_i. The n largest eigenvalues are the singular values; the l1 step of (t, sigma) is the same
//    ell1_threshold as the l1 cone; X' = sum_i sigma'_i u_i v_i' = sum_i 2 sigma'_i top(w_i) bot(w_i)' is the
//    rectangular DMMA contraction. Zero or near-zero sigma need no care: an eigenvector of an eigenvalue near 0 may
//    mix with the null space of E and is not of the form (u; v) / sqrt2, but its weight is sigma'_i, which is 0 when
//    sigma_i <= mu and sigma_i itself when mu = 0 (then Pi is the identity and the term is as small as sigma_i).
//    So such columns contribute nothing or at most their own tiny singular value, exactly as in X.
// Eigensolver status words join the sticky error flag of kernels/cones.cu (b200_cones_check).
#include "../common.cuh"
#include "../admm_api.h"
#include <cusolverDn.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <map>
#include <utility>
#include <vector>

#define ELL1_INLINE 8192   // l1 cones up to this many entries are soft-thresholded by their own CTA
#define ELL1_CHUNK 4096
#define ELL1_SMALL_T 256   // threads of the per-cone CTA (small cones / big cones)
#define ELL1_BIG_T 1024
#define NUC_T 128
#define TOL_LARGEST_CONE 1e-9  // reference sum_largest_cone.c:9

namespace {

__device__ __forceinline__ double finish(double xnew, const double *ry, const double *sv, long long row) {
  if (sv == nullptr) return xnew;
  return (ry != nullptr) ? xnew / ry[row] + sv[row] : xnew + sv[row];
}

// Threshold of the l1-norm cone projection of (t0, v), returned in every thread of the CTA:
//   Pi(t0, v) = (t0 + mu, sign(v) max(|v| - mu, 0)),   mu >= 0 the root of  sum_i max(|v_i| - mu, 0) = t0 + mu.
// mu = 0 when (t0, v) is in the cone (Pi is the identity); mu = +inf when -t0 >= max |v_i| ((t0, v) is in the polar
// cone and Pi = 0), as the reference's early exit (ell1_cone.c:107).
// Michelot's active-set iteration: A = all; mu = (sum_A |v| - t0) / (|A| + 1); A = {|v_i| > mu}; repeat until A stops
// shrinking. mu never decreases and A only shrinks, so it ends after at most n + 1 passes with the active set of the
// reference's sorted scan: the k largest magnitudes with |v|_(k) > mu >= |v|_(k+1). Sums are block sums in a fixed
// order (deterministic, no atomics). absv(i) returns |v_i|. All threads must call.
template <class F>
__device__ double ell1_threshold(int n, double t0, F absv, double *s_red /* 64 doubles */) {
  __shared__ double s_bc[2];
  double a[1] = {0.0}, mx[1] = {0.0};
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const double v = absv(i);
    a[0] += v;
    mx[0] = fmax(mx[0], v);
  }
  block_sum<1>(a, s_red);
  block_max<1>(mx, s_red + 32);
  if (threadIdx.x == 0) { s_bc[0] = a[0]; s_bc[1] = mx[0]; }
  __syncthreads();
  const double sum_all = s_bc[0], vmax = s_bc[1];
  __syncthreads();
  if (-t0 >= vmax) return INFINITY;
  double cnt = (double)n;
  double mu = (sum_all - t0) / (cnt + 1.0);
  if (!(mu > 0.0)) return 0.0;
  for (;;) {
    double r[2] = {0.0, 0.0};
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const double v = absv(i);
      if (v > mu) { r[0] += v; r[1] += 1.0; }
    }
    block_sum<2>(r, s_red);
    if (threadIdx.x == 0) { s_bc[0] = r[0]; s_bc[1] = r[1]; }
    __syncthreads();
    const double s = s_bc[0], c = s_bc[1];
    __syncthreads();
    if (c >= cnt) break;  // the active set no longer shrinks: mu is exact for it
    cnt = c;
    mu = (s - t0) / (c + 1.0);
  }
  return mu;
}

// soft thresholding of one entry (reference ell1_cone.c:139-144, 218-220)
__device__ __forceinline__ double ell1_apply(double xv, double mu, double diff) {
  const double a = fabs(xv);
  if (!(a > mu)) return 0.0;
  return xv >= 0 ? a - diff : -(a - diff);
}

// one CTA per l1 cone: off[b] = row of t, len[b] = n. Cones with n <= ELL1_INLINE are finished here; for the others
// (mu, t' - t) go to par[2 b] for k_ell1_chunks.
__global__ void k_ell1_cones(const int *__restrict__ off, const int *__restrict__ len, double *__restrict__ x,
                             const double *sv, const double *ry, double *__restrict__ par) {
  __shared__ double s_red[64];
  const int b = blockIdx.x;
  const long long base = off[b];
  const int n = len[b];
  const double t0 = x[base];
  const double *v = x + base + 1;
  const double mu = ell1_threshold(n, t0, [v](int i) { return fabs(v[i]); }, s_red);
  const double tn = (mu == INFINITY) ? 0.0 : t0 + mu;
  const double diff = tn - t0;
  if (n <= ELL1_INLINE) {
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const long long row = base + 1 + i;
      x[row] = finish(ell1_apply(x[row], mu, diff), ry, sv, row);
    }
  } else if (threadIdx.x == 0) {
    par[2 * b] = mu;
    par[2 * b + 1] = diff;
  }
  if (threadIdx.x == 0) x[base] = finish(tn, ry, sv, base);
}

// chunks of the big l1 cones: (index into par, first row, rows, -)
__global__ void k_ell1_chunks(const int4 *__restrict__ chunks, const double *__restrict__ par, double *__restrict__ x,
                              const double *sv, const double *ry) {
  const int4 ch = chunks[blockIdx.x];
  const double mu = par[2 * ch.x], diff = par[2 * ch.x + 1];
  for (int i = threadIdx.x; i < ch.z; i += blockDim.x) {
    const long long row = (long long)ch.y + i;
    x[row] = finish(ell1_apply(x[row], mu, diff), ry, sv, row);
  }
}

// nuclear cone: the embedding E = [[0, X], [X', 0]] of order N = m + n, column-major; off[b] = first row of X
__global__ void k_nuc_embed(int m, int n, int count, const int *__restrict__ off, const double *__restrict__ x,
                            double *__restrict__ mats) {
  const int b = blockIdx.y;
  if (b >= count) return;
  const int N = m + n;
  const double *X = x + off[b];
  double *M = mats + (size_t)b * N * N;
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < N * N; e += gridDim.x * blockDim.x) {
    const int I = e % N, J = e / N;
    double v = 0.0;
    if (I < m && J >= m) v = X[I + (size_t)(J - m) * m];
    else if (I >= m && J < m) v = X[J + (size_t)(I - m) * m];
    M[e] = v;
  }
}

// nuclear cone, vector step: one CTA per cone. sigma_i = max(lambda_{N-1-i}, 0), i < n (syevd sorts ascending);
// writes t' and overwrites the eigenvalues with the contraction weights: 2 sigma'_i on column N-1-i, 0 elsewhere.
__global__ void k_nuc_vector(int m, int n, int count, const int *__restrict__ off, double *__restrict__ evals,
                             double *__restrict__ x, const double *sv, const double *ry) {
  __shared__ double s_red[64];
  const int b = blockIdx.x;
  const int N = m + n;
  double *lam = evals + (size_t)b * N;
  const long long trow = (long long)off[b] - 1;
  const double t0 = x[trow];
  const double mu = ell1_threshold(n, t0, [lam, N](int i) { return fmax(lam[N - 1 - i], 0.0); }, s_red);
  const double tn = (mu == INFINITY) ? 0.0 : t0 + mu;
  const double diff = tn - t0;
  // every thread has read lam[] inside ell1_threshold (it ends with a barrier); rewrite it in place
  for (int c = threadIdx.x; c < N; c += blockDim.x) {
    double wgt = 0.0;
    if (c >= N - n) {
      const double sigma = fmax(lam[c], 0.0);
      wgt = 2.0 * ell1_apply(sigma, mu, diff);
    }
    lam[c] = wgt;
  }
  if (threadIdx.x == 0) x[trow] = finish(tn, ry, sv, trow);
}

// sum-of-largest cone, vector step: one thread per cone, the reference's sorted algorithm
// (proj_sum_largest_cone_sorted, sum_largest_cone.c:42-147) on x = eigenvalues in DESCENDING order, read through
// the ascending array e (x[i] = e[n-1-i]), and t scaled by sqrt2 as the eigenvalues are (sum_largest_eval_cone.c:111).
__global__ void k_sl_vector(int n, int count, const int *__restrict__ off, const int *__restrict__ kk,
                            double *__restrict__ evals, double *__restrict__ x, const double *sv, const double *ry) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= count) return;
  double *e = evals + (size_t)b * n;
  auto X = [e, n](int i) -> double & { return e[n - 1 - i]; };
  const int k = kk[b];
  const long long trow = (long long)off[b] - 1;
  const double sqrt2 = sqrt(2.0);
  double t = x[trow] * sqrt2;
  int nu = k, nt = 0;
  double eta = 0.0;
  const double t0 = t;
  double S = X(0);
  for (int i = 1; i < k; ++i) S += X(i);
  double a_u = X(nu - 1), a_t = X(nu);
  while (S > t + TOL_LARGEST_CONE) {
    const double ratio = (nu == k) ? 1.0 : (double)nt / (k - nu);
    const double s1 = (nu == k) ? a_u - a_t : (a_u - a_t) / (ratio - 1);
    const double s3 = (S - t) / (ratio * (nu + 1) + (k - nu));
    double s = (nu == 0) ? s3 : fmin(s3, s1);
    if (!(nu + nt == n || nt == 0)) s = fmin(s, a_t - X(nu + nt));
    eta += s * ratio;
    S -= s * (ratio * nu + k - nu);
    t = t0 + eta;
    if (nt > 0) a_t -= s;
    if (nu != 0 && s == s1) nu -= 1;
    if (nu > 0) a_u = X(nu - 1) - eta;
    nt = (nt == 0) ? 2 : nt + 1;
  }
  nt -= 1;
  for (int i = 0; i < nu; ++i) X(i) -= eta;
  for (int i = nu; i < nu + nt; ++i) X(i) = a_t;
  x[trow] = finish(t * (1.0 / sqrt2), ry, sv, trow);
}

// one batch of equally shaped matrices for cusolverDnXsyevBatched
struct EigGroup {
  int m, n;    // nuclear: X is m x n (order m + n); sum-of-largest: order n (m = 0)
  int N;       // order of the decomposed matrices
  int count;
  int *d_off;  // first row of each block's matrix (the row after t)
  int *d_k;    // sum-of-largest: k of each cone
  double *d_mats, *d_evals;
  int *d_info;
  void *d_work, *h_work;
  size_t work_bytes, h_work_bytes;
};

}  // namespace

struct B200SpecCones {
  std::vector<EigGroup> nuc, sl;
  int n_ell1_small, n_ell1_big, n_chunks;
  int *d_ell1_off, *d_ell1_len;  // small cones first, then big ones
  double *d_par;                 // 2 per big cone
  int4 *d_chunks;
  cusolverDnHandle_t solver;
  cusolverDnParams_t params;
  int *d_err;  // owned by B200Cones
};

static void free_group(EigGroup &g) {
  b200_free(g.d_off); b200_free(g.d_k); b200_free(g.d_mats); b200_free(g.d_evals); b200_free(g.d_info);
  b200_free(g.d_work); free(g.h_work);
}

extern "C" void b200_spec_destroy(B200SpecCones *c) {
  if (!c) return;
  b200_sync();
  for (auto &g : c->nuc) free_group(g);
  for (auto &g : c->sl) free_group(g);
  b200_free(c->d_ell1_off); b200_free(c->d_ell1_len); b200_free(c->d_par); b200_free(c->d_chunks);
  if (c->params) cusolverDnDestroyParams(c->params);
  b200_solver_release((void *)c->solver);
  delete c;
}

// offsets / ks: host arrays of the group; allocates the eigensolver batch of order g.N
static bool init_group(B200SpecCones *c, EigGroup &g, const std::vector<int> &offs, const std::vector<int> *ks) {
  g.count = (int)offs.size();
  g.d_off = (int *)b200_malloc((size_t)g.count * 4);
  g.d_mats = (double *)b200_malloc((size_t)g.count * g.N * g.N * 8);
  g.d_evals = (double *)b200_malloc((size_t)g.count * g.N * 8);
  g.d_info = (int *)b200_malloc((size_t)g.count * 4);
  bool ok = g.d_off && g.d_mats && g.d_evals && g.d_info && b200_h2d(g.d_off, offs.data(), offs.size() * 4) == 0;
  if (ok && ks) {
    g.d_k = (int *)b200_malloc((size_t)g.count * 4);
    ok = g.d_k && b200_h2d(g.d_k, ks->data(), ks->size() * 4) == 0;
  }
  ok = ok && b200_sync() == 0;
  size_t wd = 0, wh = 0;
  ok = ok && cusolverDnXsyevBatched_bufferSize(c->solver, c->params, CUSOLVER_EIG_MODE_VECTOR, CUBLAS_FILL_MODE_LOWER,
                                               g.N, CUDA_R_64F, g.d_mats, g.N, CUDA_R_64F, g.d_evals, CUDA_R_64F,
                                               &wd, &wh, g.count) == CUSOLVER_STATUS_SUCCESS;
  if (ok) {
    g.work_bytes = wd;
    g.h_work_bytes = wh;
    g.d_work = b200_malloc(wd ? wd : 16);
    g.h_work = wh ? malloc(wh) : nullptr;
    ok = g.d_work != nullptr && (wh == 0 || g.h_work != nullptr);
  }
  return ok;
}

extern "C" B200SpecCones *b200_spec_create(int nucsize, const int *h_nuc_m, const int *h_nuc_n, int ell1_size,
                                           const int *h_ell1, int sl_size, const int *h_sl_n, const int *h_sl_k,
                                           long long first_row, int *d_err) {
  if (b200_runtime_init() != 0) return nullptr;
  B200SpecCones *c = new B200SpecCones();  // value-initialised: counts and pointers start at 0
  c->d_err = d_err;
  long long row = first_row;
  std::map<std::pair<int, int>, std::vector<int>> nuc_by;
  for (int i = 0; i < nucsize; ++i) {
    nuc_by[{h_nuc_m[i], h_nuc_n[i]}].push_back((int)(row + 1));
    row += 1 + (long long)h_nuc_m[i] * h_nuc_n[i];
  }
  std::vector<int> small_off, small_len, big_off, big_len;
  std::vector<int4> chunks;
  for (int i = 0; i < ell1_size; ++i) {
    const int n = h_ell1[i];
    if (n <= ELL1_INLINE) {
      small_off.push_back((int)row);
      small_len.push_back(n);
    } else {
      for (int done = 0; done < n; done += ELL1_CHUNK)
        chunks.push_back(make_int4((int)big_off.size(), (int)(row + 1 + done), n - done < ELL1_CHUNK ? n - done : ELL1_CHUNK, 0));
      big_off.push_back((int)row);
      big_len.push_back(n);
    }
    row += 1 + (long long)n;
  }
  std::map<int, std::pair<std::vector<int>, std::vector<int>>> sl_by;
  for (int i = 0; i < sl_size; ++i) {
    auto &e = sl_by[h_sl_n[i]];
    e.first.push_back((int)(row + 1));
    e.second.push_back(h_sl_k[i]);
    row += 1 + (long long)h_sl_n[i] * (h_sl_n[i] + 1) / 2;
  }
  // ---- l1 cones: small cones first, then big ones (one CTA per cone each)
  c->n_ell1_small = (int)small_off.size();
  c->n_ell1_big = (int)big_off.size();
  c->n_chunks = (int)chunks.size();
  const int ncones = c->n_ell1_small + c->n_ell1_big;
  if (ncones > 0) {
    std::vector<int> offs(small_off), lens(small_len);
    offs.insert(offs.end(), big_off.begin(), big_off.end());
    lens.insert(lens.end(), big_len.begin(), big_len.end());
    c->d_ell1_off = (int *)b200_malloc((size_t)ncones * 4);
    c->d_ell1_len = (int *)b200_malloc((size_t)ncones * 4);
    c->d_par = (double *)b200_malloc((size_t)(2 * ncones) * 8);
    c->d_chunks = (int4 *)b200_malloc((chunks.size() + 1) * sizeof(int4));
    if (!c->d_ell1_off || !c->d_ell1_len || !c->d_par || !c->d_chunks ||
        b200_h2d(c->d_ell1_off, offs.data(), offs.size() * 4) != 0 ||
        b200_h2d(c->d_ell1_len, lens.data(), lens.size() * 4) != 0 ||
        (!chunks.empty() && b200_h2d(c->d_chunks, chunks.data(), chunks.size() * sizeof(int4)) != 0) ||
        b200_sync() != 0) {
      b200_spec_destroy(c);
      return nullptr;
    }
  }
  // ---- eigensolver batches
  if (!nuc_by.empty() || !sl_by.empty()) {
    c->solver = (cusolverDnHandle_t)b200_solver_acquire();
    if (!c->solver || cusolverDnCreateParams(&c->params) != CUSOLVER_STATUS_SUCCESS) {
      b200_spec_destroy(c);
      return nullptr;
    }
  }
  for (auto &kv : nuc_by) {
    EigGroup g;
    memset(&g, 0, sizeof(g));
    g.m = kv.first.first;
    g.n = kv.first.second;
    g.N = g.m + g.n;
    const bool ok = init_group(c, g, kv.second, nullptr);
    c->nuc.push_back(g);  // pushed before the check so that destroy releases what was allocated
    if (!ok) { b200_spec_destroy(c); return nullptr; }
  }
  for (auto &kv : sl_by) {
    EigGroup g;
    memset(&g, 0, sizeof(g));
    g.n = g.N = kv.first;
    const bool ok = init_group(c, g, kv.second.first, &kv.second.second);
    c->sl.push_back(g);
    if (!ok) { b200_spec_destroy(c); return nullptr; }
  }
  return c;
}

static int syevd(B200SpecCones *c, EigGroup &g, const char *what) {
  const cusolverStatus_t cs = cusolverDnXsyevBatched(
      c->solver, c->params, CUSOLVER_EIG_MODE_VECTOR, CUBLAS_FILL_MODE_LOWER, g.N, CUDA_R_64F, g.d_mats, g.N,
      CUDA_R_64F, g.d_evals, CUDA_R_64F, g.d_work, g.work_bytes, g.h_work, g.h_work_bytes, g.d_info, g.count);
  if (cs != CUSOLVER_STATUS_SUCCESS) {
    b200_set_error(what, cudaErrorUnknown, __FILE__, __LINE__);
    return -1;
  }
  b200_psd_info_or(g.count, g.d_info, c->d_err);
  return 0;
}

extern "C" int b200_spec_project(B200SpecCones *c, double *d_x, const double *d_s, const double *d_ry) {
  cudaStream_t st = (cudaStream_t)b200_stream();
  // ---- nuclear-norm cones
  for (auto &g : c->nuc) {
    dim3 eg((g.N * g.N + 255) / 256, g.count);
    k_nuc_embed<<<eg, 256, 0, st>>>(g.m, g.n, g.count, g.d_off, d_x, g.d_mats);
    b200_count_launch(1);
    if (syevd(c, g, "cusolverDnXsyevBatched (nuclear-norm cone embedding)") != 0) return -1;
    k_nuc_vector<<<g.count, NUC_T, 0, st>>>(g.m, g.n, g.count, g.d_off, g.d_evals, d_x, d_s, d_ry);
    b200_count_launch(1);
    b200_reconstruct_launch(2, g.N, g.m, g.n, g.count, g.d_off, g.d_mats, g.d_evals, d_x, d_s, d_ry);
  }
  // ---- l1-norm cones
  if (c->n_ell1_small > 0) {
    k_ell1_cones<<<c->n_ell1_small, ELL1_SMALL_T, 0, st>>>(c->d_ell1_off, c->d_ell1_len, d_x, d_s, d_ry, c->d_par);
    b200_count_launch(1);
  }
  if (c->n_ell1_big > 0) {
    k_ell1_cones<<<c->n_ell1_big, ELL1_BIG_T, 0, st>>>(c->d_ell1_off + c->n_ell1_small,
                                                       c->d_ell1_len + c->n_ell1_small, d_x, d_s, d_ry, c->d_par);
    k_ell1_chunks<<<c->n_chunks, 256, 0, st>>>(c->d_chunks, c->d_par, d_x, d_s, d_ry);
    b200_count_launch(2);
  }
  // ---- sum-of-largest-eigenvalues cones
  for (auto &g : c->sl) {
    b200_psd_unpack_launch(g.n, g.count, g.d_off, d_x, g.d_mats);
    if (syevd(c, g, "cusolverDnXsyevBatched (sum-of-largest-eigenvalues cone)") != 0) return -1;
    k_sl_vector<<<(g.count + 127) / 128, 128, 0, st>>>(g.n, g.count, g.d_off, g.d_k, g.d_evals, d_x, d_s, d_ry);
    b200_count_launch(1);
    b200_reconstruct_launch(1, g.n, g.n, g.n, g.count, g.d_off, g.d_mats, g.d_evals, d_x, d_s, d_ry);
  }
  CUDA_OK(cudaGetLastError());
  return 0;
}
