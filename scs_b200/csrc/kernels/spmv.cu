// spmv.cu -- fp64 / int32 sparse mat-vec for the SCS indirect KKT solve, sm_90a.
//
// Replaces reference linsys/scs_matrix.c:161-186 (accum_by_atrans, used for both
// A'x on the CSC arrays and A x on the explicit transpose) and the cuSPARSE
// calls of linsys/gpu/gpu.c:3-58.
//
// Every operator is a "flagged stream" (spmv_flag_kernel): nonzero-per-lane on a TMA ring, rows recovered from END
// flags with ballots and a segmented warp scan -- see the block comment above the kernel. Rows longer than a warp-tile
// are cut into "virtual rows" whose partial sums a second, tiny pass adds in order (spmv_combine_kernel).
// Static CTA partition (no atomics => a launch is bit-reproducible), 1-D TMA bulk copies
// (cp.async.bulk, L2 evict_first) of the value / index slices into shared memory with mbarrier completion,
// products rounded separately from the adds (__dmul_rn / __dadd_rn: the reference's scalar loop
// `yj += Ax[p] * x[Ai[p]]` is not contracted to fma in the oracle build), fused epilogues
// y = s | s / d[r] | fma(d[r], v[r], s) (d[r] from a vector, or from a one- or two-value table: B200_D_*)
// plus the dot product v'y with a deterministic last-block reduction and
// an optional hook that turns the dot into the CG step length on the device.
//
// Algorithmic bytes per launch (DESIGN.md): 12*nnz (11*nnz with a packed index stream) + 4*(R+1) + 8*C + 8*R (+8*R
// per extra row vector read by the epilogue).
#include "../common.cuh"
#include "../dev_api.h"
#include "../spmv_flag.cuh"
#include <mutex>
#include <stdlib.h>
#include <string.h>
#include <vector>

struct B200Spmv {
  int nrows, ncols;
  long long nnz;
  int *d_rowptr;     // stored row pointers (every row has >= 1 stored entry)
  int *d_colidx;     // column | B200_FLAG_END | B200_FLAG_SKIP
  double *d_vals;
  int grid;
  double *d_partials;
  unsigned int *d_counter;
  long long stored;  // entries held in d_colidx / d_vals: nnz + one explicit zero per empty row
  int4 *d_wt3;       // warp-tile descriptors, padded per CTA to groups of SPMV3_NCW
  int *d_cta_begin3; // first group of every CTA
  // long-row support: virtual rows + combine pass, see Spmv3Plan::vptr
  int nvrows;        // virtual rows (== nrows when no row was cut)
  int *d_vptr;       // nrows+1, or NULL
  double *d_vscratch;  // nvrows partial sums
  int borrows;       // 1: d_rowptr / d_vals / d_wt3 / d_cta_begin3 belong to another operator (renumbered-columns view)
  unsigned char *d_idx24;  // the packed index stream (b200_spmv_pack_indices; d_colidx is then NULL), or NULL
};

// Tail of both kernels. Multi-GPU (replicated modes): the last block tells every peer that this rank's partial product
// is complete; the push mode (B200_HOOK_P2P_ROUTE) needs no signal, every pushed row validates itself. Then, for
// POST_FMA_DOT, the deterministic last-block finish of the dot product and the CG step-length hook.
template <int POST>
__device__ __forceinline__ void spmv_tail(double dot_acc, double *dot_out, int hook, void *hook_arg,
                                          unsigned long long hook_val, double *partials, unsigned int *counter,
                                          double *s_red) {
  if (hook == B200_HOOK_P2P_SIGNAL) {
    __syncthreads();
    if (threadIdx.x == 0) {
      __threadfence();
      const unsigned tk = atomicAdd(counter, 1u);
      if (tk == gridDim.x - 1) {
        *counter = 0u;
        __threadfence_system();
        const B200P2pSignal *ps = reinterpret_cast<const B200P2pSignal *>(hook_arg);
        for (int r = 0; r < ps->nranks; ++r)
          if (r != ps->rank) *((volatile unsigned long long *)(ps->flags[r] + ps->rank)) = hook_val;
      }
    }
  }
  if (POST == B200_POST_FMA_DOT) {
    double acc[1] = {dot_acc};
    block_sum<1>(acc, s_red);
    if (grid_finish<1>(acc, partials, counter, 0u, s_red)) {
      if (threadIdx.x == 0) {
        *dot_out = acc[0];
        if (hook == B200_HOOK_CG_ALPHA) {
          B200CgCtl *c = reinterpret_cast<B200CgCtl *>(hook_arg);
          c->pGp = acc[0];
          c->alpha = c->ztr / acc[0];
        }
      }
    }
  }
}

// ==================================================================================
// The "flagged stream" -- nonzero-per-lane instead of row-per-lane.
//
// What bounds the SpMV of a uniformly random matrix is not HBM but the L1TEX pipe: every
// nonzero costs one wavefront for its 8-byte gather (no two lanes share a 128-byte line), and
// a row-per-thread kernel adds ~0.45 shared-memory wavefronts per nonzero on top (bank
// conflicts of the row-strided reads of values / indices, row pointers) -- ncu: L1TEX 70-80 %.
// This kernel removes everything but the gather from that pipe:
//   * the operator is stored as a FLAGGED stream: colidx carries "last entry of its row" in bit 31
//     and "explicit zero, do not gather" in bit 30 (B200_FLAG_END / B200_FLAG_SKIP, common.cuh); every empty row
//     owns one such zero entry, so row r is simply the r-th END flag and the kernel needs NO row pointers at all;
//   * the stream is cut into WARP-TILES of whole rows whose 16-byte-aligned span is <= 128
//     entries; lane l of the consumer warp owns the 4 CONSECUTIVE entries [4l, 4l+4): one
//     LDS.128 for the indices and two conflict-free LDS.128 for the values (lanes 4..7 of every
//     quarter-warp read their two halves in swapped order), then 4 independent gathers;
//   * rows are recovered in registers: 4 ballots + popc give every END its row number, a
//     sequential in-lane sum plus a warp segmented scan of the lanes' open tails (only as many
//     shuffle steps as the longest row in the warp-tile needs) gives the row sums -- fixed order,
//     so bit-reproducible run to run; a row inside one lane is still the CPU's sequential chain;
//   * a CTA stages SPMV3_NCW warp-tiles (one per consumer warp) per TMA stage: value slice,
//     index slice and the warp-tile descriptors, three bulk copies on one mbarrier; the stage is
//     released as soon as the warp has its 48 bytes per lane in registers, before the gathers
//     return, so the ring runs ahead of the gather latency.
// Rows longer than SPMV3_MAXROW entries do not fit a warp-tile: they are cut into balanced pieces
// (spmv3_piece_end), each a "virtual row" with its own END, and spmv_combine_kernel adds the pieces.
// The ring's geometry and the per-stage work of producer and consumers: spmv_flag.cuh.
static size_t spmv3_smem_bytes() {
  return (size_t)SPMV3_STAGES * (SPMV3_CAP * 12 + SPMV3_NCW * 16) + 2 * SPMV3_STAGES * 8 + 64 * 8 +
         (size_t)SPMV3_NCW * SPMV3_WT * 8;
}

// A row longer than SPMV3_MAXROW entries is cut into ceil(len / SPMV3_MAXROW) balanced pieces, the first
// len % pieces of them one entry longer; a shorter row is one piece. Returns the end of piece q, counted from the
// row's first entry. The one cut rule of the fill (spmv3_fill_row) and the virtual rows.
__host__ __device__ __forceinline__ int spmv3_piece_end(int len, int q) {
  const int pieces = len > SPMV3_MAXROW ? (len + SPMV3_MAXROW - 1) / SPMV3_MAXROW : 1;
  const int small = len / pieces, big = len % pieces;
  return (q + 1) * small + (q + 1 < big ? q + 1 : big);
}

// The stored entries of one row of `len` CSR entries (from entry a, stored from position pos): the entries, with an END
// on the last entry of the row or of each of its pieces; an empty row stores one explicit zero, SKIP | END. The one
// fill of the flagged stream: k_fill_flagged runs it per row on the device, the plan export of the CPU tests on the host.
__host__ __device__ __forceinline__ void spmv3_fill_row(int len, int a, int pos, const int *__restrict__ ci,
                                                        const double *__restrict__ va, int *__restrict__ oi,
                                                        double *__restrict__ ov) {
  if (len == 0) {
    oi[pos] = (int)(B200_FLAG_END | B200_FLAG_SKIP);
    ov[pos] = 0.0;
  }
  for (int k = 0, q = 0, e = spmv3_piece_end(len, 0); k < len; ++k) {
    const bool end = k + 1 == e;
    oi[pos + k] = end ? (int)((unsigned)ci[a + k] | B200_FLAG_END) : ci[a + k];
    ov[pos + k] = va[a + k];
    if (end) e = spmv3_piece_end(len, ++q);
  }
}

// The phases (first stored position modulo 4, bit q = phase q) at which the flag kernel sums a row of `len` <= 124
// entries exactly as it does at `phase`. The kernel cuts a row at phase q into lane pieces of 4 - q, 4, 4, ..., and
// the remainder, sums each piece sequentially in its lane and joins the pieces with the segmented scan. The result is
// the plain sequential chain ((p0 + p1) + p2) + ... in two cases only:
//   * q + len <= 4: one piece, summed in one lane (what is open from the lanes before adds an exact 0);
//   * q + len == 5: two pieces, the second holds the last entry alone: (chain of the first piece) + p[len-1].
// So a row that is plain sequential at `phase` is plain sequential at every q <= 5 - len (len 1, 2: all four phases;
// 3: 0..2; 4: 0, 1; 5: 0). Any other cut has a tree that depends on q (the scan joins two or more pieces of at least
// two entries, or three or more pieces), and such a row keeps its phase.
__host__ __device__ __forceinline__ unsigned spmv3_same_sum_phases(int len, int phase) {
  if (phase + len > 5) return 1u << phase;
  return (1u << (6 - len < 4 ? 6 - len : 4)) - 1u;
}



// IDX24: the index stream is packed (spmv3_idx24_*), else int32
template <int POST, bool IDX24>
__global__ void __launch_bounds__(SPMV3_THREADS, SPMV3_CTAS_PER_SM)
spmv_flag_kernel(const void *__restrict__ colidx, const double *__restrict__ vals,
                 const int4 *__restrict__ wt, const int *__restrict__ cta_begin,
                 const double *__restrict__ x, double *__restrict__ y, const double *init,
                 double init_sign, const double *__restrict__ d, const unsigned *__restrict__ dmask, int dform,
                 const double *__restrict__ v, double *dot_out, int hook, void *hook_arg, const int *skip,
                 double *partials, unsigned int *counter, unsigned long long hook_val) {
  // Programmatic dependent launch: nothing above pdl_wait() reads data a predecessor kernel writes -- the
  // descriptors and the matrix stream are immutable -- so barrier init and the first ring stages overlap the
  // predecessor's tail. `skip`, x, d, dmask, v, init are read only after the wait.
  extern __shared__ __align__(128) unsigned char smem_raw[];
  double *s_vals = reinterpret_cast<double *>(smem_raw);
  int *s_idx = reinterpret_cast<int *>(s_vals + SPMV3_STAGES * SPMV3_CAP);
  int4 *s_desc = reinterpret_cast<int4 *>(s_idx + SPMV3_STAGES * SPMV3_CAP);
  uint64_t *s_full = reinterpret_cast<uint64_t *>(s_desc + SPMV3_STAGES * SPMV3_NCW);
  uint64_t *s_empty = s_full + SPMV3_STAGES;
  double *s_red = reinterpret_cast<double *>(s_empty + SPMV3_STAGES);
  double *s_out = s_red + 64;  // per consumer warp: the row sums of its warp-tile, by row number

  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int g_begin = cta_begin[blockIdx.x];  // in groups of SPMV3_NCW warp-tiles
  const int nt = cta_begin[blockIdx.x + 1] - g_begin;
  // multi-GPU push mode: the routing table (static device data, written once at setup)
  __shared__ int s_rt_lo[9];
  __shared__ unsigned long long *s_rt_dst[8];
  const bool routed = (POST == B200_POST_NONE) && hook == B200_HOOK_P2P_ROUTE;
  if (routed && tid < 9) {
    const B200P2pRoute *rt = reinterpret_cast<const B200P2pRoute *>(hook_arg);
    s_rt_lo[tid] = tid <= rt->nranks ? rt->lo[tid] : 0x7fffffff;
    if (tid < 8) s_rt_dst[tid] = tid < rt->nranks ? rt->dst[tid] : nullptr;
  }
  if (tid == 0) {
#pragma unroll
    for (int s = 0; s < SPMV3_STAGES; ++s) {
      mbar_init(&s_full[s], 1);
      mbar_init(&s_empty[s], SPMV3_NCW);
    }
    mbar_fence_init();
  }
  __syncthreads();
  pdl_launch_dependents();

  double dot_acc = 0.0;
  int skipped = 0;
  const Spmv3Ring R = {s_vals, s_idx, s_desc, s_full, s_empty, s_out};
  if (wid == 0) {
    // ------------------------------------------------ producer (one elected lane)
    if (lane == 0) {
      const uint64_t pol = l2_policy_evict_first();
      const int4 *g = wt + (size_t)g_begin * SPMV3_NCW;
      int ka_n = 0, ke_n = 0;
      if (nt > 0) {
        ka_n = __ldg(&g[0].y) & ~3;
        const int4 l = __ldg(&g[SPMV3_NCW - 1]);
        ke_n = l.y + l.z;
      }
      bool waited = false;
      for (int i = 0; i < nt; ++i) {
        const int st = i % SPMV3_STAGES, use = i / SPMV3_STAGES;
        const int ka = ka_n, cnt = (ke_n - ka_n + 3) & ~3;
        if (i + 1 < nt) {  // next group's extent: issued before the wait below, so its latency hides
          ka_n = __ldg(&g[(size_t)(i + 1) * SPMV3_NCW].y) & ~3;
          const int4 l = __ldg(&g[(size_t)(i + 2) * SPMV3_NCW - 1]);
          ke_n = l.y + l.z;
        }
        if (use > 0) {
          if (!waited) {  // the first ring round was issued ahead of the predecessor's completion
            pdl_wait();
            waited = true;
            if (skip != nullptr && *((volatile const int *)skip) != 0) { skipped = i; break; }
          }
          mbar_wait(&s_empty[st], (unsigned)((use - 1) & 1));
        }
        spmv3_issue_stage<IDX24>(R, st, g, i, ka, cnt, colidx, vals, pol);
      }
      if (!waited) {
        pdl_wait();
        if (skip != nullptr && *((volatile const int *)skip) != 0) skipped = nt < SPMV3_STAGES ? nt : SPMV3_STAGES;
      }
      if (skipped) {
        // the launch is a no-op (*skip set), but `skipped` stages are in flight into this CTA's shared memory:
        // they must land before the CTA may exit
        for (int i = 0; i < skipped && i < SPMV3_STAGES; ++i) mbar_wait(&s_full[i], 0u);
      }
    }
    if (skip != nullptr) {  // the other lanes of the producer warp only need the decision for the tail below
      if (lane != 0) pdl_wait();
      skipped = (*((volatile const int *)skip) != 0) ? 1 : 0;
    }
  } else {
    // ------------------------------------------------ consumers: one warp-tile per warp per stage
    pdl_wait();
    if (skip != nullptr && *((volatile const int *)skip) != 0) skipped = 1;
    // the table forms of d (B200_D_ONE / B200_D_TWO): its values, once per launch
    constexpr bool TAB = POST == B200_POST_MUL || POST == B200_POST_FMA_DOT || POST == B200_POST_FMA;
    Spmv3Epi E = {x, y, init, init_sign, d, dmask, dform, 0.0, 0.0, v, routed, s_rt_lo, s_rt_dst, hook_val};
    if (TAB && dform != B200_D_VEC) {
      E.dt0 = d[0];
      E.dt1 = dform == B200_D_TWO ? d[1] : E.dt0;
    }
    for (int i = 0; i < (skipped ? 0 : nt); ++i)
      spmv3_consume_stage<POST, IDX24, true>(R, i % SPMV3_STAGES, (unsigned)((i / SPMV3_STAGES) & 1), wid - 1, lane,
                                             E, dot_acc);
  }

  if (skipped) return;  // uniform over the CTA: every thread read the same *skip after the predecessor completed
  spmv_tail<POST>(dot_acc, dot_out, hook, hook_arg, hook_val, partials, counter, s_red);
}

// Second pass of the long-row mode. The flag kernel has written one sum per
// VIRTUAL row into `part`; thread r adds the pieces of true row r in order, applies the epilogue and the same
// deterministic dot / hook tail as the one-pass kernel.
template <int POST>
__global__ void __launch_bounds__(256)
spmv_combine_kernel(int nrows, const int *__restrict__ vptr, const double *__restrict__ part,
                    double *__restrict__ y, const double *init, double init_sign, const double *__restrict__ d,
                    const double *__restrict__ v, double *dot_out, int hook, void *hook_arg, const int *skip,
                    double *partials, unsigned int *counter, unsigned long long hook_val) {
  if (skip != nullptr && *((volatile const int *)skip) != 0) return;
  __shared__ double s_red[64];
  double dot_acc = 0.0;
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < nrows; r += gridDim.x * blockDim.x) {
    double s = 0.0;
    for (int q = vptr[r]; q < vptr[r + 1]; ++q) s = __dadd_rn(s, part[q]);
    if (init != nullptr) s = __dadd_rn(s, init_sign * init[r]);
    const double dv = (POST != B200_POST_NONE) ? d[r] : 0.0;
    const double vv = (POST == B200_POST_FMA_DOT || POST == B200_POST_FMA) ? v[r] : 0.0;
    spmv_epilogue<POST>(s, r, y, dv, vv, dot_acc);
  }
  spmv_tail<POST>(dot_acc, dot_out, hook, hook_arg, hook_val, partials, counter, s_red);
}

// ---- host side: the virtual rows, warp-tiles and static CTA partition of a flagged stream, from its stored row
// pointers. Pure host code up to spmv3_finish (no CUDA calls): also exported for the CPU tests
// (tests/test_spmv_plan_cpu.py re-executes the kernel's lane algorithm on this plan in numpy).
struct Spmv3Plan {
  std::vector<int> rowptr;   // stored row pointers (every row has >= 1 stored entry)
  // long-row support: a row longer than SPMV3_MAXROW is cut into pieces ("virtual rows", an END flag at the end of
  // every piece); the kernel then produces one sum per virtual row and a combine pass adds the pieces of each true
  // row. vptr[r] = first virtual row of true row r, vrp = the virtual row pointers (both empty when no row was cut).
  std::vector<int> vptr, vrp;
  int nvrows = 0;
  std::vector<int4> wt;      // padded per CTA to a multiple of SPMV3_NCW: {row0, k0, cnt, nrows}
  std::vector<int> cta_begin;  // grid+1, in groups of SPMV3_NCW descriptors
  int grid = 0;
  int nwt = 0;               // real warp-tiles
};

static bool spmv3_fits(long long stored) {
  if (stored <= SPMV3_MAX_STORED) return true;
  b200_set_error("b200_spmv: a flagged stream holds at most 2^31 - 129 entries (nnz + one per empty row)",
                 cudaErrorInvalidValue, __FILE__, __LINE__);
  return false;
}

// virtual rows from the stored row pointers P.rowptr: the rows themselves unless one is longer than SPMV3_MAXROW
static void spmv3_virtual_rows(int nrows, Spmv3Plan &P) {
  const int *sp = P.rowptr.data();
  P.vptr.clear();
  P.vrp.clear();
  P.nvrows = nrows;
  int r = 0;
  while (r < nrows && sp[r + 1] - sp[r] <= SPMV3_MAXROW) ++r;
  if (r == nrows) return;
  P.vptr.resize((size_t)nrows + 1);
  P.vrp.reserve((size_t)nrows + 1);
  for (r = 0; r < nrows; ++r) {
    P.vptr[r] = (int)P.vrp.size();
    const int len = sp[r + 1] - sp[r];
    for (int q = 0, e = 0; e < len; e = spmv3_piece_end(len, q++)) P.vrp.push_back(sp[r] + e);
  }
  P.nvrows = (int)P.vrp.size();
  P.vptr[nrows] = P.nvrows;
  P.vrp.push_back(sp[nrows]);
}

// warp-tiles (whole (virtual) rows whose aligned span (k0 & ~3 .. end) is <= 128 entries) and the static CTA
// partition, from the stored (virtual) row pointers alone -- shared by every operator (plain and permuted).
// CTAs own equal counts of warp-tiles. A warp-tile holds up to 128 entries whatever its rows, so this balances the
// gathers; on the row-sorted CG copy of A it leaves 2.8x more rows on the last CTAs than on the first, but rows are
// cheap next to gathers: balancing on entries + rows (or 2 entries + rows) was 1.3 % (0.2 %) slower per CG iteration
// on C2 (H100 SXM, DESIGN.md section 3.1).
static void spmv3_tiles_from_rowptr(int grid_cap, Spmv3Plan &P) {
  const int nv = P.nvrows;
  const int *vrp = P.vrp.empty() ? P.rowptr.data() : P.vrp.data();
  std::vector<int4> real;
  real.reserve((size_t)(vrp[nv] / 100 + 16));
  for (int r = 0; r < nv;) {
    const int k0 = vrp[r], base = k0 & ~3;
    int r1 = r;
    while (r1 < nv && vrp[r1 + 1] - base <= SPMV3_WT) ++r1;
    int4 t;
    t.x = r;
    t.y = k0;
    t.z = vrp[r1] - k0;
    t.w = r1 - r;
    real.push_back(t);
    r = r1;
  }
  P.nwt = (int)real.size();
  int grid = grid_cap < P.nwt ? grid_cap : P.nwt;
  if (grid < 1) grid = 1;
  P.grid = grid;
  P.cta_begin.assign((size_t)grid + 1, 0);
  P.wt.clear();
  P.wt.reserve(real.size() + (size_t)grid * SPMV3_NCW);
  for (int c = 0; c < grid; ++c) {
    const long long a = (long long)P.nwt * c / grid, b = (long long)P.nwt * (c + 1) / grid;
    for (long long w = a; w < b; ++w) P.wt.push_back(real[(size_t)w]);
    // pad the CTA's list to whole groups with empty descriptors that continue the entry range
    const int4 last = real[(size_t)(b - 1)];
    while (P.wt.size() % SPMV3_NCW != 0) {
      int4 t;
      t.x = last.x + last.w;
      t.y = last.y + last.z;
      t.z = 0;
      t.w = 0;
      P.wt.push_back(t);
    }
    P.cta_begin[(size_t)c + 1] = (int)(P.wt.size() / SPMV3_NCW);
  }
}

// C view of a plan for the tests (host memory, owned by the handle): the stream of a CSR as the device builder fills it
// (k_stored_len and the scan, spmv3_fill_row), and what spmv3_finish computes from its stored row pointers
struct B200Spmv3PlanHost {
  Spmv3Plan plan;
  std::vector<int> idx;
  std::vector<double> vals;
};
extern "C" B200Spmv3PlanHost *b200_spmv3_plan_build(int nrows, int ncols, const int *rp, const int *ci,
                                                    const double *va, int grid_cap) {
  if (nrows <= 0 || ncols >= (1 << 30)) return nullptr;
  B200Spmv3PlanHost *h = new B200Spmv3PlanHost();
  Spmv3Plan &P = h->plan;
  P.rowptr.resize((size_t)nrows + 1);
  long long stored = 0;
  for (int r = 0; r < nrows; ++r) {
    P.rowptr[r] = (int)stored;
    stored += rp[r + 1] > rp[r] ? rp[r + 1] - rp[r] : 1;
  }
  if (!spmv3_fits(stored)) {
    delete h;
    return nullptr;
  }
  P.rowptr[nrows] = (int)stored;
  h->idx.resize((size_t)stored);
  h->vals.resize((size_t)stored);
  for (int r = 0; r < nrows; ++r)
    spmv3_fill_row(rp[r + 1] - rp[r], rp[r], P.rowptr[r], ci, va, h->idx.data(), h->vals.data());
  spmv3_virtual_rows(nrows, P);
  spmv3_tiles_from_rowptr(grid_cap, P);
  return h;
}
extern "C" void b200_spmv3_plan_free(B200Spmv3PlanHost *h) { delete h; }
extern "C" int b200_spmv3_plan_info(const B200Spmv3PlanHost *h, int *stored, int *nwt, int *ndesc, int *grid,
                                    int *ncw) {
  *stored = h->plan.rowptr.back();
  *nwt = h->plan.nwt;
  *ndesc = (int)h->plan.wt.size();
  *grid = h->plan.grid;
  *ncw = SPMV3_NCW;
  return 0;
}
extern "C" const int *b200_spmv3_plan_rowptr(const B200Spmv3PlanHost *h) { return h->plan.rowptr.data(); }
extern "C" const int *b200_spmv3_plan_idx(const B200Spmv3PlanHost *h) { return h->idx.data(); }
extern "C" const double *b200_spmv3_plan_vals(const B200Spmv3PlanHost *h) { return h->vals.data(); }
extern "C" const int *b200_spmv3_plan_desc(const B200Spmv3PlanHost *h) {
  return reinterpret_cast<const int *>(h->plan.wt.data());
}
extern "C" const int *b200_spmv3_plan_cta_begin(const B200Spmv3PlanHost *h) { return h->plan.cta_begin.data(); }
extern "C" int b200_spmv3_plan_nvrows(const B200Spmv3PlanHost *h) { return h->plan.nvrows; }
extern "C" const int *b200_spmv3_plan_vptr(const B200Spmv3PlanHost *h) {
  return h->plan.vptr.empty() ? nullptr : h->plan.vptr.data();
}

// ------------------------------------------------------------------ device side
// once per process, whichever thread launches first (std::call_once: concurrent solves may race to it)
static void spmv_set_attrs_once() {
  const int bytes = (int)spmv3_smem_bytes();
  const cudaFuncAttribute at = cudaFuncAttributeMaxDynamicSharedMemorySize;
  cudaFuncSetAttribute(spmv_flag_kernel<B200_POST_NONE, false>, at, bytes);
  cudaFuncSetAttribute(spmv_flag_kernel<B200_POST_DIV, false>, at, bytes);
  cudaFuncSetAttribute(spmv_flag_kernel<B200_POST_MUL, false>, at, bytes);
  cudaFuncSetAttribute(spmv_flag_kernel<B200_POST_FMA_DOT, false>, at, bytes);
  cudaFuncSetAttribute(spmv_flag_kernel<B200_POST_FMA, false>, at, bytes);
  // the packed index stream serves the CG loop's operators only: K1, K2 and the warm start's K2
  cudaFuncSetAttribute(spmv_flag_kernel<B200_POST_MUL, true>, at, bytes);
  cudaFuncSetAttribute(spmv_flag_kernel<B200_POST_FMA_DOT, true>, at, bytes);
  cudaFuncSetAttribute(spmv_flag_kernel<B200_POST_FMA, true>, at, bytes);
}
static void spmv_set_attrs() {
  static std::once_flag once;
  std::call_once(once, spmv_set_attrs_once);
}

// Last step of every builder, once M's stream (d_rowptr / d_colidx / d_vals, `stored`) is in place: the warp-tiles and
// the CTA partition from P's (virtual) row pointers, uploaded with the virtual-row buffers, the reduction slots and the
// ticket counter. An operator without rows (a rank's row block when there are more ranks than rows) gets no warp-tiles:
// b200_spmv returns before any launch.
static int spmv3_finish(B200Spmv *M, Spmv3Plan &P) {
  int cap = SPMV3_CTAS_PER_SM * b200_num_sms();
  const char *g = getenv("SCS_B200_SPMV_GRID");  // tests: force many groups per CTA on small matrices
  if (g && atoi(g) > 0 && atoi(g) < cap) cap = atoi(g);
  if (P.nvrows > 0) spmv3_tiles_from_rowptr(cap, P);
  M->grid = P.grid;
  M->nvrows = P.nvrows;
  M->d_partials = (double *)b200_malloc((size_t)B200_MAX_PARTIALS * 8);
  M->d_counter = (unsigned int *)b200_malloc(64);
  if (!M->d_partials || !M->d_counter || b200_memset0(M->d_counter, 64) != 0) return -1;
  if (!P.wt.empty()) {
    M->d_wt3 = (int4 *)b200_malloc(P.wt.size() * sizeof(int4));
    M->d_cta_begin3 = (int *)b200_malloc(P.cta_begin.size() * 4);
    if (!M->d_wt3 || !M->d_cta_begin3 || b200_h2d(M->d_wt3, P.wt.data(), P.wt.size() * sizeof(int4)) != 0 ||
        b200_h2d(M->d_cta_begin3, P.cta_begin.data(), P.cta_begin.size() * 4) != 0)
      return -1;
  }
  if (!P.vptr.empty()) {  // long-row mode
    M->d_vptr = (int *)b200_malloc(P.vptr.size() * 4);
    M->d_vscratch = (double *)b200_malloc((size_t)P.nvrows * 8);
    if (!M->d_vptr || !M->d_vscratch || b200_h2d(M->d_vptr, P.vptr.data(), P.vptr.size() * 4) != 0) return -1;
  }
  // the plan's host vectors go out of scope
  if (b200_sync() != 0 || cudaGetLastError() != cudaSuccess) return -1;
  spmv_set_attrs();
  return 0;
}

// ---------------------------------------------------------------------------------------------
// Construction of a flagged-stream operator from a CSR in HBM, the one builder of every operator (A and A' by
// kernels/setup.cu, P by b200_sym_build there, the tests' host CSRs through b200_spmv_create): stored row pointers (every row >= 1 entry) by a
// scan, the flagged stream by one fill kernel; only the row pointers travel back to the host for the (sequential,
// O(rows)) virtual-row and warp-tile passes. Returns NULL on failure, with the reason in b200_last_error().
__global__ void k_stored_len(int nrows, const int *__restrict__ rp, int *__restrict__ out) {
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < nrows; r += gridDim.x * blockDim.x) {
    const int len = rp[r + 1] - rp[r];
    out[r] = len > 0 ? len : 1;
  }
}
__global__ void k_fill_flagged(int nrows, const int *__restrict__ rp, const int *__restrict__ sp,
                               const int *__restrict__ ci, const double *__restrict__ va, int *__restrict__ oi,
                               double *__restrict__ ov) {
  // one lane per row (spmv3_fill_row)
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int r0 = warp * 32; r0 < nrows; r0 += nwarps * 32) {
    const int r = r0 + lane;
    if (r < nrows) {
      const int a = rp[r], len = rp[r + 1] - a, pos = sp[r];
      spmv3_fill_row(len, a, pos, ci, va, oi, ov);
    }
  }
}
extern "C" int b200_dev_exclusive_scan_int(const int *d_in, int *d_out, int count);  // kernels/setup.cu (CUB)

extern "C" B200Spmv *b200_spmv_create_dev(int nrows, int ncols, long long nnz, const int *d_rp, const int *d_ci,
                                          const double *d_va) {
  if (b200_runtime_init() != 0) return nullptr;
  if (nrows < 0 || ncols < 0 || ncols >= (1 << 30) || nrows >= (1 << 30)) {
    // bits 30/31 of the stored column indices are flags; every reader masks them
    b200_set_error("b200_spmv_create_dev: dimensions must lie in [0, 2^30)", cudaErrorInvalidValue, __FILE__,
                   __LINE__);
    return nullptr;
  }
  cudaStream_t st = (cudaStream_t)b200_stream();
  B200Spmv *M = (B200Spmv *)calloc(1, sizeof(B200Spmv));
  if (!M) return nullptr;
  M->nrows = nrows; M->ncols = ncols; M->nnz = nnz;
  int *d_len = (int *)b200_malloc((size_t)(nrows + 1) * 4);
  M->d_rowptr = (int *)b200_malloc((size_t)(nrows + 1 + 8) * 4);
  Spmv3Plan P;
  P.rowptr.resize((size_t)nrows + 1);
  bool ok = d_len && M->d_rowptr && b200_memset0(M->d_rowptr, (size_t)(nrows + 1 + 8) * 4) == 0 &&
            b200_memset0(d_len + nrows, 4) == 0;
  if (ok) {
    int g = (nrows + 255) / 256;
    if (g > 8 * b200_num_sms()) g = 8 * b200_num_sms();
    if (g > 0) k_stored_len<<<g, 256, 0, st>>>(nrows, d_rp, d_len);
    // exclusive scan over nrows + 1 items: element nrows receives the total
    ok = b200_dev_exclusive_scan_int(d_len, M->d_rowptr, nrows + 1) == 0 &&
         b200_d2h(P.rowptr.data(), M->d_rowptr, (size_t)(nrows + 1) * 4) == 0 && b200_sync() == 0;
    b200_count_launch(g > 0 ? 2 : 1);
  }
  // the int scan wraps a total of 2^31 or more; read as unsigned it is exact, since int row pointers (nnz < 2^31) and
  // nrows < 2^30 keep it below 2^32, and spmv3_fits rejects it
  const long long stored = ok ? (long long)(unsigned)P.rowptr[(size_t)nrows] : 0;
  ok = ok && spmv3_fits(stored);
  if (ok) {
    const size_t pad = (((size_t)stored + 3) & ~(size_t)3) + 8;
    M->stored = stored;
    M->d_colidx = (int *)b200_malloc(pad * 4);
    M->d_vals = (double *)b200_malloc(pad * 8);
    ok = M->d_colidx && M->d_vals && b200_memset0(M->d_colidx, pad * 4) == 0 && b200_memset0(M->d_vals, pad * 8) == 0;
    int g = (nrows + 255) / 256;
    if (g > 16 * b200_num_sms()) g = 16 * b200_num_sms();
    if (ok && g > 0) {
      k_fill_flagged<<<g, 256, 0, st>>>(nrows, d_rp, M->d_rowptr, d_ci, d_va, M->d_colidx, M->d_vals);
      b200_count_launch(1);
    }
  }
  if (ok) spmv3_virtual_rows(nrows, P);  // sequential O(rows) host pass, overlaps the fill kernel
  ok = ok && spmv3_finish(M, P) == 0;
  b200_free(d_len);
  if (!ok) {
    b200_spmv_destroy(M);
    return nullptr;
  }
  return M;
}

// an operator from a host CSR (the tests only): uploaded, then built on the device like every other
extern "C" B200Spmv *b200_spmv_create(int nrows, int ncols, const int *h_rowptr, const int *h_colidx,
                                      const double *h_vals) {
  if (b200_runtime_init() != 0) return nullptr;
  const long long nnz = h_rowptr[nrows];
  int *d_rp = (int *)b200_malloc((size_t)(nrows + 1) * 4), *d_ci = (int *)b200_malloc((size_t)nnz * 4);
  double *d_va = (double *)b200_malloc((size_t)nnz * 8);
  B200Spmv *M = nullptr;
  if (d_rp && d_ci && d_va && b200_h2d(d_rp, h_rowptr, (size_t)(nrows + 1) * 4) == 0 &&
      b200_h2d(d_ci, h_colidx, (size_t)nnz * 4) == 0 && b200_h2d(d_va, h_vals, (size_t)nnz * 8) == 0)
    M = b200_spmv_create_dev(nrows, ncols, nnz, d_rp, d_ci, d_va);
  // stream-ordered: the builder's kernels read the uploads before the blocks are handed out again
  b200_free(d_rp); b200_free(d_ci); b200_free(d_va);
  return M;
}

// ---------------------------------------------------------------------------------------------
// New values on the same pattern (scs_b200_update_matrix_device). The stream of an operator built from a CSR (rp, ci)
// holds entry k of row r at sp[r] + (k - rp[r]), sp = its stored row pointers: the fill (spmv3_fill_row) writes a row's
// entries in order from sp[r], a row cut into pieces only gets extra END flags, and an empty row is one SKIP | END
// entry. So a CSR has the operator's pattern if and only if every row has that stored length (an empty row: one SKIP
// entry) and every entry's masked column at its position is the CSR's column and not SKIP. The rows of an entry come
// from a bisection of rp (validated: nondecreasing, rp[0] = 0, rp[nrows] = nnz = the operator's nnz), so every
// position read lies inside its row's stored range.
__device__ __forceinline__ int csr_row_of(int nrows, const int *__restrict__ rp, long long k) {
  int lo = 0, hi = nrows;  // the last row r with rp[r] <= k
  while (hi - lo > 1) {
    const int mid = lo + (hi - lo) / 2;
    if (rp[mid] <= k) lo = mid; else hi = mid;
  }
  return lo;
}
__global__ void k_check_pattern(int nrows, long long nnz, const int *__restrict__ rp, const int *__restrict__ ci,
                                const int *__restrict__ sp, const int *__restrict__ oi, unsigned bit,
                                unsigned *__restrict__ d_bad) {
  const long long work = nnz > nrows ? nnz : nrows, stride = (long long)gridDim.x * blockDim.x;
  bool diff = false;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < work; t += stride) {
    if (t < nrows) {
      const int r = (int)t, len = rp[r + 1] - rp[r], slen = sp[r + 1] - sp[r];
      diff |= len == 0 ? slen != 1 || !((unsigned)oi[sp[r]] & B200_FLAG_SKIP) : slen != len;
    }
    if (t < nnz) {
      const int r = csr_row_of(nrows, rp, t);
      const int off = (int)(t - rp[r]);
      if (off < sp[r + 1] - sp[r]) {
        const unsigned v = (unsigned)oi[sp[r] + off];
        diff |= (v & B200_FLAG_SKIP) != 0 || (int)(v & B200_COLMASK) != ci[t];
      } else {
        diff = true;
      }
    }
  }
  if (diff) atomicOr(d_bad, bit);
}
__global__ void k_scatter_values(int nrows, long long nnz, const int *__restrict__ rp, const double *__restrict__ va,
                                 const int *__restrict__ sp, double *__restrict__ ov) {
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < nnz; t += (long long)gridDim.x * blockDim.x) {
    const int r = csr_row_of(nrows, rp, t);
    ov[sp[r] + (t - rp[r])] = va[t];
  }
}
static int entry_grid(long long work) {
  const long long g = (work + 255) / 256, cap = 8LL * b200_num_sms();
  return (int)(g < 1 ? 1 : g > cap ? cap : g);
}
// ORs `bit` into *d_bad (device) unless the CSR (d_rp, d_ci: nrows = M's rows, nnz entries) has M's pattern; enqueued
// only. M must keep its int32 index stream (A, A' and P do; the CG loop's packed copies do not).
extern "C" int b200_spmv_check_pattern(const B200Spmv *M, const int *d_rp, const int *d_ci, long long nnz, unsigned bit,
                                       unsigned *d_bad) {
  cudaStream_t st = (cudaStream_t)b200_stream();
  if (M->d_colidx == nullptr || M->d_rowptr == nullptr || nnz != M->nnz) {
    b200_set_error("b200_spmv_check_pattern: the operator has no int32 index stream or another nnz",
                   cudaErrorInvalidValue, __FILE__, __LINE__);
    return -1;
  }
  const long long work = nnz > M->nrows ? nnz : M->nrows;
  if (work > 0) {
    k_check_pattern<<<entry_grid(work), 256, 0, st>>>(M->nrows, nnz, d_rp, d_ci, M->d_rowptr, M->d_colidx, bit, d_bad);
    b200_count_launch(1);
  }
  CUDA_OK(cudaGetLastError());
  return 0;
}
// the values of the CSR (d_rp, d_va) into M's stream at the positions above, after a clean b200_spmv_check_pattern;
// M's explicit zeros (empty rows) keep their 0.0
extern "C" int b200_spmv_scatter_values(B200Spmv *M, const int *d_rp, const double *d_va) {
  if (M->nnz > 0) {
    k_scatter_values<<<entry_grid(M->nnz), 256, 0, (cudaStream_t)b200_stream()>>>(M->nrows, M->nnz, d_rp, d_va,
                                                                                  M->d_rowptr, M->d_vals);
    b200_count_launch(1);
  }
  CUDA_OK(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------------------------
// Reordered copies for the CG operator (DESIGN.md section 3.1 "Reordering").
// The m-space ordering INSIDE G = R_x + A' R_y^-1 A is free (tmp = R_y^-1 A p never leaves the operator), so the rows
// of A can be sorted by their smallest column index: one gather per row of K1 becomes sequential, and the matching
// entries of every column of A' become adjacent for K2.
//   b200_spmv_permuted_rows : row-permuted copy of the first `nrows` rows of the permutation of a flagged-stream
//                             operator (row `new` = row perm[new] of M); segments are copied with their flags, the
//                             warp-tiles are recomputed. Rows left out are never written (the caller leaves out
//                             empty rows only, so the entry count stays M's). Every row is placed where the kernel
//                             sums it as in M, so the copy computes bit-for-bit the row sums M computes (see below).
//                             The placement reorders rows slightly: the final order is written back to perm, and inv
//                             is computed from it;
//   b200_spmv_refresh_permuted : values only (after the resident operators were rescaled in place);
//   b200_spmv_renumbered_cols  : a VIEW of M whose stored column indices are mapped through inv[] (flags kept);
//                             row pointers, values and warp-tiles are M's own (borrowed, not copied).
//
// Lane split. The flag kernel sums a row inside one lane sequentially and combines the pieces of a row that spans lanes
// with a scan whose tree depends only on the pieces (lanes own the entries [4l, 4l+4) of the 16-byte-aligned stream;
// a leading lane that holds only explicit zeros adds exact zeros). The pieces are set by the position of the row's
// first entry modulo 4 (its phase) and its length, and spmv3_same_sum_phases gives the phases at which a row sums as it
// does in M: any phase where it is still one plain sequential chain if it is one in M, else its phase in M.
// b200_spmv_place_rows lays the rows out in their sorted order, except that at every position it takes the earliest
// of the next SPMV3_PLACE_WINDOW rows that may start there. Only when none may, up to 3 explicit zeros (SKIP, no END)
// lead a row's segment to a phase it may take. On C2-shaped matrices the zeros are 0.14 % of nnz (a window of 16: 0.9 %,
// 64: 0.01 %; keeping every row's lane pieces as in M took 30 %), and a row's smallest column moves by 0.75 columns on
// average. With the row sums equal, the CG operator computes what the plain pair computes, only faster.
#define SPMV3_PLACE_WINDOW 32

// Pure host code, exported with the phase masks for the CPU tests (tests/test_spmv_place_rows_cpu.py). sp_old: M's
// stored row pointers; perm[0..nrows): rows of M in sorted order, every one non-empty and at most SPMV3_MAXROW long. On
// return perm[0..nrows) holds the rows in the order they are laid out, each less than SPMV3_PLACE_WINDOW slots from
// where it came in, and sp_new[0..nrows] the copy's stored row pointers (a segment is its leading zeros, then the row's
// entries). Returns the copy's stored count; sp_new is valid only if that passes spmv3_fits. The result depends only
// on sp_old and the incoming perm.
extern "C" long long b200_spmv_place_rows(int nrows, const int *sp_old, int *perm, int *sp_new) {
  // The pending rows live in a ring indexed by slot % 64, with one bit mask per phase of the rows that may start there.
  // A row is placed at the latest when it is SPMV3_PLACE_WINDOW - 1 slots late, so the pending slots span less than
  // 2 * SPMV3_PLACE_WINDOW. Selecting by bit scans instead of walking a list keeps the loop nearly free of branches
  // that depend on the data: at C2 size it runs in a few tens of ms.
  static_assert(2 * SPMV3_PLACE_WINDOW <= 64, "the pending rows must fit a 64-slot ring");
  // length and phase in M of every row in sorted order, first: independent random reads of sp_old that overlap
  std::vector<int> lp((size_t)nrows);
  for (int i = 0; i < nrows; ++i) lp[(size_t)i] = (sp_old[perm[i] + 1] - sp_old[perm[i]]) << 2 | (sp_old[perm[i]] & 3);
  int ring_row[64], ring_len[64];
  unsigned char ring_mask[64];
  unsigned long long adm[4] = {0, 0, 0, 0};  // bit slot % 64: that pending row may start at phase q
  unsigned long long longm = 0;  // rows of more than SPMV3_WT - 6 entries: leading zeros may not fit their warp-tile
  auto rotr = [](unsigned long long v, int s) { return (v >> s) | (v << ((64 - s) & 63)); };
  int pending = 0, next = 0, s0 = 0;  // s0: the oldest pending slot
  long long pos = 0;
  for (int t = 0; t < nrows; ++t) {
    // perm[t] is overwritten below: every slot up to t + SPMV3_PLACE_WINDOW - 1 has been read by then
    for (; pending < SPMV3_PLACE_WINDOW && next < nrows; ++next, ++pending) {
      const int len = lp[(size_t)next] >> 2, b = next & 63;
      const unsigned m = spmv3_same_sum_phases(len, lp[(size_t)next] & 3);
      ring_row[b] = perm[next];
      ring_len[b] = len;
      ring_mask[b] = (unsigned char)m;
      for (int q = 0; q < 4; ++q) adm[q] |= (unsigned long long)(m >> q & 1u) << b;
      longm |= (unsigned long long)(len > SPMV3_WT - 6) << b;
    }
    const int c = (int)(pos & 3), sh = s0 & 63;
    int slot = -1, lead = 0;
    if (t - s0 < SPMV3_PLACE_WINDOW - 1) {
      // the earliest row that may start at c; else the earliest with the fewest leading zeros
      unsigned long long r = rotr(adm[c], sh);
      if (r) slot = s0 + __builtin_ctzll(r);
      for (int z = 1; slot < 0 && z < 4; ++z) {
        r = rotr(adm[(c + z) & 3] & ~longm, sh);
        if (r) { slot = s0 + __builtin_ctzll(r); lead = z; }
      }
    }
    if (slot < 0) {
      // the oldest row is due (or only long rows are pending): it goes now, with the zeros it needs unless they would
      // push its segment out of one warp-tile
      slot = s0;
      while (!(ring_mask[s0 & 63] >> ((c + lead) & 3) & 1u)) ++lead;
      if (c + lead + ring_len[s0 & 63] > SPMV3_WT) lead = 0;
    }
    const int b = slot & 63;
    const unsigned long long keep = ~(1ull << b);
    for (int q = 0; q < 4; ++q) adm[q] &= keep;
    longm &= keep;
    --pending;
    perm[t] = ring_row[b];
    sp_new[t] = (int)pos;
    pos += lead + ring_len[b];
    const unsigned long long left = adm[0] | adm[1] | adm[2] | adm[3];  // every row may start at some phase
    if (left) s0 += __builtin_ctzll(rotr(left, s0 & 63));
  }
  sp_new[nrows] = (int)pos;
  return pos;
}
extern "C" unsigned b200_spmv3_phase_mask(int len, int phase) { return spmv3_same_sum_phases(len, phase); }
// the packed index format, exported for the CPU tests (tests/test_spmv_packed_cpu.py)
extern "C" unsigned b200_spmv3_idx24_encode(int v) { return spmv3_idx24_encode(v); }
extern "C" int b200_spmv3_idx24_decode(unsigned e) { return spmv3_idx24_decode(e); }
extern "C" unsigned b200_spmv3_idx24_slice_bytes(int ka, int cnt) { return spmv3_idx24_slice_bytes(ka, cnt); }

__global__ void k_fill_skip(long long count, int *__restrict__ oi) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < count; k += (long long)gridDim.x * blockDim.x)
    oi[k] = (int)B200_FLAG_SKIP;
}
__global__ void k_perm_copy(int nrows, const int *__restrict__ sp_old, const int *__restrict__ sp_new,
                            const int *__restrict__ perm, const int *__restrict__ ci, const double *__restrict__ va,
                            int *__restrict__ oi, double *__restrict__ ov) {
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < nrows; r += gridDim.x * blockDim.x) {
    const int o = perm[r];
    const int a = sp_old[o], len = sp_old[o + 1] - a;
    const int b = sp_new[r + 1] - len;  // the entries close the segment; explicit zeros lead it
    for (int k = 0; k < len; ++k) {
      if (oi != nullptr) oi[b + k] = ci[a + k];
      ov[b + k] = va[a + k];
    }
  }
}
__global__ void k_renumber_cols(long long stored, const int *__restrict__ ci, const int *__restrict__ inv,
                                int *__restrict__ out) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < stored; k += (long long)gridDim.x * blockDim.x) {
    const unsigned v = (unsigned)ci[k];
    out[k] = (v & B200_FLAG_SKIP) ? (int)v : (int)((unsigned)inv[v & B200_COLMASK] | (v & B200_FLAG_END));
  }
}

__global__ void k_invert_perm(int n, const int *__restrict__ perm, int *__restrict__ inv) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) inv[perm[i]] = i;
}

extern "C" B200Spmv *b200_spmv_permuted_rows(const B200Spmv *S, int *d_perm, int *d_inv, int nrows) {
  if (!S || S->d_vptr != nullptr || nrows <= 0 || nrows > S->nrows) return nullptr;
  cudaStream_t st = (cudaStream_t)b200_stream();
  B200Spmv *M = (B200Spmv *)calloc(1, sizeof(B200Spmv));
  if (!M) return nullptr;
  M->nrows = nrows; M->ncols = S->ncols; M->nnz = S->nnz;
  // placement on the host (sequential, O(rows)): stored row pointers of S and the sorted rows come back once, the
  // placed order goes up before anything reads d_perm
  std::vector<int> h_old((size_t)S->nrows + 1), h_perm((size_t)nrows);
  Spmv3Plan P;
  P.rowptr.resize((size_t)nrows + 1);
  // no virtual rows: S cuts no row, and with its leading zeros a row's segment still fits one warp-tile
  P.nvrows = nrows;
  bool ok = b200_d2h(h_old.data(), S->d_rowptr, h_old.size() * 4) == 0 &&
            b200_d2h(h_perm.data(), d_perm, h_perm.size() * 4) == 0 && b200_sync() == 0;
  const long long pos = ok ? b200_spmv_place_rows(nrows, h_old.data(), h_perm.data(), P.rowptr.data()) : 0;
  ok = ok && spmv3_fits(pos) && b200_h2d(d_perm, h_perm.data(), h_perm.size() * 4) == 0;
  if (ok) {
    k_invert_perm<<<8 * b200_num_sms(), 256, 0, st>>>(S->nrows, d_perm, d_inv);
    b200_count_launch(1);
  }
  if (ok) {
    const size_t pad = (((size_t)pos + 3) & ~(size_t)3) + 8;
    M->stored = pos;
    M->d_rowptr = (int *)b200_malloc((size_t)(nrows + 1 + 8) * 4);
    M->d_colidx = (int *)b200_malloc(pad * 4);
    M->d_vals = (double *)b200_malloc(pad * 8);
    ok = M->d_rowptr && M->d_colidx && M->d_vals && b200_memset0(M->d_rowptr, (size_t)(nrows + 1 + 8) * 4) == 0 &&
         b200_memset0(M->d_vals, pad * 8) == 0 && b200_h2d(M->d_rowptr, P.rowptr.data(), P.rowptr.size() * 4) == 0;
    if (ok) {
      int g = (nrows + 255) / 256;
      if (g > 16 * b200_num_sms()) g = 16 * b200_num_sms();
      k_fill_skip<<<8 * b200_num_sms(), 256, 0, st>>>((long long)pad, M->d_colidx);
      k_perm_copy<<<g, 256, 0, st>>>(nrows, S->d_rowptr, M->d_rowptr, d_perm, S->d_colidx, S->d_vals, M->d_colidx,
                                     M->d_vals);
      b200_count_launch(2);
    }
  }
  ok = ok && spmv3_finish(M, P) == 0;
  if (!ok) {
    b200_spmv_destroy(M);
    return nullptr;
  }
  return M;
}
extern "C" int b200_spmv_refresh_permuted(B200Spmv *M, const B200Spmv *S, const int *d_perm) {
  cudaStream_t st = (cudaStream_t)b200_stream();
  int g = (M->nrows + 255) / 256;
  if (g > 16 * b200_num_sms()) g = 16 * b200_num_sms();
  k_perm_copy<<<g, 256, 0, st>>>(M->nrows, S->d_rowptr, M->d_rowptr, d_perm, nullptr, S->d_vals, nullptr, M->d_vals);
  b200_count_launch(1);
  CUDA_OK(cudaGetLastError());
  return 0;
}
extern "C" B200Spmv *b200_spmv_renumbered_cols(const B200Spmv *S, const int *d_inv) {
  if (!S || S->d_vptr != nullptr) return nullptr;
  cudaStream_t st = (cudaStream_t)b200_stream();
  B200Spmv *M = (B200Spmv *)calloc(1, sizeof(B200Spmv));
  if (!M) return nullptr;
  *M = *S;
  M->borrows = 1;
  const size_t pad = (((size_t)S->stored + 3) & ~(size_t)3) + 8;
  M->d_colidx = (int *)b200_malloc(pad * 4);
  M->d_partials = (double *)b200_malloc((size_t)B200_MAX_PARTIALS * 8);
  M->d_counter = (unsigned int *)b200_malloc(64);
  bool ok = M->d_colidx && M->d_partials && M->d_counter && b200_memset0(M->d_colidx, pad * 4) == 0 &&
            b200_memset0(M->d_counter, 64) == 0;
  if (ok) {
    k_renumber_cols<<<8 * b200_num_sms(), 256, 0, st>>>(S->stored, S->d_colidx, d_inv, M->d_colidx);
    b200_count_launch(1);
    ok = cudaGetLastError() == cudaSuccess && b200_sync() == 0;
  }
  if (!ok) {
    b200_spmv_destroy(M);
    return nullptr;
  }
  return M;
}

// The CG loop's operators stream their column indices packed when they have at most 2^22 columns (3 bytes per entry
// instead of 4): packed on the device, then the int32 stream is freed. Only the flag kernel reads the packed stream;
// b200_spmv_colidx of such an operator is NULL.
__global__ void k_pack_idx24(long long count, const int *__restrict__ ci, unsigned char *__restrict__ out) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < count; k += (long long)gridDim.x * blockDim.x) {
    const unsigned e = spmv3_idx24_encode(ci[k]);
    out[3 * k] = (unsigned char)e;
    out[3 * k + 1] = (unsigned char)(e >> 8);
    out[3 * k + 2] = (unsigned char)(e >> 16);
  }
}
extern "C" int b200_spmv_pack_indices(B200Spmv *M) {
  if (M->ncols > SPMV3_IDX24_MAXCOLS || M->d_idx24 != nullptr || M->d_vptr != nullptr) return 0;
  cudaStream_t st = (cudaStream_t)b200_stream();
  // the int32 stream's padded length; the last bulk copy reads up to 15 bytes past its rounded end
  const size_t pad = (((size_t)M->stored + 3) & ~(size_t)3) + 8;
  unsigned char *p = (unsigned char *)b200_malloc(3 * pad + 16);
  if (!p || b200_memset0(p + 3 * pad, 16) != 0) {
    b200_free(p);
    return -1;
  }
  k_pack_idx24<<<8 * b200_num_sms(), 256, 0, st>>>((long long)pad, M->d_colidx, p);
  b200_count_launch(1);
  if (cudaGetLastError() != cudaSuccess || b200_sync() != 0) {
    b200_free(p);
    return -1;
  }
  b200_free(M->d_colidx);
  M->d_colidx = nullptr;
  M->d_idx24 = p;
  return 0;
}

extern "C" void b200_spmv_destroy(B200Spmv *M) {
  if (!M) return;
  if (M->borrows) {  // a view: only the column indices, the reduction slots and the ticket counter are its own
    b200_free(M->d_colidx);
    b200_free(M->d_idx24);
    b200_free(M->d_partials);
    b200_free(M->d_counter);
    free(M);
    return;
  }
  b200_free(M->d_rowptr);
  b200_free(M->d_colidx);
  b200_free(M->d_idx24);
  b200_free(M->d_vals);
  b200_free(M->d_partials);
  b200_free(M->d_counter);
  b200_free(M->d_wt3);
  b200_free(M->d_cta_begin3);
  b200_free(M->d_vptr);
  b200_free(M->d_vscratch);
  free(M);
}

extern "C" int b200_spmv_nrows(const B200Spmv *M) { return M->nrows; }
extern "C" int b200_spmv_ncols(const B200Spmv *M) { return M->ncols; }
extern "C" long long b200_spmv_nnz(const B200Spmv *M) { return M->nnz; }
extern "C" const double *b200_spmv_vals(const B200Spmv *M) { return M->d_vals; }
extern "C" const int *b200_spmv_colidx(const B200Spmv *M) { return M->d_colidx; }
extern "C" const int *b200_spmv_rowptr(const B200Spmv *M) { return M->d_rowptr; }
extern "C" double b200_spmv_alg_bytes(const B200Spmv *M, int extra_row_vectors) {
  return b200_spmv_entry_bytes(M) * (double)M->nnz + 4.0 * (M->nrows + 1.0) + 8.0 * M->ncols +
         8.0 * M->nrows * (1.0 + extra_row_vectors);
}
extern "C" int b200_spmv_entry_bytes(const B200Spmv *M) { return M->d_idx24 != nullptr ? 11 : 12; }

extern "C" int b200_spmv(const B200Spmv *M, const B200SpmvArgs *a) {
  if (M->nrows == 0) return 0;
  cudaStream_t st = (cudaStream_t)b200_stream();
  const size_t smem = spmv3_smem_bytes();
  dim3 grid(M->grid), block(SPMV3_THREADS);
  if (a->hook == B200_HOOK_P2P_ROUTE && !(b200_spmv_can_route(M) && a->post == B200_POST_NONE)) {
    b200_set_error("b200_spmv: B200_HOOK_P2P_ROUTE needs the one-pass flagged-stream kernel with POST_NONE",
                   cudaErrorInvalidValue, __FILE__, __LINE__);
    return -1;
  }
  if (a->dform != B200_D_VEC && a->post != B200_POST_NONE && !b200_spmv_can_route(M)) {
    b200_set_error("b200_spmv: the table forms of d need the one-pass flagged-stream kernel", cudaErrorInvalidValue,
                   __FILE__, __LINE__);
    return -1;
  }
  if (M->d_vptr != nullptr) {
    // long-row mode: sums per virtual row, then the combine pass with the real epilogue
    spmv_flag_kernel<B200_POST_NONE, false><<<grid, block, smem, st>>>(
        M->d_colidx, M->d_vals, M->d_wt3, M->d_cta_begin3, a->d_x, M->d_vscratch, nullptr, 1.0, nullptr, nullptr,
        B200_D_VEC, nullptr, nullptr, B200_HOOK_NONE, nullptr, a->d_skip, M->d_partials, M->d_counter, 0ull);
    int cg = (M->nrows + 255) / 256;
    const int cap = 8 * b200_num_sms();
    if (cg > cap) cg = cap;
#define COMBINE(POSTV)                                                                                        \
  spmv_combine_kernel<POSTV><<<cg, 256, 0, st>>>(M->nrows, M->d_vptr, M->d_vscratch, a->d_y, a->d_init,      \
                                                 a->init_sign, a->d_d, a->d_v, a->d_dot, a->hook, a->d_hook_arg, \
                                                 a->d_skip, M->d_partials, M->d_counter, a->hook_val)
    switch (a->post) {
      case B200_POST_NONE: COMBINE(B200_POST_NONE); break;
      case B200_POST_DIV: COMBINE(B200_POST_DIV); break;
      case B200_POST_MUL: COMBINE(B200_POST_MUL); break;
      case B200_POST_FMA_DOT: COMBINE(B200_POST_FMA_DOT); break;
      case B200_POST_FMA: COMBINE(B200_POST_FMA); break;
      default: return -1;
    }
#undef COMBINE
    b200_count_launch(2);
    CUDA_OK(cudaGetLastError());
    return 0;
  }
  if (M->d_idx24 != nullptr && a->post != B200_POST_MUL && a->post != B200_POST_FMA_DOT && a->post != B200_POST_FMA) {
    b200_set_error("b200_spmv: an operator with a packed index stream takes POST_MUL / POST_FMA_DOT / POST_FMA only",
                   cudaErrorInvalidValue, __FILE__, __LINE__);
    return -1;
  }
  const void *idx = M->d_idx24 != nullptr ? (const void *)M->d_idx24 : (const void *)M->d_colidx;
#define LAUNCH_IDX(POSTV, PACKED)                                                                              \
  CUDA_OK(b200_launch(spmv_flag_kernel<POSTV, PACKED>, grid, block, smem, st, a->pdl != 0, idx,               \
                      (const double *)M->d_vals, (const int4 *)M->d_wt3, (const int *)M->d_cta_begin3, a->d_x, \
                      a->d_y, a->d_init, a->init_sign, a->d_d, a->d_dmask, a->dform, a->d_v, a->d_dot, a->hook, \
                      a->d_hook_arg,                                                                             \
                      a->d_skip, M->d_partials, M->d_counter, a->hook_val))
#define LAUNCH(POSTV)                 \
  if (M->d_idx24 != nullptr)          \
    LAUNCH_IDX(POSTV, true);          \
  else                                \
    LAUNCH_IDX(POSTV, false)
  switch (a->post) {
    case B200_POST_NONE: LAUNCH_IDX(B200_POST_NONE, false); break;
    case B200_POST_DIV: LAUNCH_IDX(B200_POST_DIV, false); break;
    case B200_POST_MUL: LAUNCH(B200_POST_MUL); break;
    case B200_POST_FMA_DOT: LAUNCH(B200_POST_FMA_DOT); break;
    case B200_POST_FMA: LAUNCH(B200_POST_FMA); break;
    default: return -1;
  }
#undef LAUNCH
#undef LAUNCH_IDX
  b200_count_launch(1);
  CUDA_OK(cudaGetLastError());
  return 0;
}
extern "C" int b200_spmv_flag_view(const B200Spmv *M, B200FlagView *out) {
  if (!b200_spmv_can_route(M)) return -1;
  out->idx = M->d_idx24 != nullptr ? (const void *)M->d_idx24 : (const void *)M->d_colidx;
  out->vals = M->d_vals;
  out->wt = M->d_wt3;
  out->cta_begin = M->d_cta_begin3;
  out->grid = M->grid;
  out->packed = M->d_idx24 != nullptr ? 1 : 0;
  out->partials = M->d_partials;
  out->counter = M->d_counter;
  return 0;
}
// B200_HOOK_P2P_ROUTE needs the one-pass kernel (no virtual rows / combine pass)
extern "C" int b200_spmv_can_route(const B200Spmv *M) { return M && M->nrows > 0 && M->d_vptr == nullptr; }
extern "C" long long b200_spmv_stored(const B200Spmv *M) { return M->stored; }

// Alternating launches of two operators (A then A'), every launch bracketed by its own CUDA
// events on the library stream: the other operator's matrix stream evicts this one's from L2,
// as in the CG loop. out_ms[0], out_ms[1] = average duration per launch of M0, M1.
extern "C" int b200_spmv_time_pair(const B200Spmv *M0, const B200Spmv *M1, int reps, double *out_ms) {
  cudaStream_t st = (cudaStream_t)b200_stream();
  const B200Spmv *Ms[2] = {M0, M1};
  double *d_x[2] = {nullptr, nullptr}, *d_y[2] = {nullptr, nullptr};
  std::vector<cudaEvent_t> ev((size_t)reps * 4);
  int rc = -1;
  for (auto &e : ev) e = nullptr;
  for (int k = 0; k < 2; ++k) {
    d_x[k] = (double *)b200_malloc((size_t)Ms[k]->ncols * 8);
    d_y[k] = (double *)b200_malloc((size_t)Ms[k]->nrows * 8);
    if (!d_x[k] || !d_y[k]) goto out;
    std::vector<double> hx((size_t)Ms[k]->ncols);
    for (size_t i = 0; i < hx.size(); ++i) hx[i] = 1.0 + 1e-3 * (double)(i % 1000);
    if (b200_h2d(d_x[k], hx.data(), hx.size() * 8) != 0) goto out;
  }
  for (auto &e : ev)
    if (cudaEventCreate(&e) != cudaSuccess) goto out;
  {
    B200SpmvArgs a[2];
    for (int k = 0; k < 2; ++k) {
      memset(&a[k], 0, sizeof(B200SpmvArgs));
      a[k].d_x = d_x[k]; a[k].d_y = d_y[k]; a[k].init_sign = 1.0; a[k].post = B200_POST_NONE;
    }
    for (int w = 0; w < 3; ++w)
      for (int k = 0; k < 2; ++k)
        if (b200_spmv(Ms[k], &a[k]) != 0) goto out;
    if (cudaStreamSynchronize(st) != cudaSuccess) goto out;
    for (int r = 0; r < reps; ++r)
      for (int k = 0; k < 2; ++k) {
        cudaEventRecord(ev[(size_t)r * 4 + 2 * k], st);
        if (b200_spmv(Ms[k], &a[k]) != 0) goto out;
        cudaEventRecord(ev[(size_t)r * 4 + 2 * k + 1], st);
      }
    if (cudaStreamSynchronize(st) != cudaSuccess) goto out;
    out_ms[0] = out_ms[1] = 0.0;
    for (int r = 0; r < reps; ++r)
      for (int k = 0; k < 2; ++k) {
        float ms = 0.f;
        cudaEventElapsedTime(&ms, ev[(size_t)r * 4 + 2 * k], ev[(size_t)r * 4 + 2 * k + 1]);
        out_ms[k] += ms;
      }
    out_ms[0] /= reps;
    out_ms[1] /= reps;
    rc = 0;
  }
out:
  for (auto &e : ev) if (e) cudaEventDestroy(e);
  for (int k = 0; k < 2; ++k) { b200_free(d_x[k]); b200_free(d_y[k]); }
  return rc;
}
