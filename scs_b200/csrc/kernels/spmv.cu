// spmv.cu -- fp64 / int32 sparse mat-vec for the SCS indirect KKT solve, sm_90a.
//
// Replaces reference linsys/scs_matrix.c:161-186 (accum_by_atrans, used for both
// A'x on the CSC arrays and A x on the explicit transpose) and the cuSPARSE
// calls of linsys/gpu/gpu.c:3-58.
//
// Two kernels:
//   * v3 "flagged stream" (spmv_flag_kernel, the default): nonzero-per-lane on a TMA ring, rows recovered from
//     END flags with ballots and a segmented warp scan -- see the block comment above the kernel. Rows longer
//     than a warp-tile are cut into "virtual rows" whose partial sums a second, tiny pass adds in order
//     (spmv_combine_kernel), so v3 serves every operator;
//   * v2 "warp-specialised row-per-lane" (spmv_ws_kernel): kept as the fallback for operators v3 cannot plan
//     (dimension / size limits) and for A/B measurements (SCS_B200_SPMV=2).
// Both: static CTA partition (no atomics => a launch is bit-reproducible), 1-D TMA bulk copies
// (cp.async.bulk, L2 evict_first) of the value / index slices into shared memory with mbarrier completion,
// products rounded separately from the adds (__dmul_rn / __dadd_rn: the reference's scalar loop
// `yj += Ax[p] * x[Ai[p]]` is not contracted to fma in the oracle build), fused epilogues
// y = s | s / d[r] | fma(d[r], v[r], s) plus the dot product v'y with a deterministic last-block reduction and
// an optional hook that turns the dot into the CG step length on the device.
//
// Algorithmic bytes per launch (DESIGN.md): 12*nnz + 4*(R+1) + 8*C + 8*R (+8*R per
// extra row vector read by the epilogue).
#include "../common.cuh"
#include "../dev_api.h"
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <thread>
#include <vector>

extern "C" int b200_host_threads(long long work_items);  // host/linsys_b200.c

// tuning knobs (overridable with -D for sweeps)
#ifndef SPMV_DEFAULT_VERSION
#define SPMV_DEFAULT_VERSION 3  // flagged stream (SCS_B200_SPMV=2 forces the warp-specialised row-per-lane kernel)
#endif
// tile descriptor: x=row0, y=nrows | (type<<28) | (lg_lanes<<24), z=k0, w=nnz
#define TILE_NORMAL 0
#define TILE_LONG_FIRST 1
#define TILE_LONG_MID 2
#define TILE_LONG_LAST 3
#define TILE_LONG_ONLY 4  // single chunk (cannot happen by construction, kept for safety)

struct B200Spmv {
  int nrows, ncols;
  long long nnz;
  int *d_rowptr;
  int *d_colidx;
  double *d_vals;
  int4 *d_tiles;
  int *d_cta_tile_begin;
  int ntiles;
  int grid;
  int tile_nnz;
  double *d_partials;
  unsigned int *d_counter;
  int version;  // 2: warp-specialised row-per-lane pipeline (fallback), 3: flagged stream
  long long stored;  // entries held in d_colidx / d_vals (v3: nnz + one explicit zero per empty row)
  int4 *d_wt3;       // v3 warp-tile descriptors, padded per CTA to groups of SPMV3_NCW
  int *d_cta_begin3; // v3: first group of every CTA
  // long-row support: virtual rows + combine pass, see Spmv3Plan::vptr
  int nvrows;        // virtual rows (== nrows when no row was cut)
  int *d_vptr;       // nrows+1, or NULL
  double *d_vscratch;  // nvrows partial sums
  int borrows;       // 1: d_rowptr / d_vals / d_wt3 / d_cta_begin3 belong to another operator (renumbered-columns view)
};

// random 8-byte gather of the dense vector: read-only path, optionally without L1 allocation
__device__ __forceinline__ double gather_ld(const double *p) {
#ifdef SPMV_GATHER_NOALLOC
  double r;
  asm volatile("ld.global.nc.L1::no_allocate.f64 %0, [%1];" : "=d"(r) : "l"(p));
  return r;
#else
  return __ldg(p);
#endif
}
// epilogue with operands fetched EARLY (before the gathers are consumed) so that their latency
// overlaps the row's chain instead of adding to it
template <int POST>
__device__ __forceinline__ void spmv_epilogue_pre(double s, int row, double *__restrict__ y, double dv,
                                                  double vv, double &dot_acc) {
  double out = s;
  if (POST == B200_POST_DIV) {
    out = s / dv;
  } else if (POST == B200_POST_MUL) {
    out = s * dv;
  } else if (POST == B200_POST_FMA_DOT) {
    out = fma(dv, vv, s);
    dot_acc = fma(vv, out, dot_acc);
  } else if (POST == B200_POST_FMA) {
    out = fma(dv, vv, s);
  }
  y[row] = out;
}

template <int POST>
__device__ __forceinline__ double spmv_epilogue(double s, int row, double *__restrict__ y,
                                                const double *__restrict__ d,
                                                const double *__restrict__ v, double &dot_acc) {
  double out = s;
  if (POST == B200_POST_DIV) {
    out = s / d[row];
  } else if (POST == B200_POST_MUL) {
    out = s * d[row];
  } else if (POST == B200_POST_FMA_DOT) {
    const double vr = v[row];
    out = fma(d[row], vr, s);
    dot_acc = fma(vr, out, dot_acc);
  } else if (POST == B200_POST_FMA) {
    out = fma(d[row], v[row], s);
  }
  y[row] = out;
  return out;
}

// ==================================================================================
// Version 2: warp-specialised pipeline.  Warp 0 is the TMA PRODUCER (one elected lane issues
// the bulk copies of the value / column-index / row-pointer slices of tile i+S as soon as the
// consumers have released the stage); warps 1..NW-1 are CONSUMERS: each takes rows of the tile
// (one row per thread for short rows), gathers x straight from global memory with up to 8
// independent loads in flight per thread, and adds the products in storage order (bit-identical
// to the sequential CPU loop).  Stages are handed over with full/empty mbarriers only -- there
// is no __syncthreads in the main loop, so a fast warp runs ahead into the next tile.
// defaults: 512 threads (1 producer + 15 consumer warps), 1536-entry tiles, 3 stages, 2 CTAs/SM =
// 148 kB of shared memory per SM, which leaves ~100 kB of the H100's 256 kB L1/shared array for the
// gathers (bigger tiles / more stages shrink L1, which the random gathers need)
#ifndef SPMV2_THREADS
#define SPMV2_THREADS 512
#endif
#ifndef SPMV2_STAGES
#define SPMV2_STAGES 3
#endif
#ifndef SPMV2_TILE_NNZ
#define SPMV2_TILE_NNZ 1536
#endif
#ifndef SPMV2_CTAS_PER_SM
#define SPMV2_CTAS_PER_SM 2
#endif
#define SPMV2_TILE_ROWS SPMV2_TILE_NNZ
#define SPMV2_CAP (SPMV2_TILE_NNZ + 8)
#define SPMV2_RCAP (SPMV2_TILE_ROWS + 8)
#define SPMV2_NCW (SPMV2_THREADS / 32 - 1)
#define SPMV2_CHUNK 8

static size_t spmv2_smem_bytes() {
  return (size_t)SPMV2_STAGES * (SPMV2_CAP * 12 + SPMV2_RCAP * 4) + 2 * SPMV2_STAGES * 8 + 64 * 8;
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

template <int POST>
__global__ void __launch_bounds__(SPMV2_THREADS, SPMV2_CTAS_PER_SM)
spmv_ws_kernel(const int *__restrict__ rowptr, const int *__restrict__ colidx,
               const double *__restrict__ vals, const int4 *__restrict__ tiles,
               const int *__restrict__ cta_tile_begin, const double *__restrict__ x,
               double *__restrict__ y, const double *init, double init_sign,
               const double *__restrict__ d, const double *__restrict__ v, double *dot_out, int hook,
               void *hook_arg, const int *skip, double *partials, unsigned int *counter,
               unsigned long long hook_val) {
  if (skip != nullptr && *((volatile const int *)skip) != 0) return;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  double *s_vals = reinterpret_cast<double *>(smem_raw);
  int *s_idx = reinterpret_cast<int *>(s_vals + SPMV2_STAGES * SPMV2_CAP);
  int *s_rp = s_idx + SPMV2_STAGES * SPMV2_CAP;
  uint64_t *s_full = reinterpret_cast<uint64_t *>(s_rp + SPMV2_STAGES * SPMV2_RCAP);
  uint64_t *s_empty = s_full + SPMV2_STAGES;
  double *s_red = reinterpret_cast<double *>(s_empty + SPMV2_STAGES);

  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int t_begin = cta_tile_begin[blockIdx.x];
  const int nt = cta_tile_begin[blockIdx.x + 1] - t_begin;
  if (tid == 0) {
#pragma unroll
    for (int s = 0; s < SPMV2_STAGES; ++s) {
      mbar_init(&s_full[s], 1);
      mbar_init(&s_empty[s], SPMV2_NCW);
    }
    mbar_fence_init();
  }
  __syncthreads();

  double dot_acc = 0.0;
  if (wid == 0) {
    // ------------------------------------------------ producer
    if (lane == 0) {
      const uint64_t pol = l2_policy_evict_first();
      for (int i = 0; i < nt; ++i) {
        const int st = i % SPMV2_STAGES, use = i / SPMV2_STAGES;
        if (use > 0) mbar_wait(&s_empty[st], (unsigned)((use - 1) & 1));
        const int4 t = tiles[t_begin + i];
        const int k0 = t.z, nnz = t.w, row0 = t.x;
        const int nrows = t.y & 0x00ffffff, type = (t.y >> 28) & 0x7;
        const int ka = k0 & ~3;
        const int cnt = (k0 + nnz - ka + 3) & ~3;
        const int ra = row0 & ~3;
        const int rcnt = (type == TILE_NORMAL) ? ((row0 + nrows + 1 - ra + 3) & ~3) : 0;
        mbar_expect_tx(&s_full[st], (unsigned)cnt * 12u + (unsigned)rcnt * 4u);
        if (cnt > 0) {
          tma_load_1d(s_vals + (size_t)st * SPMV2_CAP, vals + ka, (unsigned)cnt * 8u, &s_full[st], pol);
          tma_load_1d(s_idx + (size_t)st * SPMV2_CAP, colidx + ka, (unsigned)cnt * 4u, &s_full[st], pol);
        }
        if (rcnt > 0)
          tma_load_1d(s_rp + (size_t)st * SPMV2_RCAP, rowptr + ra, (unsigned)rcnt * 4u, &s_full[st], pol);
      }
    }
  } else {
    // ------------------------------------------------ consumers
    const int cw = wid - 1;
    double carry = 0.0;  // long-row running sum (consumer warp 0, lane 0)
    for (int i = 0; i < nt; ++i) {
      const int st = i % SPMV2_STAGES;
      const unsigned par = (unsigned)((i / SPMV2_STAGES) & 1);
      const int4 t = tiles[t_begin + i];
      const int row0 = t.x, nrows = t.y & 0x00ffffff, lg = (t.y >> 24) & 0xf, type = (t.y >> 28) & 0x7;
      const int k0 = t.z, nnz = t.w;
      const double *__restrict__ tv = s_vals + (size_t)st * SPMV2_CAP + (k0 & 3);
      const int *__restrict__ ti = s_idx + (size_t)st * SPMV2_CAP + (k0 & 3);
      const int *__restrict__ rp = s_rp + (size_t)st * SPMV2_RCAP + (row0 & 3);
      mbar_wait(&s_full[st], par);
      if (type == TILE_NORMAL && lg == 0) {
        for (int r = cw * 32 + lane; r < nrows; r += SPMV2_NCW * 32) {
          const int row = row0 + r;
          const int a = rp[r] - k0, b = rp[r + 1] - k0;
          // epilogue operands first: their (global) latency overlaps the gathers below
          const double dv = (POST != B200_POST_NONE) ? d[row] : 0.0;
          const double ev = (POST == B200_POST_FMA_DOT || POST == B200_POST_FMA) ? v[row] : 0.0;
          double s = (init != nullptr) ? init_sign * init[row] : 0.0;
          for (int k = a; k < b; k += SPMV2_CHUNK) {
            int c[SPMV2_CHUNK];
            double xv[SPMV2_CHUNK], vv[SPMV2_CHUNK];
#pragma unroll
            for (int u = 0; u < SPMV2_CHUNK; ++u) c[u] = (k + u < b) ? ti[k + u] : -1;
#pragma unroll
            for (int u = 0; u < SPMV2_CHUNK; ++u) xv[u] = (c[u] >= 0) ? gather_ld(&x[c[u]]) : 0.0;
#pragma unroll
            for (int u = 0; u < SPMV2_CHUNK; ++u) vv[u] = (c[u] >= 0) ? tv[k + u] : 0.0;
#pragma unroll
            for (int u = 0; u < SPMV2_CHUNK; ++u)
              if (c[u] >= 0) s = __dadd_rn(s, __dmul_rn(vv[u], xv[u]));
          }
          spmv_epilogue_pre<POST>(s, row, y, dv, ev, dot_acc);
        }
      } else if (type == TILE_NORMAL && lg <= 2) {
        // Few, medium rows (e.g. the 10-entry rows of A'): L = 2 or 4 lanes share a row so that all
        // consumer threads gather. Lane l of the group loads entries [base + l*CH, base + (l+1)*CH);
        // the group leader then adds the products IN STORAGE ORDER (shuffles), so the result is
        // still bit-identical to the sequential CPU loop.
        const int L = 1 << lg;
        const int lig = lane & (L - 1);
        const unsigned gmask = ((L == 2) ? 0x3u : 0xfu) << (lane & ~(L - 1));
        const int gsrc = lane & ~(L - 1);
        const int gid = (cw * 32 + lane) >> lg, ngroups = (SPMV2_NCW * 32) >> lg;
        for (int r = gid; r < nrows; r += ngroups) {
          const int row = row0 + r;
          const int a = rp[r] - k0, b = rp[r + 1] - k0;
          const double dv = (POST != B200_POST_NONE) ? d[row] : 0.0;
          const double ev = (POST == B200_POST_FMA_DOT || POST == B200_POST_FMA) ? v[row] : 0.0;
          double s = (init != nullptr) ? init_sign * init[row] : 0.0;
          for (int base = a; base < b; base += L * SPMV2_CHUNK) {
            const int k = base + lig * SPMV2_CHUNK;
            int c[SPMV2_CHUNK];
            double pr[SPMV2_CHUNK];
#pragma unroll
            for (int u = 0; u < SPMV2_CHUNK; ++u) c[u] = (k + u < b) ? ti[k + u] : -1;
#pragma unroll
            for (int u = 0; u < SPMV2_CHUNK; ++u) pr[u] = (c[u] >= 0) ? gather_ld(&x[c[u]]) : 0.0;
#pragma unroll
            for (int u = 0; u < SPMV2_CHUNK; ++u) pr[u] = (c[u] >= 0) ? __dmul_rn(tv[k + u], pr[u]) : 0.0;
            for (int l = 0; l < L; ++l) {
#pragma unroll
              for (int u = 0; u < SPMV2_CHUNK; ++u) {
                const double val = __shfl_sync(gmask, pr[u], gsrc + l);
                if (base + l * SPMV2_CHUNK + u < b) s = __dadd_rn(s, val);
              }
            }
          }
          if (lig == 0) spmv_epilogue_pre<POST>(s, row, y, dv, ev, dot_acc);
        }
      } else if (type == TILE_NORMAL) {
        // longer rows: one warp per row, lanes stride the entries, fixed shuffle tree
        for (int r = cw; r < nrows; r += SPMV2_NCW) {
          const int row = row0 + r;
          const int a = rp[r] - k0, b = rp[r + 1] - k0;
          double s = 0.0;
          for (int k = a + lane; k < b; k += 32) s = __dadd_rn(s, __dmul_rn(tv[k], __ldg(&x[ti[k]])));
          s = warp_sum(s);
          if (lane == 0) {
            if (init != nullptr) s += init_sign * init[row];
            spmv_epilogue<POST>(s, row, y, d, v, dot_acc);
          }
        }
      } else if (cw == 0) {
        // chunk of one very long row: consumer warp 0 alone, carry across chunks in lane 0
        double s = 0.0;
        for (int k = lane; k < nnz; k += 32) s = __dadd_rn(s, __dmul_rn(tv[k], __ldg(&x[ti[k]])));
        s = warp_sum(s);
        if (lane == 0) {
          if (type == TILE_LONG_FIRST || type == TILE_LONG_ONLY)
            carry = (init != nullptr) ? init_sign * init[row0] : 0.0;
          carry += s;
          if (type == TILE_LONG_LAST || type == TILE_LONG_ONLY)
            spmv_epilogue<POST>(carry, row0, y, d, v, dot_acc);
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&s_empty[st]);
    }
  }

  if (hook == B200_HOOK_P2P_SIGNAL) {
    // multi-GPU: tell every peer that this rank's partial product is complete (last block only)
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
      if (tid == 0) {
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
// Version 3: "flagged stream" -- nonzero-per-lane instead of row-per-lane.
//
// What bounds the SpMV of a uniformly random matrix is not HBM but the L1TEX pipe: every
// nonzero costs one wavefront for its 8-byte gather (no two lanes share a 128-byte line), and
// the row-per-thread kernels above add ~0.45 shared-memory wavefronts per nonzero on top (bank
// conflicts of the row-strided reads of values / indices, row pointers) -- ncu: L1TEX 70-80 %.
// v3 removes everything but the gather from that pipe:
//   * the operator is stored as a FLAGGED stream: colidx carries "last entry of its row" in bit 31
//     and "explicit zero, do not gather" in bit 30; every empty row owns one such zero entry, so
//     row r is simply the r-th END flag and the kernel needs NO row pointers at all;
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
// Rows longer than SPMV3_MAXROW entries do not fit a warp-tile: such operators keep the plain
// CSR and the v2 kernel.
// defaults: ONE CTA of 768 threads per SM (1 producer + 23 consumer warps), 3 stages = 130 kB of shared
// memory (within the H100's 227 kB per block), which leaves ~125 kB of the 256 kB L1/shared array to the gathers
#ifndef SPMV3_THREADS
#define SPMV3_THREADS 768
#endif
#ifndef SPMV3_STAGES
#define SPMV3_STAGES 3
#endif
#ifndef SPMV3_CTAS_PER_SM
#define SPMV3_CTAS_PER_SM 1
#endif
#define SPMV3_NCW (SPMV3_THREADS / 32 - 1)
#define SPMV3_WT 128
#define SPMV3_CAP (SPMV3_NCW * SPMV3_WT + 8)
#define SPMV3_MAXROW 124
#define SPMV3_END 0x80000000u
#define SPMV3_SKIP 0x40000000u

static size_t spmv3_smem_bytes() {
  return (size_t)SPMV3_STAGES * (SPMV3_CAP * 12 + SPMV3_NCW * 16) + 2 * SPMV3_STAGES * 8 + 64 * 8 +
         (size_t)SPMV3_NCW * SPMV3_WT * 8;
}

template <int POST>
__device__ __forceinline__ void spmv3_emit(double s, int row, double *__restrict__ y, const double *init,
                                           double init_sign, const double *__restrict__ d,
                                           const double *__restrict__ v, double &dot_acc) {
  if (init != nullptr) s = __dadd_rn(s, init_sign * init[row]);
  spmv_epilogue<POST>(s, row, y, d, v, dot_acc);
}

template <int POST>
__global__ void __launch_bounds__(SPMV3_THREADS, SPMV3_CTAS_PER_SM)
spmv_flag_kernel(const int *__restrict__ colidx, const double *__restrict__ vals,
                 const int4 *__restrict__ wt, const int *__restrict__ cta_begin,
                 const double *__restrict__ x, double *__restrict__ y, const double *init,
                 double init_sign, const double *__restrict__ d, const double *__restrict__ v,
                 double *dot_out, int hook, void *hook_arg, const int *skip, double *partials,
                 unsigned int *counter, unsigned long long hook_val) {
  // Programmatic dependent launch: nothing above pdl_wait() reads data a predecessor kernel writes -- the
  // descriptors and the matrix stream are immutable -- so barrier init and the first ring stages overlap the
  // predecessor's tail. `skip`, x, d, v, init are read only after the wait.
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
        mbar_expect_tx(&s_full[st], (unsigned)cnt * 12u + (unsigned)(SPMV3_NCW * 16));
        tma_load_1d(s_desc + (size_t)st * SPMV3_NCW, g + (size_t)i * SPMV3_NCW, SPMV3_NCW * 16,
                    &s_full[st], pol);
        tma_load_1d(s_idx + (size_t)st * SPMV3_CAP, colidx + ka, (unsigned)cnt * 4u, &s_full[st], pol);
        tma_load_1d(s_vals + (size_t)st * SPMV3_CAP, vals + ka, (unsigned)cnt * 8u, &s_full[st], pol);
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
    const int cw = wid - 1;
    double *ws = s_out + cw * SPMV3_WT;
    const unsigned FULL = 0xffffffffu;
    const unsigned lt = (1u << lane) - 1u;
    const unsigned le = lt | (1u << lane);
    const int sw = (lane >> 2) & 1;
    for (int i = 0; i < (skipped ? 0 : nt); ++i) {
      const int st = i % SPMV3_STAGES;
      const unsigned par = (unsigned)((i / SPMV3_STAGES) & 1);
      mbar_wait(&s_full[st], par);
      const int4 dsc = s_desc[st * SPMV3_NCW + cw];
      const int ka = s_desc[st * SPMV3_NCW].y & ~3;
      const int row0 = dsc.x, k0 = dsc.y, cnt = dsc.z;
      const int kend = k0 + cnt;
      const int kb = (k0 & ~3) + 4 * lane;  // global index of this lane's first entry
      int4 iv = make_int4(0, 0, 0, 0);
      double2 t0 = make_double2(0.0, 0.0), t1 = make_double2(0.0, 0.0);
      const bool any = (kb < kend) && (kb + 4 > k0);
      if (any) {
        const int e = kb - ka;
        iv = *reinterpret_cast<const int4 *>(s_idx + (size_t)st * SPMV3_CAP + e);
        t0 = *reinterpret_cast<const double2 *>(s_vals + (size_t)st * SPMV3_CAP + e + 2 * sw);
        t1 = *reinterpret_cast<const double2 *>(s_vals + (size_t)st * SPMV3_CAP + e + 2 - 2 * sw);
      }
      const bool v0 = any && (kb >= k0), v1 = any && (kb + 1 >= k0) && (kb + 1 < kend),
                 v2 = any && (kb + 2 >= k0) && (kb + 2 < kend), v3 = any && (kb + 3 < kend);
      const bool g0 = v0 && !(iv.x & SPMV3_SKIP), g1 = v1 && !(iv.y & SPMV3_SKIP),
                 g2 = v2 && !(iv.z & SPMV3_SKIP), g3 = v3 && !(iv.w & SPMV3_SKIP);
      // 4 independent gathers in flight per lane
      const double x0 = g0 ? gather_ld(&x[iv.x & 0x3fffffff]) : 0.0;
      const double x1 = g1 ? gather_ld(&x[iv.y & 0x3fffffff]) : 0.0;
      const double x2 = g2 ? gather_ld(&x[iv.z & 0x3fffffff]) : 0.0;
      const double x3 = g3 ? gather_ld(&x[iv.w & 0x3fffffff]) : 0.0;
      // the stage's bytes are in registers (the gather addresses depend on them): hand it back
      __syncwarp();
      if (lane == 0) mbar_arrive(&s_empty[st]);
      if (cnt == 0) continue;  // padding descriptor (warp-uniform)
      const int nrows_w = dsc.w;
      // epilogue operands of the first two rounds (rows row0 + lane, row0 + lane + 32): in flight
      // together with the gathers
      double pd0 = 0.0, pd1 = 0.0, pv0 = 0.0, pv1 = 0.0, pi0 = 0.0, pi1 = 0.0;
      {
        const bool r0ok = lane < nrows_w, r1ok = lane + 32 < nrows_w;
        if (POST != B200_POST_NONE) {
          if (r0ok) pd0 = d[row0 + lane];
          if (r1ok) pd1 = d[row0 + lane + 32];
        }
        if (POST == B200_POST_FMA_DOT || POST == B200_POST_FMA) {
          if (r0ok) pv0 = v[row0 + lane];
          if (r1ok) pv1 = v[row0 + lane + 32];
        }
        if (init != nullptr) {
          if (r0ok) pi0 = init[row0 + lane];
          if (r1ok) pi1 = init[row0 + lane + 32];
        }
      }

      const double a0 = sw ? t1.x : t0.x, a1 = sw ? t1.y : t0.y;
      const double a2 = sw ? t0.x : t1.x, a3 = sw ? t0.y : t1.y;
      const bool e0 = v0 && (iv.x < 0), e1 = v1 && (iv.y < 0), e2 = v2 && (iv.z < 0), e3 = v3 && (iv.w < 0);
      const unsigned b0 = __ballot_sync(FULL, e0), b1 = __ballot_sync(FULL, e1);
      const unsigned b2 = __ballot_sync(FULL, e2), b3 = __ballot_sync(FULL, e3);
      const unsigned ends = b0 | b1 | b2 | b3;  // lanes in which at least one row ends
      // row number (within the warp-tile) of the first END of this lane = number of ENDs in the lanes before it
      int r = __popc(b0 & lt) + __popc(b1 & lt) + __popc(b2 & lt) + __popc(b3 & lt);
      // open-row segments: the tail of lane h (the last lane <= me in which a row ends) starts the
      // row that is open when my entries begin
      const unsigned mle = ends & le;
      const int h = mle ? 31 - __clz(mle) : 0;
      const int maxdist = __reduce_max_sync(FULL, lane - h);

      const double p0 = g0 ? __dmul_rn(a0, x0) : 0.0, p1 = g1 ? __dmul_rn(a1, x1) : 0.0;
      const double p2 = g2 ? __dmul_rn(a2, x2) : 0.0, p3 = g3 ? __dmul_rn(a3, x3) : 0.0;
      // in-lane sequential sums, restarted after every END (0 + p is exact)
      double acc = p0;
      double o0 = acc;
      if (e0) acc = 0.0;
      acc = __dadd_rn(acc, p1);
      double o1 = acc;
      if (e1) acc = 0.0;
      acc = __dadd_rn(acc, p2);
      double o2 = acc;
      if (e2) acc = 0.0;
      acc = __dadd_rn(acc, p3);
      double o3 = acc;
      if (e3) acc = 0.0;
      // segmented inclusive scan of the tails (Hillis-Steele, fixed order)
      double I = acc;
      for (int dd = 1; dd <= maxdist; dd <<= 1) {
        const double up = __shfl_up_sync(FULL, I, dd);
        if (lane - dd >= h) I = __dadd_rn(up, I);
      }
      double carry = __shfl_up_sync(FULL, I, 1);
      if (lane == 0) carry = 0.0;  // warp-tiles hold whole rows: nothing is open at entry 0
      // the first END of the lane closes the row that was open on entry
      if (e0) o0 = __dadd_rn(carry, o0);
      else if (e1) o1 = __dadd_rn(carry, o1);
      else if (e2) o2 = __dadd_rn(carry, o2);
      else if (e3) o3 = __dadd_rn(carry, o3);
      // transpose through the warp's scratch: row sums by row number, then a COALESCED epilogue
      // (one row per lane and round: full-sector stores of y, one division per row, operands of the
      // first two rounds were fetched before the gathers were consumed)
      if (e0) { ws[r] = o0; ++r; }
      if (e1) { ws[r] = o1; ++r; }
      if (e2) { ws[r] = o2; ++r; }
      if (e3) { ws[r] = o3; }
      __syncwarp();
#pragma unroll
      for (int j = 0; j < SPMV3_WT / 32; ++j) {
        const int rr = lane + 32 * j;
        if (j * 32 >= nrows_w) break;  // warp-uniform
        if (rr < nrows_w) {
          const int row = row0 + rr;
          double sres = ws[rr];
          double dv, vv, iv0;
          if (j == 0) { dv = pd0; vv = pv0; iv0 = pi0; }
          else if (j == 1) { dv = pd1; vv = pv1; iv0 = pi1; }
          else {
            dv = (POST != B200_POST_NONE) ? d[row] : 0.0;
            vv = (POST == B200_POST_FMA_DOT || POST == B200_POST_FMA) ? v[row] : 0.0;
            iv0 = (init != nullptr) ? init[row] : 0.0;
          }
          if (init != nullptr) sres = __dadd_rn(sres, init_sign * iv0);
          if (routed) {  // push the row to the rank that owns it, as a self-validating 16-byte element
            int o = 0;
            while (row >= s_rt_lo[o + 1]) ++o;
            ll_store(s_rt_dst[o] + 2 * (size_t)(row - s_rt_lo[o]), sres, (unsigned)hook_val);
          } else {
            spmv_epilogue_pre<POST>(sres, row, y, dv, vv, dot_acc);
          }
        }
      }
      __syncwarp();  // the scratch is rewritten by the next warp-tile
    }
  }

  if (skipped) return;  // uniform over the CTA: every thread read the same *skip after the predecessor completed
  if (hook == B200_HOOK_P2P_SIGNAL) {
    // multi-GPU (replicated modes): tell every peer that this rank's partial product is complete (last block only).
    // The push mode (B200_HOOK_P2P_ROUTE) needs no signal: every pushed row validates itself.
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
    double accd[1] = {dot_acc};
    block_sum<1>(accd, s_red);
    if (grid_finish<1>(accd, partials, counter, 0u, s_red)) {
      if (tid == 0) {
        *dot_out = accd[0];
        if (hook == B200_HOOK_CG_ALPHA) {
          B200CgCtl *c = reinterpret_cast<B200CgCtl *>(hook_arg);
          c->pGp = accd[0];
          c->alpha = c->ztr / accd[0];
        }
      }
    }
  }
}


// Second pass of the long-row mode. The flag kernel has written one sum per
// VIRTUAL row into `part`; thread r adds the pieces of true row r in order, applies the epilogue and the same
// deterministic dot / hook tail as the one-pass kernels.
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
    spmv_epilogue<POST>(s, r, y, d, v, dot_acc);
  }
  if (hook == B200_HOOK_P2P_SIGNAL) {
    __syncthreads();
    if (threadIdx.x == 0) {
      __threadfence();
      const unsigned tk = atomicAdd(counter, 1u);
      if (tk == gridDim.x - 1) {
        *counter = 0u;
        __threadfence_system();
        const B200P2pSignal *ps = reinterpret_cast<const B200P2pSignal *>(hook_arg);
        for (int q = 0; q < ps->nranks; ++q)
          if (q != ps->rank) *((volatile unsigned long long *)(ps->flags[q] + ps->rank)) = hook_val;
      }
    }
  }
  if (POST == B200_POST_FMA_DOT) {
    double accd[1] = {dot_acc};
    block_sum<1>(accd, s_red);
    if (grid_finish<1>(accd, partials, counter, 0u, s_red)) {
      if (threadIdx.x == 0) {
        *dot_out = accd[0];
        if (hook == B200_HOOK_CG_ALPHA) {
          B200CgCtl *c = reinterpret_cast<B200CgCtl *>(hook_arg);
          c->pGp = accd[0];
          c->alpha = c->ztr / accd[0];
        }
      }
    }
  }
}

// ---- host side of v3: the flagged stream, its warp-tiles and the static CTA partition.
// Pure host code (no CUDA calls): also exported for the CPU tests (tests/test_spmv_plan_cpu.py
// re-executes the kernel's lane algorithm on this plan in numpy).
struct Spmv3Plan {
  std::vector<int> rowptr;   // stored row pointers (every row has >= 1 stored entry)
  // column | END | SKIP and the values: raw buffers, deliberately NOT value-initialised (a 120 MB memset per
  // operator at C2) -- every element is written by the fill below
  struct Raw {
    void *p = nullptr;
    ~Raw() { free(p); }
  } idx_mem, vals_mem;
  size_t stored_count = 0;
  int *idx_data() const { return static_cast<int *>(idx_mem.p); }
  double *vals_data() const { return static_cast<double *>(vals_mem.p); }
  std::vector<int4> wt;      // padded per CTA to a multiple of SPMV3_NCW: {row0, k0, cnt, nrows}
  std::vector<int> cta_begin;  // grid+1, in groups of SPMV3_NCW descriptors
  int grid = 0;
  int nwt = 0;               // real warp-tiles
  // long-row support: a row longer than SPMV3_MAXROW is cut into pieces ("virtual rows", an END flag at
  // the end of every piece); the kernel then produces one sum per virtual row and a combine pass adds the
  // pieces of each true row. vptr[r] = first virtual row of true row r (empty when no row was cut).
  std::vector<int> vptr;
  int nvrows = 0;
};

// warp-tiles (whole (virtual) rows whose aligned span (k0 & ~3 .. end) is <= 128 entries) and the static CTA
// partition, from the stored (virtual) row pointers alone -- shared by every plan builder (host, device, permuted).
// CTAs own equal counts of warp-tiles. A warp-tile holds up to 128 entries whatever its rows, so this balances the
// gathers; on the row-sorted CG copy of A it leaves 2.8x more rows on the last CTAs than on the first, but rows are
// cheap next to gathers: balancing on entries + rows (or 2 entries + rows) was 1.3 % (0.2 %) slower per CG iteration
// on C2 (H100 SXM, DESIGN.md section 3.1).
static void spmv3_tiles_from_rowptr(int nv, const int *vrp, long long stored, int grid_cap, Spmv3Plan &P) {
  std::vector<int4> real;
  real.reserve((size_t)(stored / 100 + 16));
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

static bool spmv3_build_plan(int nrows, int ncols, const int *rp, const int *ci, const double *va,
                             int grid_cap, Spmv3Plan &P, bool split_long = false) {
  if (nrows <= 0 || ncols >= (1 << 30)) return false;
  const long long nnz = rp[nrows];
  long long empties = 0, extra_pieces = 0;
  for (int r = 0; r < nrows; ++r) {
    const int len = rp[r + 1] - rp[r];
    if (len > SPMV3_MAXROW) {
      if (!split_long) return false;
      extra_pieces += (len + SPMV3_MAXROW - 1) / SPMV3_MAXROW - 1;
    }
    if (len == 0) ++empties;
  }
  if ((long long)nrows + extra_pieces > 2000000000LL) return false;
  const long long stored = nnz + empties;
  if (stored > 2000000000LL) return false;
  P.rowptr.resize((size_t)nrows + 1);
  P.stored_count = (size_t)stored;
  P.idx_mem.p = malloc(((size_t)stored + 1) * sizeof(int));
  P.vals_mem.p = malloc(((size_t)stored + 1) * sizeof(double));
  if (!P.idx_mem.p || !P.vals_mem.p) return false;
  {
    int pos = 0;
    for (int r = 0; r < nrows; ++r) {
      P.rowptr[r] = pos;
      const int len = rp[r + 1] - rp[r];
      pos += len > 0 ? len : 1;
    }
    P.rowptr[nrows] = pos;
  }
  // copy + flag the entries, rows split over host threads (disjoint output ranges)
  {
    int *out_i = P.idx_data();
    double *out_v = P.vals_data();
    const int *orp = P.rowptr.data();
    auto fill = [=](int ra, int rb) {
      for (int r = ra; r < rb; ++r) {
        const int a = rp[r], b = rp[r + 1];
        int pos = orp[r];
        if (a == b) {
          out_i[pos] = (int)(SPMV3_END | SPMV3_SKIP);
          out_v[pos] = 0.0;
        } else {
          for (int k = a; k < b; ++k, ++pos) {
            out_i[pos] = ci[k];
            out_v[pos] = va[k];
          }
          out_i[pos - 1] = (int)((unsigned)out_i[pos - 1] | SPMV3_END);
          const int len = b - a;
          if (len > SPMV3_MAXROW) {  // balanced pieces, an END after each of them
            const int pieces = (len + SPMV3_MAXROW - 1) / SPMV3_MAXROW, small = len / pieces, big = len % pieces;
            int e = orp[r];
            for (int q = 0; q < pieces - 1; ++q) {
              e += small + (q < big ? 1 : 0);
              out_i[e - 1] = (int)((unsigned)out_i[e - 1] | SPMV3_END);
            }
          }
        }
      }
    };
    const int T = b200_host_threads(stored);
    if (T <= 1) {
      fill(0, nrows);
    } else {
      std::vector<std::thread> th;
      for (int t = 0; t < T; ++t) {
        // ranges balanced by stored entries
        auto cut = [&](int q) {
          const long long target = stored * q / T;
          return (int)(std::lower_bound(P.rowptr.begin(), P.rowptr.end(), (int)target) - P.rowptr.begin());
        };
        int ra = t == 0 ? 0 : cut(t), rb = t == T - 1 ? nrows : cut(t + 1);
        if (ra > nrows) ra = nrows;
        if (rb > nrows) rb = nrows;
        if (rb > ra) {
          try {
            th.emplace_back(fill, ra, rb);
          } catch (...) {  // no more threads available: do this range here
            fill(ra, rb);
          }
        }
      }
      for (auto &x : th) x.join();
    }
  }
  // virtual row pointers: identical to the row pointers unless a row was cut into pieces
  std::vector<int> vrp_store;
  const int *vrp = P.rowptr.data();
  int nv = nrows;
  P.vptr.clear();
  P.nvrows = nrows;
  if (extra_pieces > 0) {
    nv = (int)(nrows + extra_pieces);
    vrp_store.resize((size_t)nv + 1);
    P.vptr.resize((size_t)nrows + 1);
    int v = 0;
    for (int r = 0; r < nrows; ++r) {
      P.vptr[r] = v;
      const int len = rp[r + 1] - rp[r];
      if (len > SPMV3_MAXROW) {
        const int pieces = (len + SPMV3_MAXROW - 1) / SPMV3_MAXROW, small = len / pieces, big = len % pieces;
        int e = P.rowptr[r];
        for (int q = 0; q < pieces; ++q) {
          vrp_store[v++] = e;
          e += small + (q < big ? 1 : 0);
        }
      } else {
        vrp_store[v++] = P.rowptr[r];
      }
    }
    P.vptr[nrows] = v;
    vrp_store[v] = P.rowptr[nrows];
    vrp = vrp_store.data();
    P.nvrows = nv;
  }
  spmv3_tiles_from_rowptr(nv, vrp, stored, grid_cap, P);
  return true;
}

// C view of a plan for the tests (host memory, owned by the handle)
struct B200Spmv3PlanHost {
  Spmv3Plan plan;
};
extern "C" B200Spmv3PlanHost *b200_spmv3_plan_build(int nrows, int ncols, const int *rp, const int *ci,
                                                    const double *va, int grid_cap) {
  B200Spmv3PlanHost *h = new B200Spmv3PlanHost();
  const char *lr = getenv("SCS_B200_SPMV_LONGROWS");
  const bool split = !(lr && atoi(lr) == 0);
  if (!spmv3_build_plan(nrows, ncols, rp, ci, va, grid_cap, h->plan, split)) {
    delete h;
    return nullptr;
  }
  return h;
}
extern "C" void b200_spmv3_plan_free(B200Spmv3PlanHost *h) { delete h; }
extern "C" int b200_spmv3_plan_info(const B200Spmv3PlanHost *h, int *stored, int *nwt, int *ndesc, int *grid,
                                    int *ncw) {
  *stored = (int)h->plan.stored_count;
  *nwt = h->plan.nwt;
  *ndesc = (int)h->plan.wt.size();
  *grid = h->plan.grid;
  *ncw = SPMV3_NCW;
  return 0;
}
extern "C" const int *b200_spmv3_plan_rowptr(const B200Spmv3PlanHost *h) { return h->plan.rowptr.data(); }
extern "C" const int *b200_spmv3_plan_idx(const B200Spmv3PlanHost *h) { return h->plan.idx_data(); }
extern "C" const double *b200_spmv3_plan_vals(const B200Spmv3PlanHost *h) { return h->plan.vals_data(); }
extern "C" const int *b200_spmv3_plan_desc(const B200Spmv3PlanHost *h) {
  return reinterpret_cast<const int *>(h->plan.wt.data());
}
extern "C" const int *b200_spmv3_plan_cta_begin(const B200Spmv3PlanHost *h) { return h->plan.cta_begin.data(); }
extern "C" int b200_spmv3_plan_nvrows(const B200Spmv3PlanHost *h) { return h->plan.nvrows; }
extern "C" const int *b200_spmv3_plan_vptr(const B200Spmv3PlanHost *h) {
  return h->plan.vptr.empty() ? nullptr : h->plan.vptr.data();
}

// ------------------------------------------------------------------ host side
static int lanes_log2_for(int max_row_nnz) {
  if (max_row_nnz <= 16) return 0;
  if (max_row_nnz <= 48) return 2;
  if (max_row_nnz <= 160) return 3;
  return 5;
}

static void spmv_set_attrs() {
  static bool attr_done = false;
  if (attr_done) return;
#define SET_ATTR(K, BYTES)                                                                       \
  do {                                                                                           \
    cudaFuncSetAttribute(K<B200_POST_NONE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(BYTES));    \
    cudaFuncSetAttribute(K<B200_POST_DIV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(BYTES));     \
    cudaFuncSetAttribute(K<B200_POST_MUL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(BYTES));     \
    cudaFuncSetAttribute(K<B200_POST_FMA_DOT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(BYTES)); \
    cudaFuncSetAttribute(K<B200_POST_FMA>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(BYTES));     \
  } while (0)
  SET_ATTR(spmv_ws_kernel, spmv2_smem_bytes());
  SET_ATTR(spmv_flag_kernel, spmv3_smem_bytes());
#undef SET_ATTR
  attr_done = true;
}

// v3: upload the flagged stream (it IS the operator's CSR: rowptr / colidx / vals stay a valid CSR with
// explicit zeros, flags in the two top bits of colidx) plus the warp-tile descriptors
static int spmv_upload_v3(B200Spmv *M, const Spmv3Plan &P) {
  const size_t stored = P.stored_count;
  const size_t pad = ((stored + 3) & ~(size_t)3) + 8;
  M->stored = (long long)stored;
  M->grid = P.grid;
  M->ntiles = P.nwt;
  M->tile_nnz = SPMV3_WT;
  M->d_rowptr = (int *)b200_malloc((size_t)(M->nrows + 1 + 8) * 4);
  M->d_colidx = (int *)b200_malloc(pad * 4);
  M->d_vals = (double *)b200_malloc(pad * 8);
  M->d_wt3 = (int4 *)b200_malloc(P.wt.size() * sizeof(int4));
  M->d_cta_begin3 = (int *)b200_malloc(P.cta_begin.size() * 4);
  M->d_partials = (double *)b200_malloc((size_t)B200_MAX_PARTIALS * 8);
  M->d_counter = (unsigned int *)b200_malloc(64);
  if (!M->d_rowptr || !M->d_colidx || !M->d_vals || !M->d_wt3 || !M->d_cta_begin3 || !M->d_partials ||
      !M->d_counter)
    return -1;
  int rc = 0;
  rc |= b200_memset0(M->d_rowptr, (size_t)(M->nrows + 1 + 8) * 4);
  rc |= b200_memset0(M->d_colidx, pad * 4);
  rc |= b200_memset0(M->d_vals, pad * 8);
  rc |= b200_memset0(M->d_counter, 64);
  rc |= b200_h2d(M->d_rowptr, P.rowptr.data(), (size_t)(M->nrows + 1) * 4);
  rc |= b200_h2d(M->d_colidx, P.idx_data(), stored * 4);
  rc |= b200_h2d(M->d_vals, P.vals_data(), stored * 8);
  rc |= b200_h2d(M->d_wt3, P.wt.data(), P.wt.size() * sizeof(int4));
  rc |= b200_h2d(M->d_cta_begin3, P.cta_begin.data(), P.cta_begin.size() * 4);
  M->nvrows = P.nvrows;
  if (!P.vptr.empty()) {  // long-row mode
    M->d_vptr = (int *)b200_malloc(P.vptr.size() * 4);
    M->d_vscratch = (double *)b200_malloc((size_t)P.nvrows * 8);
    if (!M->d_vptr || !M->d_vscratch) return -1;
    rc |= b200_h2d(M->d_vptr, P.vptr.data(), P.vptr.size() * 4);
  }
  rc |= b200_sync();  // the plan's host vectors go out of scope
  if (rc != 0) return -1;
  spmv_set_attrs();
  return 0;
}

extern "C" B200Spmv *b200_spmv_create(int nrows, int ncols, const int *h_rowptr,
                                      const int *h_colidx, const double *h_vals) {
  if (b200_runtime_init() != 0) return nullptr;
  if (ncols >= (1 << 30) || nrows >= (1 << 30)) {
    // bits 30/31 of the stored column indices are flags (v3); every reader masks them
    b200_set_error("b200_spmv_create: dimensions >= 2^30 are not supported", cudaErrorInvalidValue, __FILE__,
                   __LINE__);
    return nullptr;
  }
  B200Spmv *M = (B200Spmv *)calloc(1, sizeof(B200Spmv));
  if (!M) return nullptr;
  M->nrows = nrows;
  M->ncols = ncols;
  M->nnz = h_rowptr[nrows];
  M->stored = M->nnz;
  const long long nnz = M->nnz;
  const int nsm = b200_num_sms();

  {
    const char *e = getenv("SCS_B200_SPMV");
    M->version = e ? atoi(e) : SPMV_DEFAULT_VERSION;
    if (M->version < 2 || M->version > 3) M->version = SPMV_DEFAULT_VERSION;
  }
  if (M->version == 3) {
    // flagged stream; operators with a row longer than SPMV3_MAXROW keep the plain CSR + v2 kernel
    int cap = SPMV3_CTAS_PER_SM * nsm;
    const char *g = getenv("SCS_B200_SPMV_GRID");  // tests: force many groups per CTA on small matrices
    if (g && atoi(g) > 0 && atoi(g) < cap) cap = atoi(g);
    // operators with very short rows (avg below SCS_B200_SPMV_MINAVG, default 0 = never) can be sent to
    // the row-per-lane kernel instead (tuning knob)
    const char *ma = getenv("SCS_B200_SPMV_MINAVG");
    const bool too_short = ma && nrows > 0 && (double)nnz / nrows < atof(ma);
    Spmv3Plan P;
    // rows longer than a warp-tile: virtual rows + combine pass (SCS_B200_SPMV_LONGROWS=0 sends such operators
    // to the v2 kernel instead)
    const char *lr = getenv("SCS_B200_SPMV_LONGROWS");
    const bool split_long = !(lr && atoi(lr) == 0);
    if (nrows > 0 && !too_short && spmv3_build_plan(nrows, ncols, h_rowptr, h_colidx, h_vals, cap, P, split_long)) {
      if (spmv_upload_v3(M, P) != 0) {
        b200_spmv_destroy(M);
        return nullptr;
      }
      return M;
    }
    M->version = 2;
  }
  // tile size: full tiles for big matrices, smaller ones so that small matrices
  // still spread over all SMs
  const int max_tile = SPMV2_TILE_NNZ;
  const int ctas_per_sm = SPMV2_CTAS_PER_SM;
  long long want = nnz / (2LL * ctas_per_sm * nsm);
  int tile_nnz = 256 < max_tile ? 256 : max_tile;
  while (tile_nnz < max_tile && tile_nnz < want) tile_nnz <<= 1;
  if (tile_nnz > max_tile) tile_nnz = max_tile;
  M->tile_nnz = tile_nnz;
  const int tile_rows = SPMV2_TILE_ROWS;

  std::vector<int4> tiles;
  tiles.reserve((size_t)(nnz / tile_nnz + nrows / tile_rows + 16));
  std::vector<long long> weight;  // cumulative weight after each tile
  int r = 0;
  long long cumw = 0;
  while (r < nrows) {
    const int k0 = h_rowptr[r];
    const int rn = h_rowptr[r + 1] - k0;
    if (rn > tile_nnz) {
      // long row: chunks of tile_nnz
      int done = 0;
      while (done < rn) {
        int c = rn - done < tile_nnz ? rn - done : tile_nnz;
        int type = (done == 0) ? TILE_LONG_FIRST : ((done + c == rn) ? TILE_LONG_LAST : TILE_LONG_MID);
        int4 t;
        t.x = r;
        t.y = 1 | (type << 28);
        t.z = k0 + done;
        t.w = c;
        tiles.push_back(t);
        cumw += c + 64;
        weight.push_back(cumw);
        done += c;
      }
      r += 1;
      continue;
    }
    int r1 = r, cnt = 0, mx = 0;
    while (r1 < nrows && (r1 - r) < tile_rows) {
      const int rr = h_rowptr[r1 + 1] - h_rowptr[r1];
      if (rr > tile_nnz) break;           // next is a long row
      if (cnt + rr > tile_nnz) break;     // tile full
      cnt += rr;
      if (rr > mx) mx = rr;
      ++r1;
    }
    int4 t;
    t.x = r;
    int lgv = lanes_log2_for(mx);
    if (M->version == 2) {
      // v2: lg 0/1/2 = 1/2/4 lanes per row with ORDERED combine (bit-exact), 5 = warp per row (tree)
      const int nr = r1 - r, cons = SPMV2_NCW * 32;
      // sharing a 10-entry row between 2 lanes was slower on C2, so the ordered multi-lane mode is off unless
      // asked for
      lgv = 0;
      if (mx > 64) lgv = 5;
#ifdef SPMV2_ORDERED_LANES
      else if (nr * 4 <= cons) lgv = 2;
      else if (nr * 2 <= cons) lgv = 1;
#else
      (void)nr; (void)cons;
#endif
    }
    t.y = (r1 - r) | (TILE_NORMAL << 28) | (lgv << 24);
    t.z = k0;
    t.w = cnt;
    tiles.push_back(t);
    cumw += cnt + 2LL * (r1 - r) + 64;
    weight.push_back(cumw);
    r = r1;
  }
  M->ntiles = (int)tiles.size();
  int grid = ctas_per_sm * nsm;
  if (grid > M->ntiles) grid = M->ntiles;
  if (grid < 1) grid = 1;
  M->grid = grid;
  std::vector<int> begin(grid + 1, 0);
  {
    // balanced contiguous partition by cumulative weight; never split a long row
    int t = 0;
    for (int c = 1; c < grid; ++c) {
      const long long target = (cumw * c) / grid;
      while (t < M->ntiles && weight[t] <= target) ++t;
      // weight[t-1] <= target < weight[t]; boundary AFTER tile t-1 => begin = t
      int bnd = t;
      while (bnd < M->ntiles) {
        int type = (tiles[bnd].y >> 28) & 7;
        if (type == TILE_LONG_MID || type == TILE_LONG_LAST) ++bnd; else break;
      }
      if (bnd < begin[c - 1]) bnd = begin[c - 1];
      begin[c] = bnd;
      if (t < bnd) t = bnd;
    }
    begin[grid] = M->ntiles;
  }

  const size_t pad_nnz = (size_t)((nnz + 3) & ~3LL) + 8;
  M->d_rowptr = (int *)b200_malloc((size_t)(nrows + 1 + 8) * 4);
  M->d_colidx = (int *)b200_malloc(pad_nnz * 4);
  M->d_vals = (double *)b200_malloc(pad_nnz * 8);
  M->d_tiles = (int4 *)b200_malloc((size_t)(M->ntiles > 0 ? M->ntiles : 1) * sizeof(int4));
  M->d_cta_tile_begin = (int *)b200_malloc((size_t)(grid + 1) * 4);
  M->d_partials = (double *)b200_malloc((size_t)B200_MAX_PARTIALS * 8);
  M->d_counter = (unsigned int *)b200_malloc(64);
  if (!M->d_rowptr || !M->d_colidx || !M->d_vals || !M->d_tiles || !M->d_cta_tile_begin ||
      !M->d_partials || !M->d_counter) {
    b200_spmv_destroy(M);
    return nullptr;
  }
  int rc = 0;
  rc |= b200_memset0(M->d_rowptr, (size_t)(nrows + 1 + 8) * 4);
  rc |= b200_memset0(M->d_colidx, pad_nnz * 4);
  rc |= b200_memset0(M->d_vals, pad_nnz * 8);
  rc |= b200_memset0(M->d_counter, 64);
  rc |= b200_h2d(M->d_rowptr, h_rowptr, (size_t)(nrows + 1) * 4);
  if (nnz > 0) {
    rc |= b200_h2d(M->d_colidx, h_colidx, (size_t)nnz * 4);
    rc |= b200_h2d(M->d_vals, h_vals, (size_t)nnz * 8);
  }
  if (M->ntiles > 0) rc |= b200_h2d(M->d_tiles, tiles.data(), (size_t)M->ntiles * sizeof(int4));
  rc |= b200_h2d(M->d_cta_tile_begin, begin.data(), (size_t)(grid + 1) * 4);
  rc |= b200_sync();  // host vectors go out of scope
  if (rc != 0) {
    b200_spmv_destroy(M);
    return nullptr;
  }
  spmv_set_attrs();
  return M;
}

// ---------------------------------------------------------------------------------------------
// Device-side construction of a flagged-stream operator from a CSR that is ALREADY IN HBM (setup path of
// scs_init_lin_sys_work, kernels/setup.cu): stored row pointers (every row >= 1 entry) by a scan, the flagged
// stream by one fill kernel; only the row pointers travel back to the host for the (sequential, O(rows)) warp-tile
// pass. Returns NULL when the operator needs what only the host builder offers (rows longer than a warp-tile,
// forced v2, dimension limits) -- the caller then takes the host path.
__global__ void k_stored_len(int nrows, const int *__restrict__ rp, int *__restrict__ out, int *maxlen) {
  int mx = 0;
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < nrows; r += gridDim.x * blockDim.x) {
    const int len = rp[r + 1] - rp[r];
    out[r] = len > 0 ? len : 1;
    mx = len > mx ? len : mx;
  }
  mx = __reduce_max_sync(0xffffffffu, mx);
  if ((threadIdx.x & 31) == 0 && mx > 0) atomicMax(maxlen, mx);
}
__global__ void k_fill_flagged(int nrows, const int *__restrict__ rp, const int *__restrict__ sp,
                               const int *__restrict__ ci, const double *__restrict__ va, int *__restrict__ oi,
                               double *__restrict__ ov) {
  // one lane per row; a row longer than SPMV3_MAXROW gets an END at the end of every balanced piece (the "virtual
  // rows" of Spmv3Plan::vptr: the first len % pieces pieces hold one entry more) -- same cut as spmv3_build_plan
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int r0 = warp * 32; r0 < nrows; r0 += nwarps * 32) {
    const int r = r0 + lane;
    if (r < nrows) {
      const int a = rp[r], b = rp[r + 1], len = b - a;
      int pos = sp[r];
      if (a == b) {
        oi[pos] = (int)(SPMV3_END | SPMV3_SKIP);
        ov[pos] = 0.0;
      } else if (len <= SPMV3_MAXROW) {
        for (int k = a; k < b; ++k, ++pos) {
          oi[pos] = (k == b - 1) ? (int)((unsigned)ci[k] | SPMV3_END) : ci[k];
          ov[pos] = va[k];
        }
      } else {
        const int pieces = (len + SPMV3_MAXROW - 1) / SPMV3_MAXROW, small = len / pieces, big = len % pieces;
        int left = small + (big > 0 ? 1 : 0), q = 0;
        for (int k = a; k < b; ++k, ++pos) {
          const bool end = --left == 0;
          oi[pos] = end ? (int)((unsigned)ci[k] | SPMV3_END) : ci[k];
          ov[pos] = va[k];
          if (end) {
            ++q;
            left = small + (q < big ? 1 : 0);
          }
        }
      }
    }
  }
}
extern "C" int b200_dev_exclusive_scan_int(const int *d_in, int *d_out, int count);  // kernels/setup.cu (CUB)

extern "C" B200Spmv *b200_spmv_create_dev(int nrows, int ncols, long long nnz, const int *d_rp, const int *d_ci,
                                          const double *d_va) {
  if (b200_runtime_init() != 0) return nullptr;
  if (ncols >= (1 << 30) || nrows >= (1 << 30) || nrows <= 0) return nullptr;
  {
    const char *e = getenv("SCS_B200_SPMV");
    if (e && atoi(e) == 2) return nullptr;
    if (getenv("SCS_B200_SPMV_MINAVG")) return nullptr;
  }
  cudaStream_t st = (cudaStream_t)b200_stream();
  B200Spmv *M = (B200Spmv *)calloc(1, sizeof(B200Spmv));
  if (!M) return nullptr;
  M->nrows = nrows; M->ncols = ncols; M->nnz = nnz; M->version = 3;
  int *d_len = (int *)b200_malloc((size_t)(nrows + 1) * 4);
  int *d_max = (int *)b200_malloc(4);
  M->d_rowptr = (int *)b200_malloc((size_t)(nrows + 1 + 8) * 4);
  std::vector<int> h_sp;
  int h_max = 0, stored = 0;
  Spmv3Plan P;
  bool ok = d_len && d_max && M->d_rowptr;
  if (ok) {
    ok = b200_memset0(d_max, 4) == 0 && b200_memset0(M->d_rowptr, (size_t)(nrows + 1 + 8) * 4) == 0 &&
         b200_memset0(d_len + nrows, 4) == 0;
    int g = (nrows + 255) / 256;
    if (g > 8 * b200_num_sms()) g = 8 * b200_num_sms();
    if (ok) k_stored_len<<<g, 256, 0, st>>>(nrows, d_rp, d_len, d_max);
    // exclusive scan over nrows + 1 items: element nrows receives the total
    ok = ok && b200_dev_exclusive_scan_int(d_len, M->d_rowptr, nrows + 1) == 0;
    ok = ok && b200_d2h(&h_max, d_max, 4) == 0;
    h_sp.resize((size_t)nrows + 1);
    ok = ok && b200_d2h(h_sp.data(), M->d_rowptr, (size_t)(nrows + 1) * 4) == 0 && b200_sync() == 0;
    b200_count_launch(2);
  }
  {
    const char *lr = getenv("SCS_B200_SPMV_LONGROWS");
    if (ok && h_max > SPMV3_MAXROW && lr && atoi(lr) == 0) ok = false;  // long rows disabled: host builder (v2)
  }
  if (ok) {
    stored = h_sp[(size_t)nrows];
    if (stored < 0) ok = false;
  }
  if (ok) {
    const size_t pad = (((size_t)stored + 3) & ~(size_t)3) + 8;
    M->stored = stored;
    M->d_colidx = (int *)b200_malloc(pad * 4);
    M->d_vals = (double *)b200_malloc(pad * 8);
    ok = M->d_colidx && M->d_vals && b200_memset0(M->d_colidx, pad * 4) == 0 && b200_memset0(M->d_vals, pad * 8) == 0;
    if (ok) {
      int g = (nrows + 255) / 256;
      if (g > 16 * b200_num_sms()) g = 16 * b200_num_sms();
      k_fill_flagged<<<g, 256, 0, st>>>(nrows, d_rp, M->d_rowptr, d_ci, d_va, M->d_colidx, M->d_vals);
      b200_count_launch(1);
    }
  }
  if (ok) {
    int cap = SPMV3_CTAS_PER_SM * b200_num_sms();
    const char *gq = getenv("SCS_B200_SPMV_GRID");
    if (gq && atoi(gq) > 0 && atoi(gq) < cap) cap = atoi(gq);
    // virtual row pointers (sequential O(rows) host pass, overlaps the fill kernel): identical to the stored row
    // pointers unless a row is longer than a warp-tile -- then its pieces, cut exactly as k_fill_flagged cuts them
    std::vector<int> vrp_store;
    const int *vrp = h_sp.data();
    int nv = nrows;
    if (h_max > SPMV3_MAXROW) {
      long long extra = 0;
      for (int r = 0; r < nrows; ++r) {
        const int len = h_sp[(size_t)r + 1] - h_sp[r];
        if (len > SPMV3_MAXROW) extra += (len + SPMV3_MAXROW - 1) / SPMV3_MAXROW - 1;
      }
      if ((long long)nrows + extra >= (1LL << 30)) ok = false;
      if (ok) {
        nv = (int)(nrows + extra);
        vrp_store.resize((size_t)nv + 1);
        P.vptr.resize((size_t)nrows + 1);
        int v = 0;
        for (int r = 0; r < nrows; ++r) {
          P.vptr[r] = v;
          const int len = h_sp[(size_t)r + 1] - h_sp[r];
          if (len > SPMV3_MAXROW) {
            const int pieces = (len + SPMV3_MAXROW - 1) / SPMV3_MAXROW, small = len / pieces, big = len % pieces;
            int e = h_sp[r];
            for (int q = 0; q < pieces; ++q) {
              vrp_store[v++] = e;
              e += small + (q < big ? 1 : 0);
            }
          } else {
            vrp_store[v++] = h_sp[r];
          }
        }
        P.vptr[nrows] = v;
        vrp_store[v] = h_sp[(size_t)nrows];
        vrp = vrp_store.data();
      }
    }
    P.nvrows = nv;
    if (ok) spmv3_tiles_from_rowptr(nv, vrp, stored, cap, P);
    M->grid = P.grid; M->ntiles = P.nwt; M->tile_nnz = SPMV3_WT; M->nvrows = nv;
    if (ok && !P.vptr.empty()) {
      M->d_vptr = (int *)b200_malloc(P.vptr.size() * 4);
      M->d_vscratch = (double *)b200_malloc((size_t)nv * 8);
      ok = M->d_vptr && M->d_vscratch && b200_h2d(M->d_vptr, P.vptr.data(), P.vptr.size() * 4) == 0;
    }
  }
  if (ok) {
    M->d_wt3 = (int4 *)b200_malloc(P.wt.size() * sizeof(int4));
    M->d_cta_begin3 = (int *)b200_malloc(P.cta_begin.size() * 4);
    M->d_partials = (double *)b200_malloc((size_t)B200_MAX_PARTIALS * 8);
    M->d_counter = (unsigned int *)b200_malloc(64);
    ok = M->d_wt3 && M->d_cta_begin3 && M->d_partials && M->d_counter && b200_memset0(M->d_counter, 64) == 0 &&
         b200_h2d(M->d_wt3, P.wt.data(), P.wt.size() * sizeof(int4)) == 0 &&
         b200_h2d(M->d_cta_begin3, P.cta_begin.data(), P.cta_begin.size() * 4) == 0 && b200_sync() == 0 &&
         cudaGetLastError() == cudaSuccess;
  }
  b200_free(d_len);
  b200_free(d_max);
  if (!ok) {
    b200_spmv_destroy(M);
    return nullptr;
  }
  spmv_set_attrs();
  return M;
}

// ---------------------------------------------------------------------------------------------
// Reordered copies for the CG operator (DESIGN.md section 3.1 "Reordering").
// The m-space ordering INSIDE G = R_x + A' R_y^-1 A is free (tmp = R_y^-1 A p never leaves the operator), so the rows
// of A can be sorted by their smallest column index: one gather per row of K1 becomes sequential, and the matching
// entries of every column of A' become adjacent for K2.
//   b200_spmv_permuted_rows : row-permuted copy of the first `nrows` rows of the permutation of a flagged-stream
//                             operator (row `new` = row perm[new] of M); segments are copied with their flags, the
//                             warp-tiles are recomputed. Rows left out are never written (the caller leaves out
//                             empty rows only, so the entry count stays M's). Every row keeps the LANE SPLIT it has
//                             in M, so that the copy computes bit-for-bit the row sums M computes (see below);
//   b200_spmv_refresh_permuted : values only (after the resident operators were rescaled in place);
//   b200_spmv_renumbered_cols  : a VIEW of M whose stored column indices are mapped through inv[] (flags kept);
//                             row pointers, values and warp-tiles are M's own (borrowed, not copied).
//
// Lane split. The flag kernel sums a row inside one lane sequentially and combines the pieces of a row that spans lanes
// with a scan whose tree depends only on the pieces (lanes own the entries [4l, 4l+4) of the 16-byte-aligned stream;
// a leading lane that holds only explicit zeros adds exact zeros). The pieces are set by the position of the row's
// first entry modulo 4 and its length. The permuted copy therefore places every row so that it is cut into the same
// pieces as in M: a row that spans lanes in M starts at the same position modulo 4, a row that fits one lane in M fits
// one lane here. Up to 3 explicit zeros (SKIP, no END) lead a row's segment to get there. With the row sums equal, the
// CG operator computes what the plain pair computes, only faster.
__global__ void k_fill_skip(long long count, int *__restrict__ oi) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < count; k += (long long)gridDim.x * blockDim.x)
    oi[k] = (int)SPMV3_SKIP;
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
    out[k] = (v & SPMV3_SKIP) ? (int)v : (int)((unsigned)inv[v & 0x3fffffffu] | (v & SPMV3_END));
  }
}

extern "C" B200Spmv *b200_spmv_permuted_rows(const B200Spmv *S, const int *d_perm, int nrows) {
  if (!S || S->version != 3 || S->d_vptr != nullptr || nrows <= 0 || nrows > S->nrows) return nullptr;
  cudaStream_t st = (cudaStream_t)b200_stream();
  B200Spmv *M = (B200Spmv *)calloc(1, sizeof(B200Spmv));
  if (!M) return nullptr;
  M->nrows = nrows; M->ncols = S->ncols; M->nnz = S->nnz; M->version = 3; M->nvrows = nrows;
  // segment layout on the host (sequential, O(rows)): stored row pointers of M and the permutation come back once
  std::vector<int> h_old((size_t)S->nrows + 1), h_perm((size_t)nrows), h_sp((size_t)nrows + 1);
  bool ok = b200_d2h(h_old.data(), S->d_rowptr, h_old.size() * 4) == 0 &&
            b200_d2h(h_perm.data(), d_perm, h_perm.size() * 4) == 0 && b200_sync() == 0;
  long long pos = 0;
  for (int r = 0; ok && r < nrows; ++r) {
    const int a = h_old[(size_t)h_perm[(size_t)r]], len = h_old[(size_t)h_perm[(size_t)r] + 1] - a;
    const int phase = a & 3, c = (int)(pos & 3);
    int lead;
    if (phase + len <= 4) lead = c + len <= 4 ? 0 : 4 - c;  // one lane in M: one lane here
    else lead = (phase - c) & 3;                              // spans lanes in M: the same first position modulo 4
    if (c + lead + len > SPMV3_WT) lead = 0;  // a row of more than 121 entries: its warp-tile could not hold the zeros
    h_sp[(size_t)r] = (int)pos;
    pos += lead + len;
  }
  h_sp[(size_t)nrows] = (int)pos;
  if (pos > 2000000000LL) ok = false;
  M->stored = pos;
  const size_t pad = (((size_t)pos + 3) & ~(size_t)3) + 8;
  M->d_rowptr = (int *)b200_malloc((size_t)(nrows + 1 + 8) * 4);
  M->d_colidx = (int *)b200_malloc(pad * 4);
  M->d_vals = (double *)b200_malloc(pad * 8);
  M->d_partials = (double *)b200_malloc((size_t)B200_MAX_PARTIALS * 8);
  M->d_counter = (unsigned int *)b200_malloc(64);
  Spmv3Plan P;
  int g = (nrows + 255) / 256;
  if (g > 16 * b200_num_sms()) g = 16 * b200_num_sms();
  ok = ok && M->d_rowptr && M->d_colidx && M->d_vals && M->d_partials && M->d_counter;
  ok = ok && b200_memset0(M->d_rowptr, (size_t)(nrows + 1 + 8) * 4) == 0 && b200_memset0(M->d_vals, pad * 8) == 0 &&
       b200_memset0(M->d_counter, 64) == 0 && b200_h2d(M->d_rowptr, h_sp.data(), h_sp.size() * 4) == 0;
  if (ok) {
    k_fill_skip<<<8 * b200_num_sms(), 256, 0, st>>>((long long)pad, M->d_colidx);
    k_perm_copy<<<g, 256, 0, st>>>(nrows, S->d_rowptr, M->d_rowptr, d_perm, S->d_colidx, S->d_vals, M->d_colidx,
                                   M->d_vals);
    b200_count_launch(2);
    ok = cudaGetLastError() == cudaSuccess;
  }
  if (ok) {
    P.nvrows = nrows;
    spmv3_tiles_from_rowptr(nrows, h_sp.data(), M->stored, S->grid > 0 ? SPMV3_CTAS_PER_SM * b200_num_sms() : 1, P);
    M->grid = P.grid; M->ntiles = P.nwt; M->tile_nnz = SPMV3_WT;
    M->d_wt3 = (int4 *)b200_malloc(P.wt.size() * sizeof(int4));
    M->d_cta_begin3 = (int *)b200_malloc(P.cta_begin.size() * 4);
    ok = M->d_wt3 && M->d_cta_begin3 && b200_h2d(M->d_wt3, P.wt.data(), P.wt.size() * sizeof(int4)) == 0 &&
         b200_h2d(M->d_cta_begin3, P.cta_begin.data(), P.cta_begin.size() * 4) == 0 && b200_sync() == 0 &&
         cudaGetLastError() == cudaSuccess;
  }
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
  if (!S || S->version != 3 || S->d_vptr != nullptr) return nullptr;
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

extern "C" void b200_spmv_destroy(B200Spmv *M) {
  if (!M) return;
  if (M->borrows) {  // a view: only the column indices, the reduction slots and the ticket counter are its own
    b200_free(M->d_colidx);
    b200_free(M->d_partials);
    b200_free(M->d_counter);
    free(M);
    return;
  }
  b200_free(M->d_rowptr);
  b200_free(M->d_colidx);
  b200_free(M->d_vals);
  b200_free(M->d_tiles);
  b200_free(M->d_cta_tile_begin);
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
  return 12.0 * (double)M->nnz + 4.0 * (M->nrows + 1.0) + 8.0 * M->ncols +
         8.0 * M->nrows * (1.0 + extra_row_vectors);
}

extern "C" int b200_spmv(const B200Spmv *M, const B200SpmvArgs *a) {
  if (M->nrows == 0) return 0;
  cudaStream_t st = (cudaStream_t)b200_stream();
  const size_t smem = M->version == 3 ? spmv3_smem_bytes() : spmv2_smem_bytes();
  dim3 grid(M->grid), block(M->version == 3 ? SPMV3_THREADS : SPMV2_THREADS);
#define TAIL                                                                                   \
  a->d_x, a->d_y, a->d_init, a->init_sign, a->d_d, a->d_v, a->d_dot, a->hook, a->d_hook_arg,   \
      a->d_skip, M->d_partials, M->d_counter, a->hook_val
#define ARGS M->d_rowptr, M->d_colidx, M->d_vals, M->d_tiles, M->d_cta_tile_begin, TAIL
#define LAUNCH(POSTV)                                                                          \
  do {                                                                                         \
    if (M->version == 3)                                                                       \
      CUDA_OK(b200_launch(spmv_flag_kernel<POSTV>, grid, block, smem, st, a->pdl != 0,         \
                          (const int *)M->d_colidx, (const double *)M->d_vals,                 \
                          (const int4 *)M->d_wt3, (const int *)M->d_cta_begin3, TAIL));        \
    else spmv_ws_kernel<POSTV><<<grid, block, smem, st>>>(ARGS);                               \
  } while (0)
  if (a->hook == B200_HOOK_P2P_ROUTE && !(M->version == 3 && M->d_vptr == nullptr && a->post == B200_POST_NONE)) {
    b200_set_error("b200_spmv: B200_HOOK_P2P_ROUTE needs the one-pass flagged-stream kernel with POST_NONE",
                   cudaErrorInvalidValue, __FILE__, __LINE__);
    return -1;
  }
  if (M->version == 3 && M->d_vptr != nullptr) {
    // long-row mode: sums per virtual row, then the combine pass with the real epilogue
    spmv_flag_kernel<B200_POST_NONE><<<grid, block, smem, st>>>(
        M->d_colidx, M->d_vals, M->d_wt3, M->d_cta_begin3, a->d_x, M->d_vscratch, nullptr, 1.0, nullptr, nullptr,
        nullptr, B200_HOOK_NONE, nullptr, a->d_skip, M->d_partials, M->d_counter, 0ull);
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
  switch (a->post) {
    case B200_POST_NONE: LAUNCH(B200_POST_NONE); break;
    case B200_POST_DIV: LAUNCH(B200_POST_DIV); break;
    case B200_POST_MUL: LAUNCH(B200_POST_MUL); break;
    case B200_POST_FMA_DOT: LAUNCH(B200_POST_FMA_DOT); break;
    case B200_POST_FMA: LAUNCH(B200_POST_FMA); break;
    default: return -1;
  }
#undef LAUNCH
#undef ARGS
#undef TAIL
  b200_count_launch(1);
  CUDA_OK(cudaGetLastError());
  return 0;
}
extern "C" int b200_spmv_version(const B200Spmv *M) { return M->version; }
// B200_HOOK_P2P_ROUTE needs the one-pass flagged-stream kernel (no virtual rows / combine pass)
extern "C" int b200_spmv_can_route(const B200Spmv *M) { return M && M->version == 3 && M->d_vptr == nullptr; }
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
