/*
 * scs_b200_device.h -- the device-data entry points of the outer ABI (include/scs_b200.h group (1)), exported by
 * libscs_b200.so, libscs_b200_spectral.so, libscs_b200_long.so and libscs_b200_spectral_long.so.
 */
#ifndef SCS_B200_DEVICE_H
#define SCS_B200_DEVICE_H
#include "scs_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Device-data entry points: the same pipeline entered and left in GPU memory, with results bit-identical to
 * scs_init / scs_update / scs_solve on the same data.
 *  - scs_b200_init_device: d->A->{x,i,p}, d->P->{x,i,p}, d->b and d->c are DEVICE pointers on the library's device
 *    (SCS_B200_DEVICE / LOCAL_RANK; cudaMalloc'ed or managed memory); the structs, the cone with all its arrays and the
 *    settings stay in host memory. Every check of scs_init runs, the matrix checks on the device with the same
 *    messages; the operators, P's symmetric form and the equilibration are built there from device-to-device copies.
 *  - scs_b200_update_device: d_b, d_c device pointers, NULL keeps the current vector (as scs_update).
 *  - scs_b200_solve_device: d_sol->{x,y,s} device pointers (n, m, m), read for a warm start and written with the
 *    result; info in host memory.
 * The caller's arrays are only read (except d_sol). `stream` is the caller's cudaStream_t (NULL = the legacy default
 * stream): the library's work starts after what is enqueued on it at the call, and work enqueued on it after the call
 * returns runs after the library's. Workspaces are interchangeable with scs_init's: scs_update, scs_solve and
 * scs_finish take one made here, and these take one made by scs_init. Refused (NULL / -1, with a message): a host
 * pointer or memory of another device, a process that is one of several ranks (multi-GPU), or invalid data. Since
 * -1 is also SCS_UNBOUNDED, a refused scs_b200_solve_device is told apart by info: it is left untouched, while every
 * solve that starts writes info->lin_sys_solver first. The operators and the equilibration are built as scs_init builds
 * them on one GPU, with the same bits.
 * With write_data_filename or log_csv_filename set, the data needed is copied to the host (debugging modes). */
ScsWork *scs_b200_init_device(const ScsData *d, const ScsCone *k, const ScsSettings *stgs, void *stream);
scs_int scs_b200_update_device(ScsWork *w, const scs_float *d_b, const scs_float *d_c, void *stream);
scs_int scs_b200_solve_device(ScsWork *w, ScsSolution *d_sol, ScsInfo *info, scs_int warm_start, void *stream);

/* New values of A (and P) with the sparsity pattern the workspace was built with. A (and P, exactly when the
 * workspace has one) as for scs_b200_init_device: the structs in host memory, x, i, p device pointers; the same m, n,
 * p and i as at init, only x may differ. Afterwards the workspace acts exactly like a fresh init through the same door
 * with the same settings on (A, P, the current original b and c): the next solve, cold or warm from the same given
 * x, y, s, returns the same bits. The equilibration is redone as init did it, b and c are renormalised from their
 * originals, the scale goes back to stgs->scale, and AA, the box Newton warm start and the iterates are reset; the
 * operator layouts, cone workspaces, AA and CG workspaces are kept. A caller with new b and c as well calls
 * scs_b200_update_device afterwards. Refused (-1, with a message, the workspace untouched): A missing, P given or
 * missing against the workspace, another m or n, another pattern, invalid entries (init's messages), a host pointer or
 * memory of another device, a process that is one of several ranks. Accepts workspaces of scs_init too. */
scs_int scs_b200_update_matrix_device(ScsWork *w, const ScsMatrix *A, const ScsMatrix *P, void *stream);
#ifdef __cplusplus
}
#endif
#endif /* SCS_B200_DEVICE_H */
