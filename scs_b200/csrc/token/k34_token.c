/* k34_token.c -- the process-wide token of the CG loop's fused K3 + K4 kernel (kernels/cg.cu, "The fused kernel's grid
 * barrier under concurrency"). It lives in a shared object of its own, libscs_b200_token.so, which every library
 * flavour (int, spectral, DLONG, plugin-only) links by soname: the dynamic loader maps one copy per process however
 * many flavours are loaded, even each with RTLD_LOCAL, so a process has exactly one token. */
#include <stdatomic.h>

static atomic_int token;

/* 1 if the caller now holds the token, 0 if another solve does; never waits */
int b200_k34_token_take(void) {
  int expected = 0;
  return atomic_compare_exchange_strong(&token, &expected, 1);
}
void b200_k34_token_give_back(void) { atomic_store(&token, 0); }
