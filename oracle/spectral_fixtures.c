/* spectral_fixtures.c -- TEST INFRASTRUCTURE ONLY (oracle/spectral.mk). Runs the reference's spectral-cone test
 * problems that avoid the log-det cone and, through -Wl,--wrap=scs, makes each problem's scs() call first write its
 * data (ScsSettings.write_data_filename) as <outdir>/<problem>. Usage: spectral_fixtures_ref <outdir> */
#include <stdio.h>
#include <string.h>

#include "scs.h"
#include "spectral_cones_problems/graph_partitioning.h"
#include "spectral_cones_problems/robust_pca.h"
#include "spectral_cones_problems/several_nuc_cone.h"
#include "spectral_cones_problems/several_sum_largest.h"
#include "spectral_cones_problems/test_ell1_and_nuc.h"
#include "spectral_cones_problems/test_ell1_cone.h"

static const char *g_dir, *g_name;

scs_int __real_scs(const ScsData *d, const ScsCone *k, const ScsSettings *stgs, ScsSolution *sol, ScsInfo *info);
scs_int __wrap_scs(const ScsData *d, const ScsCone *k, const ScsSettings *stgs, ScsSolution *sol, ScsInfo *info) {
  char path[4096];
  ScsSettings st = *stgs;
  snprintf(path, sizeof(path), "%s/%s", g_dir, g_name);
  st.write_data_filename = path;
  st.verbose = 0;
  return __real_scs(d, k, &st, sol, info);
}

int main(int argc, char **argv) {
  static const struct {
    const char *name;
    const char *(*run)(void);
  } problems[] = {{"test_ell1_cone", test_ell1_cone}, {"test_ell1_and_nuc", test_ell1_and_nuc},
                  {"robust_pca", robust_pca}, {"several_nuc_cone", several_nuc_cone},
                  {"several_sum_largest", several_sum_largest}, {"graph_partitioning", graph_partitioning}};
  size_t i;
  int bad = 0;
  if (argc != 2) {
    fprintf(stderr, "usage: %s <outdir>\n", argv[0]);
    return 2;
  }
  g_dir = argv[1];
  for (i = 0; i < sizeof(problems) / sizeof(problems[0]); ++i) {
    const char *msg;
    g_name = problems[i].name;
    msg = problems[i].run();
    if (msg) {
      fprintf(stderr, "%s: %s\n", g_name, msg);
      bad = 1;
    }
  }
  return bad;
}
