/* logdet_fixtures.c -- TEST INFRASTRUCTURE ONLY (oracle/logdet.mk). Runs the reference's two spectral-cone test
 * problems with log-det cones and, through -Wl,--wrap=scs, makes each problem's scs() call first write its data
 * (ScsSettings.write_data_filename) as <outdir>/<problem>. Usage: logdet_fixtures_ref <outdir>
 * The vector step itself (log_cone_proj_wrapper) is exported by libscsindir_ref_spectral.so and is called from
 * oracle/make_golden_logdet.py directly. */
#include <stdio.h>
#include <string.h>

#include "scs.h"
#include "spectral_cones_problems/exp_design.h"
#include "spectral_cones_problems/several_logdet_cones.h"

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
  } problems[] = {{"exp_design", exp_design}, {"several_logdet_cones", several_logdet_cones}};
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
