# oracle/logdet.mk -- TEST INFRASTRUCTURE ONLY: the log-det fixture writer, next to oracle/spectral.mk's targets and
# built from the same reference sources and flags (which include src/spectral_cones/logdeterminant/), into oracle/_ref/
# (git-ignored):
#   logdet_fixtures_ref   oracle/logdet_fixtures.c linked with the reference's exp_design and several_logdet_cones
#                         test problems: it writes each problem's data file (oracle/make_golden_logdet.py)
# Needs $(REF); run as `make -C oracle -f logdet.mk`.
include spectral.mk

.PHONY: logdet
logdet: $(OUT)/libscsindir_ref_spectral.so $(OUT)/logdet_fixtures_ref

$(OUT)/logdet_fixtures_ref: logdet_fixtures.c | $(OUT)
	$(CC) $(COMMON) -I$(REF)/test -Wl,--wrap=scs -o $@ logdet_fixtures.c $(REF_SRC) $(BLASLD) -lm
