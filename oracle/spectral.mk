# oracle/spectral.mk -- TEST INFRASTRUCTURE ONLY: the reference's USE_SPECTRAL_CONES build, next to the builds of
# oracle/Makefile (same flags, same OpenBLAS), into oracle/_ref/ (git-ignored):
#   libscsindir_ref_spectral.so   the unmodified reference CPU-indirect backend + src/spectral_cones/**/*.c
#   spectral_fixtures_ref         oracle/spectral_fixtures.c linked with the same sources and the reference's
#                                 spectral test problems (test/spectral_cones_problems/*.h): it writes each
#                                 problem's data file (oracle/make_golden_spectral.py turns them into fixtures)
# Needs $(REF); run as `make -C oracle -f spectral.mk`.
REF   ?= /root/reference
OB    ?= /opt/prime-rl/.venv/lib/python3.12/site-packages/opencv_python_headless.libs
OBLIB ?= libopenblasp-r0-59ffcd50.3.15.so
OUT    = _ref
CC     = gcc
OPT    = -O3 -march=x86-64-v3 -fno-math-errno
INC    = -I$(REF) -I$(REF)/include -I$(REF)/linsys
COMMON = $(OPT) -w -fPIC $(INC) -DCTRLC=1 -DINDIRECT=1 -DUSE_LAPACK -DUSE_SPECTRAL_CONES
BLASLD = -L$(OB) -l:$(OBLIB) -Wl,-rpath,$(OB)

REF_SRC = $(REF)/src/aa.c $(REF)/src/cones.c $(REF)/src/ctrlc.c $(REF)/src/exp_cone.c \
          $(REF)/src/linalg.c $(REF)/src/normalize.c $(REF)/src/rw.c $(REF)/src/scs.c \
          $(REF)/src/scs_version.c $(REF)/src/util.c \
          $(REF)/linsys/scs_matrix.c $(REF)/linsys/csparse.c \
          $(REF)/linsys/cpu/indirect/private.c \
          $(wildcard $(REF)/src/spectral_cones/*.c $(REF)/src/spectral_cones/*/*.c)

.PHONY: all
all: $(OUT)/libscsindir_ref_spectral.so $(OUT)/spectral_fixtures_ref

$(OUT):
	mkdir -p $(OUT)

$(OUT)/libscsindir_ref_spectral.so: | $(OUT)
	$(CC) -shared $(COMMON) -Wl,-Bsymbolic -o $@ $(REF_SRC) $(BLASLD) -lm

$(OUT)/spectral_fixtures_ref: spectral_fixtures.c | $(OUT)
	$(CC) $(COMMON) -I$(REF)/test -Wl,--wrap=scs -o $@ spectral_fixtures.c $(REF_SRC) $(BLASLD) -lm
