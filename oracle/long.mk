# oracle/long.mk -- TEST INFRASTRUCTURE ONLY: the reference built with DLONG=1 (64-bit scs_int), next to the builds of
# oracle/Makefile and oracle/spectral.mk (same flags, same OpenBLAS), into oracle/_ref/ (git-ignored):
#   libscsindir_ref_long.so            the unmodified reference CPU-indirect backend, -DDLONG=1
#   libscsindir_ref_spectral_long.so   the same with USE_SPECTRAL_CONES and src/spectral_cones/**/*.c
#   run_tests_b200_long                the reference's own test/run_tests.c and sources with -DDLONG=1, linked against
#                                      OUR scs_b200/libscs_b200_linsys_long.so instead of its CPU-indirect private.c:
#                                      the drop-in check of INTEGRATION.md section 1 for a DLONG build
# Needs $(REF); run as `make -C oracle -f long.mk`.
REF   ?= /root/reference
OB    ?= /opt/prime-rl/.venv/lib/python3.12/site-packages/opencv_python_headless.libs
OBLIB ?= libopenblasp-r0-59ffcd50.3.15.so
OUT    = _ref
CC     = gcc
OPT    = -O3 -march=x86-64-v3 -fno-math-errno
INC    = -I$(REF) -I$(REF)/include -I$(REF)/linsys
COMMON = $(OPT) -w -fPIC $(INC) -DCTRLC=1 -DINDIRECT=1 -DUSE_LAPACK -DDLONG=1
BLASLD = -L$(OB) -l:$(OBLIB) -Wl,-rpath,$(OB)

REF_SRC = $(REF)/src/aa.c $(REF)/src/cones.c $(REF)/src/ctrlc.c $(REF)/src/exp_cone.c \
          $(REF)/src/linalg.c $(REF)/src/normalize.c $(REF)/src/rw.c $(REF)/src/scs.c \
          $(REF)/src/scs_version.c $(REF)/src/util.c \
          $(REF)/linsys/scs_matrix.c $(REF)/linsys/csparse.c \
          $(REF)/linsys/cpu/indirect/private.c
SPECTRAL_SRC = $(wildcard $(REF)/src/spectral_cones/*.c $(REF)/src/spectral_cones/*/*.c)
REF_SRC_NOLINSYS = $(filter-out $(REF)/linsys/cpu/indirect/private.c,$(REF_SRC))
B200DIR = $(abspath ../scs_b200)

.PHONY: all
all: $(OUT)/libscsindir_ref_long.so $(OUT)/libscsindir_ref_spectral_long.so $(OUT)/run_tests_b200_long

$(OUT):
	mkdir -p $(OUT)

$(OUT)/libscsindir_ref_long.so: | $(OUT)
	$(CC) -shared $(COMMON) -Wl,-Bsymbolic -o $@ $(REF_SRC) $(BLASLD) -lm

$(OUT)/libscsindir_ref_spectral_long.so: | $(OUT)
	$(CC) -shared $(COMMON) -DUSE_SPECTRAL_CONES -Wl,-Bsymbolic -o $@ $(REF_SRC) $(SPECTRAL_SRC) $(BLASLD) -lm

# the binary fixture files the tests read by relative path are copied next to the binary, as for run_tests_b200
$(OUT)/run_tests_b200_long: | $(OUT)
	$(MAKE) -C ../scs_b200/csrc linsys_long
	$(CC) $(COMMON) -I$(REF)/test -o $@ $(REF)/test/run_tests.c $(REF_SRC_NOLINSYS) \
	   -L$(B200DIR) -l:libscs_b200_linsys_long.so -Wl,-rpath,'$$ORIGIN/../../scs_b200' $(BLASLD) -lm
	mkdir -p $(OUT)/test/problems
	find $(REF)/test/problems -maxdepth 1 -type f ! -name '*.h' -exec cp {} $(OUT)/test/problems/ \;
