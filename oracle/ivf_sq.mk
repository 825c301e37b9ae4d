# oracle/ivf_sq.mk -- the reference's IVF index over SQ int8 / uint8 rows.  TEST INFRASTRUCTURE ONLY (see README.md).
#
#   make -f ivf_sq.mk ivf_sq -> _ref/libsvsref_ivf_sq.so   ref/ivf_sq_capi.cpp over the UNMODIFIED reference headers
#                                                          (ref/shims/mkl.h standing in for the BLAS), linked with the
#                                                          same distance-kernel objects as _ref/libsvsref.so
include Makefile

.PHONY: ivf_sq
ivf_sq: $(OUT)/libsvsref_ivf_sq.so

$(OUT)/ivf_sq_capi.o: ref/ivf_sq_capi.cpp ref/shims/mkl.h ref/shims/toml++/toml.h | $(OUT)/inc/fmt
	$(CXX) $(REF_CXX) -march=x86-64 -mtune=generic -c $< -o $@
$(OUT)/libsvsref_ivf_sq.so: $(OUT)/ivf_sq_capi.o $(OUT)/avx512.o $(OUT)/avx2.o
	$(CXX) -shared -o $@ $^ -lpthread
