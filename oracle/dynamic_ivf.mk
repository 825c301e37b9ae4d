# oracle/dynamic_ivf.mk -- the reference's dynamic IVF index façade.  TEST INFRASTRUCTURE ONLY (see README.md).
#
#   make -f dynamic_ivf.mk dynamic_ivf -> _ref/libsvsref_dynamic_ivf.so   ref/dynamic_ivf_capi.cpp over the UNMODIFIED reference headers (with the
#                                                 own ref/shims/mkl.h standing in for the BLAS), linked with the same
#                                                 distance-kernel objects as _ref/libsvsref.so (flags and rules from Makefile)
include Makefile

.PHONY: dynamic_ivf
dynamic_ivf: $(OUT)/libsvsref_dynamic_ivf.so

$(OUT)/dynamic_ivf_capi.o: ref/dynamic_ivf_capi.cpp ref/shims/mkl.h ref/shims/toml++/toml.h | $(OUT)/inc/fmt
	$(CXX) $(REF_CXX) -march=x86-64 -mtune=generic -c $< -o $@
$(OUT)/libsvsref_dynamic_ivf.so: $(OUT)/dynamic_ivf_capi.o $(OUT)/avx512.o $(OUT)/avx2.o
	$(CXX) -shared -o $@ $^ -lpthread
