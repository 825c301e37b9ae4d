# oracle/ivf_hier.mk -- the reference's hierarchical k-means façade.  TEST INFRASTRUCTURE ONLY (see README.md).
#
#   make -f ivf_hier.mk ivf_hier -> _ref/libsvsref_ivf_hier.so   ref/ivf_hier_capi.cpp over the UNMODIFIED reference
#                                                                headers (with the own ref/shims/mkl.h standing in for
#                                                                the BLAS), linked with the same distance-kernel objects
#                                                                as _ref/libsvsref.so (flags and rules from Makefile)
include Makefile

.PHONY: ivf_hier
ivf_hier: $(OUT)/libsvsref_ivf_hier.so

$(OUT)/ivf_hier_capi.o: ref/ivf_hier_capi.cpp ref/shims/mkl.h ref/shims/toml++/toml.h | $(OUT)/inc/fmt
	$(CXX) $(REF_CXX) -march=x86-64 -mtune=generic -c $< -o $@
$(OUT)/libsvsref_ivf_hier.so: $(OUT)/ivf_hier_capi.o $(OUT)/avx512.o $(OUT)/avx2.o
	$(CXX) -shared -o $@ $^ -lpthread
