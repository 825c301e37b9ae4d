# oracle/dynamic_flat.mk -- the reference's DynamicFlatIndex façade.  TEST INFRASTRUCTURE ONLY (see README.md).
#
#   make -f dynamic_flat.mk dynamic_flat -> _ref/libsvsref_dynamic_flat.so   ref/dynamic_flat_capi.cpp over the
#                                           UNMODIFIED reference headers, linked with the same distance-kernel objects
#                                           as _ref/libsvsref.so (flags and rules from Makefile)
include Makefile

.PHONY: dynamic_flat
dynamic_flat: $(OUT)/libsvsref_dynamic_flat.so

$(OUT)/dynamic_flat_capi.o: ref/dynamic_flat_capi.cpp ref/shims/toml++/toml.h | $(OUT)/inc/fmt
	$(CXX) $(REF_CXX) -march=x86-64 -mtune=generic -c $< -o $@
$(OUT)/libsvsref_dynamic_flat.so: $(OUT)/dynamic_flat_capi.o $(OUT)/avx512.o $(OUT)/avx2.o
	$(CXX) -shared -o $@ $^ -lpthread
