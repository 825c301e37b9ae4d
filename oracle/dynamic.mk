# oracle/dynamic.mk -- the reference's MutableVamanaIndex façade.  TEST INFRASTRUCTURE ONLY (see README.md).
#
#   make -f dynamic.mk dynamic -> _ref/libsvsref_dynamic.so   ref/dynamic_capi.cpp over the UNMODIFIED reference
#                                                             headers, linked with the same distance-kernel objects
#                                                             as _ref/libsvsref.so (flags and rules from Makefile)
include Makefile

.PHONY: dynamic
dynamic: $(OUT)/libsvsref_dynamic.so

$(OUT)/dynamic_capi.o: ref/dynamic_capi.cpp ref/shims/toml++/toml.h | $(OUT)/inc/fmt
	$(CXX) $(REF_CXX) -march=x86-64 -mtune=generic -c $< -o $@
$(OUT)/libsvsref_dynamic.so: $(OUT)/dynamic_capi.o $(OUT)/avx512.o $(OUT)/avx2.o
	$(CXX) -shared -o $@ $^ -lpthread
