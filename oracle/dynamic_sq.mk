# oracle/dynamic_sq.mk -- the reference's MutableVamanaIndex over SQ int8 / uint8 codes.  TEST INFRASTRUCTURE ONLY
# (see README.md).
#
#   make -f dynamic_sq.mk dynamic_sq -> _ref/libsvsref_dynamic_sq.so   ref/dynamic_sq_capi.cpp over the UNMODIFIED
#                                                                      reference headers, linked with the same
#                                                                      distance-kernel objects as _ref/libsvsref.so
#                                                                      (flags and rules from Makefile)
include Makefile

.PHONY: dynamic_sq
dynamic_sq: $(OUT)/libsvsref_dynamic_sq.so

$(OUT)/dynamic_sq_capi.o: ref/dynamic_sq_capi.cpp ref/shims/toml++/toml.h | $(OUT)/inc/fmt
	$(CXX) $(REF_CXX) -march=x86-64 -mtune=generic -c $< -o $@
$(OUT)/libsvsref_dynamic_sq.so: $(OUT)/dynamic_sq_capi.o $(OUT)/avx512.o $(OUT)/avx2.o
	$(CXX) -shared -o $@ $^ -lpthread
