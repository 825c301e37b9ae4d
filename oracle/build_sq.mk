# oracle/build_sq.mk -- the reference's graph builder over SQ int8 / uint8 codes.  TEST INFRASTRUCTURE ONLY (see README.md).
#
#   make -f build_sq.mk build_sq -> _ref/libsvsref_sq_build.so   ref/build_sq_capi.cpp over the UNMODIFIED reference
#                                                                headers, linked with the same distance-kernel objects
#                                                                as _ref/libsvsref.so (flags and rules from Makefile)
include Makefile

.PHONY: build_sq
build_sq: $(OUT)/libsvsref_sq_build.so

$(OUT)/build_sq_capi.o: ref/build_sq_capi.cpp ref/shims/toml++/toml.h | $(OUT)/inc/fmt
	$(CXX) $(REF_CXX) -march=x86-64 -mtune=generic -c $< -o $@
$(OUT)/libsvsref_sq_build.so: $(OUT)/build_sq_capi.o $(OUT)/avx512.o $(OUT)/avx2.o
	$(CXX) -shared -o $@ $^ -lpthread
