# oracle/build_int.mk -- the reference's graph builder over int8 / uint8 rows.  TEST INFRASTRUCTURE ONLY (see README.md).
#
#   make -f build_int.mk build_int -> _ref/libsvsref_int.so   ref/build_int_capi.cpp over the UNMODIFIED reference
#                                                             headers, linked with the same distance-kernel objects
#                                                             as _ref/libsvsref.so (flags and rules from Makefile)
include Makefile

.PHONY: build_int
build_int: $(OUT)/libsvsref_int.so

$(OUT)/build_int_capi.o: ref/build_int_capi.cpp ref/shims/toml++/toml.h | $(OUT)/inc/fmt
	$(CXX) $(REF_CXX) -march=x86-64 -mtune=generic -c $< -o $@
$(OUT)/libsvsref_int.so: $(OUT)/build_int_capi.o $(OUT)/avx512.o $(OUT)/avx2.o
	$(CXX) -shared -o $@ $^ -lpthread
