# oracle/dynamic_rows.mk -- the reference's MutableVamanaIndex façades with its stored-row reads.  TEST INFRASTRUCTURE
# ONLY (see README.md).
#
#   make -f dynamic_rows.mk dynamic_rows -> _ref/libsvsref_dynamic_rows.so     ref/dynamic_rows_capi.cpp
#                                           _ref/libsvsref_dynamic_sq_rows.so  ref/dynamic_sq_rows_capi.cpp
# each the matching façade (dynamic_capi.cpp / dynamic_sq_capi.cpp, compiled unchanged into it) plus get_distance and
# reconstruct, over the UNMODIFIED reference headers, linked with the same distance-kernel objects as _ref/libsvsref.so
# (flags and rules from Makefile)
include Makefile

.PHONY: dynamic_rows
dynamic_rows: $(OUT)/libsvsref_dynamic_rows.so $(OUT)/libsvsref_dynamic_sq_rows.so

$(OUT)/dynamic_rows_capi.o: ref/dynamic_rows_capi.cpp ref/dynamic_capi.cpp ref/shims/toml++/toml.h | $(OUT)/inc/fmt
	$(CXX) $(REF_CXX) -march=x86-64 -mtune=generic -c $< -o $@
$(OUT)/dynamic_sq_rows_capi.o: ref/dynamic_sq_rows_capi.cpp ref/dynamic_sq_capi.cpp ref/shims/toml++/toml.h | $(OUT)/inc/fmt
	$(CXX) $(REF_CXX) -march=x86-64 -mtune=generic -c $< -o $@
$(OUT)/libsvsref_dynamic_rows.so: $(OUT)/dynamic_rows_capi.o $(OUT)/avx512.o $(OUT)/avx2.o
	$(CXX) -shared -o $@ $^ -lpthread
$(OUT)/libsvsref_dynamic_sq_rows.so: $(OUT)/dynamic_sq_rows_capi.o $(OUT)/avx512.o $(OUT)/avx2.o
	$(CXX) -shared -o $@ $^ -lpthread
