# oracle/sq_set_datum.mk -- the reference's SQDataset::set_datum.  TEST INFRASTRUCTURE ONLY (see README.md).
#
#   make -f sq_set_datum.mk sq_set_datum -> _ref/libsvsref_sq_set_datum.so   ref/sq_set_datum_capi.cpp over the UNMODIFIED
#                                                                         reference headers, linked with the same
#                                                                         distance-kernel objects as _ref/libsvsref.so
include Makefile

.PHONY: sq_set_datum
sq_set_datum: $(OUT)/libsvsref_sq_set_datum.so

$(OUT)/sq_set_datum_capi.o: ref/sq_set_datum_capi.cpp ref/shims/toml++/toml.h | $(OUT)/inc/fmt
	$(CXX) $(REF_CXX) -march=x86-64 -mtune=generic -c $< -o $@
$(OUT)/libsvsref_sq_set_datum.so: $(OUT)/sq_set_datum_capi.o $(OUT)/avx512.o $(OUT)/avx2.o
	$(CXX) -shared -o $@ $^ -lpthread
