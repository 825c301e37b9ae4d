// oracle/_ref driver for the reference's SQDataset::set_datum -- TEST INFRASTRUCTURE ONLY (see oracle/README.md).
//
// A thin `extern "C"` façade over the *unmodified* reference headers (`-I/root/reference/include`, never copied),
// built by `make -C oracle -f sq_set_datum.mk` into `_ref/libsvsref_sq_set_datum.so` and linked with the same
// `avx512.o` / `avx2.o` distance kernels as `libsvsref.so`.  Tests hand it float32 rows with a scale and bias; it
// stores them into the reference's own SQDataset<int8_t / uint8_t> with that scale and bias and returns the codes:
//   quantization/scalar/scalar.h:417-429   SQDataset::set_datum
//   quantization/scalar/scalar.h:38-42     detail::compress
// This is how an add encodes its rows in the reference's dynamic IVF index over SQ data.
//
// Nothing in the product (libsvsb200.so / scalablevectorsearch_b200) links or loads this.

#include "svs/core/data.h"
#include "svs/concepts/distance.h"
#include "svs/core/distance.h"
#include "svs/quantization/scalar/scalar.h"

#include <cstdint>
#include <cstring>
#include <span>
#include <stdexcept>
#include <string>

namespace {

thread_local std::string g_error;

template <typename F> int guarded(F&& f) {
    try {
        f();
        return 0;
    } catch (const std::exception& e) {
        g_error = e.what();
        return 1;
    } catch (...) {
        g_error = "unknown exception";
        return 2;
    }
}

template <typename T> void set_data(const float* data, size_t n, size_t dim, float scale, float bias, void* codes_out) {
    auto sq = svs::quantization::scalar::SQDataset<T>(n, dim);
    sq.set_scale(scale);
    sq.set_bias(bias);
    for (size_t i = 0; i < n; ++i) sq.set_datum(i, std::span<const float>(data + i * dim, dim));
    for (size_t i = 0; i < n; ++i) {
        auto d = sq.get_datum(i);
        std::memcpy(static_cast<T*>(codes_out) + i * dim, d.data(), dim * sizeof(T));
    }
}

} // namespace

extern "C" {

const char* svsref_sq_set_datum_last_error() { return g_error.c_str(); }

/// SQDataset<int8_t> (code_type 2) or <uint8_t> (3) with the given scale and bias: set_datum of float32 rows
/// [n][dim]; the codes [n][dim] out.
int svsref_sq_set_datum(const float* data, size_t n, size_t dim, int code_type, float scale, float bias, void* codes_out) {
    return guarded([&] {
        if (code_type == 2)
            set_data<int8_t>(data, n, dim, scale, bias, codes_out);
        else if (code_type == 3)
            set_data<uint8_t>(data, n, dim, scale, bias, codes_out);
        else
            throw std::runtime_error("code_type must be 2 (int8) or 3 (uint8)");
    });
}

} // extern "C"
