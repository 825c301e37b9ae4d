// oracle/_ref driver for graph builds over scalar-quantised codes -- TEST INFRASTRUCTURE ONLY (see oracle/README.md).
//
// A thin `extern "C"` façade over the *unmodified* reference headers (`-I/root/reference/include`, never copied):
// the reference's graph construction over SQDataset<int8_t / uint8_t> with a given scale and bias, and the distance
// its builder uses between two data (the build adaptor's general distance, a DecompressionAdaptor over the metric's
// compressed distance).
//
// Reference entry points exercised (file:line under /root/reference/include/svs):
//   index/vamana/index.h:968-994                 auto_build (medoid entry point, two passes alpha = 1 then alpha)
//   extensions/vamana/scalar.h:47-95             VamanaBuildAdaptor for SQ data
//   quantization/scalar/scalar.h:547-600         DecompressionAdaptor
//   index/vamana/vamana_build.h:522-545          maybe_fix_argument(general_distance, datum i), compute(..., datum j)
//
// Nothing in the product (libsvsb200.so / scalablevectorsearch_b200) links or loads this.

#include "svs/core/data.h"
#include "svs/core/distance.h"
#include "svs/core/graph.h"
#include "svs/extensions/vamana/scalar.h"
#include "svs/index/vamana/index.h"
#include "svs/quantization/scalar/scalar.h"

#include <cstdint>
#include <span>
#include <string>

namespace {

thread_local std::string g_error;

enum DType : int { I8 = 2, U8 = 3 };
enum Metric : int { L2 = 0, IP = 1, COS = 2 };

template <typename T> using SQ = svs::quantization::scalar::SQDataset<T, svs::Dynamic, svs::lib::Allocator<T>>;

template <typename T> SQ<T> sq_of(const void* src, size_t n, size_t dim, float scale, float bias) {
    auto d = svs::data::SimpleData<T, svs::Dynamic, svs::lib::Allocator<T>>(n, dim);
    const T* p = static_cast<const T*>(src);
    for (size_t i = 0; i < n; ++i) d.set_datum(i, std::span<const T>(p + i * dim, dim));
    return SQ<T>(std::move(d), scale, bias);
}

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

// f(data, distance) for the code type and metric.
template <typename F> void with_sq(int dtype, int metric, const void* codes, size_t n, size_t dim, float scale, float bias,
                                   F&& f) {
    auto run = [&](auto data) {
        switch (metric) {
            case L2: f(std::move(data), svs::distance::DistanceL2{}); break;
            case IP: f(std::move(data), svs::distance::DistanceIP{}); break;
            case COS: f(std::move(data), svs::distance::DistanceCosineSimilarity{}); break;
            default: throw ANNEXCEPTION("bad metric {}", metric);
        }
    };
    switch (dtype) {
        case I8: run(sq_of<int8_t>(codes, n, dim, scale, bias)); break;
        case U8: run(sq_of<uint8_t>(codes, n, dim, scale, bias)); break;
        default: throw ANNEXCEPTION("int8 / uint8 codes only, got dtype {}", dtype);
    }
}

}  // namespace

extern "C" {

const char* svsref_sq_build_last_error() { return g_error.c_str(); }

/// auto_build over SQDataset<int8_t> (dtype 2) or SQDataset<uint8_t> (dtype 3) codes with the given scale and bias.
/// Output layout = n x (max_degree + 1), degree first.
int svsref_sq_build(int dtype, const void* codes, size_t n, size_t dim, int metric, float scale, float bias, float alpha,
                    size_t max_degree, size_t window, size_t max_candidates, size_t prune_to, size_t threads,
                    uint32_t* graph_out, uint32_t* entry_point_out) {
    return guarded([&] {
        auto params = svs::index::vamana::VamanaBuildParameters{alpha, max_degree, window, max_candidates, prune_to, true};
        with_sq(dtype, metric, codes, n, dim, scale, bias, [&](auto data, auto dist) {
            auto index = svs::index::vamana::auto_build(params, std::move(data), dist, threads, svs::lib::Allocator<uint32_t>{});
            index.experimental_escape_hatch([&](const auto& graph, const auto&, const auto&, auto eps) {
                *entry_point_out = eps[0];
                for (size_t i = 0; i < n; ++i) {
                    auto nb = graph.get_node(i);
                    uint32_t* row = graph_out + i * (max_degree + 1);
                    row[0] = static_cast<uint32_t>(nb.size());
                    for (size_t j = 0; j < max_degree; ++j) row[1 + j] = j < nb.size() ? nb[j] : 0;
                }
            });
        });
    });
}

/// The builder's distance between datum pairs[2p] (the query, fixed as the builder fixes it) and datum pairs[2p + 1],
/// for `npairs` pairs: the general distance of the reference's build adaptor over the SQ dataset.
int svsref_sq_build_distance(int dtype, const void* codes, size_t n, size_t dim, int metric, float scale, float bias,
                             const uint32_t* pairs, size_t npairs, float* out) {
    return guarded([&] {
        with_sq(dtype, metric, codes, n, dim, scale, bias, [&](auto data, auto dist) {
            auto adaptor = svs::index::vamana::extensions::build_adaptor(data, dist);
            auto&& general = adaptor.general_distance();
            auto accessor = adaptor.general_accessor();
            for (size_t p = 0; p < npairs; ++p) {
                const size_t i = pairs[2 * p], j = pairs[2 * p + 1];
                if (i >= n || j >= n) throw ANNEXCEPTION("pair {} out of range", p);
                const auto query = accessor(data, i);
                svs::distance::maybe_fix_argument(general, query);
                out[p] = svs::distance::compute(general, query, accessor(data, j));
            }
        });
    });
}

}  // extern "C"
