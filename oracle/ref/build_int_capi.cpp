// oracle/_ref driver for integer graph builds -- TEST INFRASTRUCTURE ONLY (see oracle/README.md).
//
// A thin `extern "C"` façade over the *unmodified* reference headers (`-I/root/reference/include`, never copied):
// the reference's graph construction over SimpleData<int8_t> / SimpleData<uint8_t>, whose default build adaptor
// uses the datum itself as the query (index/vamana/extensions.h:114-282), so every distance is int x int.
//
// Reference entry points exercised (file:line under /root/reference/include/svs):
//   index/vamana/index.h:968-994   auto_build (medoid entry point, two passes alpha = 1 then alpha)
//
// Nothing in the product (libsvsb200.so / scalablevectorsearch_b200) links or loads this.

#include "svs/core/data.h"
#include "svs/core/distance.h"
#include "svs/core/graph.h"
#include "svs/index/vamana/index.h"

#include <cstdint>
#include <span>
#include <string>

namespace {

thread_local std::string g_error;

enum DType : int { I8 = 2, U8 = 3 };
enum Metric : int { L2 = 0, IP = 1, COS = 2 };

template <typename T> using Data = svs::data::SimpleData<T, svs::Dynamic, svs::lib::Allocator<T>>;

template <typename T> Data<T> rows_of(const void* src, size_t n, size_t dim) {
    auto d = Data<T>(n, dim);
    const T* p = static_cast<const T*>(src);
    for (size_t i = 0; i < n; ++i) d.set_datum(i, std::span<const T>(p + i * dim, dim));
    return d;
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

}  // namespace

extern "C" {

const char* svsref_int_last_error() { return g_error.c_str(); }

/// auto_build over int8 (dtype 2) or uint8 (dtype 3) rows.  Output layout = n x (max_degree + 1), degree first.
int svsref_int_build(int dtype, const void* data, size_t n, size_t dim, int metric, float alpha, size_t max_degree,
                     size_t window, size_t max_candidates, size_t prune_to, size_t threads, uint32_t* graph_out,
                     uint32_t* entry_point_out) {
    return guarded([&] {
        auto params = svs::index::vamana::VamanaBuildParameters{alpha, max_degree, window, max_candidates, prune_to, true};
        auto extract = [&](const auto& index) {
            index.experimental_escape_hatch([&](const auto& graph, const auto&, const auto&, auto eps) {
                *entry_point_out = eps[0];
                for (size_t i = 0; i < n; ++i) {
                    auto nb = graph.get_node(i);
                    uint32_t* row = graph_out + i * (max_degree + 1);
                    row[0] = static_cast<uint32_t>(nb.size());
                    for (size_t j = 0; j < max_degree; ++j) row[1 + j] = j < nb.size() ? nb[j] : 0;
                }
            });
        };
        auto run = [&](auto rows) {
            auto alloc = svs::lib::Allocator<uint32_t>{};
            namespace vam = svs::index::vamana;
            switch (metric) {
                case L2: extract(vam::auto_build(params, std::move(rows), svs::distance::DistanceL2{}, threads, alloc)); break;
                case IP: extract(vam::auto_build(params, std::move(rows), svs::distance::DistanceIP{}, threads, alloc)); break;
                case COS:
                    extract(vam::auto_build(params, std::move(rows), svs::distance::DistanceCosineSimilarity{}, threads, alloc));
                    break;
                default: throw ANNEXCEPTION("bad metric {}", metric);
            }
        };
        switch (dtype) {
            case I8: run(rows_of<int8_t>(data, n, dim)); break;
            case U8: run(rows_of<uint8_t>(data, n, dim)); break;
            default: throw ANNEXCEPTION("int8 / uint8 data only, got dtype {}", dtype);
        }
    });
}

}  // extern "C"
