// ivf_hier_demo.cpp -- a program written against the reference's runtime header only
// (bindings/cpp/include/svs/runtime/ivf_index.h), linked with libsvsb200_runtime.so instead of libsvs_runtime: builds an
// IVFIndex with is_hierarchical = true (the reference's default clustering) over a float file, once with FP32 and once
// with SQI8 storage, and prints the top-k of every query at the given n_probes for each, so that a test can compare
// them with the C ABI.
#include "svs/runtime/ivf_index.h"

#include <cstdio>
#include <cstdlib>
#include <vector>

namespace rt = svs::runtime::v0;

int main(int argc, char** argv) {
    if (argc != 11) {
        std::fprintf(stderr,
                     "usage: %s <data.f32> <n> <dim> <queries.f32> <nq> <k> <centroids> <level1 clusters> <iterations> "
                     "<n_probes>\n",
                     argv[0]);
        return 2;
    }
    const size_t n = std::strtoul(argv[2], nullptr, 10), dim = std::strtoul(argv[3], nullptr, 10);
    const size_t nq = std::strtoul(argv[5], nullptr, 10), k = std::strtoul(argv[6], nullptr, 10);
    std::vector<float> data(n * dim), queries(nq * dim);
    FILE* f = std::fopen(argv[1], "rb");
    if (!f || std::fread(data.data(), 4, n * dim, f) != n * dim) return 3;
    std::fclose(f);
    f = std::fopen(argv[4], "rb");
    if (!f || std::fread(queries.data(), 4, nq * dim, f) != nq * dim) return 3;
    std::fclose(f);
    rt::IVFIndex::BuildParams bp;
    bp.num_centroids = std::strtoul(argv[7], nullptr, 10);
    bp.hierarchical_level1_clusters = std::strtoul(argv[8], nullptr, 10);
    bp.num_iterations = std::strtoul(argv[9], nullptr, 10);
    bp.is_hierarchical = true;
    rt::IVFIndex::SearchParams sp;
    sp.n_probes = std::strtoul(argv[10], nullptr, 10);
    const struct {
        const char* tag;
        rt::StorageKind kind;
    } storages[] = {{"fp32", rt::StorageKind::FP32}, {"sqi8", rt::StorageKind::SQI8}};
    for (const auto& s : storages) {
        rt::IVFIndex* index = nullptr;
        rt::Status st = rt::IVFIndex::build(&index, dim, rt::MetricType::L2, s.kind, n, data.data(), bp, sp);
        if (!st.ok()) {
            std::fprintf(stderr, "error: %s\n", st.message());
            return 1;
        }
        std::vector<float> d(nq * k);
        std::vector<size_t> l(nq * k);
        st = index->search(nq, queries.data(), k, d.data(), l.data());
        if (!st.ok()) {
            std::fprintf(stderr, "error: %s\n", st.message());
            return 1;
        }
        for (size_t i = 0; i < nq * k; ++i) std::printf("%s %zu %.9g\n", s.tag, l[i], d[i]);
        rt::IVFIndex::destroy(index);
    }
    return 0;
}
