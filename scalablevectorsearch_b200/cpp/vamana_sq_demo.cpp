// vamana_sq_demo.cpp -- a program written against the reference's runtime headers only
// (bindings/cpp/include/svs/runtime/vamana_index.h), linked with libsvsb200_runtime.so instead of libsvs_runtime, over
// SQI8 storage (int8 codes with one global scale and bias).  It builds a VamanaIndex over n float32 rows of a file
// (metric 0 = L2, 1 = inner product; graph degree R, construction window W), adds the rows and prints, for every query:
// the top-k, the top-k through an IDFilter that admits the ids divisible by 3, and the range search at `radius`.  It
// then prints the reconstruction of rows 0..3 and get_distance of the first query to rows 0..7.  It also prints
// check_storage_kind(SQI8) and the status of an add of constant rows, which cannot be compressed.
#include "svs/runtime/vamana_index.h"

#include <cstdio>
#include <cstdlib>
#include <vector>

namespace rt = svs::runtime::v0;

struct ThreeFilter final : rt::IDFilter {
    bool is_member(size_t id) const override { return id % 3 == 0; }
};

struct Results final : rt::ResultsAllocator {
    std::vector<size_t> labels;
    std::vector<float> distances;
    std::vector<size_t> counts;
    rt::SearchResultsStorage allocate(std::span<size_t> result_counts) const override {
        auto* self = const_cast<Results*>(this);
        size_t total = 0;
        for (size_t c : result_counts) total += c;
        self->counts.assign(result_counts.begin(), result_counts.end());
        self->labels.resize(total);
        self->distances.resize(total);
        return rt::SearchResultsStorage{std::span<size_t>(self->labels), std::span<float>(self->distances)};
    }
};

int main(int argc, char** argv) {
    if (argc != 11) {
        std::fprintf(stderr, "usage: %s <data.f32> <n> <dim> <queries.f32> <nq> <k> <metric> <R> <W> <radius>\n", argv[0]);
        return 2;
    }
    const size_t n = std::strtoul(argv[2], nullptr, 10), dim = std::strtoul(argv[3], nullptr, 10);
    const size_t nq = std::strtoul(argv[5], nullptr, 10), k = std::strtoul(argv[6], nullptr, 10);
    const auto metric = std::atoi(argv[7]) == 0 ? rt::MetricType::L2 : rt::MetricType::INNER_PRODUCT;
    const float radius = std::strtof(argv[10], nullptr);
    std::vector<float> data(n * dim), queries(nq * dim);
    FILE* f = std::fopen(argv[1], "rb");
    if (!f || std::fread(data.data(), 4, n * dim, f) != n * dim) return 3;
    std::fclose(f);
    f = std::fopen(argv[4], "rb");
    if (!f || std::fread(queries.data(), 4, nq * dim, f) != nq * dim) return 3;
    std::fclose(f);
    auto code = [](const rt::Status& st) { return int(st.code); };
    auto check = [](const rt::Status& st) {
        if (!st.ok()) {
            std::fprintf(stderr, "error: %s\n", st.message());
            std::exit(1);
        }
    };
    const auto SQ = rt::StorageKind::SQI8;
    std::printf("storage_sqi8 %d\n", code(rt::VamanaIndex::check_storage_kind(SQ)));
    rt::VamanaIndex::BuildParams bp;
    bp.graph_max_degree = std::strtoul(argv[8], nullptr, 10);
    bp.construction_window_size = std::strtoul(argv[9], nullptr, 10);
    rt::VamanaIndex::SearchParams sp;
    sp.search_window_size = 2 * k;

    // constant rows have no SQ scale: an error status, no index
    rt::VamanaIndex* refused = nullptr;
    check(rt::VamanaIndex::build(&refused, dim, metric, SQ, bp, sp));
    const std::vector<float> flat(n * dim, 1.5f);
    std::printf("constant %d\n", code(refused->add(n, flat.data())));
    rt::VamanaIndex::destroy(refused);

    rt::VamanaIndex* index = nullptr;
    check(rt::VamanaIndex::build(&index, dim, metric, SQ, bp, sp));
    check(index->add(n, data.data()));
    std::vector<float> d(nq * k);
    std::vector<size_t> l(nq * k);
    check(index->search(nq, queries.data(), k, d.data(), l.data()));
    for (size_t i = 0; i < nq * k; ++i) std::printf("search %zu %.9g\n", l[i], d[i]);
    ThreeFilter three;
    check(index->search(nq, queries.data(), k, d.data(), l.data(), nullptr, &three));
    for (size_t i = 0; i < nq * k; ++i) std::printf("filtered %zu %.9g\n", l[i], d[i]);
    Results range;
    check(index->range_search(nq, queries.data(), radius, range));
    for (size_t q = 0, o = 0; q < nq; ++q)
        for (size_t j = 0; j < range.counts[q]; ++j, ++o) std::printf("range %zu %zu %.9g\n", q, range.labels[o], range.distances[o]);
    const size_t rows[4] = {0, 1, 2, 3};
    std::vector<float> back(4 * dim);
    check(index->reconstruct_at(4, rows, back.data()));
    for (float v : back) std::printf("reconstruct %.9g\n", v);
    for (size_t id = 0; id < 8; ++id) {
        float dist = 0.f;
        check(index->get_distance(id, queries.data(), &dist));
        std::printf("distance %zu %.9g\n", id, dist);
    }
    rt::MemoryBreakdown mem{};
    check(index->get_memory_breakdown(&mem));
    std::printf("memory %zu %zu\n", mem.graph_bytes, mem.data_bytes);
    rt::VamanaIndex::destroy(index);
    return 0;
}
