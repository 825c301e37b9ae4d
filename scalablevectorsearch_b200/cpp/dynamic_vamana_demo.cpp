// dynamic_vamana_demo.cpp -- a program written against the reference's runtime header only
// (bindings/cpp/include/svs/runtime/dynamic_vamana_index.h), linked with libsvsb200_runtime.so instead of libsvs_runtime.
// It builds an empty DynamicVamanaIndex of the given storage kind (L2), adds row 0 alone, then rows [1, n/2) and
// [n/2, n) with labels 1000 + row, and prints a plain, an IDFilter and a range search; removes the labels whose row is a
// multiple of 10 (below the clean-up threshold) and then the odd labels (above it: the index consolidates and compacts),
// and then the multiples of 7 through remove_selected; searches again, prints get_distance and reconstruct_at of a few
// labels, the memory breakdown, and after reset and a rebuild from all rows, one more search.  It also prints the status
// codes of calls the GPU index refuses, so that a test can compare everything with the C ABI.
#include "svs/runtime/dynamic_vamana_index.h"

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

namespace rt = svs::runtime::v0;

struct ThreeFilter final : rt::IDFilter {
    bool is_member(size_t id) const override { return id % 3 == 0; }
};
struct SevenFilter final : rt::IDFilter {
    bool is_member(size_t id) const override { return id % 7 == 0; }
};

// range search results, kept per query
struct Ranges : rt::ResultsAllocator {
    mutable std::vector<size_t> labels;
    mutable std::vector<float> distances;
    mutable std::vector<size_t> counts;
    rt::SearchResultsStorage allocate(std::span<size_t> result_counts) const override {
        counts.assign(result_counts.begin(), result_counts.end());
        size_t total = 0;
        for (size_t c : counts) total += c;
        labels.assign(total, 0);
        distances.assign(total, 0.f);
        return rt::SearchResultsStorage{std::span<size_t>(labels), std::span<float>(distances)};
    }
};

int main(int argc, char** argv) {
    if (argc != 11) {
        std::fprintf(stderr,
                     "usage: %s <data.f32> <n> <dim> <queries.f32> <nq> <k> <fp32|fp16|sqi8> <graph_max_degree> "
                     "<construction_window> <radius>\n",
                     argv[0]);
        return 2;
    }
    const size_t n = std::strtoul(argv[2], nullptr, 10), dim = std::strtoul(argv[3], nullptr, 10);
    const size_t nq = std::strtoul(argv[5], nullptr, 10), k = std::strtoul(argv[6], nullptr, 10);
    const rt::StorageKind kind = std::strcmp(argv[7], "fp16") == 0   ? rt::StorageKind::FP16
                                 : std::strcmp(argv[7], "sqi8") == 0 ? rt::StorageKind::SQI8
                                                                     : rt::StorageKind::FP32;
    const float radius = std::strtof(argv[10], nullptr);
    std::vector<float> data(n * dim), queries(nq * dim);
    FILE* f = std::fopen(argv[1], "rb");
    if (!f || std::fread(data.data(), 4, n * dim, f) != n * dim) return 3;
    std::fclose(f);
    f = std::fopen(argv[4], "rb");
    if (!f || std::fread(queries.data(), 4, nq * dim, f) != nq * dim) return 3;
    std::fclose(f);
    std::vector<size_t> labels(n);
    for (size_t i = 0; i < n; ++i) labels[i] = 1000 + i;
    auto code = [](const rt::Status& st) { return int(st.code); };
    auto check = [](const rt::Status& st) {
        if (!st.ok()) {
            std::fprintf(stderr, "error: %s\n", st.message());
            std::exit(1);
        }
    };
    rt::VamanaIndex::BuildParams bp;
    bp.graph_max_degree = std::strtoul(argv[8], nullptr, 10);
    bp.construction_window_size = std::strtoul(argv[9], nullptr, 10);
    rt::VamanaIndex::SearchParams sp;
    sp.search_window_size = 2 * k;
    std::vector<float> d(nq * k);
    std::vector<size_t> l(nq * k);
    auto print_search = [&](const char* tag) {
        for (size_t i = 0; i < nq * k; ++i) std::printf("%s %zu %.9g\n", tag, l[i], d[i]);
    };

    // refusals
    rt::DynamicVamanaIndex* refused = nullptr;
    std::printf("storage_lvq8 %d\n", code(rt::DynamicVamanaIndex::check_storage_kind(rt::StorageKind::LVQ8x0)));
    std::printf("build_lvq8 %d\n", code(rt::DynamicVamanaIndex::build(&refused, dim, rt::MetricType::L2, rt::StorageKind::LVQ8x0)));
    std::printf("build_leanvec %d\n",
                code(rt::DynamicVamanaIndexLeanVec::build(&refused, dim, rt::MetricType::L2, rt::StorageKind::LeanVec4x4, 16)));
    rt::VamanaIndex::DynamicIndexParams small, large;
    small.blocksize_exp = 11;
    large.blocksize_exp = 31;
    std::printf("blocksize %d %d\n", code(rt::DynamicVamanaIndex::check_params(small)),
                code(rt::DynamicVamanaIndex::build(&refused, dim, rt::MetricType::L2, kind, bp, sp, large)));

    rt::DynamicVamanaIndex* index = nullptr;
    rt::VamanaIndex::DynamicIndexParams dp;
    dp.blocksize_exp = 20;
    check(rt::DynamicVamanaIndex::build(&index, dim, rt::MetricType::L2, kind, bp, sp, dp));
    std::printf("blocksize_bytes %zu\n", index->blocksize_bytes());
    const int uninit = code(index->search(nq, queries.data(), k, d.data(), l.data()));
    std::printf("uninit %d %zu\n", uninit, l[0]);
    std::printf("add_nolabels %d\n", code(static_cast<rt::VamanaIndex*>(index)->add(n, data.data())));

    const size_t half = n / 2;
    check(index->add(1, labels.data(), data.data()));   // one row: no graph to build yet
    check(index->add(half - 1, labels.data() + 1, data.data() + dim));
    check(index->add(n - half, labels.data() + half, data.data() + half * dim));
    check(index->search(nq, queries.data(), k, d.data(), l.data()));
    print_search("plain");
    std::printf("k0 %d\n", code(index->search(nq, queries.data(), 0, d.data(), l.data())));
    ThreeFilter three;
    check(index->search(nq, queries.data(), k, d.data(), l.data(), nullptr, &three));
    print_search("filtered");
    Ranges ranges;
    check(index->range_search(nq, queries.data(), radius, ranges, nullptr, &three));
    for (size_t q = 0, o = 0; q < nq; ++q)
        for (size_t j = 0; j < ranges.counts[q]; ++j, ++o) std::printf("range %zu %zu %.9g\n", q, ranges.labels[o], ranges.distances[o]);
    std::printf("range0 %d\n", code(index->range_search(nq, queries.data(), 0.f, ranges)));

    std::vector<size_t> tens, odd;
    for (size_t i = 0; i < n; i += 10) tens.push_back(labels[i]);
    check(index->remove(tens.size(), tens.data()));   // soft deletions below half of what is left
    std::printf("memory_remove1 %zu\n", index->get_memory_usage());
    for (size_t i = 1; i < n; i += 2)
        if (i % 10 != 0) odd.push_back(labels[i]);
    check(index->remove(odd.size(), odd.data()));   // above half: consolidate and compact
    std::printf("memory_remove2 %zu\n", index->get_memory_usage());
    size_t removed = 0;
    check(index->remove_selected(&removed, SevenFilter{}));
    std::printf("removed %zu\n", removed);
    check(index->search(nq, queries.data(), k, d.data(), l.data()));
    print_search("after");

    // stored rows: labels 1002, 1004, ... (kept), against query 0
    for (size_t i = 2; i < 40; i += 2) {
        if (labels[i] % 7 == 0 || i % 10 == 0) continue;
        float dist = 0.f;
        check(index->get_distance(labels[i], queries.data(), &dist));
        std::printf("distance %zu %.9g\n", labels[i], dist);
    }
    float unused = -1.f;
    std::printf("distance_removed %d %.9g\n", code(index->get_distance(labels[1], queries.data(), &unused)), unused);
    const size_t some[3] = {labels[2], labels[4], labels[6]};
    std::vector<float> rows(3 * dim);
    check(index->reconstruct_at(3, some, rows.data()));
    for (size_t i = 0; i < 3; ++i)
        for (size_t e = 0; e < dim; ++e) std::printf("row %zu %.9g\n", some[i], rows[i * dim + e]);
    rt::MemoryBreakdown mb;
    check(index->get_memory_breakdown(&mb));
    std::printf("memory %zu %zu %zu %zu\n", index->get_memory_usage(), mb.graph_bytes, mb.data_bytes, mb.metadata_bytes);

    check(index->reset());
    std::printf("reset %d %zu\n", code(index->search(nq, queries.data(), k, d.data(), l.data())), index->get_memory_usage());
    check(index->add(n, labels.data(), data.data()));
    check(index->search(nq, queries.data(), k, d.data(), l.data()));
    print_search("rebuilt");
    rt::DynamicVamanaIndex::destroy(index);
    return 0;
}
