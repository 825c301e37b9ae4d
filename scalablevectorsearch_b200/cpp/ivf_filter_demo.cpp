// ivf_filter_demo.cpp -- a program written against the reference's runtime headers only
// (bindings/cpp/include/svs/runtime/ivf_index.h, dynamic_ivf_index.h), linked with libsvsb200_runtime.so instead of
// libsvs_runtime: filtered searches through an IDFilter.  Over the first n0 rows of a float file (L2) it builds an
// IVFIndex with FP32 storage and one with SQI8 storage, and a DynamicIVFIndex (FP32, labels 1000 + row) from which
// every third row is removed.  Each is searched with a range filter (ids, or labels, in [n0 / 4, n0 / 2) from its
// first id) and with a filter backed by a bitmap (a fixed pseudo-random 30 % of the ids).  The FP32 IVFIndex is also
// searched with a 10 % filter (id % 10 == 3) twice: with filter_stop = 0.5, which gives up on it, and with
// filter_estimate_batch = false and filter_stop = 0.05.  Every search prints its status code and its rows.
#include "svs/runtime/dynamic_ivf_index.h"
#include "svs/runtime/ivf_index.h"

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <utility>
#include <vector>

namespace rt = svs::runtime::v0;

struct RangeFilter final : rt::IDFilter {
    size_t lo, hi;
    RangeFilter(size_t l, size_t h) : lo(l), hi(h) {}
    bool is_member(size_t id) const override { return id >= lo && id < hi; }
};

struct BitmapFilter final : rt::IDFilter {
    std::vector<uint64_t> words;
    bool is_member(size_t id) const override { return id / 64 < words.size() && (words[id / 64] >> (id % 64)) & 1u; }
};

struct TenPercentFilter final : rt::IDFilter {
    bool is_member(size_t id) const override { return id % 10 == 3; }
};

// bit i set for a fixed 30 % of i in [0, count): (i * 2654435761 mod 2^32) >> 22 below 0.3 * 1024
BitmapFilter thirty_percent(size_t count) {
    BitmapFilter f;
    f.words.assign((count + 63) / 64, 0);
    for (size_t i = 0; i < count; ++i)
        if ((uint32_t(i * 2654435761u) >> 22) < 307) f.words[i / 64] |= uint64_t(1) << (i % 64);
    return f;
}

int main(int argc, char** argv) {
    if (argc != 11) {
        std::fprintf(stderr,
                     "usage: %s <data.f32> <n> <dim> <queries.f32> <nq> <k> <centroids> <iterations> <n_probes> <n0>\n",
                     argv[0]);
        return 2;
    }
    const size_t n = std::strtoul(argv[2], nullptr, 10), dim = std::strtoul(argv[3], nullptr, 10);
    const size_t nq = std::strtoul(argv[5], nullptr, 10), k = std::strtoul(argv[6], nullptr, 10);
    const size_t n0 = std::strtoul(argv[10], nullptr, 10);
    std::vector<float> data(n * dim), queries(nq * dim);
    FILE* f = std::fopen(argv[1], "rb");
    if (!f || std::fread(data.data(), 4, n * dim, f) != n * dim) return 3;
    std::fclose(f);
    f = std::fopen(argv[4], "rb");
    if (!f || std::fread(queries.data(), 4, nq * dim, f) != nq * dim) return 3;
    std::fclose(f);
    auto check = [](const rt::Status& st) {
        if (!st.ok()) {
            std::fprintf(stderr, "error: %s\n", st.message());
            std::exit(1);
        }
    };
    rt::IVFIndex::BuildParams bp;
    bp.num_centroids = std::strtoul(argv[7], nullptr, 10);
    bp.num_iterations = std::strtoul(argv[8], nullptr, 10);
    bp.is_hierarchical = false;
    rt::IVFIndex::SearchParams sp;
    sp.n_probes = std::strtoul(argv[9], nullptr, 10);
    std::vector<float> d(nq * k);
    std::vector<size_t> l(nq * k);
    auto print = [&](const char* tag, const rt::Status& st) {
        std::printf("%s status %d\n", tag, int(st.code));
        for (size_t i = 0; i < nq * k; ++i) std::printf("%s %zu %.9g\n", tag, l[i], d[i]);
    };
    RangeFilter range(n0 / 4, n0 / 2);
    BitmapFilter bitmap = thirty_percent(n0);

    for (auto [name, kind] : {std::pair{"fp32", rt::StorageKind::FP32}, std::pair{"sqi8", rt::StorageKind::SQI8}}) {
        rt::IVFIndex* ivf = nullptr;
        check(rt::IVFIndex::build(&ivf, dim, rt::MetricType::L2, kind, n0, data.data(), bp, sp));
        const std::string tag(name);
        print((tag + "_range").c_str(), ivf->search(nq, queries.data(), k, d.data(), l.data(), nullptr, &range));
        print((tag + "_bitmap").c_str(), ivf->search(nq, queries.data(), k, d.data(), l.data(), nullptr, &bitmap));
        if (kind == rt::StorageKind::FP32) {
            TenPercentFilter ten;
            rt::IVFIndex::SearchParams stop;
            stop.filter_stop = 0.5f;   // the sampled hit rate (about 0.1) is below it: every row padded, status OK
            print("stop", ivf->search(nq, queries.data(), k, d.data(), l.data(), &stop, &ten));
            rt::IVFIndex::SearchParams no_estimate;
            no_estimate.filter_estimate_batch = false;
            no_estimate.filter_stop = 0.05f;   // per query: padded where the probed clusters' hit rate is below it
            print("no_estimate", ivf->search(nq, queries.data(), k, d.data(), l.data(), &no_estimate, &ten));
        }
        rt::IVFIndex::destroy(ivf);
    }

    std::vector<size_t> labels(n0);
    for (size_t i = 0; i < n0; ++i) labels[i] = 1000 + i;
    rt::DynamicIVFIndex* dyn = nullptr;
    check(rt::DynamicIVFIndex::build(&dyn, dim, rt::MetricType::L2, rt::StorageKind::FP32, n0, data.data(), labels.data(),
                                     bp, sp));
    std::vector<size_t> gone;
    for (size_t i = 0; i < n0; i += 3) gone.push_back(labels[i]);
    check(dyn->remove(gone.size(), gone.data()));
    RangeFilter dyn_range(1000 + n0 / 4, 1000 + n0 / 2);
    BitmapFilter dyn_bitmap = thirty_percent(1000 + n0);
    print("dynamic_range", dyn->search(nq, queries.data(), k, d.data(), l.data(), nullptr, &dyn_range));
    print("dynamic_bitmap", dyn->search(nq, queries.data(), k, d.data(), l.data(), nullptr, &dyn_bitmap));
    rt::DynamicIVFIndex::destroy(dyn);
    return 0;
}
