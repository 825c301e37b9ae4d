// ivf_sq_demo.cpp -- a program written against the reference's runtime headers only
// (bindings/cpp/include/svs/runtime/ivf_index.h, dynamic_ivf_index.h), linked with libsvsb200_runtime.so instead of
// libsvs_runtime, over SQI8 storage (int8 codes with one global scale and bias).  It builds an IVFIndex (L2) over the
// first n0 rows of a float file and prints the top-k of every query at the given n_probes.  It builds a DynamicIVFIndex
// without rows, fills it by one add of the same n0 rows (labels 1000 + row) and prints its top-k; then a
// DynamicIVFIndex over those rows, removes every third of them, adds the remaining rows with reuse_empty, removes the
// labels divisible by 7 through an IDFilter, compacts and prints its top-k.  It also prints check_storage_kind(SQI8)
// of both classes and the status of a build over constant rows, which cannot be compressed.
#include "svs/runtime/dynamic_ivf_index.h"
#include "svs/runtime/ivf_index.h"

#include <cstdio>
#include <cstdlib>
#include <vector>

namespace rt = svs::runtime::v0;

struct SevenFilter final : rt::IDFilter {
    bool is_member(size_t id) const override { return id % 7 == 0; }
};

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
    std::vector<size_t> labels(n);
    for (size_t i = 0; i < n; ++i) labels[i] = 1000 + i;
    auto code = [](const rt::Status& st) { return int(st.code); };
    auto check = [](const rt::Status& st) {
        if (!st.ok()) {
            std::fprintf(stderr, "error: %s\n", st.message());
            std::exit(1);
        }
    };
    const auto SQ = rt::StorageKind::SQI8;
    std::printf("storage_sqi8 %d %d\n", code(rt::IVFIndex::check_storage_kind(SQ)),
                code(rt::DynamicIVFIndex::check_storage_kind(SQ)));
    rt::IVFIndex::BuildParams bp;
    bp.num_centroids = std::strtoul(argv[7], nullptr, 10);
    bp.num_iterations = std::strtoul(argv[8], nullptr, 10);
    bp.is_hierarchical = false;
    rt::IVFIndex::SearchParams sp;
    sp.n_probes = std::strtoul(argv[9], nullptr, 10);
    std::vector<float> d(nq * k);
    std::vector<size_t> l(nq * k);

    // constant rows have no SQ scale: an error status, no index
    const std::vector<float> flat(n0 * dim, 1.5f);
    rt::IVFIndex* refused = nullptr;
    std::printf("constant %d %d\n", code(rt::IVFIndex::build(&refused, dim, rt::MetricType::L2, SQ, n0, flat.data(), bp, sp)),
                int(refused == nullptr));

    rt::IVFIndex* ivf = nullptr;
    check(rt::IVFIndex::build(&ivf, dim, rt::MetricType::L2, SQ, n0, data.data(), bp, sp));
    check(ivf->search(nq, queries.data(), k, d.data(), l.data()));
    for (size_t i = 0; i < nq * k; ++i) std::printf("ivf %zu %.9g\n", l[i], d[i]);
    rt::IVFIndex::destroy(ivf);

    rt::DynamicIVFIndex* empty = nullptr;
    check(rt::DynamicIVFIndex::build(&empty, dim, rt::MetricType::L2, SQ, 0, nullptr, nullptr, bp, sp));
    check(empty->add(n0, labels.data(), data.data()));   // clusters and compresses its own rows
    check(empty->search(nq, queries.data(), k, d.data(), l.data()));
    for (size_t i = 0; i < nq * k; ++i) std::printf("initial %zu %.9g\n", l[i], d[i]);
    rt::DynamicIVFIndex::destroy(empty);

    rt::DynamicIVFIndex* index = nullptr;
    check(rt::DynamicIVFIndex::build(&index, dim, rt::MetricType::L2, SQ, n0, data.data(), labels.data(), bp, sp));
    std::vector<size_t> gone;
    for (size_t i = 0; i < n0; i += 3) gone.push_back(labels[i]);
    check(index->remove(gone.size(), gone.data()));
    check(index->add(n - n0, labels.data() + n0, data.data() + n0 * dim, true));   // float32 rows, encoded
    size_t removed = 0;
    check(index->remove_selected(&removed, SevenFilter{}));
    std::printf("removed %zu\n", removed);
    check(index->consolidate());
    check(index->compact());
    check(index->search(nq, queries.data(), k, d.data(), l.data()));
    for (size_t i = 0; i < nq * k; ++i) std::printf("result %zu %.9g\n", l[i], d[i]);
    rt::DynamicIVFIndex::destroy(index);
    return 0;
}
