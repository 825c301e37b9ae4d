// flat_demo.cpp -- a program written against the reference's runtime header only
// (bindings/cpp/include/svs/runtime/flat_index.h), linked with libsvsb200_runtime.so instead of libsvs_runtime:
// builds a FlatIndex from a float file and prints the exact top-k of every query, plus the status codes of the calls
// the runtime defines as errors, so that a test can compare them.
#include "svs/runtime/flat_index.h"

#include <cstdio>
#include <cstdlib>
#include <vector>

namespace rt = svs::runtime::v0;

int main(int argc, char** argv) {
    if (argc != 7) {
        std::fprintf(stderr, "usage: %s <data.f32> <n> <dim> <queries.f32> <nq> <k>\n", argv[0]);
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
    auto code = [](const rt::Status& st) { return int(st.code); };
    std::printf("storage_fp16 %d\n", code(rt::FlatIndex::check_storage_kind(rt::StorageKind::FP16)));
    rt::FlatIndex* index = nullptr;
    rt::Status st = rt::FlatIndex::build(&index, dim, rt::MetricType::L2);
    if (!st.ok()) {
        std::fprintf(stderr, "error: %s\n", st.message());
        return 1;
    }
    std::vector<float> d(nq * k);
    std::vector<size_t> l(nq * k);
    st = index->search(nq, queries.data(), k, d.data(), l.data());
    std::printf("search_before_add %d %zu %g\n", code(st), l[0], d[0]);
    st = index->add(n, data.data());
    if (!st.ok()) {
        std::fprintf(stderr, "error: %s\n", st.message());
        return 1;
    }
    std::printf("second_add %d\n", code(index->add(n, data.data())));
    std::printf("k0 %d\n", code(index->search(nq, queries.data(), 0, d.data(), l.data())));
    st = index->search(nq, queries.data(), k, d.data(), l.data());
    if (!st.ok()) {
        std::fprintf(stderr, "error: %s\n", st.message());
        return 1;
    }
    for (size_t i = 0; i < nq * k; ++i) std::printf("result %zu %.9g\n", l[i], d[i]);
    rt::FlatIndex::destroy(index);
    return 0;
}
