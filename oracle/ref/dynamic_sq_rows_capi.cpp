// dynamic_sq_rows_capi.cpp -- TEST INFRASTRUCTURE ONLY.  The MutableVamanaIndex-over-SQDataset façade of
// dynamic_sq_capi.cpp, compiled unchanged into this translation unit, plus the index's stored-row reads on its handles:
//   index/vamana/dynamic_index.h:1306-1322  get_distance(external id, query)
//   index/vamana/dynamic_index.h:1152-1190  reconstruct_at(dst, external ids): its id check, then the rows.
// reconstruct_at itself cannot be called over SQDataset: its DecompressionAccessor (quantization/scalar/scalar.h:
// 607-620) holds a Decompressor whose output buffer is never sized (:337-355), so the first row is written out of
// bounds.  The rows are read through SQDataset::decompress_datum (:404-410) instead, which applies the same
// detail::decompress to every element.
#include "dynamic_sq_capi.cpp"

namespace {

template <typename F> void with_index(void* h, F&& f) {
    auto* base = static_cast<DynBase*>(h);
    bool done = false;
    auto attempt = [&](auto* impl) {
        if (!done && impl) {
            f(impl->index);
            done = true;
        }
    };
    attempt(dynamic_cast<DynImpl<int8_t, svs::distance::DistanceL2>*>(base));
    attempt(dynamic_cast<DynImpl<int8_t, svs::distance::DistanceIP>*>(base));
    attempt(dynamic_cast<DynImpl<int8_t, svs::distance::DistanceCosineSimilarity>*>(base));
    attempt(dynamic_cast<DynImpl<uint8_t, svs::distance::DistanceL2>*>(base));
    attempt(dynamic_cast<DynImpl<uint8_t, svs::distance::DistanceIP>*>(base));
    attempt(dynamic_cast<DynImpl<uint8_t, svs::distance::DistanceCosineSimilarity>*>(base));
    if (!done) throw ANNEXCEPTION("not a handle of this façade");
}

}  // namespace

extern "C" {

/// MutableVamanaIndex::get_distance(external_id, query) with a float32 query (fails for an id the index does not hold).
int svsref_dynamic_sq_get_distance(void* h, uint64_t id, const float* query, float* out) {
    return guarded([&] {
        with_index(h, [&](auto& index) {
            *out = static_cast<float>(index.get_distance(size_t(id), std::span<const float>(query, index.dimensions())));
        });
    });
}

/// The rows of `count` external ids as float32 (out[count][dim]), decompressed as scale * c + bias.
int svsref_dynamic_sq_reconstruct(void* h, const uint64_t* ids, size_t count, float* out) {
    return guarded([&] {
        with_index(h, [&](auto& index) {
            const size_t dim = index.dimensions();
            for (size_t i = 0; i < count; ++i)
                if (!index.has_id(ids[i])) throw ANNEXCEPTION("ID {} with value {} is out of bounds!", i, ids[i]);
            for (size_t i = 0; i < count; ++i) {
                const std::vector<float> row = index.view_data().decompress_datum(index.translate_external_id(ids[i]));
                std::memcpy(out + i * dim, row.data(), dim * sizeof(float));
            }
        });
    });
}

}  // extern "C"
