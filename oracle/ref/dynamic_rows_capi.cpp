// dynamic_rows_capi.cpp -- TEST INFRASTRUCTURE ONLY.  The MutableVamanaIndex façade of dynamic_capi.cpp, compiled
// unchanged into this translation unit, plus the index's stored-row reads on its handles:
//   index/vamana/dynamic_index.h:1152-1190  reconstruct_at(dst, external ids)
//   index/vamana/dynamic_index.h:1306-1322  get_distance(external id, query)
// over float32 / float16 rows, for every metric the façade builds.
#include "dynamic_capi.cpp"

namespace {

// f(handle's MutableVamanaIndex), whichever of the façade's instantiations the handle holds.
template <typename F> void with_index(void* h, F&& f) {
    auto* base = static_cast<DynBase*>(h);
    bool done = false;
    auto attempt = [&](auto* impl) {
        if (!done && impl) {
            f(impl->index);
            done = true;
        }
    };
    attempt(dynamic_cast<DynImpl<float, svs::distance::DistanceL2>*>(base));
    attempt(dynamic_cast<DynImpl<float, svs::distance::DistanceIP>*>(base));
    attempt(dynamic_cast<DynImpl<float, svs::distance::DistanceCosineSimilarity>*>(base));
    attempt(dynamic_cast<DynImpl<svs::Float16, svs::distance::DistanceL2>*>(base));
    attempt(dynamic_cast<DynImpl<svs::Float16, svs::distance::DistanceIP>*>(base));
    attempt(dynamic_cast<DynImpl<svs::Float16, svs::distance::DistanceCosineSimilarity>*>(base));
    if (!done) throw ANNEXCEPTION("not a handle of this façade");
}

}  // namespace

extern "C" {

/// MutableVamanaIndex::get_distance(external_id, query) with a float32 query (fails for an id the index does not hold).
int svsref_dynamic_get_distance(void* h, uint64_t id, const float* query, float* out) {
    return guarded([&] {
        with_index(h, [&](auto& index) {
            *out = static_cast<float>(index.get_distance(size_t(id), std::span<const float>(query, index.dimensions())));
        });
    });
}

/// MutableVamanaIndex::reconstruct_at: `count` rows by external id as float32 (out[count][dim]).
int svsref_dynamic_reconstruct(void* h, const uint64_t* ids, size_t count, float* out) {
    return guarded([&] {
        with_index(h, [&](auto& index) {
            auto dst = svs::data::SimpleDataView<float>(out, count, index.dimensions());
            index.reconstruct_at(dst, std::span<const uint64_t>(ids, count));
        });
    });
}

}  // extern "C"
