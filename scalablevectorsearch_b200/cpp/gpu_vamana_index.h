// gpu_vamana_index.h -- C++ host side of the drop-in boundary (SURVEY.md §8b).
//
// `svsb200::GpuVamanaIndex<Graph, Data, Dist>` is the reference's static Vamana index
// (include/svs/index/vamana/index.h:276-942) with its *batch search* re-pointed at
// libsvsb200.so.  It derives from the reference class, so every member the orchestrator
// needs (`orchestrators/vamana.h:127-275`, `orchestrators/manager.h:130-186`: parameters,
// save, reconstruct_at, calibrate, get_distance, batch iterators ...) is the reference's own
// code, unmodified, and only
//
//     search(QueryResultView<I>, queries, VamanaSearchParameters, cancel)   (index.h:564-611)
//
// is replaced.  `ManagerImpl::search` calls `impl().search(...)` on the static type
// (`manager.h:141-166` -> `index/index.h:44-55`), so type-erasing it with the reference's own
// `VamanaImpl` / `svs::Vamana` (`orchestrators/vamana.h:108-276,293-305`)
//
//     svs::Vamana v = svsb200::make_gpu_vamana<svs::lib::Types<float>>(
//         svsb200::GpuVamanaIndex{std::move(cpu_index), /*device=*/0});
//
// yields a stock `svs::Vamana` whose `search` runs on the GPU -- the object that
// `utils/search_index.cpp`, `bindings/python` and `bindings/cpp` hold.  (`svs::make_vamana`
// itself cannot be used: it re-deduces `VamanaIndex{args...}` and would slice to the CPU base,
// `orchestrators/vamana.h:711-715`.)
//
// This header compiles against the reference headers (`-I<reference>/include`); it contains
// no reference code.  Errors from the C ABI are rethrown as svs::ANNException
// (include/svs/lib/exception.h), the reference's own convention.
#pragma once

#include "svs/index/vamana/index.h"
#include "svs/orchestrators/vamana.h"
#include "svs/quantization/scalar/scalar.h"

#include "svsb200.h"

#include <memory>
#include <type_traits>
#include <vector>

namespace svsb200 {

namespace detail {
template <typename T> struct DTypeCode;
template <> struct DTypeCode<float> { static constexpr int value = SVSB200_F32; };
template <> struct DTypeCode<svs::Float16> { static constexpr int value = SVSB200_F16; };
template <> struct DTypeCode<int8_t> { static constexpr int value = SVSB200_I8; };
template <> struct DTypeCode<uint8_t> { static constexpr int value = SVSB200_U8; };

template <typename Dist> struct MetricCode;
template <> struct MetricCode<svs::distance::DistanceL2> { static constexpr int value = SVSB200_L2; };
template <> struct MetricCode<svs::distance::DistanceIP> { static constexpr int value = SVSB200_IP; };
template <> struct MetricCode<svs::distance::DistanceCosineSimilarity> {
    static constexpr int value = SVSB200_COSINE;
};

struct HandleDeleter {
    void operator()(svsb200_index* p) const { svsb200_index_destroy(p); }
};

inline void check(int rc) {
    if (rc != 0) {
        throw ANNEXCEPTION("svsb200: {}", svsb200_last_error());
    }
}
} // namespace detail

template <typename Graph, typename Data, typename Dist>
class GpuVamanaIndex : public svs::index::vamana::VamanaIndex<Graph, Data, Dist> {
  public:
    using base_type = svs::index::vamana::VamanaIndex<Graph, Data, Dist>;
    using search_parameters_type = typename base_type::search_parameters_type;

    /// Take over an assembled (or freshly built) CPU index and mirror its graph and vectors
    /// into the HBM of `device`.  The host copies stay alive for the non-search members.
    explicit GpuVamanaIndex(base_type&& cpu, int device = 0)
        : GpuVamanaIndex(std::move(cpu), std::vector<int>{device}) {}

    /// The same, replicated on several GPUs: every batch is split with the reference's own
    /// `threads::balance` (lib/threads/types.h:311-329), one slice per device -- the multi-device form of
    /// the thread-pool partition in index.h:571-574.
    GpuVamanaIndex(base_type&& cpu, const std::vector<int>& devices)
        : base_type(std::move(cpu)) {
        this->experimental_escape_hatch([&](const auto& graph,
                                            const auto& data,
                                            const auto& /*distance*/,
                                            auto entry_points) {
            if (entry_points.empty() || entry_points.size() > 32) {
                throw ANNEXCEPTION("GpuVamanaIndex takes 1 to 32 entry points");
            }
            const auto& rows = graph.get_data(); // uint32[n][max_degree + 1], degree first
            svsb200_index* raw = nullptr;
            if constexpr (svs::quantization::scalar::IsSQData<Data>) {
                using E = typename Data::element_type;
                const float aux[2] = {data.get_scale(), data.get_bias()};
                detail::check(svsb200_index_create_multi(
                    data.get_datum(0).data(),
                    detail::DTypeCode<E>::value,
                    data.size(),
                    data.dimensions(),
                    0,
                    rows.data(),
                    rows.dimensions(),
                    entry_points[0],
                    detail::MetricCode<Dist>::value,
                    SVSB200_SQ,
                    aux,
                    devices.data(),
                    devices.size(),
                    &raw
                ));
            } else {
                using E = std::remove_const_t<typename Data::element_type>;
                detail::check(svsb200_index_create_multi(
                    data.data(),
                    detail::DTypeCode<E>::value,
                    data.size(),
                    data.dimensions(),
                    0,
                    rows.data(),
                    rows.dimensions(),
                    entry_points[0],
                    detail::MetricCode<Dist>::value,
                    SVSB200_PLAIN,
                    nullptr,
                    devices.data(),
                    devices.size(),
                    &raw
                ));
            }
            handle_.reset(raw, detail::HandleDeleter{});
            if (entry_points.size() > 1) {   // index.h:304-312: every entry point seeds the walk
                std::vector<uint32_t> eps(entry_points.begin(), entry_points.end());
                detail::check(svsb200_set_entry_points(raw, eps.data(), eps.size()));
            }
        });
    }

    // Single-query search, scratch-space search etc. stay the reference's.
    using base_type::search;

    /// Batch search on the GPU: same signature and semantics as index.h:564-611.
    template <typename I, svs::data::ImmutableMemoryDataset Queries>
    void search(
        svs::QueryResultView<I> result,
        const Queries& queries,
        const search_parameters_type& sp,
        const svs::lib::DefaultPredicate& cancel = svs::lib::Returns(svs::lib::Const<false>())
    ) {
        using Q = std::remove_const_t<typename Queries::element_type>;
        static_assert(sizeof(I) == 4 || sizeof(I) == 8, "result ids must be 32 or 64 bit");
        if (queries.dimensions() != this->dimensions()) {
            throw ANNEXCEPTION(
                "Query dimensions {} do not match index dimensions {}",
                queries.dimensions(),
                this->dimensions()
            );
        }
        // The predicate is polled by this thread while the batch runs; once it fires, a device flag stops
        // every search warp at its next query / hop boundary (the reference polls at greedy_search.h:155
        // and extensions.h:579).
        const size_t nq = queries.size();
        if (nq == 0) {
            return;
        }
        auto trampoline = [](void* arg) -> int {
            return (*static_cast<const svs::lib::DefaultPredicate*>(arg))() ? 1 : 0;
        };
        detail::check(svsb200_search_cancellable(
            handle_.get(),
            queries.get_datum(0).data(),
            detail::DTypeCode<Q>::value,
            nq,
            result.n_neighbors(),
            sp.buffer_config_.get_search_window_size(),
            sp.buffer_config_.get_total_capacity(),
            sp.search_buffer_visited_set_ ? 1 : 0,
            &result.index(0, 0),
            static_cast<int>(sizeof(I)),
            &result.distance(0, 0),
            nullptr,
            +trampoline,
            const_cast<void*>(static_cast<const void*>(&cancel))
        ));
    }

    /// Devices holding a replica ("threadpool -> CUDA streams": every calling thread gets its own stream).
    size_t num_devices() const { return svsb200_index_num_devices(handle_.get()); }

    std::string name() const { return "GpuVamanaIndex (libsvsb200, sm_90a)"; }
    svsb200_index* native_handle() const { return handle_.get(); }

  private:
    std::shared_ptr<svsb200_index> handle_{};
};

template <typename Graph, typename Data, typename Dist>
GpuVamanaIndex(svs::index::vamana::VamanaIndex<Graph, Data, Dist>&&, int)
    -> GpuVamanaIndex<Graph, Data, Dist>;
template <typename Graph, typename Data, typename Dist>
GpuVamanaIndex(svs::index::vamana::VamanaIndex<Graph, Data, Dist>&&)
    -> GpuVamanaIndex<Graph, Data, Dist>;
template <typename Graph, typename Data, typename Dist>
GpuVamanaIndex(svs::index::vamana::VamanaIndex<Graph, Data, Dist>&&, const std::vector<int>&)
    -> GpuVamanaIndex<Graph, Data, Dist>;

/// Type-erase a GpuVamanaIndex into the reference's orchestrator object.
template <svs::lib::TypeList QueryTypes, typename Graph, typename Data, typename Dist>
svs::Vamana make_gpu_vamana(GpuVamanaIndex<Graph, Data, Dist>&& index) {
    using Impl = GpuVamanaIndex<Graph, Data, Dist>;
    return svs::Vamana{std::make_unique<svs::VamanaImpl<QueryTypes, Impl>>(std::move(index))};
}

} // namespace svsb200
