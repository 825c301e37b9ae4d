// slots.h -- the host side of the slots of the three dynamic indexes (dynamic Vamana, dynamic flat, dynamic IVF): every
// slot's status and external id, and the external -> slot translator (the reference's IDTranslator,
// core/translation.h).  Each index keeps one SlotTable, mirrored on the device in Replica::d_status / d_ext_ids, and
// takes its slot rules from it; what differs between the indexes is passed in by the caller (where an add starts to
// look for Empty slots, what a delete leaves behind).  Plain C++, so that the rules can be tested without CUDA.
//
// The checks run before anything changes and name their entry point ("<who>: ..."); the commits run once every device
// step of a mutation has succeeded.
#pragma once

#include <algorithm>
#include <cstddef>
#include <cstdint>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <vector>

namespace svsb200 {

int fail(const std::string& msg);   // records the calling thread's svsb200_last_error(); returns 1

// SlotMetadata of the reference's MutableVamanaIndex (index/vamana/dynamic_index.h:60-79).  The dynamic flat and IVF
// indexes use Valid and Empty only.
enum SlotStatus : uint8_t { SLOT_EMPTY = 0, SLOT_VALID = 1, SLOT_DELETED = 2 };

constexpr uint64_t kNoExternalId = ~uint64_t(0);   // reserved: marks the padding of short result rows and Empty slots

struct SlotTable {
    std::vector<uint8_t> status;                         // per slot
    std::vector<uint64_t> ext_ids;                       // per slot
    std::unordered_map<uint64_t, uint32_t> translator;   // the Valid slots' external ids -> slot
    size_t first_empty = 0;                              // first_empty_: where add_points looks for Empty slots

    size_t size() const { return translator.size(); }
    size_t num_slots() const { return status.size(); }

    // IDTranslator::insert (core/translation.h:105-127) at creation: slots 0 .. n-1 Valid with external ids `ids`.
    int assign(const char* who, const uint64_t* ids, size_t n) {
        const std::string w(who);
        std::unordered_map<uint64_t, uint32_t> t;
        t.reserve(n);
        for (size_t i = 0; i < n; ++i)
            if (ids[i] == kNoExternalId)
                return fail(w + ": external id 2^64 - 1 is reserved");
            else if (!t.emplace(ids[i], uint32_t(i)).second)
                return fail(w + ": External IDs contain repeat elements!");
        status.assign(n, SLOT_VALID);
        ext_ids.assign(ids, ids + n);
        translator = std::move(t);
        first_empty = n;
        return 0;
    }

    // translator_.insert's checks, run by add before anything changes: no id reserved, repeated or present.
    int check_new(const char* who, const uint64_t* ids, size_t count) const {
        const std::string w(who);
        std::unordered_set<uint64_t> seen;
        seen.reserve(count);
        for (size_t i = 0; i < count; ++i) {
            if (ids[i] == kNoExternalId) return fail(w + ": external id 2^64 - 1 is reserved");
            if (!seen.insert(ids[i]).second) return fail(w + ": External IDs contain repeat elements!");
            if (translator.count(ids[i]))
                return fail(w + ": External ID " + std::to_string(ids[i]) + " already exists!");
        }
        return 0;
    }

    // translator_.check_external_exist (core/translation.h:395-407), run by delete before anything changes: every id
    // present, once.  *slots = their slots.
    int find(const char* who, const uint64_t* ids, size_t count, std::vector<uint32_t>* slots) const {
        slots->clear();
        slots->reserve(count);
        std::unordered_set<uint64_t> seen;
        seen.reserve(count);
        for (size_t i = 0; i < count; ++i) {
            auto it = translator.find(ids[i]);
            if (it == translator.end() || !seen.insert(ids[i]).second)
                return fail(std::string(who) + ": External ID " + std::to_string(ids[i]) + " does not exist!");
            slots->push_back(it->second);
        }
        return 0;
    }

    // The slots of `count` added rows: Empty ones from slot `from` on, then appended ones.  Returns the number of slots
    // afterwards (the caller checks it against its limit before using *slots).
    size_t choose(size_t count, size_t from, std::vector<uint32_t>* slots) const {
        slots->clear();
        slots->reserve(count);
        for (size_t s = from; s < status.size() && slots->size() < count; ++s)
            if (status[s] == SLOT_EMPTY) slots->push_back(uint32_t(s));
        const size_t n = status.size() + (count - slots->size());
        for (size_t s = status.size(); s < n; ++s) slots->push_back(uint32_t(s));
        return n;
    }

    // The rows of external ids `ids` are now Valid in `slots` (from choose); appended slots past the ones the table
    // holds come in Empty, and the ones not used stay so.  slots_out (may be NULL) receives the slots.
    void commit_add(const std::vector<uint32_t>& slots, const uint64_t* ids, uint64_t* slots_out) {
        if (slots.empty()) return;
        const size_t n = std::max<size_t>(status.size(), size_t(slots.back()) + 1);
        status.resize(n, SLOT_EMPTY);
        ext_ids.resize(n, kNoExternalId);
        for (size_t i = 0; i < slots.size(); ++i) {
            status[slots[i]] = SLOT_VALID;
            ext_ids[slots[i]] = ids[i];
            translator.emplace(ids[i], slots[i]);
            if (slots_out) slots_out[i] = slots[i];
        }
        first_empty = std::max<size_t>(first_empty, size_t(slots.back()) + 1);
    }

    // The entries of external ids `ids` in `slots` (from find) are deleted.  to = SLOT_EMPTY (delete_entry of the
    // dynamic flat and IVF indexes): the external id is cleared and first_empty moves back to the slot.  to =
    // SLOT_DELETED (the Vamana index's soft delete): the slot keeps its external id until consolidation.
    void commit_delete(const std::vector<uint32_t>& slots, const uint64_t* ids, uint8_t to) {
        for (size_t i = 0; i < slots.size(); ++i) {
            status[slots[i]] = to;
            translator.erase(ids[i]);
            if (to == SLOT_EMPTY) {
                ext_ids[slots[i]] = kNoExternalId;
                first_empty = std::min<size_t>(first_empty, slots[i]);
            }
        }
    }

    // nonmissing_indices: compaction's new -> old slot order (the Valid slots, ascending), and *ext their external ids.
    std::vector<uint32_t> valid_slots(std::vector<uint64_t>* ext) const {
        std::vector<uint32_t> new_to_old;
        new_to_old.reserve(translator.size());
        ext->clear();
        ext->reserve(translator.size());
        for (size_t s = 0; s < status.size(); ++s)
            if (status[s] == SLOT_VALID) {
                new_to_old.push_back(uint32_t(s));
                ext->push_back(ext_ids[s]);
            }
        return new_to_old;
    }

    // After compaction: slots 0 .. m-1 Valid with external ids `ext` (from valid_slots).
    void commit_compact(std::vector<uint64_t> ext) {
        const size_t m = ext.size();
        status.assign(m, SLOT_VALID);
        ext_ids = std::move(ext);
        for (size_t i = 0; i < m; ++i) translator[ext_ids[i]] = uint32_t(i);
        first_empty = m;
    }

    // all_ids: the external ids of the Valid slots in slot order (out NULL: their number only).
    int ids(const char* who, uint64_t* out, size_t* count) const {
        if (!count) return fail(std::string(who) + ": NULL count");
        if (out) {
            if (*count < translator.size()) return fail(std::string(who) + ": output too small");
            size_t o = 0;
            for (size_t s = 0; s < status.size(); ++s)
                if (status[s] == SLOT_VALID) out[o++] = ext_ids[s];
        }
        *count = translator.size();
        return 0;
    }

    int has_id(const char* who, uint64_t id, int* out) const {
        if (!out) return fail(std::string(who) + ": NULL output");
        *out = translator.count(id) ? 1 : 0;
        return 0;
    }

    // The status and external id of every slot (either output may be NULL).
    void export_to(uint8_t* status_out, uint64_t* ext_ids_out) const {
        if (status_out) std::copy(status.begin(), status.end(), status_out);
        if (ext_ids_out) std::copy(ext_ids.begin(), ext_ids.end(), ext_ids_out);
    }
};

}  // namespace svsb200
