// A C interface to svsb200::SlotTable (scalablevectorsearch_b200/csrc/slots.h) for tests/test_slot_table.py, which
// compiles it with the host C++ compiler: the slot rules of the dynamic indexes without CUDA.
#include "slots.h"

#include <string>

namespace svsb200 {
static std::string last_error;
int fail(const std::string& msg) {
    last_error = msg;
    return 1;
}
}  // namespace svsb200

using svsb200::SlotTable;

extern "C" {
const char* st_last_error() { return svsb200::last_error.c_str(); }
void* st_new() { return new SlotTable(); }
void st_free(void* t) { delete static_cast<SlotTable*>(t); }
int st_assign(void* t, const uint64_t* ids, size_t n) { return static_cast<SlotTable*>(t)->assign("t", ids, n); }
// An add as an index runs it: the checks, then the slots from `from`, then the commit.  from_num_slots: the dynamic
// IVF index's rule (append unless reuse_empty); otherwise the dynamic flat and Vamana indexes' (from first_empty).
int st_add(void* p, const uint64_t* ids, size_t count, int reuse_empty, int from_num_slots, uint64_t* slots_out) {
    SlotTable& t = *static_cast<SlotTable*>(p);
    if (int rc = t.check_new("t", ids, count)) return rc;
    std::vector<uint32_t> slots;
    t.choose(count, reuse_empty ? 0 : from_num_slots ? t.num_slots() : t.first_empty, &slots);
    t.commit_add(slots, ids, slots_out);
    return 0;
}
int st_delete(void* p, const uint64_t* ids, size_t count, uint8_t to) {
    SlotTable& t = *static_cast<SlotTable*>(p);
    std::vector<uint32_t> slots;
    if (int rc = t.find("t", ids, count, &slots)) return rc;
    t.commit_delete(slots, ids, to);
    return 0;
}
void st_compact(void* p) {
    SlotTable& t = *static_cast<SlotTable*>(p);
    std::vector<uint64_t> ext;
    t.valid_slots(&ext);
    t.commit_compact(std::move(ext));
}
size_t st_num_slots(void* t) { return static_cast<SlotTable*>(t)->num_slots(); }
size_t st_size(void* t) { return static_cast<SlotTable*>(t)->size(); }
size_t st_first_empty(void* t) { return static_cast<SlotTable*>(t)->first_empty; }
void st_export(void* t, uint8_t* status, uint64_t* ext) { static_cast<SlotTable*>(t)->export_to(status, ext); }
int st_ids(void* t, uint64_t* out, size_t* count) { return static_cast<SlotTable*>(t)->ids("t", out, count); }
int st_has_id(void* t, uint64_t id, int* out) { return static_cast<SlotTable*>(t)->has_id("t", id, out); }
}
