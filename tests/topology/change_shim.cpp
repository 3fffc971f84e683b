// Test shim of tests/test_constraint_changes.py: replay_changes and compose_lane_ops of bepuphysics2_b200/csrc/bepu_topology.h behind a
// ctypes-friendly C interface, holding a ChangeState between calls as a context does. Built with g++ together with bepu_topology.cpp; the product
// never loads it.
#include <cstring>

#include "bepu_topology.h"

using namespace bepucuda;

extern "C" {

// meta: int32[n][4] (batch, type batch, type id, ConstraintCount); refs[i]: ref_words[i] body references of source i (fallback sources; else 0).
void* change_create(int n, const int32_t* meta, const int32_t* const* refs, const int32_t* ref_words, int batch_count) {
    ChangeState* st = new ChangeState();
    st->batch_count = batch_count;
    for (int i = 0; i < n; ++i)
        st->sources.push_back({meta[4 * i], meta[4 * i + 1], meta[4 * i + 2], meta[4 * i + 3], std::vector<int32_t>(refs[i], refs[i] + ref_words[i])});
    return st;
}
void change_destroy(void* st) { delete (ChangeState*)st; }

// One call on a copy of the state, committed only when it succeeds (as bepucuda_add_constraints / bepucuda_remove_constraints do). On success:
// copies_out[*copy_count][4] the lane copies in order (compose != 0: compose_lane_ops of them), remap_out[i] the index of source i after the call
// (-1: removed; new sources included), and the state's sources compacted. Returns the replay's code, or -100 when `capacity` copies do not fit.
int change_apply(void* stp, int remove, int W, int threshold, int body_count, int count, const int32_t* locations, const int32_t* records, int compose, int capacity,
                 int32_t* copies_out, int* copy_count, int32_t* remap_out) {
    ChangeState& st = *(ChangeState*)stp;
    ChangeState next = st;
    std::vector<LaneCopy> ops;
    std::string error;
    const int rc = replay_changes(&next, remove != 0, W, threshold, body_count, count, (const bepucuda_constraint_location*)locations, records, &ops, &error);
    if (rc != 0) return rc;
    if (compose) ops = compose_lane_ops(ops);
    if ((int)ops.size() > capacity) return -100;
    std::memcpy(copies_out, ops.data(), ops.size() * sizeof(LaneCopy));
    *copy_count = (int)ops.size();
    ChangeState kept;
    kept.batch_count = next.batch_count;
    for (size_t i = 0; i < next.sources.size(); ++i) {
        remap_out[i] = next.sources[i].type_batch_index >= 0 ? (int32_t)kept.sources.size() : -1;
        if (next.sources[i].type_batch_index >= 0) kept.sources.push_back(next.sources[i]);
    }
    st = kept;
    return 0;
}

// meta_out: int32[n][4] of the current sources; returns n. *batch_count: the batch count.
int change_sources(void* stp, int32_t* meta_out, int* batch_count) {
    const ChangeState& st = *(ChangeState*)stp;
    for (size_t i = 0; i < st.sources.size(); ++i) {
        const ChangeSource& s = st.sources[i];
        const int32_t m[4] = {s.batch_index, s.type_batch_index, s.type_id, s.count};
        std::memcpy(meta_out + 4 * i, m, sizeof(m));
    }
    *batch_count = st.batch_count;
    return (int)st.sources.size();
}

}  // extern "C"
