// Test shim of tests/test_constraint_write.py: resolve_location and PrestepWriteQueue of bepuphysics2_b200/csrc/bepu_topology.h behind a
// ctypes-friendly C interface, next to the plans of tests/topology/topology_shim.cpp. Built with g++ together with bepu_topology.cpp; the product
// never loads it.
#include <cstring>

#include "bepu_topology.h"

using namespace bepucuda;

extern "C" {

// Plans the sources as topology_plan does (single context), then resolves every location (int32[count][4], bepucuda_constraint_location):
// out[i] = {return code, device type batch, slot, inverse entry}. Returns the plan's code.
int locations_resolve(int n, const int32_t* meta, const int32_t* const* refs, int W, int fallback_threshold, int batch_count, int body_count, int count,
                      const int32_t* locations, int64_t* out) {
    std::vector<SourceView> sources;
    for (int i = 0; i < n; ++i) sources.push_back({meta[4 * i], meta[4 * i + 1], meta[4 * i + 2], meta[4 * i + 3], refs[i]});
    TopologyPlan plan;
    std::string error;
    const int rc = plan_topology(sources, W, fallback_threshold, batch_count, body_count, false, &plan, &error);
    if (rc != 0) return rc;
    for (int i = 0; i < count; ++i, out += 4) {
        const bepucuda_constraint_location l{locations[4 * i], locations[4 * i + 1], locations[4 * i + 2], locations[4 * i + 3]};
        ResolvedLocation r{-7, {-7, -7}, -7};  // what an error leaves untouched
        out[0] = resolve_location(plan, l, &r);
        out[1] = r.at.type_batch;
        out[2] = r.at.slot;
        out[3] = r.inverse_entry;
    }
    return 0;
}

// A queue over `type_batches` device type batches of `bundles` bundles each. Puts `count` writes (slots int32[count][2], rows
// float[count][rows_per_write]) into it in order, `rounds` times with a clear() in between. Returns the queue length; out_slots / out_rows
// (float[count][rows_per_write]) receive its entries in queue order.
int write_queue(int type_batches, int bundles, int rounds, int count, const int32_t* slots, const float* rows, int rows_per_write, int32_t* out_slots, float* out_rows) {
    TopologyPlan plan;
    plan.tbs.resize((size_t)type_batches);
    for (PlannedTypeBatch& tb : plan.tbs) tb.bundle_count = bundles;
    PrestepWriteQueue q;
    q.plan(plan);
    for (int round = 0; round < rounds; ++round) {
        q.clear();
        for (int i = 0; i < count; ++i) q.put(DeviceSlot{slots[2 * i], slots[2 * i + 1]}, rows + (size_t)i * rows_per_write, rows_per_write);
    }
    for (size_t i = 0; i < q.writes.size(); ++i) {
        out_slots[2 * i] = q.writes[i].at.type_batch;
        out_slots[2 * i + 1] = q.writes[i].at.slot;
        std::memcpy(out_rows + i * rows_per_write, q.rows.data() + q.writes[i].row0, (size_t)rows_per_write * sizeof(float));
    }
    return (int)q.writes.size();
}

}  // extern "C"
