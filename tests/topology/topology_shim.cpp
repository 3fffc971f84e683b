// Test shim for tests/test_topology.py: plan_topology and build_stage_program of bepuphysics2_b200/csrc/bepu_topology.h behind a ctypes-friendly
// C interface. Built with g++ together with bepu_topology.cpp; the product never loads it.
#include <cstring>

#include "bepu_topology.h"

using namespace bepucuda;

struct PlanHandle {
    TopologyPlan plan;
    int rc;
    std::string error;
};

extern "C" {

// meta: per source (batch_index, type_batch_index, type_id, count); refs[i]: its host references (AOSOA-W) or null
void* topology_plan(int n, const int32_t* meta, const int32_t* const* refs, int W, int fallback_threshold, int batch_count, int body_count, int peer_mode) {
    std::vector<SourceView> sources;
    for (int i = 0; i < n; ++i) sources.push_back({meta[4 * i], meta[4 * i + 1], meta[4 * i + 2], meta[4 * i + 3], refs[i]});
    PlanHandle* h = new PlanHandle;
    h->rc = plan_topology(sources, W, fallback_threshold, batch_count, body_count, peer_mode != 0, &h->plan, &h->error);
    return h;
}
int topology_plan_error(void* h, char* message, int capacity) {
    const PlanHandle* p = (const PlanHandle*)h;
    std::strncpy(message, p->error.c_str(), (size_t)capacity - 1);
    message[capacity - 1] = 0;
    return p->rc;
}
// type batches, map slots, work items, device batches, sources, all_work_count, sync_batch_count, fallback_levels, constraint_count, inc_begin, inc_count
void topology_plan_sizes(void* h, int64_t* out) {
    const TopologyPlan& p = ((PlanHandle*)h)->plan;
    const int64_t v[] = {(int64_t)p.tbs.size(), (int64_t)p.maps.size(), (int64_t)p.work.size(), (int64_t)p.batches.size(), (int64_t)p.source_live.size(), p.all_work_count,
                         p.sync_batch_count, p.fallback_levels, p.constraint_count, p.inc_begin, p.inc_count};
    std::memcpy(out, v, sizeof(v));
}
// per type batch: type_id, bundle_count, device_batch, source, map_offset
void topology_plan_tbs(void* h, int64_t* out) {
    for (const PlannedTypeBatch& t : ((PlanHandle*)h)->plan.tbs) {
        const int64_t v[] = {t.type_id, t.bundle_count, t.device_batch, t.source, t.map_offset};
        std::memcpy(out, v, sizeof(v));
        out += 5;
    }
}
void topology_plan_maps(void* h, int32_t* out) {
    const TopologyPlan& p = ((PlanHandle*)h)->plan;
    if (!p.maps.empty()) std::memcpy(out, p.maps.data(), p.maps.size() * 4);
}
// per work item: type batch, bundle, live lanes
void topology_plan_work(void* h, int32_t* out) {
    const TopologyPlan& p = ((PlanHandle*)h)->plan;
    for (size_t i = 0; i < p.work.size(); ++i) {
        out[3 * i] = p.work[i].type_batch;
        out[3 * i + 1] = p.work[i].bundle;
        out[3 * i + 2] = p.bundle_live[i];
    }
}
// per device batch: begin, count, contacts_only
void topology_plan_batches(void* h, int32_t* out) {
    for (const TopologyPlan::Batch& b : ((PlanHandle*)h)->plan.batches) {
        out[0] = b.begin; out[1] = b.count; out[2] = b.contacts_only;
        out += 3;
    }
}
void topology_plan_source_live(void* h, int32_t* out) {
    const TopologyPlan& p = ((PlanHandle*)h)->plan;
    if (!p.source_live.empty()) std::memcpy(out, p.source_live.data(), p.source_live.size() * 4);
}
void topology_plan_free(void* h) { delete (PlanHandle*)h; }

void* topology_program(void* plan, int substeps, const int32_t* iterations, int kinematic_count, int integrate_velocity_for_kinematics, int peer_mode, int body_count) {
    return new StageProgram(build_stage_program(((PlanHandle*)plan)->plan, std::vector<int32_t>(iterations, iterations + substeps), kinematic_count,
                                                integrate_velocity_for_kinematics != 0, peer_mode != 0, body_count));
}
// ops, exchange_count, stage_count, constraint_iterations, algorithmic_bytes
void topology_program_sizes(void* h, int64_t* out) {
    const StageProgram& p = *(StageProgram*)h;
    const int64_t v[] = {(int64_t)p.ops.size(), p.exchange_count, p.stage_count, p.constraint_iterations, p.algorithmic_bytes};
    std::memcpy(out, v, sizeof(v));
}
// per op: stage, work_begin, work_count, exchange, exchange_index, launch_flags, algorithmic_bytes
void topology_program_ops(void* h, int64_t* out) {
    for (const StageOp& op : ((StageProgram*)h)->ops) {
        const int64_t v[] = {op.stage, op.work_begin, op.work_count, op.exchange, op.exchange_index, op.launch_flags, op.algorithmic_bytes};
        std::memcpy(out, v, sizeof(v));
        out += 7;
    }
}
void topology_program_free(void* h) { delete (StageProgram*)h; }

}  // extern "C"
