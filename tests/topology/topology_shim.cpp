// Test shim of the planner tests (loaded by tests/planner.py): get_type_info, plan_topology (plain and per rank), its inverse slot map,
// build_stage_program, exchange_targets, resolve_stage_launch, same_launches and integrated_warm_start_launch of bepuphysics2_b200/csrc/
// bepu_topology.h behind a ctypes-friendly C interface. Built with g++ together with bepu_topology.cpp; the product never loads it.
#include <cstring>

#include "bepu_topology.h"
#include "bepu_type_table.h"

using namespace bepucuda;

struct PlanHandle {
    TopologyPlan plan;
    int rc;
    std::string error;
};

extern "C" {

// meta: per source (batch_index, type_batch_index, type_id, count); refs[i]: its host references (AOSOA-W) or null. In peer mode the plan is
// `rank`'s, with `fallback_rank` the rank that owns the fallback batch (-1 = none).
void* topology_plan(int n, const int32_t* meta, const int32_t* const* refs, int W, int fallback_threshold, int batch_count, int body_count, int peer_mode,
                    int rank, int fallback_rank) {
    std::vector<SourceView> sources;
    for (int i = 0; i < n; ++i) sources.push_back({meta[4 * i], meta[4 * i + 1], meta[4 * i + 2], meta[4 * i + 3], refs[i]});
    PlanHandle* h = new PlanHandle;
    h->rc = plan_topology(sources, W, fallback_threshold, batch_count, body_count, peer_mode != 0, &h->plan, &h->error, rank, fallback_rank);
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
int64_t topology_plan_inverse_size(void* h) { return (int64_t)((PlanHandle*)h)->plan.inverse.size(); }
// per source: its device type batch (synchronized) and its first inverse entry (fallback); per entry: device type batch, slot
void topology_plan_inverse(void* h, int32_t* source_type_batch, int64_t* source_inverse_offset, int32_t* inverse) {
    const TopologyPlan& p = ((PlanHandle*)h)->plan;
    std::memcpy(source_type_batch, p.source_type_batch.data(), p.source_type_batch.size() * 4);
    std::memcpy(source_inverse_offset, p.source_inverse_offset.data(), p.source_inverse_offset.size() * 8);
    for (size_t i = 0; i < p.inverse.size(); ++i) {
        inverse[2 * i] = p.inverse[i].type_batch;
        inverse[2 * i + 1] = p.inverse[i].slot;
    }
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
// per op: stage, work_begin, work_count, exchange, exchange_index, launch_flags (kOp* facts), algorithmic_bytes
void topology_program_ops(void* h, int64_t* out) {
    for (const StageOp& op : ((StageProgram*)h)->ops) {
        const int64_t v[] = {op.stage, op.work_begin, op.work_count, op.exchange, op.exchange_index, op.launch_flags, op.algorithmic_bytes};
        std::memcpy(out, v, sizeof(v));
        out += 7;
    }
}
void topology_program_free(void* h) { delete (StageProgram*)h; }

// exchange_targets of the peer-mode program of `plan` with per-device-batch boundary counts; out: kShardMaxExchanges cumulative targets
int topology_exchange_targets(void* plan, int substeps, const int32_t* iterations, int kinematic_count, int integrate_velocity_for_kinematics, int body_count,
                              const int32_t* boundary_count, unsigned long long* out) {
    const TopologyPlan& p = ((PlanHandle*)plan)->plan;
    const StageProgram prog = build_stage_program(p, std::vector<int32_t>(iterations, iterations + substeps), kinematic_count, integrate_velocity_for_kinematics != 0, true,
                                                  body_count);
    std::vector<unsigned long long> targets;
    std::string error;
    const int rc = exchange_targets(prog, std::vector<int32_t>(boundary_count, boundary_count + p.batches.size()), &targets, &error);
    if (rc == 0) std::memcpy(out, targets.data(), targets.size() * sizeof(unsigned long long));
    return rc;
}
int topology_max_exchanges() { return kShardMaxExchanges; }

// ops: n rows of topology_program_ops; out[i] = kernel, flags of op i
void topology_resolve(const int64_t* ops, int n, int integrator_extensions, int angular_mode, int profile, int32_t* out) {
    const LaunchContext lc{integrator_extensions != 0, angular_mode, profile != 0};
    for (int i = 0; i < n; ++i, ops += 7) {
        const StageOp op{(int32_t)ops[0], (int32_t)ops[1], (int32_t)ops[2], (int32_t)ops[3], (uint32_t)ops[4], (int32_t)ops[5], ops[6]};
        const StageLaunch l = resolve_stage_launch(op, lc);
        out[2 * i] = l.kernel;
        out[2 * i + 1] = l.flags;
    }
}
int topology_same_launches(int extensions_a, int angular_mode_a, int profile_a, int extensions_b, int angular_mode_b, int profile_b) {
    return same_launches(LaunchContext{extensions_a != 0, angular_mode_a, profile_a != 0}, LaunchContext{extensions_b != 0, angular_mode_b, profile_b != 0});
}
int topology_deep_batch_bundles() { return kDeepBatchBundles; }
// get_type_info: the name (null for an id without a type); out: the other TypeInfo fields in order, then the filter counts of the table row
const char* topology_type_info(int type_id, int64_t* out) {
    const TypeInfo* t = get_type_info(type_id);
    if (!t) return nullptr;
    const TypeRow& r = *type_row(type_id);
    const int64_t v[] = {t->bodies, t->prestep_rows, t->impulse_rows, t->contacts, t->solve_bytes, t->warm_start_bytes, t->incremental_bytes,
                         r.solve_read, r.solve_written, r.warm_start_read, r.warm_start_written};
    std::memcpy(out, v, sizeof(v));
    return t->name;
}
// which contact-only WarmStart instantiation launch_stage (csrc/bepu_solver_kernels.cu) runs for a resolved launch: 1 = the integrated one
int topology_integrated_warm_start_launch(int stage, int kernel, int flags) { return integrated_warm_start_launch(stage, StageLaunch{kernel, flags}) ? 1 : 0; }

}  // extern "C"
