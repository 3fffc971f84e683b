// Constraint topology: type registry, device batches and work list (plan_topology), stage program (build_stage_program). Plain C++: no CUDA
// runtime call, so that the CPU suite can check what the device is told to run.
#include "bepu_topology.h"

#include <algorithm>
#include <cstring>
#include <numeric>

#include "../../include/bepucuda.h"

namespace bepucuda {

// ---- type registry -------------------------------------------------------------------------------------------------------
// SURVEY.md §8d algorithmic bytes:
//   solve       = 4 * (P + 2D + n + sum(R_i + W_i))        R/W from the type's Solve access filters
//   warm start  = 4 * (P + D + n + sum(R'_i + W'_i))       (non-integrating lane, WarmStart filters)
//   incremental = 4 * (P_read + contacts_written + n + 6n)
// Filters (IBodyAccessFilter.cs:L38-126): pos 3, orientation 4, lin 3, ang 3, inertia tensor 6, mass 1.
static TypeInfo make_contact(int bodies, int prestep, int impulses, int contacts, const char* name) {
    TypeInfo t{};
    t.bodies = bodies; t.prestep_rows = prestep; t.impulse_rows = impulses; t.contacts = contacts; t.name = name;
    const int body_rw = 13 + 6;  // AccessNoPose: velocity 6 + inertia 7 read, velocity 6 written
    t.solve_bytes = 4 * (prestep + 2 * impulses + bodies + bodies * body_rw);
    t.warm_start_bytes = 4 * (prestep + impulses + bodies + bodies * body_rw);
    t.incremental_bytes = 4 * (prestep + contacts + bodies + 6 * bodies);
    return t;
}
static TypeInfo make_joint(int bodies, int prestep, int impulses, int solve_r, int solve_w, int ws_r, int ws_w, const char* name) {
    TypeInfo t{};
    t.bodies = bodies; t.prestep_rows = prestep; t.impulse_rows = impulses; t.contacts = 0; t.name = name;
    t.solve_bytes = 4 * (prestep + 2 * impulses + bodies + solve_r + solve_w);
    t.warm_start_bytes = 4 * (prestep + impulses + bodies + ws_r + ws_w);
    t.incremental_bytes = 0;
    return t;
}
struct Registry {
    TypeInfo types[64];
    bool present[64];
    Registry() {
        std::memset(present, 0, sizeof(present));
        auto add = [&](int id, TypeInfo t) { types[id] = t; present[id] = true; };
        add(0, make_contact(1, 11, 4, 1, "Contact1OneBody")); add(1, make_contact(1, 15, 5, 2, "Contact2OneBody"));
        add(2, make_contact(1, 19, 6, 3, "Contact3OneBody")); add(3, make_contact(1, 23, 7, 4, "Contact4OneBody"));
        add(4, make_contact(2, 14, 4, 1, "Contact1")); add(5, make_contact(2, 18, 5, 2, "Contact2"));
        add(6, make_contact(2, 22, 6, 3, "Contact3")); add(7, make_contact(2, 26, 7, 4, "Contact4"));
        add(8, make_contact(1, 18, 6, 2, "Contact2NonconvexOneBody")); add(9, make_contact(1, 25, 9, 3, "Contact3NonconvexOneBody"));
        add(10, make_contact(1, 32, 12, 4, "Contact4NonconvexOneBody"));
        add(15, make_contact(2, 21, 6, 2, "Contact2Nonconvex")); add(16, make_contact(2, 28, 9, 3, "Contact3Nonconvex"));
        add(17, make_contact(2, 35, 12, 4, "Contact4Nonconvex"));
#define BEPU_REGISTER_JOINTS
#include "bepu_joint_registry.inc"
#undef BEPU_REGISTER_JOINTS
    }
};
static const Registry& registry() {
    static Registry r;
    return r;
}
const TypeInfo* get_type_info(int type_id) {
    if (type_id < 0 || type_id >= 64 || !registry().present[type_id]) return nullptr;
    return &registry().types[type_id];
}

// ---- device batches and work list ----------------------------------------------------------------------------------------
static bool dynamic_ref(int32_t enc) { return enc >= 0 && !((uint32_t)enc & kRefKinematicBit); }

int plan_topology(const std::vector<SourceView>& sources, int W, int fallback_threshold, int batch_count, int body_count, bool peer_mode, TopologyPlan* plan,
                  std::string* error) {
    TopologyPlan& p = *plan;
    p = TopologyPlan{};
    // sources in (batch, type batch) order
    std::vector<int> order(sources.size());
    std::iota(order.begin(), order.end(), 0);
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) {
        const SourceView &x = sources[(size_t)a], &y = sources[(size_t)b];
        return x.batch_index != y.batch_index ? x.batch_index < y.batch_index : x.type_batch_index < y.type_batch_index;
    });
    p.source_live.assign(sources.size(), 0);
    p.source_bundle_base.assign(sources.size(), 0);
    for (int si : order) {
        p.source_bundle_base[(size_t)si] = p.source_bundles;
        p.source_bundles += (sources[(size_t)si].count + W - 1) / W;
    }
    std::vector<std::vector<int>> batch_tbs;  // device batch -> device type batches
    auto add_tb = [&](int source, int device_batch, int constraints, int64_t map_offset) {
        batch_tbs[(size_t)device_batch].push_back((int)p.tbs.size());
        p.tbs.push_back({sources[(size_t)source].type_id, (constraints + 31) / 32, device_batch, source, map_offset, 0, 0, 0});
    };

    // synchronized batches: device batch index == host batch index (empty batches stay as empty slots), so ranks of a sharded graph agree on
    // batch numbers
    for (int si : order) {
        const SourceView& s = sources[(size_t)si];
        if (s.batch_index >= fallback_threshold) continue;
        while ((int)batch_tbs.size() <= s.batch_index) batch_tbs.emplace_back();
        add_tb(si, s.batch_index, s.count, -1);
        p.source_live[(size_t)si] = s.count;
        p.constraint_count += s.count;
    }
    if (peer_mode) {
        // every rank runs the exchange point of every batch, also of batches it has no constraint in
        while ((int)batch_tbs.size() < std::min(batch_count, fallback_threshold)) batch_tbs.emplace_back();
        for (const SourceView& s : sources)
            if (s.batch_index >= fallback_threshold) {
                *error = "end_constraints: the sequential fallback batch is not supported across ranks";
                return BEPUCUDA_ERR_BAD_STATE;
            }
    }
    p.sync_batch_count = (int)batch_tbs.size();

    // Fallback levelisation. The reference executes fallback bundles one after another on a single thread (Solver_Solve.cs:L546-583); within a
    // bundle no dynamic body repeats (TypeProcessor.cs:L338-359). A constraint's level is 1 + the highest level of any earlier-bundle constraint
    // sharing a dynamic body with it: executing levels in order with a barrier in between preserves every read-after-write of the sequential
    // loop, so results are identical.
    std::vector<int32_t> last_level;  // per body: highest level assigned so far (0 = none)
    struct Slot { int level; int rank; int constraint; };  // rank: position of the source in `order`
    std::vector<Slot> slots;
    std::vector<int> lane_level((size_t)W);
    for (size_t rank = 0; rank < order.size(); ++rank) {
        const SourceView& s = sources[(size_t)order[rank]];
        if (s.batch_index < fallback_threshold) continue;
        if (last_level.empty()) last_level.assign((size_t)body_count, 0);
        const int nb = get_type_info(s.type_id)->bodies;
        const int bundles = (s.count + W - 1) / W;
        auto ref = [&](int k, int b, int l) { return s.refs[((size_t)k * nb + b) * W + l]; };
        for (int k = 0; k < bundles; ++k) {
            // all lanes of a bundle read the state left by earlier bundles
            for (int l = 0; l < W; ++l) {
                lane_level[(size_t)l] = 0;
                if (k * W + l >= s.count || ref(k, 0, l) < 0) continue;  // padding, hole
                int lvl = 0;
                for (int b = 0; b < nb; ++b) {
                    const int32_t enc = ref(k, b, l);
                    if (!dynamic_ref(enc)) continue;
                    const uint32_t idx = (uint32_t)enc & kRefIndexMask;
                    if ((int)idx >= body_count) {
                        *error = "end_constraints: body reference out of range";
                        return BEPUCUDA_ERR_INVALID_ARGUMENT;
                    }
                    lvl = std::max(lvl, last_level[idx]);
                }
                lane_level[(size_t)l] = lvl + 1;
            }
            for (int l = 0; l < W; ++l) {
                if (lane_level[(size_t)l] == 0) continue;
                for (int b = 0; b < nb; ++b)
                    if (dynamic_ref(ref(k, b, l))) last_level[(uint32_t)ref(k, b, l) & kRefIndexMask] = lane_level[(size_t)l];
                // TypeProcessor.cs:L338-359: a fallback bundle never holds a dynamic body twice (two lanes of one level would race on its record)
                for (int l2 = 0; l2 < l; ++l2) {
                    if (lane_level[(size_t)l2] == 0) continue;
                    for (int b = 0; b < nb; ++b) {
                        const int32_t e1 = ref(k, b, l);
                        if (!dynamic_ref(e1)) continue;
                        for (int b2 = 0; b2 < nb; ++b2) {
                            const int32_t e2 = ref(k, b2, l2);
                            if (dynamic_ref(e2) && (((uint32_t)e1 ^ (uint32_t)e2) & kRefIndexMask) == 0) {
                                *error = "end_constraints: a fallback bundle references the same dynamic body more than once";
                                return BEPUCUDA_ERR_BATCH_INVARIANT;
                            }
                        }
                    }
                }
                slots.push_back({lane_level[(size_t)l], (int)rank, k * W + l});
                ++p.source_live[(size_t)order[rank]];
                ++p.constraint_count;
            }
        }
    }
    // one device batch per level; within it one device type batch per source, its slots mapped to the source constraints
    std::stable_sort(slots.begin(), slots.end(), [](const Slot& a, const Slot& b) { return a.level != b.level ? a.level < b.level : a.rank < b.rank; });
    for (size_t i = 0; i < slots.size();) {
        const int level = slots[i].level;
        batch_tbs.emplace_back();
        ++p.fallback_levels;
        while (i < slots.size() && slots[i].level == level) {
            const int rank = slots[i].rank;
            size_t j = i;
            while (j < slots.size() && slots[j].level == level && slots[j].rank == rank) ++j;
            add_tb(order[(size_t)rank], (int)batch_tbs.size() - 1, (int)(j - i), (int64_t)p.maps.size());
            for (size_t q = i; q < j; ++q) p.maps.push_back(slots[q].constraint);
            p.maps.resize((size_t)p.tbs.back().map_offset + (size_t)p.tbs.back().bundle_count * 32, -1);
            i = j;
        }
    }

    // arenas of the AOSOA-32 image
    for (PlannedTypeBatch& tb : p.tbs) {
        const TypeInfo* t = get_type_info(tb.type_id);
        tb.refs_offset = p.refs_words;
        tb.prestep_offset = p.prestep_words;
        tb.impulse_offset = p.impulse_words;
        p.refs_words += (size_t)tb.bundle_count * t->bodies * 32;
        p.prestep_words += (size_t)tb.bundle_count * t->prestep_rows * 32;
        p.impulse_words += (size_t)tb.bundle_count * t->impulse_rows * 32;
    }

    // work lists: per device batch (one warp per bundle), then the incremental-update list over all contact bundles
    auto add_bundles = [&](int tb) {
        const PlannedTypeBatch& d = p.tbs[(size_t)tb];
        for (int k = 0; k < d.bundle_count; ++k) {
            p.work.push_back({tb, k});
            // identity-mapped type batches: lanes beyond the source count are padding; mapped (fallback level) ones: -1 entries are padding
            int live = 0;
            if (d.map_offset < 0) live = std::max(0, std::min(32, sources[(size_t)d.source].count - k * 32));
            else for (int l = 0; l < 32; ++l) live += p.maps[(size_t)d.map_offset + (size_t)k * 32 + l] >= 0;
            p.bundle_live.push_back(live);
        }
    };
    for (const auto& list : batch_tbs) {
        const int begin = (int)p.work.size();
        bool contacts_only = true;
        for (int tb : list) {
            contacts_only = contacts_only && get_type_info(p.tbs[(size_t)tb].type_id)->contacts > 0;
            add_bundles(tb);
        }
        p.batches.push_back({begin, (int)p.work.size() - begin, contacts_only ? 1 : 0});
    }
    p.all_work_count = (int)p.work.size();
    p.inc_begin = p.all_work_count;
    for (size_t tb = 0; tb < p.tbs.size(); ++tb)
        if (get_type_info(p.tbs[tb].type_id)->contacts > 0) add_bundles((int)tb);
    p.inc_count = (int)p.work.size() - p.inc_begin;
    return BEPUCUDA_OK;
}

std::vector<WorkRecord> work_records(const TopologyPlan& plan, int32_t* refs, float* prestep, float* impulses) {
    std::vector<WorkRecord> records(plan.work.size());
    for (size_t i = 0; i < plan.work.size(); ++i) {
        const WorkItem& w = plan.work[i];
        const PlannedTypeBatch& tb = plan.tbs[(size_t)w.type_batch];
        const TypeInfo* t = get_type_info(tb.type_id);
        WorkRecord& r = records[i];
        r.refs = refs + tb.refs_offset + (size_t)w.bundle * t->bodies * 32;
        r.prestep = prestep + tb.prestep_offset + (size_t)w.bundle * t->prestep_rows * 32;
        r.impulses = impulses + tb.impulse_offset + (size_t)w.bundle * t->impulse_rows * 32;
        r.type_id = tb.type_id;
        r.live_lanes = plan.bundle_live[i];
    }
    return records;
}

// ---- stage program ---------------------------------------------------------------------------------------------------------
StageProgram build_stage_program(const TopologyPlan& plan, const std::vector<int32_t>& iterations, int kinematic_count, bool integrate_velocity_for_kinematics,
                                 bool peer_mode, int body_count) {
    StageProgram prog;
    std::vector<StageOp>& ops = prog.ops;
    auto push = [&](int32_t stage, int32_t begin, int32_t count, int32_t exchange, int32_t flags, int64_t bytes) {
        ops.push_back({stage, begin, count, exchange, 0u, flags, bytes});
    };
    // algorithmic bytes of one pass over a slice of the work list, summed once per device batch (a program repeats every batch many times)
    auto work_bytes = [&](int32_t begin, int32_t count, int32_t TypeInfo::*per) {
        int64_t bytes = 0;
        for (int32_t w = begin; w < begin + count; ++w)
            bytes += (int64_t)(get_type_info(plan.tbs[(size_t)plan.work[(size_t)w].type_batch].type_id)->*per) * plan.bundle_live[(size_t)w];
        return bytes;
    };
    std::vector<int64_t> warm_start_bytes, solve_bytes;
    for (const TopologyPlan::Batch& bw : plan.batches) {
        warm_start_bytes.push_back(work_bytes(bw.begin, bw.count, &TypeInfo::warm_start_bytes));
        solve_bytes.push_back(work_bytes(bw.begin, bw.count, &TypeInfo::solve_bytes));
    }
    auto batch_stages = [&](int32_t stage, int32_t flags) {
        // in peer mode every rank runs the exchange point of every batch, also of one it has no constraint in
        for (size_t b = 0; b < plan.batches.size(); ++b) {
            const TopologyPlan::Batch& bw = plan.batches[b];
            if (bw.count > 0 || (peer_mode && (int)b < plan.sync_batch_count))
                push(stage, bw.begin, bw.count, peer_mode ? (int32_t)b : kNoExchange, flags | (bw.contacts_only ? kLaunchContactsOnly : 0),
                     stage == kStageSolve ? solve_bytes[b] : warm_start_bytes[b]);
        }
    };
    // In substeps > 0 the incremental contact update integrates the pose and world inertia of every body that a constraint lane integrates, and
    // the WarmStart stages only integrate velocity. That update is exact there: a body's pose update depends on its pose, its local inertia and its
    // velocity at the start of the substep, and nothing writes those between the start of the substep and the WarmStart of the body's first batch
    // (the incremental update writes rows, the kinematic pass kinematic bodies, and earlier batches do not reference the body). Peer-sharded
    // solves keep the integration in the owning lane, which also pushes the new records to the peers.
    const int32_t bodies_integrated = plan.inc_count > 0 && !peer_mode ? kLaunchBodiesIntegrated : 0;
    const int64_t incremental_bytes = work_bytes(plan.inc_begin, plan.inc_count, &TypeInfo::incremental_bytes);
    const int64_t kinematic_bytes = (int64_t)kinematic_count * 108;  // per-body passes: 108 bytes per body
    const int substeps = (int)iterations.size();
    for (int s = 0; s < substeps; ++s) {
        if (s > 0) {
            // peer sharding: what peers pushed in the last Solve stages must have arrived before the contact update reads velocities
            if (peer_mode) push(kStageKinematic, 0, 0, kRankBarrier, 0, 0);
            if (plan.inc_count > 0) push(kStageIncremental, plan.inc_begin, plan.inc_count, kNoExchange, bodies_integrated, incremental_bytes);
            if (kinematic_count > 0) push(kStageKinematic, 0, kinematic_count, kNoExchange, 0, kinematic_bytes);
        } else if (integrate_velocity_for_kinematics && kinematic_count > 0) {
            push(kStageKinematicFirst, 0, kinematic_count, kNoExchange, 0, kinematic_bytes);
        }
        // all ranks meet before the first stage of a substep's WarmStart: after every peer's last Solve stage has completed, before any peer's
        // WarmStart stage stores into this rank's arrays
        if (peer_mode) push(kStageKinematic, 0, 0, kRankBarrier, 0, 0);
        if (s == 0) batch_stages(kStageWarmStartFirst, 0);
        else batch_stages(kStageWarmStart, bodies_integrated);
        for (int it = 0; it < iterations[(size_t)s]; ++it) batch_stages(kStageSolve, 0);
    }
    if (peer_mode) push(kStageKinematic, 0, 0, kRankBarrier, 0, 0);  // ... and before the final pose pass reads them
    push(kStageFinalPose, 0, body_count, kNoExchange, 0, (int64_t)body_count * 108);

    const StageOp* previous = nullptr;  // last launched stage (rank barriers write nothing)
    for (StageOp& op : ops) {
        op.exchange_index = prog.exchange_count;
        if (op.exchange != kNoExchange) ++prog.exchange_count;
        if (op.exchange == kRankBarrier) continue;
        if (op.stage <= kStageIncremental) {
            // Row prefetch in the PDL prologue (constraint_stage_kernel): allowed when the stage launched immediately before neither rewrites this
            // stage's prestep rows (the incremental contact update does) nor its impulses (a stage of the same batch does: single-batch scenes).
            if (op.stage != kStageIncremental && previous && previous->stage != kStageIncremental && !(previous->stage <= kStageSolve && previous->work_begin == op.work_begin))
                op.launch_flags |= kLaunchPrefetchRows;
            // Body-record loads in the PDL prologue (constraint_stage_body): allowed for a WarmStart / Solve stage when the stage launched immediately
            // before belongs to this solve (what ran before the solve, such as a body upload, has no stage to order against) and is not the WarmStart
            // of the same batch, the only stage that writes the records these loads read: world inertia and pose of this batch's bodies, the pose
            // of an integrating one.
            if (op.stage <= kStageSolve && previous && !(previous->stage <= kStageWarmStart && previous->work_begin == op.work_begin))
                op.launch_flags |= kLaunchPrefetchBodies;
        }
        if (op.stage == kStageFinalPose ? body_count > 0 : op.work_count > 0) previous = &op;
        if (op.work_count > 0 || op.stage == kStageFinalPose) ++prog.stage_count;
        if (op.stage != kStageKinematicFirst && op.stage != kStageKinematic) prog.algorithmic_bytes += op.algorithmic_bytes;
    }
    int64_t iterations_per_constraint = 0;
    for (int32_t n : iterations) iterations_per_constraint += n;
    prog.constraint_iterations = plan.constraint_count * iterations_per_constraint;
    return prog;
}

int exchange_targets(const StageProgram& program, const std::vector<int32_t>& boundary_count, std::vector<unsigned long long>* targets, std::string* error) {
    if (program.exchange_count + 1 > (uint32_t)kShardMaxExchanges) {
        *error = "peer sharding: more than 4095 exchange points per solve";
        return BEPUCUDA_ERR_BAD_STATE;
    }
    targets->assign((size_t)kShardMaxExchanges, 0ull);
    unsigned long long arrived = 0;
    for (const StageOp& op : program.ops) {
        if (op.exchange == kNoExchange) continue;
        if (op.exchange >= 0 && op.work_count > 0) arrived += (unsigned long long)boundary_count[(size_t)op.exchange];
        (*targets)[op.exchange_index] = arrived;
    }
    targets->back() = arrived;
    return BEPUCUDA_OK;
}

std::vector<int32_t> sort_boundary_first(const TopologyPlan& plan, const uint8_t* is_boundary, std::vector<WorkRecord>& records) {
    std::vector<int32_t> boundary_count(plan.batches.size(), 0);
    std::vector<WorkRecord> sorted;
    for (size_t b = 0; b < plan.batches.size(); ++b) {
        const int begin = plan.batches[b].begin, count = plan.batches[b].count;
        sorted.clear();
        for (int pass = 0; pass < 2; ++pass)
            for (int i = begin; i < begin + count; ++i)
                if ((is_boundary[(size_t)i] != 0) == (pass == 0)) {
                    WorkRecord r = records[(size_t)i];
                    r.live_lanes = (r.live_lanes & ~kRecordBoundaryBit) | (pass == 0 ? kRecordBoundaryBit : 0);
                    sorted.push_back(r);
                    boundary_count[b] += pass == 0;
                }
        std::copy(sorted.begin(), sorted.end(), records.begin() + begin);
    }
    return boundary_count;
}

}  // namespace bepucuda
