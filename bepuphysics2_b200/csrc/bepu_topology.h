// Constraint topology of libbepucuda, decided on the host without the CUDA runtime: the type registry, which device batch every constraint
// runs in (synchronized batches, then the dependency levels of the sequential fallback batch), the work list the stage kernels walk, and the
// stage program of one solve with the launch flags of every stage. bepucuda_api.cu turns a plan into device tables; tests/test_topology.py
// checks plans on the CPU.
#pragma once
#include <string>
#include <vector>

#include "bepu_layout_kernels.h"

namespace bepucuda {

// bodies / prestep floats / impulse floats per BatchTypeId, contacts per manifold (0 for joints: only contacts have an incremental update),
// and SURVEY.md §8d algorithmic bytes per evaluation
struct TypeInfo {
    int32_t bodies, prestep_rows, impulse_rows, contacts;
    int32_t solve_bytes, warm_start_bytes, incremental_bytes;
    const char* name;
};
const TypeInfo* get_type_info(int type_id);  // nullptr if unsupported

// One uploaded type batch (TypeBatch.cs:L10-27). `refs` (host AOSOA-W body references) is read only for fallback sources.
struct SourceView {
    int32_t batch_index, type_batch_index, type_id, count;
    const int32_t* refs;
};

// A device type batch: a whole synchronized source, or the constraints of one fallback source that share a dependency level.
struct PlannedTypeBatch {
    int32_t type_id;
    int32_t bundle_count;    // 32-lane bundles
    int32_t device_batch;
    int32_t source;          // index into the planned sources
    int64_t map_offset;      // fallback levels: first slot of its 32 * bundle_count entries in TopologyPlan::maps; -1 = identity
    size_t refs_offset, prestep_offset, impulse_offset;  // 32-bit words into the AOSOA-32 arenas
};

struct TopologyPlan {
    std::vector<PlannedTypeBatch> tbs;
    std::vector<int32_t> maps;                // per slot of a fallback level: the source constraint, -1 = padding
    std::vector<WorkItem> work;               // grouped by device batch, then the incremental list
    std::vector<int32_t> bundle_live;         // live constraints per work item (parallel to `work`)
    struct Batch { int32_t begin, count, contacts_only; };
    std::vector<Batch> batches;               // per device batch: its slice of `work`; every bundle of it is a contact
    int32_t inc_begin = 0, inc_count = 0;     // the incremental contact update: every contact bundle once
    int32_t all_work_count = 0;               // work[0 .. all_work_count) covers every bundle once
    int32_t sync_batch_count = 0, fallback_levels = 0;
    int64_t constraint_count = 0;
    std::vector<int32_t> source_live;         // constraints actually present per source (fallback type batches may contain holes)
    std::vector<int32_t> source_bundle_base;  // per source: its first host-width bundle in the per-bundle flag array
    int32_t source_bundles = 0;
    size_t refs_words = 0, prestep_words = 0, impulse_words = 0;
};

// Plans the device batches of `sources` (bundle width W; batches from fallback_threshold on form the sequential fallback batch). Returns
// BEPUCUDA_OK, or an error code with `error` set: BEPUCUDA_ERR_BAD_STATE for a fallback batch in peer mode, BEPUCUDA_ERR_INVALID_ARGUMENT for a
// fallback body reference out of range, BEPUCUDA_ERR_BATCH_INVARIANT for a fallback bundle that holds a dynamic body twice.
int plan_topology(const std::vector<SourceView>& sources, int W, int fallback_threshold, int batch_count, int body_count, bool peer_mode, TopologyPlan* plan,
                  std::string* error);

// What the solver kernels read per work item, with the plan's offsets applied to the arena bases.
std::vector<WorkRecord> work_records(const TopologyPlan& plan, int32_t* refs, float* prestep, float* impulses);

// Stage program entry, walked by the host when it issues or captures a frame.
struct StageOp {
    int32_t stage;
    int32_t work_begin;       // into the work list (constraint stages) / unused
    int32_t work_count;       // warps of work (constraint stages), bodies (final pose), kinematics (kinematic stages)
    int32_t exchange;         // peer sharding: kRankBarrier, the device batch of a sharded WarmStart / Solve stage, or kNoExchange
    uint32_t exchange_index;  // exchange points before this op in the solve (FrameParams::exchange_base, ShardStage)
    int32_t launch_flags;     // kLaunchContactsOnly | kLaunchPrefetchRows | kLaunchPrefetchBodies | kLaunchBodiesIntegrated
    int64_t algorithmic_bytes;  // SURVEY.md §8d bytes of the stage
};
constexpr int32_t kNoExchange = -1, kRankBarrier = -2;

struct StageProgram {
    std::vector<StageOp> ops;
    uint32_t exchange_count = 0;        // exchange points per solve
    int64_t stage_count = 0;            // (batch, stage) barriers per solve
    int64_t constraint_iterations = 0;  // constraint_count * sum of the velocity iterations
    int64_t algorithmic_bytes = 0;      // constraint stages and the final pose pass; neither the kinematic passes nor the per-body acceleration records
};

// Solver_Solve.cs:L1419-1479, then PoseIntegrator.IntegrateAfterSubstepping.
StageProgram build_stage_program(const TopologyPlan& plan, const std::vector<int32_t>& iterations, int kinematic_count, bool integrate_velocity_for_kinematics,
                                 bool peer_mode, int body_count);

// Peer sharding: cumulative boundary bundles of this rank through each exchange point of one solve, kShardMaxExchanges slots, the last one the
// per-solve total (ShardStage). BEPUCUDA_ERR_BAD_STATE when the program has too many exchange points.
int exchange_targets(const StageProgram& program, const std::vector<int32_t>& boundary_count, std::vector<unsigned long long>* targets, std::string* error);

// Peer sharding: moves the boundary records (is_boundary[i] != 0) of every device batch to its front, marks them with kRecordBoundaryBit and
// returns how many each batch has.
std::vector<int32_t> sort_boundary_first(const TopologyPlan& plan, const uint8_t* is_boundary, std::vector<WorkRecord>& records);

}  // namespace bepucuda
