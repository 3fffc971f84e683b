// Constraint topology of libbepucuda, decided on the host without the CUDA runtime: the type registry, which device batch every constraint
// runs in (synchronized batches, then the dependency levels of the sequential fallback batch), the work list the stage kernels walk, and the
// stage program of one solve, and how each of its stages is launched. bepucuda_api.cu turns a plan into device tables; tests/test_topology.py
// checks plans and launches on the CPU.
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
    int32_t fallback_rank = -1;               // peer sharding: the rank that runs the whole fallback batch, -1 = none (no rank may have one)
    int64_t constraint_count = 0;
    std::vector<int32_t> source_live;         // constraints actually present per source (fallback type batches may contain holes)
    std::vector<int32_t> source_bundle_base;  // per source: its first host-width bundle in the per-bundle flag array
    int32_t source_bundles = 0;
    size_t refs_words = 0, prestep_words = 0, impulse_words = 0;
};

// Plans the device batches of `sources` (bundle width W; batches from fallback_threshold on form the sequential fallback batch). In peer mode,
// `rank` is this rank and `fallback_rank` the rank that owns every fallback constraint (bepucuda_shard_set_fallback_rank; -1 = none): only that
// rank may have fallback sources, and it levelises them as a single context does. Returns BEPUCUDA_OK, or an error code with `error` set:
// BEPUCUDA_ERR_BAD_STATE for a fallback source in peer mode on a rank other than the fallback rank (or with none set), BEPUCUDA_ERR_INVALID_ARGUMENT
// for a fallback body reference out of range, BEPUCUDA_ERR_BATCH_INVARIANT for a fallback bundle that holds a dynamic body twice.
int plan_topology(const std::vector<SourceView>& sources, int W, int fallback_threshold, int batch_count, int body_count, bool peer_mode, TopologyPlan* plan,
                  std::string* error, int rank = 0, int fallback_rank = -1);

// What the solver kernels read per work item, with the plan's offsets applied to the arena bases.
std::vector<WorkRecord> work_records(const TopologyPlan& plan, int32_t* refs, float* prestep, float* impulses);

// Stage program entry, walked by the host when it issues or captures a frame.
struct StageOp {
    int32_t stage;
    int32_t work_begin;       // into the work list (constraint stages) / unused
    int32_t work_count;       // warps of work (constraint stages), bodies (final pose), kinematics (kinematic stages)
    int32_t exchange;         // peer sharding: kRankBarrier, the device batch of a sharded WarmStart / Solve stage, or kNoExchange
    uint32_t exchange_index;  // exchange points before this op in the solve (FrameParams::exchange_base, ShardStage)
    int32_t launch_flags;     // kOp* below: facts about the op, from which resolve_stage_launch derives its launch
    int64_t algorithmic_bytes;  // SURVEY.md §8d bytes of the stage
};
constexpr int32_t kNoExchange = -1, kRankBarrier = -2;
// Facts about a constraint op:
//   kOpRowsFree: the op launched just before it writes neither this batch's prestep rows (the incremental contact update does) nor its impulses (a
//   stage of the same batch does);
//   kOpContactsOnly: every bundle of the device batch is a contact;
//   kOpBodiesFree: the op launched just before it is a stage of this solve and not the WarmStart of the same batch, the only stage that writes
//   the world inertia and pose of this batch's bodies, and the pose of those it integrates;
//   kOpIntegrable: the incremental op and the WarmStart ops of substeps > 0 of a solve with contacts that is not peer-sharded. Their pose half of
//   the integration may move from the WarmStart stages to the incremental update: a body's pose update depends on its pose, its local inertia and
//   its velocity at the start of the substep, and nothing writes those between the start of the substep and the WarmStart of the body's first
//   batch (the incremental update writes rows, the kinematic pass kinematic bodies, and earlier batches do not reference the body).
constexpr int32_t kOpRowsFree = 2, kOpContactsOnly = 8, kOpBodiesFree = 16, kOpIntegrable = 32;
// WarmStartFirst / WarmStart / Solve ops of at least this many bundles run the deep kernel (the deep budget in bepu_solver_kernels.cu, which
// checks its copy of the threshold against this one).
constexpr int32_t kDeepBatchBundles = 2150;

// What a launch depends on besides its op. A captured graph bakes the resolved launches in, so it is re-captured unless same_launches holds for
// the context it was captured with and the current one.
struct LaunchContext {
    bool integrator_extensions;  // per-body accelerations or point gravity are set
    int32_t angular_mode;        // bepucuda_integrator_desc::angular_integration_mode
    bool profile;                // bepucuda_profile_stages: every launch timed alone, without PDL and without prologue loads
};
struct StageLaunch {
    int32_t kernel;  // StageKernel (constraint ops; kKernelFull otherwise)
    int32_t flags;   // kLaunch*
};
// The one place that decides how an op of the stage program is launched: which instantiation runs, what its prologue loads before the
// grid-dependency wait, and whether the incremental update integrates the bodies' poses.
StageLaunch resolve_stage_launch(const StageOp& op, const LaunchContext& lc);
// Whether resolve_stage_launch launches every op alike in both contexts.
bool same_launches(const LaunchContext& a, const LaunchContext& b);
// Whether a resolved launch runs the contact-only WarmStart instantiation that has no pose integration (launch_stage, bepu_solver_kernels.cu):
// the incremental update of its substep integrates the poses. Its prologue compiles the world-inertia loads only, and it has no kExt.
constexpr bool integrated_warm_start_launch(int32_t stage, const StageLaunch& l) {
    return stage == kStageWarmStart && l.kernel == kKernelContacts && (l.flags & kLaunchBodiesIntegrated) != 0;
}

struct StageProgram {
    std::vector<StageOp> ops;
    uint32_t exchange_count = 0;        // exchange points per solve
    int64_t stage_count = 0;            // (batch, stage) barriers per solve
    int64_t constraint_iterations = 0;  // constraint_count * sum of the velocity iterations
    int64_t algorithmic_bytes = 0;      // constraint stages and the final pose pass; neither the kinematic passes nor the per-body acceleration records
};

// Solver_Solve.cs:L1419-1479, then PoseIntegrator.IntegrateAfterSubstepping. In peer mode with a fallback rank (TopologyPlan::fallback_rank), the
// fallback part of every WarmStart and Solve pass is ONE exchange point on every rank: every level op of it carries the same exchange_index on the
// fallback rank, and a zero-work op holds its place on the others.
StageProgram build_stage_program(const TopologyPlan& plan, const std::vector<int32_t>& iterations, int kinematic_count, bool integrate_velocity_for_kinematics,
                                 bool peer_mode, int body_count);

// Peer sharding: cumulative boundary bundles of this rank through each exchange point of one solve, kShardMaxExchanges slots, the last one the
// per-solve total (ShardStage); the level ops of a fallback section add up into their one exchange point. BEPUCUDA_ERR_BAD_STATE when the program
// has too many exchange points.
int exchange_targets(const StageProgram& program, const std::vector<int32_t>& boundary_count, std::vector<unsigned long long>* targets, std::string* error);

// Peer sharding: moves the boundary records (is_boundary[i] != 0) of every device batch to its front, marks them with kRecordBoundaryBit and
// returns how many each batch has.
std::vector<int32_t> sort_boundary_first(const TopologyPlan& plan, const uint8_t* is_boundary, std::vector<WorkRecord>& records);

}  // namespace bepucuda
