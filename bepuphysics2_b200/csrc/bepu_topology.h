// Constraint topology of libbepucuda, decided on the host without the CUDA runtime: the type registry, which device batch every constraint
// runs in (synchronized batches, then the dependency levels of the sequential fallback batch), the work list the stage kernels walk, and the
// stage program of one solve, and how each of its stages is launched. bepucuda_api.cu turns a plan into device tables; tests/test_topology.py
// checks plans and launches on the CPU.
#pragma once
#include <string>
#include <vector>

#include "../../include/bepucuda.h"
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
    // The inverse, for reads by host location (bepucuda_read_constraints). A synchronized source is one device type batch with identity slots;
    // the constraints of a fallback source are spread over the type batches of its levels.
    std::vector<int32_t> source_type_batch;      // per source: its device type batch if synchronized, else -1
    std::vector<int64_t> source_inverse_offset;  // per source: the first of its `count` entries in `inverse` if fallback, else -1
    std::vector<DeviceSlot> inverse;             // per fallback source constraint: the slot that maps to it, {-1, -1} for a hole
    std::vector<int32_t> source_count;           // per source: its ConstraintCount, holes of a fallback source included
    std::vector<int32_t> location_source;        // per host batch index * 64 + type id: the source of that type batch, -1 = none
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

// A host location (bepucuda_constraint_location, Solver.HandleToConstraint) resolved against a plan.
struct ResolvedLocation {
    int32_t source;         // index into the planned sources
    DeviceSlot at;          // the device slot of the constraint; {-1, -1} for a hole of the sequential fallback batch
    int64_t inverse_entry;  // a fallback source's constraint: its entry in TopologyPlan::inverse; -1 for a synchronized source
};
// The one resolution of bepucuda_read_constraints and bepucuda_write_constraints: the source by (batch, type id), then the identity slot of a
// synchronized type batch or the inverse map of the fallback levels. BEPUCUDA_ERR_INVALID_ARGUMENT (out untouched) when the location names no
// constraint of the active set: set_index != 0, a batch out of range, a type id without a type batch in that batch, or an index outside
// [0, ConstraintCount).
int resolve_location(const TopologyPlan& plan, const bepucuda_constraint_location& location, ResolvedLocation* out);

// The prestep writes of bepucuda_write_constraints waiting for the next solve, one per device slot: a later write to a slot replaces the earlier
// one, in place, so the queue holds each written constraint once, in the order the slots were first written.
struct PrestepWriteQueue {
    std::vector<PrestepWrite> writes;
    std::vector<float> rows;              // the prestep rows of every write, back to back (PrestepWrite::row0)
    // Takes the device type batches of a new plan (bepucuda_end_constraints) and drops every write.
    void plan(const TopologyPlan& p);
    // rows: the `count` prestep floats of the constraint at `at`, a slot of the plan (count: its type's prestep_rows)
    void put(DeviceSlot at, const float* rows, int count);
    void clear();

  private:
    std::vector<int64_t> slot_base_;      // per device type batch: its first slot in entry_of_slot_
    int64_t slots_ = 0;
    std::vector<int32_t> entry_of_slot_;  // per device slot: its entry of `writes`, -1 = none (allocated by the first write of a plan)
};

// bepucuda_write_bodies on the host. check_body_write: BEPUCUDA_ERR_INVALID_ARGUMENT for count < 0 or a NULL pointer with count > 0,
// BEPUCUDA_ERR_BAD_STATE before the first bepucuda_upload_bodies, BEPUCUDA_ERR_INVALID_ARGUMENT for an index outside [0, body_count); *why names
// the failure. Duplicates and count == 0 are OK.
int check_body_write(bool bodies_uploaded, int32_t body_count, const void* body_dynamics, int32_t count, const int32_t* body_indices, const char** why);
// The staging of an unregistered buffer: out[i][0 .. 16) = floats 0-15 (pose and velocity) of the 128-B record body_indices[i], in list order.
void gather_motion_halves(const void* body_dynamics, const int32_t* body_indices, int32_t count, float* out);

// bepucuda_add_constraints / bepucuda_remove_constraints on the host: Solver.Add's placement checked and Solver.Remove's lane moves replayed on the
// context's type batches (its sources), without the rows. A fallback source keeps its AOSOA-W body references (W lanes per row, `count`'s bundles),
// which tell holes from constraints; a synchronized one needs none. A source removed by the replay keeps its place with type_batch_index -1, and
// a new one is appended, so that the lane ops of one call index the sources of the state before it and after it alike.
struct ChangeSource {
    int32_t batch_index, type_batch_index, type_id, count;
    std::vector<int32_t> refs;
};
struct ChangeState {
    std::vector<ChangeSource> sources;
    int32_t batch_count = 0;
};
// Applies `count` entries in list order to *state and appends their lane copies (LaneCopy, in the order the reference writes the lanes) to *ops. Adds (remove = false; records: the 64-word records of the
// entries): a synchronized location must be the end of its type batch, a type id without a type batch in the batch opens one at index 0, batch
// batch_count opens a new batch, and a fallback location must be an empty lane of an existing bundle or the first lane of a new one at the end;
// word 0 must be the location's type id and every body reference must name a body below body_count (bit 30: kinematic). Removes
// (TypeProcessor.Remove, TypeProcessor.cs:L634-720): a synchronized one pulls the last constraint into the hole; a fallback one clears its lane
// and, when that empties the bundle, pulls the last bundle into it and recomputes ConstraintCount from the new last bundle (L647-693). An emptied
// type batch is swap-removed from its batch (ConstraintBatch.RemoveTypeBatchIfEmpty, ConstraintBatch.cs:L170-185), and trailing empty batches are
// dropped (Solver.RemoveBatchIfEmpty, Solver.cs:L1294-1336). BEPUCUDA_ERR_INVALID_ARGUMENT with *error set for the first entry that breaks a rule;
// *state is then partly changed, so callers replay on a copy.
int replay_changes(ChangeState* state, bool remove, int W, int fallback_threshold, int body_count, int32_t count, const bepucuda_constraint_location* locations,
                   const int32_t* records, std::vector<LaneCopy>* ops, std::string* error);
// The lane ops of one call as one parallel step: per written lane, in the order lanes were first written, the lane of the state BEFORE the call
// whose rows it ends with (or kLaneClear / kLaneNew). A lane cleared and later copied elsewhere carries only its cleared body references there.
std::vector<LaneCopy> compose_lane_ops(const std::vector<LaneCopy>& ops);

// bepucuda_remove_bodies on the host: `count` BodySet.RemoveAt (BodySet.cs:L83-111) in list order on `body_count` bodies, each on the state the
// entries before it left (the count drops by one and, when the index is below the new count, the last body moves into its slot), composed into
// one parallel step. *final_count = body_count - count; moved_to[i] (count entries): the new index of the body that was at final_count + i, or -1
// when it was removed. Every moved body comes from [final_count, body_count) and goes to a distinct slot below final_count, and that slot's body
// was removed, so the moves of one step neither read nor write each other's records. BEPUCUDA_ERR_INVALID_ARGUMENT with *error set for count < 0,
// a NULL list with count > 0, or the first index outside [0, count at that entry); nothing else is written then.
int replay_body_removes(int32_t body_count, int32_t count, const int32_t* body_indices, int32_t* final_count, std::vector<int32_t>* moved_to, std::string* error);

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
