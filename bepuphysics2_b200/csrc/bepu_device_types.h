// Shared host/device plain structs of libbepucuda: how the active set lives in HBM.
//
// Bodies: four arrays of 32-byte records (one 32-B DRAM sector each, two LDG.128 per record), so a Solve lane touches
// exactly two sectors per body (velocity + world inertia) instead of the reference's 128-B AOS BodyDynamics record
// (BepuPhysics/BodyProperties.cs:L318-338) or 13 scattered SoA planes:
//   pose[i]          = { q.x q.y q.z q.w | p.x p.y p.z 0 }
//   velocity[i]      = { lin.x lin.y lin.z 0 | ang.x ang.y ang.z 0 }
//   inertia_local[i] = { xx yx yy zx | zy zz inv_mass 0 }     (inverse inertia tensor, body space)
//   inertia_world[i] = same, world space; valid between a velocity integration and the next pose integration
//
// Constraints: every type batch is AOSOA with a 32-lane bundle (one warp per bundle, lane = constraint): each row of
// body references / prestep data / accumulated impulses is one 128-B line.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace bepucuda {

// Device body reference encoding (host encoding: Bodies_GatherScatter.cs:L107-139 has bit 30 = kinematic, -1 = empty).
// The device adds bit 29: "this constraint lane owns the integration of this body" (the reference keeps that in
// per-type-batch IndexSets, Solver_Solve.cs:L951-1044), so WarmStart needs no second flag stream.
// Bit 28: "some lane of this lane's SOURCE (host-width) bundle owns an integration for this body slot". Only consulted in the
// momentum-conserving angular modes, where the reference's first-substep IntegrateVelocity applies the angular update to every
// lane of a partially integrating bundle before masking (TypeProcessor.cs:L1251-1283), making results bundle-composition dependent.
constexpr uint32_t kRefIndexMask = 0x0FFFFFFFu;
constexpr uint32_t kRefBundleIntegratesBit = 1u << 28;
constexpr uint32_t kRefIntegrateBit = 1u << 29;
constexpr uint32_t kRefKinematicBit = 1u << 30;
constexpr int32_t kRefEmpty = -1;

struct BodyBuffers {
    float4* pose;
    float4* velocity;
    float4* inertia_local;
    float4* inertia_world;
    const uint8_t* constrained;  // 1 if the body is referenced by any constraint or is a constrained kinematic
    const int32_t* first_batch;  // lowest device batch that references the body as a dynamic body (its integrating lane's), INT32_MAX if none
    int32_t count;
};

struct DeviceTypeBatch {
    int32_t type_id;
    int32_t bundle_count;      // 32-lane bundles
    int32_t device_batch;      // index of the device batch (synchronized batches, then fallback levels)
    int32_t pad;
    int32_t* refs;             // [bundle][body slot][32]
    float* prestep;            // [bundle][prestep row][32]
    float* impulses;           // [bundle][impulse row][32]
};

// Per-frame scalars read by every stage kernel through a pointer, so a captured CUDA graph survives dt changes.
struct FrameParams {
    float dt;                  // substep dt
    float inverse_dt;
    float gravity_dt[3];       // PrepareForIntegration(substep dt) products (Demos/DemoCallbacks.cs:L79-86)
    float linear_damping_dt;
    float angular_damping_dt;
    float final_dt;            // dt the final pass uses for unconstrained bodies
    float final_gravity_dt[3];
    float final_linear_damping_dt;
    float final_angular_damping_dt;
    int32_t final_steps;       // integration steps for unconstrained bodies in the final pass
    int32_t angular_mode;
    int32_t integrate_velocity_for_kinematics;
    uint32_t exchange_base;    // peer sharding: number of cross-GPU exchange points executed before this solve (the flag barrier counts them)
    uint32_t shard_solve_index;  // peer sharding: solves since the arrival targets were last published (the arrival counters keep counting)
    // bepucuda_set_body_accelerations / bepucuda_set_point_gravity: the optional velocity terms after the declarative callback
    uint32_t accelerations[2];     // device address of the per-body array {a.xyz 0 | alpha.xyz 0} (active-set index) as two words, which keeps the
                                   // struct 4-byte aligned like every field the stage kernels copy; read only with kIntegrateAccelerations
    uint32_t integrate_extensions;  // kIntegrateAccelerations | kIntegratePointGravity; 0 = the declarative callback alone
    float attractor_center[3];
    float attractor_dt;            // PrepareForIntegration(substep dt) of the point gravity: dt * strength
    float final_attractor_dt;      // the same with final_dt
};
constexpr uint32_t kIntegrateAccelerations = 1u, kIntegratePointGravity = 2u;

enum Stage : int32_t {
    kStageWarmStartFirst = 0,  // substep 0: integrate velocity only (DisallowPoseIntegration)
    kStageWarmStart = 1,       // substep > 0: integrate pose then velocity
    kStageSolve = 2,
    kStageIncremental = 3,
    kStageKinematicFirst = 4,
    kStageKinematic = 5,
    kStageFinalPose = 6,
};

// One entry per warp of a stage launch: which bundle of which device type batch.
struct WorkItem {
    int32_t type_batch;
    int32_t bundle;
};

// What a solver warp needs to process one bundle, in ONE 32-byte record (two LDG.128): no dependent work-item -> type-batch -> pointer chain.
// Pointers address the bundle's row 0, lane 0.
struct alignas(32) WorkRecord {
    int32_t* refs;
    float* prestep;
    float* impulses;
    int32_t type_id;
    int32_t live_lanes;
};

// Peer sharding (bepucuda_shard_*): where the other ranks' body arrays and flag blocks are mapped in this process.
constexpr int kMaxShardRanks = 8;
struct ShardPeers {
    float4* pose[kMaxShardRanks];
    float4* velocity[kMaxShardRanks];
    float4* inertia_world[kMaxShardRanks];
    unsigned long long* flags[kMaxShardRanks];  // flags[r][w]: rank r's block, slot written by rank w
    int32_t rank, rank_count;
};
// One sharded stage = one exchange point. Bundles that touch a body another rank references ("boundary" bundles, kRecordBoundaryBit in
// WorkRecord::live_lanes, sorted to the front of the batch) first wait until every peer's boundary bundles of all earlier exchange points have
// arrived, and announce their own arrival to every peer (one fire-and-forget red.add over NVLink) once their peer stores are out. Interior bundles
// neither wait nor announce, so the NVLink round trip hides behind them. A rank's flag block (u64 slots):
//   [0, 8)  barrier flags, slot w written by rank w (shard_barrier_kernel)
//   [16, 24) arrival counters, slot w incremented by rank w's boundary bundles
//   [32 + w * kShardMaxExchanges ...) rank w's arrival targets: slot e = its boundary bundles through exchange point e of one solve, cumulative;
//                                     the last slot holds the per-solve total
struct ShardStage {
    uint32_t exchange_index;
    int32_t* error_flag;
};
constexpr int kShardCounterSlot = 16;
constexpr int kShardTargetSlot = 32;
constexpr int kShardMaxExchanges = 4096;
constexpr size_t kShardFlagBlockWords = kShardTargetSlot + (size_t)kMaxShardRanks * kShardMaxExchanges;
constexpr int32_t kRecordBoundaryBit = 1 << 30;

}  // namespace bepucuda
