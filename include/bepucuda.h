/*
 * libbepucuda — C ABI of the H100-native constraint solver + integrator for bepuphysics2.
 *
 * This is the drop-in boundary. The reference has no FFI at this seam (SURVEY.md §8b): the
 * solver is a C# class constructed inside Simulation.Create. The entry points below are what
 * a C# `CudaTimestepper : ITimestepper` (BepuPhysics/ITimestepper.cs:L15-34) P/Invokes in
 * place of `simulation.Solve(dt, threadDispatcher)` (BepuPhysics/Simulation.cs:L278-290).
 * Every pointer is a raw host pointer taken straight from the reference's own pinned
 * `Buffer<T>.Memory` fields (BepuUtilities/Memory/Buffer.cs:L13-21); no layout conversion is
 * required on the C# side. INTEGRATION.md shows the binding.
 *
 * Conventions
 *   - every function returns an int32 status: 0 = ok, negative = error; the message for the
 *     last error on a context is available through bepucuda_last_error.
 *   - no exceptions cross the boundary; a context is used from one thread at a time.
 *   - the context owns all device memory, streams, CUDA graphs and events.
 *   - there is NO CPU fallback: if no CUDA device is usable, bepucuda_create fails with
 *     BEPUCUDA_ERR_NO_DEVICE.
 */
#ifndef BEPUCUDA_H
#define BEPUCUDA_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BEPUCUDA_OK 0
#define BEPUCUDA_ERR_INVALID_ARGUMENT (-1)
#define BEPUCUDA_ERR_NO_DEVICE (-2)
#define BEPUCUDA_ERR_CUDA (-3)
/* Unknown constraint type id: the host shim should fall back to Simulation.Solve for the frame. */
#define BEPUCUDA_ERR_UNSUPPORTED_TYPE (-4)
/* A synchronized batch references the same dynamic body twice (ConstraintBatch invariant,
 * BepuPhysics/Solver.cs:L348-960 debug validators). */
#define BEPUCUDA_ERR_BATCH_INVARIANT (-5)
#define BEPUCUDA_ERR_BAD_STATE (-6)
#define BEPUCUDA_ERR_OUT_OF_MEMORY (-7)

typedef struct bepucuda_ctx bepucuda_ctx;

/* How the (substep, stage, batch) sequence of Solver.Solve (Solver_Solve.cs:L1419-1479) is sequenced
 * on the device. */
enum bepucuda_execution_mode {
    BEPUCUDA_EXEC_GRAPH = 0,      /* one kernel per (batch, stage) chained by programmatic dependent launch, whole frame captured in a CUDA graph */
    BEPUCUDA_EXEC_STREAM = 2      /* the same launches issued directly on the stream, no graph (profiling with ncu) */
    /* 1 and 3 were a persistent cooperative kernel (grid barrier per stage) and a dataflow kernel (per-body version dependencies); both measured
     * slower than the graph on every benchmark configuration and were removed: bepucuda_create rejects them. */
};

typedef struct bepucuda_config {
    int32_t device_ordinal;   /* CUDA device to own; one context <-> one GPU */
    /* 1 = kernels compiled with -fmad=false: bit-identical to a non-contracting fp32 CPU evaluation
     * (RyuJIT does not contract Vector<float> expressions; SURVEY.md §7-5). 0 = FMA contraction on (fast). */
    int32_t strict_fp;
    int32_t execution_mode;   /* enum bepucuda_execution_mode */
    int32_t reserved[5];      /* reserved: ignored by bepucuda_create */
} bepucuda_config;

/* Declarative stand-in for the user's IPoseIntegratorCallbacks struct (BepuPhysics/PoseIntegrator.cs:L42-94).
 * Covers Demos/DemoCallbacks.cs:L12-105 (DemoPoseIntegratorCallbacks) exactly:
 *   PrepareForIntegration(dt): linearDampingDt = pow(clamp(1 - linear_damping, 0, 1), dt), same angular, gravityDt = gravity * dt
 *   IntegrateVelocity: v.linear = (v.linear + gravityDt) * linearDampingDt; v.angular *= angularDampingDt
 * This is the one API narrowing of the drop-in (SURVEY.md §7 hard part 4). */
typedef struct bepucuda_integrator_desc {
    float gravity[3];
    float linear_damping;
    float angular_damping;
    int32_t angular_integration_mode;           /* AngularIntegrationMode: 0 Nonconserving, 1 ConserveMomentum, 2 ConserveMomentumWithGyroscopicTorque */
    int32_t allow_substeps_for_unconstrained;   /* IPoseIntegratorCallbacks.AllowSubstepsForUnconstrainedBodies */
    int32_t integrate_velocity_for_kinematics;  /* IPoseIntegratorCallbacks.IntegrateVelocityForKinematics */
} bepucuda_integrator_desc;

/* Replaces SimulationProfiler's Solver / PoseIntegrator stage timers (BepuPhysics/SimulationProfiler.cs:L6-75). */
typedef struct bepucuda_timings {
    float solve_ms;                 /* device time of the last bepucuda_solve (CUDA events on the context stream) */
    float upload_ms;                /* device-side time of the uploads since the previous solve (H2D copies + transposes) */
    float download_ms;              /* device-side time of the last downloads */
    int64_t constraint_count;       /* active constraints (empty fallback lanes excluded) */
    int64_t constraint_iterations;  /* sum over substeps of constraint_count * velocity_iterations(substep) */
    int64_t stage_count;            /* (batch, stage) barriers executed per solve */
    int64_t kernel_launches;        /* kernels launched (or graph kernel nodes executed) by the last solve */
    int64_t algorithmic_bytes;      /* SURVEY.md §8d compulsory-traffic model for the last solve */
    int64_t h2d_bytes;              /* bytes copied host->device since the previous solve */
    int64_t d2h_bytes;              /* bytes copied device->host by the last downloads */
    int32_t device_batch_count;     /* synchronized batches + fallback dependency levels */
    int32_t fallback_level_count;   /* dependency levels the sequential fallback batch was split into */
    int64_t graph_captures;         /* CUDA graphs this context has captured (BEPUCUDA_EXEC_GRAPH): one per stage program and launch context */
} bepucuda_timings;

/* Lifetime. Replaces: construction of Solver<TIntegrationCallbacks> in Simulation.Create (Simulation.cs:L135-141). */
int32_t bepucuda_create(const bepucuda_config* cfg, bepucuda_ctx** out);
int32_t bepucuda_destroy(bepucuda_ctx* ctx);
const char* bepucuda_last_error(bepucuda_ctx* ctx);

/* Static type registry query (mirrors TypeProcessor.BodiesPerConstraint / ConstrainedDegreesOfFreedom,
 * Constraints/TypeProcessor.cs:L31-39, and sizeof(TPrestepData)/sizeof(Vector<float>)).
 * Returns BEPUCUDA_ERR_UNSUPPORTED_TYPE for ids the device cannot solve. */
int32_t bepucuda_type_info(int32_t type_id, int32_t* bodies_per_constraint, int32_t* prestep_floats, int32_t* impulse_floats);

/* Optional: page-lock a host range (e.g. a BufferPool block, BepuUtilities/Memory/BufferPool.cs:L42) so the
 * per-frame copies run at full PCIe/C2C speed. */
int32_t bepucuda_host_register(bepucuda_ctx* ctx, void* ptr, int64_t bytes);
int32_t bepucuda_host_unregister(bepucuda_ctx* ctx, void* ptr);

/* Replaces: Solver.SubstepCount / VelocityIterationCount / VelocityIterationScheduler / FallbackBatchThreshold
 * (BepuPhysics/SolveDescription.cs:L21-38). The scheduler is pre-evaluated host-side into one iteration count per
 * substep (Solver_Solve.cs:L743-751). Batches with index >= fallback_batch_threshold are treated as the
 * sequential fallback batch (Solver.cs:L1878-1884). */
int32_t bepucuda_set_solve_description(bepucuda_ctx* ctx, int32_t substep_count,
                                       const int32_t* velocity_iterations_per_substep,
                                       int32_t fallback_batch_threshold);
/* Replaces: the TIntegrationCallbacks type argument of Solver<T>/PoseIntegrator<T>. */
int32_t bepucuda_set_integrator(bepucuda_ctx* ctx, const bepucuda_integrator_desc* desc);

/* Two optional terms after the declarative callback, for IntegrateVelocity bodies the descriptor cannot express. Each is applied wherever the
 * reference calls IntegrateVelocity and keeps its result: the integrating lane of WarmStart (TypeProcessor.cs:L1204-1283), the kinematic prepasses
 * when integrate_velocity_for_kinematics (PoseIntegrator.cs:L451-535), the final pass of unconstrained bodies (L632-645, L707-712) and
 * bepucuda_predict_bounding_boxes (L339-341, L428). With dt and position what the reference passes the callback at that site (the dt of its
 * PrepareForIntegration; the pose after this substep's pose integration in WarmStart of substeps > 0 and in the kinematic pose prepass):
 *   v.linear  += a_linear[i] * dt;  v.angular += a_angular[i] * dt                     (not damped)
 *   offset = position - center;  d = |offset|;  v.linear -= (attractorDt * offset) * (1 / max(1, d * d * d)),  attractorDt = dt * strength
 * Neither term set: exactly the declarative callback, with no extra arithmetic.
 *
 * bepucuda_set_body_accelerations: per-body accelerations, as Demos/Demos/PerBodyGravityDemo.cs:L20-89 applies them (there: a_linear = (0, g_i, 0)).
 * 8 floats per body {ax, ay, az, 0, alpha_x, alpha_y, alpha_z, 0} indexed by active-set body index, the record shape of a velocity. Copied to
 * the device (counted in h2d_bytes / upload_ms); the caller's buffer is free when the call returns. NULL clears them. body_count must equal the
 * one of the last bepucuda_upload_bodies (else BEPUCUDA_ERR_INVALID_ARGUMENT); if the body count changes afterwards, bepucuda_solve,
 * bepucuda_profile_stages and bepucuda_predict_bounding_boxes return BEPUCUDA_ERR_BAD_STATE before any device work until they are set again or
 * cleared. A peer-sharded rank is given the whole array, like its bodies.
 * bepucuda_set_point_gravity: gravity towards a point, Demos/Demos/PlanetDemo.cs:L20-48 (center = PlanetCenter, strength = Gravity). A frame
 * parameter like the integrator's gravity: changing it does not rebuild the captured graph. enabled = 0 switches it off (center may be NULL).
 * Arbitrary callback code and per-body damping are not covered. */
int32_t bepucuda_set_body_accelerations(bepucuda_ctx* ctx, const float* accelerations, int32_t body_count);
int32_t bepucuda_set_point_gravity(bepucuda_ctx* ctx, int32_t enabled, const float* center, float strength);

/* Replaces: reads of Bodies.ActiveSet.DynamicsState (BepuPhysics/BodySet.cs:L33). `body_dynamics` is the raw
 * Buffer<BodyDynamics>.Memory: body_count records of 128 B (BepuPhysics/BodyProperties.cs:L11-46,L318-338). */
int32_t bepucuda_upload_bodies(bepucuda_ctx* ctx, const void* body_dynamics, int32_t body_count);

/* Replaces: iteration over Solver.ActiveSet.Batches[b].TypeBatches[t] (BepuPhysics/Solver.cs:L24-29,
 * Constraints/TypeBatch.cs:L10-27). source_bundle_width = Vector<float>.Count on the host. */
int32_t bepucuda_begin_constraints(bepucuda_ctx* ctx, int32_t source_bundle_width, int32_t batch_count);
/* body_references / prestep / accumulated_impulses are TypeBatch.BodyReferences / PrestepData / AccumulatedImpulses
 * .Memory in the reference's AOSOA layout (row = Vector<T>; bundle k lane i = constraint k*W+i,
 * BepuUtilities/BundleIndexing.cs:L50). constraint_count = TypeBatch.ConstraintCount (includes interior empty
 * lanes in the fallback batch). The accumulated_impulses pointer is retained until the next
 * bepucuda_begin_constraints so bepucuda_download_impulses can write results back in place. */
int32_t bepucuda_upload_type_batch(bepucuda_ctx* ctx, int32_t batch_index, int32_t type_batch_index, int32_t type_id,
                                   int32_t constraint_count,
                                   const int32_t* body_references, const float* prestep, float* accumulated_impulses);
/* Replaces: Solver.ConstrainedKinematicHandles (Solver.cs:L68), already mapped handle->index through
 * Bodies.HandleToLocation. */
int32_t bepucuda_set_constrained_kinematics(bepucuda_ctx* ctx, const int32_t* body_indices, int32_t count);
/* Replaces: Solver.PrepareConstraintIntegrationResponsibilities (Solver_Solve.cs:L1072-1388): validates the batch
 * invariant, levelises the fallback batch, computes which constraint lane owns each body's integration, builds the
 * stage program and (re)captures the CUDA graph when topology changed. */
int32_t bepucuda_end_constraints(bepucuda_ctx* ctx);

/* Refresh only the per-frame contact data of an already-uploaded type batch (same topology): what the narrow phase
 * rewrites every frame (CollisionDetection/NarrowPhaseConstraintUpdate.cs:L81-135). */
int32_t bepucuda_update_type_batch(bepucuda_ctx* ctx, int32_t batch_index, int32_t type_batch_index,
                                   const float* prestep, float* accumulated_impulses);

/* Device-side contact constraint update, first slice (SURVEY.md §8 f2): the accumulated impulses of contact type batches STAY on the device between
 * frames. Replaces, for a manifold whose constraint type did not change, the impulse half of NarrowPhase.UpdateConstraint
 * (CollisionDetection/NarrowPhaseConstraintUpdate.cs:L147-196): GatherOldImpulses -> RedistributeImpulses (L81-135) -> ScatterNewImpulses
 * (ContactConstraintAccessor.cs:L36-78). The host keeps writing the new description into TypeBatch.PrestepData
 * (Solver.ApplyDescriptionWithoutWaking) and passes that buffer as before.
 *   feature ids: ConstraintCache.FeatureId0.. of the pair (CollisionDetection/PairCache.cs), one int32 per contact: [constraint][contact], contact
 *   count given by the type id (convex 1-4, nonconvex 2-4). Only contact type ids (0-10, 15-17) are accepted.
 * bepucuda_set_contact_features stores the ids that belong to the impulses uploaded with bepucuda_upload_type_batch (call it between
 * begin/end_constraints or any time after). bepucuda_update_contacts uploads the frame's prestep data and NEW feature ids; at the next solve the
 * penetration impulses are redistributed from the old to the new ids on the device (matched ids keep their impulse, the unmatched share the
 * remainder equally); friction impulses are kept, as in the reference. No impulse bytes cross the bus in either direction.
 * A solve transposes in only the rows uploaded since the previous one: every type batch the frame did not name (joint type batches, contact type
 * batches without an update) keeps its device rows, accumulated impulses and incrementally updated depths included. bepucuda_update_type_batch
 * on a contact type batch hands its impulses back to the host: the next solve uses the uploaded ones and does not redistribute, even when
 * bepucuda_update_contacts was called for it in the same frame. The device then still takes the uploaded impulses to belong to the feature ids
 * it held before that frame (the last bepucuda_set_contact_features or redistribution); if they belong to other ids (the host redistributed
 * them itself), call bepucuda_set_contact_features with those ids before the next bepucuda_update_contacts.
 * bepucuda_update_contacts returns BEPUCUDA_ERR_INVALID_ARGUMENT for a type batch without contacts, BEPUCUDA_ERR_BAD_STATE before
 * bepucuda_set_contact_features or when called twice for a type batch without a solve in between. From a registered (mapped) buffer the ids are
 * read by the next solve: keep the buffer unchanged until then. */
int32_t bepucuda_set_contact_features(bepucuda_ctx* ctx, int32_t batch_index, int32_t type_batch_index, const int32_t* feature_ids);
int32_t bepucuda_update_contacts(bepucuda_ctx* ctx, int32_t batch_index, int32_t type_batch_index, const float* prestep, const int32_t* new_feature_ids);
/* The motion half of BodyDynamics only: floats 0-15 of every 128-B record (pose + velocity, BodyProperties.cs:L318-338); the inertia half does not
 * change from frame to frame (local inertia) or is recomputed by the solve (world inertia). 64 B per body over the bus instead of 128. The body
 * count must equal the one of the last bepucuda_upload_bodies. */
int32_t bepucuda_upload_body_motion(bepucuda_ctx* ctx, const void* body_dynamics, int32_t body_count);
int32_t bepucuda_download_body_motion(bepucuda_ctx* ctx, void* body_dynamics_out, int32_t body_count);
/* Write the motion of listed bodies straight into the device's body state: what the host changed through BodyReference between frames (an
 * ApplyImpulse, a new velocity, a teleport, a kinematic mover's pose) without sending the motion of every body. The host mutates its own
 * Bodies.ActiveSet.DynamicsState as before (after bepucuda_download_body_motion it is current) and names the active-set indices it touched.
 *   body_dynamics: the whole DynamicsState buffer, 128-B records as for bepucuda_upload_body_motion; body_indices: count active-set indices.
 *   For each listed index, floats 0-15 of its record (pose and velocity) replace the device's pose and velocity. Local and world inertia are never
 *   written: the stage kernels load local inertia before their grid-dependency wait, and a kinematic <-> dynamic change also changes the constraints'
 *   kinematic bits, so an inertia change goes through bepucuda_upload_bodies and a describe (begin/upload/end_constraints).
 *   Duplicates are allowed and write the same record; count == 0 is OK and changes nothing.
 * Stream-ordered with bepucuda_upload_bodies and bepucuda_upload_body_motion (whichever is called last wins for a body), and seen by the next
 * bepucuda_solve / bepucuda_profile_stages, by bepucuda_predict_bounding_boxes and by bepucuda_download_body_motion / bepucuda_download_bodies, before
 * any solve too. From a buffer registered with bepucuda_host_register one kernel reads the listed records straight from mapped memory when the stream
 * reaches the write: keep them unchanged until then (the next download or synchronize). From any other buffer the listed 64-B halves are gathered
 * into a context-owned pinned staging buffer during the call, and the caller's buffers are free when it returns. The index list is always copied.
 * Adds count * (64 + 4) bytes to h2d_bytes, inside upload_ms; never re-captures the graph. A peer-sharded rank is given the same list as every
 * other rank, as it is given all bodies.
 * BEPUCUDA_ERR_INVALID_ARGUMENT for count < 0, a NULL pointer with count > 0, or an index outside [0, body_count of the last bepucuda_upload_bodies);
 * BEPUCUDA_ERR_BAD_STATE before the first bepucuda_upload_bodies. All are checked before any device work, and a failing call writes nothing. */
int32_t bepucuda_write_bodies(bepucuda_ctx* ctx, const void* body_dynamics, int32_t count, const int32_t* body_indices);

/* Replaces: Solver.Solve (Solver_Solve.cs:L1415-1484) + PoseIntegrator.IntegrateAfterSubstepping
 * (PoseIntegrator.cs:L707-726). Asynchronous on the context stream. */
int32_t bepucuda_solve(bepucuda_ctx* ctx, float dt);
/* Blocks until prior work is done. */
int32_t bepucuda_synchronize(bepucuda_ctx* ctx);

/* Replaces: the in-place writes to Bodies.ActiveSet.DynamicsState done by ScatterVelocities/ScatterPose/ScatterInertia
 * (Bodies_GatherScatter.cs:L484-753). Writes pose, velocity and world inertia into 128-B records; local inertia and
 * padding floats of the destination are left untouched. Blocks until done. */
int32_t bepucuda_download_bodies(bepucuda_ctx* ctx, void* body_dynamics_out, int32_t body_count);
/* Replaces: in-place accumulated impulse updates in TypeBatch.AccumulatedImpulses. Writes every registered host
 * impulse buffer (the narrow phase reads them next frame). Blocks until done. */
int32_t bepucuda_download_impulses(bepucuda_ctx* ctx);
/* Replaces: in-place prestep mutation by IncrementallyUpdateForSubstep (contact depths). Test/diagnostic use. */
int32_t bepucuda_download_prestep(bepucuda_ctx* ctx, int32_t batch_index, int32_t type_batch_index, float* prestep_out);

/* Read listed constraints straight from the device rows, without moving anything else: the state behind NarrowPhase.TryExtractSolverContactData
 * (CollisionDetection/NarrowPhase.cs:L136-145) and Solver.EnumerateAccumulatedImpulses / GetAccumulatedImpulseMagnitude[Squared]
 * (Solver.cs:L1535-1574) on the resident path, where the host's TypeBatch.AccumulatedImpulses and PrestepData go stale after the first frame.
 *   bepucuda_constraint_location: Solver.HandleToConstraint[handle] (ConstraintLocation.cs). set_index 0 is the active set, the only one the device
 *   holds; type_id selects the type batch of that id in batch batch_index.
 *   records_out: count records of 64 int32 (256 B), in the order of `locations`; duplicates are allowed.
 *     word 0      type id
 *     word 1      1 = a live constraint, 0 = an empty lane (a hole of the sequential fallback batch); then words 2-63 are 0
 *     words 2-5   the body references as TypeBatch.BodyReferences holds them: active-set index, bit 30 for a kinematic body, -1 for a slot the type
 *                 does not have
 *     words 6-17  accumulated impulses (float bits) in the row order of <Type>AccumulatedImpulses, EnumerateAccumulatedImpulses' order; then 0
 *     words 18-52 prestep (float bits) in the row order of <Type>PrestepData; then 0
 *     words 53-63 0
 * The rows are the device's as of the later of the last bepucuda_end_constraints and the last bepucuda_solve / bepucuda_profile_stages: for contacts
 * the impulses after redistribution and solve and the depths the incremental update left, what the reference's TypeBatch holds after Solver.Solve.
 * Rows uploaded since then (bepucuda_update_type_batch, bepucuda_update_contacts) are pending and not visible before the next solve.
 * Locations are resolved against the type batches of the last bepucuda_end_constraints. Read after the solve and before the host changes its
 * constraint set: once collision detection has added or removed constraints (which moves IndexInTypeBatch), an index still in range names the
 * device row of another constraint until the next describe.
 * Writes no device state and no host memory but records_out, leaves the captured graph in place, and blocks until the records are written.
 * BEPUCUDA_ERR_BAD_STATE before the first bepucuda_end_constraints and in peer mode (a rank holds its constraints compacted, so host locations do not
 * address them). BEPUCUDA_ERR_INVALID_ARGUMENT for a NULL pointer with count > 0, set_index != 0, a batch out of range, a type id without a type batch
 * in that batch, or an index at or beyond its ConstraintCount; all are checked before any device work and nothing is written. count == 0 is OK. */
typedef struct bepucuda_constraint_location {
    int32_t set_index, batch_index, type_id, index_in_type_batch;
} bepucuda_constraint_location;
int32_t bepucuda_read_constraints(bepucuda_ctx* ctx, int32_t count, const bepucuda_constraint_location* locations, int32_t* records_out);

/* Write the prestep rows of listed constraints straight into the device rows, leaving their accumulated impulses as they are. Replaces
 * Solver.ApplyDescriptionWithoutWaking(ConstraintReference, description) (Solver.cs:L1149-1180) against the device rows on the resident path, where
 * bepucuda_update_type_batch would also send the host's stale accumulated impulses of the whole type batch: the host calls Solver.ApplyDescription
 * on its own buffers as before (waking stays with the host; the device holds the active set only), then forwards the changed lanes here.
 *   locations: as for bepucuda_read_constraints (Solver.HandleToConstraint[handle]), resolved against the type batches of the last
 *   bepucuda_end_constraints.
 *   records: count records of 64 int32 in the layout bepucuda_read_constraints returns, so a record read, patched and written back works as is.
 *   Word 0 must equal the location's type id; words 18 .. 18 + P - 1 are applied, P = prestep_floats of the type (bepucuda_type_info), the
 *   <Type>PrestepData rows in the reference's order. Every other word is ignored: no body reference and no accumulated impulse is written, as
 *   ApplyDescription writes neither. The caller's buffers are free when the call returns.
 * Writes are queued and applied by the next bepucuda_solve / bepucuda_profile_stages, after that frame's whole-type-batch rows
 * (bepucuda_update_type_batch, bepucuda_update_contacts) are transposed in and the impulses redistributed: a write wins over a whole-type-batch upload
 * of the same frame, whichever was called first. Several writes to one constraint before a solve, in one call or across calls, resolve to the last.
 * Until that solve a write is pending: bepucuda_read_constraints and bepucuda_download_prestep do not see it. bepucuda_begin_constraints drops the
 * pending writes (the describe uploads the host's buffers, which already hold what ApplyDescription wrote). Writing a contact's prestep sets its
 * depths to the written values, as the reference's ApplyDescription does.
 * The solve uploads 12 B per distinct constraint written plus its P prestep floats (bepucuda_timings h2d_bytes), inside the upload window
 * (upload_ms); a write does not re-capture the graph.
 * BEPUCUDA_ERR_BAD_STATE before the first bepucuda_end_constraints, between begin and end, and in peer mode. BEPUCUDA_ERR_INVALID_ARGUMENT for every
 * location bepucuda_read_constraints rejects, a location that names a hole of the sequential fallback batch, a word 0 other than the location's
 * type id, a NULL pointer with count > 0, and count < 0. All are checked before anything is queued, and a failing call queues nothing. count == 0
 * is OK and changes nothing. */
int32_t bepucuda_write_constraints(bepucuda_ctx* ctx, int32_t count, const bepucuda_constraint_location* locations, const int32_t* records);

/* Add and remove listed constraints of the device rows: Solver.Add (Solver.cs:L1182-1199; TypeProcessor.AllocateInTypeBatch L314,
 * AllocateInTypeBatchForFallback L451) and Solver.Remove (Solver.cs:L1385-1405 -> RemoveFromBatch L1344-1358, TypeProcessor.Remove L634-720,
 * ConstraintBatch.RemoveTypeBatchIfEmpty ConstraintBatch.cs:L170-185, Solver.RemoveBatchIfEmpty L1294-1336) on the resident path, where a describe
 * would first need every impulse downloaded and then send every type batch back up. The host runs Solver.Add / Solver.Remove on its own buffers as
 * before and decides every location; the device replays the reference's lane moves (the swap-remove of a synchronized type batch, the lane clear and
 * bundle pull of the fallback batch, the removal of emptied type batches and of trailing empty batches), so that afterwards every location the
 * host holds names the same constraint on the device.
 *   Entries apply in list order, each in the state the entries before it left. locations[i]: the Solver.HandleToConstraint entry the host's own
 *   call produced (add) or consumed (remove). Make one call per run of adds or removes, in the order the host applied them; the reference's narrow
 *   phase adds first (OnPreflush) and removes after (the ConstraintRemover jobs of NarrowPhase.Flush).
 *   Add placement must be Solver.Add's: in a synchronized batch index_in_type_batch == the type batch's ConstraintCount; a type id without a type
 *   batch in the batch opens one (index 0) at TypeBatches.Count; batch_index == the batch count opens a batch; in the fallback batch the index names
 *   an empty lane or the first lane of a new bundle at the end.
 *   records: count records of 64 int32 in the layout of bepucuda_read_constraints. Word 0 is the type id, words 2-5 the body references (bit 30:
 *   kinematic), words 6.. the accumulated impulses and words 18.. the prestep, all written as given: zero impulses for a new pair; for a contact
 *   whose type changed, the impulses the host redistributed from the old constraint it read with bepucuda_read_constraints before removing it
 *   (NarrowPhase.UpdateConstraint gathers them before the remove).
 *   feature_ids: 4 int32 per entry, the ids of the entry's impulses for the next bepucuda_update_contacts (words past its contact count ignored);
 *   NULL is allowed when no entry is a contact type, and then no feature id is written.
 *   constrained_kinematics: Solver.ConstrainedKinematicHandles after the host's changes, mapped to active-set indices, as for
 *   bepucuda_set_constrained_kinematics.
 * After a successful call the context is as if the host had described its current buffers, except that every row of a constraint that already
 * existed comes from the device (its accumulated impulses, incrementally updated depths and resident feature ids) and only the listed entries
 * crossed the bus: 16 B per lane copy plus, per add entry, its 256-B record and, with feature_ids, 16 B (bepucuda_timings h2d_bytes, inside
 * upload_ms). An add entry is one lane copy; a synchronized remove is at most one, a fallback remove one lane clear and, when it pulls a bundle,
 * W copies (the clear lane among them). Reads, writes, bepucuda_find_sleepable_islands and bepucuda_update_contacts take the new locations at once;
 * the next solve re-captures the graph. The host buffers passed to bepucuda_upload_type_batch / bepucuda_update_type_batch of a type batch that
 * took an add may since have been reallocated: until that type batch is passed again (bepucuda_update_type_batch or a describe),
 * bepucuda_download_impulses returns BEPUCUDA_ERR_BAD_STATE; bepucuda_read_constraints reads its impulses. The device rows of grown and removed
 * type batches are reused by later growth; a describe releases them all. A contact type batch that never had bepucuda_set_contact_features
 * keeps refusing bepucuda_update_contacts after adds; a type batch the adds create keeps the feature ids they bring.
 * BEPUCUDA_ERR_BAD_STATE before the first bepucuda_end_constraints, between begin and end, in peer mode, and while rows are pending
 * (bepucuda_update_type_batch, bepucuda_update_contacts, bepucuda_set_contact_features or bepucuda_write_constraints since the last solve; a frame
 * is solve, changes, then that frame's uploads and writes). BEPUCUDA_ERR_INVALID_ARGUMENT for count < 0, a NULL pointer with count > 0 (feature_ids
 * aside), a placement other than the above, a word 0 other than the location's type id, a body reference out of range, a remove of a hole or at or
 * beyond ConstraintCount, and a constrained kinematic index out of range. These are found by a dry run of the whole list on the host: a failing
 * call does no device work and changes nothing. An add that breaks the batch invariant (a synchronized batch holding a dynamic body twice) is
 * found by the ownership pass: BEPUCUDA_ERR_BATCH_INVARIANT, and the context needs a describe (bepucuda_solve returns BEPUCUDA_ERR_BAD_STATE until
 * begin/end_constraints). count == 0 re-plans with the new constrained kinematics. */
int32_t bepucuda_add_constraints(bepucuda_ctx* ctx, int32_t count, const bepucuda_constraint_location* locations, const int32_t* records, const int32_t* feature_ids,
                                 const int32_t* constrained_kinematics, int32_t kinematic_count);
int32_t bepucuda_remove_constraints(bepucuda_ctx* ctx, int32_t count, const bepucuda_constraint_location* locations, const int32_t* constrained_kinematics,
                                    int32_t kinematic_count);

int32_t bepucuda_get_timings(bepucuda_ctx* ctx, bepucuda_timings* out);

/* Replaces SimulationProfiler.Start/End (SimulationProfiler.cs:L25-60): CUDA events on the context stream, 16 slots. */
int32_t bepucuda_event_record(bepucuda_ctx* ctx, int32_t slot);
int32_t bepucuda_event_elapsed_ms(bepucuda_ctx* ctx, int32_t slot_begin, int32_t slot_end, float* ms);

/* Per-stage-kind device time of ONE frame, measured with a CUDA event pair around every stage launch (plain stream launches, no graph, no
 * programmatic dependent launch between stages).
 * Index by stage kind: 0 WarmStart(first substep), 1 WarmStart, 2 Solve, 3 IncrementallyUpdateForSubstep, 4/5 kinematic prepasses, 6 final pose pass.
 * algorithmic_bytes follows SURVEY.md §8d. Advances the simulation exactly like bepucuda_solve(ctx, dt), with the same kernel launches. A peer-mode
 * context (bepucuda_shard_import*) returns BEPUCUDA_ERR_BAD_STATE before any device work: one rank alone cannot meet its peers at the rank
 * barriers. */
typedef struct bepucuda_stage_profile {
    float ms[8];
    int64_t launches[8];
    int64_t algorithmic_bytes[8];
} bepucuda_stage_profile;
int32_t bepucuda_profile_stages(bepucuda_ctx* ctx, float dt, bepucuda_stage_profile* out);

/* PredictBoundingBoxes on the device (SURVEY.md §8 f4): the stage DefaultTimestepper runs right before collision detection
 * (PoseIntegrator.PredictBoundingBoxes, PoseIntegrator.cs:L307-370, L424-444), over the body state the solver keeps resident. Per active body:
 * the sleep-candidacy update (UpdateSleepCandidacy, L286-304: |v|^2 + |w|^2 of the CURRENT velocity against BodyActivity.SleepThreshold), the
 * velocity callback with PrepareForIntegration(dt) applied to a copy of the velocity (the integrated velocity is used for the prediction only and
 * is not stored, L339; kinematics only when IntegrateVelocityForKinematics), and for the convex primitive shapes the bounding box and speculative
 * margin BoundingBoxBatcher.ExecuteConvexBatch computes (Collidables/BoundingBoxBatcher.cs:L142-222; IConvexShape.GetBounds of Sphere.cs:L149-160,
 * Capsule.cs:L226-239, Box.cs:L211-222, Cylinder.cs:L222-235; BoundingBoxHelpers.cs:L12-58).
 *   bepucuda_body_shape.type: the reference's shape type id -- 0 sphere (a = radius), 1 capsule (a = radius, b = half length), 2 box (a, b, c = half
 *   width, height, length), 4 cylinder (a = radius, b = half length). Any other value (no shape; triangle, hull, compound, mesh: their bounds stay
 *   on the host) yields valid = 0 for that body; its activity is still updated.
 *   bepucuda_body_activity = BodyActivity (BodyProperties.cs:L386-416), updated in place.
 *   bounds_out: 8 floats per body {min.x, min.y, min.z, speculative margin, max.x, max.y, max.z, valid (1 or 0)}.
 * Uses the body arrays as they are on the device (after bepucuda_upload_bodies / bepucuda_solve) and the integrator set by bepucuda_set_integrator.
 * Results are bit-identical to a non-contracting fp32 evaluation of the reference's expressions. Blocks until the outputs are written. */
typedef struct bepucuda_body_shape {
    int32_t type;
    float a, b, c;
    float minimum_speculative_margin;   /* Collidable.MinimumSpeculativeMargin */
    float maximum_speculative_margin;   /* Collidable.MaximumSpeculativeMargin */
    int32_t allow_expansion_beyond_speculative_margin;  /* Collidable.Continuity.AllowExpansionBeyondSpeculativeMargin */
    int32_t reserved;
} bepucuda_body_shape;
typedef struct bepucuda_body_activity {
    float sleep_threshold;
    uint8_t minimum_timesteps_under_threshold;
    uint8_t timesteps_under_threshold_count;
    uint8_t sleep_candidate;
    uint8_t reserved;
} bepucuda_body_activity;
int32_t bepucuda_set_body_shapes(bepucuda_ctx* ctx, const bepucuda_body_shape* shapes, int32_t body_count);
int32_t bepucuda_predict_bounding_boxes(bepucuda_ctx* ctx, float dt, bepucuda_body_activity* activities, float* bounds_out);

/* Add and remove listed bodies of the device-resident body state: Bodies.Add (Bodies.cs:L183-212 -> BodySet.Add, BodySet.cs:L68-81) and the
 * body half of Bodies.RemoveAt (Bodies.cs:L244-260 -> RemoveFromActiveSet L214-239, BodySet.RemoveAt BodySet.cs:L83-111,
 * Solver.UpdateForBodyMemoryMove Solver.cs:L1444-1482, TypeProcessor.UpdateForBodyMemoryMove TypeProcessor.cs:L807-817,
 * SequentialFallbackBatch.UpdateForDynamicBodyMemoryMove SequentialFallbackBatch.cs:L220-227) on the resident path, where a change in the body
 * count would otherwise need bepucuda_download_impulses and a describe.
 *   bepucuda_add_bodies appends count 128-B BodyDynamics records (what BodySet.Add wrote at [Count, Count + count)), inertia included, in order
 *   at the current body count. No constraint references the new bodies: add their constraints afterwards with bepucuda_add_constraints.
 *   bepucuda_remove_bodies applies body_indices in list order, each a BodySet.RemoveAt on the state the entries before it left: the body count
 *   drops by one and, when the index is below the new count, the last body moves into that slot. Duplicates name whatever body sits at that index
 *   at that point. Every constraint reference to a moved body takes its new index (the kinematic bit kept), and so do the constrained kinematic
 *   indices of the context (a removed one leaves them). Remove the bodies' constraints first (bepucuda_remove_constraints), as RemoveAt does.
 * Per-body arrays set for the current body count move with the bodies: bepucuda_set_body_accelerations and bepucuda_set_body_shapes. An add
 * appends shapes[count] and accelerations[count * 8] to them; NULL for an array the context holds leaves that array at its old count, and then
 * bepucuda_solve / bepucuda_predict_bounding_boxes return BEPUCUDA_ERR_BAD_STATE until it is set again or cleared.
 * Afterwards every call takes the new indices and count: the body uploads, writes and downloads, bepucuda_read_constraints,
 * bepucuda_find_sleepable_islands and the constraint change calls. The next solve re-captures the graph. Bus cost (bepucuda_timings h2d_bytes,
 * inside upload_ms): an add 128 B per body plus 32 B per appended shape and acceleration record; a remove 4 B per index, its composed move table
 * (the new index of each body at or above the new count). A remove re-plans the constraint rows as the constraint change calls do.
 * BEPUCUDA_ERR_BAD_STATE before the first bepucuda_end_constraints, between begin and end, in peer mode, and while rows are pending (as for the
 * constraint change calls). BEPUCUDA_ERR_INVALID_ARGUMENT for count < 0, a NULL body_dynamics / body_indices with count > 0, a body count past
 * 2^28 - 1, an index outside [0, body count at that entry), and a removed body that a live constraint references. The index checks run on the
 * host and the reference check on the device rows, both before any record, row, count or kinematic index changes: a failing call changes
 * nothing. count == 0 is OK and changes nothing. */
int32_t bepucuda_add_bodies(bepucuda_ctx* ctx, const void* body_dynamics, int32_t count, const bepucuda_body_shape* shapes, const float* accelerations);
int32_t bepucuda_remove_bodies(bepucuda_ctx* ctx, int32_t count, const int32_t* body_indices);

/* Device-side batch colouring (SURVEY.md §8 f3). Replaces, for a whole constraint set at once, the batch search Solver.Add runs per constraint
 * (Solver.cs:L1182-1199: the first batch whose referenced-handle set holds none of the constraint's dynamic bodies; kinematic references never
 * block, GetBlockingBodyHandles L1058-1078; index == fallback_batch_threshold is the fallback batch and accepts everything, TryAllocateInBatch
 * L1093-1140; the narrow phase's FindCandidateBatch L984-1014 is the same search). The result is IDENTICAL to running that first-fit search
 * sequentially over the constraints in ascending key order:
 *   BEPUCUDA_COLOR_INSERTION_ORDER  key = constraint index: the batches the reference's Solver.Add sequence produces from an empty solver;
 *   BEPUCUDA_COLOR_HASHED_ORDER     key = (bepucuda_color_hash(index) << 32) | index: a fixed pseudo-random order, which bounds the number of
 *                                   dependent device rounds by O(log n) on bounded-degree constraint graphs (insertion order can chain);
 *   BEPUCUDA_COLOR_BY_PRIORITY      key = (priorities[index] << 32) | index. With priorities = the constraints' CURRENT batch indices no
 *                                   constraint moves to a higher batch and none could move lower afterwards: the fixed point the reference's
 *                                   BatchCompressor (BatchCompressor.cs:L233) approaches a few constraints per frame.
 * encoded_body_references: [constraint][slot] with `bodies_per_constraint` (1..4) slots per constraint: active-set body index, bit 30 set for a
 * kinematic body (Bodies_GatherScatter.cs:L107-139), -1 for an unused slot. body_count bounds the indices. batch_indices_out[i] receives the batch
 * of constraint i (0 .. fallback_batch_threshold), *batch_count_out the number of batches, *rounds_out the dependent device rounds it took
 * (both optional). Host buffers are caller-owned and only used during the call, which blocks until the result is written. */
#define BEPUCUDA_COLOR_INSERTION_ORDER 0
#define BEPUCUDA_COLOR_HASHED_ORDER 1
#define BEPUCUDA_COLOR_BY_PRIORITY 2
int32_t bepucuda_color_constraints(bepucuda_ctx* ctx, int32_t constraint_count, int32_t bodies_per_constraint, const int32_t* encoded_body_references,
                                   int32_t body_count, int32_t fallback_batch_threshold, int32_t order, const uint32_t* priorities,
                                   int32_t* batch_indices_out, int32_t* batch_count_out, int32_t* rounds_out);
/* The hash behind BEPUCUDA_COLOR_HASHED_ORDER: h = i * 0x9E3779B1; h ^= h >> 15; h *= 0x85EBCA77; h ^= h >> 13; h *= 0xC2B2AE3D; h ^= h >> 16 (uint32). */
uint32_t bepucuda_color_hash(uint32_t constraint_index);

/* Sleepable islands on the device: the search of Simulation.Sleep (IslandSleeper.CollectIsland with the SleepPredicate,
 * BepuPhysics/IslandSleeper.cs:L85-223), for every island of the constraint graph the device holds at once instead of from a sampled fraction of
 * the active bodies (TestedFractionPerFrame, Update L925-963).
 *   graph: two active-set bodies share an island when one constraint of the last bepucuda_end_constraints references both -- every batch, the
 *     sequential fallback batch included, every body slot of 1- to 4-body types. Kinematic references connect islands like any other: CollectIsland
 *     walks Solver.EnumerateConnectedBodyReferences, which reports decoded references (Solver.cs:L1781-1784). Empty lanes (-1) are skipped. A body
 *     no constraint references is an island of its own.
 *   island_of_body_out[b] (optional, body_count entries): the smallest active-set index in b's island. The label is unique, so the result does not
 *     depend on the order of the device's atomics.
 *   An island is sleepable when every body in it has activities[i].sleep_candidate != 0 -- exactly when CollectIsland(start, SleepPredicate)
 *     returns true for any start body in it. sleepable_roots_out receives the labels of the sleepable islands in ascending order,
 *     sleepable_body_counts_out their body counts (so the host can apply TargetSleptFraction itself), *sleepable_count_out how many there are;
 *     both arrays need room for body_count entries. *rounds_out (optional): hook-and-shortcut rounds the device ran (each ends with one flag read by the host; they grow like log n,
 *     not like the island's diameter).
 * Reads only activities[i].sleep_candidate; reads and writes no body, impulse or prestep state and leaves the captured graph valid. Blocks until the
 * outputs are written. BEPUCUDA_ERR_BAD_STATE before the first bepucuda_end_constraints and in peer mode (a rank holds only its own constraints);
 * BEPUCUDA_ERR_INVALID_ARGUMENT when body_count differs from the last bepucuda_upload_bodies or a required pointer is NULL. */
int32_t bepucuda_find_sleepable_islands(bepucuda_ctx* ctx, const bepucuda_body_activity* activities, int32_t body_count, int32_t* island_of_body_out,
                                        int32_t* sleepable_roots_out, int32_t* sleepable_body_counts_out, int32_t* sleepable_count_out, int32_t* rounds_out);

/* Multi-GPU, ONE constraint graph over several GPUs with direct NVLink peer stores (SURVEY.md §8e; replaces the reference's multithreaded batch
 * dispatch, Solver_Solve.cs:L458-654, where workers split the constraints of a batch). Bodies are partitioned into owner slabs by the host; every
 * rank (one context per GPU, normally one process per GPU) uploads ALL bodies (only its own slab and the halo it references are kept current) and
 * ONLY ITS OWN constraints, compacted, under their original batch indices, so every rank has the same batch layout. A WarmStart / Solve stage
 * stores each record it writes for a body other ranks also reference straight into those ranks' body arrays (peer memory opened from CUDA IPC
 * handles), from the registers of the lane that computed it, and announces the arrival in their flag blocks; bundles that read such a body in a
 * later stage first wait for those arrivals. Rank barriers in peer memory open every substep and precede the contact update and the final pose
 * pass: no host round trip, no collective library. Within a batch no dynamic body is referenced twice, so exactly one rank writes a given body in
 * a given stage, and every rank's copy of a body it references is bit-identical to the single-GPU solve at every stage.
 *   bepucuda_shard_export: IPC handles of this context's pose / velocity / world-inertia arrays and of its flag block (call after
 *     bepucuda_upload_bodies; the arrays must not be re-allocated afterwards, i.e. keep the body count).
 *   bepucuda_shard_import: this rank's index, the rank count (<= 8) and every rank's exported handles, in rank order.
 *   bepucuda_shard_set_global: per body, the lowest batch index that references it as a dynamic body on ANY rank (INT32_MAX if none) -- the owner of
 *     its integration, Solver_Solve.cs:L951-1044 -- and whether any rank constrains it (final pose pass, PoseIntegrator.cs:L537-693).
 *   bepucuda_shard_set_body_masks: rank_masks[body] has bit r set when rank r references the body (NULL: BEPUCUDA_ERR_INVALID_ARGUMENT).
 *   bepucuda_shard_set_fallback_rank: the rank in [0, rank_count) that owns EVERY constraint of the sequential fallback batch, or -1 (the default) for
 *     none; call it on every rank with the same value, before bepucuda_end_constraints. That rank uploads the fallback type batches as the host has
 *     them (not compacted: the device levelises them by host bundle, Solver_Solve.cs:L546-583 runs them on one worker) and runs the whole fallback
 *     part of every WarmStart / Solve pass, while the other ranks hand off once before and once after it. Out of range, or a context not in peer
 *     mode: BEPUCUDA_ERR_INVALID_ARGUMENT.
 * Call order: upload_bodies, shard_export, (exchange handles), shard_import, shard_set_global, shard_set_body_masks, shard_set_fallback_rank (graphs
 * with a fallback batch), begin/upload/end_constraints.
 * In peer mode bepucuda_end_constraints returns BEPUCUDA_ERR_BAD_STATE when shard_set_body_masks was not called for the current body count, and when
 * a constraint of the sequential fallback batch is uploaded on a rank other than the fallback rank (or no fallback rank is set; the message names the
 * fallback rank). Every rank must have finished uploading a frame's bodies before any rank's bepucuda_solve can complete its first stage: the solve
 * starts with a rank barrier, so issuing upload and solve on each rank in that order is enough. BEPUCUDA_EXEC_GRAPH or _STREAM. */
typedef struct bepucuda_ipc_handles {
    unsigned char bytes[4][64];
} bepucuda_ipc_handles;
int32_t bepucuda_shard_export(bepucuda_ctx* ctx, bepucuda_ipc_handles* out);
int32_t bepucuda_shard_import(bepucuda_ctx* ctx, int32_t rank, int32_t rank_count, const bepucuda_ipc_handles* all_ranks);
/* The same for ranks that live in ONE process (one host thread per context): the other ranks' arrays are taken from their contexts directly
 * (peer access is enabled between different devices) instead of through IPC handles. all_ranks[rank] must be ctx itself. */
int32_t bepucuda_shard_import_contexts(bepucuda_ctx* ctx, int32_t rank, int32_t rank_count, bepucuda_ctx* const* all_ranks);
int32_t bepucuda_shard_set_global(bepucuda_ctx* ctx, const int32_t* first_batch_per_body, const uint8_t* constrained_per_body);
int32_t bepucuda_shard_set_body_masks(bepucuda_ctx* ctx, const uint8_t* rank_masks);
int32_t bepucuda_shard_set_fallback_rank(bepucuda_ctx* ctx, int32_t rank);

#ifdef __cplusplus
}
#endif
#endif /* BEPUCUDA_H */
