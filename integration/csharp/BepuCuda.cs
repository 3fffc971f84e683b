// P/Invoke surface of libbepucuda (include/bepucuda.h). Not compiled in this repository (no .NET toolchain in the build image); it is the
// binding a bepuphysics2 maintainer adds next to their application. Every entry point replaces the reference call cited in the header.
using System;
using System.Runtime.InteropServices;

namespace BepuCuda
{
    [StructLayout(LayoutKind.Sequential)] public unsafe struct IpcHandles { public fixed byte Bytes[256]; }
    [StructLayout(LayoutKind.Sequential)]
    public unsafe struct Config { public int DeviceOrdinal, StrictFp, ExecutionMode; public fixed int Reserved[5]; }

    [StructLayout(LayoutKind.Sequential)]
    public unsafe struct IntegratorDesc
    {
        public fixed float Gravity[3];
        public float LinearDamping, AngularDamping;
        public int AngularIntegrationMode, AllowSubstepsForUnconstrained, IntegrateVelocityForKinematics;
    }

    [StructLayout(LayoutKind.Sequential)]
    public struct Timings
    {
        public float SolveMs, UploadMs, DownloadMs;
        public long ConstraintCount, ConstraintIterations, StageCount, KernelLaunches, AlgorithmicBytes, H2DBytes, D2HBytes;
        public int DeviceBatchCount, FallbackLevelCount;
        public long GraphCaptures;
    }

    [StructLayout(LayoutKind.Sequential)]
    public unsafe struct StageProfile
    {
        public fixed float Ms[8];
        public fixed long Launches[8];
        public fixed long AlgorithmicBytes[8];
    }

    /// <summary>bepucuda_constraint_location: Solver.HandleToConstraint[handle] (ConstraintLocation.cs); SetIndex 0 is the active set. Named apart
    /// from BepuPhysics.ConstraintLocation so that code importing both namespaces still compiles.</summary>
    [StructLayout(LayoutKind.Sequential)]
    public struct CudaConstraintLocation { public int SetIndex, BatchIndex, TypeId, IndexInTypeBatch; }

    public static unsafe class Native
    {
        const string Lib = "bepucuda";
        [DllImport(Lib)] public static extern int bepucuda_create(Config* cfg, IntPtr* ctx);
        [DllImport(Lib)] public static extern int bepucuda_destroy(IntPtr ctx);
        [DllImport(Lib)] public static extern IntPtr bepucuda_last_error(IntPtr ctx);
        [DllImport(Lib)] public static extern int bepucuda_type_info(int typeId, int* bodies, int* prestepFloats, int* impulseFloats);
        [DllImport(Lib)] public static extern int bepucuda_host_register(IntPtr ctx, void* ptr, long bytes);
        [DllImport(Lib)] public static extern int bepucuda_host_unregister(IntPtr ctx, void* ptr);
        [DllImport(Lib)] public static extern int bepucuda_set_solve_description(IntPtr ctx, int substepCount, int* velocityIterationsPerSubstep, int fallbackBatchThreshold);
        [DllImport(Lib)] public static extern int bepucuda_set_integrator(IntPtr ctx, IntegratorDesc* desc);
        /// <summary>Optional terms after the declarative callback: per-body accelerations (PerBodyGravityDemo) and gravity towards a point (PlanetDemo).</summary>
        [DllImport(Lib)] public static extern int bepucuda_set_body_accelerations(IntPtr ctx, float* accelerations, int bodyCount);
        [DllImport(Lib)] public static extern int bepucuda_set_point_gravity(IntPtr ctx, int enabled, float* center, float strength);
        [DllImport(Lib)] public static extern int bepucuda_upload_bodies(IntPtr ctx, void* bodyDynamics, int bodyCount);
        [DllImport(Lib)] public static extern int bepucuda_begin_constraints(IntPtr ctx, int sourceBundleWidth, int batchCount);
        [DllImport(Lib)] public static extern int bepucuda_upload_type_batch(IntPtr ctx, int batchIndex, int typeBatchIndex, int typeId, int constraintCount, void* bodyReferences, void* prestep, void* accumulatedImpulses);
        [DllImport(Lib)] public static extern int bepucuda_set_constrained_kinematics(IntPtr ctx, int* bodyIndices, int count);
        [DllImport(Lib)] public static extern int bepucuda_end_constraints(IntPtr ctx);
        [DllImport(Lib)] public static extern int bepucuda_update_type_batch(IntPtr ctx, int batchIndex, int typeBatchIndex, void* prestep, void* accumulatedImpulses);
        [DllImport(Lib)] public static extern int bepucuda_set_contact_features(IntPtr ctx, int batchIndex, int typeBatchIndex, int* featureIds);
        [DllImport(Lib)] public static extern int bepucuda_update_contacts(IntPtr ctx, int batchIndex, int typeBatchIndex, void* prestep, int* newFeatureIds);
        [DllImport(Lib)] public static extern int bepucuda_upload_body_motion(IntPtr ctx, void* bodyDynamics, int bodyCount);
        [DllImport(Lib)] public static extern int bepucuda_download_body_motion(IntPtr ctx, void* bodyDynamicsOut, int bodyCount);
        /// <summary>Pose and velocity (floats 0-15) of the listed active-set records of DynamicsState into the device's body state; inertia is never written.</summary>
        [DllImport(Lib)] public static extern int bepucuda_write_bodies(IntPtr ctx, void* bodyDynamics, int count, int* bodyIndices);
        [DllImport(Lib)] public static extern int bepucuda_solve(IntPtr ctx, float dt);
        [DllImport(Lib)] public static extern int bepucuda_synchronize(IntPtr ctx);
        [DllImport(Lib)] public static extern int bepucuda_download_bodies(IntPtr ctx, void* bodyDynamicsOut, int bodyCount);
        [DllImport(Lib)] public static extern int bepucuda_download_impulses(IntPtr ctx);
        [DllImport(Lib)] public static extern int bepucuda_download_prestep(IntPtr ctx, int batchIndex, int typeBatchIndex, float* prestepOut);
        /// <summary>Records of 64 ints (type id, live, body references, accumulated impulses, prestep) of the listed constraints, read from the device rows.</summary>
        [DllImport(Lib)] public static extern int bepucuda_read_constraints(IntPtr ctx, int count, CudaConstraintLocation* locations, int* recordsOut);
        /// <summary>Queues the prestep rows (words 18 on) of records in the read layout for the listed constraints; the next solve writes them into the
        /// device rows and keeps their accumulated impulses (Solver.ApplyDescription on the resident path).</summary>
        [DllImport(Lib)] public static extern int bepucuda_write_constraints(IntPtr ctx, int count, CudaConstraintLocation* locations, int* records);
        [DllImport(Lib)] public static extern int bepucuda_get_timings(IntPtr ctx, Timings* timings);
        [DllImport(Lib)] public static extern int bepucuda_event_record(IntPtr ctx, int slot);
        [DllImport(Lib)] public static extern int bepucuda_event_elapsed_ms(IntPtr ctx, int slotBegin, int slotEnd, float* ms);
        [DllImport(Lib)] public static extern int bepucuda_profile_stages(IntPtr ctx, float dt, StageProfile* profile);
        [DllImport(Lib)] public static extern int bepucuda_shard_export(IntPtr ctx, IpcHandles* handles);
        [DllImport(Lib)] public static extern int bepucuda_shard_import(IntPtr ctx, int rank, int rankCount, IpcHandles* allRanks);
        [DllImport(Lib)] public static extern int bepucuda_shard_set_global(IntPtr ctx, int* firstBatchPerBody, byte* constrainedPerBody);
        [DllImport(Lib)] public static extern int bepucuda_shard_set_body_masks(IntPtr ctx, byte* rankMasks);
        [DllImport(Lib)] public static extern int bepucuda_shard_import_contexts(IntPtr ctx, int rank, int rankCount, IntPtr* allRanks);
        /// <summary>The rank that runs the whole sequential fallback batch of a sharded graph (-1: none); same value on every rank, before end_constraints.</summary>
        [DllImport(Lib)] public static extern int bepucuda_shard_set_fallback_rank(IntPtr ctx, int rank);
        /// <summary>PredictBoundingBoxes on the device: sleep candidacy + bounds and speculative margins of sphere / capsule / box / cylinder bodies from the resident body state.</summary>
        [DllImport(Lib)] public static extern int bepucuda_set_body_shapes(IntPtr ctx, BodyShape* shapes, int bodyCount);
        [DllImport(Lib)] public static extern int bepucuda_predict_bounding_boxes(IntPtr ctx, float dt, BodyActivity* activities, float* boundsOut);
        /// <summary>Device-side batch colouring: the batch Solver.Add's first-fit search would pick for every constraint of a list (order 0 = add order, 1 = hashed, 2 = priorities).</summary>
        [DllImport(Lib)] public static extern int bepucuda_color_constraints(IntPtr ctx, int constraintCount, int bodiesPerConstraint, int* encodedBodyReferences, int bodyCount, int fallbackBatchThreshold, int order, uint* priorities, int* batchIndicesOut, int* batchCountOut, int* roundsOut);
        [DllImport(Lib)] public static extern uint bepucuda_color_hash(uint constraintIndex);
        [DllImport(Lib)] public static extern int bepucuda_add_constraints(IntPtr ctx, int count, CudaConstraintLocation* locations, int* records, int* featureIds, int* constrainedKinematics, int kinematicCount);
        [DllImport(Lib)] public static extern int bepucuda_remove_constraints(IntPtr ctx, int count, CudaConstraintLocation* locations, int* constrainedKinematics, int kinematicCount);
        [DllImport(Lib)] public static extern int bepucuda_add_bodies(IntPtr ctx, void* bodyDynamics, int count, BodyShape* shapes, float* accelerations);
        [DllImport(Lib)] public static extern int bepucuda_remove_bodies(IntPtr ctx, int count, int* bodyIndices);
        /// <summary>Sleepable islands on the device: per body the smallest body index of its island, and the islands whose bodies are all sleep candidates (ascending, with body counts).
        /// Call after bepucuda_solve and before IncrementallyOptimizeDataStructures; see INTEGRATION.md.</summary>
        [DllImport(Lib)] public static extern int bepucuda_find_sleepable_islands(IntPtr ctx, BodyActivity* activities, int bodyCount, int* islandOfBodyOut, int* sleepableRootsOut, int* sleepableBodyCountsOut, int* sleepableCountOut, int* roundsOut);
    }
}
