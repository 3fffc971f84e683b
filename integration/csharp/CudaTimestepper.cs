// CudaTimestepper<TCallbacks> : ITimestepper — DefaultTimestepper.Timestep (BepuPhysics/DefaultTimestepper.cs:L28-43) with the Solve stage on the GPU.
// Not compiled here (no .NET toolchain in the build image). Usage:
//   var callbacks = new DemoPoseIntegratorCallbacks(gravity, linearDamping, angularDamping);
//   Simulation.Create(pool, narrowPhaseCallbacks, callbacks, solveDescription,
//                     new CudaTimestepper<DemoPoseIntegratorCallbacks>(callbacks, gravity, linearDamping, angularDamping));
// The device integrates velocities with the declarative descriptor (gravity, damping) — it cannot call the user's IntegrateVelocity — so the three
// BEHAVIOURAL properties of the callbacks (IPoseIntegratorCallbacks, PoseIntegrator.cs:L42-94) are taken from the SAME callbacks instance the
// simulation was created with, and checked again every frame against the simulation's own copy: the two paths cannot diverge silently.
using System;
using System.Numerics;
using BepuPhysics;
using BepuUtilities;
using BepuCuda;

public unsafe class CudaTimestepper<TCallbacks> : ITimestepper, IDisposable where TCallbacks : struct, IPoseIntegratorCallbacks
{
    public event TimestepperStageHandler BeforeCollisionDetection;   // ITimestepper.cs:L20
    public event TimestepperStageHandler CollisionsDetected;         // ITimestepper.cs:L25
    /// <summary>Set when the application subscribes to Solver.SubstepStarted / SubstepEnded (Solver_Solve.cs:L1423,L1478): the device solve raises
    /// neither, so frames are then solved by simulation.Solve on the CPU.</summary>
    public bool SubstepEventsInUse;
    IntPtr ctx;
    IntegratorDesc integrator;
    ulong uploadedTopology;   // signature of the constraint graph the device currently holds (0 = none)
    float[] bodyAccelerations;  // SetBodyAccelerations: 8 floats per active-set body index, uploaded after the bodies every frame (null = none)

    /// <summary>Per-body accelerations added as a * dt after the declarative callback (PerBodyGravityDemo's IntegrateVelocity): 8 floats per
    /// active-set body index {ax, ay, az, 0, alpha_x, alpha_y, alpha_z, 0}. The application keeps the array in step with the active set (its length is
    /// checked against the body count every frame); null switches them off.</summary>
    public void SetBodyAccelerations(float[] accelerations) => bodyAccelerations = accelerations;

    /// <summary>Gravity towards a point after the declarative callback (PlanetDemo's IntegrateVelocity: center = PlanetCenter, strength = Gravity);
    /// null switches it off.</summary>
    public void SetPointGravity(Vector3? center, float strength)
    {
        if (center is Vector3 c)
        {
            var xyz = stackalloc float[3] { c.X, c.Y, c.Z };
            Check(Native.bepucuda_set_point_gravity(ctx, 1, xyz, strength));
        }
        else
        {
            Check(Native.bepucuda_set_point_gravity(ctx, 0, null, 0));
        }
    }

    public CudaTimestepper(in TCallbacks callbacks, Vector3 gravity, float linearDamping = 0.03f, float angularDamping = 0.03f, int device = 0, bool strict = false)
    {
        Config cfg = default; cfg.DeviceOrdinal = device; cfg.StrictFp = strict ? 1 : 0; cfg.ExecutionMode = 0;
        IntPtr c; Check(Native.bepucuda_create(&cfg, &c)); ctx = c;
        integrator.Gravity[0] = gravity.X; integrator.Gravity[1] = gravity.Y; integrator.Gravity[2] = gravity.Z;
        integrator.LinearDamping = linearDamping; integrator.AngularDamping = angularDamping;   // DemoPoseIntegratorCallbacks (Demos/DemoCallbacks.cs:L12-105)
        integrator.AngularIntegrationMode = (int)callbacks.AngularIntegrationMode;               // PoseIntegrator.cs:L59
        integrator.AllowSubstepsForUnconstrained = callbacks.AllowSubstepsForUnconstrainedBodies ? 1 : 0;   // L66
        integrator.IntegrateVelocityForKinematics = callbacks.IntegrateVelocityForKinematics ? 1 : 0;             // L72
    }

    bool CallbacksMatch(Simulation simulation)
    {
        if (simulation.PoseIntegrator is not PoseIntegrator<TCallbacks> poseIntegrator) return false;
        ref var live = ref poseIntegrator.Callbacks;
        return (int)live.AngularIntegrationMode == integrator.AngularIntegrationMode
            && (live.AllowSubstepsForUnconstrainedBodies ? 1 : 0) == integrator.AllowSubstepsForUnconstrained
            && (live.IntegrateVelocityForKinematics ? 1 : 0) == integrator.IntegrateVelocityForKinematics;
    }

    public void Timestep(Simulation simulation, float dt, IThreadDispatcher threadDispatcher = null)
    {
        simulation.Sleep(threadDispatcher);
        simulation.PredictBoundingBoxes(dt, threadDispatcher);
        BeforeCollisionDetection?.Invoke(dt, threadDispatcher);
        simulation.CollisionDetection(dt, threadDispatcher);
        CollisionsDetected?.Invoke(dt, threadDispatcher);
        // CPU path, as before, when the frame cannot run on the device: an unsupported constraint type, callbacks whose behavioural properties differ
        // from the descriptor this timestepper was built with, or substep events in use.
        if (SubstepEventsInUse || !CallbacksMatch(simulation) || !SolveOnDevice(simulation, dt))
            simulation.Solve(dt, threadDispatcher);
        simulation.IncrementallyOptimizeDataStructures(threadDispatcher);
    }

    bool SolveOnDevice(Simulation simulation, float dt)
    {
        var solver = simulation.Solver;
        ref var bodies = ref simulation.Bodies.ActiveSet;
        // SolveDescription (SolveDescription.cs:L21-38): the scheduler is evaluated host-side (Solver_Solve.cs:L743-751).
        var iterations = stackalloc int[solver.SubstepCount];
        // GetVelocityIterationCountForSubstepIndex: a scheduler result below 1 falls back to VelocityIterationCount (Solver_Solve.cs:L743-751).
        for (int i = 0; i < solver.SubstepCount; ++i)
        {
            int scheduled = solver.VelocityIterationScheduler == null ? solver.VelocityIterationCount : solver.VelocityIterationScheduler(i);
            iterations[i] = scheduled < 1 ? solver.VelocityIterationCount : scheduled;
        }
        Check(Native.bepucuda_set_solve_description(ctx, solver.SubstepCount, iterations, solver.FallbackBatchThreshold));
        fixed (IntegratorDesc* d = &integrator) Check(Native.bepucuda_set_integrator(ctx, d));
        Check(Native.bepucuda_upload_bodies(ctx, bodies.DynamicsState.Memory, bodies.Count));                       // BodySet.cs:L33
        if (bodyAccelerations == null) Check(Native.bepucuda_set_body_accelerations(ctx, null, 0));
        else fixed (float* a = bodyAccelerations) Check(Native.bepucuda_set_body_accelerations(ctx, a, bodyAccelerations.Length / 8));

        // Frames whose constraint graph did not change (same type batches, same body references, same kinematics) only refresh what the
        // narrow phase rewrote: the device keeps its batch analysis and the captured CUDA graph (INTEGRATION.md, performance notes).
        ref var set = ref solver.ActiveSet;
        ulong topology = TopologySignature(simulation);
        if (topology == uploadedTopology)
        {
            for (int b = 0; b < set.Batches.Count; ++b)
            {
                ref var batch = ref set.Batches[b];
                for (int t = 0; t < batch.TypeBatches.Count; ++t)
                {
                    ref var tb = ref batch.TypeBatches[t];
                    Check(Native.bepucuda_update_type_batch(ctx, b, t, tb.PrestepData.Memory, tb.AccumulatedImpulses.Memory));
                }
            }
        }
        else
        {
            uploadedTopology = 0;
            Check(Native.bepucuda_begin_constraints(ctx, Vector<float>.Count, set.Batches.Count));
            for (int b = 0; b < set.Batches.Count; ++b)
            {
                ref var batch = ref set.Batches[b];
                for (int t = 0; t < batch.TypeBatches.Count; ++t)
                {
                    ref var tb = ref batch.TypeBatches[t];                                                             // TypeBatch.cs:L10-27
                    int rc = Native.bepucuda_upload_type_batch(ctx, b, t, tb.TypeId, tb.ConstraintCount, tb.BodyReferences.Memory, tb.PrestepData.Memory, tb.AccumulatedImpulses.Memory);
                    if (rc == -4) return false;   // BEPUCUDA_ERR_UNSUPPORTED_TYPE
                    Check(rc);
                }
            }
            var kinematics = stackalloc int[Math.Max(1, solver.ConstrainedKinematicHandles.Count)];                   // Solver.cs:L68
            for (int i = 0; i < solver.ConstrainedKinematicHandles.Count; ++i)
                kinematics[i] = simulation.Bodies.HandleToLocation[solver.ConstrainedKinematicHandles[i]].Index;
            Check(Native.bepucuda_set_constrained_kinematics(ctx, kinematics, solver.ConstrainedKinematicHandles.Count));
            Check(Native.bepucuda_end_constraints(ctx));
            uploadedTopology = topology;
        }

        Check(Native.bepucuda_solve(ctx, dt));                                                                         // Simulation.cs:L278-290
        Check(Native.bepucuda_download_bodies(ctx, bodies.DynamicsState.Memory, bodies.Count));
        Check(Native.bepucuda_download_impulses(ctx));   // narrow phase redistributes them next frame (NarrowPhaseConstraintUpdate.cs:L81-135)
        return true;
    }

    // FNV-1a over everything bepucuda_end_constraints analyses: batch / type batch shape, every body reference, the constrained kinematics.
    // (~8 bytes per constraint body: a few hundred microseconds for 300 k contacts, against a graph re-capture per frame.)
    static ulong TopologySignature(Simulation simulation)
    {
        var solver = simulation.Solver;
        ref var set = ref solver.ActiveSet;
        ulong h = 14695981039346656037UL;
        void Mix(ulong v) { h = (h ^ v) * 1099511628211UL; }
        Mix((ulong)simulation.Bodies.ActiveSet.Count); Mix((ulong)set.Batches.Count); Mix((ulong)Vector<float>.Count);
        for (int b = 0; b < set.Batches.Count; ++b)
        {
            ref var batch = ref set.Batches[b];
            Mix((ulong)batch.TypeBatches.Count);
            for (int t = 0; t < batch.TypeBatches.Count; ++t)
            {
                ref var tb = ref batch.TypeBatches[t];
                Mix((ulong)tb.TypeId); Mix((ulong)tb.ConstraintCount);
                int bundles = (tb.ConstraintCount + Vector<int>.Count - 1) / Vector<int>.Count;
                int words = bundles * solver.TypeProcessors[tb.TypeId].BodiesPerConstraint * Vector<int>.Count / 2;   // int32 pairs
                var refs = (ulong*)tb.BodyReferences.Memory;
                for (int i = 0; i < words; ++i) Mix(refs[i]);
            }
        }
        for (int i = 0; i < solver.ConstrainedKinematicHandles.Count; ++i) Mix((ulong)solver.ConstrainedKinematicHandles[i].Value);
        return h == 0 ? 1 : h;
    }

    void Check(int rc) { if (rc != 0) throw new InvalidOperationException(System.Runtime.InteropServices.Marshal.PtrToStringAnsi(Native.bepucuda_last_error(ctx))); }
    public void Dispose() { if (ctx != IntPtr.Zero) { Native.bepucuda_destroy(ctx); ctx = IntPtr.Zero; } }
}
