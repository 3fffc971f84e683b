"""TEST INFRASTRUCTURE: the reference's single-threaded frame, restated a second time, independently of oracle/bepu_oracle.cpp's driver.

The constraint functions, PoseIntegration and the convex bounds are calls into the transpiled reference (oracle/_ref/libbepu_ref.so: ref_eval_lane,
ref_eval_integration, ref_convex_bounds), which tests/test_oracle_pinned_to_reference.py and tests/test_bounds.py pin. Everything else (which batch and
lane integrates a body, the stage order, the masks, the callbacks, the final pose pass, sleep candidacy, impulse redistribution) is written here from
the reference's C# text, in numpy float32 in the C# operation order, with the line of each step cited. MathF.Pow is libm's powf.

It works bundle-wise where the reference does: WarmStart integrates a whole bundle under a lane mask, IntegrateBundlesAfterSubstepping and
PredictBoundingBoxes walk body bundles of Vector<float>.Count lanes. It mutates a host `Simulation`'s buffers in place, like oracle.binding.solve, so
tests/util.snapshot and compare apply unchanged.

`mutation` names one driver decision to get wrong on purpose (MUTATIONS); tests/test_oracle_driver_pinned_to_reference.py shows that the scene
matrix notices each of them. Nothing in the product imports this file."""
import ctypes as C
import ctypes.util
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBRARY = os.path.join(ROOT, "oracle", "_ref", "libbepu_ref.so")
FP = C.POINTER(C.c_float)
f32 = np.float32
DYNAMIC_LIMIT = 1 << 30  # Bodies.DynamicLimit = KinematicMask (Bodies_GatherScatter.cs:L107-139)
REFERENCE_MASK = (1 << 30) - 1  # Bodies.BodyReferenceMask
CONTACT_TYPES = (0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 15, 16, 17)  # the only functions with RequiresIncrementalSubstepUpdates => true (ContactConvexTypes.cs, ContactNonconvexTypes.cs)

MUTATIONS = (
    "pose_in_substep_zero",  # WarmStartBlock<AllowPoseIntegration> on substep 0 too (Solver_Solve.cs:L1447-1454)
    "every_batch_integrates",  # integration flags for every batch referencing a body, not only the first (Solver_Solve.cs:L1174-1181)
    "fallback_last_slot",  # the fallback batch's owner is the latest (type batch, index) instead of the earliest (Solver_Solve.cs:L996-1019)
    "kinematic_velocity_prepass_ignores_flag",  # IntegrateKinematicVelocities runs although IntegrateVelocityForKinematics is false (Solver_Solve.cs:L1437-1441)
    "incremental_after_kinematic_pose",  # IntegrateKinematicPosesAndVelocities before the incremental contact update (Solver_Solve.cs:L1426-1436)
    "final_constrained_full_dt",  # constrained bodies take their last pose step with dt instead of substepDt (PoseIntegrator.cs:L587-594)
    "final_constrained_pose_every_step",  # with AllowSubstepsForUnconstrainedBodies, constrained lanes are not masked out after step 0 (L660-667)
    "callback_sees_stepped_position",  # the final pass hands the callback the position after the step (PoseIntegrator.cs:L631-638)
    "final_prepare_substep_dt",  # PrepareForIntegration(substepDt) in the final pass although unconstrained bodies take one dt step (L706-708)
    "sleep_reads_integrated_velocity",  # sleep candidacy measured after the velocity callback (PoseIntegrator.cs:L334-341)
    "kinematic_test_bits",  # Bodies.IsKinematic as an integer comparison of the OR of the bits (Bodies.cs:L326-331 compares floats)
    "unmatched_zero_impulse",  # unmatched contacts start at zero instead of sharing the unmatched impulse (NarrowPhaseConstraintUpdate.cs:L110-131)
)

_LIB = None
_LIBM = None


def library():
    """The transpiled reference, or None where it was not built (no checkout of the reference's C# sources)."""
    global _LIB
    if _LIB is None and os.path.exists(LIBRARY):
        lib = C.CDLL(LIBRARY)
        lib.ref_eval_lane.argtypes = [C.c_int32, C.c_int32, FP, C.c_float, C.c_void_p, C.c_void_p, FP, C.c_int32]
        lib.ref_eval_integration.argtypes = [C.c_int32, FP, FP]
        lib.ref_convex_bounds.argtypes = [C.c_int32, FP, FP, C.c_int32, FP, FP, FP, FP, C.c_float, FP]
        _LIB = lib
    return _LIB


def _powf(x, y):
    global _LIBM
    if _LIBM is None:
        _LIBM = C.CDLL(ctypes.util.find_library("m"))
        _LIBM.powf.argtypes, _LIBM.powf.restype = [C.c_float, C.c_float], C.c_float
    return f32(_LIBM.powf(float(x), float(y)))


def _ptr(a):
    return a.ctypes.data_as(FP)


def _check(mutation):
    assert mutation is None or mutation in MUTATIONS, mutation


# ---- PoseIntegration (PoseIntegrator.cs:L146-253), through the transpiled reference ----------------------------------------------------------------
def _integration(op, inputs, n):
    out = np.zeros(n, dtype=f32)
    assert library().ref_eval_integration(op, _ptr(np.ascontiguousarray(np.concatenate(inputs), dtype=f32)), _ptr(out)) == 0
    return out


def integrate_orientation(q, w, half_dt):
    return _integration(0, [q, w, [half_dt]], 4)


def rotate_inverse_inertia(local, q):
    return _integration(1, [local, q], 6)


def conserve_momentum(previous_orientation, local, world, w):
    return _integration(2, [previous_orientation, local, world, w], 3)


def gyroscopic(q, local, w, dt):
    return _integration(3, [q, local, w, [dt]], 3)


def _length(v):  # Vector3Wide.Length: sqrt(x x + y y + z z)
    return np.sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2])


def _length_squared(v):
    return v[0] * v[0] + v[1] * v[1] + v[2] * v[2]


def is_kinematic(local_inertia7, mutation=None):
    """Bodies.IsKinematic (Bodies.cs:L326-331): Vector.Equals(BitwiseOr(seven floats), Vector<float>.Zero), a float comparison of the OR."""
    bits = np.bitwise_or.reduce(np.ascontiguousarray(local_inertia7, dtype=f32).view(np.uint32))
    if mutation == "kinematic_test_bits":
        return bool(bits == 0)
    return bool(np.array([bits], dtype=np.uint32).view(f32)[0] == f32(0.0))


# ---- the callbacks: DemoCallbacks.cs:L79-105, PerBodyGravityDemo.cs:L57-88, PlanetDemo.cs:L36-46 ---------------------------------------------------
class Callbacks:
    def __init__(self, integrator, accelerations=None, center=None, strength=0.0):
        self.gravity = np.array(list(integrator.gravity), dtype=f32)
        self.linear_damping, self.angular_damping = f32(integrator.linear_damping), f32(integrator.angular_damping)
        self.angular_mode = int(integrator.angular_integration_mode)
        self.allow_substeps = bool(integrator.allow_substeps_for_unconstrained)
        self.integrate_kinematics = bool(integrator.integrate_velocity_for_kinematics)
        self.accelerations = None if accelerations is None else np.ascontiguousarray(accelerations, dtype=f32).reshape(-1, 8)
        self.center = None if center is None else np.array(center, dtype=f32)
        self.strength = f32(strength)

    def prepare(self, dt):
        """PrepareForIntegration: DemoCallbacks.cs:L79-86 (Pow(Clamp(1 - damping, 0, 1), dt), Gravity * dt), PlanetDemo.cs:L36-40 (dt * Gravity)."""
        dt = f32(dt)
        self.linear_damping_dt = _powf(min(max(f32(1) - self.linear_damping, f32(0)), f32(1)), dt)
        self.angular_damping_dt = _powf(min(max(f32(1) - self.angular_damping, f32(0)), f32(1)), dt)
        self.gravity_dt = self.gravity * dt
        self.attractor_dt = dt * self.strength

    def integrate_velocity(self, body_index, position, dt, lin, ang):
        """IntegrateVelocity for one lane. body_index is the lane's entry of the bodyIndices vector: -1 for lanes outside the integration mask
        (TypeProcessor.cs:L1290-1293, PoseIntegrator.cs:L331-332, L618-620), which read no per-body data (PerBodyGravityDemo.cs:L74-83)."""
        lin = (lin + self.gravity_dt) * self.linear_damping_dt
        ang = ang * self.angular_damping_dt
        if self.accelerations is not None:
            a = self.accelerations[body_index] if body_index >= 0 else np.zeros(8, dtype=f32)
            lin = lin + a[0:3] * f32(dt)
            ang = ang + a[4:7] * f32(dt)
        if self.center is not None:
            offset = position - self.center
            distance = _length(offset)
            inverse = f32(1) / max(f32(1), distance * distance * distance)  # Vector3Wide / Vector<float>: times the reciprocal (Vector3Wide.cs:L357-363)
            lin = lin - (self.attractor_dt * offset) * inverse
        return lin, ang


# ---- bodies (BodyProperties.cs:L318-338: orientation 0-3, position 4-6, linear 8-10, angular 12-14, local inertia 16-22, world inertia 24-30) ------
class _Lane:
    __slots__ = ("enc", "index", "q", "pos", "lin", "ang", "inertia", "dt")


def _gather(bodies, enc, world):  # Bodies.GatherState (Bodies_GatherScatter.cs:L267-478)
    s = _Lane()
    s.enc, s.index = int(enc), int(enc) & REFERENCE_MASK
    r = bodies[s.index]
    s.q, s.pos, s.lin, s.ang = r[0:4].copy(), r[4:7].copy(), r[8:11].copy(), r[12:15].copy()
    s.inertia = (r[24:31] if world else r[16:23]).copy()
    return s


def _scatter_velocity(bodies, s):  # ScatterVelocities skips kinematic and empty lanes (Bodies_GatherScatter.cs:L626-753)
    if (s.enc & 0xFFFFFFFF) < DYNAMIC_LIMIT:
        bodies[s.index, 8:11], bodies[s.index, 12:15] = s.lin, s.ang


# ---- Solver.PrepareConstraintIntegrationResponsibilities (Solver_Solve.cs:L951-1044, L1072-1388) ---------------------------------------------------
def integration_responsibilities(batches, body_count, fallback_threshold, W, constrained_kinematics, mutation=None):
    """Returns (flags, constrained): flags[b][t] = None where batch b's type batch t integrates nothing (coarse responsibility false), otherwise one
    boolean array per body slot over the constraints; constrained = the merged constrained body set plus the constrained kinematics."""
    def referenced(batch):  # batchReferencedHandles: the dynamic bodies a batch references (kinematics never block)
        out = np.zeros(body_count, dtype=bool)
        for tb in batch:
            refs = tb.body_references.transpose(1, 0, 2).reshape(tb.bodies, -1)[:, :tb.constraint_count].astype(np.int64) & 0xFFFFFFFF
            out[refs[refs < DYNAMIC_LIMIT]] = True
        return out

    merged = referenced(batches[0]) if batches else np.zeros(body_count, dtype=bool)  # L1100-1102: starts as batch 0's set
    flags = [[None] * len(batch) for batch in batches]
    for b in range(1, len(batches)):
        mine = referenced(batches[b])
        first = mine & ~merged  # L1156-1166: firstObservedBundle = ~merged & batch; merged |= batch
        if mutation == "every_batch_integrates":
            first = mine.copy()
        merged |= mine
        if not first.any():  # batchHasAnyIntegrationResponsibilities false: no region is computed (L1229-1246)
            continue
        fallback = b == fallback_threshold
        earliest = {}
        if fallback:  # L996-1019: the body's earliest constraint in the fallback batch by ((typeBatchIndex << 32) | indexInTypeBatch)
            for t, tb in enumerate(batches[b]):
                for c in range(tb.constraint_count):
                    for slot in range(tb.bodies):
                        enc = int(tb.body_references[c // W, slot, c % W])
                        if enc == -1:
                            continue
                        key, body = (t << 32) | c, enc & REFERENCE_MASK
                        if mutation == "fallback_last_slot":
                            earliest[body] = max(earliest.get(body, -1), key)
                        else:
                            earliest[body] = min(earliest.get(body, 1 << 63), key)
        for t, tb in enumerate(batches[b]):
            per_slot = np.zeros((tb.bodies, tb.constraint_count), dtype=bool)
            for c in range(tb.constraint_count):  # ComputeIntegrationResponsibilitiesForConstraintRegion (L951-1044)
                for slot in range(tb.bodies):
                    enc = int(tb.body_references[c // W, slot, c % W])
                    if fallback and enc == -1:
                        continue
                    body = enc & REFERENCE_MASK
                    if first[body] and (not fallback or earliest[body] == ((t << 32) | c)):
                        per_slot[slot, c] = True
            if per_slot.any():  # L1032-1043: coarse responsibility = any flag of any slot
                flags[b][t] = per_slot
    constrained = merged.copy()
    constrained[np.asarray(constrained_kinematics, dtype=np.int64)] = True  # L1372-1381
    return flags, constrained


# ---- TypeProcessor.GatherAndIntegrate + WarmStart / Solve / IncrementallyUpdateForSubstep ----------------------------------------------------------
def _integrate_pose_and_velocity(cb, s, dt, active):
    """IntegratePoseAndVelocity (TypeProcessor.cs:L1204-1248) for one lane; `active` is its integration mask bit. s.inertia is local on entry, world
    on exit."""
    dt = f32(dt)
    half_dt = dt * f32(0.5)
    new_position = s.pos + s.lin * dt
    if active:
        s.pos = new_position
    local = s.inertia
    previous_lin, previous_ang = s.lin, s.ang
    previous_orientation = s.q
    new_orientation = integrate_orientation(s.q, s.ang, half_dt)
    if active:
        s.q = new_orientation
    world = rotate_inverse_inertia(local[0:6], s.q)
    if cb.angular_mode == 1:
        s.ang = conserve_momentum(previous_orientation, local[0:6], world, s.ang)
    elif cb.angular_mode == 2:
        s.ang = gyroscopic(s.q, local[0:6], s.ang, dt)
    lin, ang = cb.integrate_velocity(s.index if active else -1, s.pos, dt, s.lin, s.ang)  # L1244: the callback sees the integrated pose
    s.lin, s.ang = (lin, ang) if active else (previous_lin, previous_ang)
    s.inertia = np.concatenate([world, local[6:7]])


def _integrate_velocity(cb, s, dt, active, conditional):
    """IntegrateVelocity (TypeProcessor.cs:L1251-1283) for one lane: the angular step runs on every lane, only the callback's result is masked, and
    only under BatchShouldConditionallyIntegrate."""
    dt = f32(dt)
    local = s.inertia
    world = rotate_inverse_inertia(local[0:6], s.q)
    if cb.angular_mode == 1:
        previous_orientation = integrate_orientation(s.q, s.ang, dt * f32(-0.5))
        s.ang = conserve_momentum(previous_orientation, local[0:6], world, s.ang)
    elif cb.angular_mode == 2:
        s.ang = gyroscopic(s.q, local[0:6], s.ang, dt)
    lin, ang = cb.integrate_velocity(s.index if active else -1, s.pos, dt, s.lin, s.ang)
    if active or not conditional:
        s.lin, s.ang = lin, ang
    s.inertia = np.concatenate([world, local[6:7]])


def _lanes(tb, bundle, W):
    """The occupied lanes of a bundle: lanes past the constraint count and the fallback batch's holes (-1 in every slot) carry nothing."""
    return [l for l in range(W) if bundle * W + l < tb.constraint_count and int(tb.body_references[bundle, 0, l]) != -1]


def _eval(tb, stage, bundle, lane, lanes_state, dt, W):
    lib = library()
    states = np.zeros((tb.bodies, 14), dtype=f32)
    velocities = np.zeros((tb.bodies, 6), dtype=f32)
    for slot, s in enumerate(lanes_state):
        states[slot] = np.concatenate([s.pos, s.q, s.inertia])
        velocities[slot] = np.concatenate([s.lin, s.ang])
    pre = tb.prestep.ctypes.data + ((bundle * tb.prestep_rows) * W + lane) * 4
    imp = tb.accumulated_impulses.ctypes.data + ((bundle * tb.impulse_rows) * W + lane) * 4
    assert lib.ref_eval_lane(tb.type_id, stage, _ptr(states), f32(dt), pre, imp, _ptr(velocities), W) == 0
    for slot, s in enumerate(lanes_state):
        s.lin, s.ang = velocities[slot, 0:3].copy(), velocities[slot, 3:6].copy()


def _warm_start_bundle(bodies, cb, tb, bundle, batch_index, flags, allow_pose, dt, W):
    """WarmStartBlock (Solver_Solve.cs:L185-210) -> TypeProcessor.WarmStart: GatherAndIntegrate per body slot (TypeProcessor.cs:L1298-1397), the
    WarmStart function per lane, ScatterVelocities."""
    lanes = _lanes(tb, bundle, W)
    gathered = {l: [None] * tb.bodies for l in lanes}
    for slot in range(tb.bodies):
        refs = tb.body_references[bundle, slot]
        if batch_index == 0:  # BatchShouldAlwaysIntegrate: mask = lanes below DynamicLimit
            mode, mask = "always", [(int(refs[l]) & 0xFFFFFFFF) < DYNAMIC_LIMIT for l in range(W)]
        elif flags is None:  # coarse responsibility false: BatchShouldNeverIntegrate
            mode, mask = "never", None
        else:  # BundleShouldIntegrate (TypeProcessor.cs:L1155-1202)
            mask = [bundle * W + l < tb.constraint_count and bool(flags[slot, bundle * W + l]) for l in range(W)]
            mode = "conditional" if any(mask) else "never"
        for l in lanes:
            s = _gather(bodies, refs[l], world=mode == "never")
            if mode != "never":
                if allow_pose:
                    _integrate_pose_and_velocity(cb, s, dt, mask[l])
                    if mask[l]:  # ScatterPose, ScatterInertia under the integration mask
                        bodies[s.index, 0:4], bodies[s.index, 4:7], bodies[s.index, 24:31] = s.q, s.pos, s.inertia
                else:
                    _integrate_velocity(cb, s, dt, mask[l], conditional=mode == "conditional")
                    if mask[l]:
                        bodies[s.index, 24:31] = s.inertia
            gathered[l][slot] = s
    for l in lanes:
        _eval(tb, 0, bundle, l, gathered[l], dt, W)
    for l in lanes:
        for s in gathered[l]:
            _scatter_velocity(bodies, s)


def _solve_bundle(bodies, tb, bundle, dt, W, stage):
    lanes = _lanes(tb, bundle, W)
    gathered = {l: [_gather(bodies, tb.body_references[bundle, slot, l], world=True) for slot in range(tb.bodies)] for l in lanes}
    for l in lanes:
        _eval(tb, stage, bundle, l, gathered[l], dt, W)
    if stage == 1:
        for l in lanes:
            for s in gathered[l]:
                _scatter_velocity(bodies, s)


# ---- PoseIntegrator kinematic prepasses (PoseIntegrator.cs:L451-535) --------------------------------------------------------------------------------
def _kinematic_velocities(bodies, cb, kinematics, dt):  # IntegrateKinematicVelocities: the callback at the gathered pose, every existing lane
    for index in kinematics:
        s = _gather(bodies, index, world=False)
        s.lin, s.ang = cb.integrate_velocity(s.index, s.pos, dt, s.lin, s.ang)
        bodies[s.index, 8:11], bodies[s.index, 12:15] = s.lin, s.ang


def _kinematic_poses_and_velocities(bodies, cb, kinematics, dt):  # IntegrateKinematicPosesAndVelocities: pose, then (optionally) velocity
    dt = f32(dt)
    for index in kinematics:
        s = _gather(bodies, index, world=False)
        s.pos = s.pos + s.lin * dt
        s.q = integrate_orientation(s.q, s.ang, dt * f32(0.5))
        bodies[s.index, 0:4], bodies[s.index, 4:7] = s.q, s.pos
        if cb.integrate_kinematics:
            s.lin, s.ang = cb.integrate_velocity(s.index, s.pos, dt, s.lin, s.ang)
            bodies[s.index, 8:11], bodies[s.index, 12:15] = s.lin, s.ang


# ---- PoseIntegrator.IntegrateAfterSubstepping (PoseIntegrator.cs:L537-726), bundle-wise ------------------------------------------------------------
def _after_substepping(bodies, cb, constrained, dt, substep_count, W, mutation):
    dt = f32(dt)
    substep_dt = dt / f32(substep_count)
    velocity_dt = substep_dt if cb.allow_substeps else dt  # L704-708
    cb.prepare(substep_dt if mutation == "final_prepare_substep_dt" else velocity_dt)
    n = bodies.shape[0]
    for start in range(0, n, W):
        count = min(W, n - start)
        unconstrained = [not constrained[start + i] for i in range(count)]
        any_unconstrained = any(unconstrained)
        lanes = []
        for i in range(count):
            s = _gather(bodies, start + i, world=False)
            if cb.allow_substeps:
                s.dt = substep_dt
            else:
                s.dt = dt if unconstrained[i] else substep_dt  # ConditionalSelect(unconstrainedMask, dt, substepDt)
            if mutation == "final_constrained_full_dt" and not unconstrained[i]:
                s.dt = dt
            integrate_velocity = unconstrained[i] and (cb.integrate_kinematics or not is_kinematic(s.inertia, mutation))  # L602-613
            lanes.append((s, integrate_velocity))
        any_velocity = any(v for _, v in lanes)
        if not any_unconstrained:  # L684-691: pose only, one step
            for s, _ in lanes:
                s.q = integrate_orientation(s.q, s.ang, s.dt * f32(0.5))
                s.pos = s.pos + s.lin * s.dt
                bodies[s.index, 0:4], bodies[s.index, 4:7] = s.q, s.pos
            continue
        steps = substep_count if cb.allow_substeps else 1
        for step in range(steps):  # L624-682: velocity, then pose
            for i, (s, integrate_velocity) in enumerate(lanes):
                if any_velocity and integrate_velocity and mutation != "callback_sees_stepped_position":
                    s.lin, s.ang = cb.integrate_velocity(s.index, s.pos, s.dt, s.lin, s.ang)
                if any_velocity and integrate_velocity and mutation == "callback_sees_stepped_position":
                    s.lin, s.ang = cb.integrate_velocity(s.index, s.pos + s.lin * s.dt, s.dt, s.lin, s.ang)
                s.pos = s.pos + s.lin * s.dt
                half_dt = s.dt * f32(0.5)
                if cb.angular_mode == 1:
                    previous_orientation = s.q
                    s.q = integrate_orientation(s.q, s.ang, half_dt)
                    world = rotate_inverse_inertia(s.inertia[0:6], s.q)
                    s.ang = conserve_momentum(previous_orientation, s.inertia[0:6], world, s.ang)
                elif cb.angular_mode == 2:
                    s.q = integrate_orientation(s.q, s.ang, half_dt)
                    s.ang = gyroscopic(s.q, s.inertia[0:6], s.ang, s.dt)
                else:
                    s.q = integrate_orientation(s.q, s.ang, half_dt)
                pose = True  # integratePoseMask: every existing lane on step 0, unconstrained lanes only after it (L660-667)
                if cb.allow_substeps and step > 0 and mutation != "final_constrained_pose_every_step":
                    pose = unconstrained[i]
                if pose:
                    bodies[s.index, 0:4], bodies[s.index, 4:7] = s.q, s.pos
                if any_velocity and integrate_velocity:  # ScatterVelocities through velocityMaskedBodyIndices
                    bodies[s.index, 8:11], bodies[s.index, 12:15] = s.lin, s.ang


# ---- Simulation.Solve: Solver.Solve single-threaded path (Solver_Solve.cs:L1415-1479), then IntegrateAfterSubstepping -------------------------------
def solve(sim, dt, accelerations=None, center=None, strength=0.0, mutation=None):
    """One frame of the reference's Solve on `sim`'s host buffers, in place (bodies, prestep, accumulated impulses)."""
    _check(mutation)
    assert library() is not None, "the transpiled reference is not built"
    W = sim.bundle_width
    bodies = sim.bodies
    tbs = sim.type_batches()
    batches = [[tb for tb in tbs if tb.batch_index == b] for b in range(sim.batch_count)]
    for batch in batches:
        assert [tb.type_batch_index for tb in batch] == list(range(len(batch)))
    kinematics = [int(k) for k in sim.constrained_kinematics]
    cb = Callbacks(sim.integrator, accelerations, center, strength)
    flags, constrained = integration_responsibilities(batches, sim.body_count, sim.fallback_batch_threshold, W, kinematics, mutation)
    substep_count = len(sim.velocity_iterations)
    substep_dt = f32(dt) / f32(substep_count)
    cb.prepare(substep_dt)  # L1417-1418
    for substep in range(substep_count):
        if substep > 0:
            if mutation == "incremental_after_kinematic_pose":
                _kinematic_poses_and_velocities(bodies, cb, kinematics, substep_dt)
            for batch in batches:  # L1427-1438: IncrementallyUpdateForSubstep of the types that require it
                for tb in batch:
                    if tb.type_id in CONTACT_TYPES:
                        for k in range(tb.bundle_count):
                            _solve_bundle(bodies, tb, k, substep_dt, W, stage=2)
            if mutation != "incremental_after_kinematic_pose":
                _kinematic_poses_and_velocities(bodies, cb, kinematics, substep_dt)  # L1439
        elif cb.integrate_kinematics or mutation == "kinematic_velocity_prepass_ignores_flag":
            _kinematic_velocities(bodies, cb, kinematics, substep_dt)  # L1441-1444
        allow_pose = substep > 0 or mutation == "pose_in_substep_zero"
        for b, batch in enumerate(batches):  # L1446-1460
            for t, tb in enumerate(batch):
                for k in range(tb.bundle_count):
                    _warm_start_bundle(bodies, cb, tb, k, b, flags[b][t], allow_pose, substep_dt, W)
        for _ in range(sim.velocity_iterations[substep]):  # L1461-1473
            for batch in batches:
                for tb in batch:
                    for k in range(tb.bundle_count):
                        _solve_bundle(bodies, tb, k, substep_dt, W, stage=1)
    _after_substepping(bodies, cb, constrained, dt, substep_count, W, mutation)  # Simulation.cs:L278-290


# ---- PoseIntegrator.PredictBoundingBoxes (PoseIntegrator.cs:L307-370, L424-444) ---------------------------------------------------------------------
def update_sleep_candidacy(energy, activity):
    """UpdateSleepCandidacy (PoseIntegrator.cs:L286-304) on one BODY_ACTIVITY_DTYPE record."""
    if energy > activity["sleep_threshold"]:
        activity["timesteps_under_threshold_count"] = 0
        activity["sleep_candidate"] = 0
    elif activity["timesteps_under_threshold_count"] < 255:
        activity["timesteps_under_threshold_count"] += 1
        if activity["timesteps_under_threshold_count"] >= activity["minimum_timesteps_under_threshold"]:
            activity["sleep_candidate"] = 1


def predict_bounding_boxes(bodies, shapes, activities, dt, integrator, accelerations=None, center=None, strength=0.0, bundle_width=8, mutation=None):
    """Bounds of every body: bounds[n, 8] = {min.xyz, speculative margin, max.xyz, valid}, activities updated in place. Body bundles are
    `bundle_width` (Vector<float>.Count) lanes wide. Shapes without a convex GetBounds here (valid = 0) get no bounds, their activity still counts."""
    _check(mutation)
    lib = library()
    assert lib is not None, "the transpiled reference is not built"
    bodies = np.ascontiguousarray(bodies, dtype=f32).reshape(-1, 32)
    n = bodies.shape[0]
    dt = f32(dt)
    cb = Callbacks(integrator, accelerations, center, strength)
    cb.prepare(dt)  # L427
    out = np.zeros((n, 8), dtype=f32)
    for start in range(0, n, bundle_width):
        count = min(bundle_width, n - start)
        lanes = [_gather(bodies, start + i, world=False) for i in range(count)]
        if cb.integrate_kinematics:  # L322-329
            mask = [True] * count
        else:
            mask = [not is_kinematic(s.inertia, mutation) for s in lanes]
        energies = [_length_squared(s.lin) + _length_squared(s.ang) for s in lanes]  # L332
        if any(mask):  # L334-335: the callback runs on the whole bundle and its result is kept in every lane; masked lanes carry index -1
            for s, m in zip(lanes, mask):
                s.lin, s.ang = cb.integrate_velocity(s.index if m else -1, s.pos, dt, s.lin, s.ang)
        for i, s in enumerate(lanes):
            body = start + i
            energy = _length_squared(s.lin) + _length_squared(s.ang) if mutation == "sleep_reads_integrated_velocity" else energies[i]
            update_sleep_candidacy(energy, activities[body])
            shape = shapes[body]
            if int(shape["type"]) not in (0, 1, 2, 4):
                continue
            # BoundingBoxBatcher.ExecuteConvexBatch (BoundingBoxBatcher.cs:L176-197) with the shape's GetBounds, transpiled
            dims = np.array([shape["a"], shape["b"], shape["c"]], dtype=f32)
            margins = np.array([shape["minimum_speculative_margin"], shape["maximum_speculative_margin"]], dtype=f32)
            r = np.zeros(7, dtype=f32)
            assert lib.ref_convex_bounds(int(shape["type"]), _ptr(dims), _ptr(margins), int(shape["allow_expansion_beyond_speculative_margin"]), _ptr(s.q), _ptr(s.pos),
                                         _ptr(np.ascontiguousarray(s.lin)), _ptr(np.ascontiguousarray(s.ang)), dt, _ptr(r)) == 0
            out[body, 0:7], out[body, 7] = r, f32(1)
    return out


# ---- NarrowPhase.UpdateConstraint, same-type branch (NarrowPhaseConstraintUpdate.cs:L81-196) ------------------------------------------------------
def redistribute_impulses(old_feature_ids, old_impulses, new_feature_ids, mutation=None):
    """RedistributeImpulses (L81-135): returns the new impulses; old_impulses is consumed (matched entries zeroed) like the reference's buffer."""
    _check(mutation)
    old = np.array(old_impulses, dtype=f32)
    new = np.full(len(new_feature_ids), f32(-1), dtype=f32)  # a negative impulse flags 'unmatched'
    unmatched = 0
    for i, feature in enumerate(new_feature_ids):
        for j, old_feature in enumerate(old_feature_ids):
            if old_feature == feature:
                new[i] = old[j]
                old[j] = f32(0)
                break
        if new[i] < 0:
            unmatched += 1
    if unmatched > 0:
        total = f32(0)
        for value in old:
            total = total + value
        per = total / f32(unmatched)
        for i in range(len(new)):
            if new[i] < 0:
                new[i] = f32(0) if mutation == "unmatched_zero_impulse" else per
    return new


def penetration_rows(type_id):
    """The accumulated-impulse rows GatherOldImpulses / ScatterNewImpulses address (ContactConstraintAccessor.cs:L36-78): after the Vector2Wide tangent
    friction of a convex manifold, and NonconvexAccumulatedImpulses.Penetration ({Tangent.X, Tangent.Y, Penetration} per contact) otherwise."""
    if 0 <= type_id <= 7:
        return [2 + i for i in range((type_id & 3) + 1)]
    count = type_id - 6 if 8 <= type_id <= 10 else type_id - 13
    assert 15 <= type_id <= 17 or 8 <= type_id <= 10
    return [3 * i + 2 for i in range(count)]


def update_contact_impulses(tb, old_feature_ids, new_feature_ids, mutation=None):
    """UpdateConstraint for every constraint of a contact type batch whose new manifold has the same type: gather, redistribute, scatter in place."""
    rows = penetration_rows(tb.type_id)
    W = tb.accumulated_impulses.shape[2]
    for c in range(tb.constraint_count):
        bundle, lane = c // W, c % W
        old = [tb.accumulated_impulses[bundle, r, lane] for r in rows]
        new = redistribute_impulses(list(old_feature_ids[c]), old, list(new_feature_ids[c]), mutation)
        for r, value in zip(rows, new):
            tb.accumulated_impulses[bundle, r, lane] = value
