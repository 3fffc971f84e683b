"""GPU parity tests: libbepucuda (through the C ABI, via the host mirror's CudaTimestepper) against the CPU oracle on identical seeded
scenes. Strict build (-fmad=false): bit-exact on body poses/velocities/world inertias, accumulated impulses and contact depths.
Fast build (FMA contraction on): fp32 tolerance stated per test."""
import numpy as np
import pytest

from bepuphysics2_b200 import scenes
from bepuphysics2_b200.native import EXEC_GRAPH, EXEC_STREAM
from tests import util

pytestmark = pytest.mark.gpu
DT = 1.0 / 60.0


def _parity(scene, exact=True, mode=EXEC_GRAPH, frames=1, rel_rms=1e-3, max_abs=5e-2, **kw):
    a = util.make_sim(scene, **kw)
    b = util.make_sim(scene, **kw)
    ref = util.run_oracle(a, DT, frames=frames)
    got = util.run_gpu(b, DT, frames=frames, strict=exact, mode=mode)
    util.compare(ref, got, exact=exact, rel_rms=rel_rms, max_abs=max_abs)
    return got


def test_box_stack_config1_bit_exact(libs):
    """BASELINE config 1: 256-body box stack, Contact4 only, 1 velocity iteration."""
    got = _parity(scenes.box_stacks(16, 16), substeps=1, velocity_iterations=1)
    assert got["timings"]["constraint_count"] == 256
    assert got["timings"]["device_batch_count"] == 2


@pytest.mark.parametrize("mode", [EXEC_GRAPH, EXEC_STREAM])
def test_box_stack_substepped_all_execution_modes(libs, mode):
    _parity(scenes.box_stacks(8, 12), mode=mode, substeps=4, velocity_iterations=2, frames=3)


def test_shape_pile_all_convex_types_bit_exact(libs):
    """Types 0-7 (1-4 contacts, one and two body), 8 substeps x 2 iterations like BASELINE config 2, several frames."""
    got = _parity(scenes.shape_pile(3000, seed=5), substeps=8, velocity_iterations=2, frames=2)
    assert got["timings"]["constraint_iterations"] == got["timings"]["constraint_count"] * 16


def test_shape_pile_nonconvex_types_bit_exact(libs):
    _parity(scenes.shape_pile(2000, seed=7, nonconvex_fraction=0.5), substeps=3, velocity_iterations=[1, 2, 3])


def test_shape_pile_stream_mode_bit_exact(libs):
    _parity(scenes.shape_pile(5000, seed=11), mode=EXEC_STREAM, substeps=4, velocity_iterations=2, frames=2)


def test_bundle_width_4_and_16_sources(libs):
    """The host's Vector<float>.Count only changes the source layout; results are identical."""
    for w in (4, 16):
        _parity(scenes.shape_pile(800, seed=3), bundle_width=w, substeps=2, velocity_iterations=2)


def test_sequential_fallback_batch_bit_exact(libs):
    """Hub bodies exceed the fallback threshold: the fallback batch is levelised on the device, results match the sequential CPU loop."""
    scene = scenes.fallback_stress(600, hubs=3, seed=5)
    got = _parity(scene, fallback_batch_threshold=8, substeps=2, velocity_iterations=2, frames=2)
    assert got["timings"]["fallback_level_count"] > 8


def test_fast_build_within_tolerance(libs):
    """FMA-contracted + approximate sqrt build on contacts: relative RMS error <= 1e-5 and max abs error <= 1e-4 on velocities, poses and
    accumulated impulses after one frame of 8 substeps x 2 iterations."""
    _parity(scenes.shape_pile(3000, seed=5), exact=False, rel_rms=1e-5, max_abs=1e-4, substeps=8, velocity_iterations=2)


def test_unconstrained_and_kinematic_bodies(libs):
    """Bodies with no constraints take the IntegrateAfterSubstepping path; kinematics referenced by constraints take the prepass."""
    scene = scenes.box_stacks(4, 4)
    extra = scenes.make_bodies(np.array([[100, 5, 0], [120, 5, 0]], dtype=np.float32), linear=np.array([[1, 2, 3], [0, 0, 0]], dtype=np.float32),
                               angular=np.array([[0.5, 0.1, -0.3], [0, 1, 0]], dtype=np.float32), inverse_mass=np.array([1, 0], dtype=np.float32),
                               inverse_inertia=np.array([[2, 0, 2, 0, 0, 2], [0, 0, 0, 0, 0, 0]], dtype=np.float32))
    scene["bodies"] = np.concatenate([scene["bodies"], extra])
    scene["bodies"][0, 8:11] = (0.2, 0.0, 0.1)  # moving kinematic ground
    scene["bodies"][0, 12:15] = (0.0, 0.3, 0.0)
    for allow in (0, 1):
        integ = util.bp.IntegratorDesc.default()
        integ.allow_substeps_for_unconstrained = allow
        _parity(scene, substeps=3, velocity_iterations=1, integrator=integ, frames=2)


@pytest.mark.parametrize("angular_mode", [1, 2])
def test_momentum_conserving_angular_modes(libs, angular_mode):
    integ = util.bp.IntegratorDesc.default()
    integ.angular_integration_mode = angular_mode
    _parity(scenes.shape_pile(500, seed=9), substeps=3, velocity_iterations=1, integrator=integ)


def test_ragdolls_all_joint_types_bit_exact(libs):
    """BASELINE config 3 topology: BallSocket, SwingLimit, TwistLimit, TwistServo, SwivelHinge, Hinge, AngularMotor + contacts vs a kinematic tube."""
    got = _parity(scenes.ragdolls(60, seed=5), substeps=1, velocity_iterations=4, frames=3)
    assert got["timings"]["constraint_count"] > 60 * 58


def test_device_resident_frames_without_reupload(libs):
    """Several solves without re-uploading anything (the bench's device-resident loop): the captured graph is replayed on the state the previous
    solve left on the device."""
    import bepuphysics2_b200 as bp

    scene = scenes.shape_pile(2000, seed=13)
    a = util.make_sim(scene, substeps=2, velocity_iterations=2)
    b = util.make_sim(scene, substeps=2, velocity_iterations=2)
    ref = util.run_oracle(a, DT, frames=4)
    ts = bp.CudaTimestepper(b, strict_fp=True, execution_mode=EXEC_GRAPH)
    ts.describe()
    for _ in range(3):
        ts.solve_device_only(DT)
    ts.solve(DT, download=True)
    ts.download_prestep()
    ts.close()
    util.compare(ref, util.snapshot(b), exact=True)


def test_ragdolls_substepped_servo_variant_bit_exact(libs):
    """AngularServo variant (RagdollDemo.cs:L199) with 8 substeps x 2 iterations."""
    _parity(scenes.ragdolls(40, seed=6, motor="servo"), substeps=8, velocity_iterations=2, frames=2)


def test_ragdolls_stream_mode_fast_within_tolerance(libs):
    """Fast build on joints: relative RMS error <= 1e-3, max abs error <= 2e-2 after one frame (the twist/servo angle
    measurements go through acos near 1, which amplifies rounding: see tests/tools/fast_error_stats.py)."""
    _parity(scenes.ragdolls(60, seed=5), exact=False, mode=EXEC_STREAM, rel_rms=1e-3, max_abs=2e-2, substeps=1, velocity_iterations=4)


def test_registered_host_buffers_refresh_flow_bit_exact(libs):
    """The per-frame flow of a host application: page-locked (registered) buffers, refresh (bodies + prestep + impulses re-uploaded through the batched
    zero-copy kernel), solve, download into the same buffers. Several frames, strict build, against the oracle."""
    import bepuphysics2_b200 as bp

    scene = scenes.shape_pile(4000, seed=21)
    a = util.make_sim(scene, substeps=3, velocity_iterations=2)
    b = util.make_sim(scene, substeps=3, velocity_iterations=2)
    ref = util.run_oracle(a, DT, frames=3)
    ts = bp.CudaTimestepper(b, strict_fp=True)
    ts.register_host_buffers()
    ts.describe()
    for f in range(3):
        if f > 0:
            ts.refresh()
        ts.solve(DT, download=True)
        ts.download_prestep()
    t = ts.timings()
    ts.close()
    assert t.h2d_bytes > 0 and t.d2h_bytes > 0
    util.compare(ref, util.snapshot(b), exact=True)


@pytest.mark.parametrize("type_id", sorted(scenes.JOINT_ZOO_TYPES))
def test_each_remaining_joint_type_bit_exact(libs, type_id):
    """One scene per constraint type of DefaultTypes.cs beyond the ragdoll set (1, 2, 3 and 4 body types), substepped, several frames so that
    warm starting sees non-zero accumulated impulses."""
    got = _parity(scenes.joint_zoo(300, 150, seed=20 + type_id, types=[type_id]), substeps=3, velocity_iterations=2, frames=3)
    assert got["timings"]["constraint_count"] == 150


@pytest.mark.parametrize("mode", [EXEC_GRAPH, EXEC_STREAM])
def test_joint_zoo_all_types_together_all_execution_modes(libs, mode):
    """All 22 remaining types in one scene (many batches, kinematic partners, 3- and 4-body constraints) in every execution mode."""
    _parity(scenes.joint_zoo(1500, 120, seed=6), mode=mode, substeps=2, velocity_iterations=2, frames=2)


def test_joint_zoo_with_fallback_batch_and_momentum_conserving_integration(libs):
    """Low fallback threshold pushes multi-body joints into the sequential fallback batch; ConserveMomentum exercises the bundle-wide
    first-substep quirk with 1-, 3- and 4-body bundles."""
    integ = util.bp.IntegratorDesc.default()
    integ.angular_integration_mode = 1
    got = _parity(scenes.joint_zoo(250, 60, seed=9), fallback_batch_threshold=4, substeps=2, velocity_iterations=2, frames=2, integrator=integ)
    assert got["timings"]["fallback_level_count"] > 0


def test_profile_stages_advances_like_solve(libs):
    """bepucuda_profile_stages runs one frame with an event pair around every launch and must advance the simulation exactly like bepucuda_solve:
    bodies, impulses and contact depths bit for bit against the oracle, and as many launches as a graph solve of the same description. The scene
    runs every stage kind: contacts (incremental update), joints in the sequential fallback batch, constrained kinematics with
    IntegrateVelocityForKinematics (both kinematic prepasses), several substeps."""
    import bepuphysics2_b200 as bp

    integ = util.bp.IntegratorDesc.default()
    integ.integrate_velocity_for_kinematics = 1
    scene = scenes.merge(scenes.joint_zoo(250, 60, seed=9), scenes.shape_pile(300, seed=2))
    kw = dict(fallback_batch_threshold=4, substeps=3, velocity_iterations=2, integrator=integ)
    ref = util.run_oracle(util.make_sim(scene, **kw), DT)
    sim = util.make_sim(scene, **kw)
    ts = bp.CudaTimestepper(sim, strict_fp=True)
    try:
        ts.describe()
        profile = ts.profile_stages(DT)
        ts.download_bodies()
        ts.download_impulses()
        ts.download_prestep()
    finally:
        ts.close()
    util.compare(ref, util.snapshot(sim), exact=True)
    assert all(profile.launches[stage] > 0 for stage in range(7))
    graph = util.run_gpu(util.make_sim(scene, **kw), DT, strict=True, mode=EXEC_GRAPH)
    assert graph["timings"]["fallback_level_count"] > 0
    assert sum(profile.launches) == graph["timings"]["kernel_launches"]


def test_joint_zoo_fast_build_within_tolerance(libs):
    """Fast (FMA, approximate sqrt) build on the full zoo after one frame: relative RMS error <= 1e-3, max abs error <= 5e-2."""
    _parity(scenes.joint_zoo(1500, 120, seed=6), exact=False, rel_rms=1e-3, max_abs=5e-2, substeps=2, velocity_iterations=2)


@pytest.mark.parametrize("mode", [EXEC_GRAPH, EXEC_STREAM])
def test_edge_cases_no_constraints_single_body_and_per_substep_iteration_schedule(libs, mode):
    """Degenerate inputs through the whole C-ABI sequence: bodies without any constraint (only IntegrateAfterSubstepping runs), a single constrained
    body, a one-constraint scene, and a per-substep velocity-iteration schedule that contains a zero."""
    free = {"bodies": scenes.make_bodies(np.array([[0, 5, 0], [3, 1, 2]], dtype=np.float32), linear=np.array([[1, 0, 0], [0, 2, 0]], dtype=np.float32),
                                         angular=np.array([[0.1, 0.2, 0.3], [0, 0, 1]], dtype=np.float32), inverse_mass=np.array([1, 0.5], dtype=np.float32),
                                         inverse_inertia=np.array([[1, 0, 1, 0, 0, 1], [2, 0, 3, 0, 0, 4]], dtype=np.float32)), "constraints": []}
    _parity(free, mode=mode, substeps=3, velocity_iterations=2, frames=2)
    one = scenes.joint_zoo(2, 1, seed=3, kinematic_fraction=0.0, types=[44])  # one one-body servo on one of two bodies
    _parity(one, mode=mode, substeps=2, velocity_iterations=1, frames=2)
    _parity(scenes.shape_pile(300, seed=2), mode=mode, substeps=3, velocity_iterations=[2, 0, 1], frames=2)


@pytest.mark.parametrize("seed", range(6))
def test_randomised_mixed_scenes_bit_exact(libs, seed):
    """Seeded random combinations: a pile (convex + nonconvex contacts), ragdolls, the joint zoo and free bodies merged into one simulation; random
    substep count, per-substep iteration schedule, host bundle width, fallback threshold, angular integration mode and execution mode."""
    rng = np.random.default_rng(1000 + seed)
    parts = [scenes.shape_pile(int(rng.integers(200, 900)), seed=int(rng.integers(1, 99)), nonconvex_fraction=float(rng.choice([0.0, 0.4]))),
             scenes.ragdolls(int(rng.integers(3, 12)), seed=int(rng.integers(1, 99)), motor=str(rng.choice(["motor", "servo"]))),
             scenes.joint_zoo(int(rng.integers(150, 400)), int(rng.integers(8, 30)), seed=int(rng.integers(1, 99))),
             {"bodies": scenes.make_bodies(rng.uniform(-5, 5, size=(5, 3)).astype(np.float32) + 200, linear=rng.uniform(-1, 1, size=(5, 3)).astype(np.float32),
                                           angular=rng.uniform(-1, 1, size=(5, 3)).astype(np.float32), inverse_mass=np.ones(5, dtype=np.float32),
                                           inverse_inertia=np.tile(np.array([[1, 0, 2, 0, 0, 3]], dtype=np.float32), (5, 1))), "constraints": []}]
    scene = scenes.merge(*parts)
    substeps = int(rng.integers(1, 5))
    iterations = [int(x) for x in rng.integers(1, 4, size=substeps)]
    integ = util.bp.IntegratorDesc.default()
    integ.angular_integration_mode = int(rng.integers(0, 3))
    integ.allow_substeps_for_unconstrained = int(rng.integers(0, 2))
    _parity(scene, mode=int(rng.choice([EXEC_GRAPH, EXEC_STREAM])), bundle_width=int(rng.choice([4, 8, 16])),
            fallback_batch_threshold=int(rng.choice([6, 64])), substeps=substeps, velocity_iterations=iterations, integrator=integ, frames=2)


@pytest.mark.parametrize("mode", [EXEC_GRAPH, EXEC_STREAM])
def test_fast_build_is_run_to_run_deterministic(libs, mode):
    """The reference's own determinism harness (Demos/SpecializedTests/DeterminismTest.cs) repeats a simulation and demands bitwise identical
    results. The strict build is bit-identical to the oracle, hence deterministic; this holds the default FMA build to the same standard: no
    result may depend on which CTA of a stage runs first (scene large enough for every stage to span many CTAs, several frames)."""
    scene = scenes.merge(scenes.shape_pile(20000, seed=5, nonconvex_fraction=0.2), scenes.ragdolls(100, seed=5))
    runs = [util.run_gpu(util.make_sim(scene, substeps=4, velocity_iterations=2), DT, frames=3, strict=False, mode=mode) for _ in range(3)]
    for other in runs[1:]:
        util.compare(runs[0], other, exact=True)


@pytest.mark.parametrize("mode", [EXEC_GRAPH, EXEC_STREAM])
def test_kinematic_velocity_integration_all_execution_modes(libs, mode):
    """IntegrateVelocityForKinematics = true (PoseIntegrator.cs:L451-487 first substep, L493-535 later substeps): the callback's gravity and damping
    are applied to constrained kinematic bodies by the prepass, so a moving kinematic ground accelerates under the stacks resting on it, and an
    UNconstrained kinematic takes the velocity callback in IntegrateAfterSubstepping (L596-597 `integrateVelocity`)."""
    scene = scenes.box_stacks(5, 6)
    extra = scenes.make_bodies(np.array([[100, 5, 0], [120, 5, 0]], dtype=np.float32), linear=np.array([[1, 2, 3], [0.5, 0, -0.25]], dtype=np.float32),
                               angular=np.array([[0.5, 0.1, -0.3], [0, 1, 0]], dtype=np.float32), inverse_mass=np.array([1, 0], dtype=np.float32),
                               inverse_inertia=np.array([[2, 0, 2, 0, 0, 2], [0, 0, 0, 0, 0, 0]], dtype=np.float32))
    scene["bodies"] = np.concatenate([scene["bodies"], extra])
    scene["bodies"][0, 8:11] = (0.2, 0.05, 0.1)   # moving, spinning, constrained kinematic ground
    scene["bodies"][0, 12:15] = (0.0, 0.3, 0.05)
    for allow in (0, 1):
        integ = util.bp.IntegratorDesc.default()
        integ.integrate_velocity_for_kinematics = 1
        integ.allow_substeps_for_unconstrained = allow
        a = util.make_sim(scene, substeps=3, velocity_iterations=2, integrator=integ)
        assert len(a.constrained_kinematics) == 1
        before = a.bodies[0, 8:11].copy()
        got = _parity(scene, mode=mode, substeps=3, velocity_iterations=2, integrator=integ, frames=3)
        # the prepass really ran: gravity changed the kinematic's linear velocity (it would stay constant with the flag off)
        assert not np.array_equal(got["bodies"][0, 8:11], before)
        assert got["bodies"][0, 9] < before[1]


def test_kinematic_velocity_integration_with_joints_and_momentum_modes(libs):
    """The same flag on the joint zoo (5 % kinematic partners of 1-4 body joints) with the gyroscopic angular mode: the kinematic prepass
    never applies a momentum-conserving update (PoseIntegrator.cs:L451-535 integrate pose + callback only)."""
    integ = util.bp.IntegratorDesc.default()
    integ.integrate_velocity_for_kinematics = 1
    integ.angular_integration_mode = 2
    scene = scenes.joint_zoo(600, 40, seed=31, kinematic_fraction=0.15)
    kin = np.flatnonzero(scene["bodies"][:, 22] == 0)
    scene["bodies"][kin, 8:11] = np.random.default_rng(3).uniform(-0.5, 0.5, size=(kin.size, 3)).astype(np.float32)
    _parity(scene, substeps=3, velocity_iterations=2, integrator=integ, frames=2)


@pytest.mark.parametrize("mode", [EXEC_GRAPH, EXEC_STREAM])
def test_benchmark_scale_pile_bit_exact(libs, mode):
    """BASELINE config 2 at its own size (100 k bodies, ~333 k manifolds, 8 substeps x 2 iterations): the strict build against the oracle, bit for
    bit, several frames. Unlike the small scenes a stage here is hundreds of CTAs and several grids are in flight under programmatic dependent launch."""
    scene = scenes.shape_pile(100_000, seed=5)
    kw = dict(substeps=8, velocity_iterations=2)
    a = util.make_sim(scene, **kw)
    ref = util.run_oracle(a, DT, frames=2, threads=16, simd=True)
    for _ in range(2):  # a race would not show every time
        got = util.run_gpu(util.make_sim(scene, **kw), DT, frames=2, strict=True, mode=mode)
        util.compare(ref, got, exact=True)


def _fast_drift(scene, frames, **kw):
    """Runs `frames` frames (refresh between them, like a host application) through the oracle and through the default fast build and returns
    the per-quantity relative RMS / max abs differences of the final body state."""
    a, b = util.make_sim(scene, **kw), util.make_sim(scene, **kw)
    ref = util.run_oracle(a, DT, frames=frames, threads=16, simd=True)
    got = util.run_gpu(b, DT, frames=frames, strict=False)
    out = {}
    for label, cols in (("position", np.r_[4:7]), ("orientation", np.r_[0:4]), ("linear", np.r_[8:11]), ("angular", np.r_[12:15])):
        x, y = ref["bodies"][:, cols].astype(np.float64), got["bodies"][:, cols].astype(np.float64)
        assert np.isfinite(y).all(), label
        d = np.abs(x - y)
        out[label] = (float(np.sqrt((d ** 2).sum() / max((x ** 2).sum(), 1e-300))), float(d.max()))
    imp_num = imp_den = 0.0
    for ta, tb in zip(ref["type_batches"], got["type_batches"]):
        v = np.broadcast_to(ta["valid"][:, None, :], ta["impulses"].shape)
        x, y = np.where(v, ta["impulses"], 0).astype(np.float64), np.where(v, tb["impulses"], 0).astype(np.float64)
        assert np.isfinite(y).all()
        imp_num += ((x - y) ** 2).sum()
        imp_den += (x ** 2).sum()
    out["impulses"] = (float(np.sqrt(imp_num / max(imp_den, 1e-300))), 0.0)
    print("fast-build drift after %d frames:" % frames, {k: "%.2e / %.2e" % v for k, v in out.items()})
    return out


def test_fast_build_benchmark_scale_multi_frame_drift_bound(libs):
    """The BENCHMARKED build (FMA contraction, approximate sqrt) at the benchmark's own size, 8 frames of 8 x 2 with per-frame refresh. A
    contracting evaluation of a chaotic system separates from the non-contracting one; tests/tools/drift_curve.py measures the growth
    with a CPU proxy (frame 8, 3000-body pile: position 1.1e-8, linear 3.4e-7, angular 6.4e-7 relative RMS). Bound asserted here: 100x that."""
    d = _fast_drift(scenes.shape_pile(100_000, seed=5), 8, substeps=8, velocity_iterations=2)
    assert d["position"][0] <= 1e-6 and d["orientation"][0] <= 1e-5
    assert d["linear"][0] <= 5e-5 and d["angular"][0] <= 1e-4
    assert d["impulses"][0] <= 2e-2  # 2.4e-3 on an H100: many contact impulses sit at the clamp, where a last-bit difference switches them on or off


def test_fast_build_ragdoll_tube_multi_frame_drift_bound(libs):
    """Config-3-shaped scene (ragdolls: BallSocket / SwingLimit / TwistLimit / TwistServo / SwivelHinge / Hinge / AngularMotor + contacts), 1 x 4,
    8 frames. CPU-proxy growth at frame 8: position 2.4e-7, linear 2.4e-5, angular 2.5e-4 relative RMS; bound: 20x."""
    d = _fast_drift(scenes.ragdolls(2000, seed=5), 8, substeps=1, velocity_iterations=4)
    assert d["position"][0] <= 5e-6 and d["linear"][0] <= 5e-4 and d["angular"][0] <= 5e-3


def test_fast_build_fallback_stress_multi_frame_drift_bound(libs):
    """Config-5-shaped scene (hub bodies above the fallback threshold: levelised sequential fallback batch), 1 x 4, 8 frames."""
    d = _fast_drift(scenes.fallback_stress(5000, hubs=5, seed=5), 8, substeps=1, velocity_iterations=4)
    assert d["position"][0] <= 1e-5 and d["linear"][0] <= 1e-3 and d["angular"][0] <= 1e-2
