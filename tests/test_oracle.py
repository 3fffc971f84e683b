"""CPU tests that pin the oracle itself. The reference ships no golden numeric vectors for the solver path (SURVEY.md §8c); the arithmetic is pinned to the C# text by
tests/test_oracle_pinned_to_reference.py, and for the DRIVER (unpinned) the
oracle is anchored on analytic known answers and internal consistency: scalar vs 8-wide evaluation, thread-count invariance, bundle-width invariance,
momentum conservation, steady-state stack impulses, and joint error decay."""
import numpy as np
import pytest

import bepuphysics2_b200 as bp
from bepuphysics2_b200 import scenes
from tests import planner, util

DT = 1.0 / 60.0


def test_stacked_boxes_carry_the_weight_above_them(libs):
    """Steady state: the penetration impulses of the manifold under k boxes sum to (k) * m * g * dt (SURVEY.md §8c known answer)."""
    sim = util.make_sim(scenes.box_stacks(2, 8), substeps=1, velocity_iterations=8)
    for _ in range(200):
        util.ob.solve(sim, DT)
    g_dt = 10.0 * DT
    for tb in sim.type_batches():
        W = sim.bundle_width
        for c in range(tb.constraint_count):
            a = int(tb.body_references[c // W, 0, c % W])
            level = (a - 1) % 8  # boxes are numbered bottom-up within a column
            carried = 8 - level
            pen = tb.accumulated_impulses[c // W, 2:6, c % W].sum()
            assert pen == pytest.approx(carried * g_dt, rel=2e-2)


def test_scalar_and_simd_evaluation_are_bit_identical(libs):
    scene = scenes.shape_pile(1500, seed=4, nonconvex_fraction=0.3)
    a = util.run_oracle(util.make_sim(scene, substeps=4, velocity_iterations=2), DT, frames=2, simd=False)
    b = util.run_oracle(util.make_sim(scene, substeps=4, velocity_iterations=2), DT, frames=2, simd=True)
    util.compare(a, b, exact=True)


def test_ragdolls_scalar_and_simd_are_bit_identical(libs):
    scene = scenes.ragdolls(30, seed=4)
    a = util.run_oracle(util.make_sim(scene, substeps=2, velocity_iterations=3), DT, frames=2, simd=False)
    b = util.run_oracle(util.make_sim(scene, substeps=2, velocity_iterations=3), DT, frames=2, simd=True)
    util.compare(a, b, exact=True)


@pytest.mark.parametrize("name,threads", [("pile", 4), ("pile", 3), ("fallback", 3), ("ragdolls", 5), ("mixed_with_terms", 4)])
def test_thread_count_does_not_change_results(libs, name, threads):
    """The worker loop (one share of every batch stage per worker, spin sync between stages, fallback batch on worker 0) against one thread.
    mixed_with_terms: contacts, ragdolls and a joint zoo with kinematic velocity integration, per-body accelerations and point gravity."""
    scene = {"pile": lambda: scenes.shape_pile(3000, seed=8), "fallback": lambda: scenes.fallback_stress(1500, hubs=2, seed=8), "ragdolls": lambda: scenes.ragdolls(40, seed=8),
             "mixed_with_terms": lambda: scenes.merge(scenes.box_stacks(4, 6), scenes.ragdolls(6, seed=3), scenes.joint_zoo(400, 20, seed=4))}[name]()
    integ, terms = None, {}
    if name == "mixed_with_terms":
        integ = bp.IntegratorDesc.default()
        integ.integrate_velocity_for_kinematics = 1
        accelerations = np.random.default_rng(5).uniform(-5, 5, size=(scene["bodies"].shape[0], 8)).astype(np.float32)
        accelerations[:, 3] = accelerations[:, 7] = 0.0
        terms = {"accelerations": accelerations, "center": (0, -30, 0), "strength": 500.0}
    a = util.run_oracle(util.make_sim(scene, substeps=3, velocity_iterations=2, integrator=integ), DT, frames=2, threads=1, simd=True, **terms)
    b = util.run_oracle(util.make_sim(scene, substeps=3, velocity_iterations=2, integrator=integ), DT, frames=2, threads=threads, simd=True, **terms)
    util.compare(a, b, exact=True)


def test_bundle_width_does_not_change_results(libs):
    """Synchronized batches commute, so the host's Vector<float>.Count must not matter (nonconserving angular mode)."""
    scene = scenes.shape_pile(800, seed=3)
    snaps = [util.run_oracle(util.make_sim(scene, bundle_width=w, substeps=2, velocity_iterations=2), DT) for w in (4, 8, 16)]
    for s in snaps[1:]:
        assert np.array_equal(snaps[0]["bodies"][:, util.MEANINGFUL], s["bodies"][:, util.MEANINGFUL])


def test_two_body_contacts_conserve_linear_momentum(libs):
    """With gravity and damping off, two-body constraints exchange momentum only: sum(m v) is conserved to rounding."""
    scene = scenes.shape_pile(600, seed=6, one_body_fraction=0.0)
    integ = bp.IntegratorDesc.default()
    integ.gravity[1] = 0.0
    integ.linear_damping = 0.0
    integ.angular_damping = 0.0
    sim = util.make_sim(scene, substeps=2, velocity_iterations=3, integrator=integ)
    m = 1.0 / sim.bodies[:, 22]
    before = (sim.bodies[:, 8:11] * m[:, None]).sum(axis=0)
    util.ob.solve(sim, DT)
    after = (sim.bodies[:, 8:11] * m[:, None]).sum(axis=0)
    np.testing.assert_allclose(after, before, atol=2e-3)


def test_zero_impulse_warm_start_is_identity_and_unconstrained_bodies_fall(libs):
    """A body with no constraints integrates v = (v + g dt) * damping^dt, p += v dt (IntegrateAfterSubstepping, unconstrained path)."""
    scene = {"bodies": scenes.make_bodies(np.array([[0, 10, 0]], dtype=np.float32), inverse_mass=np.array([1], dtype=np.float32), inverse_inertia=np.array([[1, 0, 1, 0, 0, 1]], dtype=np.float32)),
             "constraints": [], "description": "one free body"}
    sim = util.make_sim(scene, substeps=4, velocity_iterations=1)
    util.ob.solve(sim, DT)
    damp = np.float32(0.97) ** np.float32(DT)
    v = np.float32(-10.0 * DT) * damp
    assert sim.bodies[0, 9] == pytest.approx(v, rel=1e-6)
    assert sim.bodies[0, 5] == pytest.approx(10.0 + v * DT, rel=1e-6)


def test_ball_socket_pulls_anchors_together(libs):
    """Two bodies joined by a BallSocket with separated anchors: the anchor error shrinks every frame (error * ERP bias, BallSocket.cs:L66-86)."""
    bodies = scenes.make_bodies(np.array([[0, 0, 0], [1.5, 0, 0]], dtype=np.float32), inverse_mass=np.array([1, 1], dtype=np.float32),
                                inverse_inertia=np.array([[1, 0, 1, 0, 0, 1]] * 2, dtype=np.float32))
    pre = np.r_[[0.5, 0, 0], [-0.5, 0, 0], scenes.spring(30, 1)].astype(np.float32)[None, :]
    scene = {"bodies": bodies, "constraints": [(22, np.array([[0, 1]], dtype=np.int32), pre)], "description": "ball socket"}
    integ = bp.IntegratorDesc.default()
    integ.gravity[1] = 0.0
    sim = util.make_sim(scene, substeps=1, velocity_iterations=4, integrator=integ)
    errors = []
    for _ in range(30):
        util.ob.solve(sim, DT)
        b = sim.bodies
        errors.append(abs((b[1, 4] - 0.5) - (b[0, 4] + 0.5)))
    assert errors[-1] < 0.02 * 0.5
    assert errors[10] < errors[0]


def test_sin_cos_approximations_through_orientation_integration(libs):
    """A free body spinning at w about z for one second returns a rotation of |w| radians: pins MathHelper.Sin/Cos restatements (error < 1e-5)."""
    w = 2.0
    scene = {"bodies": scenes.make_bodies(np.zeros((1, 3), dtype=np.float32), angular=np.array([[0, 0, w]], dtype=np.float32), inverse_mass=np.array([1], dtype=np.float32),
                                          inverse_inertia=np.array([[1, 0, 1, 0, 0, 1]], dtype=np.float32)), "constraints": [], "description": "spinner"}
    integ = bp.IntegratorDesc.default()
    integ.gravity[1] = 0.0
    integ.angular_damping = 0.0
    sim = util.make_sim(scene, integrator=integ)
    for _ in range(60):
        util.ob.solve(sim, DT)
    q = sim.bodies[0, 0:4]
    assert q[2] == pytest.approx(np.sin(w / 2), abs=2e-5)
    assert q[3] == pytest.approx(np.cos(w / 2), abs=2e-5)
    assert np.linalg.norm(q) == pytest.approx(1.0, abs=1e-6)


def test_fallback_batch_runs_sequentially(libs):
    """With a tiny fallback threshold most constraints land in the fallback batch; parallel oracle threads must not change the result."""
    scene = scenes.fallback_stress(300, hubs=2, seed=1)
    a = util.run_oracle(util.make_sim(scene, fallback_batch_threshold=4, substeps=2, velocity_iterations=2), DT, threads=1)
    b = util.run_oracle(util.make_sim(scene, fallback_batch_threshold=4, substeps=2, velocity_iterations=2), DT, threads=4)
    util.compare(a, b, exact=True)


def test_merged_scene_islands_evolve_independently(libs):
    """scenes.merge puts independent islands into one simulation; each island must evolve exactly as it does alone (batching interleaves them, the
    arithmetic per constraint and per body does not change)."""
    pile, dolls = scenes.shape_pile(400, seed=3), scenes.ragdolls(5, seed=4)
    alone_a = util.run_oracle(util.make_sim(pile, substeps=2, velocity_iterations=2), DT, frames=2)["bodies"]
    alone_b = util.run_oracle(util.make_sim(dolls, substeps=2, velocity_iterations=2), DT, frames=2)["bodies"]
    both = util.run_oracle(util.make_sim(scenes.merge(pile, dolls), substeps=2, velocity_iterations=2), DT, frames=2)["bodies"]
    n = alone_a.shape[0]
    assert np.array_equal(both[:n, util.MOTION], alone_a[:, util.MOTION])
    assert np.array_equal(both[n:, util.MOTION], alone_b[:, util.MOTION])


def test_oracle_output_is_stable_across_rounds(libs):
    """tests/golden/oracle_hashes.json (made by tests/golden/make_oracle_hashes.py) pins the checker to itself: every GPU parity test leans on the
    oracle, so a silent change to it must fail here first."""
    import json
    import os
    import sys

    here = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    sys.path.insert(0, here)
    import make_oracle_hashes as m

    with open(os.path.join(here, "oracle_hashes.json")) as f:
        want = json.load(f)
    assert sorted(want) == sorted(m.CASES)
    for name in m.CASES:
        assert m.digest(name) == want[name], "oracle output changed for %s" % name


def _inactive(scene):
    """The same constraint graph with every contact far out of reach (depth -100): the constraints apply nothing, but their batches still decide
    which lane integrates which body."""
    out = {"bodies": scene["bodies"].copy(), "constraints": [], "description": scene.get("description", "")}
    for type_id, handles, pre in scene["constraints"]:
        pre = pre.copy()
        rows = planner.depth_rows(type_id)
        assert rows  # contacts only: a joint would still apply impulses
        pre[:, rows] = -100.0
        out["constraints"].append((type_id, handles, pre))
    return out


@pytest.mark.parametrize("name,substeps", [("pile", 1), ("pile", 5), ("fallback", 3)])
def test_every_body_is_integrated_exactly_once_per_substep(libs, name, substeps):
    """The invariant of the reference's commented-out validators (Solver_Solve.cs:L1298-1361): across the batches' integration responsibilities,
    the kinematic prepass and IntegrateAfterSubstepping, every dynamic body gets exactly one velocity integration and one pose integration per
    substep — whatever batch it was first seen in, fallback batch included. With constraints that apply nothing, every constrained body must
    then match the closed-form trajectory (float64); a body integrated twice or never is off by g * dt_substep."""
    if name == "pile":
        scene = _inactive(scenes.shape_pile(3000, seed=11))
    else:
        scene = _inactive(scenes.fallback_stress(1500, hubs=2, seed=11))
    rng = np.random.default_rng(3)
    n = scene["bodies"].shape[0]
    dynamic = scene["bodies"][:, 22] > 0
    scene["bodies"][:, 8:11] = np.where(dynamic[:, None], rng.normal(0, 1, (n, 3)), 0).astype(np.float32)
    before = scene["bodies"].astype(np.float64)
    sim = util.make_sim(scene, substeps=substeps, velocity_iterations=2)
    assert max(tb.batch_index for tb in sim.type_batches()) >= (64 if name == "fallback" else 4)  # 64 = the sequential fallback batch
    constrained = np.zeros(n, dtype=bool)
    for tb in sim.type_batches():
        refs = tb.body_references
        constrained[(refs[refs >= 0] & 0x3FFFFFFF)] = True
    util.ob.solve(sim, DT)
    h = DT / substeps
    damp = 0.97 ** h
    v = before[:, 8:11].copy()
    p = before[:, 4:7].copy()
    for _ in range(substeps):
        v = (v + np.array([0, -10.0 * h, 0])) * damp
        p = p + v * h
    sel = constrained & dynamic
    assert sel.sum() > 0.9 * dynamic.sum()
    after = sim.bodies.astype(np.float64)
    # (a wrong integration count is off by |g| * h = 0.03 .. 0.17 in velocity)
    assert np.abs(after[sel, 8:11] - v[sel]).max() < 2e-5
    assert np.abs(after[sel, 4:7] - p[sel]).max() < 2e-5 * max(1.0, np.abs(p).max())
    # unconstrained dynamic bodies take one full-length step (AllowSubstepsForUnconstrainedBodies = false, PoseIntegrator.cs:L537-693)
    free = dynamic & ~constrained
    if free.any():
        vf = (before[free, 8:11] + np.array([0, -10.0 * DT, 0])) * 0.97 ** DT
        assert np.abs(after[free, 8:11] - vf).max() < 2e-5
        assert np.abs(after[free, 4:7] - (before[free, 4:7] + vf * DT)).max() < 2e-5 * max(1.0, np.abs(p).max())
