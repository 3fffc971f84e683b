"""Pins the oracle's DRIVER (oracle/bepu_oracle.cpp: which batch and lane integrates a body, the WarmStart masks, the kinematic prepasses, the final
pose pass, the callbacks, PredictBoundingBoxes' per-body glue, impulse redistribution) to a second, independent restatement of the reference's
single-threaded frame (tests/reference_frame.py), which runs on the transpiled reference's own arithmetic (oracle/_ref/libbepu_ref.so).

CPU, bit for bit: (a) ob.solve, scalar and 8-wide, on a scene matrix; (b) ob.predict_bounding_boxes; (c) ob.update_contact_impulses and the
redistribution itself; (d) every named misreading of the reference (reference_frame.MUTATIONS) changes the result of a named case. These need the
transpiled library, built by oracle/ref_transpile/build_ref.py where a checkout of the reference's C# sources is at hand; the restatement's answers
on the matrix are also committed as digests (tests/golden/reference_frame_digests.json, tests/golden/make_reference_frame_digests.py), so the
oracle is held to them everywhere.
GPU: the strict build, in both execution modes, equals the same digests on the whole matrix (full re-upload frames, and a resident sequence whose
impulse redistribution runs on the device); bepucuda_predict_bounding_boxes equals them on (b); the fast build stays within the tolerances the
existing fast tests apply to the same scene families.

One disagreement is known and left as it is: PredictBoundingBoxes (PoseIntegrator.cs:L322-335) hands the velocity callback whole body bundles and
keeps every lane's result, and DemoCallbacks ignores the integration mask, so in the reference a kinematic body sharing a bundle of
Vector<float>.Count bodies with a dynamic one gets its predicted velocity integrated. That depends on the host's SIMD width; the project follows
the callback's mask. The bounds cases keep kinematic bodies in bundles of their own, where both readings agree."""
import ctypes as C
import hashlib
import json
import os

import numpy as np
import pytest

import bepuphysics2_b200 as bp
from bepuphysics2_b200 import native, scenes
from oracle import binding as ob
from tests import reference_frame as rf
from tests import util

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DIGESTS = os.path.join(ROOT, "tests", "golden", "reference_frame_digests.json")
DT = 1.0 / 60.0
FRAMES = 2
needs_reference = pytest.mark.skipif(rf.library() is None, reason="the transpiled reference (oracle/_ref/libbepu_ref.so) is not built here")


def _loose_bodies(seed):
    """Unconstrained bodies: dynamic ones, +0 kinematic ones and one kinematic with -0.0 components, all moving."""
    rng = np.random.default_rng(seed)
    n = 7
    bodies = scenes.make_bodies(rng.uniform(-20, 20, size=(n, 3)).astype(np.float32), linear=rng.normal(size=(n, 3)).astype(np.float32),
                                angular=rng.normal(size=(n, 3)).astype(np.float32), inverse_mass=np.ones(n, dtype=np.float32),
                                inverse_inertia=np.tile(np.array([[1.5, 0.1, 2, 0, 0.2, 3]], dtype=np.float32), (n, 1)))
    bodies[[1, 4, 6], 16:23] = 0.0
    bodies[6, [16, 19, 22]] = -0.0
    return {"bodies": bodies, "constraints": []}


def _accelerations(n, seed):
    a = np.random.default_rng(seed).uniform(-5, 5, size=(n, 8)).astype(np.float32)
    a[:, 3] = a[:, 7] = 0.0
    return a


# name -> (what it is for, scene, Simulation keywords[, solve keywords]); every case runs FRAMES frames
def _cases():
    loose = _loose_bodies
    return {
        "contacts_w8": ("the 14 contact types (0-10, 15-17), incremental depth updates, partial last bundles, iteration schedule [1, 2]",
                        scenes.shape_pile(80, seed=1, one_body_fraction=0.25, nonconvex_fraction=0.4), dict(bundle_width=8, substeps=2, velocity_iterations=[1, 2]), {}),
        "contacts_w4_accelerations": ("contacts at width 4, one substep of three iterations, per-body accelerations",
                                      scenes.shape_pile(60, seed=6, one_body_fraction=0.3, nonconvex_fraction=0.5), dict(bundle_width=4, substeps=1, velocity_iterations=3),
                                      dict(accelerations=True)),
        "joints_w4_kinematics_integrated": ("the joint zoo at width 4 with constrained kinematics, integrate_velocity_for_kinematics = 1, angular mode 1, "
                                            "point gravity, schedule [2, 0, 1]",
                                            scenes.joint_zoo(150, 4, seed=2, kinematic_fraction=0.1),
                                            dict(bundle_width=4, substeps=3, velocity_iterations=[2, 0, 1], integrator=util.integrator(angular_integration_mode=1, integrate_velocity_for_kinematics=1)),
                                            dict(center=(0.0, -30.0, 0.0), strength=500.0)),
        "joints_w16_kinematics_not_integrated": ("the joint zoo at width 16, constrained kinematics with integrate_velocity_for_kinematics = 0, angular mode 2",
                                                 scenes.joint_zoo(150, 4, seed=3, kinematic_fraction=0.1),
                                                 dict(bundle_width=16, substeps=2, velocity_iterations=1, integrator=util.integrator(angular_integration_mode=2))),
        "ragdolls_four_substeps": ("ragdolls with motors and servos (types 22, 25-27, 29, 30, 46, 47) in a kinematic tube, loose bodies between them, "
                                   "4 substeps [1, 0, 2, 1], allow_substeps_for_unconstrained = 1, both velocity terms",
                                   scenes.merge(scenes.ragdolls(2, seed=4), loose(7), scenes.ragdolls(1, seed=5, motor="servo")),
                                   dict(bundle_width=8, substeps=4, velocity_iterations=[1, 0, 2, 1], integrator=util.integrator(allow_substeps_for_unconstrained=1, integrate_velocity_for_kinematics=1)),
                                   dict(accelerations=True, center=(0.0, -40.0, 0.0), strength=300.0)),
        "fallback_w8": ("a fallback batch (threshold 3) with holes, hubs in several of its type batches, bodies first seen in batches > 0",
                        scenes.fallback_stress(100, hubs=3, seed=5), dict(bundle_width=8, substeps=2, velocity_iterations=1, fallback_batch_threshold=3), {}),
        "fallback_w16_angular": ("a fallback batch at threshold 2 and width 16, angular mode 1, three substeps",
                                 scenes.fallback_stress(70, hubs=2, seed=8), dict(bundle_width=16, substeps=3, velocity_iterations=[1, 1, 0], fallback_batch_threshold=2,
                                                                                  integrator=util.integrator(angular_integration_mode=1))),
        "loose_bodies_allow0": ("unconstrained dynamic and kinematic bodies (one with -0.0 inertia) in body bundles with constrained ones, "
                                "allow_substeps_for_unconstrained = 0, angular mode 1, kinematics not integrated",
                                scenes.merge(scenes.joint_zoo(40, 1, seed=9, kinematic_fraction=0.1), loose(10), scenes.shape_pile(30, seed=9), loose(11)),
                                dict(bundle_width=8, substeps=3, velocity_iterations=[1, 2, 1], integrator=util.integrator(angular_integration_mode=1)), dict(center=(5.0, -20.0, 0.0), strength=200.0)),
        "loose_bodies_allow1": ("the same bodies with allow_substeps_for_unconstrained = 1, angular mode 2, kinematics integrated, per-body accelerations",
                                scenes.merge(scenes.joint_zoo(40, 1, seed=9, kinematic_fraction=0.1), loose(10), scenes.shape_pile(30, seed=9), loose(11)),
                                dict(bundle_width=4, substeps=3, velocity_iterations=[0, 2, 1], integrator=util.integrator(angular_integration_mode=2, allow_substeps_for_unconstrained=1, integrate_velocity_for_kinematics=1)),
                                dict(accelerations=True)),
    }


CASES = _cases()


def make_case(name):
    """(simulation, solve keywords) of a matrix case, freshly built."""
    _, scene, sim_kw, *solve_kw = CASES[name]
    sim = util.make_sim(scene, **sim_kw)
    kw = dict(solve_kw[0]) if solve_kw else {}
    if kw.get("accelerations"):
        kw["accelerations"] = _accelerations(sim.body_count, 3)
    else:
        kw.pop("accelerations", None)
    return sim, kw


def digest(snap):
    """SHA-256 over the bits of a util.snapshot: meaningful body floats, then per type batch the impulses and prestep of valid lanes."""
    h = hashlib.sha256()
    h.update(np.ascontiguousarray(snap["bodies"][:, util.MEANINGFUL]).view(np.uint32).tobytes())
    for tb in snap["type_batches"]:
        for what in ("impulses", "prestep"):
            valid = np.broadcast_to(tb["valid"][:, None, :], tb[what].shape)
            h.update(np.where(valid, tb[what], np.float32(0)).view(np.uint32).tobytes())
    return h.hexdigest()


def run_reference(name, mutation=None):
    sim, kw = make_case(name)
    for _ in range(FRAMES):
        rf.solve(sim, DT, mutation=mutation, **kw)
    return util.snapshot(sim)


def run_oracle(name, simd=False, frames=FRAMES):
    sim, kw = make_case(name)
    for _ in range(frames):
        ob.solve(sim, DT, simd=simd, **kw)
    return util.snapshot(sim)


# ---- (b) PredictBoundingBoxes cases -------------------------------------------------------------------------------------------------------------
def bounds_case(seed, kinematics, terms):
    """Bodies in 12 bundles of 8 (the reference's Vector<float>.Count on AVX2); bundles 2, 5 and 9 are kinematic, with +0 and with -0.0 components;
    every shape type id (3, 5, 6, 7 and -1 have no convex bounds here: valid = 0); sleep thresholds around the bodies' energies, counts at 254
    and 255, MinimumTimestepsUnderThreshold 0."""
    rng = np.random.default_rng(seed)
    n = 96
    q = rng.normal(size=(n, 4))
    q = (q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32)
    lin = (rng.normal(size=(n, 3)) * rng.choice([0.0, 0.05, 2.0, 40.0], size=(n, 1))).astype(np.float32)
    ang = (rng.normal(size=(n, 3)) * rng.choice([0.0, 0.05, 3.0, 100.0], size=(n, 1))).astype(np.float32)
    bodies = scenes.make_bodies(rng.uniform(-30, 30, size=(n, 3)).astype(np.float32), orientation=q, linear=lin, angular=ang,
                                inverse_mass=rng.uniform(0.5, 2, size=n).astype(np.float32),
                                inverse_inertia=np.tile(np.array([[1, 0.1, 2, 0, 0.2, 3]], dtype=np.float32), (n, 1)))
    for b in (2, 5, 9):
        bodies[8 * b:8 * b + 8, 16:23] = 0.0
        bodies[8 * b + 1, 22] = -0.0  # inverse mass -0
        bodies[8 * b + 2, 16:23] = -0.0  # every component -0
        bodies[8 * b + 3, [17, 20]] = -0.0
    shapes = np.zeros(n, dtype=native.BODY_SHAPE_DTYPE)
    shapes["type"] = np.resize(np.array([0, 1, 2, 4, 0, 1, 2, 4, 3, 5, 6, 7, -1], dtype=np.int32), n)
    shapes["a"], shapes["b"], shapes["c"] = (rng.uniform(0.05, 2.0, size=n) for _ in range(3))
    shapes["minimum_speculative_margin"] = rng.choice([0.0, 0.01, 0.2], size=n)
    shapes["maximum_speculative_margin"] = rng.choice([0.05, 1.0, 3.40282347e+38], size=n)
    shapes["allow_expansion_beyond_speculative_margin"] = rng.integers(0, 2, size=n)
    activities = np.zeros(n, dtype=native.BODY_ACTIVITY_DTYPE)
    energy = (lin.astype(np.float64) ** 2).sum(1) + (ang.astype(np.float64) ** 2).sum(1)
    activities["sleep_threshold"] = (energy * rng.choice([0.5, 1.0, 2.0], size=n)).astype(np.float32)
    activities["minimum_timesteps_under_threshold"] = rng.choice([0, 1, 2, 3, 255], size=n)
    activities["timesteps_under_threshold_count"] = rng.choice([0, 1, 254, 255], size=n)
    activities["sleep_candidate"] = rng.integers(0, 2, size=n)
    kw = dict(accelerations=_accelerations(n, seed), center=(1.0, -25.0, 2.0), strength=400.0) if terms else {}
    return bodies, shapes, activities, util.integrator(integrate_velocity_for_kinematics=kinematics), kw


BOUNDS_CASES = {"kinematics0": (11, 0, False), "kinematics1": (12, 1, False), "kinematics0_terms": (13, 0, True), "kinematics1_terms": (14, 1, True)}
BOUNDS_FRAMES = 3


def bounds_reference(name, mutation=None):
    bodies, shapes, activities, integ, kw = bounds_case(*BOUNDS_CASES[name])
    out = [rf.predict_bounding_boxes(bodies, shapes, activities, DT, integ, mutation=mutation, **kw) for _ in range(BOUNDS_FRAMES)]
    return np.stack(out), activities


def bounds_oracle(name):
    bodies, shapes, activities, integ, kw = bounds_case(*BOUNDS_CASES[name])
    out = [ob.predict_bounding_boxes(bodies, shapes, activities, DT, integ, **kw) for _ in range(BOUNDS_FRAMES)]
    return np.stack(out), activities


def bounds_digest(bounds, activities):
    return hashlib.sha256(np.ascontiguousarray(bounds).view(np.uint32).tobytes() + activities.view(np.uint8).tobytes()).hexdigest()


# ---- (c) redistribution cases -------------------------------------------------------------------------------------------------------------------
def contact_batches():
    """A simulation holding every contact type id, impulses >= 0 on every row, and per type batch (old ids, new ids) with the four patterns by
    constraint index mod 4: all matched (permuted), none matched, duplicated old and new ids, and partly matched."""
    sim = util.make_sim(scenes.shape_pile(80, seed=1, one_body_fraction=0.25, nonconvex_fraction=0.4), bundle_width=8)
    rng = np.random.default_rng(21)
    ids = {}
    for tb in sim.type_batches():
        tb.accumulated_impulses[:] = rng.choice([0.0, 0.125, 0.5, 3.0, 7.25], size=tb.accumulated_impulses.shape).astype(np.float32)
        n = native.contact_count(tb.type_id)
        old = rng.integers(0, 50, size=(tb.constraint_count, n)).astype(np.int32)
        new = old.copy()
        for c in range(tb.constraint_count):
            pattern = c % 4
            if pattern == 0:
                new[c] = rng.permutation(old[c])
            elif pattern == 1:
                new[c] = 100 + np.arange(n)
            elif pattern == 2:
                old[c, :] = old[c, 0]
                new[c, :] = old[c, 0]
                if n > 1:
                    new[c, -1] = 99
            else:
                new[c, n // 2:] = 200 + np.arange(n - n // 2)
        ids[(tb.batch_index, tb.type_batch_index)] = (old, new)
    return sim, ids


# ---- (d) the case that catches each misreading --------------------------------------------------------------------------------------------------
CATCHES = {
    "pose_in_substep_zero": ("solve", "contacts_w8"),
    "every_batch_integrates": ("solve", "contacts_w8"),
    "fallback_last_slot": ("solve", "fallback_w8"),
    "kinematic_velocity_prepass_ignores_flag": ("solve", "joints_w16_kinematics_not_integrated"),
    "incremental_after_kinematic_pose": ("solve", "ragdolls_four_substeps"),
    "final_constrained_full_dt": ("solve", "contacts_w8"),
    "final_constrained_pose_every_step": ("solve", "loose_bodies_allow1"),
    "callback_sees_stepped_position": ("solve", "loose_bodies_allow0"),
    "final_prepare_substep_dt": ("solve", "loose_bodies_allow0"),
    "sleep_reads_integrated_velocity": ("bounds", "kinematics0"),
    "kinematic_test_bits": ("bounds", "kinematics0"),
    "unmatched_zero_impulse": ("redistribution", None),
}


def _digests():
    with open(DIGESTS) as f:
        return json.load(f)


# ---- CPU ------------------------------------------------------------------------------------------------------------------------------------------
def test_matrix_covers_what_it_claims(libs):
    types, widths, fallback = set(), set(), False
    for name in CASES:
        sim, _ = make_case(name)
        widths.add(sim.bundle_width)
        for tb in sim.type_batches():
            types.add(tb.type_id)
            fallback = fallback or (tb.batch_index == sim.fallback_batch_threshold and (tb.body_references[:, 0, :] == -1).any())
    assert sorted(types) == sorted(t for t in range(64) if ob.type_info(t) is not None) and len(types) == 44
    assert widths == {4, 8, 16} and fallback
    modes = {CASES[n][2].get("integrator", util.integrator()).angular_integration_mode for n in CASES}
    assert modes == {0, 1, 2}
    assert set(_digests()["solve"]) == set(CASES) and set(_digests()["bounds"]) == set(BOUNDS_CASES)


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_solve_equals_the_committed_reference_digests(libs, name):
    """Runs everywhere: the scalar and the 8-wide oracle (where the width is 8) against the restatement's stored answers."""
    want = _digests()["solve"][name]
    assert digest(run_oracle(name)) == want
    if CASES[name][2]["bundle_width"] == 8:
        assert digest(run_oracle(name, simd=True)) == want


@pytest.mark.parametrize("name", sorted(BOUNDS_CASES))
def test_oracle_bounds_equal_the_committed_reference_digests(libs, name):
    assert bounds_digest(*bounds_oracle(name)) == _digests()["bounds"][name]


@needs_reference
@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_solve_equals_the_restatement_bit_for_bit(libs, name):
    ref = run_reference(name)
    assert digest(ref) == _digests()["solve"][name], "the committed digest is not the restatement's answer"
    util.compare(ref, run_oracle(name), exact=True)
    if CASES[name][2]["bundle_width"] == 8:
        util.compare(ref, run_oracle(name, simd=True), exact=True)


@needs_reference
@pytest.mark.parametrize("name", sorted(BOUNDS_CASES))
def test_oracle_bounds_equal_the_restatement_bit_for_bit(libs, name):
    want, want_activities = bounds_reference(name)
    got, got_activities = bounds_oracle(name)
    assert bounds_digest(want, want_activities) == _digests()["bounds"][name]
    assert np.array_equal(want.view(np.uint32), got.view(np.uint32))
    assert np.array_equal(want_activities.view(np.uint8), got_activities.view(np.uint8))
    # the case reaches what it claims: bounds both valid and not, saturated counts, fresh sleep candidates
    assert set(np.unique(want[0, :, 7])) == {0.0, 1.0}
    assert (want_activities["timesteps_under_threshold_count"] == 255).any() and (want_activities["sleep_candidate"] == 1).any()


@needs_reference
def test_oracle_redistribution_equals_the_restatement(libs):
    want, ids = contact_batches()
    got, _ = contact_batches()
    for tw, tg in zip(want.type_batches(), got.type_batches()):
        old, new = ids[(tw.batch_index, tw.type_batch_index)]
        rf.update_contact_impulses(tw, old, new)
        ob.update_contact_impulses(tg, old, new)
        assert np.array_equal(tw.accumulated_impulses.view(np.uint32), tg.accumulated_impulses.view(np.uint32)), "type %d" % tw.type_id
    assert sorted({tb.type_id for tb in want.type_batches()}) == list(rf.CONTACT_TYPES)
    # old and new contact counts that differ (a manifold that changed its contact count changes type: UpdateConstraint's other branch)
    lib = ob.load()
    lib.oracle_redistribute_impulses.argtypes = [C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
    rng = np.random.default_rng(4)
    for old_count in range(1, 5):
        for new_count in range(1, 5):
            for _ in range(8):
                old_ids = rng.integers(0, 6, size=old_count).astype(np.int32)
                new_ids = rng.integers(0, 6, size=new_count).astype(np.int32)
                old = rng.choice([0.0, 0.25, 1.5, 9.0], size=old_count).astype(np.float32)
                expect = rf.redistribute_impulses(old_ids, old.copy(), new_ids)
                out, scratch = np.zeros(new_count, dtype=np.float32), old.copy()
                lib.oracle_redistribute_impulses(old_count, old_ids.ctypes.data, scratch.ctypes.data, new_count, new_ids.ctypes.data, out.ctypes.data)
                assert np.array_equal(expect.view(np.uint32), out.view(np.uint32)), (old_ids, new_ids, old)


def _redistribution_differs(mutation):
    want, ids = contact_batches()
    got, _ = contact_batches()
    for tw, tg in zip(want.type_batches(), got.type_batches()):
        old, new = ids[(tw.batch_index, tw.type_batch_index)]
        rf.update_contact_impulses(tw, old, new, mutation=mutation)
        ob.update_contact_impulses(tg, old, new)
        if not np.array_equal(tw.accumulated_impulses, tg.accumulated_impulses):
            return True
    return False


@needs_reference
@pytest.mark.parametrize("mutation", rf.MUTATIONS)
def test_each_misreading_of_the_reference_is_caught(libs, mutation):
    part, name = CATCHES[mutation]
    if part == "solve":
        differs = digest(run_reference(name, mutation)) != digest(run_oracle(name))
    elif part == "bounds":
        bounds, activities = bounds_reference(name, mutation)
        differs = bounds_digest(bounds, activities) != bounds_digest(*bounds_oracle(name))
    else:
        differs = _redistribution_differs(mutation)
    assert differs, "%s: case %s does not notice it" % (mutation, name)


# ---- GPU ------------------------------------------------------------------------------------------------------------------------------------------
def _device_frames(name, strict, mode, frames=FRAMES):
    sim, kw = make_case(name)
    ts = bp.CudaTimestepper(sim, strict_fp=strict, execution_mode=mode)
    try:
        ts.describe()
        if "accelerations" in kw:
            ts.set_body_accelerations(kw["accelerations"])
        if "center" in kw:
            ts.set_point_gravity(kw["center"], kw["strength"])
        for f in range(frames):
            if f > 0:
                ts.refresh()
            ts.solve(DT, download=True)
            ts.download_prestep()
    finally:
        ts.close()
    return util.snapshot(sim)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [native.EXEC_GRAPH, native.EXEC_STREAM])
@pytest.mark.parametrize("name", sorted(CASES))
def test_strict_build_equals_the_restatement(libs, name, mode):
    got = _device_frames(name, True, mode)
    if digest(got) != _digests()["solve"][name]:
        util.compare(run_oracle(name), got, exact=True)  # the oracle carries the same digest: name the first differing buffer
        raise AssertionError("%s: the device differs from the restatement's digest" % name)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [native.EXEC_GRAPH, native.EXEC_STREAM])
@pytest.mark.parametrize("name", [n for n in sorted(CASES) if n.startswith(("contacts", "loose"))])
def test_strict_build_resident_redistribution_equals_the_restatement(libs, name, mode):
    """One frame, then the narrow phase's same-type update on the device (set_contact_features, update_contacts) and a second frame; the host side is
    the same frame with the redistribution restated (reference_frame.update_contact_impulses when the library is here, the pinned oracle otherwise)."""
    host, kw = make_case(name)
    dev, _ = make_case(name)
    ids = {}
    rng = np.random.default_rng(31)
    for tb in host.type_batches():
        n = native.contact_count(tb.type_id)
        if n:
            old = rng.integers(0, 8, size=(tb.constraint_count, n)).astype(np.int32)
            new = np.where(rng.random(old.shape) < 0.5, old, rng.integers(0, 8, size=old.shape)).astype(np.int32)
            ids[(tb.batch_index, tb.type_batch_index)] = (old, new)
    solve = rf.solve if rf.library() is not None else ob.solve
    update = rf.update_contact_impulses if rf.library() is not None else ob.update_contact_impulses
    new_prestep = {(tb.batch_index, tb.type_batch_index): tb.prestep.copy() for tb in host.type_batches()}  # the new manifolds' data: the same as frame 1's here
    solve(host, DT, **kw)
    for tb in host.type_batches():
        key = (tb.batch_index, tb.type_batch_index)
        if key in ids:
            tb.prestep[:] = new_prestep[key]
            update(tb, *ids[key])
    solve(host, DT, **kw)
    ts = bp.CudaTimestepper(dev, strict_fp=True, execution_mode=mode)
    try:
        ts.describe()
        if "accelerations" in kw:
            ts.set_body_accelerations(kw["accelerations"])
        if "center" in kw:
            ts.set_point_gravity(kw["center"], kw["strength"])
        ts.set_contact_features({k: v[0] for k, v in ids.items()})
        ts.solve_device_only(DT)
        ts.update_contacts({k: v[1] for k, v in ids.items()})
        ts.solve_device_only(DT)
        ts.download_bodies()
        ts.download_impulses()
        ts.download_prestep()
    finally:
        ts.close()
    util.compare(util.snapshot(host), util.snapshot(dev), exact=True)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(BOUNDS_CASES))
def test_device_bounds_equal_the_restatement(libs, name):
    bodies, shapes, activities, integ, kw = bounds_case(*BOUNDS_CASES[name])
    sim = bp.Simulation(integrator=integ)
    sim.add_bodies(bodies)
    ts = bp.CudaTimestepper(sim, strict_fp=True)
    try:
        ts.describe()
        ts.set_body_shapes(shapes)
        if kw:
            ts.set_body_accelerations(kw["accelerations"])
            ts.set_point_gravity(kw["center"], kw["strength"])
        got = np.stack([ts.predict_bounding_boxes(DT, activities) for _ in range(BOUNDS_FRAMES)])
    finally:
        ts.close()
    assert bounds_digest(got, activities) == _digests()["bounds"][name]


@pytest.mark.gpu
@pytest.mark.parametrize("name", [n for n in sorted(CASES) if n != "ragdolls_four_substeps"])
def test_fast_build_within_the_existing_tolerances(libs, name):
    """The bound the existing fast tests hold these scene families to after one frame: util.compare's defaults (relative RMS <= 1e-3, max abs
    <= 5e-2), as in smoke(). Ragdolls are held to it only at one substep of four iterations
    (tests/test_integrator_extensions.py::test_fast_build_within_joint_tolerance); the ragdoll case here, four substeps with the schedule
    [1, 0, 2, 1], leaves the servo impulses at a relative RMS of 1.4e-3, and this file adds no new bound."""
    util.compare(run_oracle(name, frames=1), _device_frames(name, False, native.EXEC_GRAPH, frames=1), exact=False)
