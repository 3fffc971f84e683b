"""Pose and world-inertia integration in the incremental contact update (kLaunchBodiesIntegrated). In substeps > 0 of a solve with contacts,
the launch of IncrementallyUpdateForSubstep carries one thread per body that integrates the pose and rotates the inverse inertia of every body a
constraint lane integrates, and the WarmStart stages integrate velocity only. CPU: where the stage program sets the flag (topology shim of
tests/test_topology.py), and the shared pose arithmetic of csrc/bepu_integration.cuh compiled for the host against the oracle, bit for bit. GPU:
the strict build against the oracle, bit for bit, on the scenes and schedules that exercise the split."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from bepuphysics2_b200 import native, scenes, sharding
from oracle import binding as ob
from tests import test_topology as topo
from tests import util

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.join(ROOT, "tests", "device_on_host")
CSRC = os.path.join(ROOT, "bepuphysics2_b200", "csrc")
BODIES_INTEGRATED = 32
DT = 1.0 / 60.0
f32 = np.float32

shim = topo.shim


# ---- CPU: the stage program --------------------------------------------------------------------------------------------------------------------------

def _flagged(ops):
    return (ops[:, 5] & BODIES_INTEGRATED) != 0


@pytest.mark.parametrize("iterations", [[1], [2, 2], [0, 2, 1], [3, 0, 1, 2]])
@pytest.mark.parametrize("integrate_velocity_for_kinematics", [False, True])
def test_flag_sits_on_the_incremental_update_and_the_later_warm_starts(libs, shim, iterations, integrate_velocity_for_kinematics):
    sim = util.make_sim(topo.mixed_scene(5), fallback_batch_threshold=6)
    kinematic_count = len(sim.constrained_kinematics)
    p = topo.plan(shim, topo.sim_sources(sim), 8, 6, sim.batch_count, sim.body_count)
    assert p.inc_count > 0 and p.fallback_levels > 0
    ops, totals = p.program(iterations, kinematic_count, integrate_velocity_for_kinematics, False, sim.body_count)
    stage = ops[:, 0]
    want = (stage == topo.INCREMENTAL) | (stage == topo.WS)
    assert _flagged(ops).tolist() == want.tolist()
    assert (stage == topo.INCREMENTAL).sum() == len(iterations) - 1
    assert (stage == topo.WS).sum() == (len(iterations) - 1) * int((p.batches[:, 1] > 0).sum())
    # substep 0 (WarmStartFirst) and its kinematic prepass never carry it; the flag changes no other bit of the program
    assert not _flagged(ops[stage == topo.WS_FIRST]).any()
    assert not _flagged(ops[(stage == topo.KIN) | (stage == topo.KIN_FIRST) | (stage == topo.SOLVE) | (stage == topo.FINAL)]).any()
    topo.check_program(p, ops, totals, iterations, sim.body_count, kinematic_count, integrate_velocity_for_kinematics, False)


def test_flag_is_absent_without_contacts_and_in_peer_mode(libs, shim):
    joints = util.make_sim(scenes.joint_zoo(600, 20, seed=4, kinematic_fraction=0.1))
    p = topo.plan(shim, topo.sim_sources(joints), 8, 64, joints.batch_count, joints.body_count)
    assert p.inc_count == 0
    ops, _ = p.program([2, 1, 2], len(joints.constrained_kinematics), True, False, joints.body_count)
    assert (ops[:, 0] == topo.WS).any() and not _flagged(ops).any()

    sim = util.make_sim(scenes.merge(scenes.shape_pile(1500, seed=13), scenes.ragdolls(4, seed=14)))
    shards, _, _, _ = sharding.partition(sim, 2)
    for r in range(2):
        sources = [(d["batch_index"], d["type_batch_index"], d["type_id"], d["count"], d["refs"]) for d in shards[r]]
        p = topo.plan(shim, sources, sim.bundle_width, sim.fallback_batch_threshold, sim.batch_count, sim.body_count, peer_mode=True)
        assert p.inc_count > 0
        ops, _ = p.program([2, 1, 3], len(sim.constrained_kinematics), True, True, sim.body_count)
        assert (ops[:, 0] == topo.INCREMENTAL).any() and not _flagged(ops).any()


# ---- CPU: the shared pose arithmetic -------------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def pose_on_host(tmp_path_factory):
    lib = str(tmp_path_factory.mktemp("pose_on_host") / "libpose_integration.so")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-march=x86-64-v3", "-Wall", "-Wno-unused-function", "-Wno-unknown-pragmas",
                           "-I", os.path.join(HERE, "stubs"), "-I", CSRC, "-shared", "-fPIC", "-o", lib, os.path.join(HERE, "pose_integration.cpp")])
    dll = C.CDLL(lib)
    dll.pose_integration_on_host.argtypes = [C.POINTER(C.c_float), C.POINTER(C.c_float)]
    return dll


def _ptr(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def test_pose_integration_helper_matches_the_oracle_bit_for_bit(libs, pose_on_host):
    """integrate_pose_and_inertia against the oracle's orientation integration and inertia rotation (PoseIntegrator.cs:L146-175) and the float32
    position update p + v dt, on random states, including the |w| <= 1e-15 identity branch."""
    orc = ob.load()
    orc.oracle_eval_integration.argtypes = [C.c_int32, C.POINTER(C.c_float), C.POINTER(C.c_float)]
    rng = np.random.default_rng(23)
    for trial in range(2000):
        lin = rng.normal(0, 3, 3).astype(f32)
        ang = (rng.normal(0, 1, 3) * 10.0 ** rng.uniform(-3, 1.5)).astype(f32)
        if trial % 100 == 0:
            ang[:] = 0.0
        dt = f32(1.0 / rng.choice([60.0, 240.0, 480.0]))
        r = np.linalg.qr(rng.normal(0, 1, (3, 3)))[0]
        m = r @ np.diag(rng.uniform(0.3, 5.0, 3)) @ r.T
        local = np.array([m[0, 0], m[1, 0], m[1, 1], m[2, 0], m[2, 1], m[2, 2]], dtype=f32)
        pos = rng.normal(0, 20, 3).astype(f32)
        q = rng.normal(0, 1, 4)
        q = (q / np.linalg.norm(q)).astype(f32)
        inp = np.ascontiguousarray(np.r_[lin, ang, dt, local, pos, q], dtype=f32)
        got = np.zeros(13, dtype=f32)
        assert pose_on_host.pose_integration_on_host(_ptr(inp), _ptr(got)) == 0

        q_want = np.zeros(6, dtype=f32)
        assert orc.oracle_eval_integration(0, _ptr(np.ascontiguousarray(np.r_[q, ang, dt * f32(0.5)], dtype=f32)), _ptr(q_want)) == 0
        world_want = np.zeros(6, dtype=f32)
        assert orc.oracle_eval_integration(1, _ptr(np.ascontiguousarray(np.r_[local, q_want[:4]], dtype=f32)), _ptr(world_want)) == 0
        want = np.r_[pos + lin * dt, q_want[:4], world_want].astype(f32)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), "trial %d: %s vs %s" % (trial, got, want)


# ---- GPU: the strict build against the oracle -------------------------------------------------------------------------------------------------------

def _integrator(kinematics=0, angular_mode=0):
    d = native.IntegratorDesc.default()
    d.integrate_velocity_for_kinematics = kinematics
    d.angular_integration_mode = angular_mode
    return d


def _parity(scene, mode=native.EXEC_GRAPH, frames=3, terms=False, profile=False, **kw):
    a, b = util.make_sim(scene, **kw), util.make_sim(scene, **kw)
    acc = np.random.default_rng(31).uniform(-5, 5, size=(a.body_count, 8)).astype(f32) if terms else None
    center, strength = ((1.0, -40.0, 2.0), 800.0) if terms else (None, 0.0)
    for _ in range(frames):
        ob.solve(a, DT, accelerations=acc, center=center, strength=strength)
    ts = native.CudaTimestepper(b, strict_fp=True, execution_mode=mode)
    try:
        ts.describe()
        if terms:
            ts.set_body_accelerations(acc)
            ts.set_point_gravity(center, strength)
        for f in range(frames):
            if f > 0:
                ts.refresh()
            if profile:
                ts.profile_stages(DT)
                ts.download_bodies()
                ts.download_impulses()
            else:
                ts.solve(DT, download=True)
            ts.download_prestep()
    finally:
        ts.close()
    util.compare(util.snapshot(a), util.snapshot(b), exact=True)


def _kinematic_pile():
    """A pile on moving, spinning constrained kinematic grounds, plus an unconstrained kinematic."""
    scene = scenes.merge(scenes.box_stacks(5, 6), scenes.shape_pile(1500, seed=8))
    kin = np.flatnonzero(scene["bodies"][:, 22] == 0)
    assert kin.size > 0
    rng = np.random.default_rng(4)
    scene["bodies"][kin, 8:11] = rng.uniform(-0.3, 0.3, size=(kin.size, 3)).astype(f32)
    scene["bodies"][kin, 12:15] = rng.uniform(-0.2, 0.2, size=(kin.size, 3)).astype(f32)
    return scene


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [native.EXEC_GRAPH, native.EXEC_STREAM])
def test_pile_with_kinematics_bit_exact(libs, mode):
    _parity(_kinematic_pile(), mode=mode, substeps=4, velocity_iterations=2, integrator=_integrator(kinematics=1))


@pytest.mark.gpu
def test_mixed_scene_with_fallback_batch_bit_exact(libs):
    scene = scenes.merge(topo.mixed_scene(9), scenes.fallback_stress(600, hubs=3, seed=5))
    _parity(scene, fallback_batch_threshold=6, substeps=3, velocity_iterations=2, integrator=_integrator(kinematics=1))


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [native.EXEC_GRAPH, native.EXEC_STREAM])
def test_accelerations_and_point_gravity_bit_exact(libs, mode):
    """These contexts keep the pose integration in the WarmStart stages: the flagged program must still give the oracle's answer there."""
    scene = scenes.merge(scenes.shape_pile(2000, seed=12, nonconvex_fraction=0.3), scenes.ragdolls(6, seed=13))
    _parity(scene, mode=mode, terms=True, substeps=3, velocity_iterations=2, integrator=_integrator(kinematics=1))


@pytest.mark.gpu
@pytest.mark.parametrize("iterations", [[0, 2, 1], [2, 0, 0, 1]])
def test_iteration_schedules_with_zeros_bit_exact(libs, iterations):
    _parity(scenes.shape_pile(3000, seed=14), substeps=len(iterations), velocity_iterations=iterations)


@pytest.mark.gpu
def test_profile_stages_integrates_like_solve(libs):
    _parity(scenes.merge(scenes.shape_pile(1500, seed=15), scenes.ragdolls(4, seed=16)), frames=2, profile=True, substeps=3, velocity_iterations=2,
            integrator=_integrator(kinematics=1))


@pytest.mark.gpu
@pytest.mark.parametrize("angular_mode", [1, 2])
def test_momentum_conserving_modes_keep_the_warm_start_integration(libs, angular_mode):
    _parity(scenes.merge(scenes.shape_pile(1500, seed=17), scenes.ragdolls(4, seed=18)), frames=2, substeps=3, velocity_iterations=2,
            integrator=_integrator(kinematics=1, angular_mode=angular_mode))


@pytest.mark.gpu
def test_joints_only_scene_bit_exact(libs):
    _parity(scenes.joint_zoo(800, 30, seed=19, kinematic_fraction=0.1), substeps=3, velocity_iterations=2, integrator=_integrator(kinematics=1))
