"""Per-body accelerations and point gravity after the declarative velocity callback (bepucuda_set_body_accelerations /
bepucuda_set_point_gravity; PerBodyGravityDemo.cs and PlanetDemo.cs of the reference). The oracle of the terms is
tests/integrator_extensions/oracle_integrator_extensions.cpp: the oracle's translation unit with the driver functions that call IntegrateVelocity
restated. CPU: that oracle against closed forms, its scalar against its 8-wide evaluation, per-body gravity against uniform gravity, no terms
against oracle_solve, and the CUDA arithmetic compiled for the host against it. GPU: the strict build against it bit for bit at every
integration site, the fast build within tolerance, and the error rules."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from bepuphysics2_b200 import native, scenes, sharding
from oracle import binding as ob
from tests import util

DT = 1.0 / 60.0
f32 = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.join(ROOT, "tests", "integrator_extensions")
_LIBS = {}


class Terms(C.Structure):
    """bepu_oracle::ext::Terms of oracle_integrator_extensions.cpp."""
    _fields_ = [("accelerations", C.c_void_p), ("point_gravity", C.c_int32), ("center", C.c_float * 3), ("strength", C.c_float)]


def _compile(name, source, flags):
    """Both test libraries are compiled once per process into a temporary directory: the tree itself may be read-only."""
    if name not in _LIBS:
        if "dir" not in _LIBS:
            _LIBS["dir"] = tempfile.mkdtemp(prefix="bepu_integrator_extensions_")
            atexit.register(shutil.rmtree, _LIBS["dir"], True)
        lib = os.path.join(_LIBS["dir"], name)
        subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-march=x86-64-v3", "-Wall",
                               "-Wno-unused-function", "-Wno-psabi"] + flags + ["-o", lib, os.path.join(HERE, source)])
        _LIBS[name] = C.CDLL(lib)
    return _LIBS[name]


def _oracle_ext():
    lib = _compile("liboracle_integrator_extensions.so", "oracle_integrator_extensions.cpp", ["-fopenmp", "-I", os.path.join(ROOT, "oracle")])
    lib.oracle_ext_solve.argtypes = [C.POINTER(ob.OracleScene), C.POINTER(Terms), C.c_float]
    lib.oracle_ext_predict_bounding_boxes.argtypes = [C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p, C.c_float, C.c_float, C.c_int32,
                                                      C.POINTER(Terms), C.c_void_p]
    lib.oracle_ext_eval.argtypes = [C.c_void_p, C.c_void_p]
    return lib


def _terms(accelerations, center, strength):
    t = Terms()
    acc = None if accelerations is None else np.ascontiguousarray(accelerations, dtype=np.float32).reshape(-1, 8)
    t.accelerations = acc.ctypes.data if acc is not None and acc.size else None
    t.point_gravity = 0 if center is None else 1
    if center is not None:
        for i in range(3):
            t.center[i] = float(np.float32(center[i]))
        t.strength = float(np.float32(strength))
    return t, acc


def solve_ex(simulation, dt, accelerations=None, center=None, strength=0.0, simd=False):
    """ob.solve on `simulation`'s buffers in place, with the terms (oracle_ext_solve; one worker)."""
    terms, acc = _terms(accelerations, center, strength)
    assert acc is None or acc.shape[0] == simulation.body_count
    per_batch = [[] for _ in range(simulation.batch_count)]
    for tb in simulation.type_batches():
        per_batch[tb.batch_index].append(tb)
    keep = []
    batches = (ob.OracleBatch * max(simulation.batch_count, 1))()
    for b, tbs in enumerate(per_batch):
        arr = (ob.OracleTypeBatch * max(len(tbs), 1))()
        for i, tb in enumerate(tbs):
            arr[i].type_id, arr[i].constraint_count = tb.type_id, tb.constraint_count
            arr[i].body_references, arr[i].prestep, arr[i].accumulated_impulses = tb.body_references.ctypes.data, tb.prestep.ctypes.data, tb.accumulated_impulses.ctypes.data
        keep.append(arr)
        batches[b].type_batch_count, batches[b].type_batches = len(tbs), arr
    sc = ob.OracleScene()
    sc.bodies = simulation.bodies.ctypes.data if simulation.body_count else None
    sc.body_count, sc.batch_count, sc.batches, sc.bundle_width = simulation.body_count, simulation.batch_count, batches, simulation.bundle_width
    its = (C.c_int32 * len(simulation.velocity_iterations))(*simulation.velocity_iterations)
    sc.substep_count, sc.velocity_iterations, sc.fallback_batch_threshold = len(simulation.velocity_iterations), its, simulation.fallback_batch_threshold
    d = simulation.integrator
    for i in range(3):
        sc.gravity[i] = d.gravity[i]
    sc.linear_damping, sc.angular_damping, sc.angular_integration_mode = d.linear_damping, d.angular_damping, d.angular_integration_mode
    sc.allow_substeps_for_unconstrained, sc.integrate_velocity_for_kinematics = d.allow_substeps_for_unconstrained, d.integrate_velocity_for_kinematics
    kin = np.ascontiguousarray(simulation.constrained_kinematics, dtype=np.int32)
    sc.constrained_kinematics, sc.constrained_kinematic_count = (kin.ctypes.data if kin.size else None), int(kin.size)
    sc.threads, sc.simd = 1, 1 if simd else 0
    rc = _oracle_ext().oracle_ext_solve(C.byref(sc), C.byref(terms), dt)
    assert rc == 0, "oracle_ext_solve failed: %d" % rc


def predict_bounding_boxes_ex(bodies, shapes, activities, dt, integrator, accelerations=None, center=None, strength=0.0):
    """ob.predict_bounding_boxes with the terms (oracle_ext_predict_bounding_boxes); activities updated in place."""
    bodies = np.ascontiguousarray(bodies, dtype=np.float32).reshape(-1, 32)
    n = bodies.shape[0]
    shapes = np.ascontiguousarray(shapes)
    terms, acc = _terms(accelerations, center, strength)
    bounds = np.zeros((max(n, 1), 8), dtype=np.float32)
    gravity = (C.c_float * 3)(*integrator.gravity)
    rc = _oracle_ext().oracle_ext_predict_bounding_boxes(n, bodies.ctypes.data, shapes.ctypes.data, activities.ctypes.data, dt, gravity, integrator.linear_damping,
                                                         integrator.angular_damping, int(integrator.integrate_velocity_for_kinematics), C.byref(terms), bounds.ctypes.data)
    assert rc == 0
    return bounds[:n]


def _integrator(gravity=(0.0, -10.0, 0.0), damping=0.03, angular_mode=0, allow_substeps=0, kinematics=0):
    d = native.IntegratorDesc.default()
    for i in range(3):
        d.gravity[i] = gravity[i]
    d.linear_damping = d.angular_damping = damping
    d.angular_integration_mode = angular_mode
    d.allow_substeps_for_unconstrained = allow_substeps
    d.integrate_velocity_for_kinematics = kinematics
    return d


def _accelerations(n, seed, scale=5.0):
    a = np.random.default_rng(seed).uniform(-scale, scale, size=(n, 8)).astype(np.float32)
    a[:, 3] = a[:, 7] = 0.0
    return a


def _one_body(position, linear, angular, **integ):
    scene = {"bodies": scenes.make_bodies(np.array([position], dtype=np.float32), linear=np.array([linear], dtype=np.float32),
                                          angular=np.array([angular], dtype=np.float32), inverse_mass=np.array([1], dtype=np.float32),
                                          inverse_inertia=np.array([[1, 0, 1, 0, 0, 1]], dtype=np.float32)), "constraints": []}
    return scene


# ---- CPU -------------------------------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("allow_substeps", [0, 1])
def test_unconstrained_body_takes_a_times_dt(libs, allow_substeps):
    """One unconstrained body, damping 0: every step v' = (v + g dt) * 1 + a dt, then p' = p + v' dt, in float32 in that order."""
    substeps = 3
    g = f32(-10.0)
    a = _accelerations(1, 1)
    sim = util.make_sim(_one_body((1, 2, 3), (0.5, -1.0, 2.0), (0.25, -0.5, 0.75)), substeps=substeps, velocity_iterations=1,
                        integrator=_integrator(gravity=(0.0, -10.0, 0.0), damping=0.0, allow_substeps=allow_substeps))
    v = sim.bodies[0, 8:11].copy()
    w = sim.bodies[0, 12:15].copy()
    p = sim.bodies[0, 4:7].copy()
    solve_ex(sim, DT, accelerations=a)
    dt = f32(DT) / f32(substeps) if allow_substeps else f32(DT)
    for _ in range(substeps if allow_substeps else 1):
        v = (v + np.array([0, g * dt, 0], dtype=f32)) * f32(1.0)
        v = v + a[0, 0:3] * dt
        w = w * f32(1.0) + a[0, 4:7] * dt
        p = p + v * dt
    assert np.array_equal(sim.bodies[0, 8:11], v)
    assert np.array_equal(sim.bodies[0, 12:15], w)
    assert np.array_equal(sim.bodies[0, 4:7], p)


def test_point_gravity_one_step(libs):
    """PlanetDemo's callback for one step: v' = v - (dt * strength * offset) * (1 / max(1, |offset|^3))."""
    center, strength = np.array([0.5, -20.0, 3.0], dtype=f32), f32(1000.0)
    sim = util.make_sim(_one_body((4, 7, -2), (0.0, 0.0, 0.0), (0.0, 0.0, 0.0)), integrator=_integrator(gravity=(0, 0, 0), damping=0.0))
    pos = sim.bodies[0, 4:7].copy()
    solve_ex(sim, DT, center=center, strength=strength)
    offset = pos - center
    d = np.sqrt(offset[0] * offset[0] + offset[1] * offset[1] + offset[2] * offset[2])
    inverse = f32(1.0) / max(f32(1.0), d * d * d)
    v = np.zeros(3, dtype=f32) - (offset * (f32(DT) * strength)) * inverse
    assert np.array_equal(sim.bodies[0, 8:11], v)
    assert np.array_equal(sim.bodies[0, 4:7], pos + v * f32(DT))


def _mixed_scene():
    return scenes.merge(scenes.box_stacks(4, 6), scenes.ragdolls(6, seed=3), scenes.joint_zoo(400, 20, seed=4))


@pytest.mark.parametrize("angular_mode", [0, 1, 2])
def test_scalar_and_eight_wide_oracle_agree_with_both_terms(libs, angular_mode):
    scene = _mixed_scene()
    integ = _integrator(angular_mode=angular_mode, kinematics=1)
    a, b = (util.make_sim(scene, substeps=3, velocity_iterations=2, integrator=integ) for _ in range(2))
    acc = _accelerations(a.body_count, 5)
    for _ in range(2):
        solve_ex(a, DT, accelerations=acc, center=(0, -30, 0), strength=500.0)
        solve_ex(b, DT, accelerations=acc, center=(0, -30, 0), strength=500.0, simd=True)
    util.compare(util.snapshot(a), util.snapshot(b), exact=True)


def test_per_body_acceleration_equal_to_gravity_matches_uniform_gravity(libs):
    """Damping 0: (v + g dt) * 1 with gravity g equals (v + 0) * 1 + g dt with gravity 0 and a = g, elementwise."""
    scene = scenes.box_stacks(4, 6)
    extra = scenes.make_bodies(np.array([[50, 5, 0], [60, 5, 0]], dtype=np.float32), linear=np.array([[1, 2, 3], [0, 1, 0]], dtype=np.float32),
                               inverse_mass=np.array([1, 1], dtype=np.float32), inverse_inertia=np.array([[2, 0, 2, 0, 0, 2]] * 2, dtype=np.float32))
    scene["bodies"] = np.concatenate([scene["bodies"], extra])
    uniform = util.make_sim(scene, substeps=4, velocity_iterations=2, integrator=_integrator(gravity=(0, -10, 0), damping=0.0))
    per_body = util.make_sim(scene, substeps=4, velocity_iterations=2, integrator=_integrator(gravity=(0, 0, 0), damping=0.0))
    acc = np.zeros((per_body.body_count, 8), dtype=np.float32)
    acc[:, 1] = -10.0
    for _ in range(2):
        ob.solve(uniform, DT)
        solve_ex(per_body, DT, accelerations=acc)
    cols = util.MEANINGFUL
    assert (uniform.bodies[:, cols] == per_body.bodies[:, cols]).all()


def test_no_extension_is_oracle_solve_bit_for_bit(libs):
    scene = _mixed_scene()
    a, b = (util.make_sim(scene, substeps=2, velocity_iterations=2, integrator=_integrator(kinematics=1)) for _ in range(2))
    ob.solve(a, DT)
    solve_ex(b, DT)
    util.compare(util.snapshot(a), util.snapshot(b), exact=True)


def test_extension_source_on_host_matches_the_oracle_bit_for_bit():
    """integrate_velocity_extensions of csrc/bepu_integration.cuh compiled for the host against the oracle's statement, on random operands."""
    dev = _compile("libdevice_integrator_extensions_on_host.so", "device_integrator_extensions_on_host.cpp",
                   ["-I", os.path.join(ROOT, "tests", "device_on_host", "stubs"), "-I", os.path.join(ROOT, "bepuphysics2_b200", "csrc")])
    dev.device_integrator_extensions_on_host_eval.argtypes = [C.c_void_p, C.c_void_p]
    orc = _oracle_ext()
    rng = np.random.default_rng(17)
    for k in range(4000):
        x = np.zeros(22, dtype=np.float32)
        x[0:12] = rng.normal(0, 5, size=12)
        x[12] = rng.uniform(1e-3, 0.05)
        x[13:19] = rng.normal(0, 3 if k % 2 else 50, size=6)
        x[19] = rng.uniform(-100, 100)
        x[20], x[21] = (k >> 1) & 1, 1 if k % 4 != 1 else 0
        a, b = np.zeros(6, dtype=np.float32), np.zeros(6, dtype=np.float32)
        assert dev.device_integrator_extensions_on_host_eval(x.ctypes.data, a.ctypes.data) == 0
        assert orc.oracle_ext_eval(x.ctypes.data, b.ctypes.data) == 0
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), (k, x, a, b)


# ---- GPU -------------------------------------------------------------------------------------------------------------------------------------------

CENTER, STRENGTH = (1.0, -40.0, 2.0), 800.0


def _gpu_parity(scene, frames=2, mode=native.EXEC_GRAPH, exact=True, resident=False, rel_rms=1e-3, max_abs=5e-2, **kw):
    a, b = util.make_sim(scene, **kw), util.make_sim(scene, **kw)
    acc = _accelerations(a.body_count, 11)
    for _ in range(frames):
        solve_ex(a, DT, accelerations=acc, center=CENTER, strength=STRENGTH)
    ts = native.CudaTimestepper(b, strict_fp=exact, execution_mode=mode)
    try:
        ts.describe()
        ts.set_body_accelerations(acc)
        ts.set_point_gravity(CENTER, STRENGTH)
        for f in range(frames):
            if resident and f < frames - 1:
                ts.solve_device_only(DT)
                continue
            if f > 0 and not resident:
                ts.refresh()
            ts.solve(DT, download=True)
            ts.download_prestep()
    finally:
        ts.close()
    util.compare(util.snapshot(a), util.snapshot(b), exact=exact, rel_rms=rel_rms, max_abs=max_abs)


GPU_SCENES = {
    "box_stacks": lambda: scenes.box_stacks(8, 10),
    "joint_zoo": lambda: scenes.joint_zoo(1200, 40, seed=8, kinematic_fraction=0.05),
    "ragdolls": lambda: scenes.ragdolls(30, seed=5),
}


@pytest.mark.gpu
@pytest.mark.parametrize("scene", sorted(GPU_SCENES))
@pytest.mark.parametrize("mode", [native.EXEC_GRAPH, native.EXEC_STREAM])
def test_scenes_bit_exact(libs, scene, mode):
    _gpu_parity(GPU_SCENES[scene](), mode=mode, substeps=3, velocity_iterations=2, integrator=_integrator(kinematics=1))


@pytest.mark.gpu
@pytest.mark.parametrize("angular_mode", [0, 1, 2])
@pytest.mark.parametrize("allow_substeps", [0, 1])
def test_angular_modes_and_unconstrained_bodies_bit_exact(libs, angular_mode, allow_substeps):
    scene = scenes.joint_zoo(800, 30, seed=9, kinematic_fraction=0.05)
    extra = scenes.make_bodies(np.array([[100, 5, 0], [120, 5, 0], [140, 0, 0]], dtype=np.float32), linear=np.array([[1, 2, 3], [0, 0, 0], [0, 1, 0]], dtype=np.float32),
                               angular=np.array([[0.5, 0.1, -0.3], [0, 1, 0], [0, 0, 0]], dtype=np.float32), inverse_mass=np.array([1, 0, 1], dtype=np.float32),
                               inverse_inertia=np.array([[2, 0, 2, 0, 0, 2], [0, 0, 0, 0, 0, 0], [1, 0.1, 2, 0, 0.2, 3]], dtype=np.float32))
    scene["bodies"] = np.concatenate([scene["bodies"], extra])
    _gpu_parity(scene, substeps=3, velocity_iterations=1, integrator=_integrator(angular_mode=angular_mode, allow_substeps=allow_substeps, kinematics=1))


@pytest.mark.gpu
def test_resident_frames_bit_exact(libs):
    _gpu_parity(scenes.merge(scenes.box_stacks(6, 8), scenes.ragdolls(10, seed=2)), frames=4, resident=True, substeps=2, velocity_iterations=2,
                integrator=_integrator(kinematics=1))


@pytest.mark.gpu
def test_fast_build_within_joint_tolerance(libs):
    """DESIGN §5's joint tolerance for the fast build: relative RMS <= 1e-3, max abs <= 2e-2 after one frame."""
    _gpu_parity(scenes.ragdolls(60, seed=5), frames=1, exact=False, rel_rms=1e-3, max_abs=2e-2, substeps=1, velocity_iterations=4)


@pytest.mark.gpu
def test_predict_bounding_boxes_with_both_terms(libs):
    rng = np.random.default_rng(3)
    sim = util.make_sim(scenes.shape_pile(600, seed=2), substeps=1, velocity_iterations=1, integrator=_integrator(kinematics=1))
    n = sim.body_count
    shapes = np.zeros(n, dtype=native.BODY_SHAPE_DTYPE)
    shapes["type"] = rng.choice([0, 1, 2, 4], size=n)
    shapes["a"], shapes["b"], shapes["c"] = (rng.uniform(0.1, 1.0, size=n) for _ in range(3))
    shapes["minimum_speculative_margin"], shapes["maximum_speculative_margin"] = 0.0, 1e3
    activities = np.zeros(n, dtype=native.BODY_ACTIVITY_DTYPE)
    activities["sleep_threshold"], activities["minimum_timesteps_under_threshold"] = 0.01, 4
    acc = _accelerations(n, 4, scale=50.0)
    ref_act = activities.copy()
    ref = predict_bounding_boxes_ex(sim.bodies, shapes, ref_act, DT, sim.integrator, accelerations=acc, center=CENTER, strength=STRENGTH)
    plain = ob.predict_bounding_boxes(sim.bodies, shapes, activities.copy(), DT, sim.integrator)
    assert not np.array_equal(ref, plain)
    ts = native.CudaTimestepper(sim, strict_fp=True)
    try:
        ts.describe()
        ts.set_body_shapes(shapes)
        ts.set_body_accelerations(acc)
        ts.set_point_gravity(CENTER, STRENGTH)
        got = ts.predict_bounding_boxes(DT, activities)
    finally:
        ts.close()
    assert np.array_equal(ref.view(np.uint32), got.view(np.uint32))
    assert np.array_equal(ref_act, activities)


@pytest.mark.gpu
def test_profile_stages_advances_like_solve(libs):
    scene = scenes.merge(scenes.box_stacks(6, 8), scenes.joint_zoo(400, 20, seed=6))
    a, b = (util.make_sim(scene, substeps=2, velocity_iterations=2, integrator=_integrator(kinematics=1)) for _ in range(2))
    acc = _accelerations(a.body_count, 12)
    solve_ex(a, DT, accelerations=acc, center=CENTER, strength=STRENGTH)
    ts = native.CudaTimestepper(b, strict_fp=True)
    try:
        ts.describe()
        ts.set_body_accelerations(acc)
        ts.set_point_gravity(CENTER, STRENGTH)
        ts.profile_stages(DT)
        ts.download_bodies()
        ts.download_impulses()
        ts.download_prestep()
    finally:
        ts.close()
    util.compare(util.snapshot(a), util.snapshot(b), exact=True)


@pytest.mark.gpu
def test_two_shard_ranks_bit_exact(libs):
    """Every rank holds every body and is given the whole acceleration array; the owning lane's results travel through the peer stores."""
    sim = util.make_sim(scenes.merge(scenes.shape_pile(1200, seed=21), scenes.ragdolls(12, seed=22)), substeps=3, velocity_iterations=2, integrator=_integrator())
    acc = _accelerations(sim.body_count, 13)
    solvers = [sharding.ShardedSolver(sim, r, 2, 0, strict_fp=True) for r in range(2)]
    try:
        for s in solvers:
            s.export_handles()
        for s in solvers:
            s.import_contexts(solvers)
        for s in solvers:
            s.describe()
            s._check(s._cuda.bepucuda_set_body_accelerations(s._ctx, acc.ctypes.data, sim.body_count))
            center = np.array(CENTER, dtype=np.float32)
            s._check(s._cuda.bepucuda_set_point_gravity(s._ctx, 1, center.ctypes.data, C.c_float(STRENGTH)))
        for s in solvers:
            s.synchronize()
        for _ in range(2):
            solve_ex(sim, DT, accelerations=acc, center=CENTER, strength=STRENGTH)
            for s in solvers:
                s.solve(DT)
        for s in solvers:
            got = s.download()
            mine = s.referenced_bodies()
            assert np.array_equal(sim.bodies[mine][:, util.MOTION].view(np.uint32), got[mine][:, util.MOTION].view(np.uint32)), "rank %d" % s.rank
    finally:
        for s in solvers:
            s.close()


@pytest.mark.gpu
def test_argument_and_state_errors(libs):
    scene = scenes.box_stacks(4, 4)
    sim = util.make_sim(scene, substeps=2, velocity_iterations=1)
    ts = native.CudaTimestepper(sim, strict_fp=True)
    try:
        ts.describe()
        with pytest.raises(native.BepuCudaError) as e:
            ts.set_body_accelerations(np.zeros((sim.body_count + 1, 8), dtype=np.float32))
        assert e.value.code == -1  # BEPUCUDA_ERR_INVALID_ARGUMENT
        ts.set_body_accelerations(np.zeros((sim.body_count, 8), dtype=np.float32))
        more = np.concatenate([sim.bodies, sim.bodies[-1:]])
        ts._check(ts._cuda.bepucuda_upload_bodies(ts._ctx, more.ctypes.data, more.shape[0]))
        for call in (lambda: ts.solve_device_only(DT), lambda: ts.profile_stages(DT), lambda: ts.predict_bounding_boxes(DT, np.zeros(more.shape[0], dtype=native.BODY_ACTIVITY_DTYPE))):
            with pytest.raises(native.BepuCudaError) as e:
                call()
            assert e.value.code == -6  # BEPUCUDA_ERR_BAD_STATE
        ts.set_body_accelerations(None)
        ts._check(ts._cuda.bepucuda_upload_bodies(ts._ctx, sim.bodies.ctypes.data, sim.body_count))
    finally:
        ts.close()


@pytest.mark.gpu
def test_cleared_terms_equal_a_context_that_never_set_them(libs):
    scene = scenes.merge(scenes.box_stacks(4, 6), scenes.joint_zoo(300, 20, seed=2))
    a, b = (util.make_sim(scene, substeps=2, velocity_iterations=2, integrator=_integrator(kinematics=1)) for _ in range(2))
    ref = util.run_gpu(a, DT, frames=2)
    ts = native.CudaTimestepper(b, strict_fp=True)
    try:
        ts.describe()
        ts.set_body_accelerations(_accelerations(b.body_count, 3))
        ts.set_point_gravity(CENTER, STRENGTH)
        ts.set_body_accelerations(None)
        ts.set_point_gravity(None, 0.0)
        for f in range(2):
            if f > 0:
                ts.refresh()
            ts.solve(DT, download=True)
            ts.download_prestep()
    finally:
        ts.close()
    util.compare(ref, util.snapshot(b), exact=True)
