"""ORACLE — test infrastructure only. ctypes loader for oracle/libbepu_oracle.so and a helper that runs it on a host `Simulation`'s buffers
(in place, like the reference's Simulation.Solve). Parity: the arithmetic is pinned to the reference's C# text (oracle/ref_transpile); the solver driver is unpinned (see oracle/bepu_math.h)."""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


class OracleTypeBatch(C.Structure):
    _fields_ = [("type_id", C.c_int32), ("constraint_count", C.c_int32), ("body_references", C.c_void_p), ("prestep", C.c_void_p), ("accumulated_impulses", C.c_void_p)]


class OracleBatch(C.Structure):
    _fields_ = [("type_batch_count", C.c_int32), ("type_batches", C.POINTER(OracleTypeBatch))]


class OracleIntegratorTerms(C.Structure):
    _fields_ = [("accelerations", C.c_void_p), ("point_gravity", C.c_int32), ("center", C.c_float * 3), ("strength", C.c_float)]


class OracleScene(C.Structure):
    _fields_ = [
        ("bodies", C.c_void_p), ("body_count", C.c_int32), ("batch_count", C.c_int32), ("batches", C.POINTER(OracleBatch)), ("bundle_width", C.c_int32),
        ("substep_count", C.c_int32), ("velocity_iterations", C.POINTER(C.c_int32)), ("fallback_batch_threshold", C.c_int32),
        ("gravity", C.c_float * 3), ("linear_damping", C.c_float), ("angular_damping", C.c_float), ("angular_integration_mode", C.c_int32),
        ("allow_substeps_for_unconstrained", C.c_int32), ("integrate_velocity_for_kinematics", C.c_int32),
        ("constrained_kinematics", C.c_void_p), ("constrained_kinematic_count", C.c_int32), ("threads", C.c_int32), ("simd", C.c_int32),
        ("terms", OracleIntegratorTerms),
    ]


def _terms(body_count, accelerations, center, strength):
    """The optional velocity terms: per-body accelerations (body_count x 8 floats {a.xyz 0 | alpha.xyz 0}) and point gravity toward `center`
    with `strength` (None: off). Returns the struct and the array it points into, which the caller keeps alive."""
    t = OracleIntegratorTerms()
    acc = None
    if accelerations is not None:
        acc = np.ascontiguousarray(accelerations, dtype=np.float32).reshape(-1, 8)
        assert acc.shape[0] == body_count
        t.accelerations = acc.ctypes.data if acc.size else None
    if center is not None:
        t.point_gravity = 1
        t.center[:] = [float(c) for c in center]
        t.strength = strength
    return t, acc


def build(force=False):
    lib = os.path.join(HERE, "libbepu_oracle.so")
    srcs = [os.path.join(HERE, f) for f in ("bepu_oracle.cpp", "bepu_oracle.h", "bepu_math.h", "bepu_contacts.h", "bepu_joints.h", "bepu_joints_more.h")]
    if force or not os.path.exists(lib) or any(os.path.getmtime(s) > os.path.getmtime(lib) for s in srcs):
        r = subprocess.run(["make", "-C", HERE] + (["-B"] if force else []), stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if r.returncode != 0:
            raise RuntimeError("oracle build failed:\n" + r.stdout)
    return lib


def load():
    global _LIB
    if _LIB is None:
        path = os.path.join(HERE, "libbepu_oracle.so")
        if not os.path.exists(path):
            build()
        os.environ.setdefault("OMP_WAIT_POLICY", "passive")  # libgomp's default spin-wait collapses when the container has fewer CPUs than it reports
        _LIB = C.CDLL(path)
        _LIB.oracle_solve.argtypes = [C.POINTER(OracleScene), C.c_float]
        _LIB.oracle_type_info.argtypes = [C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
    return _LIB


def type_info(type_id):
    b, p, d = C.c_int32(), C.c_int32(), C.c_int32()
    if load().oracle_type_info(type_id, C.byref(b), C.byref(p), C.byref(d)) != 0:
        return None
    return b.value, p.value, d.value


def max_threads():
    return load().oracle_max_threads()


def scene(simulation, threads=1, simd=False, accelerations=None, center=None, strength=0.0):
    """The oracle_scene of `simulation`'s buffers with the optional velocity terms (see _terms), and the ctypes objects it points into, which the
    caller keeps alive while the scene is used."""
    tbs = simulation.type_batches()
    batch_count = simulation.batch_count
    per_batch = [[] for _ in range(batch_count)]
    for tb in tbs:
        per_batch[tb.batch_index].append(tb)
    keep = []
    batches = (OracleBatch * max(batch_count, 1))()
    for b in range(batch_count):
        arr = (OracleTypeBatch * max(len(per_batch[b]), 1))()
        for i, tb in enumerate(per_batch[b]):
            arr[i].type_id = tb.type_id
            arr[i].constraint_count = tb.constraint_count
            arr[i].body_references = tb.body_references.ctypes.data
            arr[i].prestep = tb.prestep.ctypes.data
            arr[i].accumulated_impulses = tb.accumulated_impulses.ctypes.data
        keep.append(arr)
        batches[b].type_batch_count = len(per_batch[b])
        batches[b].type_batches = arr
    sc = OracleScene()
    bodies = simulation.bodies
    sc.bodies = bodies.ctypes.data if simulation.body_count else None
    sc.body_count = simulation.body_count
    sc.batch_count = batch_count
    sc.batches = batches
    sc.bundle_width = simulation.bundle_width
    its = (C.c_int32 * len(simulation.velocity_iterations))(*simulation.velocity_iterations)
    sc.substep_count = len(simulation.velocity_iterations)
    sc.velocity_iterations = its
    sc.fallback_batch_threshold = simulation.fallback_batch_threshold
    d = simulation.integrator
    for i in range(3):
        sc.gravity[i] = d.gravity[i]
    sc.linear_damping, sc.angular_damping = d.linear_damping, d.angular_damping
    sc.angular_integration_mode = d.angular_integration_mode
    sc.allow_substeps_for_unconstrained = d.allow_substeps_for_unconstrained
    sc.integrate_velocity_for_kinematics = d.integrate_velocity_for_kinematics
    kin = np.ascontiguousarray(simulation.constrained_kinematics, dtype=np.int32)
    sc.constrained_kinematics = kin.ctypes.data if kin.size else None
    sc.constrained_kinematic_count = int(kin.size)
    sc.threads = threads
    sc.simd = 1 if simd else 0
    sc.terms, acc = _terms(simulation.body_count, accelerations, center, strength)
    return sc, (tbs, keep, batches, bodies, its, kin, acc)


def solve(simulation, dt, threads=1, simd=False, accelerations=None, center=None, strength=0.0):
    """Runs the oracle's Simulation.Solve restatement in place on `simulation`'s buffers (bodies, prestep depths, accumulated impulses), with the
    optional velocity terms of bepucuda_set_body_accelerations / bepucuda_set_point_gravity (see _terms)."""
    lib = load()
    sc, keep = scene(simulation, threads, simd, accelerations, center, strength)  # keep: alive until oracle_solve returns
    rc = lib.oracle_solve(C.byref(sc), dt)
    if rc != 0:
        raise RuntimeError("oracle_solve failed: %d" % rc)


def update_contact_impulses(type_batch, old_feature_ids, new_feature_ids):
    """NarrowPhase.UpdateConstraint, same-type branch, on a host type batch's accumulated impulses in place (NarrowPhaseConstraintUpdate.cs:L81-183)."""
    lib = load()
    lib.oracle_update_contact_impulses.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    old = np.ascontiguousarray(old_feature_ids, dtype=np.int32)
    new = np.ascontiguousarray(new_feature_ids, dtype=np.int32)
    rc = lib.oracle_update_contact_impulses(type_batch.type_id, type_batch.constraint_count, type_batch.accumulated_impulses.shape[2], type_batch.accumulated_impulses.ctypes.data,
                                            old.ctypes.data, new.ctypes.data)
    if rc != 0:
        raise ValueError("not a contact constraint type: %d" % type_batch.type_id)


def first_fit_batches(refs, body_count, fallback_threshold=64, order=0, priorities=None):
    """Sequential restatement of Solver.Add's batch search (Solver.cs:L1182-1199) over refs[n, slots] (encoded body references, -1 = unused slot)."""
    lib = load()
    refs = np.ascontiguousarray(refs, dtype=np.int32)
    n, slots = refs.shape
    out = np.full(n, -1, dtype=np.int32)
    pr = None if priorities is None else np.ascontiguousarray(priorities, dtype=np.uint32)
    lib.oracle_first_fit_batches.argtypes = [C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]
    count = lib.oracle_first_fit_batches(n, slots, refs.ctypes.data, body_count, fallback_threshold, order, None if pr is None else pr.ctypes.data, out.ctypes.data)
    if count < 0:
        raise ValueError("oracle_first_fit_batches failed: %d" % count)
    return out, count


def predict_bounding_boxes(bodies, shapes, activities, dt, integrator, accelerations=None, center=None, strength=0.0):
    """PoseIntegrator.PredictBoundingBoxes restated (PoseIntegrator.cs:L307-370): bodies[n, 32], shapes / activities as the record arrays of
    bepuphysics2_b200.native (activities updated in place), velocity terms as for solve. Returns bounds[n, 8] = {min.xyz, speculative margin,
    max.xyz, valid}."""
    lib = load()
    bodies = np.ascontiguousarray(bodies, dtype=np.float32).reshape(-1, 32)
    n = bodies.shape[0]
    assert shapes.shape[0] == n and activities.shape[0] == n and shapes.dtype.itemsize == 32 and activities.dtype.itemsize == 8
    shapes = np.ascontiguousarray(shapes)
    bounds = np.zeros((max(n, 1), 8), dtype=np.float32)
    gravity = (C.c_float * 3)(*integrator.gravity)
    terms, acc = _terms(n, accelerations, center, strength)
    lib.oracle_predict_bounding_boxes.argtypes = [C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p, C.c_float, C.c_float, C.c_int32, C.c_void_p,
                                                  C.POINTER(OracleIntegratorTerms)]
    rc = lib.oracle_predict_bounding_boxes(n, bodies.ctypes.data, shapes.ctypes.data, activities.ctypes.data, dt, gravity, integrator.linear_damping, integrator.angular_damping,
                                           int(integrator.integrate_velocity_for_kinematics), bounds.ctypes.data, C.byref(terms))
    assert rc == 0
    return bounds[:n]
