"""bepucuda_write_bodies: the motion of listed bodies written straight into the device's body state, what the host changed through BodyReference
between resident frames (include/bepucuda.h).
CPU part: the host-side index check and the staging gather of csrc/bepu_topology.cpp, through tests/topology/body_write_shim.cpp, and the test's own
ApplyImpulse against a float64 evaluation.
GPU part: resident frames (prestep and feature ids through bepucuda_update_contacts) on twins: A sends every body's motion
(bepucuda_upload_body_motion), B only the changed bodies (bepucuda_write_bodies), and the oracle's host twin applies the same changes. Then the
ordering rules, the byte count, the errors and peer mode."""
import ctypes as C
import os

import numpy as np
import pytest

import bepuphysics2_b200 as bp
from bepuphysics2_b200 import _build, scenes, sharding
from bepuphysics2_b200.native import (BODY_ACTIVITY_DTYPE, BODY_SHAPE_DTYPE, ERR_BAD_STATE, ERR_INVALID_ARGUMENT, EXEC_GRAPH, EXEC_STREAM,
                                      SHAPE_SPHERE)
from oracle import binding as ob
from tests import harness, util
from tests.planner import CSRC, ROOT
from tests.resident import initial_features, narrow_phase_like_update, push_bodies

DT = 1.0 / 60.0
MOTION_FLOATS = 16  # floats 0-15 of a 128-B BodyDynamics record: pose and velocity
WRITE_BYTES = 64 + 4  # per listed index: its motion half and the index


# ---- CPU: the index check and the staging gather --------------------------------------------------------------------------------------------------
def body_write_shim():
    cuda_include = os.path.join(os.path.dirname(os.path.dirname(_build.NVCC)), "include")
    dll = harness.load("body_write_shim", [os.path.join(ROOT, "tests", "topology", "body_write_shim.cpp"), os.path.join(CSRC, "bepu_topology.cpp")],
                       ["-O2", "-std=c++17", "-Wall", "-shared", "-fPIC", "-I", cuda_include], includes=[CSRC, os.path.join(ROOT, "include")])
    vp, i32 = C.c_void_p, C.c_int32
    dll.body_write_check.argtypes = [i32, i32, vp, i32, vp]
    dll.body_write_gather.argtypes = [vp, vp, i32, vp]
    return dll


def test_the_index_check_rejects_every_invalid_input_and_accepts_duplicates():
    dll = body_write_shim()
    n = 50
    bodies = np.zeros((n, 32), dtype=np.float32)
    good = np.array([0, 7, 7, 49, 0, 3], dtype=np.int32)

    def check(indices, count=None, uploaded=True, body_count=n, dynamics=bodies):
        idx = None if indices is None else np.ascontiguousarray(indices, dtype=np.int32)
        return dll.body_write_check(int(uploaded), body_count, None if dynamics is None else dynamics.ctypes.data,
                                    len(idx) if count is None else count, None if idx is None else idx.ctypes.data)

    assert check(good) == 0, "duplicates are allowed"
    assert check(None, count=0, dynamics=None) == 0, "count == 0 needs no buffers"
    assert check(good, count=0) == 0
    assert check(good, count=-1) == ERR_INVALID_ARGUMENT
    assert check(None, count=1) == ERR_INVALID_ARGUMENT
    assert check(good, dynamics=None) == ERR_INVALID_ARGUMENT
    assert check(np.r_[good, -1]) == ERR_INVALID_ARGUMENT
    assert check(np.r_[good, n]) == ERR_INVALID_ARGUMENT
    assert check(np.r_[good, np.iinfo(np.int32).min]) == ERR_INVALID_ARGUMENT
    assert check(good, body_count=49) == ERR_INVALID_ARGUMENT, "49 is outside a 49-body upload"
    assert check(good, uploaded=False) == ERR_BAD_STATE
    assert check(None, count=0, dynamics=None, uploaded=False) == ERR_BAD_STATE
    assert check(good, count=-1, uploaded=False) == ERR_INVALID_ARGUMENT, "a malformed call is an argument error first"


def test_the_staging_gather_takes_the_motion_half_of_exactly_the_listed_records_in_order():
    dll = body_write_shim()
    rng = np.random.default_rng(3)
    bodies = rng.standard_normal((300, 32)).astype(np.float32)
    indices = np.r_[rng.integers(0, 300, 500), 299, 0, 0].astype(np.int32)
    out = np.full((len(indices) + 1, MOTION_FLOATS), np.float32(np.nan))
    dll.body_write_gather(bodies.ctypes.data, indices.ctypes.data, len(indices), out.ctypes.data)
    assert np.array_equal(out[:-1].view(np.uint32), bodies[indices, :MOTION_FLOATS].view(np.uint32))
    assert np.isnan(out[-1]).all(), "nothing past the list is written"


# ---- the host's changes -----------------------------------------------------------------------------------------------------------------------------
def rotate_inverse_inertia(q, m):
    """PoseIntegration.RotateInverseInertia (PoseIntegrator.cs:L102-110) in float32, in the reference's operation order: Matrix3x3.CreateFromQuaternion,
    then Symmetric3x3.RotationSandwich. q: [n, 4] (x, y, z, w), m: [n, 6] (XX, YX, YY, ZX, ZY, ZZ). Returns [n, 6]."""
    x, y, z, w = q.T
    one = np.float32(1)
    qx2, qy2, qz2 = x + x, y + y, z + z
    YY, ZZ, XX = qy2 * y, qz2 * z, qx2 * x
    XY, ZW, XZ, YW, XW, YZ = qx2 * y, qz2 * w, qx2 * z, qy2 * w, qx2 * w, qy2 * z
    r = [[one - YY - ZZ, XY + ZW, XZ - YW], [XY - ZW, one - XX - ZZ, YZ + XW], [XZ + YW, YZ - XW, one - XX - YY]]  # rows X, Y, Z
    mxx, myx, myy, mzx, mzy, mzz = m.T
    i = [[r[0][c] * mxx + r[1][c] * myx + r[2][c] * mzx, r[0][c] * myx + r[1][c] * myy + r[2][c] * mzy, r[0][c] * mzx + r[1][c] * mzy + r[2][c] * mzz]
         for c in range(3)]
    out = [i[0][0] * r[0][0] + i[0][1] * r[1][0] + i[0][2] * r[2][0],
           i[1][0] * r[0][0] + i[1][1] * r[1][0] + i[1][2] * r[2][0], i[1][0] * r[0][1] + i[1][1] * r[1][1] + i[1][2] * r[2][1],
           i[2][0] * r[0][0] + i[2][1] * r[1][0] + i[2][2] * r[2][0], i[2][0] * r[0][1] + i[2][1] * r[1][1] + i[2][2] * r[2][1],
           i[2][0] * r[0][2] + i[2][1] * r[1][2] + i[2][2] * r[2][2]]
    return np.stack(out, axis=1).astype(np.float32)


def apply_impulse(bodies, index, impulse, offset):
    """BodyReference.ApplyImpulse(impulse, impulseOffset, ref localInertia, ref pose, ref velocity) (BodyReference.cs:L351-356) on one record: the
    world inverse inertia from the local one and the current orientation, then ApplyLinearImpulse and ApplyAngularImpulse."""
    rec = bodies[index]
    s = rotate_inverse_inertia(rec[None, 0:4], rec[None, 16:22])[0]
    rec[8:11] += impulse * rec[22]
    a = np.array([offset[1] * impulse[2] - offset[2] * impulse[1], offset[2] * impulse[0] - offset[0] * impulse[2],
                  offset[0] * impulse[1] - offset[1] * impulse[0]], dtype=np.float32)
    rec[12:15] += np.array([a[0] * s[0] + a[1] * s[1] + a[2] * s[3], a[0] * s[1] + a[1] * s[2] + a[2] * s[4], a[0] * s[3] + a[1] * s[4] + a[2] * s[5]],
                           dtype=np.float32)


def test_apply_impulse_follows_the_rotated_inverse_inertia():
    rng = np.random.default_rng(5)
    bodies = np.zeros((40, 32), dtype=np.float32)
    q = rng.standard_normal((40, 4))
    bodies[:, 0:4] = q / np.linalg.norm(q, axis=1, keepdims=True)
    a = rng.standard_normal((40, 3, 3))
    local = np.einsum("nij,nkj->nik", a, a) + np.eye(3)  # symmetric positive definite
    bodies[:, 16:22] = local[:, [0, 1, 1, 2, 2, 2], [0, 0, 1, 0, 1, 2]]
    bodies[:, 22] = rng.uniform(0.5, 2, 40)
    before = bodies.copy()
    impulse, offset = rng.standard_normal((40, 3)).astype(np.float32), rng.standard_normal((40, 3)).astype(np.float32)
    for k in range(40):
        apply_impulse(bodies, k, impulse[k], offset[k])
    qq = before[:, 0:4].astype(np.float64)
    x, y, z, w = qq.T
    R = np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], -1),
                  np.stack([2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)], -1),
                  np.stack([2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], -1)], 1)  # world <- local
    world = R @ local @ R.transpose(0, 2, 1)
    dw = np.einsum("nij,nj->ni", world, np.cross(offset.astype(np.float64), impulse.astype(np.float64)))
    assert np.allclose(bodies[:, 12:15] - before[:, 12:15], dw, rtol=1e-4, atol=1e-4)
    assert np.allclose(bodies[:, 8:11] - before[:, 8:11], impulse * before[:, 22:23], rtol=1e-6, atol=1e-6)


def change_bodies(sim, frame, kinematic, seed=21):
    """What a host does between frames through BodyReference, deterministic in (frame, seed) and the bodies' state: push_bodies' velocity kick of a
    fifth of the bodies, an ApplyImpulse at an offset on a few dynamic bodies (a tank's recoil, a character standing on a body), a teleport, and a
    constrained kinematic mover's next pose and velocity. Returns the indices touched, in order (overlaps included)."""
    rng = np.random.default_rng((seed, frame))
    b = sim.bodies
    push_bodies(sim, frame)
    kicked = np.arange(frame % 5, sim.body_count, 5)
    dynamic = np.flatnonzero(b[:, 22] != 0)
    hit = rng.choice(dynamic, size=min(8, len(dynamic)), replace=False)
    for k in hit:
        apply_impulse(b, k, rng.uniform(-0.05, 0.05, 3).astype(np.float32), rng.uniform(-0.5, 0.5, 3).astype(np.float32))
    teleported = rng.choice(dynamic, size=1)
    b[teleported, 4:7] += np.float32(0.002)
    moved = []
    if kinematic is not None:
        b[kinematic, 4:7] += b[kinematic, 8:11] * np.float32(DT)
        b[kinematic, 8:11] = np.float32([0.5 * np.sin(frame), 0.0, 0.25])
        b[kinematic, 12:15] = np.float32([0.0, 0.0, 0.25 + 0.05 * frame])
        moved = [kinematic]
    return np.concatenate([kicked, hit, teleported, moved]).astype(np.int32)


# ---- GPU: twins ---------------------------------------------------------------------------------------------------------------------------------------
ZOO = lambda: scenes.merge(scenes.shape_pile(1500, seed=41, nonconvex_fraction=0.4), scenes.joint_zoo(600, per_type=20, seed=42),
                           scenes.ragdolls(10, seed=43))
SCENES = {
    "pile_width4": (lambda: scenes.shape_pile(2000, seed=33, nonconvex_fraction=0.3), dict(bundle_width=4)),
    "pile_width16": (lambda: scenes.shape_pile(2000, seed=34, nonconvex_fraction=0.3), dict(bundle_width=16)),
    "ragdolls": (lambda: scenes.ragdolls(24, seed=5), {}),
    "zoo_fallback": (ZOO, dict(fallback_batch_threshold=6, holes=True)),
}
MODES = {"graph": EXEC_GRAPH, "stream": EXEC_STREAM}


def make_sim(scene, bundle_width=8, fallback_batch_threshold=64, holes=False):
    sim = util.make_sim(scene, bundle_width=bundle_width, fallback_batch_threshold=fallback_batch_threshold, substeps=3, velocity_iterations=2)
    if holes:
        assert util.punch_fallback_holes(sim) > 0
    return sim


def same_bits(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint32), np.ascontiguousarray(b).view(np.uint32))


def state(ts, sim):
    """Bodies, accumulated impulses and prestep rows of every type batch after the full downloads."""
    ts.download_bodies()
    ts.download_impulses()
    ts.download_prestep()
    tbs = sim.type_batches()
    return [sim.bodies.copy()] + [tb.accumulated_impulses.copy() for tb in tbs] + [tb.prestep.copy() for tb in tbs]


def host_state(sim):
    tbs = sim.type_batches()
    return [sim.bodies.copy()] + [tb.accumulated_impulses.copy() for tb in tbs] + [tb.prestep.copy() for tb in tbs]


def constrained_kinematic(sim):
    kin = sim.constrained_kinematics
    return int(kin[0]) if len(kin) else None


def twin_frames(case, mode, register, strict=True, write=True, frames=4):
    """Resident frames of twins A (every body's motion up) and B (bepucuda_write_bodies of the changed indices; nothing when not `write`) next to
    the oracle's host twin. Returns per frame whether B's motion equalled A's and the host twin's, the three final states, whether a constrained
    kinematic body was moved, and the per-frame (h2d of B - h2d of A, expected difference, graph captures of B)."""
    make, kw = SCENES[case]
    scene = make()
    host, a, b = make_sim(scene, **kw), make_sim(scene, **kw), make_sim(scene, **kw)
    kinematic = constrained_kinematic(host)
    rngs = [np.random.default_rng(77) for _ in range(3)]
    ts_a = bp.CudaTimestepper(a, strict_fp=strict, execution_mode=mode)
    ts_b = bp.CudaTimestepper(b, strict_fp=strict, execution_mode=mode)
    same_a, same_host, accounting = [], [], []
    try:
        for ts in (ts_a, ts_b):
            if register:
                ts.register_host_buffers()
            ts.describe()
        feats = [initial_features(s, r) for s, r in zip((host, a, b), rngs)]
        ts_a.set_contact_features(feats[1])
        ts_b.set_contact_features(feats[2])
        for frame in range(frames):
            if frame > 0:
                new = [narrow_phase_like_update(s, f, r) for s, f, r in zip((host, a, b), feats, rngs)]
                for tb in host.type_batches():
                    key = (tb.batch_index, tb.type_batch_index)
                    if key in new[0]:
                        ob.update_contact_impulses(tb, feats[0][key], new[0][key])
                for f, n in zip(feats, new):
                    f.update({key: ids.copy() for key, ids in n.items()})
                change_bodies(host, frame, kinematic)
                change_bodies(a, frame, kinematic)
                indices = change_bodies(b, frame, kinematic)
                ts_a.upload_body_motion()
                ts_a.update_contacts(new[1])
                if write:
                    ts_b.write_bodies(indices)
                ts_b.update_contacts(new[2])
            ob.solve(host, DT)
            ts_a.solve_device_only(DT)
            ts_b.solve_device_only(DT)
            ts_a.download_body_motion()
            ts_b.download_body_motion()
            ta, tb_ = ts_a.timings(), ts_b.timings()
            if frame > 0:
                accounting.append((tb_.h2d_bytes - ta.h2d_bytes, (WRITE_BYTES * len(indices) if write else 0) - 64 * b.body_count, tb_.graph_captures))
            same_a.append(same_bits(a.bodies[:, :MOTION_FLOATS], b.bodies[:, :MOTION_FLOATS]))
            same_host.append(same_bits(host.bodies[:, util.MOTION], b.bodies[:, util.MOTION]))
        got_a, got_b = state(ts_a, a), state(ts_b, b)
    finally:
        ts_a.close()
        ts_b.close()
    return same_a, same_host, (host_state(host), got_a, got_b, host), kinematic is not None, accounting


def assert_on_the_oracle(want, got, host):
    assert same_bits(want[0][:, util.MEANINGFUL], got[0][:, util.MEANINGFUL])
    tbs = host.type_batches()
    for k, tb in enumerate(tbs):
        live = (tb.body_references[:, 0, :] >= 0)[:, None, :]
        for what, offset in (("impulses", 1), ("prestep", 1 + len(tbs))):
            assert same_bits(np.where(live, want[offset + k], 0), np.where(live, got[offset + k], 0)), "%s of type batch %s" % (what, (tb.batch_index, tb.type_id))


@pytest.mark.gpu
@pytest.mark.parametrize("buffers", ["registered", "unregistered"])
@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("case", sorted(SCENES))
def test_writes_of_the_changed_bodies_match_the_full_upload_and_the_oracle(libs, case, mode, buffers):
    same_a, same_host, (want, got_a, got_b, host), moved_kinematic, accounting = twin_frames(case, MODES[mode], buffers == "registered")
    assert all(same_a), same_a
    assert all(same_host), same_host
    assert all(same_bits(x, y) for x, y in zip(got_a, got_b)), "final bodies, impulses and prestep of B equal A's byte for byte"
    assert_on_the_oracle(want, got_b, host)
    assert moved_kinematic == (case != "pile_width4" and case != "pile_width16")
    captures = accounting[0][2]
    for got, expected, graph_captures in accounting:
        assert got == expected
        assert graph_captures == captures, "a write never re-captures the graph"


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["pile_width16", "zoo_fallback"])
def test_fast_build_writes_match_the_full_upload_byte_for_byte(libs, case):
    same_a, _, (_, got_a, got_b, _), _, _ = twin_frames(case, EXEC_GRAPH, case == "pile_width16", strict=False)
    assert all(same_a), same_a
    assert all(same_bits(x, y) for x, y in zip(got_a, got_b))


@pytest.mark.gpu
def test_without_the_write_the_twin_leaves_the_full_upload(libs):
    same_a, same_host, (_, got_a, got_b, _), _, _ = twin_frames("zoo_fallback", EXEC_GRAPH, False, write=False)
    assert same_a[0] and not all(same_a[1:]) and not all(same_host[1:])
    assert not same_bits(got_a[0][:, util.MOTION], got_b[0][:, util.MOTION])


# ---- GPU: ordering ----------------------------------------------------------------------------------------------------------------------------------
def raw_write(ts, bodies, indices, count=None):
    idx = None if indices is None else np.ascontiguousarray(indices, dtype=np.int32)
    return ts._cuda.bepucuda_write_bodies(ts._ctx, None if bodies is None else bodies.ctypes.data, len(idx) if count is None else count,
                                          None if idx is None or idx.size == 0 else idx.ctypes.data)


def motion(ts, sim):
    out = sim.bodies.copy()
    ts._check(ts._cuda.bepucuda_download_body_motion(ts._ctx, out.ctypes.data, sim.body_count))
    return out[:, :MOTION_FLOATS].copy()


def device_bodies(ts, sim):
    out = sim.bodies.copy()
    ts._check(ts._cuda.bepucuda_download_bodies(ts._ctx, out.ctypes.data, sim.body_count))
    return out


def small_sim():
    return make_sim(scenes.merge(scenes.shape_pile(600, seed=3, nonconvex_fraction=0.3), scenes.ragdolls(6, seed=5)))


def expected_motion(base, source, indices):
    """Pose and velocity as the device holds them after `source`'s listed records were written over `base`: the padding floats 7, 11 and 15 are 0."""
    want = base[:, :MOTION_FLOATS].copy()
    want[indices] = source[indices, :MOTION_FLOATS]
    want[:, [7, 11, 15]] = 0
    return want


@pytest.mark.gpu
@pytest.mark.parametrize("buffers", ["registered", "unregistered"])
def test_the_last_of_a_write_and_a_full_upload_wins_and_downloads_see_it_before_a_solve(libs, buffers):
    sim = small_sim()
    ts = bp.CudaTimestepper(sim, strict_fp=True)
    try:
        if buffers == "registered":
            ts.register_host_buffers()
        ts.describe()
        rng = np.random.default_rng(8)
        base = sim.bodies.copy()
        changed = base.copy()
        idx = rng.choice(sim.body_count, size=40, replace=False).astype(np.int32)
        changed[idx, :MOTION_FLOATS] += rng.uniform(-1, 1, (40, MOTION_FLOATS)).astype(np.float32)
        source = changed if buffers == "unregistered" else sim.bodies  # a registered source is the registered buffer itself
        # a write after a full upload wins
        sim.bodies[:] = base
        ts.upload_body_motion()
        if buffers == "registered":
            ts.synchronize()  # the full upload has read the mapped buffer
            sim.bodies[:] = changed
        assert raw_write(ts, source, idx) == 0
        assert same_bits(motion(ts, sim), expected_motion(base, changed, idx))
        # the inertia halves are the uploaded ones, and download_bodies sees the write too
        full = device_bodies(ts, sim)
        assert same_bits(full[:, 16:23], base[:, 16:23])
        assert same_bits(full[:, util.MOTION], changed[:, util.MOTION])
        # a full upload after a write wins
        if buffers == "unregistered":
            assert raw_write(ts, changed, idx) == 0
        sim.bodies[:] = base
        ts.upload_body_motion()
        assert same_bits(motion(ts, sim), expected_motion(base, base, idx))
        # duplicates within a call write the same record, and of two calls the last wins
        first, last = base.copy(), base.copy()
        first[idx, 8:11] += np.float32(1)
        last[idx, 8:11] -= np.float32(1)
        if buffers == "unregistered":
            assert raw_write(ts, first, np.r_[idx, idx, idx[:5]]) == 0
            assert raw_write(ts, last, np.r_[idx[::-1], idx]) == 0
        else:
            sim.bodies[:] = first
            assert raw_write(ts, sim.bodies, np.r_[idx, idx, idx[:5]]) == 0
            ts.synchronize()
            sim.bodies[:] = last
            assert raw_write(ts, sim.bodies, np.r_[idx[::-1], idx]) == 0
        assert same_bits(motion(ts, sim), expected_motion(base, last, idx))
    finally:
        ts.close()


@pytest.mark.gpu
def test_predict_bounding_boxes_sees_a_write_before_any_solve(libs):
    sims = [small_sim(), small_sim()]
    ctxs = [bp.CudaTimestepper(s, strict_fp=True) for s in sims]
    try:
        n = sims[0].body_count
        shapes = np.zeros(n, dtype=BODY_SHAPE_DTYPE)
        shapes["type"], shapes["a"] = SHAPE_SPHERE, 0.5
        shapes["maximum_speculative_margin"] = np.float32(np.inf)
        for ts in ctxs:
            ts.describe()
            ts.set_body_shapes(shapes)

        def predict(ts):
            act = np.zeros(n, dtype=BODY_ACTIVITY_DTYPE)
            act["sleep_threshold"], act["minimum_timesteps_under_threshold"] = 0.01, 32
            return ts.predict_bounding_boxes(DT, act).copy()

        before = predict(ctxs[0])
        idx = np.arange(0, n, 7, dtype=np.int32)
        for s in sims:
            s.bodies[idx, 4:7] += np.float32(3)  # teleports
            s.bodies[idx, 8:11] += np.float32(2)
        ctxs[0].write_bodies(idx)
        ctxs[1].upload_body_motion()
        got, want = predict(ctxs[0]), predict(ctxs[1])
        assert same_bits(got, want)
        moved = np.zeros(n, dtype=bool)
        moved[idx] = True
        assert not np.array_equal(got[moved], before[moved]) and same_bits(got[~moved], before[~moved])
    finally:
        for ts in ctxs:
            ts.close()


# ---- GPU: errors ------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_rejected_writes_leave_the_device_bodies_as_they_were(libs):
    sim = small_sim()
    fresh = bp.CudaTimestepper(sim, strict_fp=True)
    ts = bp.CudaTimestepper(sim, strict_fp=True)
    try:
        idx = np.array([0, 1, 2], dtype=np.int32)
        assert raw_write(fresh, sim.bodies, idx) == ERR_BAD_STATE, "before upload_bodies"
        assert raw_write(fresh, None, None, count=0) == ERR_BAD_STATE
        ts.describe()
        ts.solve_device_only(DT)
        before = device_bodies(ts, sim)
        changed = sim.bodies.copy()
        changed[:, 8:11] += np.float32(1)
        n = sim.body_count
        assert raw_write(ts, changed, idx, count=-1) == ERR_INVALID_ARGUMENT
        assert raw_write(ts, None, idx) == ERR_INVALID_ARGUMENT
        assert raw_write(ts, changed, None, count=3) == ERR_INVALID_ARGUMENT
        assert raw_write(ts, changed, np.r_[idx, -1]) == ERR_INVALID_ARGUMENT
        assert raw_write(ts, changed, np.r_[idx, n]) == ERR_INVALID_ARGUMENT, "the last listed index is out of range: nothing before it is written"
        assert raw_write(ts, changed, np.r_[n + 1000, idx]) == ERR_INVALID_ARGUMENT
        assert raw_write(ts, None, None, count=0) == 0
        assert raw_write(ts, changed, idx, count=0) == 0
        assert same_bits(device_bodies(ts, sim), before)
    finally:
        fresh.close()
        ts.close()


# ---- GPU: peer mode ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_a_two_rank_shard_given_the_same_writes_stays_on_the_single_context(libs):
    """Ranks as contexts of one process on device 0 (util.run_ranks), each given the same list as the single context."""
    scene = scenes.merge(scenes.shape_pile(800, seed=4), scenes.ragdolls(6, seed=5))
    single = make_sim(scene)
    ranks_sim = make_sim(scene)
    kinematic = constrained_kinematic(single)
    ts = bp.CudaTimestepper(single, strict_fp=True)
    solvers = [sharding.ShardedSolver(ranks_sim, r, 2, 0, strict_fp=True) for r in range(2)]
    try:
        ts.describe()
        for s in solvers:
            s.export_handles()
        for s in solvers:
            s.import_contexts(solvers)
        for s in solvers:
            s.describe()
        for frame in range(4):
            if frame > 0:
                indices = change_bodies(single, frame, kinematic)
                ts.write_bodies(indices)
                for s in solvers:
                    s.bodies[indices, :MOTION_FLOATS] = single.bodies[indices, :MOTION_FLOATS]
                    s._check(s._cuda.bepucuda_write_bodies(s._ctx, s.bodies.ctypes.data, len(indices), indices.ctypes.data))
            ts.solve_device_only(DT)
            util.solve_all(solvers, DT)
            ts.download_body_motion()
            for s in solvers:
                s._check(s._cuda.bepucuda_download_body_motion(s._ctx, s.bodies.ctypes.data, ranks_sim.body_count))
                mine = s.referenced_bodies()
                assert mine.size > 0
                assert same_bits(single.bodies[mine][:, util.MOTION], s.bodies[mine][:, util.MOTION]), "rank %d, frame %d" % (s.rank, frame)
    finally:
        ts.close()
        for s in solvers:
            s.close()
