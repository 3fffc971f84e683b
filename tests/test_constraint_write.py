"""bepucuda_write_constraints: prestep rows of listed constraints written straight into the device rows, their accumulated impulses left in place
(Solver.ApplyDescription on the resident path, include/bepucuda.h).
CPU part: the shared location resolver (resolve_location) and the write queue of csrc/bepu_topology.cpp, through tests/topology/location_shim.cpp,
against the forward maps of the planner (tests/planner.py).
GPU part: twins held to the oracle bit for bit with every change sent through the write alone; the write route against the whole-type-batch route;
the queue's semantics (last write wins, writes win over whole-batch uploads, pending until the solve, dropped by a describe); and the errors."""
import os

import numpy as np
import pytest

import bepuphysics2_b200 as bp
from bepuphysics2_b200 import _build, scenes, sharding
from bepuphysics2_b200.native import ERR_BAD_STATE, ERR_INVALID_ARGUMENT, EXEC_GRAPH, EXEC_STREAM, contact_count
from oracle import binding as ob
from tests import harness, util
from tests.planner import CSRC, ROOT, constraints_of, inverse_of, plan, sim_sources
from tests.resident import initial_features, push_bodies

DT = 1.0 / 60.0
PRESTEP = 18  # first prestep word of a record
WRITE_BYTES = 12  # PrestepWrite: the device slot and the first of its prestep floats, which follow it in the upload


# ---- CPU: the resolver and the queue ------------------------------------------------------------------------------------------------------------
def location_shim():
    import ctypes as C

    cuda_include = os.path.join(os.path.dirname(os.path.dirname(_build.NVCC)), "include")
    dll = harness.load("location_shim", [os.path.join(ROOT, "tests", "topology", "location_shim.cpp"), os.path.join(CSRC, "bepu_topology.cpp")],
                       ["-O2", "-std=c++17", "-Wall", "-shared", "-fPIC", "-I", cuda_include], includes=[CSRC, os.path.join(ROOT, "include")])
    vp, i32 = C.c_void_p, C.c_int32
    dll.locations_resolve.argtypes = [i32, vp, vp, i32, i32, i32, i32, i32, vp, vp]
    dll.write_queue.argtypes = [i32, i32, i32, i32, vp, vp, i32, vp, vp]
    return dll


def resolve_all(sources, W, threshold, batch_count, body_count, locations):
    """[n, 4]: return code, device type batch, slot, inverse entry of every location (int32[n, 4] with the set index first)."""
    import ctypes as C

    dll = location_shim()
    meta = np.array([s[:4] for s in sources], dtype=np.int32).reshape(len(sources), 4)
    refs = [np.ascontiguousarray(s[4], dtype=np.int32) for s in sources]
    ptrs = (C.c_void_p * max(len(sources), 1))(*[r.ctypes.data for r in refs])
    loc = np.ascontiguousarray(locations, dtype=np.int32).reshape(-1, 4)
    out = np.zeros((max(len(loc), 1), 4), dtype=np.int64)
    assert dll.locations_resolve(len(sources), meta.ctypes.data, ptrs, W, threshold, batch_count, body_count, len(loc), loc.ctypes.data, out.ctypes.data) == 0
    return out[:len(loc)]


def with_set(locations, set_index=0):
    loc = np.asarray(locations, dtype=np.int32).reshape(-1, 3)
    return np.concatenate([np.full((len(loc), 1), set_index, dtype=np.int32), loc], axis=1)


@pytest.mark.parametrize("case", ["mixed_w8", "fallback_stress_w4", "holes_w16"])
def test_the_resolver_sends_every_location_to_the_slot_of_the_forward_maps(libs, case):
    scene, W, threshold = {"mixed_w8": (lambda: scenes.merge(scenes.shape_pile(1200, seed=3, nonconvex_fraction=0.3), scenes.joint_zoo(400, per_type=8, seed=4)), 8, 6),
                           "fallback_stress_w4": (lambda: scenes.fallback_stress(3000, hubs=6, seed=7), 4, 4),
                           "holes_w16": (lambda: scenes.merge(scenes.shape_pile(800, seed=5), scenes.joint_zoo(300, per_type=6, seed=6)), 16, 3)}[case]
    sim = util.make_sim(scene(), bundle_width=W, fallback_batch_threshold=threshold)
    punched = util.punch_fallback_holes(sim) if case == "holes_w16" else 0
    sources = sim_sources(sim)
    p = plan(sources, W, threshold, sim.batch_count, sim.body_count)
    assert p.fallback_levels > 0
    source_tb, offsets, _ = inverse_of(p)
    forward = {}
    for tb in range(len(p.tbs)):
        for slot, c in enumerate(constraints_of(p, sources, tb)):
            if c >= 0:
                forward[(int(p.tbs[tb, 3]), int(c))] = (tb, slot)
    locations = sim.constraint_locations()
    got = resolve_all(sources, W, threshold, sim.batch_count, sim.body_count, with_set(locations))
    assert (got[:, 0] == 0).all()
    source_of = {(s[0], s[2]): k for k, s in enumerate(sources)}
    holes = 0
    for (batch, type_id, i), (_, tb, slot, entry) in zip(locations.tolist(), got.tolist()):
        s = source_of[(batch, type_id)]
        if batch < threshold:
            assert (tb, slot, entry) == (source_tb[s], i, -1), "a synchronized source: identity slots"
        elif sources[s][4][i // W, 0, i % W] < 0:
            holes += 1
            assert (tb, slot, entry) == (-1, -1, offsets[s] + i), "a hole resolves to no slot"
        else:
            assert (tb, slot, entry) == forward[(s, i)] + (offsets[s] + i,), (batch, type_id, i)
    assert holes >= punched
    # locations of no constraint are rejected and leave the output as it was
    tb = sim.type_batches()[0]
    present = {(t.batch_index, t.type_id) for t in sim.type_batches()}
    missing_type = next(t for t in range(64) if bp.type_info(t) and (tb.batch_index, t) not in present)
    bad = [[1, tb.batch_index, tb.type_id, 0], [0, -1, tb.type_id, 0], [0, sim.batch_count, tb.type_id, 0], [0, tb.batch_index, missing_type, 0],
           [0, tb.batch_index, 64, 0], [0, tb.batch_index, -1, 0], [0, tb.batch_index, tb.type_id, tb.constraint_count], [0, tb.batch_index, tb.type_id, -1]]
    got = resolve_all(sources, W, threshold, sim.batch_count, sim.body_count, bad)
    assert (got[:, 0] == ERR_INVALID_ARGUMENT).all() and (got[:, 1:] == -7).all()


@pytest.mark.parametrize("rounds", [1, 2])
def test_the_write_queue_keeps_one_entry_per_slot_and_the_last_write(rounds):
    """rounds = 2: the same writes again after a clear(), as the next frame's writes follow a solve."""
    dll = location_shim()
    rng = np.random.default_rng(4)
    n, rows = 5000, 23
    slots = np.stack([rng.integers(0, 4, n), rng.integers(0, 300, n)], axis=1).astype(np.int32)
    values = rng.standard_normal((n, rows)).astype(np.float32)
    out_slots = np.zeros((n, 2), dtype=np.int32)
    out_rows = np.zeros((n, rows), dtype=np.float32)
    count = dll.write_queue(4, 10, rounds, n, slots.ctypes.data, values.ctypes.data, rows, out_slots.ctypes.data, out_rows.ctypes.data)
    keys = [tuple(s) for s in slots.tolist()]
    first = list(dict.fromkeys(keys))
    last = {k: i for i, k in enumerate(keys)}
    assert count == len(first) < n
    assert [tuple(s) for s in out_slots[:count].tolist()] == first, "entries in the order their slots were first written"
    for slot, got in zip(first, out_rows[:count]):
        assert np.array_equal(got, values[last[slot]]), slot


# ---- GPU helpers ----------------------------------------------------------------------------------------------------------------------------------
def records_of(sim, locations):
    """Records in the layout of bepucuda_read_constraints with the type id and the prestep rows of the host's buffers (what ApplyDescription left
    there); every other word 0."""
    loc = np.asarray(locations, dtype=np.int32).reshape(-1, 3)
    out = np.zeros((len(loc), 64), dtype=np.int32)
    W = sim.bundle_width
    for tb in sim.type_batches():
        sel = np.flatnonzero((loc[:, 0] == tb.batch_index) & (loc[:, 1] == tb.type_id))
        i = loc[sel, 2]
        out[sel, 0] = tb.type_id
        out[sel, PRESTEP:PRESTEP + tb.prestep_rows] = tb.prestep[i // W, :, i % W].view(np.int32)
    return out


def apply_records(sim, locations, records):
    """Solver.ApplyDescription on the host's buffers: the prestep rows of the records into their lanes, in order (a later duplicate wins)."""
    loc = np.asarray(locations, dtype=np.int32).reshape(-1, 3)
    W = sim.bundle_width
    for tb in sim.type_batches():
        for k in np.flatnonzero((loc[:, 0] == tb.batch_index) & (loc[:, 1] == tb.type_id)):
            i = loc[k, 2]
            tb.prestep[i // W, :, i % W] = records[k, PRESTEP:PRESTEP + tb.prestep_rows].view(np.float32)


def changed(records, rng):
    """New descriptions for the records: an AngularMotor gets a new target velocity, an AngularServo a new target orientation; every other joint
    moves its last three (settings) rows by up to 1 %, a contact every row. Huge and non-finite values (unlimited forces) stay."""
    rec = records.copy()
    f = rec[:, PRESTEP:PRESTEP + 35].view(np.float32)
    for type_id in np.unique(rec[:, 0]).tolist():
        k = np.flatnonzero(rec[:, 0] == type_id)
        P = bp.type_info(type_id)[1]
        if type_id == 30:  # AngularMotor: TargetVelocityLocalA
            f[k, 0:3] = rng.uniform(-2, 2, (len(k), 3))
        elif type_id == 29:  # AngularServo: TargetRelativeRotationLocalA
            axis = rng.standard_normal((len(k), 3))
            half = rng.uniform(-0.3, 0.3, (len(k), 1))
            f[k, 0:4] = np.concatenate([axis / np.linalg.norm(axis, axis=1, keepdims=True) * np.sin(half), np.cos(half)], axis=1)
        else:
            rows = slice(0, P) if contact_count(type_id) else slice(max(0, P - 3), P)
            v = f[k, rows]
            keep = np.isfinite(v) & (np.abs(v) < 1e30)
            f[k, rows] = np.where(keep, v * (1 + rng.uniform(-0.01, 0.01, v.shape)), v).astype(np.float32)
    return rec


def live_locations(sim):
    """Every location that holds a constraint (fallback holes left out), and which of them are joints."""
    loc = sim.constraint_locations()
    W = sim.bundle_width
    live = np.zeros(len(loc), dtype=bool)
    at = 0
    for tb in sim.type_batches():
        i = np.arange(tb.constraint_count)
        live[at:at + tb.constraint_count] = tb.body_references[i // W, 0, i % W] >= 0
        at += tb.constraint_count
    loc = loc[live]
    joints = np.array([contact_count(int(t)) == 0 for t in loc[:, 1]], dtype=bool)
    return loc, joints


def pick(rng, loc, joints, fraction=0.1, contacts=20):
    """A random `fraction` of the joints and at least one joint of every joint type, plus `contacts` contacts (200 in a scene without joints)."""
    j = rng.permutation(np.flatnonzero(joints))
    c = np.flatnonzero(~joints)
    one_per_type = j[np.unique(loc[j, 1], return_index=True)[1]]
    chosen = [j[:max(1, int(fraction * len(j)))], one_per_type] if len(j) else []
    if len(c):
        chosen.append(rng.choice(c, size=min(contacts if len(j) else 200, len(c)), replace=False))
    return loc[np.concatenate(chosen)]


def same_bits(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint32), np.ascontiguousarray(b).view(np.uint32))


def state(ts, sim):
    """Bodies, accumulated impulses and prestep rows of every type batch after the full downloads."""
    ts.download_bodies()
    ts.download_impulses()
    ts.download_prestep()
    tbs = sim.type_batches()
    return [sim.bodies.copy()] + [tb.accumulated_impulses.copy() for tb in tbs] + [tb.prestep.copy() for tb in tbs]


def same_state(a, b):
    return len(a) == len(b) and all(same_bits(x, y) for x, y in zip(a, b))


MOTOR_RAGDOLLS = lambda: scenes.merge(scenes.ragdolls(24, seed=5, motor="motor"), scenes.ragdolls(24, seed=6, motor="servo"))
ZOO = lambda: scenes.merge(scenes.shape_pile(1500, seed=41, nonconvex_fraction=0.4), scenes.joint_zoo(600, per_type=20, seed=42),
                           scenes.ragdolls(10, seed=43, motor="motor"), scenes.ragdolls(10, seed=44, motor="servo"))
SCENES = {
    "ragdolls": (MOTOR_RAGDOLLS, {}),
    "zoo_fallback": (ZOO, dict(fallback_batch_threshold=6, holes=True)),
    "pile_width4": (lambda: scenes.shape_pile(2000, seed=33, nonconvex_fraction=0.3), dict(bundle_width=4)),
    "pile_width16": (lambda: scenes.shape_pile(2000, seed=34, nonconvex_fraction=0.3), dict(bundle_width=16)),
}
MODES = {"graph": EXEC_GRAPH, "stream": EXEC_STREAM}


def make_sim(scene, bundle_width=8, fallback_batch_threshold=64, holes=False, substeps=3, velocity_iterations=2):
    sim = util.make_sim(scene, bundle_width=bundle_width, fallback_batch_threshold=fallback_batch_threshold, substeps=substeps, velocity_iterations=velocity_iterations)
    if holes:
        assert util.punch_fallback_holes(sim) > 0
    return sim


# ---- GPU: twins held to the oracle ----------------------------------------------------------------------------------------------------------------
def twin_frames(case, mode, write=True, frames=4, seed=11):
    """Resident frames of a device twin next to the oracle's host twin. Before every frame but the first, random constraints get new descriptions:
    the host twin in its buffers (ApplyDescription), the device twin only through bepucuda_write_constraints. Returns whether the body motion
    agreed bit for bit after every frame, the host twin's and the device twin's final state, and the type ids changed."""
    make, kw = SCENES[case]
    scene = make()
    host, dev = make_sim(scene, **kw), make_sim(scene, **kw)
    rng = np.random.default_rng(seed)
    loc, joints = live_locations(host)
    ts = bp.CudaTimestepper(dev, strict_fp=True, execution_mode=mode)
    agreed, types = True, set()
    try:
        ts.describe()
        for frame in range(frames):
            if frame > 0:
                chosen = pick(rng, loc, joints)
                records = changed(records_of(host, chosen), rng)
                types.update(records[:, 0].tolist())
                apply_records(host, chosen, records)
                if write:
                    ts.write_constraints(chosen, records)
                push_bodies(host, frame)
                push_bodies(dev, frame)
                ts.upload_body_motion()
            ob.solve(host, DT)
            ts.solve_device_only(DT)
            ts.download_body_motion()
            agreed = agreed and same_bits(host.bodies[:, util.MOTION], dev.bodies[:, util.MOTION])
            assert agreed or not write, "frame %d" % frame
        got = state(ts, dev)
    finally:
        ts.close()
    want = [host.bodies.copy()] + [tb.accumulated_impulses.copy() for tb in host.type_batches()] + [tb.prestep.copy() for tb in host.type_batches()]
    return agreed, want, got, types, host


@pytest.mark.gpu
@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("case", sorted(SCENES))
def test_writes_alone_keep_the_device_twin_on_the_oracle(libs, case, mode):
    agreed, want, got, types, host = twin_frames(case, MODES[mode])
    assert agreed
    # final downloads: bodies (every meaningful float), then impulses and prestep on live lanes
    assert same_bits(want[0][:, util.MEANINGFUL], got[0][:, util.MEANINGFUL])
    tbs = host.type_batches()
    for k, tb in enumerate(tbs):
        live = (tb.body_references[:, 0, :] >= 0)[:, None, :]
        for what, offset in (("impulses", 1), ("prestep", 1 + len(tbs))):
            assert same_bits(np.where(live, want[offset + k], 0), np.where(live, got[offset + k], 0)), "%s of type batch %s" % (what, (tb.batch_index, tb.type_id))
    if case == "ragdolls":
        assert {29, 30} <= types
    if case == "zoo_fallback":
        assert len({t for t in types if not contact_count(t)}) == 30 and any(contact_count(t) for t in types)
        assert any(tb.batch_index >= 6 for tb in tbs)


@pytest.mark.gpu
def test_without_the_writes_the_device_twin_leaves_the_oracle(libs):
    agreed, want, got, _, _ = twin_frames("zoo_fallback", EXEC_GRAPH, write=False)
    assert not agreed and not same_bits(want[0][:, util.MOTION], got[0][:, util.MOTION])


# ---- GPU: the write route against the whole-type-batch route ---------------------------------------------------------------------------------------
BUILDS = {"strict_graph": (True, EXEC_GRAPH), "strict_stream": (True, EXEC_STREAM), "fast_graph": (False, EXEC_GRAPH), "fast_stream": (False, EXEC_STREAM)}


def resident_context(sim, strict=True, mode=EXEC_GRAPH, frames=2):
    ts = bp.CudaTimestepper(sim, strict_fp=strict, execution_mode=mode)
    ts.describe()
    for _ in range(frames):
        ts.solve_device_only(DT)
    return ts


@pytest.mark.gpu
@pytest.mark.parametrize("build", sorted(BUILDS))
def test_the_write_route_and_the_whole_type_batch_route_give_the_same_frames(libs, build):
    strict, mode = BUILDS[build]
    make, kw = SCENES["zoo_fallback"]
    scene = make()
    sim_w, sim_u = make_sim(scene, **kw), make_sim(scene, **kw)
    rng = np.random.default_rng(5)
    loc, joints = live_locations(sim_w)
    ts_w, ts_u = resident_context(sim_w, strict, mode), resident_context(sim_u, strict, mode)
    try:
        for _ in range(2):
            chosen = pick(rng, loc, joints)
            # the records a host would build: the device's current rows of those lanes with a new description
            records = changed(ts_w.read_constraints(chosen), rng)
            ts_w.write_constraints(chosen, records)
            ts_u.download_impulses()
            ts_u.download_prestep()
            apply_records(sim_u, chosen, records)
            named = {(int(b), int(t)) for b, t, _ in chosen.tolist()}
            for tb in sim_u.type_batches():
                if (tb.batch_index, tb.type_id) in named:
                    ts_u._check(ts_u._cuda.bepucuda_update_type_batch(ts_u._ctx, tb.batch_index, tb.type_batch_index, tb.prestep.ctypes.data,
                                                                      tb.accumulated_impulses.ctypes.data))
            ts_w.solve_device_only(DT)
            ts_u.solve_device_only(DT)
        ts_w.solve_device_only(DT)
        ts_u.solve_device_only(DT)
        assert same_state(state(ts_w, sim_w), state(ts_u, sim_u))
    finally:
        ts_w.close()
        ts_u.close()


# ---- GPU: semantics -------------------------------------------------------------------------------------------------------------------------------
def small_scene():
    return scenes.merge(scenes.shape_pile(600, seed=3, nonconvex_fraction=0.3), scenes.joint_zoo(300, per_type=6, seed=4), scenes.ragdolls(6, seed=5, motor="servo"))


def joint_locations(sim, n, rng):
    loc, joints = live_locations(sim)
    return loc[rng.choice(np.flatnonzero(joints), size=n, replace=False)]


def prestep_words(records):
    return [r[PRESTEP:PRESTEP + bp.type_info(int(r[0]))[1]] for r in records]


@pytest.mark.gpu
def test_the_last_write_to_a_constraint_wins_within_and_across_calls(libs):
    sim = make_sim(small_scene())
    rng = np.random.default_rng(1)
    ts = resident_context(sim)
    try:
        loc = joint_locations(sim, 40, rng)
        now = ts.read_constraints(loc)
        a, b, c = changed(now, rng), changed(now, rng), changed(now, rng)
        # one call: every location twice, a then b; a second call: c for the first half
        ts.write_constraints(np.concatenate([loc, loc]), np.concatenate([a, b]))
        ts.write_constraints(loc[:20], c[:20])
        ts.solve_device_only(DT)
        got = ts.read_constraints(loc)  # joint prestep rows are not moved by a solve
        want = np.concatenate([c[:20], b[20:]])
        assert all(np.array_equal(x, y) for x, y in zip(prestep_words(got), prestep_words(want)))
    finally:
        ts.close()


@pytest.mark.gpu
@pytest.mark.parametrize("order", ["write_first", "upload_first"])
@pytest.mark.parametrize("upload", ["update_type_batch", "update_contacts"])
def test_a_write_wins_over_a_whole_type_batch_upload_of_the_same_frame(libs, upload, order):
    """Context A: the whole-batch upload carries the old rows and a write the new ones; context B: the whole-batch upload carries the new rows. The
    next frame is the same."""
    scene = small_scene()
    sims = [make_sim(scene), make_sim(scene)]
    rng = np.random.default_rng(2)
    ctxs = [resident_context(s) for s in sims]
    try:
        loc, joints = live_locations(sims[0])
        want_contacts = upload == "update_contacts"
        tb = next(t for t in sims[0].type_batches() if bool(contact_count(t.type_id)) == want_contacts and t.constraint_count > 8)
        i = rng.choice(tb.constraint_count, size=5, replace=False)
        chosen = np.stack([np.full(5, tb.batch_index), np.full(5, tb.type_id), i], axis=1).astype(np.int32)
        for ts, sim in zip(ctxs, sims):
            ts.download_impulses()
            ts.download_prestep()
        records = changed(records_of(sims[0], chosen), rng)
        apply_records(sims[1], chosen, records)
        features = {}
        if want_contacts:
            features = initial_features(sims[0], np.random.default_rng(3))
            for ts in ctxs:
                ts.set_contact_features(features)

        def whole(ts, sim):
            if want_contacts:
                ts.update_contacts({(tb.batch_index, tb.type_batch_index): features[(tb.batch_index, tb.type_batch_index)]})
            else:
                t = next(x for x in sim.type_batches() if (x.batch_index, x.type_batch_index) == (tb.batch_index, tb.type_batch_index))
                ts._check(ts._cuda.bepucuda_update_type_batch(ts._ctx, t.batch_index, t.type_batch_index, t.prestep.ctypes.data, t.accumulated_impulses.ctypes.data))

        if order == "write_first":
            ctxs[0].write_constraints(chosen, records)
            whole(ctxs[0], sims[0])
        else:
            whole(ctxs[0], sims[0])
            ctxs[0].write_constraints(chosen, records)
        whole(ctxs[1], sims[1])
        for ts in ctxs:
            ts.solve_device_only(DT)
        assert same_state(state(ctxs[0], sims[0]), state(ctxs[1], sims[1]))
    finally:
        for ts in ctxs:
            ts.close()


@pytest.mark.gpu
def test_a_pending_write_is_seen_after_the_solve_only_and_a_describe_drops_it(libs):
    sim = make_sim(small_scene())
    rng = np.random.default_rng(3)
    ts = bp.CudaTimestepper(sim, strict_fp=True)
    try:
        ts.describe()
        loc = joint_locations(sim, 30, rng)
        before = ts.read_constraints(loc)
        new = changed(before, rng)
        ts.write_constraints(loc, new)  # right after the describe, before the first solve
        assert np.array_equal(ts.read_constraints(loc), before), "pending until the solve"
        ts.solve_device_only(DT)
        got = ts.read_constraints(loc)
        assert all(np.array_equal(x, y) for x, y in zip(prestep_words(got), prestep_words(new)))
        # a describe uploads the host's buffers and drops what is pending
        ts.write_constraints(loc, changed(before, rng))
        ts.describe()
        ts.solve_device_only(DT)
        assert all(np.array_equal(x, y) for x, y in zip(prestep_words(ts.read_constraints(loc)), prestep_words(records_of(sim, loc))))
    finally:
        ts.close()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", sorted(MODES))
def test_writing_back_what_was_read_changes_nothing_and_counts_its_bytes(libs, mode):
    scene = small_scene()
    sims = [make_sim(scene), make_sim(scene)]
    ctxs = [resident_context(s, mode=MODES[mode]) for s in sims]
    try:
        loc, _ = live_locations(sims[0])
        loc = loc[np.random.default_rng(4).choice(len(loc), size=500, replace=False)]
        captures = [ts.timings().graph_captures for ts in ctxs]
        records = ctxs[0].read_constraints(loc)
        ctxs[0].write_constraints(np.concatenate([loc, loc[:50]]), np.concatenate([records, records[:50]]))  # 50 duplicates: 500 distinct
        for ts in ctxs:
            ts.solve_device_only(DT)
        t = [ts.timings() for ts in ctxs]
        assert [x.graph_captures for x in t] == captures
        assert t[0].h2d_bytes - t[1].h2d_bytes == 500 * WRITE_BYTES + 4 * sum(bp.type_info(int(r[0]))[1] for r in records)
        for ts in ctxs:
            ts.solve_device_only(DT)
        assert same_state(state(ctxs[0], sims[0]), state(ctxs[1], sims[1]))
    finally:
        for ts in ctxs:
            ts.close()


@pytest.mark.gpu
def test_every_contact_of_the_100k_body_pile_in_one_call(libs):
    # one substep: no incremental depth update moves the written rows before they are read back
    sim = make_sim(scenes.shape_pile(100_000, seed=5), substeps=1, velocity_iterations=2)
    ts = resident_context(sim, frames=1)
    try:
        loc = sim.constraint_locations()
        assert len(loc) > 300_000
        new = changed(ts.read_constraints(loc), np.random.default_rng(6))
        ts.write_constraints(loc, new)
        ts.solve_device_only(DT)
        got = ts.read_constraints(loc)
        assert np.array_equal(got[:, 0], new[:, 0])
        assert np.array_equal(got[:, PRESTEP:53], new[:, PRESTEP:53])
    finally:
        ts.close()


# ---- GPU: errors ----------------------------------------------------------------------------------------------------------------------------------
def raw_write(ts, locations, records, n=None):
    loc = np.ascontiguousarray(locations, dtype=np.int32).reshape(-1, 4)
    rec = np.ascontiguousarray(records, dtype=np.int32).reshape(-1, 64)
    return ts._cuda.bepucuda_write_constraints(ts._ctx, len(loc) if n is None else n, loc.ctypes.data if loc.size else None, rec.ctypes.data if rec.size else None)


@pytest.mark.gpu
def test_errors_queue_nothing(libs):
    scene = scenes.merge(scenes.shape_pile(600, seed=3), scenes.joint_zoo(200, per_type=6, seed=4))
    sims = [make_sim(scene, fallback_batch_threshold=3, holes=True), make_sim(scene, fallback_batch_threshold=3, holes=True)]
    ctxs = [bp.CudaTimestepper(s, strict_fp=True) for s in sims]
    try:
        ts, sim = ctxs[0], sims[0]
        good_loc, _ = live_locations(sim)
        good_loc = with_set(good_loc[:: max(1, len(good_loc) // 64)])
        good = changed(records_of(sim, good_loc[:, 1:]), np.random.default_rng(7))
        assert raw_write(ts, good_loc, good) == ERR_BAD_STATE  # before end_constraints
        for c in ctxs:
            c.describe()
            c.solve_device_only(DT)
        ts._check(ts._cuda.bepucuda_begin_constraints(ts._ctx, sim.bundle_width, sim.batch_count))
        assert raw_write(ts, good_loc, good) == ERR_BAD_STATE  # between begin and end
        for c in ctxs:
            c.describe()
        tb = sim.type_batches()[0]
        present = {(t.batch_index, t.type_id) for t in sim.type_batches()}
        missing_type = next(t for t in range(64) if bp.type_info(t) and (tb.batch_index, t) not in present)
        hole = next([t.batch_index, t.type_id, int(i)] for t in sim.type_batches() if t.batch_index >= 3
                    for i in range(t.constraint_count) if t.body_references[i // sim.bundle_width, 0, i % sim.bundle_width] < 0)
        bad = {"set": [1, tb.batch_index, tb.type_id, 0], "negative_batch": [0, -1, tb.type_id, 0], "batch_out_of_range": [0, sim.batch_count, tb.type_id, 0],
               "type_without_type_batch": [0, tb.batch_index, missing_type, 0], "type_out_of_range": [0, tb.batch_index, 64, 0],
               "index_at_count": [0, tb.batch_index, tb.type_id, tb.constraint_count], "negative_index": [0, tb.batch_index, tb.type_id, -1],
               "hole": [0] + hole}
        for name, location in bad.items():
            rec = np.zeros((1, 64), dtype=np.int32)
            rec[0, 0] = location[2]
            assert raw_write(ts, np.concatenate([good_loc, [location]]), np.concatenate([good, rec])) == ERR_INVALID_ARGUMENT, name
        wrong = good.copy()
        wrong[-1, 0] = (wrong[-1, 0] + 1) % 64
        assert raw_write(ts, good_loc, wrong) == ERR_INVALID_ARGUMENT  # word 0 is not the location's type id
        assert ts._cuda.bepucuda_write_constraints(ts._ctx, 1, None, good.ctypes.data) == ERR_INVALID_ARGUMENT
        assert ts._cuda.bepucuda_write_constraints(ts._ctx, 1, good_loc.ctypes.data, None) == ERR_INVALID_ARGUMENT
        assert raw_write(ts, good_loc, good, n=-1) == ERR_INVALID_ARGUMENT
        assert ts._cuda.bepucuda_write_constraints(ts._ctx, 0, None, None) == 0
        for c in ctxs:
            c.solve_device_only(DT)
        assert same_state(state(ctxs[0], sims[0]), state(ctxs[1], sims[1]))
    finally:
        for c in ctxs:
            c.close()


@pytest.mark.gpu
def test_peer_mode_is_refused(libs):
    """A rank holds its constraints compacted, so host locations do not address them (ranks as contexts of one process on one device)."""
    sim = util.make_sim(scenes.shape_pile(400, seed=4), substeps=2, velocity_iterations=1)
    solvers = [sharding.ShardedSolver(sim, r, 2, 0, strict_fp=True) for r in range(2)]
    try:
        for s in solvers:
            s.export_handles()
        for s in solvers:
            s.import_contexts(solvers)
        for s in solvers:
            s.describe()
        tb = sim.type_batches()[0]
        loc = np.array([[0, tb.batch_index, tb.type_id, 0]], dtype=np.int32)
        rec = np.zeros((1, 64), dtype=np.int32)
        rec[0, 0] = tb.type_id
        s = solvers[0]
        assert s._cuda.bepucuda_write_constraints(s._ctx, 1, loc.ctypes.data, rec.ctypes.data) == ERR_BAD_STATE
    finally:
        for s in solvers:
            s.close()
