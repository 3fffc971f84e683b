"""Body adds and removes on the device-resident state (bepucuda_add_bodies / bepucuda_remove_bodies). On the CPU: replay_body_removes in
bepu_topology.cpp against BodySet.RemoveAt applied step by step, its dry run, and the host mirror's Bodies.Remove with handles. On the GPU: a
resident twin that only forwards its changes, held to the oracle's host twin after every frame, and to a describing twin."""
import ctypes as C
import os

import numpy as np
import pytest

import bepuphysics2_b200 as bp
from bepuphysics2_b200 import _build, scenes, sharding
from bepuphysics2_b200.native import BODY_ACTIVITY_DTYPE, BODY_SHAPE_DTYPE, ERR_BAD_STATE, ERR_INVALID_ARGUMENT, EXEC_GRAPH, EXEC_STREAM, contact_count
from oracle import binding as ob
from tests import harness, util
from tests.resident import body_frame, lane_record, live_handles, projectile_prestep, remove_a_ragdoll

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "bepuphysics2_b200", "csrc")
DT = 1.0 / 60.0
KINEMATIC = 1 << 30
INDEX = (1 << 30) - 1


# ---- CPU: the composed replay against BodySet.RemoveAt step by step -------------------------------------------------------------------------------
def body_shim():
    cuda_include = os.path.join(os.path.dirname(os.path.dirname(_build.NVCC)), "include")
    dll = harness.load("body_change_shim", [os.path.join(ROOT, "tests", "topology", "body_change_shim.cpp"), os.path.join(CSRC, "bepu_topology.cpp")],
                       ["-O2", "-std=c++17", "-Wall", "-shared", "-fPIC", "-I", cuda_include], includes=[CSRC, os.path.join(ROOT, "include")])
    dll.body_removes.argtypes = [C.c_int32, C.c_int32, C.c_void_p, C.POINTER(C.c_int32), C.c_void_p]
    return dll


def replay(body_count, indices):
    """(code, final count, moved_to) of replay_body_removes; on a failure the outputs hold the sentinels they were given."""
    idx = np.ascontiguousarray(indices, dtype=np.int32)
    final = C.c_int32(-7)
    moved = np.full(max(len(idx), 1), -9, dtype=np.int32)
    rc = body_shim().body_removes(body_count, len(idx), idx.ctypes.data if len(idx) else None, C.byref(final), moved.ctypes.data)
    return rc, final.value, moved[:len(idx)]


def remove_at_step_by_step(records, indices):
    """BodySet.RemoveAt of each index in order on a copy of `records`; returns the records and, per final slot, the original index it holds."""
    records, at = list(records), list(range(len(records)))
    for i in indices:
        assert 0 <= i < len(at)
        last, last_record = at.pop(), records.pop()
        if i < len(at):
            at[i], records[i] = last, last_record
    return records, at


@pytest.mark.parametrize("seed", range(6))
def test_composed_moves_equal_remove_at_step_by_step(libs, seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 400))
    cases = [rng.integers(0, np.arange(n, max(n - 60, 0), -1)) for _ in range(4)]   # each entry within the count at that entry
    cases += [[n - 1], list(range(n - 1, -1, -1)), [0] * n, [n - 1, 0, 0, n - 4 if n > 4 else 0][:min(n, 4)]]  # last (no move), down to zero, duplicates
    for indices in cases:
        indices = [int(i) for i in indices]
        records = [("body", k) for k in range(n)]
        want_records, want_at = remove_at_step_by_step(records, indices)
        rc, final, moved = replay(n, indices)
        assert rc == 0 and final == n - len(indices) == len(want_at)
        # the composed moves applied in one step
        one_step = list(records[:final])
        for i, to in enumerate(moved):
            if to >= 0:
                assert to < final and final + i >= final
                one_step[to] = records[final + i]
        assert one_step == want_records
        # the index map: every survivor at or above the final count moved to the slot it holds after the sequence
        for i, to in enumerate(moved):
            assert (to >= 0) == ((final + i) in want_at)
            if to >= 0:
                assert want_at[to] == final + i
        assert len(set(int(t) for t in moved if t >= 0)) == int((moved >= 0).sum())


def test_the_dry_run_rejects_every_malformed_list(libs):
    shim = body_shim()
    final = C.c_int32(-7)
    moved = np.full(4, -9, dtype=np.int32)
    assert shim.body_removes(10, -1, None, C.byref(final), moved.ctypes.data) == ERR_INVALID_ARGUMENT
    assert shim.body_removes(10, 2, None, C.byref(final), moved.ctypes.data) == ERR_INVALID_ARGUMENT
    for bad in ([10], [-1], [3, 9], [9, 9], [0] * 11):
        rc, f, m = replay(10, bad)
        assert rc == ERR_INVALID_ARGUMENT, bad
        assert f == -7 and (m == -9).all()
    assert final.value == -7 and (moved == -9).all()
    rc, f, _ = replay(10, [])
    assert rc == 0 and f == 10


# ---- CPU: the mirror's Bodies.Remove --------------------------------------------------------------------------------------------------------------
def constraint_bodies(scene):
    """Per constraint handle of a freshly built scene: its body handles."""
    return [np.asarray(h, dtype=np.int32) for _, handles, _ in scene["constraints"] for h in handles]


def check_mirror(sim, bodies_of, dynamics_of):
    """Every live constraint references HandleToLocation of its bodies, kinematic bits kept; every body's record is its own; the constrained
    kinematics are the kinematic bodies live constraints reference."""
    handles = sim.body_handles
    assert len(set(handles.tolist())) == sim.body_count
    for index, h in enumerate(handles):
        assert sim.body_index(h) == index
        assert util.bits(sim.bodies[index]).tolist() == util.bits(dynamics_of[int(h)]).tolist()
    refs, batches = sim.constraint_references()
    kinematic = set()
    for c in np.flatnonzero(batches >= 0):
        want = np.array([sim.body_index(h) for h in bodies_of[c]], dtype=np.int32)
        got = refs[c, :len(want)]
        assert np.array_equal(got & INDEX, want), c
        is_kin = np.array([not sim.bodies[i, 16:23].any() for i in want])
        assert np.array_equal((got & KINEMATIC) != 0, is_kin), c
        kinematic |= set(want[is_kin].tolist())
    assert sorted(sim.constrained_kinematics.tolist()) == sorted(kinematic)


@pytest.mark.parametrize("case", ["zoo_w8_fallback", "ragdolls_w4"])
def test_the_mirror_keeps_references_and_kinematics_on_their_bodies(libs, case):
    scene = scenes.merge(scenes.joint_zoo(300, per_type=8, seed=4, kinematic_fraction=0.1), scenes.shape_pile(300, seed=5)) if case.startswith("zoo") else \
        scenes.ragdolls(12, seed=3)
    sim = util.make_sim(scene, bundle_width=8 if "w8" in case else 4, fallback_batch_threshold=4 if "fallback" in case else 64)
    assert np.array_equal(sim.body_handles, np.arange(sim.body_count))  # handles are indices until a body is removed
    bodies_of = constraint_bodies(scene)
    dynamics_of = {int(h): sim.bodies[i].copy() for i, h in enumerate(sim.body_handles)}
    kin_before = len(sim.constrained_kinematics)
    rng = np.random.default_rng(2)
    for step in range(6):
        doomed = rng.choice(sim.body_handles, size=max(1, sim.body_count // 20), replace=False)
        sim.remove_bodies(doomed)
        for h in doomed:
            assert sim.body_index(int(h)) == -1
            del dynamics_of[int(h)]
        check_mirror(sim, bodies_of, dynamics_of)
        new = scenes.make_bodies(rng.normal(size=(3, 3)), inverse_mass=[1, 1, 1], inverse_inertia=[[1, 0, 1, 0, 0, 1]] * 3)
        first = sim.add_bodies(new)
        added = sim.body_handles[-3:]
        assert added[0] == first
        for h, r in zip(added, new):
            dynamics_of[int(h)] = r
        check_mirror(sim, bodies_of, dynamics_of)
    if case.startswith("zoo"):
        assert kin_before > 0
    # the pool hands out the last freed handle first
    h = int(sim.body_handles[-1])
    sim.remove_bodies([h])
    assert sim.add_bodies(scenes.make_bodies([[0, 0, 0]])) == h


# ---- GPU: the resident twin against the oracle's host twin ----------------------------------------------------------------------------------------
ZOO = lambda: scenes.merge(scenes.shape_pile(1200, seed=41, nonconvex_fraction=0.4), scenes.joint_zoo(500, per_type=16, seed=42), scenes.ragdolls(8, seed=43))
GPU_SCENES = {
    "pile_w4": (lambda: scenes.shape_pile(2000, seed=33, nonconvex_fraction=0.3), dict(bundle_width=4)),
    "pile_w16": (lambda: scenes.shape_pile(2000, seed=34, nonconvex_fraction=0.3), dict(bundle_width=16)),
    "zoo_fallback_w8": (ZOO, dict(bundle_width=8, fallback_batch_threshold=6)),
}
MODES = {"graph": EXEC_GRAPH, "stream": EXEC_STREAM}


def make_twin(scene, bundle_width=8, fallback_batch_threshold=64):
    return util.make_sim(scene, bundle_width=bundle_width, fallback_batch_threshold=fallback_batch_threshold, substeps=3, velocity_iterations=2)


def same_bodies(a, b):
    return util.bits(a.bodies[:, util.MEANINGFUL]).tolist() == util.bits(b.bodies[:, util.MEANINGFUL]).tolist()


def resident_twins(make, kw, mode, frames=4, spawn=12, removes=8, forward=True, strict=True, prepare=None, frame_hook=None):
    """Frames of a resident twin next to the oracle's host twin: both make the same body and constraint changes before every frame but the first;
    the resident twin forwards them with bepuhost_cuda_change. Returns whether the bodies agreed bit for bit after every frame, the timings of each
    frame, the two simulations, and the resident twin's records of every live constraint."""
    scene = make()
    host, dev = make_twin(scene, **kw), make_twin(scene, **kw)
    extra = prepare(host) if prepare else None
    if prepare:
        prepare(dev)
    rng_h, rng_d = np.random.default_rng(7), np.random.default_rng(7)
    ts = bp.CudaTimestepper(dev, strict_fp=strict, execution_mode=mode)
    agreed, timings = True, []
    try:
        ts.describe()
        for frame in range(frames):
            if frame > 0:
                if frame_hook:
                    frame_hook(host, frame, extra)
                    frame_hook(dev, frame, extra)
                body_frame(host, rng_h, spawn, removes, extra)
                adds = body_frame(dev, rng_d, spawn, removes, extra)
                if forward:
                    ts.change(np.zeros((adds, 4), dtype=np.int32))
            ob.solve(host, DT)
            ts.solve_device_only(DT)
            if forward:
                ts.download_bodies()
                agreed = agreed and same_bodies(host, dev)
            else:
                ts.download_body_motion()
                n = min(host.body_count, dev.body_count)
                agreed = agreed and util.bits(host.bodies[:n, util.MOTION]).tolist() == util.bits(dev.bodies[:n, util.MOTION]).tolist()
            timings.append(ts.timings())
        live = live_handles(dev)
        records = ts.read_constraints(np.array([(0,) + dev.constraint_location(int(h)) for h in live], dtype=np.int32)) if forward else None
    finally:
        ts.close()
    return agreed, timings, host, dev, records


def check_records(host, dev, records):
    live = live_handles(dev)
    assert np.array_equal(live, live_handles(host))
    assert np.array_equal(records, np.stack([lane_record(host, int(h)) for h in live]))


@pytest.mark.gpu
@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("case", sorted(GPU_SCENES))
def test_the_resident_twin_stays_on_the_oracle_through_body_adds_and_removes(libs, case, mode):
    make, kw = GPU_SCENES[case]
    agreed, timings, host, dev, records = resident_twins(make, kw, MODES[mode])
    assert agreed
    check_records(host, dev, records)
    assert not np.array_equal(dev.body_handles, np.arange(dev.body_count))  # bodies moved
    if mode == "graph":
        captures = [t.graph_captures for t in timings]
        assert all(b - a == 1 for a, b in zip(captures, captures[1:]))
    if "fallback" in case:
        assert any(tb.batch_index >= 6 for tb in dev.type_batches())


@pytest.mark.gpu
def test_whole_ragdolls_are_removed_on_the_resident_path(libs):
    make = lambda: scenes.merge(scenes.ragdolls(24, seed=5, motor="motor"), scenes.ragdolls(24, seed=6, motor="servo"))
    agreed, _, host, dev, records = resident_twins(make, dict(bundle_width=8), EXEC_GRAPH, spawn=4, removes=2, frame_hook=remove_a_ragdoll)
    assert agreed
    check_records(host, dev, records)


def add_kinematic_mover(sim):
    """A kinematic body appended last, joined to body 5 by a contact, so that the first removal moves it."""
    mover = scenes.make_bodies([[0, 4, 0]], linear=[[0.5, 0, 0]])
    h = sim.add_bodies(mover)
    sim.add_constraints(4, np.array([[5, h]], dtype=np.int32), projectile_prestep(np.random.default_rng(1), 1))
    return h


@pytest.mark.gpu
@pytest.mark.parametrize("mode", sorted(MODES))
def test_a_constrained_kinematic_moved_by_a_removal(libs, mode):
    seen = []

    def hook(sim, frame, mover):
        if frame == 1:
            sim.remove_bodies([int(sim.body_handles[2])])  # the last body, the mover, takes index 2
            assert sim.body_index(mover) == 2 and 2 in sim.constrained_kinematics.tolist()
            seen.append(True)

    agreed, _, host, dev, records = resident_twins(lambda: scenes.shape_pile(1500, seed=8), dict(bundle_width=8), MODES[mode], spawn=0, removes=3,
                                                   prepare=add_kinematic_mover, frame_hook=hook)
    assert agreed and seen
    check_records(host, dev, records)


@pytest.mark.gpu
def test_without_the_change_calls_the_twins_differ(libs):
    make, kw = GPU_SCENES["pile_w4"]
    agreed, _, _, _, _ = resident_twins(make, kw, EXEC_GRAPH, frames=3, spawn=0, removes=8, forward=False)
    assert not agreed


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["pile_w16", "zoo_fallback_w8"])
def test_the_fast_build_resident_twin_matches_a_describing_twin(libs, case):
    """Fast build: the resident twin against a device twin that downloads everything and describes again after its changes, byte for byte; and
    find_sleepable_islands on both after the changes."""
    make, kw = GPU_SCENES[case]
    scene = make()
    a, b = make_twin(scene, **kw), make_twin(scene, **kw)
    rng_a, rng_b = np.random.default_rng(3), np.random.default_rng(3)
    ta, tb = bp.CudaTimestepper(a, strict_fp=False), bp.CudaTimestepper(b, strict_fp=False)
    try:
        ta.describe()
        tb.describe()
        for frame in range(4):
            if frame > 0:
                body_frame(a, rng_a, 10, 6)
                ta.describe()
                adds = body_frame(b, rng_b, 10, 6)
                tb.change(np.zeros((adds, 4), dtype=np.int32))
            ta.solve(DT, download=True)
            ta.download_prestep()
            tb.solve_device_only(DT)
            tb.download_bodies()
            assert same_bodies(a, b), frame
        live = live_handles(b)
        got = tb.read_constraints(np.array([(0,) + b.constraint_location(int(h)) for h in live], dtype=np.int32))
        assert np.array_equal(got, np.stack([lane_record(a, int(h)) for h in live]))
        activities = np.zeros(b.body_count, dtype=BODY_ACTIVITY_DTYPE)
        activities["sleep_candidate"] = np.arange(b.body_count) % 3 != 0
        ia, ib = ta.find_sleepable_islands(activities), tb.find_sleepable_islands(activities)
        for x, y in zip(ia[:3], ib[:3]):
            assert np.array_equal(x, y)
    finally:
        ta.close()
        tb.close()


def random_shapes(rng, n):
    s = np.zeros(n, dtype=BODY_SHAPE_DTYPE)
    s["type"] = rng.choice([0, 1, 2, 4], size=n)
    s["a"], s["b"], s["c"] = rng.uniform(0.1, 1, size=(3, n)).astype(np.float32)
    s["maximum_speculative_margin"] = np.float32(0.2)
    return s


@pytest.mark.gpu
def test_per_body_arrays_follow_the_bodies(libs):
    """Shapes and accelerations move with removed bodies and take appended records on adds: bounding boxes and a solve equal a describing twin
    that sets both arrays again. NULL arrays on an add leave the arrays at the old count: BEPUCUDA_ERR_BAD_STATE until they are set again."""
    rng = np.random.default_rng(5)
    scene = {"bodies": scenes.shape_pile(600, seed=2)["bodies"], "constraints": []}
    a, b = make_twin(scene), make_twin(scene)
    shapes = {int(h): s for h, s in zip(a.body_handles, random_shapes(rng, a.body_count))}
    acc = {int(h): r for h, r in zip(a.body_handles, rng.normal(size=(a.body_count, 8)).astype(np.float32))}
    ta, tb = bp.CudaTimestepper(a, strict_fp=True), bp.CudaTimestepper(b, strict_fp=True)
    arrays = lambda sim: (np.array([shapes[int(h)] for h in sim.body_handles], dtype=BODY_SHAPE_DTYPE), np.stack([acc[int(h)] for h in sim.body_handles]))
    try:
        for ts, sim in ((ta, a), (tb, b)):
            ts.describe()
            s, c = arrays(sim)
            ts.set_body_shapes(s)
            ts.set_body_accelerations(c)
        for frame in range(3):
            doomed = rng.choice(a.body_count, size=25, replace=False)
            handles = [int(a.body_handles[i]) for i in doomed]
            order = []
            for h in handles:  # each index read just before its removal, as the reference's RemoveAt sees it
                order.append(a.body_index(h))
                a.remove_bodies([h])
                b.remove_bodies([h])
            ta.remove_bodies(order)
            new = a.bodies[rng.integers(0, a.body_count, size=40)].copy()
            new[:, 4] += 10
            first = a.add_bodies(new)
            b.add_bodies(new)
            added = a.body_handles[-40:]
            s_new, c_new = random_shapes(rng, 40), rng.normal(size=(40, 8)).astype(np.float32)
            for h, s, c in zip(added, s_new, c_new):
                shapes[int(h)], acc[int(h)] = s, c
            ta.add_bodies(new, s_new, c_new)
            tb.describe()
            s, c = arrays(b)
            tb.set_body_shapes(s)
            tb.set_body_accelerations(c)
            act_a = np.zeros(a.body_count, dtype=BODY_ACTIVITY_DTYPE)
            act_b = act_a.copy()
            assert np.array_equal(util.bits(ta.predict_bounding_boxes(DT, act_a)), util.bits(tb.predict_bounding_boxes(DT, act_b)))
            for ts in (ta, tb):
                ts.solve_device_only(DT)
                ts.download_bodies()
            assert same_bodies(a, b), frame
        a.add_bodies(new[:2])
        ta.add_bodies(new[:2])
        for call in (lambda: ta.solve_device_only(DT), lambda: ta.predict_bounding_boxes(DT, np.zeros(a.body_count, dtype=BODY_ACTIVITY_DTYPE))):
            with pytest.raises(bp.BepuCudaError) as e:
                call()
            assert e.value.code == ERR_BAD_STATE
    finally:
        ta.close()
        tb.close()


@pytest.mark.gpu
def test_growth_keeps_every_record(libs):
    """Adds past twice the initial body count, in several calls: every record downloads as it was given, and the frames stay on the oracle."""
    make = lambda: scenes.shape_pile(300, seed=6)
    agreed, _, host, dev, records = resident_twins(make, dict(bundle_width=8), EXEC_GRAPH, frames=5, spawn=120, removes=5)
    assert agreed and dev.body_count > 2 * 300
    check_records(host, dev, records)


def unconstrained(sim, rng, n):
    """n random bodies no constraint references, as handles."""
    refs, batches = sim.constraint_references()
    used = set((refs[batches >= 0] & INDEX)[refs[batches >= 0] >= 0].tolist())
    free = [i for i in range(sim.body_count) if i not in used]
    return [int(sim.body_handles[i]) for i in rng.choice(free, size=n, replace=False)]


@pytest.mark.gpu
def test_bus_bytes_and_captures_follow_the_entries(libs):
    scene = scenes.shape_pile(1500, seed=12)
    sim = make_twin(scene)
    rng = np.random.default_rng(8)
    ts = bp.CudaTimestepper(sim, strict_fp=True)
    try:
        ts.describe()
        ts.solve_device_only(DT)
        captures = ts.timings().graph_captures
        sim.remove_bodies(unconstrained(sim, rng, 7))
        ts.change()
        ts.solve_device_only(DT)
        t = ts.timings()
        assert t.h2d_bytes == 7 * 4 and t.graph_captures == captures + 1
        sim.add_bodies(scenes.make_bodies(rng.normal(size=(5, 3)), inverse_mass=np.ones(5), inverse_inertia=[[1, 0, 1, 0, 0, 1]] * 5))
        ts.change()
        ts.solve_device_only(DT)
        t = ts.timings()
        assert t.h2d_bytes == 5 * 128 and t.graph_captures == captures + 2
        ts.solve_device_only(DT)
        assert ts.timings().graph_captures == captures + 2
    finally:
        ts.close()


@pytest.mark.gpu
def test_refused_calls_change_nothing(libs):
    """A removal of a body a live constraint references, an index out of range and a call with pending rows are refused: the body records and the
    read-back rows stay byte-identical, nothing is captured, and the next solve matches a twin that never made them."""
    scene = scenes.shape_pile(800, seed=21)
    sims = [make_twin(scene, bundle_width=8, fallback_batch_threshold=4) for _ in range(2)]
    solvers = [bp.CudaTimestepper(s, strict_fp=True) for s in sims]
    try:
        for ts in solvers:
            ts.describe()
            ts.solve_device_only(DT)
        sim, ts = sims[1], solvers[1]
        live = live_handles(sim)
        locs = np.array([(0,) + sim.constraint_location(int(h)) for h in live], dtype=np.int32)
        refs, _ = sim.constraint_references()
        referenced = int(refs[live[0], 0] & INDEX)
        ts.download_bodies()
        before_bodies, before_rows = sim.bodies.copy(), ts.read_constraints(locs)
        captures = ts.timings().graph_captures
        for call in (lambda: ts.remove_bodies([referenced]), lambda: ts.remove_bodies([sim.body_count]), lambda: ts.remove_bodies([sim.body_count - 1, sim.body_count - 1]),
                     lambda: ts.remove_bodies([-1])):
            with pytest.raises(bp.BepuCudaError) as e:
                call()
            assert e.value.code == ERR_INVALID_ARGUMENT
        assert ts._cuda.bepucuda_remove_bodies(ts._ctx, -1, None) == ERR_INVALID_ARGUMENT
        assert ts._cuda.bepucuda_add_bodies(ts._ctx, None, 1, None, None) == ERR_INVALID_ARGUMENT
        ts.write_constraints(locs[:1], before_rows[:1])  # pending rows
        solvers[0].write_constraints(locs[:1], before_rows[:1])
        for call in (lambda: ts.remove_bodies([0]), lambda: ts.add_bodies(sim.bodies[:1])):
            with pytest.raises(bp.BepuCudaError) as e:
                call()
            assert e.value.code == ERR_BAD_STATE
        ts.download_bodies()
        assert util.bits(sim.bodies).tolist() == util.bits(before_bodies).tolist()
        assert np.array_equal(ts.read_constraints(locs), before_rows)
        for ts_ in solvers:
            ts_.solve_device_only(DT)
            ts_.download_bodies()
        assert ts.timings().graph_captures == captures
        assert same_bodies(sims[0], sims[1])
    finally:
        for ts_ in solvers:
            ts_.close()


@pytest.mark.gpu
def test_peer_mode_is_refused(libs):
    sim = util.make_sim(scenes.shape_pile(400, seed=4), substeps=2, velocity_iterations=1)
    solvers = [sharding.ShardedSolver(sim, r, 2, 0, strict_fp=True) for r in range(2)]
    try:
        for s in solvers:
            s.export_handles()
        for s in solvers:
            s.import_contexts(solvers)
        for s in solvers:
            s.describe()
        s = solvers[0]
        idx = np.array([0], dtype=np.int32)
        assert s._cuda.bepucuda_remove_bodies(s._ctx, 1, idx.ctypes.data) == ERR_BAD_STATE
        assert s._cuda.bepucuda_add_bodies(s._ctx, sim.bodies[:1].ctypes.data, 1, None, None) == ERR_BAD_STATE
    finally:
        for s in solvers:
            s.close()
