"""bepucuda_read_constraints: records of listed constraints read straight from the device rows (include/bepucuda.h), the state behind
NarrowPhase.TryExtractSolverContactData and Solver.EnumerateAccumulatedImpulses on the resident path.
CPU part: the planner's inverse slot map (csrc/bepu_topology.cpp) against its forward map, through the topology shim (tests/planner.py).
GPU part: after resident frames with device-side redistribution, every record equals the host buffers after the full downloads, word for word; subsets
come back in the order given; the call changes nothing; and each error leaves the output untouched."""
import numpy as np
import pytest

import bepuphysics2_b200 as bp
from bepuphysics2_b200 import scenes, sharding
from bepuphysics2_b200.native import ERR_BAD_STATE, ERR_INVALID_ARGUMENT, EXEC_GRAPH, EXEC_STREAM
from tests import planner, util
from tests.planner import constraints_of, inverse_of, plan, sim_sources
from tests.resident import initial_features, narrow_phase_like_update, push_bodies

DT = 1.0 / 60.0
CONVEX = {t for t in planner.CONTACT_TYPES if "Normal.X" in planner.TYPE_LAYOUTS[t]["prestep_rows"]}  # one normal per manifold
NONCONVEX = planner.CONTACT_TYPES - CONVEX


# ---- CPU: the inverse slot map -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["mixed_w8", "fallback_stress_w4", "holes_w16"])
def test_inverse_map_sends_every_fallback_constraint_to_its_slot_and_holes_nowhere(libs, case):
    scene, W, threshold = {"mixed_w8": (lambda: scenes.merge(scenes.shape_pile(1200, seed=3, nonconvex_fraction=0.3), scenes.joint_zoo(400, per_type=8, seed=4)), 8, 6),
                           "fallback_stress_w4": (lambda: scenes.fallback_stress(3000, hubs=6, seed=7), 4, 4),
                           "holes_w16": (lambda: scenes.merge(scenes.shape_pile(800, seed=5), scenes.joint_zoo(300, per_type=6, seed=6)), 16, 3)}[case]
    sim = util.make_sim(scene(), bundle_width=W, fallback_batch_threshold=threshold)
    holes = util.punch_fallback_holes(sim) if case == "holes_w16" else 0
    sources = sim_sources(sim)
    p = plan(sources, W, threshold, sim.batch_count, sim.body_count)
    assert p.fallback_levels > 0
    source_tb, offsets, inverse = inverse_of(p)
    # the forward maps: (device type batch, slot) -> source constraint
    forward = {}
    for tb in range(len(p.tbs)):
        for slot, c in enumerate(constraints_of(p, sources, tb)):
            if c >= 0:
                forward[(int(p.tbs[tb, 3]), int(c))] = (tb, slot)
    seen_holes = 0
    for s, (batch, _, type_id, count, refs) in enumerate(sources):
        if batch < threshold:
            assert offsets[s] == -1 and p.tbs[source_tb[s], 3] == s and p.tbs[source_tb[s], 4] == -1, "a synchronized source is one identity-mapped type batch"
            continue
        assert source_tb[s] == -1 and offsets[s] >= 0
        for i in range(count):
            tb, slot = inverse[offsets[s] + i]
            hole = refs[i // W, 0, i % W] < 0
            if hole:
                seen_holes += 1
                assert (tb, slot) == (-1, -1), "a hole maps to no slot"
            else:
                assert forward[(s, i)] == (tb, slot), "source %d constraint %d" % (s, i)
                assert constraints_of(p, sources, tb)[slot] == i and p.tbs[tb, 3] == s
    assert seen_holes >= holes  # punched holes, and any the scene has itself
    assert len(inverse) == sum(s[3] for s in sources if s[0] >= threshold)


# ---- GPU ---------------------------------------------------------------------------------------------------------------------------------
def expected_records(sim, locations):
    """The records the host's own buffers give (after download_impulses / download_prestep): what bepucuda_read_constraints must return."""
    tbs = {(tb.batch_index, tb.type_id): tb for tb in sim.type_batches()}
    W = sim.bundle_width
    out = np.zeros((len(locations), 64), dtype=np.int32)
    for k, (batch, type_id, i) in enumerate(np.asarray(locations).reshape(-1, 3)):
        tb = tbs[(int(batch), int(type_id))]
        b, lane = i // W, i % W
        out[k, 0] = type_id
        refs = tb.body_references[b, :, lane]
        if refs[0] < 0:  # a hole of the fallback batch
            continue
        out[k, 1] = 1
        out[k, 2:6] = -1
        out[k, 2:2 + tb.bodies] = refs
        out[k, 6:6 + tb.impulse_rows] = tb.accumulated_impulses[b, :, lane].view(np.int32)
        out[k, 18:18 + tb.prestep_rows] = tb.prestep[b, :, lane].view(np.int32)
    return out


def resident(scene, frames=3, bundle_width=8, fallback_batch_threshold=64, mode=EXEC_GRAPH, strict=True, holes=False, seed=77, substeps=3, velocity_iterations=2):
    """A described timestepper after `frames` resident frames: narrow-phase-like updates with random feature ids, so that redistribution and the
    incremental depth updates have moved the device rows away from the host's. Returns (simulation, timestepper)."""
    sim = util.make_sim(scene, bundle_width=bundle_width, fallback_batch_threshold=fallback_batch_threshold, substeps=substeps, velocity_iterations=velocity_iterations)
    if holes:
        assert util.punch_fallback_holes(sim) > 0
    rng = np.random.default_rng(seed)
    ts = bp.CudaTimestepper(sim, strict_fp=strict, execution_mode=mode)
    ts.register_host_buffers()
    ts.describe()
    features = initial_features(sim, rng)
    ts.set_contact_features(features)
    for frame in range(frames):
        if frame > 0:
            new = narrow_phase_like_update(sim, features, rng)
            push_bodies(sim, frame)
            ts.upload_body_motion()
            ts.update_contacts(new)
            features.update(new)
        ts.solve_device_only(DT)
    return sim, ts


def check_all_locations(sim, ts):
    locations = sim.constraint_locations()
    got = ts.read_constraints(locations)
    ts.download_impulses()
    ts.download_prestep()
    want = expected_records(sim, locations)
    assert got.shape == (len(locations), 64)
    bad = np.flatnonzero((got != want).any(axis=1))
    assert bad.size == 0, "%d of %d records differ, first %s: got %s want %s" % (bad.size, len(got), locations[bad[0]], got[bad[0]], want[bad[0]])
    return got


SCENES = {
    "convex_pile": (lambda: scenes.shape_pile(3000, seed=31), {}),
    "nonconvex_pile": (lambda: scenes.shape_pile(3000, seed=32, nonconvex_fraction=0.6), {}),
    "ragdolls": (lambda: scenes.ragdolls(40, seed=5), {}),
    "zoo_fallback": (lambda: scenes.merge(scenes.shape_pile(1500, seed=41, nonconvex_fraction=0.4), scenes.joint_zoo(600, per_type=20, seed=42),
                                          scenes.ragdolls(10, seed=43, motor="motor"), scenes.ragdolls(10, seed=44, motor="servo")),
                     dict(fallback_batch_threshold=6, holes=True)),
    "pile_width4": (lambda: scenes.shape_pile(2000, seed=33, nonconvex_fraction=0.3), dict(bundle_width=4)),
    "pile_width16": (lambda: scenes.shape_pile(2000, seed=34, nonconvex_fraction=0.3), dict(bundle_width=16)),
}
BUILDS = {"strict_graph": (True, EXEC_GRAPH), "fast_stream": (False, EXEC_STREAM), "strict_stream": (True, EXEC_STREAM), "fast_graph": (False, EXEC_GRAPH)}


@pytest.mark.gpu
@pytest.mark.parametrize("build", sorted(BUILDS))
@pytest.mark.parametrize("case", sorted(SCENES))
def test_every_record_equals_the_full_downloads(libs, case, build):
    make, kw = SCENES[case]
    strict, mode = BUILDS[build]
    sim, ts = resident(make(), strict=strict, mode=mode, **kw)
    try:
        got = check_all_locations(sim, ts)
        types = set(int(t) for t in got[:, 0])
        if case == "convex_pile":
            assert CONVEX <= types
        if case == "nonconvex_pile":
            assert NONCONVEX <= types
        if case == "zoo_fallback":
            assert len(types) == 44, sorted(types)
            assert ts.timings().fallback_level_count > 0
            holes = got[:, 1] == 0
            assert holes.any() and not got[holes, 2:].any()
    finally:
        ts.close()


@pytest.mark.gpu
def test_every_manifold_of_the_100k_body_pile_in_one_call(libs):
    sim, ts = resident(scenes.shape_pile(100_000, seed=5), frames=2, substeps=4, velocity_iterations=2)
    try:
        got = check_all_locations(sim, ts)
        assert len(got) > 300_000
    finally:
        ts.close()


@pytest.mark.gpu
def test_a_subset_in_random_order_with_duplicates_comes_back_in_that_order(libs):
    make, kw = SCENES["zoo_fallback"]
    sim, ts = resident(make(), **kw)
    try:
        everything = sim.constraint_locations()
        rng = np.random.default_rng(9)
        pick = rng.integers(0, len(everything), size=777)
        pick[100:120] = pick[0]  # duplicates
        subset = everything[pick]
        full = ts.read_constraints(everything)
        got = ts.read_constraints(subset)
        assert np.array_equal(got, full[pick])
        assert np.array_equal(ts.read_constraints(subset[:1]), full[pick[:1]])
        assert ts.read_constraints(np.zeros((0, 3), dtype=np.int32)).shape == (0, 64)
    finally:
        ts.close()


def _frame_after(read, mode):
    """Resident frames, then (optionally) a read of every constraint, then one more frame. Returns the state that frame leaves, and the graphs the
    context had captured before the read and after the frame."""
    sim, ts = resident(SCENES["zoo_fallback"][0](), mode=mode, **SCENES["zoo_fallback"][1])
    try:
        tbs = sim.type_batches()
        canary = [tb.accumulated_impulses.copy() for tb in tbs]
        for tb in tbs:
            tb.accumulated_impulses[:] = np.float32(-1234.5)  # the registered host impulse buffers: the read must not write them
        captures = [ts.timings().graph_captures]
        if read:
            ts.read_constraints(sim.constraint_locations())
        assert all((tb.accumulated_impulses == np.float32(-1234.5)).all() for tb in tbs), "the call wrote a host impulse buffer"
        ts.solve_device_only(DT)
        captures.append(ts.timings().graph_captures)
        for tb, c in zip(tbs, canary):
            tb.accumulated_impulses[:] = c
        ts.download_bodies()
        ts.download_impulses()
        return sim.bodies.copy(), [tb.accumulated_impulses.copy() for tb in tbs], captures
    finally:
        ts.close()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [EXEC_GRAPH, EXEC_STREAM], ids=["graph", "stream"])
def test_the_call_changes_nothing(libs, mode):
    bodies_a, impulses_a, captures_a = _frame_after(True, mode)
    bodies_b, impulses_b, captures_b = _frame_after(False, mode)
    assert np.array_equal(bodies_a.view(np.uint32), bodies_b.view(np.uint32))
    assert all(np.array_equal(a.view(np.uint32), b.view(np.uint32)) for a, b in zip(impulses_a, impulses_b))
    # the resident frames captured one graph in graph mode (none in stream mode); the frame after the read replays it
    assert captures_a == captures_b == ([1, 1] if mode == EXEC_GRAPH else [0, 0])


def _canary_records(n):
    return np.full((max(n, 1), 64), 0x5A5A5A5A, dtype=np.int32)


def _raw_read(ts, locations, n=None, records=None):
    loc = np.ascontiguousarray(locations, dtype=np.int32).reshape(-1, 4)
    count = len(loc) if n is None else n
    return ts._cuda.bepucuda_read_constraints(ts._ctx, count, loc.ctypes.data if loc.size else None, None if records is None else records.ctypes.data)


@pytest.mark.gpu
def test_errors_leave_the_records_untouched(libs):
    sim = util.make_sim(scenes.merge(scenes.shape_pile(600, seed=3), scenes.joint_zoo(200, per_type=6, seed=4)), substeps=2, velocity_iterations=1)
    ts = bp.CudaTimestepper(sim, strict_fp=True)
    try:
        good = np.array([[0, tb.batch_index, tb.type_id, tb.constraint_count - 1] for tb in sim.type_batches()], dtype=np.int32)
        records = _canary_records(len(good))
        assert _raw_read(ts, good, records=records) == ERR_BAD_STATE  # before end_constraints
        assert (records == 0x5A5A5A5A).all()
        ts.describe()
        ts.solve_device_only(DT)
        tb = sim.type_batches()[0]
        present = {(t.batch_index, t.type_id) for t in sim.type_batches()}
        missing_type = next(t for t in range(64) if bp.type_info(t) and (tb.batch_index, t) not in present)
        bad = {"set": [1, tb.batch_index, tb.type_id, 0], "negative_batch": [0, -1, tb.type_id, 0], "batch_out_of_range": [0, sim.batch_count, tb.type_id, 0],
               "type_without_type_batch": [0, tb.batch_index, missing_type, 0], "type_out_of_range": [0, tb.batch_index, 64, 0],
               "index_at_count": [0, tb.batch_index, tb.type_id, tb.constraint_count], "negative_index": [0, tb.batch_index, tb.type_id, -1]}
        for name, location in bad.items():
            locations = np.concatenate([good, np.array([location], dtype=np.int32)])
            records = _canary_records(len(locations))
            assert _raw_read(ts, locations, records=records) == ERR_INVALID_ARGUMENT, name
            assert (records == 0x5A5A5A5A).all(), name
        records = _canary_records(len(good))
        assert _raw_read(ts, good, records=None) == ERR_INVALID_ARGUMENT  # NULL output
        assert ts._cuda.bepucuda_read_constraints(ts._ctx, 1, None, records.ctypes.data) == ERR_INVALID_ARGUMENT  # NULL locations
        assert _raw_read(ts, good, n=-1, records=records) == ERR_INVALID_ARGUMENT
        assert ts._cuda.bepucuda_read_constraints(ts._ctx, 0, None, None) == 0
        assert (records == 0x5A5A5A5A).all()
        assert _raw_read(ts, good, records=records) == 0 and (records[:, 1] == 1).all()
    finally:
        ts.close()


@pytest.mark.gpu
def test_peer_mode_is_refused(libs):
    """A rank holds its constraints compacted, so host locations do not address them: BAD_STATE before any device work (ranks as contexts of one
    process on one device, as tests/test_sharding.py runs them)."""
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
        records = _canary_records(1)
        s = solvers[0]
        assert s._cuda.bepucuda_read_constraints(s._ctx, 1, loc.ctypes.data, records.ctypes.data) == ERR_BAD_STATE
        assert (records == 0x5A5A5A5A).all()
    finally:
        for s in solvers:
            s.close()
