"""Constraint adds and removes on the device-resident rows (bepucuda_add_constraints / bepucuda_remove_constraints). On the CPU: the replay of
Solver.Add / Solver.Remove in bepu_topology.cpp against the host mirror's own Solver.Remove, step by step, and its dry run. On the GPU: a resident twin
that only forwards its changes, held to the oracle's host twin after every frame."""
import ctypes as C
import os

import numpy as np
import pytest

import bepuphysics2_b200 as bp
from bepuphysics2_b200 import _build, scenes, sharding
from bepuphysics2_b200.native import ERR_BAD_STATE, ERR_INVALID_ARGUMENT, EXEC_GRAPH, EXEC_STREAM, contact_count
from oracle import binding as ob
from tests import harness, planner, util
from tests.resident import lane_record, live_handles, type_batch_at

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "bepuphysics2_b200", "csrc")
DT = 1.0 / 60.0
CLEAR, NEW = -1, -2  # kLaneClear / kLaneNew


# ---- the mirror ---------------------------------------------------------------------------------------------------------------------------------
def write_impulses(sim, handle, record):
    b, t, i = sim.constraint_location(handle)
    tb = type_batch_at(sim, b, t)
    W = sim.bundle_width
    tb.accumulated_impulses[i // W, :, i % W] = record[6:6 + tb.impulse_rows].view(np.float32)


def remove_run(sim, handles):
    """Solver.Remove of each handle in order; returns the locations the removes consumed, int32[n, 4]."""
    locs = []
    for h in handles:
        locs.append((0,) + sim.constraint_location(int(h)))
        sim.remove_constraints([int(h)])
    return np.array(locs, dtype=np.int32).reshape(-1, 4)


def add_run(sim, adds):
    """Solver.Add of (type id, body handles, prestep) in order; returns (handles, locations int32[n, 4], records int32[n, 64])."""
    handles, locs, records = [], [], []
    for type_id, bodies, prestep in adds:
        h = sim.add_constraints(type_id, np.asarray(bodies).reshape(1, -1), np.asarray(prestep).reshape(1, -1))
        handles.append(h)
        locs.append((0,) + sim.constraint_location(h))
        records.append(lane_record(sim, h))
    return handles, np.array(locs, dtype=np.int32).reshape(-1, 4), np.array(records, dtype=np.int32).reshape(-1, 64)


def random_changes(sim, rng, fraction, original):
    """A frame of collision detection: a fraction of the live constraints removed and re-added (same bodies and description, so the pair keeps
    its meaning), as remove + add runs. Returns (removed handles, adds)."""
    live = live_handles(sim)
    pick = rng.choice(live, size=max(1, int(len(live) * fraction)), replace=False)
    adds = [original[int(h)] for h in pick]
    return pick, adds


def scene_original(scene):
    """Per handle of a freshly built scene: (type id, body handles, prestep) in add order."""
    out = []
    for type_id, handles, prestep in scene["constraints"]:
        for h, p in zip(handles, prestep):
            out.append((type_id, np.asarray(h, dtype=np.int32), np.asarray(p, dtype=np.float32)))
    return out


# ---- CPU: the replay against the mirror --------------------------------------------------------------------------------------------------------
def change_shim():
    cuda_include = os.path.join(os.path.dirname(os.path.dirname(_build.NVCC)), "include")
    dll = harness.load("change_shim", [os.path.join(ROOT, "tests", "topology", "change_shim.cpp"), os.path.join(CSRC, "bepu_topology.cpp")],
                       ["-O2", "-std=c++17", "-Wall", "-shared", "-fPIC", "-I", cuda_include], includes=[CSRC, os.path.join(ROOT, "include")])
    vp, i32 = C.c_void_p, C.c_int32
    dll.change_create.restype = vp
    dll.change_create.argtypes = [i32, vp, vp, vp, i32]
    dll.change_destroy.argtypes = [vp]
    dll.change_apply.argtypes = [vp, i32, i32, i32, i32, i32, vp, vp, i32, i32, vp, C.POINTER(i32), vp]
    dll.change_sources.argtypes = [vp, vp, C.POINTER(i32)]
    return dll


class Replay:
    """A ChangeState of the shim, created from a simulation's type batches, with the lane each handle sits in tracked through the lane copies."""

    def __init__(self, sim):
        self.dll, self.sim = change_shim(), sim
        self.W, self.threshold = sim.bundle_width, sim.fallback_batch_threshold
        tbs = sim.type_batches()
        meta = np.array([[tb.batch_index, tb.type_batch_index, tb.type_id, tb.constraint_count] for tb in tbs], dtype=np.int32).reshape(-1, 4)
        refs = [np.ascontiguousarray(tb.body_references if tb.batch_index >= self.threshold else np.zeros(0), dtype=np.int32).reshape(-1) for tb in tbs]
        words = np.array([r.size for r in refs], dtype=np.int32)
        ptrs = (C.c_void_p * max(len(refs), 1))(*[r.ctypes.data for r in refs])
        self.state = self.dll.change_create(len(tbs), meta.ctypes.data, ptrs, words.ctypes.data, sim.batch_count)
        keys = {(tb.batch_index, tb.type_id): s for s, tb in enumerate(tbs)}
        self.lanes = {}
        for h in live_handles(sim):
            b, t, i = sim.constraint_location(int(h))
            self.lanes[(keys[(b, t)], i)] = int(h)

    def close(self):
        self.dll.change_destroy(self.state)

    def sources(self):
        meta = np.zeros((4096, 4), dtype=np.int32)
        bc = C.c_int32()
        n = self.dll.change_sources(self.state, meta.ctypes.data, C.byref(bc))
        return meta[:n], bc.value

    def apply(self, remove, locations, records=None, new_handles=(), compose=False):
        """Returns (code, copies); on success the tracked lanes follow the copies (in order, or from the state before the call when composed)."""
        loc = np.ascontiguousarray(locations, dtype=np.int32).reshape(-1, 4)
        rec = None if records is None else np.ascontiguousarray(records, dtype=np.int32).reshape(-1, 64)
        cap = 64 * (len(loc) + 1) * self.W
        copies = np.zeros((cap, 4), dtype=np.int32)
        remap = np.full(4096, -1, dtype=np.int32)
        n = C.c_int32()
        rc = self.dll.change_apply(self.state, int(remove), self.W, self.threshold, self.sim.body_count, len(loc), loc.ctypes.data, None if rec is None else rec.ctypes.data,
                                   int(compose), cap, copies.ctypes.data, C.byref(n), remap.ctypes.data)
        if rc != 0:
            return rc, None
        copies = copies[:n.value]
        before = dict(self.lanes)
        for d_s, d_i, s_s, s_i in copies:
            src = before if compose else self.lanes
            self.lanes[(d_s, d_i)] = None if s_s == CLEAR else new_handles[s_i] if s_s == NEW else src.get((s_s, s_i))
        self.lanes = {(int(remap[s]), i): h for (s, i), h in self.lanes.items() if remap[s] >= 0}
        return 0, copies

    def check(self):
        """Counts, (batch, type batch, type id) keys and the lane of every live handle agree with the mirror."""
        meta, batch_count = self.sources()
        want = sorted((tb.batch_index, tb.type_batch_index, tb.type_id, tb.constraint_count) for tb in self.sim.type_batches())
        assert sorted(map(tuple, meta.tolist())) == want
        assert batch_count == self.sim.batch_count
        keys = {(int(m[0]), int(m[2])): s for s, m in enumerate(meta)}
        for h in live_handles(self.sim):
            b, t, i = self.sim.constraint_location(int(h))
            assert self.lanes.get((keys[(b, t)], i)) == int(h), "handle %d at %s" % (h, (b, t, i))


def check_mirror(sim, original):
    """Solver.Remove's invariants in the mirror: every live handle's lane holds its own body references and description, synchronized type batches
    have no hole below ConstraintCount, and fallback holes are -1."""
    W = sim.bundle_width
    live = live_handles(sim)
    occupied = set()
    for h in live:
        b, t, i = sim.constraint_location(int(h))
        tb = type_batch_at(sim, b, t)
        assert i < tb.constraint_count and (b, t, i) not in occupied
        occupied.add((b, t, i))
        type_id, bodies, prestep = original[int(h)]
        assert type_id == t
        assert np.array_equal(tb.body_references[i // W, :, i % W] & ((1 << 30) - 1), bodies)
        assert util.bits(tb.prestep[i // W, :, i % W]).tolist() == util.bits(prestep).tolist()
    for tb in sim.type_batches():
        assert tb.constraint_count > 0
        for i in range(tb.constraint_count):
            held = (tb.batch_index, tb.type_id, i) in occupied
            if tb.batch_index < sim.fallback_batch_threshold:
                assert held
            else:
                assert held == (tb.body_references[i // W, 0, i % W] >= 0)
    assert len(live) == len(occupied)


CPU_CASES = {
    "pile_w4": (lambda: scenes.shape_pile(300, seed=3, nonconvex_fraction=0.3), 4, 64),
    "pile_w8_fallback": (lambda: scenes.shape_pile(300, seed=4), 8, 3),
    "stress_w4": (lambda: scenes.fallback_stress(600, hubs=4, seed=7), 4, 4),
    "zoo_w16": (lambda: scenes.merge(scenes.joint_zoo(200, per_type=6, seed=4), scenes.ragdolls(4, seed=5)), 16, 5),
}


def _replay_removes(sim, replay, handles, compose, seen, original):
    meta, batches = replay.sources()
    locs = remove_run(sim, handles)
    rc, copies = replay.apply(True, locs, compose=compose)
    assert rc == 0
    fallback = meta[:, 0] >= replay.threshold
    seen["sync_swap"] |= any(c[2] >= 0 and not fallback[c[2]] for c in copies)
    seen["fallback_clear"] |= bool((locs[:, 1] >= replay.threshold).any())
    seen["bundle_pull"] |= any(c[2] >= 0 and fallback[c[2]] and c[1] // replay.W != c[3] // replay.W for c in copies)
    after = {(int(m[0]), int(m[2])): int(m[3]) for m in replay.sources()[0]}
    for m in meta[fallback]:
        n = after.get((int(m[0]), int(m[2])), 0)
        seen["bundle_shrink"] |= (n + replay.W - 1) // replay.W < (int(m[3]) + replay.W - 1) // replay.W
    seen["type_batch_gone"] |= len(after) < len(meta)
    seen["batch_dropped"] |= replay.sources()[1] < batches
    replay.check()
    check_mirror(sim, original)


def _replay_adds(sim, replay, adds, compose, seen, original):
    meta, batches = replay.sources()
    handles, locs, records = add_run(sim, adds)
    original += adds
    rc, copies = replay.apply(False, locs, records, new_handles=handles, compose=compose)
    assert rc == 0 and len(copies) == len(handles)
    seen["new_type_batch"] |= any((int(l[1]), int(l[2])) not in {(int(m[0]), int(m[2])) for m in meta} for l in locs)
    seen["new_batch"] |= replay.sources()[1] > batches
    replay.check()
    check_mirror(sim, original)


@pytest.mark.parametrize("compose", [False, True])
@pytest.mark.parametrize("case", sorted(CPU_CASES))
def test_the_replay_follows_the_mirror_step_by_step(libs, case, compose):
    """Frames of random changes: even steps add the replacement pairs first and remove the old ones after, as the narrow phase does (the new pairs
    then find their bodies taken and go to higher or new batches), odd steps remove first; the last step removes the whole last batch and adds it
    back."""
    make, W, threshold = CPU_CASES[case]
    scene = make()
    sim = util.make_sim(scene, bundle_width=W, fallback_batch_threshold=threshold)
    original = scene_original(scene)
    rng = np.random.default_rng(len(case) + compose)
    replay = Replay(sim)
    seen = dict.fromkeys(["sync_swap", "fallback_clear", "bundle_pull", "bundle_shrink", "type_batch_gone", "batch_dropped", "new_type_batch", "new_batch"], False)
    try:
        replay.check()
        for step in range(12):
            removed, adds = random_changes(sim, rng, 0.08 if step % 3 else 0.3, original)
            rng.shuffle(adds)
            if step % 2 == 0:
                _replay_adds(sim, replay, adds, compose, seen, original)
                _replay_removes(sim, replay, removed, compose, seen, original)
            else:
                _replay_removes(sim, replay, removed, compose, seen, original)
                _replay_adds(sim, replay, adds, compose, seen, original)
        _, batches = sim.constraint_references()
        last = np.flatnonzero(batches == sim.batch_count - 1)
        adds = [original[int(h)] for h in last]
        _replay_removes(sim, replay, last, compose, seen, original)
        _replay_adds(sim, replay, adds, compose, seen, original)
    finally:
        replay.close()
    assert seen["sync_swap"] and seen["type_batch_gone"] and seen["batch_dropped"] and seen["new_type_batch"] and seen["new_batch"], seen
    if any(tb.batch_index >= threshold for tb in sim.type_batches()):
        assert seen["fallback_clear"] and seen["bundle_pull"] and seen["bundle_shrink"], seen


def test_a_run_that_empties_the_last_batch_drops_it_and_an_add_opens_it_again(libs):
    scene = scenes.shape_pile(200, seed=9)
    sim = util.make_sim(scene, bundle_width=8)
    original = scene_original(scene)
    replay = Replay(sim)
    try:
        last = sim.batch_count - 1
        _, batches = sim.constraint_references()
        doomed = np.flatnonzero(batches == last)
        rc, _ = replay.apply(True, remove_run(sim, doomed))
        assert rc == 0 and sim.batch_count == last
        replay.check()
        adds = [original[int(h)] for h in doomed]
        handles, locs, records = add_run(sim, adds)
        assert locs[:, 1].max() == last  # the pairs need that batch again
        assert replay.apply(False, locs, records, new_handles=handles)[0] == 0
        replay.check()
    finally:
        replay.close()


def test_the_dry_run_rejects_every_malformed_list_and_changes_nothing(libs):
    sim = util.make_sim(scenes.shape_pile(300, seed=4), bundle_width=8, fallback_batch_threshold=3)
    util.punch_fallback_holes(sim)
    replay = Replay(sim)
    try:
        tbs = sim.type_batches()
        sync = next(tb for tb in tbs if tb.batch_index == 0)
        fb = next(tb for tb in tbs if tb.batch_index >= 3)
        W = 8
        holes = [i for i in range(fb.constraint_count) if fb.body_references[i // W, 0, i % W] < 0]
        occupied = next(i for i in range(fb.constraint_count) if fb.body_references[i // W, 0, i % W] >= 0)
        h = int(live_handles(sim)[0])
        good = lane_record(sim, h)
        b, t, i = sim.constraint_location(h)

        def rec(type_id, refs=None):
            r = good.copy()
            r[0] = type_id
            if refs is not None:
                r[2:2 + len(refs)] = refs
            return r

        meta_before = replay.sources()
        bad_adds = [
            ((0, b, t, type_batch_at(sim, b, t).constraint_count + 1), rec(t)),  # synchronized add past the end
            ((0, b, t, 0), rec(t)),                                              # synchronized add over a constraint
            ((0, b, t, type_batch_at(sim, b, t).constraint_count), rec(t + 1 if t < 10 else 0)),  # word 0 differs
            ((0, b, t, type_batch_at(sim, b, t).constraint_count), rec(t, [sim.body_count])),     # body out of range
            ((0, sim.batch_count + 1, t, 0), rec(t)),                            # batch past the new one
            ((0, fb.batch_index, fb.type_id, occupied), rec(fb.type_id)),        # fallback lane in use
            ((1, b, t, type_batch_at(sim, b, t).constraint_count), rec(t)),      # not the active set
            ((0, 0, 63, 0), rec(63)),                                            # no such type
        ]
        for k, (loc, r) in enumerate(bad_adds):
            assert replay.apply(False, [loc], [r], new_handles=[-1])[0] == ERR_INVALID_ARGUMENT, loc
            if k == 0:
                continue  # after an add at the end, index ConstraintCount + 1 is the end
            # a bad entry after a good one: the good one is not committed either
            loc0 = (0, b, t, type_batch_at(sim, b, t).constraint_count)
            assert replay.apply(False, [loc0, loc], [rec(t), r], new_handles=[-1, -1])[0] == ERR_INVALID_ARGUMENT, loc
        bad_removes = [(0, sync.batch_index, sync.type_id, sync.constraint_count), (0, b, t, -1), (0, sim.batch_count, t, 0), (2, b, t, i)]
        bad_removes += [(0, fb.batch_index, fb.type_id, j) for j in holes[:2]]
        for loc in bad_removes:
            assert replay.apply(True, [loc])[0] == ERR_INVALID_ARGUMENT, loc
            assert replay.apply(True, [(0, b, t, i), loc])[0] == ERR_INVALID_ARGUMENT, loc
        # the same constraint twice: the second names a moved or missing lane only if it is past the end
        last = (0, sync.batch_index, sync.type_id, sync.constraint_count - 1)
        assert replay.apply(True, [last, last])[0] == ERR_INVALID_ARGUMENT
        after = replay.sources()
        assert np.array_equal(meta_before[0], after[0]) and meta_before[1] == after[1]
        replay.check()
        assert holes, "the scene's fallback batch has holes"
    finally:
        replay.close()


# ---- GPU: the resident twin against the oracle's host twin ---------------------------------------------------------------------------------------
ZOO = lambda: scenes.merge(scenes.shape_pile(1200, seed=41, nonconvex_fraction=0.4), scenes.joint_zoo(500, per_type=16, seed=42), scenes.ragdolls(8, seed=43))
GPU_SCENES = {
    "pile_w4": (lambda: scenes.shape_pile(2000, seed=33, nonconvex_fraction=0.3), dict(bundle_width=4)),
    "pile_w16": (lambda: scenes.shape_pile(2000, seed=34, nonconvex_fraction=0.3), dict(bundle_width=16)),
    "ragdolls_w8": (lambda: scenes.merge(scenes.ragdolls(24, seed=5, motor="motor"), scenes.ragdolls(24, seed=6, motor="servo")), dict(bundle_width=8)),
    "zoo_fallback_w8": (ZOO, dict(bundle_width=8, fallback_batch_threshold=6)),
}
MODES = {"graph": EXEC_GRAPH, "stream": EXEC_STREAM}


def make_twin(scene, bundle_width=8, fallback_batch_threshold=64):
    return util.make_sim(scene, bundle_width=bundle_width, fallback_batch_threshold=fallback_batch_threshold, substeps=3, velocity_iterations=2)


def change_frame(sim, rng, original, fraction, carried):
    """Removes and re-adds a fraction of the constraints of `sim`; a re-added constraint takes the impulses `carried(handle)` returns for the
    removed one (read before the remove) when that is not None. Returns the number of adds and removes."""
    removed, adds = random_changes(sim, rng, fraction, original)
    kept = [carried(int(h)) for h in removed]
    remove_run(sim, removed)
    handles, _, _ = add_run(sim, adds)
    original += adds
    for h, record in zip(handles, kept):
        if record is not None:
            write_impulses(sim, h, record)
    return len(adds), len(removed)


def resident_twins(case, mode, strict=True, frames=4, fraction=0.03, forward=True, seed=5):
    """Frames of a resident twin next to the oracle's host twin. Before every frame but the first both twins remove and re-add the same
    constraints; the host twin carries the removed constraints' impulses from its buffers, the resident twin from bepucuda_read_constraints, and
    forwards its changes with bepuhost_cuda_change. Returns whether the body motion agreed bit for bit after every frame, the timings of each frame,
    and the two simulations with the resident twin's records at every live handle."""
    make, kw = GPU_SCENES[case]
    scene = make()
    host, dev = make_twin(scene, **kw), make_twin(scene, **kw)
    orig_h, orig_d = scene_original(scene), scene_original(scene)
    rng_h, rng_d = np.random.default_rng(seed), np.random.default_rng(seed)
    ts = bp.CudaTimestepper(dev, strict_fp=strict, execution_mode=mode)
    agreed, timings = True, []
    try:
        ts.describe()
        for frame in range(frames):
            if frame > 0:
                change_frame(host, rng_h, orig_h, fraction, lambda h: lane_record(host, h))
                read = lambda h: ts.read_constraints([(0,) + dev.constraint_location(h)])[0]
                adds, _ = change_frame(dev, rng_d, orig_d, fraction, read)
                if forward:
                    ts.change(np.zeros((adds, 4), dtype=np.int32))
            ob.solve(host, DT)
            ts.solve_device_only(DT)
            ts.download_body_motion()
            timings.append(ts.timings())
            agreed = agreed and util.bits(host.bodies[:, util.MOTION]).tolist() == util.bits(dev.bodies[:, util.MOTION]).tolist()
        live = live_handles(dev)
        records = ts.read_constraints(np.array([(0,) + dev.constraint_location(int(h)) for h in live], dtype=np.int32)) if forward else None
    finally:
        ts.close()
    return agreed, timings, host, dev, records


@pytest.mark.gpu
@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("case", sorted(GPU_SCENES))
def test_the_resident_twin_stays_on_the_oracle_through_adds_and_removes(libs, case, mode):
    agreed, timings, host, dev, records = resident_twins(case, MODES[mode])
    assert agreed
    live = live_handles(dev)
    assert np.array_equal(live, live_handles(host))
    want = np.stack([lane_record(host, int(h)) for h in live])
    assert np.array_equal(records, want)
    captures = [t.graph_captures for t in timings]
    if mode == "graph":
        assert all(b - a == 1 for a, b in zip(captures, captures[1:]))
    if "fallback" in case:
        assert any(tb.batch_index >= 6 for tb in dev.type_batches())


@pytest.mark.gpu
def test_without_the_change_calls_the_twins_differ(libs):
    agreed, _, host, dev, _ = resident_twins("pile_w4", EXEC_GRAPH, frames=3, forward=False)
    assert not agreed


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["pile_w16", "zoo_fallback_w8"])
def test_the_fast_build_resident_twin_matches_a_describing_twin(libs, case):
    """Fast build: the resident twin against a device twin that downloads everything and describes again after its changes, byte for byte."""
    make, kw = GPU_SCENES[case]
    scene = make()
    a, b = make_twin(scene, **kw), make_twin(scene, **kw)
    orig_a, orig_b = scene_original(scene), scene_original(scene)
    rng_a, rng_b = np.random.default_rng(3), np.random.default_rng(3)
    ta, tb = bp.CudaTimestepper(a, strict_fp=False), bp.CudaTimestepper(b, strict_fp=False)
    try:
        ta.describe()
        tb.describe()
        for frame in range(4):
            if frame > 0:
                change_frame(a, rng_a, orig_a, 0.05, lambda h: lane_record(a, h))
                ta.describe()
                adds, _ = change_frame(b, rng_b, orig_b, 0.05, lambda h: tb.read_constraints([(0,) + b.constraint_location(h)])[0])
                tb.change(np.zeros((adds, 4), dtype=np.int32))
            ta.solve(DT, download=True)
            ta.download_prestep()
            tb.solve_device_only(DT)
            tb.download_body_motion()
            assert util.bits(a.bodies[:, util.MOTION]).tolist() == util.bits(b.bodies[:, util.MOTION]).tolist(), frame
        live = live_handles(b)
        got = tb.read_constraints(np.array([(0,) + b.constraint_location(int(h)) for h in live], dtype=np.int32))
        assert np.array_equal(got, np.stack([lane_record(a, int(h)) for h in live]))
    finally:
        ta.close()
        tb.close()


@pytest.mark.gpu
def test_bus_bytes_and_captures_follow_the_entries(libs):
    scene = scenes.shape_pile(1500, seed=12)
    sim = make_twin(scene, bundle_width=8, fallback_batch_threshold=4)
    original = scene_original(scene)
    rng = np.random.default_rng(8)
    ts = bp.CudaTimestepper(sim, strict_fp=True)
    try:
        ts.describe()
        ts.solve_device_only(DT)
        captures = ts.timings().graph_captures
        replay = Replay(sim)
        removed, adds = random_changes(sim, rng, 0.05, original)
        locs = remove_run(sim, removed)
        _, copies = replay.apply(True, locs, compose=True)
        replay.close()
        ts.remove_constraints(locs)
        ts.solve_device_only(DT)
        t = ts.timings()
        assert t.h2d_bytes == 16 * len(copies) and t.graph_captures == captures + 1
        handles, locs, records = add_run(sim, adds)
        ts.add_constraints(locs, records, np.zeros((len(adds), 4), dtype=np.int32))
        ts.solve_device_only(DT)
        t2 = ts.timings()
        assert t2.h2d_bytes == len(adds) * (16 + 256 + 16) and t2.graph_captures == captures + 2
    finally:
        ts.close()


@pytest.mark.gpu
def test_refused_calls_change_nothing(libs):
    """A pending-rows call and malformed lists are refused before any device work: the next solve matches a twin that never made them."""
    scene = scenes.shape_pile(800, seed=21)
    sims = [make_twin(scene, bundle_width=8, fallback_batch_threshold=4) for _ in range(2)]
    solvers = [bp.CudaTimestepper(s, strict_fp=True) for s in sims]
    try:
        for ts in solvers:
            ts.describe()
            ts.solve_device_only(DT)
        sim, ts = sims[1], solvers[1]
        h = int(live_handles(sim)[0])
        loc = np.array([(0,) + sim.constraint_location(h)], dtype=np.int32)
        rec = lane_record(sim, h)[None]
        ts.write_constraints(loc, rec)  # pending rows
        with pytest.raises(bp.BepuCudaError) as e:
            ts.remove_constraints(loc)
        assert e.value.code == ERR_BAD_STATE
        solvers[0].write_constraints(loc, rec)
        for ts_ in solvers:
            ts_.solve_device_only(DT)
        bad = rec.copy()
        bad[0, 0] = 63
        for call in (lambda: ts.add_constraints(loc, rec, np.zeros((1, 4), dtype=np.int32)),  # index over a constraint
                     lambda: ts.add_constraints(loc, bad, np.zeros((1, 4), dtype=np.int32)),
                     lambda: ts.remove_constraints(np.array([[0, 0, loc[0, 2], 1 << 20]], dtype=np.int32)),
                     lambda: ts.remove_constraints(loc, kinematics=[sim.body_count])):
            with pytest.raises(bp.BepuCudaError) as e:
                call()
            assert e.value.code == ERR_INVALID_ARGUMENT
        assert ts._cuda.bepucuda_remove_constraints(ts._ctx, -1, None, None, 0) == ERR_INVALID_ARGUMENT
        for ts_ in solvers:
            ts_.solve_device_only(DT)
            ts_.download_bodies()
        assert util.bits(sims[0].bodies[:, util.MEANINGFUL]).tolist() == util.bits(sims[1].bodies[:, util.MEANINGFUL]).tolist()
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
        tb = sim.type_batches()[0]
        loc = np.array([[0, tb.batch_index, tb.type_id, 0]], dtype=np.int32)
        s = solvers[0]
        assert s._cuda.bepucuda_remove_constraints(s._ctx, 1, loc.ctypes.data, None, 0) == ERR_BAD_STATE
    finally:
        for s in solvers:
            s.close()


# ---- GPU: contacts with feature ids through the change calls and bepucuda_update_contacts -----------------------------------------------------
CONVEX_GROWABLE = {0, 1, 2, 4, 5, 6}  # convex manifolds that can take one more contact (type id + 1)


def grown_prestep(type_id, prestep):
    """The description of the same manifold with one more contact, a copy of its last one (a contact-count change makes a new type id)."""
    depth = planner.depth_rows(type_id)
    assert planner.depth_rows(type_id + 1) == depth + [depth[-1] + 4]
    end = depth[-1] + 1
    return np.concatenate([prestep[:end], prestep[end - 4:end], prestep[end:]]).astype(np.float32)


def redistribute(old_type, old_impulses, old_ids, new_type, new_ids):
    """NarrowPhase.RedistributeImpulses across a type change: a penetration impulse follows its feature id, the unmatched new contacts share what
    the unmatched old ones held; the friction and twist rows are carried in order."""
    old_pen, new_pen = planner.penetration_rows(old_type), planner.penetration_rows(new_type)
    out = np.zeros(len(planner.TYPE_LAYOUTS[new_type]["impulse_rows"]), dtype=np.float32)
    rest_old = [r for r in range(len(old_impulses)) if r not in old_pen]
    rest_new = [r for r in range(len(out)) if r not in new_pen]
    out[rest_new] = old_impulses[rest_old]
    left, unmatched = np.float32(0), []
    for k, fid in enumerate(old_ids):
        if fid not in new_ids:
            left += old_impulses[old_pen[k]]
    for k, fid in enumerate(new_ids):
        if fid in old_ids:
            out[new_pen[k]] = old_impulses[old_pen[list(old_ids).index(fid)]]
        else:
            unmatched.append(k)
    for k in unmatched:
        out[new_pen[k]] = left / np.float32(len(unmatched))
    return out


def lane_handles(sim):
    """{(batch, type id, index): handle} of every live constraint."""
    return {sim.constraint_location(int(h)): int(h) for h in live_handles(sim)}


def feature_arrays(sim, feat):
    """Per contact type batch, int32[ConstraintCount, contacts] of the handles' feature ids (0 in holes)."""
    where = lane_handles(sim)
    out = {}
    for tb in sim.type_batches():
        n = contact_count(tb.type_id)
        if n:
            a = np.zeros((tb.constraint_count, n), dtype=np.int32)
            for i in range(tb.constraint_count):
                h = where.get((tb.batch_index, tb.type_id, i))
                if h is not None:
                    a[i] = feat[h]
            out[(tb.batch_index, tb.type_batch_index)] = a
    return out


def contact_changes(sim, rng, feat, fraction, read):
    """One frame's collision detection on a contact pile: a fraction of the manifolds is replaced, with the adds made before the removes (as the
    narrow phase does). A replaced manifold either keeps its type (its impulses and feature ids carried) or gains a contact (new type id: its
    impulses redistributed by feature id, one new id). read(handle): the constraint's 64-word record, read before the host changes anything. Returns the feature ids of the adds in order, padded to 4, and how many manifolds changed type."""
    pick = rng.choice(live_handles(sim), size=max(1, int(len(live_handles(sim)) * fraction)), replace=False)
    grow = rng.random(len(pick)) < 0.3
    fresh = rng.integers(1 << 21, 1 << 22, size=len(pick), dtype=np.int32)
    add_ids, changed = [], [0]

    def readd(handles, grow_mask, fresh_ids):
        plans = []
        for h, g, f in zip(handles, grow_mask, fresh_ids):
            rec = read(int(h))
            t = int(rec[0])
            tb = type_batch_at(sim, *sim.constraint_location(int(h))[:2])
            bodies = rec[2:2 + tb.bodies] & ((1 << 30) - 1)
            prestep = rec[18:18 + tb.prestep_rows].view(np.float32)
            impulses = rec[6:6 + tb.impulse_rows].view(np.float32)
            if g and t in CONVEX_GROWABLE:
                ids = np.append(feat[int(h)], f).astype(np.int32)
                plans.append((t + 1, bodies, grown_prestep(t, prestep), redistribute(t, impulses, feat[int(h)], t + 1, ids), ids))
                changed[0] += 1
            else:
                plans.append((t, bodies, prestep.copy(), impulses.copy(), feat[int(h)].copy()))
        for t, bodies, prestep, impulses, ids in plans:
            new = sim.add_constraints(t, bodies.reshape(1, -1), prestep.reshape(1, -1))
            b, _, i = sim.constraint_location(new)
            tb = type_batch_at(sim, b, t)
            tb.accumulated_impulses[i // sim.bundle_width, :, i % sim.bundle_width] = impulses
            feat[new] = ids
            add_ids.append(np.pad(ids, (0, 4 - len(ids))))

    readd(pick, grow, fresh)
    for h in pick:
        sim.remove_constraints([int(h)])
        del feat[int(h)]
    return np.array(add_ids, dtype=np.int32).reshape(-1, 4), changed[0]


def reopen_last_batch(sim, feat, read):
    """Removes every constraint of the last batch (the batch goes) and adds them back with their impulses and feature ids (their pairs need the
    batch again). Returns the feature ids of the adds, padded to 4."""
    _, batches = sim.constraint_references()
    last = np.flatnonzero(batches == sim.batch_count - 1)
    kept = [(read(int(h)), feat[int(h)].copy()) for h in last]
    count = sim.batch_count
    for h in last:
        sim.remove_constraints([int(h)])
        del feat[int(h)]
    assert sim.batch_count < count
    add_ids = []
    for rec, ids in kept:
        t = int(rec[0])
        info = planner.TYPE_LAYOUTS[t]
        new = sim.add_constraints(t, (rec[2:2 + info["bodies"]] & ((1 << 30) - 1)).reshape(1, -1), rec[18:18 + len(info["prestep_rows"])].view(np.float32).reshape(1, -1))
        write_impulses(sim, new, rec)
        feat[new] = ids
        add_ids.append(np.pad(ids, (0, 4 - len(ids))))
    assert sim.batch_count == count, "the last batch's pairs need it again"
    return np.array(add_ids, dtype=np.int32).reshape(-1, 4)


def narrow_phase_ids(sim, feat, rng):
    """New feature ids for every live contact (a fifth replaced) and fresh depths for every contact type batch; returns (old, new) arrays."""
    old = feature_arrays(sim, feat)
    for h in sorted(feat):
        ids = feat[h].copy()
        change = rng.random(ids.shape) < 0.2
        ids[change] = rng.integers(1 << 20, 1 << 21, size=int(change.sum()), dtype=np.int32)
        feat[h] = ids
    for tb in sim.type_batches():
        for r in planner.depth_rows(tb.type_id):
            tb.prestep[:, r, :] = rng.uniform(-0.02, 0.05, size=tb.prestep[:, r, :].shape).astype(np.float32)
    return old, feature_arrays(sim, feat)


CONTACT_CASES = {"w8": dict(bundle_width=8), "w4_fallback": dict(bundle_width=4, fallback_batch_threshold=5)}


@pytest.mark.gpu
@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("case", sorted(CONTACT_CASES))
def test_contact_changes_with_feature_ids_stay_on_the_oracle(libs, case, mode):
    """The resident frame with changes: solve, the change calls (with the adds' feature ids), update_contacts with new ids and depths, solve. The
    host twin redistributes on the oracle. Type-changing contacts, carried impulses, and a frame that drops and re-opens the last batch; bodies
    bit for bit after every frame, every live constraint word for word at the end."""
    kw = CONTACT_CASES[case]
    scene = scenes.shape_pile(2000, seed=51)
    host, dev = make_twin(scene, **kw), make_twin(scene, **kw)
    rng0 = np.random.default_rng(4)
    feat_h = {int(h): rng0.integers(0, 1 << 20, size=contact_count(host.constraint_location(int(h))[1]), dtype=np.int32) for h in live_handles(host)}
    feat_d = {h: ids.copy() for h, ids in feat_h.items()}
    rng_h, rng_d = np.random.default_rng(9), np.random.default_rng(9)
    ts = bp.CudaTimestepper(dev, strict_fp=True, execution_mode=MODES[mode])
    grown = 0
    try:
        ts.describe()
        ts.set_contact_features(feature_arrays(dev, feat_d))
        for frame in range(4):
            if frame > 0:
                read_h = lambda h: lane_record(host, h)
                read_d = lambda h: ts.read_constraints([(0,) + dev.constraint_location(h)])[0]
                contact_changes(host, rng_h, feat_h, 0.03, read_h)
                ids, changed = contact_changes(dev, rng_d, feat_d, 0.03, read_d)
                assert (ids != 0).any()
                grown += changed
                ts.change(ids)
                if frame == 2:  # device reads need the host's locations forwarded first
                    reopen_last_batch(host, feat_h, read_h)
                    ts.change(reopen_last_batch(dev, feat_d, read_d))
                old_h, new_h = narrow_phase_ids(host, feat_h, rng_h)
                _, new_d = narrow_phase_ids(dev, feat_d, rng_d)
                for tb in host.type_batches():
                    key = (tb.batch_index, tb.type_batch_index)
                    if key in new_h:
                        ob.update_contact_impulses(tb, old_h[key], new_h[key])
                ts.update_contacts(new_d)
            ob.solve(host, DT)
            ts.solve_device_only(DT)
            ts.download_body_motion()
            assert util.bits(host.bodies[:, util.MOTION]).tolist() == util.bits(dev.bodies[:, util.MOTION]).tolist(), "frame %d" % frame
        live = live_handles(dev)
        assert np.array_equal(live, live_handles(host))
        got = ts.read_constraints(np.array([(0,) + dev.constraint_location(int(h)) for h in live], dtype=np.int32))
        assert np.array_equal(got, np.stack([lane_record(host, int(h)) for h in live]))
    finally:
        ts.close()
    assert grown > 0
    if "fallback" in case:
        assert any(tb.batch_index >= 5 for tb in dev.type_batches())
