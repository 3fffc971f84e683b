"""Sleepable islands (bepucuda_find_sleepable_islands): the search of IslandSleeper.CollectIsland with the SleepPredicate (IslandSleeper.cs:L85-223)
over every island of the constraint graph the device holds.

CPU: a restatement of CollectIsland (tests/islands/collect_island.cpp, the checker) partitions the bodies exactly as scipy's connected components do on the same graph (random graphs
of 1- to 4-body types, kinematic bridges, empty fallback lanes, unconstrained bodies, a 131 072-body chain), and its sleepable verdict matches
closed forms. GPU: the device result is IDENTICAL to the checker's (labels, roots, counts) on those graphs and on the benchmark scenes, calls repeat
exactly, the call leaves the next solve byte for byte as it was, the error cases are reported, and the round count stays logarithmic on the chain."""
import ctypes as C

import numpy as np
import pytest
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components

import bepuphysics2_b200 as bp
from bepuphysics2_b200 import native, scenes, sharding
from tests import island_checker, util

DT = 1.0 / 60.0
# type ids by bodies per constraint: a one-body convex contact, a two-body convex contact, AreaConstraint (3), VolumeConstraint (4)
TYPE_OF_BODIES = {1: 0, 2: 4, 3: 36, 4: 32}


def _bodies(n, kinematic=()):
    rng = np.random.default_rng(n)
    inv_mass = np.ones(n, dtype=np.float32)
    inv_inertia = np.tile(np.array([1, 0, 1, 0, 0, 1], dtype=np.float32), (n, 1))
    kinematic = np.asarray(kinematic, dtype=np.int64)
    inv_mass[kinematic] = 0.0
    inv_inertia[kinematic] = 0.0
    return scenes.make_bodies(rng.uniform(-10, 10, size=(n, 3)), inverse_mass=inv_mass, inverse_inertia=inv_inertia)


def _constraints(handles_by_count, seed=0):
    """Scene constraints from {bodies per constraint: int32[m, k] handles}; prestep values are arbitrary (the search reads only references)."""
    rng = np.random.default_rng(seed)
    out = []
    for k, h in sorted(handles_by_count.items()):
        if len(h):
            t = TYPE_OF_BODIES[k]
            out.append((t, np.asarray(h, dtype=np.int32).reshape(-1, k), rng.uniform(0.1, 1.0, size=(len(h), bp.type_info(t)[1])).astype(np.float32)))
    return out


def random_graph(seed, n=3000, per_kind=(400, 900, 150, 100), kinematic_count=12):
    """Bodies 0 .. n-1 with a few kinematics; constraints of 1, 2, 3 and 4 bodies on distinct random bodies (slot 0 always dynamic); about a
    tenth of the bodies stay unconstrained."""
    rng = np.random.default_rng(seed)
    kinematic = rng.choice(np.arange(1, n), size=kinematic_count, replace=False)
    dynamic = np.setdiff1d(np.arange(n), kinematic)
    reach = rng.choice(n, size=int(n * 0.9), replace=False)
    handles = {}
    for k, m in zip((1, 2, 3, 4), per_kind):
        rows = []
        while len(rows) < m:
            row = [int(rng.choice(dynamic))] + [int(x) for x in rng.choice(reach, size=k - 1)]
            if len(set(row)) == k:
                rows.append(row)
        handles[k] = np.array(rows, dtype=np.int32).reshape(-1, k)
    return {"bodies": _bodies(n, kinematic), "constraints": _constraints(handles, seed)}


def chain(n, seed=0):
    """One chain through all n bodies, visited in a random order (so the device cannot finish in one hook pass)."""
    order = np.random.default_rng(seed).permutation(n).astype(np.int32)
    return {"bodies": _bodies(n), "constraints": _constraints({2: np.stack([order[:-1], order[1:]], axis=1)})}


def bridged_piles(pile=200, kinematic_bridge=True):
    """Two chains of `pile` bodies each and, last, one body that both chains' ends touch: a kinematic body (or a dynamic one). Plus one separate
    dynamic pair."""
    n = 2 * pile + 3
    bridge = 2 * pile
    a = np.arange(pile, dtype=np.int32)
    b = np.arange(pile, 2 * pile, dtype=np.int32)
    pairs = np.concatenate([np.stack([a[:-1], a[1:]], 1), np.stack([b[:-1], b[1:]], 1), [[a[-1], bridge], [b[0], bridge], [bridge + 1, bridge + 2]]]).astype(np.int32)
    return {"bodies": _bodies(n, [bridge] if kinematic_bridge else []), "constraints": _constraints({2: pairs})}


def edges_of(type_batches, bundle_width):
    """Per live lane, edges from its first live body to each other one (decoded references), straight from the reference-layout buffers."""
    us, vs = [], []
    for tb in type_batches:
        refs = np.asarray(tb.body_references)  # [bundle, slot, W]
        lanes = refs.transpose(0, 2, 1).reshape(-1, refs.shape[1])[:tb.constraint_count]
        dec = np.where(lanes >= 0, lanes & 0x3FFFFFFF, -1)
        for s in range(1, dec.shape[1]):
            ok = (dec[:, 0] >= 0) & (dec[:, s] >= 0)
            us.append(dec[ok, 0])
            vs.append(dec[ok, s])
    return (np.concatenate(us) if us else np.zeros(0, np.int64)), (np.concatenate(vs) if vs else np.zeros(0, np.int64))


def expected(type_batches, bundle_width, n, candidates):
    """scipy's connected components of the same graph, in the call's form: (smallest index per body, sleepable roots ascending, their sizes)."""
    u, v = edges_of(type_batches, bundle_width)
    graph = coo_matrix((np.ones(u.shape[0]), (u, v)), shape=(n, n))
    _, comp = connected_components(graph, directed=False)
    lowest = np.full(comp.max() + 1, n, dtype=np.int64)
    np.minimum.at(lowest, comp, np.arange(n))
    labels = lowest[comp].astype(np.int32)
    blocked = np.zeros(comp.max() + 1, dtype=bool)
    np.logical_or.at(blocked, comp, np.asarray(candidates) == 0)
    sizes = np.bincount(comp)
    keep = np.sort(np.flatnonzero(~blocked), kind="stable")
    order = np.argsort(lowest[keep])
    return labels, lowest[keep][order].astype(np.int32), sizes[keep][order].astype(np.int32)


def checker(sim, candidates):
    return island_checker.find_sleepable_islands(sim.type_batches(), sim.body_count, sim.bundle_width, candidates)


def candidates_for(n, seed, p_block=0.002):
    rng = np.random.default_rng(seed)
    return (rng.random(n) >= p_block).astype(np.uint8)


def check_against_scipy(sim, candidates):
    want = expected(sim.type_batches(), sim.bundle_width, sim.body_count, candidates)
    got = checker(sim, candidates)
    for w, g, what in zip(want, got, ("labels", "roots", "counts")):
        assert np.array_equal(w, g), what
    return got


# ---- CPU: the checker against scipy and closed forms -------------------------------------------------------------------------------------------------
def test_checker_partition_is_scipys_on_random_graphs(libs):
    for seed in range(4):
        sim = util.make_sim(random_graph(seed))
        labels, roots, counts = check_against_scipy(sim, candidates_for(sim.body_count, seed, p_block=0.01))
        assert len(np.unique(labels)) > 100 and len(roots) > 10  # many islands, some of them sleepable
        assert {tb.type_id for tb in sim.type_batches()} == set(TYPE_OF_BODIES.values())


def test_checker_kinematic_bridge_joins_two_piles(libs):
    for kinematic in (True, False):
        sim = util.make_sim(bridged_piles(kinematic_bridge=kinematic))
        labels, _, _ = check_against_scipy(sim, np.ones(sim.body_count, dtype=np.uint8))
        assert sorted(np.unique(labels).tolist()) == [0, 401]  # the piles and their bridge are one island, the separate pair another


def test_checker_skips_empty_fallback_lanes(libs):
    sim = util.make_sim(scenes.fallback_stress(600, hubs=3, seed=5), fallback_batch_threshold=8)
    assert util.punch_fallback_holes(sim) > 10
    check_against_scipy(sim, candidates_for(sim.body_count, 3))


def test_checker_unconstrained_bodies_are_islands_of_their_own(libs):
    scene = random_graph(7, n=500, per_kind=(10, 30, 5, 5))
    sim = util.make_sim(scene)
    labels, roots, counts = check_against_scipy(sim, np.ones(500, dtype=np.uint8))
    u, v = edges_of(sim.type_batches(), sim.bundle_width)
    free = np.setdiff1d(np.arange(500), np.concatenate([u, v]))
    assert free.size > 100
    assert np.array_equal(labels[free], free)
    assert np.isin(free, roots).all() and (counts[np.searchsorted(roots, free)] == 1).all()


def test_checker_on_a_131072_body_chain(libs):
    n = 131072
    sim = util.make_sim(chain(n))
    labels, roots, counts = check_against_scipy(sim, np.ones(n, dtype=np.uint8))
    assert (labels == 0).all() and roots.tolist() == [0] and counts.tolist() == [n]


def test_checker_sleepable_verdict_on_closed_forms(libs):
    sim = util.make_sim(random_graph(11, n=800, per_kind=(40, 200, 20, 20)))
    n = sim.body_count
    labels, roots, counts = checker(sim, np.ones(n, dtype=np.uint8))
    assert np.array_equal(roots, np.unique(labels)) and counts.sum() == n  # all candidates: every island sleeps
    assert checker(sim, np.zeros(n, dtype=np.uint8))[1].size == 0  # none: no island
    one_per_island = np.ones(n, dtype=np.uint8)
    one_per_island[roots] = 0
    assert checker(sim, one_per_island)[1].size == 0
    # a kinematic body that is not a candidate blocks the island it bridges, and only that one
    sim = util.make_sim(bridged_piles())
    c = np.ones(sim.body_count, dtype=np.uint8)
    c[400] = 0
    _, roots, counts = checker(sim, c)
    assert roots.tolist() == [401] and counts.tolist() == [2]


# ---- GPU: the device against the checker---------------------------------------------------------------------------------------------------------------
def activities(candidates):
    a = np.zeros(len(candidates), dtype=native.BODY_ACTIVITY_DTYPE)
    a["sleep_threshold"] = 0.01
    a["sleep_candidate"] = candidates
    return a


def device(sim, candidates, repeat=1, mode=native.EXEC_GRAPH):
    ts = bp.CudaTimestepper(sim, execution_mode=mode)
    try:
        ts.describe()
        return [ts.find_sleepable_islands(activities(candidates)) for _ in range(repeat)]
    finally:
        ts.close()


def check_device(sim, candidates, repeat=1):
    want = checker(sim, candidates)
    runs = device(sim, candidates, repeat)
    for labels, roots, counts, rounds in runs:
        for w, g, what in zip(want, (labels, roots, counts), ("labels", "roots", "counts")):
            assert np.array_equal(w, g), what
        assert rounds >= 1 or sim.constraint_count == 0
    return runs[0]


@pytest.mark.gpu
def test_device_matches_the_checker_on_random_graphs_at_every_bundle_width(libs):
    for W in (4, 8, 16):
        for seed in range(3):
            sim = util.make_sim(random_graph(seed), bundle_width=W)
            for candidates in (candidates_for(sim.body_count, seed, p_block=0.01), np.ones(sim.body_count, dtype=np.uint8)):
                check_device(sim, candidates)
        sim = util.make_sim(bridged_piles(), bundle_width=W)
        c = np.ones(sim.body_count, dtype=np.uint8)
        c[400] = 0
        check_device(sim, c)
        sim = util.make_sim(scenes.fallback_stress(600, hubs=3, seed=5), bundle_width=W, fallback_batch_threshold=8)
        util.punch_fallback_holes(sim)
        check_device(sim, candidates_for(sim.body_count, W))


@pytest.mark.gpu
def test_device_matches_the_checker_on_the_benchmark_scenes(libs):
    """C2 (100 k-body pile), C3 (ragdolls in a kinematic tube), C5 (levelised fallback batch); every body a candidate and a few blocked."""
    for name, scene, kw in (("C2", scenes.shape_pile(100_000, seed=5), {}), ("C3", scenes.ragdolls(seed=5), {}), ("C5", scenes.fallback_stress(seed=5), {})):
        sim = util.make_sim(scene, **kw)
        for candidates in (np.ones(sim.body_count, dtype=np.uint8), candidates_for(sim.body_count, 1, p_block=0.001)):
            _, roots, _, rounds = check_device(sim, candidates)
            print("%s: %d bodies, %d sleepable islands, %d rounds" % (name, sim.body_count, roots.size, rounds))


@pytest.mark.gpu
def test_device_matches_the_checker_on_the_million_body_pile(libs):
    sim = util.make_sim(scenes.shape_pile(1_000_000, seed=5), substeps=4, velocity_iterations=2)
    check_device(sim, candidates_for(sim.body_count, 2, p_block=0.0005))


@pytest.mark.gpu
def test_repeated_calls_give_identical_outputs(libs):
    sim = util.make_sim(scenes.shape_pile(20_000, seed=3))
    runs = check_device(sim, candidates_for(sim.body_count, 4), repeat=1)
    again = device(sim, candidates_for(sim.body_count, 4), repeat=3)
    for run in again:
        for a, b in zip(runs, run):
            assert np.array_equal(a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [native.EXEC_GRAPH, native.EXEC_STREAM])
def test_the_call_leaves_the_next_solve_unchanged(libs, mode):
    """Three frames of solve + search against three solves: byte-identical bodies and impulses (the search touches no solver state and does not
    invalidate the captured graph)."""
    scene = scenes.merge(scenes.shape_pile(3000, seed=9), scenes.ragdolls(20, seed=9), scenes.fallback_stress(600, hubs=3, seed=9))
    snaps = []
    for search in (True, False):
        sim = util.make_sim(scene, substeps=2, velocity_iterations=2)
        ts = bp.CudaTimestepper(sim, execution_mode=mode)
        try:
            ts.describe()
            for frame in range(3):
                ts.solve_device_only(DT)
                if search:
                    ts.find_sleepable_islands(activities(candidates_for(sim.body_count, frame)))
            launches = ts.timings().kernel_launches
            ts.download_bodies()
            ts.download_impulses()
        finally:
            ts.close()
        snaps.append((util.snapshot(sim), launches))
    util.compare(snaps[0][0], snaps[1][0], exact=True)
    assert snaps[0][1] == snaps[1][1]


@pytest.mark.gpu
def test_errors(libs):
    sim = util.make_sim(random_graph(0, n=300, per_kind=(10, 40, 5, 5)))
    n = sim.body_count
    ts = bp.CudaTimestepper(sim)
    try:
        with pytest.raises(bp.BepuCudaError) as e:  # before the first end_constraints
            ts.find_sleepable_islands(activities(np.ones(n, dtype=np.uint8)))
        assert e.value.code == native.ERR_BAD_STATE
        ts.describe()
        with pytest.raises(bp.BepuCudaError) as e:  # another body count than the last upload
            ts.find_sleepable_islands(activities(np.ones(n - 1, dtype=np.uint8)))
        assert e.value.code == native.ERR_INVALID_ARGUMENT
        cuda = ts._cuda
        count, act = C.c_int32(), activities(np.ones(n, dtype=np.uint8))
        out = np.zeros(n, dtype=np.int32)
        for args in ((None, out.ctypes.data, out.ctypes.data, C.byref(count)), (act.ctypes.data, None, out.ctypes.data, C.byref(count)),
                     (act.ctypes.data, out.ctypes.data, None, C.byref(count)), (act.ctypes.data, out.ctypes.data, out.ctypes.data, None)):
            a, r, c, k = args
            assert cuda.bepucuda_find_sleepable_islands(ts._ctx, a, n, None, r, c, k, None) == native.ERR_INVALID_ARGUMENT
        labels, roots, counts, _ = ts.find_sleepable_islands(act)  # the context still works
        assert counts.sum() == n and np.array_equal(roots, np.unique(labels))
    finally:
        ts.close()
    # peer mode: a one-rank shard on this GPU
    solver = sharding.ShardedSolver(sim, 0, 1, device=0)
    try:
        solver.export_handles()
        solver.import_contexts([solver])
        solver.describe()  # a rank whose constraint description is complete
        labels = np.zeros(n, dtype=np.int32)
        count = C.c_int32()
        rc = solver._cuda.bepucuda_find_sleepable_islands(solver._ctx, activities(np.ones(n, dtype=np.uint8)).ctypes.data, n, None, labels.ctypes.data, labels.ctypes.data,
                                                          C.byref(count), None)
        assert rc == native.ERR_BAD_STATE
        assert b"peer mode" in solver._cuda.bepucuda_last_error(solver._ctx)
    finally:
        solver.close()


@pytest.mark.gpu
def test_round_count_is_logarithmic(libs):
    """Min-label propagation would take the chain's diameter in rounds (131 071); hooking roots and pointing every body at its root takes O(log n)."""
    n = 131072
    sim = util.make_sim(chain(n))
    labels, roots, counts, rounds = check_device(sim, np.ones(n, dtype=np.uint8))
    assert (labels == 0).all() and counts.tolist() == [n]
    sim = util.make_sim(scenes.shape_pile(100_000, seed=5))
    _, _, _, pile_rounds = device(sim, np.ones(sim.body_count, dtype=np.uint8))[0]
    print("rounds: %d on the %d-body chain, %d on C2" % (rounds, n, pile_rounds))
    assert rounds <= 64
    assert pile_rounds <= 64
