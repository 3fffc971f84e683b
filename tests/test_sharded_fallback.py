"""A constraint graph with a sequential fallback batch split over several ranks: one rank, the fallback rank, owns every fallback constraint and runs
the whole fallback batch in its dependency levels; every rank has one exchange point per fallback section (the fallback part of one WarmStart or
Solve pass). On the CPU: the partitioner (sharding.partition / fallback_rank), and the plan, the stage program and the arrival targets through the
topology shims. On the GPU: several ranks as contexts of one process on one device against the oracle run on the whole graph, bit for bit."""
import ctypes as C
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from bepuphysics2_b200 import _build, native, scenes, sharding
from tests import test_topology as topo
from tests import util

DT = 1.0 / 60.0
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "bepuphysics2_b200", "csrc")
EXECUTION_MODES = {"graph": native.EXEC_GRAPH, "stream": native.EXEC_STREAM}
OLD_MESSAGE = "end_constraints: the sequential fallback batch is not supported across ranks"

SCENES = {"fallback_stress": (lambda: scenes.fallback_stress(3000, hubs=6, seed=7), 4),
          "joint_zoo": (lambda: scenes.joint_zoo(600, per_type=30, seed=11, kinematic_fraction=0.2), 4)}


def _sim(case, **kw):
    scene, threshold = SCENES[case]
    return util.make_sim(scene(), fallback_batch_threshold=threshold, **kw)


def _live(tb):
    """Live constraints of a type batch (holes of the fallback batch excluded)."""
    return np.flatnonzero(tb.body_references.transpose(0, 2, 1).reshape(-1, tb.body_references.shape[1])[:tb.constraint_count, 0] >= 0)


# ---- partition ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", sorted(SCENES))
@pytest.mark.parametrize("rank_count", [2, 3])
def test_partition_puts_the_whole_fallback_batch_on_one_rank_verbatim(case, rank_count):
    sim = _sim(case)
    threshold = sim.fallback_batch_threshold
    shards, first_batch, constrained, masks = sharding.partition(sim, rank_count)
    fallback = sharding.fallback_rank(sim, rank_count)
    by_key = {(tb.batch_index, tb.type_batch_index): tb for tb in sim.type_batches()}
    assert any(b >= threshold for b, _ in by_key) and 0 <= fallback < rank_count

    # the rule: the slab holding the most first dynamic bodies of fallback constraints, lowest rank on a tie
    votes = np.zeros(rank_count, dtype=np.int64)
    for (b, _), tb in by_key.items():
        if b >= threshold:
            refs = tb.body_references.transpose(0, 2, 1).reshape(-1, tb.body_references.shape[1])[:tb.constraint_count]
            for row in refs[_live(tb)]:
                dyn = [int(x) & sharding.INDEX_MASK for x in row if x >= 0 and not x & sharding.KINEMATIC_BIT]
                if dyn:
                    votes[dyn[0] * rank_count // sim.body_count] += 1
    assert fallback == int(np.flatnonzero(votes == votes.max())[0])

    seen = {k: np.zeros(tb.constraint_count, dtype=np.int32) for k, tb in by_key.items()}
    expect_masks = np.zeros(sim.body_count, dtype=np.uint8)
    expect_first = np.full(sim.body_count, sharding.INT32_MAX, dtype=np.int64)
    for r, shard in enumerate(shards):
        for d in shard:
            key = (d["batch_index"], d["type_batch_index"])
            g = by_key[key]
            nb = d["refs"].shape[1]
            packed = d["refs"].transpose(0, 2, 1).reshape(-1, nb)[:d["count"]]
            if key[0] >= threshold:
                # the host's type batch as it is: bundles, lanes and holes, and its rows
                assert r == fallback, "a fallback type batch on rank %d, fallback rank %d" % (r, fallback)
                assert d["count"] == g.constraint_count and np.array_equal(d["source"], np.arange(g.constraint_count))
                for mine, host in (("refs", g.body_references), ("prestep", g.prestep), ("impulses", g.accumulated_impulses)):
                    assert np.array_equal(d[mine].view(np.uint32), host.view(np.uint32)), mine
                seen[key][_live(g)] += 1
                packed = packed[_live(g)]
            else:
                seen[key][d["source"]] += 1
            dyn = (packed >= 0) & ((packed & sharding.KINEMATIC_BIT) == 0)
            idx = (packed & sharding.INDEX_MASK)[dyn]
            expect_masks[idx] |= np.uint8(1 << r)
            np.minimum.at(expect_first, idx, key[0])
    for key, count in seen.items():
        live = np.zeros(count.shape[0], dtype=bool)
        live[_live(by_key[key]) if key[0] >= threshold else slice(None)] = True
        assert (count[live] == 1).all() and (count[~live] == 0).all(), key
    assert np.array_equal(expect_masks, masks)
    assert np.array_equal(expect_first, first_batch.astype(np.int64))
    expect_constrained = expect_first != sharding.INT32_MAX
    expect_constrained[np.asarray(sim.constrained_kinematics, dtype=np.int64)] = True
    assert np.array_equal(constrained != 0, expect_constrained)


def test_partition_without_a_fallback_batch_names_no_fallback_rank():
    sim = util.make_sim(scenes.shape_pile(1500, seed=13))
    assert sharding.fallback_rank(sim, 3) == -1
    assert all(d["batch_index"] < sim.fallback_batch_threshold for shard in sharding.partition(sim, 3)[0] for d in shard)


_GLOO_SCRIPT = r"""
import hashlib, sys
import torch.distributed as dist
sys.path.insert(0, %r)
from bepuphysics2_b200 import scenes, sharding
from tests import util
dist.init_process_group("gloo")
rank, world = dist.get_rank(), dist.get_world_size()
sim = util.make_sim(scenes.fallback_stress(2000, hubs=4, seed=9), fallback_batch_threshold=4)
fallback = sharding.fallback_rank(sim, world)
shards, first_batch, constrained, masks = sharding.partition(sim, world)
digest = hashlib.sha256(first_batch.tobytes() + constrained.tobytes() + masks.tobytes()).hexdigest()
got = [None] * world
dist.all_gather_object(got, (fallback, digest))
assert fallback >= 0 and len(set(got)) == 1, "ranks disagree on the fallback rank or the global tables: %%s" %% got
if rank == 0:
    print("OK", fallback)
dist.destroy_process_group()
"""


def test_gloo_ranks_agree_on_the_fallback_rank(tmp_path):
    script = tmp_path / "ranks.py"
    script.write_text(_GLOO_SCRIPT % ROOT)
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "3", "--master-addr", "127.0.0.1", "--master-port", "29547", str(script)],
                       cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0 and "OK" in r.stdout, r.stdout[-3000:]


# ---- plan, stage program and arrival targets ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def peer_shim():
    here = os.path.join(ROOT, "tests", "topology")
    lib = os.path.join(here, "libfallback_shim.so")
    srcs = [os.path.join(here, "topology_shim.cpp"), os.path.join(here, "fallback_shim.cpp"), os.path.join(CSRC, "bepu_topology.cpp")]
    deps = srcs + [os.path.join(CSRC, f) for f in ("bepu_topology.h", "bepu_device_types.h", "bepu_layout_kernels.h", "bepu_joint_registry.inc")]
    if not os.path.exists(lib) or any(os.path.getmtime(s) > os.path.getmtime(lib) for s in deps):
        cuda_include = os.path.join(os.path.dirname(os.path.dirname(_build.NVCC)), "include")
        subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-Wall", "-shared", "-fPIC", "-I", CSRC, "-I", cuda_include, "-o", lib] + srcs)
    dll = C.CDLL(lib)
    vp, i32 = C.c_void_p, C.c_int32
    dll.topology_plan.restype = vp
    dll.topology_plan.argtypes = [i32, vp, vp, i32, i32, i32, i32, i32]
    dll.topology_plan_peer.restype = vp
    dll.topology_plan_peer.argtypes = [i32, vp, vp, i32, i32, i32, i32, i32, i32]
    dll.topology_plan_error.argtypes = [vp, C.c_char_p, i32]
    for name in ("sizes", "tbs", "maps", "work", "batches", "source_live"):
        getattr(dll, "topology_plan_" + name).argtypes = [vp, vp]
    dll.topology_plan_free.argtypes = [vp]
    dll.topology_program.restype = vp
    dll.topology_program.argtypes = [vp, i32, vp, i32, i32, i32, i32]
    dll.topology_program_sizes.argtypes = [vp, vp]
    dll.topology_program_ops.argtypes = [vp, vp]
    dll.topology_program_free.argtypes = [vp]
    dll.topology_resolve.argtypes = [vp, i32, i32, i32, i32, vp]
    dll.topology_exchange_targets.argtypes = [vp, i32, vp, i32, i32, i32, vp, vp]
    return dll


def plan_peer(dll, sources, W, threshold, batch_count, body_count, rank, fallback_rank):
    """topology_plan in peer mode for `rank`: a topo.Plan, or (error code, message)."""
    n = len(sources)
    meta = np.array([s[:4] for s in sources], dtype=np.int32).reshape(n, 4)
    refs = [np.ascontiguousarray(s[4], dtype=np.int32) for s in sources]
    ptrs = (C.c_void_p * max(n, 1))(*[r.ctypes.data for r in refs])
    h = dll.topology_plan_peer(n, meta.ctypes.data, ptrs, W, threshold, batch_count, body_count, rank, fallback_rank)
    message = C.create_string_buffer(256)
    rc = dll.topology_plan_error(h, message, 256)
    if rc != 0:
        dll.topology_plan_free(h)
        return rc, message.value.decode()
    return topo.Plan(dll, h)


def shard_sources(shard):
    return [(d["batch_index"], d["type_batch_index"], d["type_id"], d["count"], d["refs"]) for d in shard]


def fallback_levels(p, sources):
    """Per planned type batch of the fallback levels: (level, source (batch, type batch), type id, bundles, source constraint per slot)."""
    out = []
    for t in range(len(p.tbs)):
        type_id, bundles, device_batch, source, map_offset = (int(v) for v in p.tbs[t])
        if map_offset >= 0:
            out.append((device_batch - p.sync_batch_count, tuple(sources[source][:2]), type_id, bundles, p.maps[map_offset:map_offset + 32 * bundles].tolist()))
    return out


def exchange_points(ops):
    """Per exchange point of a program, in order: (stage, rank barrier or not), and the op rows that carry it."""
    points = {}
    for op in ops[ops[:, 3] != topo.NO_EXCHANGE]:
        points.setdefault(int(op[4]), []).append(op)
    assert sorted(points) == list(range(len(points))), "exchange indices are consecutive"
    return [(int(rows[0][0]), int(rows[0][3]) == topo.RANK_BARRIER) for _, rows in sorted(points.items())], [rows for _, rows in sorted(points.items())]


@pytest.mark.parametrize("case", sorted(SCENES))
@pytest.mark.parametrize("rank_count", [2, 3])
def test_every_rank_runs_one_exchange_point_per_fallback_section(libs, peer_shim, case, rank_count):
    sim = _sim(case)
    W, threshold = sim.bundle_width, sim.fallback_batch_threshold
    shards, _, _, _ = sharding.partition(sim, rank_count)
    fallback = sharding.fallback_rank(sim, rank_count)
    kinematic_count = len(sim.constrained_kinematics)
    plans = [plan_peer(peer_shim, shard_sources(shards[r]), W, threshold, sim.batch_count, sim.body_count, r, fallback) for r in range(rank_count)]
    assert all(isinstance(p, topo.Plan) for p in plans)

    # the fallback rank levelises its verbatim type batches exactly as one context given the whole graph does
    whole = topo.plan(peer_shim, topo.sim_sources(sim), W, threshold, sim.batch_count, sim.body_count)
    mine = plans[fallback]
    assert mine.fallback_levels == whole.fallback_levels > 1
    assert fallback_levels(mine, shard_sources(shards[fallback])) == fallback_levels(whole, topo.sim_sources(sim))
    assert all(p.fallback_levels == 0 for r, p in enumerate(plans) if r != fallback)
    assert len({p.sync_batch_count for p in plans}) == 1

    rng = np.random.default_rng(rank_count)
    for iterations in ([1], [2, 1, 3]):
        passes = sum(1 + n for n in iterations)
        sequences = []
        for r, p in enumerate(plans):
            ops, totals = p.program(iterations, kinematic_count, True, True, sim.body_count)
            topo.check_launches(peer_shim, ops, True)
            sequence, rows = exchange_points(ops)
            assert totals["exchange_count"] == len(sequence)
            sequences.append(sequence)
            sections = [i for i, rs in enumerate(rows) if int(rs[0][3]) >= p.sync_batch_count]
            assert len(sections) == passes, "one exchange point per fallback section"
            if r == fallback:
                # the rank's program is the single-context order of its batches (levels included) ...
                want = topo.expected_program(p, iterations, kinematic_count, True, True, sim.body_count)
                assert np.array_equal(ops[:, :4], want[:, :4])
                # ... with the levels of a section on one exchange point, in order, every one of them
                for i in sections:
                    assert [int(op[3]) for op in rows[i]] == list(range(p.sync_batch_count, p.sync_batch_count + p.fallback_levels))
            else:
                for i in sections:
                    assert len(rows[i]) == 1 and rows[i][0][2] == 0, "a zero-work op holds the section's place"
            # arrival targets: every op of a section adds its boundary bundles to the section's one exchange point
            boundary = rng.integers(1, 6, size=len(p.batches)).astype(np.int32)
            boundary[p.batches[:, 1] == 0] = 0
            targets = np.zeros(peer_shim.topology_max_exchanges(), dtype=np.uint64)
            its = np.asarray(iterations, dtype=np.int32)
            assert peer_shim.topology_exchange_targets(p.handle, its.size, its.ctypes.data, kinematic_count, 1, sim.body_count, boundary.ctypes.data, targets.ctypes.data) == 0
            total = 0
            for i, rs in enumerate(rows):
                arrived = sum(int(boundary[int(op[3])]) for op in rs if op[3] >= 0 and op[2] > 0)
                assert int(targets[i]) - total == arrived, "exchange point %d" % i
                total += arrived
                if i in sections and r == fallback:
                    assert arrived == int(boundary[p.sync_batch_count:].sum()) > 0
            assert int(targets[-1]) == total
        assert all(s == sequences[0] for s in sequences), "every rank runs the same exchange sequence"


@pytest.mark.parametrize("case", sorted(SCENES))
def test_a_fallback_type_batch_off_the_fallback_rank_is_refused(libs, peer_shim, case):
    sim = _sim(case)
    W, threshold = sim.bundle_width, sim.fallback_batch_threshold
    shards, _, _, _ = sharding.partition(sim, 2)
    fallback = sharding.fallback_rank(sim, 2)
    other = 1 - fallback
    sources = shard_sources(shards[fallback])
    code, message = plan_peer(peer_shim, sources, W, threshold, sim.batch_count, sim.body_count, other, fallback)
    assert code == topo.ERR_BAD_STATE and ("fallback rank %d" % fallback) in message
    # no fallback rank set: the message peer mode has always given
    assert plan_peer(peer_shim, sources, W, threshold, sim.batch_count, sim.body_count, fallback, -1) == (topo.ERR_BAD_STATE, OLD_MESSAGE)
    assert topo.plan(peer_shim, sources, W, threshold, sim.batch_count, sim.body_count, peer_mode=True) == (topo.ERR_BAD_STATE, OLD_MESSAGE)


# ---- on the GPU -----------------------------------------------------------------------------------------------------------------------------
def _solve_all(solvers):
    """One frame on every rank, each issued from a host thread of its own (one host thread per context, include/bepucuda.h): the fallback rank
    issues a launch per level and section, thousands per frame, and once the launch queue is full its issuing thread blocks until the device drains
    it, which needs the other ranks' frames issued too."""
    with ThreadPoolExecutor(max_workers=len(solvers)) as pool:
        list(pool.map(lambda s: s.solve(DT), solvers))


def _one_process_ranks(scene, rank_count, frames, mode, **kw):
    """`rank_count` contexts on device 0; every rank's referenced bodies and its own live constraints' impulses and prestep rows against the oracle
    run on the whole graph, bit for bit. Returns the solvers' fallback rank."""
    from oracle import binding as ob

    sim = util.make_sim(scene, **kw)
    solvers = [sharding.ShardedSolver(sim, r, rank_count, 0, strict_fp=True, execution_mode=EXECUTION_MODES[mode]) for r in range(rank_count)]
    try:
        for s in solvers:
            s.export_handles()
        for s in solvers:
            s.import_contexts(solvers)
        for s in solvers:
            s.describe()
        for s in solvers:
            s.synchronize()
        fallback = solvers[0].fallback_rank
        assert fallback >= 0 and all(s.fallback_rank == fallback for s in solvers)
        for s in solvers:
            assert (s.timings().fallback_level_count > 0) == (s.rank == fallback)
        for _ in range(frames):
            ob.solve(sim, DT)
            _solve_all(solvers)
        by_key = {(tb.batch_index, tb.type_batch_index): tb for tb in sim.type_batches()}
        for s in solvers:
            got = s.download()
            mine = s.referenced_bodies()
            assert np.array_equal(sim.bodies[mine][:, util.MOTION].view(np.uint32), got[mine][:, util.MOTION].view(np.uint32)), "rank %d bodies (%s)" % (s.rank, mode)
            for d in s.shard:
                g = by_key[(d["batch_index"], d["type_batch_index"])]
                # a fallback type batch is the host's own (source = identity): its live lanes; a synchronized one is compacted
                ref_lanes, have_lanes = (_live(g), _live(g)) if d["batch_index"] >= sim.fallback_batch_threshold else (d["source"], np.arange(d["count"]))
                for what, ref_rows in (("impulses", g.accumulated_impulses), ("prestep", g.prestep)):
                    ref = ref_rows.transpose(0, 2, 1).reshape(-1, ref_rows.shape[1])[ref_lanes]
                    have = d[what].transpose(0, 2, 1).reshape(-1, d[what].shape[1])[have_lanes]
                    assert np.array_equal(ref.view(np.uint32), have.view(np.uint32)), "rank %d %s of batch %d (%s)" % (s.rank, what, d["batch_index"], mode)
        assert int(((solvers[0].masks & (solvers[0].masks - 1)) != 0).sum()) > 0
        return fallback
    finally:
        for s in solvers:
            s.close()


@pytest.mark.gpu
@pytest.mark.parametrize("rank_count,mode", [(2, "graph"), (3, "graph"), (2, "stream"), (3, "stream")])
def test_fallback_stress_over_several_ranks_bit_exact(libs, rank_count, mode):
    _one_process_ranks(scenes.fallback_stress(3000, hubs=6, seed=7), rank_count, frames=3, mode=mode, fallback_batch_threshold=4, substeps=2, velocity_iterations=2)


@pytest.mark.gpu
def test_joint_zoo_with_multi_body_joints_and_kinematics_in_the_fallback_batch_bit_exact(libs):
    """Three- and four-body joints and kinematic partners in the fallback batch: the pushes of body slots 2 and 3 from the fallback levels."""
    _one_process_ranks(scenes.joint_zoo(1200, per_type=60, seed=8, kinematic_fraction=0.15), 2, frames=2, mode="graph", fallback_batch_threshold=4, substeps=3,
                       velocity_iterations=2)


@pytest.mark.gpu
def test_mixed_scene_with_a_fallback_batch_over_two_ranks_bit_exact(libs):
    """Contacts, ragdolls, joints and hubs in one graph, several substeps, both execution modes: the incremental contact update and the rank barriers
    between substeps meet the fallback sections."""
    scene = scenes.merge(scenes.shape_pile(1200, seed=21), scenes.ragdolls(8, seed=22), scenes.joint_zoo(300, 20, seed=23), scenes.fallback_stress(800, hubs=3, seed=24))
    for mode in ("graph", "stream"):
        _one_process_ranks(scene, 2, frames=2, mode=mode, fallback_batch_threshold=6, substeps=3, velocity_iterations=2)


@pytest.mark.gpu
def test_momentum_conserving_angular_mode_with_the_fallback_batch_on_one_rank_bit_exact(libs):
    """ConserveMomentum's first-substep quirk depends on the host bundles (bit 28): the fallback rank's verbatim type batches keep it. Threshold 1
    leaves batch 0 synchronized, where every dynamic lane integrates its bodies and compaction cannot change the quirk."""
    integ = util.bp.IntegratorDesc.default()
    integ.angular_integration_mode = 1
    _one_process_ranks(scenes.joint_zoo(600, 40, seed=9), 2, frames=2, mode="graph", fallback_batch_threshold=1, substeps=2, velocity_iterations=2, integrator=integ)


@pytest.mark.gpu
def test_fallback_rank_argument_and_state_errors_come_before_device_work(libs):
    sim = util.make_sim(scenes.fallback_stress(600, hubs=3, seed=5), fallback_batch_threshold=4, substeps=2, velocity_iterations=1)
    solvers = [sharding.ShardedSolver(sim, r, 2, 0, strict_fp=True) for r in range(2)]
    try:
        for s in solvers:
            s.export_handles()
        s, cuda = solvers[0], solvers[0]._cuda
        assert cuda.bepucuda_shard_set_fallback_rank(s._ctx, 0) == topo.ERR_INVALID_ARGUMENT  # not in peer mode yet
        assert "peer mode" in cuda.bepucuda_last_error(s._ctx).decode()
        for t in solvers:
            t.import_contexts(solvers)
        for bad in (2, -2):
            assert cuda.bepucuda_shard_set_fallback_rank(s._ctx, bad) == topo.ERR_INVALID_ARGUMENT
        fallback = s.fallback_rank
        other = solvers[1 - fallback]
        # the fallback rank's type batches uploaded on the other rank: refused by end_constraints, naming the fallback rank, with the bodies as uploaded
        for fallback_rank, message in ((fallback, "fallback rank %d" % fallback), (-1, OLD_MESSAGE)):
            other._check(cuda.bepucuda_shard_set_fallback_rank(other._ctx, fallback_rank))
            other._check(cuda.bepucuda_shard_set_global(other._ctx, other.first_batch.ctypes.data, other.constrained.ctypes.data))
            other._check(cuda.bepucuda_begin_constraints(other._ctx, sim.bundle_width, sim.batch_count))
            for d in solvers[fallback].shard:
                other._check(cuda.bepucuda_upload_type_batch(other._ctx, d["batch_index"], d["type_batch_index"], d["type_id"], d["count"], d["refs"].ctypes.data,
                                                             d["prestep"].ctypes.data, d["impulses"].ctypes.data))
            other._check(cuda.bepucuda_shard_set_body_masks(other._ctx, other.masks.ctypes.data))
            with pytest.raises(native.BepuCudaError) as e:
                other._check(cuda.bepucuda_end_constraints(other._ctx))
            assert e.value.code == topo.ERR_BAD_STATE and message in str(e.value)
        got = np.zeros_like(sim.bodies)
        other._check(cuda.bepucuda_download_bodies(other._ctx, got.ctypes.data, sim.body_count))
        assert np.array_equal(sim.bodies[:, util.MOTION].view(np.uint32), got[:, util.MOTION].view(np.uint32))
        # described as the partitioner says, both ranks solve and match the oracle
        from oracle import binding as ob

        for t in solvers:
            t.describe()
        ob.solve(sim, DT)
        _solve_all(solvers)
        for t in solvers:
            mine = t.referenced_bodies()
            got = t.download()
            assert np.array_equal(sim.bodies[mine][:, util.MOTION].view(np.uint32), got[mine][:, util.MOTION].view(np.uint32))
    finally:
        for s in solvers:
            s.close()
