"""One constraint graph over several GPUs (SURVEY.md §8e): the host partitioner (CPU: invariants, and a world-size-2 gloo run showing both ranks derive
the same global tables from the same scene) and, on the GPU, several ranks as contexts of one process on one device against the oracle, bit for bit."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

from bepuphysics2_b200 import native, scenes, sharding
from tests import util

DT = 1.0 / 60.0
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXECUTION_MODES = {"graph": native.EXEC_GRAPH, "stream": native.EXEC_STREAM}


def _global_rows(sim):
    rows = {}
    for tb in sim.type_batches():
        nb = tb.body_references.shape[1]
        rows[(tb.batch_index, tb.type_batch_index)] = tb.body_references.transpose(0, 2, 1).reshape(-1, nb)[:tb.constraint_count]
    return rows


@pytest.mark.parametrize("rank_count", [2, 3, 8])
def test_partition_covers_every_constraint_once_and_masks_name_the_referencing_ranks(rank_count):
    sim = util.make_sim(scenes.shape_pile(3000, seed=3), substeps=2, velocity_iterations=2)
    shards, first_batch, constrained, masks = sharding.partition(sim, rank_count)
    rows = _global_rows(sim)
    seen = {k: np.zeros(v.shape[0], dtype=np.int32) for k, v in rows.items()}
    expect_masks = np.zeros(sim.body_count, dtype=np.uint8)
    expect_first = np.full(sim.body_count, sharding.INT32_MAX, dtype=np.int64)
    for r, shard in enumerate(shards):
        for tb in shard:
            key = (tb["batch_index"], tb["type_batch_index"])
            seen[key][tb["source"]] += 1
            # the compacted rows are the global rows of the source constraints, in the order the shard stores them
            nb = tb["refs"].shape[1]
            packed = tb["refs"].transpose(0, 2, 1).reshape(-1, nb)[:tb["count"]]
            assert np.array_equal(packed, rows[key][tb["source"]])
            assert (tb["refs"].transpose(0, 2, 1).reshape(-1, nb)[tb["count"]:] == -1).all()
            dyn = (packed >= 0) & ((packed & sharding.KINEMATIC_BIT) == 0)
            idx = (packed & sharding.INDEX_MASK)[dyn]
            expect_masks[idx] |= np.uint8(1 << r)
            np.minimum.at(expect_first, idx, tb["batch_index"])
            # boundary constraints (a dynamic body some other rank references too) come first
            boundary = (((masks[packed & sharding.INDEX_MASK] & ~np.uint8(1 << r)) != 0) & dyn).any(axis=1)
            assert not (np.diff(boundary.astype(np.int8)) > 0).any()
    for key, count in seen.items():
        assert (count == 1).all(), key
    assert np.array_equal(expect_masks, masks)
    assert np.array_equal(expect_first, first_batch.astype(np.int64))
    assert np.array_equal(constrained != 0, expect_first != sharding.INT32_MAX)  # no constrained kinematics in this scene
    # within a batch no dynamic body is written by two ranks: what one rank pushes never collides with another rank's write
    for batch in range(sim.batch_count):
        writers = np.zeros(sim.body_count, dtype=np.int32)
        for shard in shards:
            touched = np.zeros(sim.body_count, dtype=bool)
            for tb in shard:
                if tb["batch_index"] == batch:
                    touched[tb["idx"][tb["dynamic"]]] = True
            writers += touched
        assert writers.max() <= 1


_GLOO_SCRIPT = r"""
import hashlib, sys
import numpy as np
import torch.distributed as dist
sys.path.insert(0, %r)
from bepuphysics2_b200 import scenes, sharding
from tests import util
dist.init_process_group("gloo")
rank, world = dist.get_rank(), dist.get_world_size()
sim = util.make_sim(scenes.shape_pile(1500, seed=9), substeps=2, velocity_iterations=1)
shards, first_batch, constrained, masks = sharding.partition(sim, world)
digest = hashlib.sha256(first_batch.tobytes() + constrained.tobytes() + masks.tobytes()).hexdigest()
mine = sum(tb["count"] for tb in shards[rank])
got = [None] * world
dist.all_gather_object(got, (digest, mine))
assert len({d for d, _ in got}) == 1, "ranks disagree on the global tables"
assert sum(m for _, m in got) == sim.constraint_count
if rank == 0:
    print("OK", sim.constraint_count, [m for _, m in got])
dist.destroy_process_group()
"""


def test_two_gloo_ranks_derive_the_same_global_tables(tmp_path):
    script = tmp_path / "ranks.py"
    script.write_text(_GLOO_SCRIPT % ROOT)
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port", "29533", str(script)],
                       cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0 and "OK" in r.stdout, r.stdout[-3000:]


def _one_process_ranks(sim_scene, rank_count, frames, mode, libs, **kw):
    """`rank_count` contexts on device 0, wired to one another with bepucuda_shard_import_contexts; every rank's referenced bodies and its own
    impulses and prestep rows (contact depths written by the incremental update) against the oracle run on the whole graph."""
    from oracle import binding as ob

    sim = util.make_sim(sim_scene, **kw)
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
        for _ in range(frames):
            ob.solve(sim, DT)
            for s in solvers:  # asynchronous launches: the ranks' frames run side by side on the device and meet at their exchange points
                s.solve(DT)
        by_key = {(tb.batch_index, tb.type_batch_index): tb for tb in sim.type_batches()}
        for s in solvers:
            got = s.download()
            mine = s.referenced_bodies()
            assert mine.size > 0
            assert np.array_equal(sim.bodies[mine][:, util.MOTION].view(np.uint32), got[mine][:, util.MOTION].view(np.uint32)), "rank %d bodies (%s)" % (s.rank, mode)
            for tb in s.shard:
                g = by_key[(tb["batch_index"], tb["type_batch_index"])]
                for what, ref_rows in (("impulses", g.accumulated_impulses), ("prestep", g.prestep)):
                    ref = ref_rows.transpose(0, 2, 1).reshape(-1, ref_rows.shape[1])[tb["source"]]
                    have = tb[what].transpose(0, 2, 1).reshape(-1, tb[what].shape[1])[:tb["count"]]
                    assert np.array_equal(ref.view(np.uint32), have.view(np.uint32)), "rank %d %s of batch %d (%s)" % (s.rank, what, tb["batch_index"], mode)
        shared = int(((solvers[0].masks & (solvers[0].masks - 1)) != 0).sum())
        assert shared > 0
    finally:
        for s in solvers:
            s.close()


@pytest.mark.gpu
@pytest.mark.parametrize("rank_count,mode", [(2, "graph"), (3, "graph"), (2, "stream")])
def test_one_graph_over_several_ranks_bit_exact(libs, rank_count, mode):
    _one_process_ranks(scenes.shape_pile(2500, seed=6), rank_count, frames=3, mode=mode, libs=libs, substeps=4, velocity_iterations=2)


@pytest.mark.gpu
def test_one_graph_over_two_ranks_ragdolls_bit_exact(libs):
    _one_process_ranks(scenes.ragdolls(60, seed=2), 2, frames=2, mode="graph", libs=libs, substeps=2, velocity_iterations=2)


@pytest.mark.gpu
def test_one_graph_over_two_ranks_joint_zoo_bit_exact(libs):
    """Three- and four-body constraints, kinematic bodies, every joint type: the pushes of body slots 2 and 3 and the kinematic stages."""
    _one_process_ranks(scenes.joint_zoo(1200, per_type=60, seed=8), 2, frames=2, mode="graph", libs=libs, substeps=3, velocity_iterations=2)


@pytest.mark.gpu
def test_one_graph_over_two_ranks_mixed_scene_bit_exact(libs):
    """Contacts, ragdolls and a joint zoo in one graph, several substeps, in both execution modes: the incremental contact update between substeps
    reads velocities that other ranks stored, and each rank's contact depths must still match the oracle bit for bit."""
    scene = scenes.merge(scenes.shape_pile(1200, seed=21), scenes.ragdolls(12, seed=22), scenes.joint_zoo(300, 20, seed=23))
    for mode in ("graph", "stream"):
        _one_process_ranks(scene, 2, frames=2, mode=mode, libs=libs, substeps=3, velocity_iterations=2)


@pytest.mark.gpu
def test_peer_mode_needs_body_masks(libs):
    """NULL masks are an argument error, and a rank whose masks are missing cannot build its stage program: end_constraints reports it before any
    device work. Both are plain argument / state errors (no solve, so no rank barrier runs); describing with masks afterwards succeeds."""
    sim = util.make_sim(scenes.shape_pile(400, seed=4), substeps=2, velocity_iterations=1)
    solvers = [sharding.ShardedSolver(sim, r, 2, 0, strict_fp=True) for r in range(2)]
    try:
        for s in solvers:
            s.export_handles()
        for s in solvers:
            s.import_contexts(solvers)
        s, cuda = solvers[0], solvers[0]._cuda
        with pytest.raises(native.BepuCudaError) as e:
            s._check(cuda.bepucuda_shard_set_body_masks(s._ctx, None))
        assert e.value.code == -1  # BEPUCUDA_ERR_INVALID_ARGUMENT
        s._check(cuda.bepucuda_shard_set_global(s._ctx, s.first_batch.ctypes.data, s.constrained.ctypes.data))
        s._check(cuda.bepucuda_begin_constraints(s._ctx, sim.bundle_width, sim.batch_count))
        for tb in s.shard:
            s._check(cuda.bepucuda_upload_type_batch(s._ctx, tb["batch_index"], tb["type_batch_index"], tb["type_id"], tb["count"], tb["refs"].ctypes.data,
                                                     tb["prestep"].ctypes.data, tb["impulses"].ctypes.data))
        with pytest.raises(native.BepuCudaError) as e:
            s._check(cuda.bepucuda_end_constraints(s._ctx))
        assert e.value.code == -6 and "shard_set_body_masks" in str(e.value)  # BEPUCUDA_ERR_BAD_STATE
        s.describe()
    finally:
        for s in solvers:
            s.close()


@pytest.mark.gpu
def test_profile_stages_is_refused_in_peer_mode(libs):
    """A stage profile is a frame of one rank alone, which cannot meet its peers at the rank barriers: a described peer-mode context refuses it
    before any device work, so its bodies stay as uploaded."""
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
        profile = native.StageProfile()
        assert s._cuda.bepucuda_profile_stages(s._ctx, DT, ctypes.byref(profile)) == -6  # BEPUCUDA_ERR_BAD_STATE
        assert sum(profile.launches) == 0
        mine = s.referenced_bodies()
        got = s.download()
        assert np.array_equal(sim.bodies[mine][:, util.MOTION].view(np.uint32), got[mine][:, util.MOTION].view(np.uint32))
    finally:
        for s in solvers:
            s.close()
