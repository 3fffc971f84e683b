"""One constraint graph over several GPUs (SURVEY.md §8e): host-side partitioner + driver of the bepucuda_shard_* entry points.

The reference splits the constraints of every batch over its worker threads (Solver_Solve.cs:L458-654); here the split is over GPUs. Bodies are cut
into contiguous index slabs (the active set of a pile is spatially coherent in index order, like the reference's body memory after its
cache-optimising sorts); a constraint belongs to the rank that owns its first dynamic body. Every rank uploads ALL bodies and only ITS constraints,
compacted, under their original batch indices, so batch k means the same colour on every rank. What crosses GPUs after a (batch, stage): the records
the stage wrote for bodies that another rank references too (direct NVLink peer stores from the lanes that computed them, then a flag barrier).
The sequential fallback batch is the exception: one rank, the fallback rank, owns all of it and uploads its type batches as the host has them.
"""
import ctypes as C

import numpy as np

from . import native

INDEX_MASK = 0x3FFFFFFF      # host body reference: bits 0-29 index, bit 30 kinematic (Bodies_GatherScatter.cs:L107-139)
KINEMATIC_BIT = 1 << 30
INT32_MAX = 0x7FFFFFFF


class IpcHandles(C.Structure):
    _fields_ = [("bytes", (C.c_ubyte * 64) * 4)]


def _constraint_owners(simulation, rank_count):
    """Per type batch: (tb, flat refs [constraint, body slot], body indices, dynamic mask, owner rank: the slab of the constraint's first dynamic body,
    rank 0 if it has none, -1 for a hole), and whether the constraint has a dynamic body."""
    n = simulation.body_count
    owner_of_body = (np.arange(n, dtype=np.int64) * rank_count) // max(n, 1)
    for tb in simulation.type_batches():
        refs = tb.body_references  # [bundles, bodies, W]
        nb = refs.shape[1]
        flat = refs.transpose(0, 2, 1).reshape(-1, nb)[:tb.constraint_count]  # [constraint, body slot]
        valid = flat[:, 0] >= 0
        idx = flat & INDEX_MASK
        dynamic = (flat >= 0) & ((flat & KINEMATIC_BIT) == 0)
        first_dyn = np.argmax(dynamic, axis=1)
        has_dyn = dynamic.any(axis=1)
        first_body = np.where(has_dyn, idx[np.arange(idx.shape[0]), first_dyn], 0)  # holes of the fallback batch have no body
        owner = np.where(has_dyn, owner_of_body[first_body], 0)
        yield tb, flat, idx, dynamic, np.where(valid, owner, -1), valid & has_dyn


def fallback_rank(simulation, rank_count):
    """The rank that runs the whole sequential fallback batch (bepucuda_shard_set_fallback_rank), -1 when the graph has none: the rank whose body slab
    holds the most first dynamic bodies of fallback constraints, the lowest on a tie. It depends on the scene alone, so every rank derives the same."""
    counts, any_fallback = np.zeros(rank_count, dtype=np.int64), False
    for tb, _, _, _, owner, has_dyn in _constraint_owners(simulation, rank_count):
        if tb.batch_index >= simulation.fallback_batch_threshold and tb.constraint_count > 0:
            any_fallback = True
            counts += np.bincount(owner[has_dyn], minlength=rank_count)
    return int(np.argmax(counts)) if any_fallback else -1


def partition(simulation, rank_count):
    """Splits the host simulation's type batches by owner rank. Returns (shards, first_batch, constrained, masks):
    shards[r] = list of dicts {batch_index, type_batch_index, type_id, count, refs, prestep, impulses, source (indices into the global type batch)};
    first_batch[body] = lowest batch referencing it as a dynamic body (INT32_MAX if none); constrained[body]; masks[body] = bit r set when rank r references it.
    Every constraint of the sequential fallback batch belongs to fallback_rank(), whose type batches are the host's verbatim (source = identity):
    the device levelises them by host bundle, so repacking would change the levels and the result."""
    n = simulation.body_count
    W = simulation.bundle_width
    fallback = fallback_rank(simulation, rank_count)
    first_batch = np.full(n, INT32_MAX, dtype=np.int32)
    constrained = np.zeros(n, dtype=np.uint8)
    masks = np.zeros(n, dtype=np.uint8)
    shards = [[] for _ in range(rank_count)]
    per_tb = []
    for tb, flat, idx, dynamic, owner, _ in _constraint_owners(simulation, rank_count):
        if tb.batch_index >= simulation.fallback_batch_threshold:
            owner = np.where(owner >= 0, fallback, -1)
        for s in range(flat.shape[1]):
            sel = (owner >= 0) & dynamic[:, s]
            np.minimum.at(first_batch, idx[sel, s], tb.batch_index)
            constrained[idx[sel, s]] = 1
            np.bitwise_or.at(masks, idx[sel, s], (1 << owner[sel]).astype(np.uint8))
        per_tb.append((tb, flat, idx, dynamic, owner))
    constrained[np.asarray(simulation.constrained_kinematics, dtype=np.int64)] = 1
    for tb, flat, idx, dynamic, owner in per_tb:
        if tb.batch_index >= simulation.fallback_batch_threshold:
            if tb.constraint_count > 0:
                shards[fallback].append({"batch_index": tb.batch_index, "type_batch_index": tb.type_batch_index, "type_id": tb.type_id, "count": tb.constraint_count,
                                         "source": np.arange(tb.constraint_count), "refs": tb.body_references.copy(), "prestep": tb.prestep.copy(),
                                         "impulses": tb.accumulated_impulses.copy(), "idx": idx, "dynamic": dynamic})
            continue
        pre = tb.prestep.transpose(0, 2, 1).reshape(-1, tb.prestep.shape[1])[:tb.constraint_count]
        imp = tb.accumulated_impulses.transpose(0, 2, 1).reshape(-1, tb.accumulated_impulses.shape[1])[:tb.constraint_count]
        for r in range(rank_count):
            mine = np.flatnonzero(owner == r)
            if mine.size == 0:
                continue
            # constraints that write a body another rank references go first: they fill few bundles, which the device schedules ahead of the rest
            # and which alone take part in the stage's flag barrier (ShardStage in bepu_device_types.h)
            boundary = (((masks[idx[mine]] & ~np.uint8(1 << r)) != 0) & dynamic[mine]).any(axis=1)
            mine = np.concatenate([mine[boundary], mine[~boundary]])
            m = mine.size
            bundles = (m + W - 1) // W

            def pack(rows, fill, dtype):
                out = np.full((bundles * W, rows.shape[1]), fill, dtype=dtype)
                out[:m] = rows[mine]
                return np.ascontiguousarray(out.reshape(bundles, W, rows.shape[1]).transpose(0, 2, 1))

            shards[r].append({"batch_index": tb.batch_index, "type_batch_index": tb.type_batch_index, "type_id": tb.type_id, "count": m, "source": mine,
                              "refs": pack(flat, -1, np.int32), "prestep": pack(pre, 0, np.float32), "impulses": pack(imp, 0, np.float32),
                              "idx": idx[mine], "dynamic": dynamic[mine]})
    return shards, first_batch, constrained, masks


class ShardedSolver:
    """One rank of a sharded solve, straight on the C ABI. `exchange_handles(bytes) -> [bytes per rank]` moves the IPC handles between the ranks
    (torch.distributed.all_gather_object in the tools; a direct call when several contexts live in one process)."""

    def __init__(self, simulation, rank, rank_count, device, strict_fp=False, execution_mode=native.EXEC_GRAPH):
        self._cuda, _ = native.load_libraries()
        for name, args in (("bepucuda_shard_export", [C.c_void_p, C.POINTER(IpcHandles)]), ("bepucuda_shard_import", [C.c_void_p, C.c_int32, C.c_int32, C.POINTER(IpcHandles)]),
                           ("bepucuda_shard_set_global", [C.c_void_p, C.c_void_p, C.c_void_p]),
                           ("bepucuda_shard_set_body_masks", [C.c_void_p, C.c_void_p]), ("bepucuda_shard_import_contexts", [C.c_void_p, C.c_int32, C.c_int32, C.POINTER(C.c_void_p)]),
                           ("bepucuda_shard_set_fallback_rank", [C.c_void_p, C.c_int32])):
            getattr(self._cuda, name).argtypes = args
        self.sim, self.rank, self.rank_count = simulation, rank, rank_count
        cfg = native.Config()
        cfg.device_ordinal, cfg.strict_fp, cfg.execution_mode = device, int(bool(strict_fp)), execution_mode
        ctx = C.c_void_p()
        rc = self._cuda.bepucuda_create(C.byref(cfg), C.byref(ctx))
        if rc != 0:
            raise native.BepuCudaError(rc, "bepucuda_create failed")
        self._ctx = ctx
        self.shards, self.first_batch, self.constrained, self.masks = partition(simulation, rank_count)
        self.fallback_rank = fallback_rank(simulation, rank_count)
        self.shard = self.shards[rank]
        self.bodies = simulation.bodies.copy()

    def _check(self, rc):
        if rc != 0:
            raise native.BepuCudaError(rc, self._cuda.bepucuda_last_error(self._ctx).decode())

    def export_handles(self):
        sim = self.sim
        its = (C.c_int32 * len(sim.velocity_iterations))(*sim.velocity_iterations)
        self._check(self._cuda.bepucuda_set_solve_description(self._ctx, len(sim.velocity_iterations), its, sim.fallback_batch_threshold))
        self._check(self._cuda.bepucuda_set_integrator(self._ctx, C.byref(sim.integrator)))
        self._check(self._cuda.bepucuda_upload_bodies(self._ctx, self.bodies.ctypes.data, sim.body_count))
        h = IpcHandles()
        self._check(self._cuda.bepucuda_shard_export(self._ctx, C.byref(h)))
        return bytes(h)

    def import_handles(self, all_handles):
        arr = (IpcHandles * self.rank_count)()
        for r, raw in enumerate(all_handles):
            C.memmove(C.byref(arr[r]), raw, C.sizeof(IpcHandles))
        self._check(self._cuda.bepucuda_shard_import(self._ctx, self.rank, self.rank_count, arr))

    def import_contexts(self, solvers):
        """All ranks in this process: `solvers` in rank order (each after export_handles)."""
        arr = (C.c_void_p * self.rank_count)(*[s._ctx for s in solvers])
        self._check(self._cuda.bepucuda_shard_import_contexts(self._ctx, self.rank, self.rank_count, arr))

    def describe(self):
        sim = self.sim
        self._check(self._cuda.bepucuda_shard_set_global(self._ctx, self.first_batch.ctypes.data, self.constrained.ctypes.data))
        if self.fallback_rank >= 0:
            self._check(self._cuda.bepucuda_shard_set_fallback_rank(self._ctx, self.fallback_rank))
        self._check(self._cuda.bepucuda_begin_constraints(self._ctx, sim.bundle_width, sim.batch_count))
        for tb in self.shard:
            self._check(self._cuda.bepucuda_upload_type_batch(self._ctx, tb["batch_index"], tb["type_batch_index"], tb["type_id"], tb["count"], tb["refs"].ctypes.data,
                                                              tb["prestep"].ctypes.data, tb["impulses"].ctypes.data))
        self._check(self._cuda.bepucuda_shard_set_body_masks(self._ctx, self.masks.ctypes.data))
        kin = np.ascontiguousarray(sim.constrained_kinematics, dtype=np.int32)
        self._check(self._cuda.bepucuda_set_constrained_kinematics(self._ctx, kin.ctypes.data if kin.size else None, int(kin.size)))
        self._check(self._cuda.bepucuda_end_constraints(self._ctx))

    def solve(self, dt):
        self._check(self._cuda.bepucuda_solve(self._ctx, dt))

    def synchronize(self):
        self._check(self._cuda.bepucuda_synchronize(self._ctx))

    def timings(self):
        t = native.Timings()
        self._check(self._cuda.bepucuda_get_timings(self._ctx, C.byref(t)))
        return t

    def download(self):
        """Bodies (valid for the bodies this rank references) and this rank's impulses / prestep back into its shard arrays."""
        self._check(self._cuda.bepucuda_download_bodies(self._ctx, self.bodies.ctypes.data, self.sim.body_count))
        self._check(self._cuda.bepucuda_download_impulses(self._ctx))
        for tb in self.shard:
            self._check(self._cuda.bepucuda_download_prestep(self._ctx, tb["batch_index"], tb["type_batch_index"], tb["prestep"].ctypes.data))
        return self.bodies

    def referenced_bodies(self):
        return np.flatnonzero((self.masks >> self.rank) & 1)

    def close(self):
        if getattr(self, "_ctx", None):
            self._cuda.bepucuda_destroy(self._ctx)
            self._ctx = None
