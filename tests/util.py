"""Shared helpers of the test-suite: build identical host simulations, run the oracle / the GPU on them, compare buffers."""
import ctypes as C
from concurrent.futures import ThreadPoolExecutor

import numpy as np

import bepuphysics2_b200 as bp
from bepuphysics2_b200 import native, scenes, sharding
from oracle import binding as ob

EXECUTION_MODES = {"graph": native.EXEC_GRAPH, "stream": native.EXEC_STREAM}
MEANINGFUL = np.r_[0:7, 8:11, 12:15, 16:23, 24:31]  # floats of a BodyDynamics record that carry data (padding excluded)
MOTION = np.r_[0:7, 8:11, 12:15]


def make_sim(scene, bundle_width=8, substeps=1, velocity_iterations=1, fallback_batch_threshold=64, integrator=None):
    sim = bp.Simulation(bundle_width=bundle_width, fallback_batch_threshold=fallback_batch_threshold, substeps=substeps, velocity_iterations=velocity_iterations, integrator=integrator)
    scenes.build(scene, sim)
    return sim


def integrator(**fields):
    """IntegratorDesc.default() with the named fields set (gravity as a 3-sequence)."""
    d = bp.IntegratorDesc.default()
    for name, value in fields.items():
        if name == "gravity":
            for i in range(3):
                d.gravity[i] = value[i]
        else:
            assert hasattr(d, name), name
            setattr(d, name, value)
    return d


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def float_ptr(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def punch_fallback_holes(sim, every=5):
    """Empties every `every`-th lane of the fallback type batches in place (what removing a constraint from the fallback batch leaves behind)."""
    punched = 0
    for tb in sim.type_batches():
        if tb.batch_index < sim.fallback_batch_threshold:
            continue
        W = tb.body_references.shape[2]
        for i in range(0, tb.constraint_count - 1, every):  # interior lanes: the last one keeps ConstraintCount meaningful
            tb.body_references[i // W, :, i % W] = -1
            punched += 1
    return punched


def snapshot(sim):
    """Copies of everything the solve mutates: bodies, per type batch prestep and accumulated impulses (valid lanes only)."""
    out = {"bodies": sim.bodies.copy(), "type_batches": []}
    for tb in sim.type_batches():
        refs = tb.body_references
        valid = refs[:, 0, :] >= 0
        out["type_batches"].append({"key": (tb.batch_index, tb.type_batch_index, tb.type_id), "valid": valid, "prestep": tb.prestep.copy(), "impulses": tb.accumulated_impulses.copy()})
    return out


def run_oracle(sim, dt, frames=1, threads=1, simd=False, accelerations=None, center=None, strength=0.0):
    for _ in range(frames):
        ob.solve(sim, dt, threads=threads, simd=simd, accelerations=accelerations, center=center, strength=strength)
    return snapshot(sim)


def run_gpu(sim, dt, frames=1, strict=True, mode=0, download_prestep=True, terms=None, profile=False, resident=False):
    """`frames` frames of `sim` on the device, refreshed from the host between them. terms = (accelerations, center, strength): set right after
    describe. profile: each frame runs through profile_stages, then download_bodies and download_impulses. resident: every frame but the last is
    solve_device_only, and nothing is refreshed. The snapshot also carries the timings and "launches": the launch count of the last profile, or
    timings().kernel_launches."""
    ts = bp.CudaTimestepper(sim, strict_fp=strict, execution_mode=mode)
    try:
        ts.describe()
        if terms is not None:
            ts.set_body_accelerations(terms[0])
            ts.set_point_gravity(terms[1], terms[2])
        for f in range(frames):
            if resident and f < frames - 1:
                ts.solve_device_only(dt)
                continue
            if f > 0 and not resident:
                ts.refresh()
            if profile:
                launches = sum(ts.profile_stages(dt).launches)
                ts.download_bodies()
                ts.download_impulses()
            else:
                ts.solve(dt, download=True)
            if download_prestep:
                ts.download_prestep()
        timings = ts.timings()
    finally:
        ts.close()
    snap = snapshot(sim)
    snap["timings"] = timings.as_dict()
    snap["launches"] = launches if profile else timings.kernel_launches
    return snap


def solve_all(solvers, dt):
    """One frame on every rank, each issued from a host thread of its own (one host thread per context, include/bepucuda.h): a rank's issuing
    thread blocks once its launch queue is full (the fallback rank issues a launch per level and section, thousands per frame) until the device
    drains it, which needs the other ranks' frames issued too."""
    with ThreadPoolExecutor(max_workers=len(solvers)) as pool:
        list(pool.map(lambda s: s.solve(dt), solvers))


def run_ranks(scene, rank_count, frames, mode, dt=1.0 / 60.0, **kw):
    """`rank_count` contexts on device 0, wired to one another with bepucuda_shard_import_contexts, against the oracle run on the whole graph, bit
    for bit after `frames` frames: every rank's referenced bodies and its own live constraints' impulses and prestep rows (contact depths written by
    the incremental update). A fallback type batch is the host's own (source = identity): its live lanes are compared; a synchronized one is
    compacted: `source` against arange(count). `mode`: a key of EXECUTION_MODES. Returns the solvers' fallback rank (-1 = no fallback batch)."""
    sim = make_sim(scene, **kw)
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
        assert all(s.fallback_rank == fallback for s in solvers)
        for s in solvers:
            assert (s.timings().fallback_level_count > 0) == (s.rank == fallback)
        for _ in range(frames):
            ob.solve(sim, dt)
            solve_all(solvers, dt)  # the ranks' frames run side by side on the device and meet at their exchange points
        by_key = {(tb.batch_index, tb.type_batch_index): tb for tb in sim.type_batches()}
        for s in solvers:
            got = s.download()
            mine = s.referenced_bodies()
            assert mine.size > 0
            assert np.array_equal(sim.bodies[mine][:, MOTION].view(np.uint32), got[mine][:, MOTION].view(np.uint32)), "rank %d bodies (%s)" % (s.rank, mode)
            for d in s.shard:
                g = by_key[(d["batch_index"], d["type_batch_index"])]
                if d["batch_index"] >= sim.fallback_batch_threshold:
                    live = np.flatnonzero(g.body_references.transpose(0, 2, 1).reshape(-1, g.body_references.shape[1])[:g.constraint_count, 0] >= 0)
                    ref_lanes, have_lanes = live, live
                else:
                    ref_lanes, have_lanes = d["source"], np.arange(d["count"])
                for what, ref_rows in (("impulses", g.accumulated_impulses), ("prestep", g.prestep)):
                    ref = ref_rows.transpose(0, 2, 1).reshape(-1, ref_rows.shape[1])[ref_lanes]
                    have = d[what].transpose(0, 2, 1).reshape(-1, d[what].shape[1])[have_lanes]
                    assert np.array_equal(ref.view(np.uint32), have.view(np.uint32)), "rank %d %s of batch %d (%s)" % (s.rank, what, d["batch_index"], mode)
        assert int(((solvers[0].masks & (solvers[0].masks - 1)) != 0).sum()) > 0
        return fallback
    finally:
        for s in solvers:
            s.close()


def compare(a, b, exact=True, rel_rms=1e-3, max_abs=5e-2):
    """Asserts two snapshots agree: bodies (meaningful floats), accumulated impulses and prestep on valid lanes.
    exact: bit-for-bit (the strict -fmad=false build against the non-contracting oracle).
    otherwise (FMA-contracted, approximate sqrt build): per quantity, relative RMS error <= rel_rms and max abs error <= max_abs."""
    def check(x, y, what):
        if exact:
            # bit patterns only: -0.0 against +0.0 is a difference, and so are two NaNs with different payloads
            bits_x, bits_y = bits(x), bits(y)
            if not np.array_equal(bits_x, bits_y):
                bad = np.argwhere(bits_x != bits_y)
                diff = np.abs(x.astype(np.float64) - y.astype(np.float64))
                raise AssertionError("%s differs at %d positions (first %s), max abs diff %g" % (what, bad.shape[0], bad[0].tolist(), np.nanmax(diff)))
        else:
            x64, y64 = x.astype(np.float64), y.astype(np.float64)
            assert np.isfinite(y64).all(), "%s: non-finite values" % what
            d = np.abs(x64 - y64)
            denom = np.sqrt((x64 ** 2).sum())
            rms = np.sqrt((d ** 2).sum()) / denom if denom > 0 else d.max(initial=0.0)
            assert rms <= rel_rms, "%s: relative RMS error %.3e > %.1e" % (what, rms, rel_rms)
            assert d.max(initial=0.0) <= max_abs, "%s: max abs error %.3e > %.1e" % (what, d.max(), max_abs)

    for label, cols in (("body poses", np.r_[0:7]), ("body linear velocities", np.r_[8:11]), ("body angular velocities", np.r_[12:15]), ("body inertias", np.r_[16:23, 24:31])):
        check(a["bodies"][:, cols], b["bodies"][:, cols], label)
    assert len(a["type_batches"]) == len(b["type_batches"])
    for ta, tb in zip(a["type_batches"], b["type_batches"]):
        assert ta["key"] == tb["key"]
        va = np.broadcast_to(ta["valid"][:, None, :], ta["impulses"].shape)
        check(np.where(va, ta["impulses"], 0), np.where(va, tb["impulses"], 0), "impulses of type batch %s" % (ta["key"],))
        vp = np.broadcast_to(ta["valid"][:, None, :], ta["prestep"].shape)
        check(np.where(vp, ta["prestep"], 0), np.where(vp, tb["prestep"], 0), "prestep of type batch %s" % (ta["key"],))
