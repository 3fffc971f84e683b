"""Shared helpers of the test-suite: build identical host simulations, run the oracle / the GPU on them, compare buffers."""
import numpy as np

import bepuphysics2_b200 as bp
from bepuphysics2_b200 import scenes
from oracle import binding as ob

MEANINGFUL = np.r_[0:7, 8:11, 12:15, 16:23, 24:31]  # floats of a BodyDynamics record that carry data (padding excluded)
MOTION = np.r_[0:7, 8:11, 12:15]


def make_sim(scene, bundle_width=8, substeps=1, velocity_iterations=1, fallback_batch_threshold=64, integrator=None):
    sim = bp.Simulation(bundle_width=bundle_width, fallback_batch_threshold=fallback_batch_threshold, substeps=substeps, velocity_iterations=velocity_iterations, integrator=integrator)
    scenes.build(scene, sim)
    return sim


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


def run_gpu(sim, dt, frames=1, strict=True, mode=0, download_prestep=True):
    ts = bp.CudaTimestepper(sim, strict_fp=strict, execution_mode=mode)
    try:
        ts.describe()
        for f in range(frames):
            if f > 0:
                ts.refresh()
            ts.solve(dt, download=True)
            if download_prestep:
                ts.download_prestep()
        timings = ts.timings()
    finally:
        ts.close()
    snap = snapshot(sim)
    snap["timings"] = timings.as_dict()
    return snap


def compare(a, b, exact=True, rel_rms=1e-3, max_abs=5e-2):
    """Asserts two snapshots agree: bodies (meaningful floats), accumulated impulses and prestep on valid lanes.
    exact: bit-for-bit (the strict -fmad=false build against the non-contracting oracle).
    otherwise (FMA-contracted, approximate sqrt build): per quantity, relative RMS error <= rel_rms and max abs error <= max_abs."""
    def check(x, y, what):
        if exact:
            # bit patterns only: -0.0 against +0.0 is a difference, and so are two NaNs with different payloads
            bits_x, bits_y = np.ascontiguousarray(x).view(np.uint32), np.ascontiguousarray(y).view(np.uint32)
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
