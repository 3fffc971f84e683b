"""Cost of the optional velocity terms (bepucuda_set_body_accelerations + bepucuda_set_point_gravity) on the bench's C2 (100 k-body pile, 8 x 2)
and C3 (ragdoll tube, 1 x 4) scenes: the same scene on two contexts, one with random per-body accelerations and an attractor, one without,
timed in alternating rounds of device-resident graph solves (CUDA events on the context stream). Prints one JSON line per scene."""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import bepuphysics2_b200 as bp  # noqa: E402
from bepuphysics2_b200 import scenes  # noqa: E402

DT = 1.0 / 60.0
SCENES = {
    "c2_pile_100k_8x2": (lambda: scenes.shape_pile(100_000, seed=5), 8, 2),
    "c3_ragdoll_tube_10k_1x4": (lambda: scenes.ragdolls(10_000, seed=5), 1, 4),
}


def timed(ts, steps):
    ts.event_record(0)
    for _ in range(steps):
        ts.solve_device_only(DT)
    ts.event_record(1)
    return ts.event_elapsed_ms(0, 1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--steps", type=int, default=50)
    args = ap.parse_args()
    for name, (make, substeps, iterations) in SCENES.items():
        sim = bp.Simulation(bundle_width=8, substeps=substeps, velocity_iterations=iterations)
        scenes.build(make(), sim)
        plain, ext = bp.CudaTimestepper(sim), bp.CudaTimestepper(sim)
        for ts in (plain, ext):
            ts.describe()
        acc = np.random.default_rng(1).uniform(-1, 1, size=(sim.body_count, 8)).astype(np.float32)
        acc[:, 3] = acc[:, 7] = 0.0
        ext.set_body_accelerations(acc)
        ext.set_point_gravity((0.0, -1000.0, 0.0), 1.0e5)
        for ts in (plain, ext):
            timed(ts, 5)  # graph capture and warm-up
        ms = {"plain": [], "extensions": []}
        for _ in range(args.rounds):
            ms["plain"].append(timed(plain, args.steps))
            ms["extensions"].append(timed(ext, args.steps))
        out = {"scene": name, "bodies": sim.body_count, "steps_per_round": args.steps}
        for k, v in ms.items():
            out[k + "_ms"] = {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))}
        out["overhead_pct"] = 100.0 * (out["extensions_ms"]["median"] / out["plain_ms"]["median"] - 1.0)
        print(json.dumps(out), flush=True)
        plain.close()
        ext.close()


if __name__ == "__main__":
    main()
