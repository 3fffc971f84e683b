"""Measurement: a frame of C2 (the 100 k-body shape pile) in which the game removes a number of bodies (Bodies.Remove: their contacts first) and
fires as many projectiles (Bodies.Add, each with one new contact), sent to the device either as the change calls (bepuhost_cuda_change:
bepucuda_remove_constraints, bepucuda_remove_bodies, bepucuda_add_bodies, bepucuda_add_constraints on the resident state) or as
bepucuda_download_impulses before the host's changes and a full describe after them. Fast build, graph mode, pageable host buffers. Two twin
simulations, one per route, alternate frame by frame; each frame is changes, solve (which re-captures the graph), download_body_motion.
Per route and body count: medians over the timed frames of the device time of the route's calls (CUDA events around them) and of their host wall
clock, the wall clock of the whole frame, and the bytes up. Prints one JSON line per route with the card it ran on, and writes the lines to --out
when given."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import bepuphysics2_b200 as bp  # noqa: E402
from bepuphysics2_b200 import scenes  # noqa: E402

DT = 1.0 / 60.0


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, limit = [x.strip() for x in q.stdout.splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": limit}


def host_changes(sim, rng, count):
    """Bodies.Remove of `count` random bodies, then Bodies.Add of `count` projectiles with one contact each. Returns the constraint adds."""
    sim.remove_bodies(rng.choice(sim.body_handles, size=count, replace=False))
    new = sim.bodies[rng.integers(0, sim.body_count, size=count)].copy()
    new[:, 5] += 3
    new[:, 8:11] = rng.normal(size=(count, 3))
    new[:, 16:23] = [1, 0, 1, 0, 0, 1, 1]
    sim.add_bodies(new)
    added = sim.body_handles[-count:]
    partners = sim.body_handles[rng.integers(0, sim.body_count - count, size=count)]
    prestep = scenes.convex_prestep(rng.uniform(-0.2, 0.2, size=(count, 1, 3)), np.full((count, 1), 0.01), np.tile([0, 1, 0], (count, 1)),
                                    offset_b=rng.uniform(-0.2, 0.2, size=(count, 3)))
    sim.add_constraints(4, np.stack([added, partners], axis=1), prestep)
    return count


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bodies", type=int, default=100_000)
    ap.add_argument("--frames", type=int, default=8, help="timed frames per route and body count")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--counts", default="10,100,1000", help="bodies removed and spawned per frame")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    scene = scenes.shape_pile(args.bodies, seed=5)
    info = card()
    lines = []
    for count in [int(c) for c in args.counts.split(",")]:
        twins = {}
        for route in ("change", "describe"):
            sim = bp.Simulation(bundle_width=8, substeps=8, velocity_iterations=2)
            scenes.build(scene, sim)
            ts = bp.CudaTimestepper(sim, strict_fp=False)
            ts.describe()
            ts.solve_device_only(DT)
            twins[route] = (sim, ts, np.random.default_rng(7))
        samples = {r: {"device_ms": [], "wall_ms": [], "frame_wall_ms": [], "h2d_bytes": []} for r in twins}
        for frame in range(args.warmup + args.frames):
            for route, (sim, ts, rng) in twins.items():
                start = time.perf_counter()
                if route == "change":
                    adds = host_changes(sim, rng, count)
                    t0 = time.perf_counter()
                    ts.event_record(0)
                    ts.change(np.zeros((adds, 4), dtype=np.int32))
                    ts.event_record(1)
                    ts.synchronize()
                    wall = time.perf_counter() - t0
                    device = ts.event_elapsed_ms(0, 1)
                else:
                    t0 = time.perf_counter()
                    ts.event_record(0)
                    ts.download_impulses()
                    ts.event_record(1)
                    wall = time.perf_counter() - t0
                    device = ts.event_elapsed_ms(0, 1)
                    host_changes(sim, rng, count)
                    t0 = time.perf_counter()
                    ts.event_record(2)
                    ts.describe()
                    ts.event_record(3)
                    ts.synchronize()
                    wall += time.perf_counter() - t0
                    device += ts.event_elapsed_ms(2, 3)
                ts.solve_device_only(DT)
                ts.download_body_motion()
                t = ts.timings()
                if frame >= args.warmup:
                    s = samples[route]
                    s["device_ms"].append(device)
                    s["wall_ms"].append(wall * 1e3)
                    s["frame_wall_ms"].append((time.perf_counter() - start) * 1e3)
                    s["h2d_bytes"].append(t.h2d_bytes)
        for route, (sim, ts, _) in twins.items():
            s = samples[route]
            line = dict(info, route=route, count=count, bodies=sim.body_count, constraints=int(sum(tb.constraint_count for tb in sim.type_batches())),
                        frames=args.frames, **{"median_" + k: float(np.median(v)) for k, v in s.items()})
            print(json.dumps(line), flush=True)
            lines.append(line)
            ts.close()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write("\n".join(json.dumps(x) for x in lines) + "\n")


if __name__ == "__main__":
    main()
