"""Cost of a motor change on the resident path: C3 (10 k ragdolls, 150 k AngularMotors, 4 substeps x 8 iterations) with the target velocity of
every ragdoll's 15 AngularMotors changed every frame, through
  write:        bepucuda_write_constraints of the changed motors, then the solve;
  write_one:    the same for one ragdoll's 15 motors only (a frame in which one car or tank steers);
  type_batch:   what a host needs without it: bepucuda_download_impulses (the host's impulses are stale after the first resident frame), then
                bepucuda_update_type_batch of every AngularMotor type batch, then the solve;
  no_change:    the solve alone.
The new targets are written into the records / the host's prestep buffers (Solver.ApplyDescription) before the timed window. Per frame: CUDA
events on the context stream around the route's calls and the solve, the upload window and solve time the context reports (bepucuda_timings
upload_ms + solve_ms), and the wall clock around the same calls and a synchronize; the median over --frames frames after --warmup, with the routes
taking turns frame by frame. Prints the card and its power limit, then one JSON line per route."""
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
ANGULAR_MOTOR = 30


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True, check=True)
    return q.stdout.strip().splitlines()[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ragdolls", type=int, default=10_000)
    ap.add_argument("--frames", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    sim = bp.Simulation(bundle_width=8, substeps=4, velocity_iterations=8)
    scenes.build(scenes.ragdolls(args.ragdolls, seed=5, motor="motor"), sim)
    ts = bp.CudaTimestepper(sim, strict_fp=False)
    ts.register_host_buffers()
    ts.describe()
    ts.solve_device_only(DT)
    W = sim.bundle_width
    motors = [tb for tb in sim.type_batches() if tb.type_id == ANGULAR_MOTOR]
    locations = sim.constraint_locations()
    locations = locations[locations[:, 1] == ANGULAR_MOTOR]
    assert len(locations) == 15 * args.ragdolls, len(locations)
    records = ts.read_constraints(locations)
    rng = np.random.default_rng(3)

    def describe_write():
        records[:, 18:21] = rng.uniform(-1, 1, (len(locations), 3)).astype(np.float32).view(np.int32)

    def write_route():
        ts.write_constraints(locations, records)

    def write_one_route():
        ts.write_constraints(locations[:15], records[:15])

    def describe_type_batch():
        for tb in motors:
            tb.prestep[:, 0:3, :] = rng.uniform(-1, 1, (tb.bundle_count, 3, W)).astype(np.float32)

    def type_batch_route():
        ts.download_impulses()
        for tb in motors:
            ts._check(ts._cuda.bepucuda_update_type_batch(ts._ctx, tb.batch_index, tb.type_batch_index, tb.prestep.ctypes.data, tb.accumulated_impulses.ctypes.data))

    routes = {"write": (describe_write, write_route), "write_one": (describe_write, write_one_route), "type_batch": (describe_type_batch, type_batch_route), "no_change": (lambda: None, lambda: None)}
    results = {name: {"event_ms": [], "upload_plus_solve_ms": [], "wall_ms": [], "h2d_bytes": 0} for name in routes}
    # the routes alternate frame by frame, so that drift of the clocks or of other work on the card falls on all of them alike
    for frame in range(args.warmup + args.frames):
        for name, (describe, route) in routes.items():
            describe()
            ts.synchronize()
            t0 = time.perf_counter()
            ts.event_record(0)
            route()
            ts.solve_device_only(DT)
            ts.event_record(1)
            ts.synchronize()
            wall = (time.perf_counter() - t0) * 1e3
            t = ts.timings()
            if frame >= args.warmup:
                r = results[name]
                r["event_ms"].append(ts.event_elapsed_ms(0, 1))
                r["upload_plus_solve_ms"].append((t.upload_ms if name != "no_change" else 0.0) + t.solve_ms)
                r["wall_ms"].append(wall)
                r["h2d_bytes"] = int(t.h2d_bytes)
    for name, r in results.items():
        print(json.dumps({"route": name, "changed_motors": {"write_one": 15, "no_change": 0}.get(name, len(locations)), "frames": args.frames,
                          "event_ms": float(np.median(r["event_ms"])), "upload_plus_solve_ms": float(np.median(r["upload_plus_solve_ms"])),
                          "wall_ms": float(np.median(r["wall_ms"])), "h2d_bytes": r["h2d_bytes"]}), flush=True)
    ts.close()


if __name__ == "__main__":
    main()
