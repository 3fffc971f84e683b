"""Cost of bepucuda_read_constraints on C2 (100 k-body pile, 333 k manifolds, 8 substeps x 2 iterations) for 1, 1 000, 100 000 and every location,
against what a host needs without it: bepucuda_download_impulses plus bepucuda_download_prestep of every type batch. Each is timed with CUDA
events on the context stream around the call and with the wall clock around it (every call blocks until its results are on the host); the
median over --calls calls after one warm-up call. The records go either to a new pageable array per call (what read_constraints does without
`out`; the copy then also pays the array's first-touch page faults) or to one registered, page-locked buffer reused by every call, as a host
that reads every frame keeps it. The locations are a seeded random sample of the scene's. Prints the card and its power limit, then one JSON
line per measurement."""
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
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True, check=True)
    return q.stdout.strip().splitlines()[0]


def timed(ts, call, calls):
    """Median event time and wall time of `calls` calls after one warm-up call."""
    call()
    events, walls = [], []
    for _ in range(calls):
        ts.synchronize()
        t0 = time.perf_counter()
        ts.event_record(0)
        call()
        ts.event_record(1)
        walls.append((time.perf_counter() - t0) * 1e3)
        events.append(ts.event_elapsed_ms(0, 1))
    return float(np.median(events)), float(np.median(walls))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--bodies", type=int, default=100_000)
    args = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    sim = bp.Simulation(bundle_width=8, substeps=8, velocity_iterations=2)
    scenes.build(scenes.shape_pile(args.bodies, seed=5), sim)
    ts = bp.CudaTimestepper(sim, strict_fp=False)
    ts.register_host_buffers()
    ts.describe()
    ts.solve_device_only(DT)
    everything = sim.constraint_locations()
    # the records as a host keeps them across frames: one page-locked buffer, registered once (bepucuda_host_register)
    backing = np.zeros(len(everything) * 64 + 2048, dtype=np.int32)  # page-aligned start and a whole number of pages
    skip = (-backing.ctypes.data % 4096) // 4
    pinned = backing[skip:skip + ((len(everything) * 64 + 1023) // 1024) * 1024]
    ts.register_array(pinned)
    rng = np.random.default_rng(1)
    for n in (1, 1000, 100_000, len(everything)):
        locations = everything if n == len(everything) else everything[rng.choice(len(everything), size=n, replace=False)]
        for output, out in (("new_pageable_array", None), ("registered_buffer", pinned)):
            ms, wall = timed(ts, lambda: ts.read_constraints(locations, out=out), args.calls)
            print(json.dumps({"call": "read_constraints", "output": output, "locations": n, "event_ms": ms, "wall_ms": wall, "bytes_out": n * 256}), flush=True)
    ms, wall = timed(ts, lambda: (ts.download_impulses(), ts.download_prestep()), args.calls)
    print(json.dumps({"call": "download_impulses+download_prestep", "constraints": len(everything), "type_batches": len(sim.type_batches()), "event_ms": ms,
                      "wall_ms": wall}), flush=True)
    ts.close()


if __name__ == "__main__":
    main()
