"""Cost of bepucuda_find_sleepable_islands on C2 (100 k-body pile), C3 (ragdoll tube, 10 k ragdolls) and C4 (1 M-body pile): CUDA events on the
context stream around the call (device work plus the host's one flag read per round), the call's wall clock, and its rounds; beside it the
CPU restatement of CollectIsland that the tests hold the call to (tests/islands/collect_island.cpp) on one host core, as the reference's
single-threaded traversal runs. Every body is a sleep candidate except a seeded 0.1 %, and the device result is checked against the restatement's.
Prints the card and its power limit, then one JSON line per scene."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import bepuphysics2_b200 as bp  # noqa: E402
from bepuphysics2_b200 import native, scenes  # noqa: E402
from tests import island_checker  # noqa: E402

SCENES = {
    "c2_pile_100k": lambda: scenes.shape_pile(100_000, seed=5),
    "c3_ragdoll_tube_10k": lambda: scenes.ragdolls(10_000, seed=5),
    "c4_pile_1m": lambda: scenes.shape_pile(1_000_000, seed=5),
}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True, check=True)
    return q.stdout.strip().splitlines()[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--cpu-calls", type=int, default=3)
    ap.add_argument("--scenes", default=",".join(SCENES))
    args = ap.parse_args()
    os.sched_setaffinity(0, {sorted(os.sched_getaffinity(0))[0]})  # the CPU restatement on one core
    print(json.dumps({"card": card()}), flush=True)
    for name in args.scenes.split(","):
        sim = bp.Simulation(bundle_width=8)
        scenes.build(SCENES[name](), sim)
        n = sim.body_count
        candidates = (np.random.default_rng(1).random(n) >= 0.001).astype(np.uint8)
        activities = np.zeros(n, dtype=native.BODY_ACTIVITY_DTYPE)
        activities["sleep_candidate"] = candidates
        ts = bp.CudaTimestepper(sim)
        ts.describe()
        got = ts.find_sleepable_islands(activities)  # warm-up: module load, scratch buffers
        device_ms, wall_ms = [], []
        for _ in range(args.calls):
            ts.event_record(0)
            t0 = time.perf_counter()
            labels, roots, counts, rounds = ts.find_sleepable_islands(activities)
            wall_ms.append(1e3 * (time.perf_counter() - t0))
            ts.event_record(1)
            device_ms.append(ts.event_elapsed_ms(0, 1))
        ts.close()
        cpu_ms = []
        for _ in range(args.cpu_calls):
            t0 = time.perf_counter()
            want = island_checker.find_sleepable_islands(sim.type_batches(), n, sim.bundle_width, candidates)
            cpu_ms.append(1e3 * (time.perf_counter() - t0))
        assert all(np.array_equal(a, b) for a, b in zip(want, got[:3])), "device and CPU restatement differ on " + name
        stat = lambda v: {"median": round(float(np.median(v)), 3), "min": round(float(np.min(v)), 3), "max": round(float(np.max(v)), 3)}
        print(json.dumps({"scene": name, "bodies": n, "constraints": sim.constraint_count, "islands": int(np.unique(labels).size), "sleepable_islands": int(roots.size),
                          "rounds": rounds, "device_ms": stat(device_ms), "wall_ms": stat(wall_ms), "cpu_one_core_ms": stat(cpu_ms)}), flush=True)


if __name__ == "__main__":
    main()
