"""Development sweep (not part of the bench contract): device-resident ms/step of one scene under different execution modes."""
import argparse
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import numpy as np
import torch

import bepuphysics2_b200 as bp
from bepuphysics2_b200 import scenes
from bepuphysics2_b200.native import EXEC_GRAPH, EXEC_STREAM

ap = argparse.ArgumentParser()
ap.add_argument("--bodies", type=int, default=100_000)
ap.add_argument("--scene", default="shape_pile")
ap.add_argument("--substeps", type=int, default=8)
ap.add_argument("--iterations", type=int, default=2)
ap.add_argument("--steps", type=int, default=10)
ap.add_argument("--cpu", action="store_true")
args = ap.parse_args()
DT = 1 / 60

if args.scene == "shape_pile":
    scene = scenes.shape_pile(args.bodies, seed=5)
elif args.scene == "ragdolls":
    scene = scenes.ragdolls(args.bodies // 16, seed=5)
else:
    scene = scenes.fallback_stress(args.bodies, hubs=max(1, args.bodies // 1000), seed=5)
print(scene["description"], flush=True)
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")


def run(mode, do_flush=True, strict=False):
    sim = bp.Simulation(substeps=args.substeps, velocity_iterations=args.iterations)
    t0 = time.time()
    scenes.build(scene, sim)
    build_s = time.time() - t0
    ts = bp.CudaTimestepper(sim, strict_fp=strict, execution_mode=mode)
    t0 = time.time()
    ts.describe()
    ts.synchronize()
    describe_s = time.time() - t0
    ms = []
    for i in range(args.steps + 3):
        if do_flush:
            flush.fill_(1)
            torch.cuda.synchronize()
        ts.solve_device_only(DT)
        t = ts.timings()
        if i >= 3:
            ms.append(t.solve_ms)
    ci = t.constraint_iterations
    name = {EXEC_GRAPH: "graph", EXEC_STREAM: "stream"}[mode]
    print("%-10s flush=%d strict=%d : %.3f ms/step (min %.3f)  %.2f G CI/s  batches=%d stages=%d alg=%.1f GB/s  [build %.1fs describe %.2fs]" % (
        name, do_flush, strict, np.mean(ms), np.min(ms), ci / np.mean(ms) / 1e6, t.device_batch_count, t.stage_count, t.algorithmic_bytes / np.mean(ms) / 1e6, build_s, describe_s), flush=True)
    ts.close()


run(EXEC_GRAPH)
if os.environ.get("SWEEP", "full") != "graph":
    run(EXEC_STREAM)
    run(EXEC_GRAPH, strict=True)

if args.cpu:
    from oracle import binding as ob

    print("affinity", len(os.sched_getaffinity(0)), "cpu.max", open("/sys/fs/cgroup/cpu.max").read().strip() if os.path.exists("/sys/fs/cgroup/cpu.max") else None, flush=True)
    for threads in (1, 8, 16, 32, 64, 128):
        sim = bp.Simulation(substeps=args.substeps, velocity_iterations=args.iterations)
        scenes.build(scene, sim)
        ob.solve(sim, DT, threads=threads, simd=True)
        t0 = time.time()
        ob.solve(sim, DT, threads=threads, simd=True)
        dt = time.time() - t0
        print("cpu threads=%d: %.1f ms/frame  %.1f M CI/s" % (threads, dt * 1e3, sim.constraint_count * args.substeps * args.iterations / dt / 1e6), flush=True)
