"""Minimal ncu target: build one scene, describe it, run a couple of frames as plain stream launches (no graph) so every stage is its own kernel."""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bepuphysics2_b200 as bp
from bepuphysics2_b200 import scenes
from bepuphysics2_b200.native import EXEC_STREAM

ap = argparse.ArgumentParser()
ap.add_argument("--bodies", type=int, default=100_000)
ap.add_argument("--scene", default="shape_pile")
ap.add_argument("--frames", type=int, default=2)
ap.add_argument("--substeps", type=int, default=8)
ap.add_argument("--iterations", type=int, default=2)
args = ap.parse_args()
scene = scenes.shape_pile(args.bodies, seed=5) if args.scene == "shape_pile" else scenes.ragdolls(args.bodies // 16, seed=5)
sim = bp.Simulation(substeps=args.substeps, velocity_iterations=args.iterations)
scenes.build(scene, sim)
ts = bp.CudaTimestepper(sim, execution_mode=EXEC_STREAM)
ts.describe()
for _ in range(args.frames):
    ts.solve_device_only(1 / 60)
ts.synchronize()
t = ts.timings()
print(scene["description"], "solve_ms", t.solve_ms, "batches", t.device_batch_count)
ts.close()
