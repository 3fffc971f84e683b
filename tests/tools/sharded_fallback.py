"""One constraint graph WITH a sequential fallback batch over N GPUs (bepucuda_shard_*, bepucuda_shard_set_fallback_rank), one process per GPU. The
scene is config 5 (fallback stress: hubs with far more than FallbackBatchThreshold constraints), so most constraints run in the fallback levels of
the fallback rank while the other ranks wait at one exchange point per fallback section:

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29513 tests/tools/sharded_fallback.py --check --bodies 20000
    ... tests/tools/sharded_fallback.py --bodies 50000 --substeps 1 --iterations 4 --steps 20        (timing; prints one line on rank 0)

--check: strict build, every rank compares the bodies it references and its own constraints' impulses (live lanes) with the oracle's solve of the
WHOLE graph, bit for bit, over several frames. Expect no speedup over one GPU: the fallback section is serial on one GPU, as it is on one worker in
the reference."""
import argparse
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import torch
import torch.distributed as dist

import bepuphysics2_b200 as bp
from bepuphysics2_b200 import scenes, sharding

ap = argparse.ArgumentParser()
ap.add_argument("--bodies", type=int, default=20000)
ap.add_argument("--substeps", type=int, default=1)
ap.add_argument("--iterations", type=int, default=4)
ap.add_argument("--frames", type=int, default=3)
ap.add_argument("--steps", type=int, default=20)
ap.add_argument("--check", action="store_true")
ap.add_argument("--stream", action="store_true")
args = ap.parse_args()

rank, world, local = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
DT = 1.0 / 60.0

scene = scenes.fallback_stress(args.bodies, hubs=max(1, args.bodies // 1000), seed=5)
sim = bp.Simulation(bundle_width=8, substeps=args.substeps, velocity_iterations=args.iterations)
scenes.build(scene, sim)
solver = sharding.ShardedSolver(sim, rank, world, local, strict_fp=args.check, execution_mode=bp.native.EXEC_STREAM if args.stream else bp.native.EXEC_GRAPH)
mine = solver.export_handles()
gathered = [None] * world
dist.all_gather_object(gathered, mine)
solver.import_handles(gathered)
solver.describe()
solver.synchronize()
dist.barrier()
levels = solver.timings().fallback_level_count

if args.check:
    from oracle import binding as ob

    for _ in range(args.frames):
        ob.solve(sim, DT)
        solver.solve(DT)
    got = solver.download()
    ref = sim.bodies
    mine_bodies = solver.referenced_bodies()
    ok = True
    for label, cols in (("poses", np.r_[0:7]), ("linear velocities", np.r_[8:11]), ("angular velocities", np.r_[12:15])):
        diff = (ref[mine_bodies][:, cols].view(np.uint32) != got[mine_bodies][:, cols].view(np.uint32)).any(axis=1)
        if diff.any():
            ok = False
            print("rank %d: %s differ for %d of %d referenced bodies (first body %d)" % (rank, label, diff.sum(), mine_bodies.size, mine_bodies[np.flatnonzero(diff)[0]]), flush=True)
    by_key = {(tb.batch_index, tb.type_batch_index): tb for tb in sim.type_batches()}
    for d in solver.shard:
        g = by_key[(d["batch_index"], d["type_batch_index"])]
        nb = g.body_references.shape[1]
        if d["batch_index"] >= sim.fallback_batch_threshold:  # the host's own type batch: its live lanes
            lanes = np.flatnonzero(g.body_references.transpose(0, 2, 1).reshape(-1, nb)[:g.constraint_count, 0] >= 0)
            ref_lanes, have_lanes = lanes, lanes
        else:
            ref_lanes, have_lanes = d["source"], np.arange(d["count"])
        ref_imp = g.accumulated_impulses.transpose(0, 2, 1).reshape(-1, g.accumulated_impulses.shape[1])[ref_lanes]
        got_imp = d["impulses"].transpose(0, 2, 1).reshape(-1, d["impulses"].shape[1])[have_lanes]
        if not np.array_equal(ref_imp.view(np.uint32), got_imp.view(np.uint32)):
            ok = False
            print("rank %d: impulses of batch %d type %d differ" % (rank, d["batch_index"], d["type_id"]), flush=True)
            break
    flag = torch.tensor([1 if ok else 0], device="cuda")
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    if rank == 0:
        print("sharded over %d GPUs with the fallback batch on rank %d (%d levels): %d bodies, %d constraints, %d frames of %d x %d: %s" % (
            world, solver.fallback_rank, levels, args.bodies, sim.constraint_count, args.frames, args.substeps, args.iterations,
            "BIT-EXACT vs the oracle on every rank" if flag.item() else "MISMATCH"), flush=True)
    code = 0 if flag.item() else 1
else:
    for _ in range(3):
        solver.solve(DT)
    solver.synchronize()
    ms = []
    for _ in range(args.steps):
        dist.barrier()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        solver.solve(DT)
        solver.synchronize()
        ms.append((time.perf_counter() - t0) * 1e3)
    t = solver.timings()
    dev_ms = torch.tensor([float(np.median(ms)), t.solve_ms], device="cuda", dtype=torch.float64)
    dist.all_reduce(dev_ms, op=dist.ReduceOp.MAX)
    if rank == 0:
        name = torch.cuda.get_device_name(local)
        print("%s x %d, fallback batch on rank %d (%d levels): %d bodies, %d constraints, %d x %d: wall %.3f ms/step (median), device %.3f ms/step (max over ranks)" % (
            name, world, solver.fallback_rank, levels, args.bodies, sim.constraint_count, args.substeps, args.iterations, dev_ms[0].item(), dev_ms[1].item()), flush=True)
    code = 0
solver.close()
dist.barrier()
dist.destroy_process_group()
sys.exit(code)
