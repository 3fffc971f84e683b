"""One constraint graph over N GPUs with NVLink peer stores + flag barrier (bepucuda_shard_*), one process per GPU:

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29511 tests/tools/sharded_peer.py --check --bodies 20000
    ... tests/tools/sharded_peer.py --bodies 1000000 --substeps 4 --iterations 2 --steps 20        (timing; prints one line on rank 0)

--check: strict build, every rank compares the bodies it references and its own constraints' impulses with the oracle's single-threaded solve of
the WHOLE graph, bit for bit, over several frames."""
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
ap.add_argument("--substeps", type=int, default=4)
ap.add_argument("--iterations", type=int, default=2)
ap.add_argument("--frames", type=int, default=3)
ap.add_argument("--steps", type=int, default=20)
ap.add_argument("--check", action="store_true")
ap.add_argument("--stream", action="store_true")
args = ap.parse_args()

rank, world, local = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
torch.cuda.set_device(local)
if os.environ.get("NCCL_DEBUG", "").upper() == "VERSION":
    os.environ["NCCL_DEBUG"] = "WARN"
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
DT = 1.0 / 60.0

scene = scenes.shape_pile(args.bodies, seed=5)
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

if args.check:
    from oracle import binding as ob

    for _ in range(args.frames):
        ob.solve(sim, DT, threads=8, simd=True)
        solver.solve(DT)
    got = solver.download()
    ref = sim.bodies
    mine_bodies = solver.referenced_bodies()
    ok = True
    for label, cols in (("poses", np.r_[0:7]), ("linear velocities", np.r_[8:11]), ("angular velocities", np.r_[12:15])):
        same = np.array_equal(ref[mine_bodies][:, cols].view(np.uint32), got[mine_bodies][:, cols].view(np.uint32))
        ok &= same
        if not same:
            bad = np.flatnonzero((ref[mine_bodies][:, cols].view(np.uint32) != got[mine_bodies][:, cols].view(np.uint32)).any(axis=1))
            print("rank %d: %s differ for %d of %d referenced bodies (first body %d)" % (rank, label, bad.size, mine_bodies.size, mine_bodies[bad[0]]), flush=True)
    by_key = {(tb.batch_index, tb.type_batch_index): tb for tb in sim.type_batches()}
    for tb in solver.shard:
        g = by_key[(tb["batch_index"], tb["type_batch_index"])]
        ref_imp = g.accumulated_impulses.transpose(0, 2, 1).reshape(-1, g.accumulated_impulses.shape[1])[tb["source"]]
        got_imp = tb["impulses"].transpose(0, 2, 1).reshape(-1, tb["impulses"].shape[1])[:tb["count"]]
        if not np.array_equal(ref_imp.view(np.uint32), got_imp.view(np.uint32)):
            ok = False
            print("rank %d: impulses of batch %d type %d differ" % (rank, tb["batch_index"], tb["type_id"]), flush=True)
            break
    flag = torch.tensor([1 if ok else 0], device="cuda")
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    shared = int(((solver.masks & (solver.masks - 1)) != 0).sum())
    if rank == 0:
        print("sharded over %d GPUs: %d bodies (%d shared between ranks), %d constraints, %d frames of %d x %d: %s" % (
            world, args.bodies, shared, sim.constraint_count, args.frames, args.substeps, args.iterations, "BIT-EXACT vs the oracle on every rank" if flag.item() else "MISMATCH"), flush=True)
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
    dev_ms = torch.tensor([float(np.mean(ms)), t.solve_ms], device="cuda", dtype=torch.float64)
    dist.all_reduce(dev_ms, op=dist.ReduceOp.MAX)
    mine_count = torch.tensor([sum(tb["count"] for tb in solver.shard)], device="cuda", dtype=torch.float64)
    dist.all_reduce(mine_count, op=dist.ReduceOp.SUM)
    if rank == 0:
        ci = sim.constraint_count * args.substeps * args.iterations
        shared = int(((solver.masks & (solver.masks - 1)) != 0).sum())
        print("sharded over %d GPUs: %d bodies (%d shared), %d constraints (%d uploaded), %d x %d: wall %.3f ms/step, device %.3f ms/step (max over ranks), %.3f G constraint-iterations/s" % (
            world, args.bodies, shared, sim.constraint_count, int(mine_count.item()), args.substeps, args.iterations, dev_ms[0].item(), dev_ms[1].item(), ci / (dev_ms[1].item() * 1e-3) / 1e9), flush=True)
    code = 0
solver.close()
dist.barrier()
dist.destroy_process_group()
sys.exit(code)
