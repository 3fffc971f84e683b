"""Per-stage timeline of the 100 k-body pile (C2) on the GPU: torch.profiler with CUDA activities over solves in EXEC_STREAM mode, where the stages
still launch with programmatic dependent launch (bepucuda_profile_stages serialises them). Every constraint stage kernel is mapped onto the stage
program in launch order and the table gives, per (stage kind, device batch): bundles, the instantiation that ran, the mean kernel duration and the
mean start-to-start interval (this stage's start to the next stage kernel's start: what the stage adds to the dependent chain).

    python tests/tools/stage_timeline.py [--solves 10] [--json out.json] [--tree DIR]

--tree imports the package from another checkout (a built tree of an older commit), so that two versions can be compared in one run."""
import argparse
import collections
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
STAGES = {0: "warm_start_first", 1: "warm_start", 2: "solve", 3: "incremental"}
KERNEL = re.compile(r"constraint_stage_kernel(?:_sharded)?<(\d+), (\d+), (true|false)(?:, (true|false))?>")


def card():
    """Name, power limit and SM clock of the card, read without changing anything."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], stdout=subprocess.PIPE,
                             stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip().splitlines()
        name, power, sm, sm_max = [p.strip() for p in out[0].split(",")]
        return {"name": name, "power_limit": power, "sm_clock_after_run": sm, "sm_clock_max": sm_max}
    except Exception as e:  # noqa: BLE001
        return {"error": "nvidia-smi: %s" % e}


def kernel_events(trace_path):
    with open(trace_path) as f:
        trace = json.load(f)
    events = [e for e in trace.get("traceEvents", []) if e.get("cat") == "kernel" and e.get("ph") == "X"]
    events.sort(key=lambda e: e["ts"])
    return events


def timeline(events):
    """Maps the constraint stage kernels onto the stage program. Within one substep the program is WarmStart b0 .. bN-1, then the Solve stages
    b0 .. bN-1 once per velocity iteration, so the batch of a WarmStart is its place in the run of WarmStart launches and the batch of a Solve its
    place in the run of Solve launches modulo N."""
    rows = collections.OrderedDict()
    batches = 0
    run_stage, run_length = None, 0
    ours = [e for e in events if "bepu_" in e["name"]]
    for i, e in enumerate(ours):
        m = KERNEL.search(e["name"])
        if not m:
            run_stage, run_length = None, 0
            continue
        stage = int(m.group(1))
        kind = STAGES[stage]
        if stage != run_stage:
            run_stage, run_length = stage, 0
        if stage in (0, 1):
            batch = run_length
            batches = run_length + 1
        elif stage == 2:
            batch = run_length % max(batches, 1)
        else:
            batch = 0
        run_length += 1
        nxt = ours[i + 1]["ts"] if i + 1 < len(ours) else None
        variant = "minb=%s%s%s" % (m.group(2), " ext" if m.group(3) == "true" else "", " contacts" if m.group(4) == "true" else "")
        grid = e.get("args", {}).get("grid", [0])[0]
        r = rows.setdefault((kind, batch), {"kind": kind, "batch": batch, "bundles": grid * 2, "variants": set(), "dur": [], "s2s": []})
        r["variants"].add(variant)
        r["dur"].append(e["dur"])
        if nxt is not None:
            r["s2s"].append(nxt - e["ts"])
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bodies", type=int, default=100_000)
    ap.add_argument("--substeps", type=int, default=8)
    ap.add_argument("--iterations", type=int, default=2)
    ap.add_argument("--solves", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--strict", action="store_true")
    ap.add_argument("--tree", default=ROOT, help="repository tree whose package is imported (built in place)")
    ap.add_argument("--json", help="also write the table as JSON to this path")
    args = ap.parse_args()

    sys.path.insert(0, os.path.abspath(args.tree))
    import torch
    from torch.profiler import ProfilerActivity, profile

    import bepuphysics2_b200 as bp
    from bepuphysics2_b200 import scenes
    from bepuphysics2_b200.native import EXEC_STREAM

    if not torch.cuda.is_available():
        raise SystemExit("stage_timeline.py: no CUDA device")
    sim = bp.Simulation(bundle_width=8, fallback_batch_threshold=64, substeps=args.substeps, velocity_iterations=args.iterations)
    scenes.build(scenes.shape_pile(args.bodies, seed=5), sim)
    ts = bp.CudaTimestepper(sim, device=0, strict_fp=args.strict, execution_mode=EXEC_STREAM)
    ts.register_host_buffers()
    ts.describe()
    ts.synchronize()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")  # > the 50 MB L2, as in bench.py

    def solve():
        flush.fill_(1)
        torch.cuda.synchronize()
        ts.solve_device_only(1.0 / 60.0)
        ts.synchronize()

    for _ in range(args.warmup):
        solve()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.solves):
            solve()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(path)
        events = kernel_events(path)
    rows = timeline(events)
    info = card()
    print("stage timeline: shape_pile %d bodies, %d x %d, %d solves, %s build, tree %s" % (args.bodies, args.substeps, args.iterations, args.solves,
                                                                                           "strict" if args.strict else "fast", os.path.abspath(args.tree)))
    print("card: %s" % json.dumps(info))
    print("%-17s %5s %7s %-22s %9s %9s" % ("stage", "batch", "bundles", "instantiation", "dur us", "s2s us"))
    out = []
    total = collections.defaultdict(float)
    for r in rows.values():
        dur = sum(r["dur"]) / len(r["dur"])
        s2s = sum(r["s2s"]) / len(r["s2s"]) if r["s2s"] else float("nan")
        launches_per_solve = len(r["dur"]) / args.solves
        if r["s2s"]:
            total[r["kind"]] += s2s * launches_per_solve
        variants = ",".join(sorted(r["variants"]))
        print("%-17s %5d %7d %-22s %9.2f %9.2f" % (r["kind"], r["batch"], r["bundles"], variants, dur, s2s))
        out.append({"kind": r["kind"], "batch": r["batch"], "bundles": r["bundles"], "instantiation": variants, "mean_us": dur, "start_to_start_us": s2s,
                    "launches_per_solve": launches_per_solve})
    for kind, us in total.items():
        print("per solve, %-17s start-to-start sum %8.1f us" % (kind, us))
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": info, "bodies": args.bodies, "substeps": args.substeps, "iterations": args.iterations, "solves": args.solves, "rows": out,
                       "start_to_start_us_per_solve": dict(total)}, f, indent=1)


if __name__ == "__main__":
    main()
