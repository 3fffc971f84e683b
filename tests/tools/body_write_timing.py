"""Measurement: the resident frame of C2 (the 100 k-body shape pile) with the host's body changes sent as every body's motion
(bepucuda_upload_body_motion) against bepucuda_write_bodies of 1, 1 000, 20 000 (push_bodies' fifth) and 100 000 listed indices. Fast build, graph
mode, registered buffers. The routes alternate frame by frame; each frame is body step, update_contacts, solve, download_body_motion.
Per route: medians over the timed frames of the body step (CUDA events around it; host wall clock of the call) and of the whole frame (events;
wall clock, which ends in the download's synchronize), and the bytes up. Prints one JSON line per route with the card it ran on, and writes the
lines to --out when given."""
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
from bepuphysics2_b200.native import contact_count  # noqa: E402

COUNTS = [1, 1_000, 20_000, 100_000]
KICK = np.float32(1e-3)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, limit = [x.strip() for x in q.stdout.splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": limit}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bodies", type=int, default=100_000)
    ap.add_argument("--frames", type=int, default=40, help="timed frames per route")
    ap.add_argument("--warmup", type=int, default=5, help="untimed frames per route")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    sim = bp.Simulation(bundle_width=8, substeps=8, velocity_iterations=2)
    scenes.build(scenes.shape_pile(args.bodies, seed=5), sim)
    n = sim.body_count
    ts = bp.CudaTimestepper(sim, strict_fp=False)
    ts.register_host_buffers()
    tbs = [tb for tb in sim.type_batches() if contact_count(tb.type_id)]
    rng = np.random.default_rng(1)
    pool = rng.integers(0, 1 << 20, size=sum(tb.constraint_count * contact_count(tb.type_id) for tb in tbs), dtype=np.int32)
    feats, at = {}, 0
    for tb in tbs:
        k = tb.constraint_count * contact_count(tb.type_id)
        feats[(tb.batch_index, tb.type_batch_index)] = pool[at:at + k].reshape(tb.constraint_count, -1)
        at += k
    ts.register_array(pool)
    ts.describe()
    ts.set_contact_features(feats)

    routes = {"upload_body_motion": None}
    for c in COUNTS:
        if c <= n:
            routes["write_bodies_%d" % c] = np.sort(rng.choice(n, size=c, replace=False)).astype(np.int32)
    fifth = np.arange(0, n, 5)
    samples = {r: {"body_event_ms": [], "body_wall_ms": [], "frame_event_ms": [], "frame_wall_ms": [], "h2d_bytes": []} for r in routes}

    def frame(route, timed):
        idx = routes[route]
        sim.bodies[fifth if idx is None else idx, 9] += KICK  # the host's change
        t0 = time.perf_counter()
        ts.event_record(0)
        if idx is None:
            ts.upload_body_motion()
        else:
            ts.write_bodies(idx)
        ts.event_record(1)
        t1 = time.perf_counter()
        ts.update_contacts(feats)
        ts.solve_device_only(1 / 60)
        ts.event_record(2)
        ts.download_body_motion()  # synchronizes
        t2 = time.perf_counter()
        if timed:
            s = samples[route]
            s["body_event_ms"].append(ts.event_elapsed_ms(0, 1))
            s["frame_event_ms"].append(ts.event_elapsed_ms(0, 2))
            s["body_wall_ms"].append((t1 - t0) * 1e3)
            s["frame_wall_ms"].append((t2 - t0) * 1e3)
            s["h2d_bytes"].append(ts.timings().h2d_bytes)

    for i in range(args.warmup + args.frames):
        for route in routes:  # alternated frame by frame
            frame(route, i >= args.warmup)
    ts.close()

    info = card()
    update_bytes = None
    results = []
    for route, s in samples.items():
        idx = routes[route]
        body_bytes = n * 64 if idx is None else len(idx) * 68
        h2d = int(np.median(s["h2d_bytes"]))
        update_bytes = h2d - body_bytes
        r = {"route": route, "listed": n if idx is None else len(idx), "bodies": n, "frames": len(s["frame_wall_ms"]), "body_bytes_up": body_bytes,
             "h2d_bytes": h2d}
        r.update({k: round(float(np.median(v)), 4) for k, v in s.items() if k != "h2d_bytes"})
        r.update(info)
        results.append(r)
    full = results[0]
    for key in ("body_event_ms", "frame_event_ms", "frame_wall_ms"):
        # the listed count above which the full upload is cheaper, by linear interpolation between the measured counts
        pts = [(r["listed"], r[key]) for r in results[1:]]
        cross = None
        for (c0, t0), (c1, t1) in zip(pts, pts[1:]):
            if t0 <= full[key] < t1:
                cross = int(c0 + (full[key] - t0) * (c1 - c0) / (t1 - t0))
        full["crossover_" + key] = cross if cross is not None else ("above %d" % pts[-1][0] if pts[-1][1] <= full[key] else "below %d" % pts[0][0])
    full["update_contacts_h2d_bytes"] = update_bytes
    lines = [json.dumps(r) for r in results]
    print("\n".join(lines))
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
