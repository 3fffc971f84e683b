"""Diagnostic: where the time of the resident-impulses end-to-end frame goes (each call followed by a synchronize)."""
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import bepuphysics2_b200 as bp
from bepuphysics2_b200 import scenes
from bepuphysics2_b200.native import contact_count

sim = bp.Simulation(bundle_width=8, substeps=8, velocity_iterations=2)
scenes.build(scenes.shape_pile(100_000, seed=5), sim)
ts = bp.CudaTimestepper(sim)
ts.register_host_buffers()
tbs = [tb for tb in sim.type_batches() if contact_count(tb.type_id)]
pool = np.random.default_rng(1).integers(0, 1 << 20, size=sum(tb.constraint_count * contact_count(tb.type_id) for tb in tbs), dtype=np.int32)
feats, at = {}, 0
for tb in tbs:
    n = tb.constraint_count * contact_count(tb.type_id)
    feats[(tb.batch_index, tb.type_batch_index)] = pool[at:at + n].reshape(tb.constraint_count, -1)
    at += n
ts.register_array(pool)
ts.describe()
ts.set_contact_features(feats)
acc = {}
def timed(name, fn):
    t = time.perf_counter(); fn(); ts.synchronize(); acc[name] = acc.get(name, 0.0) + time.perf_counter() - t
for i in range(13):
    if i == 3:
        acc.clear()
    timed("upload_body_motion", ts.upload_body_motion)
    timed("update_contacts", lambda: ts.update_contacts(feats))
    timed("solve (incl. refresh: flush, transpose, redistribute)", lambda: ts.solve_device_only(1 / 60))
    timed("download_body_motion", ts.download_body_motion)
    timed("refresh (regular path)", ts.refresh)
    timed("solve+download (regular path)", lambda: ts.solve(1 / 60, download=True))
for k, v in acc.items():
    print("%-60s %.3f ms" % (k, v / 10 * 1e3))
