"""Diagnostic for the resident-impulses path: isolates body round trip, redistribution and the following solve."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import bepuphysics2_b200 as bp
from bepuphysics2_b200 import scenes
from oracle import binding as ob
from tests import util
from tests.resident import initial_features, narrow_phase_like_update

DT = 1 / 60.0
scene = scenes.shape_pile(3000, seed=31)
kw = dict(substeps=3, velocity_iterations=2)
host, dev = util.make_sim(scene, **kw), util.make_sim(scene, **kw)
rng_h, rng_d = np.random.default_rng(77), np.random.default_rng(77)
feat_h, feat_d = initial_features(host, rng_h), initial_features(dev, rng_d)
ts = bp.CudaTimestepper(dev, strict_fp=True)
ts.register_host_buffers()
ts.describe()
ts.set_contact_features(feat_d)
cols = np.r_[0:7, 8:11, 12:15]
def bodies_equal(tag):
    same = np.array_equal(host.bodies[:, cols].view(np.uint32), dev.bodies[:, cols].view(np.uint32))
    print(tag, "bodies equal:", same, flush=True)
def rows_equal(tag):
    bad_i = bad_p = 0
    for a, b in zip(host.type_batches(), dev.type_batches()):
        valid = a.body_references[:, 0, :] >= 0
        vi = np.broadcast_to(valid[:, None, :], a.accumulated_impulses.shape)
        bad_i += int((np.where(vi, a.accumulated_impulses, 0).view(np.uint32) != np.where(vi, b.accumulated_impulses, 0).view(np.uint32)).sum())
        vp = np.broadcast_to(valid[:, None, :], a.prestep.shape)
        bad_p += int((np.where(vp, a.prestep, 0).view(np.uint32) != np.where(vp, b.prestep, 0).view(np.uint32)).sum())
    print(tag, "impulse words differing:", bad_i, "prestep words differing:", bad_p, flush=True)
for frame in range(4):
    if frame > 0:
        new_h = narrow_phase_like_update(host, feat_h, rng_h)
        for tb in host.type_batches():
            key = (tb.batch_index, tb.type_batch_index)
            ob.update_contact_impulses(tb, feat_h[key], new_h[key])
        feat_h = new_h
        new_d = narrow_phase_like_update(dev, feat_d, rng_d)
        print("new ids equal:", all(np.array_equal(new_h[k], new_d[k]) for k in new_h))
        ts.upload_body_motion()
        ts.update_contacts(new_d)
        feat_d = new_d
    ob.solve(host, DT)
    ts.solve_device_only(DT)
    ts.download_body_motion()
    if "--timings" in sys.argv:
        t = ts.timings()
        print("d2h", t.d2h_bytes, "h2d", t.h2d_bytes, "solve_ms %.3f" % t.solve_ms)
    bodies_equal("frame %d" % frame)
    if "--downloads" in sys.argv:
        ts.download_impulses(); ts.download_prestep()
        rows_equal("after frame %d" % frame)
ts.download_impulses(); ts.download_prestep()
rows_equal("end")
ts.close()
