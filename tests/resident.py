"""Frames of the resident device path (accumulated impulses kept on the device and redistributed there from the old to the new contact feature
ids) next to the oracle's host path on a twin simulation, and the narrow-phase-like updates, body changes and per-frame descriptions that drive
them."""
import ctypes as C

import numpy as np

import bepuphysics2_b200 as bp
from bepuphysics2_b200 import scenes
from bepuphysics2_b200.native import EXEC_GRAPH, contact_count
from oracle import binding as ob
from tests import planner, util

DT = 1.0 / 60.0
REFERENCE_MASK = (1 << 30) - 1  # the body index bits of an encoded body reference


def live_handles(sim):
    _, batches = sim.constraint_references()
    return np.flatnonzero(batches >= 0)


def type_batch_at(sim, batch, type_id):
    return next(tb for tb in sim.type_batches() if tb.batch_index == batch and tb.type_id == type_id)


def lane_record(sim, handle):
    """The 64-word record (bepucuda_read_constraints layout) of a constraint from the host's buffers."""
    b, t, i = sim.constraint_location(handle)
    tb = type_batch_at(sim, b, t)
    W = sim.bundle_width
    r = np.zeros(64, dtype=np.int32)
    r[0], r[1] = t, 1
    r[2:2 + tb.bodies] = tb.body_references[i // W, :, i % W]
    r[2 + tb.bodies:6] = -1
    r[6:6 + tb.impulse_rows] = tb.accumulated_impulses[i // W, :, i % W].view(np.int32)
    r[18:18 + tb.prestep_rows] = tb.prestep[i // W, :, i % W].view(np.int32)
    return r


def projectile_prestep(rng, m):
    return scenes.convex_prestep(rng.uniform(-0.2, 0.2, size=(m, 1, 3)), np.full((m, 1), 0.01), np.tile([0, 1, 0], (m, 1)), offset_b=rng.uniform(-0.2, 0.2, size=(m, 3)))


def body_frame(sim, rng, spawn, removes, kinematic_mover=None):
    """One frame of a game on the host: `removes` random bodies go (Bodies.Remove: their constraints first), then `spawn` projectiles are fired,
    copies of random bodies 3 m higher with a velocity, each with a new contact to a random body. Returns the number of constraint adds."""
    if removes:
        pool = sim.body_handles
        if kinematic_mover is not None:
            pool = pool[pool != kinematic_mover]
        sim.remove_bodies(rng.choice(pool, size=removes, replace=False))
    if not spawn:
        return 0
    src = rng.integers(0, sim.body_count, size=spawn)
    new = sim.bodies[src].copy()
    new[:, 5] += 3
    new[:, 8:11] = rng.normal(size=(spawn, 3))
    new[:, 16:23] = np.where(new[:, 16:23].any(axis=1, keepdims=True), new[:, 16:23], [1, 0, 1, 0, 0, 1, 1])  # projectiles are dynamic
    sim.add_bodies(new)
    added = sim.body_handles[-spawn:]
    partners = sim.body_handles[rng.integers(0, sim.body_count - spawn, size=spawn)]
    sim.add_constraints(4, np.stack([added, partners], axis=1), projectile_prestep(rng, spawn))
    return spawn


def remove_a_ragdoll(sim, frame, extra):
    """Removes every body joined to a random body by joints (one whole ragdoll)."""
    refs, batches = sim.constraint_references()
    joint = np.array([contact_count(sim.constraint_location(int(c))[1]) == 0 if batches[c] >= 0 else False for c in range(len(batches))])
    rng = np.random.default_rng(frame)
    seed_index = int(rng.integers(0, sim.body_count))
    group, todo = {seed_index}, [seed_index]
    while todo:
        b = todo.pop()
        for c in np.flatnonzero(joint & ((refs & REFERENCE_MASK) == b).any(axis=1) & (refs >= 0).any(axis=1)):
            for r in refs[c]:
                if r >= 0 and (r & REFERENCE_MASK) not in group:
                    group.add(int(r & REFERENCE_MASK))
                    todo.append(int(r & REFERENCE_MASK))
    sim.remove_bodies([int(sim.body_handles[i]) for i in sorted(group)])


def set_description(ts, sim):
    """What a C# host sends at the start of every frame (integration/csharp/CudaTimestepper.cs): the simulation's solve description and
    integrator, through the C ABI."""
    its = (C.c_int32 * len(sim.velocity_iterations))(*sim.velocity_iterations)
    ts._check(ts._cuda.bepucuda_set_solve_description(ts._ctx, len(sim.velocity_iterations), its, sim.fallback_batch_threshold))
    ts._check(ts._cuda.bepucuda_set_integrator(ts._ctx, C.byref(sim.integrator)))


def set_terms(ts, terms):
    """The velocity terms of a frame's solve keywords (accelerations, center, strength) on the context: set, or cleared where they are absent."""
    ts.set_body_accelerations(terms.get("accelerations"))
    ts.set_point_gravity(terms.get("center"), terms.get("strength", 0.0))


def initial_features(sim, rng):
    return {(tb.batch_index, tb.type_batch_index): rng.integers(0, 1 << 20, size=(tb.constraint_count, contact_count(tb.type_id)), dtype=np.int32)
            for tb in sim.type_batches() if contact_count(tb.type_id)}


def narrow_phase_like_update(sim, features, rng):
    """What a frame of collision detection does to an unchanged topology: new depths, and some contacts replaced by new features. Touches the
    contact type batches named in `features` only."""
    new = {}
    for tb in sim.type_batches():
        key = (tb.batch_index, tb.type_batch_index)
        if key not in features:
            continue
        ids = features[key].copy()
        n = ids.shape[1]
        change = rng.random(ids.shape) < 0.2
        ids[change] = rng.integers(1 << 20, 1 << 21, size=int(change.sum()), dtype=np.int32)
        swap = rng.random(ids.shape[0]) < 0.3  # the narrow phase often reports the same features in another order
        if n > 1:
            ids[swap] = ids[swap][:, ::-1]
        new[key] = ids
        for r in planner.depth_rows(tb.type_id):  # the narrow phase writes fresh depths every frame (whatever the solver's incremental updates left in the row)
            tb.prestep[:, r, :] = rng.uniform(-0.02, 0.05, size=tb.prestep[:, r, :].shape).astype(np.float32)
    return new


def _type_batch(sim, key):
    return next(tb for tb in sim.type_batches() if (tb.batch_index, tb.type_batch_index) == key)


def update_type_batch(ts, tb):
    """bepucuda_update_type_batch of one type batch from the simulation's own buffers (what bepuhost_cuda_refresh does for every type batch)."""
    ts._check(ts._cuda.bepucuda_update_type_batch(ts._ctx, tb.batch_index, tb.type_batch_index, tb.prestep.ctypes.data, tb.accumulated_impulses.ctypes.data))


KICK = 0.01  # m/s: far above the last bit of any velocity, small enough not to stress the joints


def push_bodies(sim, frame):
    """What a host does to the bodies between frames (a character controller, a user drag): here a fifth of the bodies gets a small kick of
    linear velocity. Applied to both twins, so a motion upload that did nothing would show."""
    sim.bodies[frame % 5::5, 9] += np.float32(KICK)


def _take_state(host, source, features, feat_h):
    """The host twin takes the state of `source` (a simulation whose device run was downloaded): bodies, prestep, accumulated impulses, and the
    feature ids those impulses belong to."""
    host.bodies[:] = source.bodies
    for th, src in zip(host.type_batches(), source.type_batches()):
        th.prestep[:] = src.prestep
        th.accumulated_impulses[:] = src.accumulated_impulses
    feat_h.clear()
    feat_h.update({key: ids.copy() for key, ids in features.items()})


def resident_frames(scene, frames=4, bundle_width=8, fallback_batch_threshold=64, mode=EXEC_GRAPH, strict=True, register=True, pool=False, named=None,
                     joint_reset=False, seed=77, take_state=None, push=True):
    """Frames of f2 through the device path next to the oracle's host path on a twin simulation. Host: narrow-phase-like update, RedistributeImpulses
    (ob.update_contact_impulses), solve. Device: upload_body_motion + update_contacts (or update_contacts_from_pool, the sequence bench.py times),
    solve_device_only, download_body_motion; the motion halves must agree bit for bit after every frame (strict build). One download_bodies,
    download_impulses and download_prestep at the end. named(frame, keys): the contact type batches a frame updates (all by default); the others
    keep what the last solve left on both sides. joint_reset: every frame also zeroes the accumulated impulses of one joint type batch on both
    twins (a re-created joint) and sends it through bepucuda_update_type_batch. push: before every update both twins' bodies get the same velocity
    kick (push_bodies). take_state = (frame, source simulation, its feature ids): after that frame the host twin takes that state (_take_state), so
    that the frame after it can be held to one-frame tolerances in the fast build. Returns (host, dev, device timings, replaced contact count,
    the device's feature ids)."""
    kw = dict(bundle_width=bundle_width, fallback_batch_threshold=fallback_batch_threshold, substeps=3, velocity_iterations=2)
    host, dev = util.make_sim(scene, **kw), util.make_sim(scene, **kw)
    rng_h, rng_d = np.random.default_rng(seed), np.random.default_rng(seed)
    ts = bp.CudaTimestepper(dev, strict_fp=strict, execution_mode=mode)
    try:
        if register:
            ts.register_host_buffers()
        ts.describe()
        feat_h, feat_d = initial_features(host, rng_h), initial_features(dev, rng_d)
        if pool:
            pool_d, views = ts.contact_feature_pool()
            ts.register_array(pool_d)
            assert sorted(views) == sorted(feat_d)
            for key, ids in feat_d.items():
                views[key][:] = ids
            ts.set_contact_feature_pool(pool_d)
        else:
            ts.set_contact_features(feat_d)
        joints = [(tb.batch_index, tb.type_batch_index) for tb in host.type_batches() if not contact_count(tb.type_id)]
        assert joints or not joint_reset
        replaced = 0
        for frame in range(frames):
            if frame > 0:
                keys = sorted(feat_h) if named is None else named(frame, sorted(feat_h))
                new_h = narrow_phase_like_update(host, {k: feat_h[k] for k in keys}, rng_h)
                new_d = narrow_phase_like_update(dev, {k: feat_d[k] for k in keys}, rng_d)
                if pool:
                    for key, ids in new_d.items():
                        views[key][:] = ids
                    new_h = {key: views[key] for key in new_h}  # the host redistributes through the pool's views
                for tb in host.type_batches():
                    key = (tb.batch_index, tb.type_batch_index)
                    if key in new_h:
                        ob.update_contact_impulses(tb, feat_h[key], new_h[key])
                        replaced += int((new_h[key] >= (1 << 20)).sum())
                feat_h.update({key: ids.copy() for key, ids in new_h.items()})
                if push:
                    push_bodies(host, frame)
                    push_bodies(dev, frame)
                if pool:
                    ts.update_contacts_from_pool(pool_d)
                else:
                    ts.upload_body_motion()
                    ts.update_contacts(new_d)
                feat_d.update(new_d)
                if joint_reset:
                    key = joints[frame % len(joints)]
                    _type_batch(host, key).accumulated_impulses[:] = 0.0
                    tb = _type_batch(dev, key)
                    tb.accumulated_impulses[:] = 0.0
                    update_type_batch(ts, tb)
            ob.solve(host, DT)
            ts.solve_device_only(DT)
            ts.download_body_motion()
            t = ts.timings()
            assert t.d2h_bytes == dev.body_count * 64
            assert np.array_equal(host.bodies[:, util.MOTION].view(np.uint32), dev.bodies[:, util.MOTION].view(np.uint32)) or not strict, "frame %d" % frame
            if take_state is not None and frame == take_state[0]:
                _take_state(host, take_state[1], take_state[2], feat_h)
        ts.download_bodies()  # the motion-only download leaves the host's world-inertia half untouched: fetch it once for the full comparison
        ts.download_impulses()
        ts.download_prestep()
        timings = ts.timings()
    finally:
        ts.close()
    return host, dev, timings, replaced, feat_d
