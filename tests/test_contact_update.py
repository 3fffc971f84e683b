"""Device-side contact constraint update, first slice (SURVEY.md §8 f2): accumulated impulses stay resident on the device and are redistributed there
from the old to the new contact feature ids (NarrowPhase.RedistributeImpulses, CollisionDetection/NarrowPhaseConstraintUpdate.cs:L81-135), and
only the motion half of BodyDynamics crosses the bus. CPU part: the oracle's restatement of RedistributeImpulses against hand-worked cases.
GPU part: several frames of (narrow-phase-like update -> solve) through the resident path against the host path of the oracle, bit for bit."""
import ctypes as C

import numpy as np
import pytest

import bepuphysics2_b200 as bp
from bepuphysics2_b200 import scenes
from bepuphysics2_b200.native import ERR_BAD_STATE, ERR_INVALID_ARGUMENT, EXEC_STREAM, contact_count
from oracle import binding as ob
from tests import planner, resident, util

DT = 1.0 / 60.0


def _redistribute(old_ids, old_imp, new_ids):
    lib = ob.load()
    ip, fp = C.POINTER(C.c_int32), C.POINTER(C.c_float)
    lib.oracle_redistribute_impulses.argtypes = [C.c_int32, ip, fp, C.c_int32, ip, fp]
    oi = np.array(old_ids, dtype=np.int32)
    om = np.array(old_imp, dtype=np.float32)
    ni = np.array(new_ids, dtype=np.int32)
    out = np.zeros(len(new_ids), dtype=np.float32)
    lib.oracle_redistribute_impulses(len(old_ids), oi.ctypes.data_as(ip), om.ctypes.data_as(fp), len(new_ids), ni.ctypes.data_as(ip), out.ctypes.data_as(fp))
    return out


def test_redistribute_impulses_known_answers(libs):
    """NarrowPhaseConstraintUpdate.cs:L81-135 on cases worked by hand."""
    # all matched, permuted: every new contact takes the impulse of the old contact with its id
    assert np.array_equal(_redistribute([10, 11, 12, 13], [1, 2, 3, 4], [13, 10, 12, 11]), np.array([4, 1, 3, 2], dtype=np.float32))
    # one new contact unmatched: it receives what the vanished old contact had
    assert np.array_equal(_redistribute([10, 11, 12, 13], [1, 2, 3, 4], [10, 99, 12, 13]), np.array([1, 2, 3, 4], dtype=np.float32))
    # two unmatched share the remainder (2 + 4) / 2 equally
    assert np.array_equal(_redistribute([10, 11, 12, 13], [1, 2, 3, 4], [10, 98, 12, 99]), np.array([1, 3, 3, 3], dtype=np.float32))
    # nothing matches: the total is spread evenly
    assert np.array_equal(_redistribute([1, 2], [3, 5], [7, 8]), np.array([4, 4], dtype=np.float32))
    # fewer new contacts than old, one match: matched keeps its own, nothing unmatched -> the rest is dropped
    assert np.array_equal(_redistribute([1, 2, 3], [3, 5, 7], [2]), np.array([5], dtype=np.float32))
    # duplicate ids: the inner loop always stops at the FIRST old contact with the id (only its impulse is zeroed, L96-101), so the second new contact matches it again and gets 0
    assert np.array_equal(_redistribute([5, 5], [2, 6], [5, 5]), np.array([2, 0], dtype=np.float32))


def _pile(nonconvex=0.0):
    return scenes.shape_pile(3000, seed=31, nonconvex_fraction=nonconvex)


def _mixed():
    return scenes.merge(scenes.shape_pile(1500, seed=41, nonconvex_fraction=0.3), scenes.joint_zoo(600, per_type=20, seed=42), scenes.ragdolls(20, seed=43))


# scene, keyword arguments of resident.resident_frames
RESIDENT_CASES = {
    "pile": (lambda: _pile(0.0), {}),
    "pile_nonconvex": (lambda: _pile(0.5), {}),
    "pile_width4": (lambda: _pile(0.3), dict(bundle_width=4)),
    "pile_width16": (lambda: _pile(0.3), dict(bundle_width=16)),
    "pile_stream": (lambda: _pile(0.3), dict(mode=EXEC_STREAM)),
    "pile_unregistered": (lambda: _pile(0.3), dict(register=False)),
    "pile_feature_pool": (lambda: _pile(0.3), dict(pool=True)),
    "fallback_levels": (lambda: scenes.fallback_stress(2000, hubs=4, seed=5), dict(fallback_batch_threshold=8)),
    "ragdolls_graph": (lambda: scenes.ragdolls(60, seed=5), {}),
    "ragdolls_stream": (lambda: scenes.ragdolls(60, seed=5), dict(mode=EXEC_STREAM)),
    "mixed_graph": (_mixed, {}),
    "mixed_stream": (_mixed, dict(mode=EXEC_STREAM)),
    "mixed_unregistered_feature_pool": (_mixed, dict(register=False, pool=True)),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(RESIDENT_CASES))
def test_resident_impulses_with_device_side_redistribution_bit_exact(libs, case):
    """The f2 frame against the host path, bit for bit, for several frames: contact piles at host bundle widths 4 / 8 / 16, the levelised fallback
    batches (slot map), joints solved next to the contacts (their impulses stay resident and warm-start the next frame as on the host), both
    execution modes, both upload routes (mapped host buffers and cudaMemcpy2DAsync through the staging image) and the feature-pool walker."""
    make, kw = RESIDENT_CASES[case]
    host, dev, timings, replaced, _ = resident.resident_frames(make(), **kw)
    util.compare(util.snapshot(host), util.snapshot(dev), exact=True)
    contacts = sum(tb.constraint_count * contact_count(tb.type_id) for tb in host.type_batches())
    assert replaced > 0.2 * contacts  # the test really replaced contacts
    if case == "fallback_levels":
        assert timings.fallback_level_count > 0
    if case.startswith(("ragdolls", "mixed")):
        joints = [tb for tb in host.type_batches() if not contact_count(tb.type_id)]
        assert joints and any(np.abs(tb.accumulated_impulses).max() > 0 for tb in joints)


def _every_other(frame, keys):
    return [k for i, k in enumerate(keys) if (i + frame) % 2 == 0]


@pytest.mark.gpu
@pytest.mark.parametrize("joint_reset", [False, True], ids=["contacts_only", "with_joint_update"])
def test_partial_frames_keep_the_device_rows_of_type_batches_not_sent(libs, joint_reset):
    """Frames that name only every other contact type batch (alternating): the others keep on the device the depths and impulses the last solve
    left, as the host does. With joint_reset one joint type batch per frame also goes up through bepucuda_update_type_batch with zeroed impulses,
    and only that one: the other joints keep warm-starting from their resident impulses."""
    host, dev, _, _, _ = resident.resident_frames(_mixed(), frames=5, named=_every_other, joint_reset=joint_reset)
    util.compare(util.snapshot(host), util.snapshot(dev), exact=True)


def _all_contact_types_scene(seed=3):
    """One type batch per contact type id (0-10, 15-17), alternately of 1 and 33 constraints, every constraint on bodies of its own (so each type
    batch sits whole in batch 0). Bodies and prestep rows come from the seeded pile."""
    pile = scenes.shape_pile(3000, seed=seed, nonconvex_fraction=0.5)
    by_type = {int(t): (h, p) for t, h, p in pile["constraints"]}
    types = sorted(planner.CONTACT_TYPES)
    assert all(t in by_type for t in types)
    constraints, next_body = [], 0
    for i, t in enumerate(types):
        h, p = by_type[t]
        count = 1 if i % 2 == 0 else 33
        nb = h.shape[1]
        handles = np.arange(next_body, next_body + count * nb, dtype=np.int32).reshape(count, nb)
        next_body += count * nb
        constraints.append((t, handles, np.ascontiguousarray(np.resize(p, (count, p.shape[1])), dtype=np.float32)))
    bodies = np.ascontiguousarray(np.resize(pile["bodies"], (next_body, pile["bodies"].shape[1])), dtype=np.float32)
    return {"bodies": bodies, "constraints": constraints, "description": "every contact type, type batches of 1 and 33"}


def _crafted_ids(rng, count, n):
    """(old, new) feature ids of `count` constraints of n contacts, cycling through: all matched and permuted; none matched; duplicates in old,
    in new and in both; INT32_MIN / INT32_MAX / negative ids; partially matched."""
    lo, hi = np.iinfo(np.int32).min, np.iinfo(np.int32).max
    old = np.zeros((count, n), dtype=np.int32)
    new = np.zeros((count, n), dtype=np.int32)
    for c in range(count):
        o = rng.choice(1000, size=n, replace=False).astype(np.int32) - 500
        kind = (c + n) % 7
        if kind == 0:
            nw = rng.permutation(o)
        elif kind == 1:
            nw = o + 1000
        elif kind == 2:
            o[:] = o[0]
            nw = rng.permutation(np.r_[o[:1], np.arange(n - 1) + 2000]).astype(np.int32)
        elif kind == 3:
            nw = np.full(n, o[-1], dtype=np.int32)
        elif kind == 4:
            o[:] = o[0]
            nw = np.full(n, o[0], dtype=np.int32)
        elif kind == 5:
            o = np.array([lo, hi, -1, 0][:n], dtype=np.int32)
            nw = np.array([hi, lo, -2, 0][:n], dtype=np.int32)
        else:
            nw = o.copy()
            nw[::2] = lo + c
        old[c], new[c] = o, nw
    return old, new


@pytest.mark.gpu
def test_redistribution_edges_through_the_kernel(libs):
    """redistribute_impulses_kernel on every contact type id, type batches of 1 and 33 constraints, crafted id pairs and impulses of 0, subnormals,
    ordinary values and values whose sum overflows to inf. Solved with the schedule [0] (one substep, no velocity iterations) so that WarmStart
    leaves the accumulated impulses as the redistribution wrote them: download_impulses must equal ob.update_contact_impulses bit for bit, the
    untouched friction and twist rows included."""
    scene = _all_contact_types_scene()
    host, dev = util.make_sim(scene, velocity_iterations=[0]), util.make_sim(scene, velocity_iterations=[0])
    rng = np.random.default_rng(12)
    fmax = np.finfo(np.float32).max
    values = np.array([0.0, 1e-45, 2e-40, 0.125, 0.75, 3.0, fmax * 0.5, fmax * 0.75, fmax], dtype=np.float32)
    old_ids, new_ids = {}, {}
    counts = set()
    for th, td in zip(host.type_batches(), dev.type_batches()):
        key, n = (th.batch_index, th.type_batch_index), contact_count(th.type_id)
        assert n and th.batch_index == 0
        counts.add(th.constraint_count)
        acc = rng.uniform(-1, 1, size=th.accumulated_impulses.shape).astype(np.float32)  # friction / twist rows: ordinary values, both signs
        for r in planner.penetration_rows(th.type_id):
            acc[:, r, :] = values[rng.integers(0, values.size, size=acc[:, r, :].shape)]
        th.accumulated_impulses[:] = acc
        td.accumulated_impulses[:] = acc
        old_ids[key], new_ids[key] = _crafted_ids(rng, th.constraint_count, n)
    assert {tb.type_id for tb in host.type_batches()} == planner.CONTACT_TYPES and counts == {1, 33}
    ts = bp.CudaTimestepper(dev, strict_fp=True)
    try:
        ts.describe()
        ts.set_contact_features(old_ids)
        ts.upload_body_motion()
        ts.update_contacts(new_ids)
        ts.solve_device_only(DT)
        ts.download_impulses()
    finally:
        ts.close()
    for tb in host.type_batches():
        key = (tb.batch_index, tb.type_batch_index)
        ob.update_contact_impulses(tb, old_ids[key], new_ids[key])
    util.compare(util.snapshot(host), util.snapshot(dev) | {"bodies": host.bodies}, exact=True)
    pen = np.concatenate([tb.accumulated_impulses[:, planner.penetration_rows(tb.type_id), :].ravel() for tb in host.type_batches()])
    assert np.isinf(pen).any() and (pen == 0).any() and ((pen > 0) & (pen < np.finfo(np.float32).tiny)).any()


@pytest.mark.gpu
def test_topology_change_after_resident_frames(libs):
    """Resident frames, then download_impulses (the resident, redistributed impulses back into the host's buffers), new bodies and constraints
    on both twins, a new describe, new feature ids and more resident frames: still the host path bit for bit."""
    scene = _mixed()
    kw = dict(substeps=3, velocity_iterations=2)
    host, dev = util.make_sim(scene, **kw), util.make_sim(scene, **kw)
    rng_h, rng_d = np.random.default_rng(5), np.random.default_rng(5)
    extra = scenes.merge(scenes.shape_pile(300, seed=51), scenes.ragdolls(2, seed=52))
    ts = bp.CudaTimestepper(dev, strict_fp=True)  # host buffers unregistered: adding bodies and constraints may move them
    try:
        for epoch in range(2):
            if epoch:
                ts.download_bodies()
                ts.download_impulses()
                ts.download_prestep()  # the depths the incremental updates moved (a narrow phase would rewrite them)
                for sim in (host, dev):
                    base = sim.body_count
                    sim.add_bodies(extra["bodies"])
                    for type_id, handles, prestep in extra["constraints"]:
                        sim.add_constraints(type_id, handles + base, prestep)
            ts.describe()
            feat_h, feat_d = resident.initial_features(host, rng_h), resident.initial_features(dev, rng_d)
            ts.set_contact_features(feat_d)
            for frame in range(3):
                if frame > 0:
                    new_h = resident.narrow_phase_like_update(host, feat_h, rng_h)
                    for tb in host.type_batches():
                        key = (tb.batch_index, tb.type_batch_index)
                        if key in new_h:
                            ob.update_contact_impulses(tb, feat_h[key], new_h[key])
                    feat_h = new_h
                    feat_d = resident.narrow_phase_like_update(dev, feat_d, rng_d)
                    ts.upload_body_motion()
                    ts.update_contacts(feat_d)
                ob.solve(host, DT)
                ts.solve_device_only(DT)
                ts.download_body_motion()
        ts.download_bodies()
        ts.download_impulses()
        ts.download_prestep()
    finally:
        ts.close()
    util.compare(util.snapshot(host), util.snapshot(dev), exact=True)


def _resident_bytes():
    with open("/proc/self/status") as f:
        return next(int(line.split()[1]) << 10 for line in f if line.startswith("VmRSS:"))


@pytest.mark.gpu
def test_feature_ids_sent_again_every_frame_hold_no_host_memory(libs):
    """bepucuda_set_contact_features after end_constraints from unregistered buffers, again and again, as a host that sends the feature ids every
    frame does: type batches whose ids are each under 256 KB, 512 MB sent in all. The process's resident memory grows by far less than that, and
    the ids of the last call are the ones the next update_contacts redistributes from: that frame matches the host path bit for bit."""
    kw = dict(substeps=3, velocity_iterations=2)
    host, dev = util.make_sim(_pile(0.3), **kw), util.make_sim(_pile(0.3), **kw)
    rng_h, rng_d = np.random.default_rng(9), np.random.default_rng(9)
    ts = bp.CudaTimestepper(dev, strict_fp=True)
    try:
        ts.describe()
        feat_h, feat_d = resident.initial_features(host, rng_h), resident.initial_features(dev, rng_d)
        ts.set_contact_features(feat_d)
        ob.solve(host, DT)
        ts.solve_device_only(DT)  # resident impulses that belong to feat_d
        ts.download_body_motion()
        assert max(ids.nbytes for ids in feat_d.values()) < 256 << 10
        wrong = {key: ids + (1 << 21) for key, ids in feat_d.items()}  # match nothing: a device that kept these would redistribute differently
        per_call = sum(ids.nbytes for ids in feat_d.values())
        calls = -(-(512 << 20) // per_call)
        before = _resident_bytes()
        for i in range(calls):
            ts.set_contact_features(feat_d if i == calls - 1 else wrong)
        ts.synchronize()
        grown = _resident_bytes() - before
        assert grown < 32 << 20, "resident memory grew by %d MB while %d MB of feature ids were sent" % (grown >> 20, (calls * per_call) >> 20)
        new_h = resident.narrow_phase_like_update(host, feat_h, rng_h)
        for tb in host.type_batches():
            key = (tb.batch_index, tb.type_batch_index)
            if key in new_h:
                ob.update_contact_impulses(tb, feat_h[key], new_h[key])
        ts.upload_body_motion()
        ts.update_contacts(resident.narrow_phase_like_update(dev, feat_d, rng_d))
        ob.solve(host, DT)
        ts.solve_device_only(DT)
        ts.download_bodies()
        ts.download_impulses()
        ts.download_prestep()
    finally:
        ts.close()
    util.compare(util.snapshot(host), util.snapshot(dev), exact=True)


@pytest.mark.gpu
def test_update_contacts_state_errors(libs):
    """update_contacts before set_contact_features and twice without a solve: BAD_STATE; on a joint type batch: INVALID_ARGUMENT. update_type_batch
    after update_contacts hands the impulses back to the host: the next solve starts from the host's values (no redistribution)."""
    scene = scenes.merge(scenes.shape_pile(600, seed=8), scenes.ragdolls(4, seed=9))
    host, dev = util.make_sim(scene), util.make_sim(scene)
    rng = np.random.default_rng(4)
    ts = bp.CudaTimestepper(dev, strict_fp=True)
    try:
        ts.describe()
        feats = resident.initial_features(dev, rng)
        key = sorted(feats)[0]
        with pytest.raises(bp.BepuCudaError) as e:
            ts.update_contacts({key: feats[key]})
        assert e.value.code == ERR_BAD_STATE
        ts.set_contact_features(feats)
        joint = next(tb for tb in dev.type_batches() if not contact_count(tb.type_id))
        ids = np.zeros((joint.constraint_count, 4), dtype=np.int32)
        rc = ts._cuda.bepucuda_update_contacts(ts._ctx, joint.batch_index, joint.type_batch_index, joint.prestep.ctypes.data, ids.ctypes.data)
        assert rc == ERR_INVALID_ARGUMENT
        ts.solve_device_only(DT)
        ob.solve(host, DT)
        ts.download_bodies()
        ts.download_impulses()
        ts.download_prestep()
        util.compare(util.snapshot(host), util.snapshot(dev), exact=True)
        new = {k: v + 1 for k, v in feats.items()}  # nothing matches: every contact would get the mean of the old impulses
        ts.update_contacts(new)
        with pytest.raises(bp.BepuCudaError) as e:
            ts.update_contacts(new)
        assert e.value.code == ERR_BAD_STATE
        for tb in dev.type_batches():  # the host takes every contact type batch back, with its own impulses (the ones the last solve left)
            if contact_count(tb.type_id):
                resident.update_type_batch(ts, tb)
        ts.solve_device_only(DT)
        ob.solve(host, DT)  # no redistribution on the host either
        ts.download_bodies()
        ts.download_impulses()
        ts.download_prestep()
    finally:
        ts.close()
    util.compare(util.snapshot(host), util.snapshot(dev), exact=True)


def _within_one_frame_tolerances(a, b, rel_rms=1e-3, max_abs=2e-2):
    """DESIGN §5's fast-build bounds, per quantity: body poses, linear and angular velocities, and the accumulated impulses and prestep rows of
    all contact type batches together and of all joint type batches together (valid lanes), each within relative RMS and max abs error."""
    def check(x, y, what):
        x, y = np.asarray(x, dtype=np.float64), np.asarray(y, dtype=np.float64)
        assert np.isfinite(y).all(), "%s: non-finite values" % what
        d = np.abs(x - y)
        rms = np.sqrt((d ** 2).sum() / (x ** 2).sum())
        assert rms <= rel_rms, "%s: relative RMS error %.3e > %.1e" % (what, rms, rel_rms)
        assert d.max() <= max_abs, "%s: max abs error %.3e > %.1e" % (what, d.max(), max_abs)

    for label, cols in (("body poses", np.r_[0:7]), ("body linear velocities", np.r_[8:11]), ("body angular velocities", np.r_[12:15])):
        check(a["bodies"][:, cols], b["bodies"][:, cols], label)
    for kind, select in (("contact", lambda t: contact_count(t) > 0), ("joint", lambda t: contact_count(t) == 0)):
        for rows in ("impulses", "prestep"):
            pairs = [(ta[rows].transpose(0, 2, 1)[ta["valid"]], tb[rows].transpose(0, 2, 1)[ta["valid"]])
                     for ta, tb in zip(a["type_batches"], b["type_batches"]) if select(ta["key"][2])]
            check(np.concatenate([x.ravel() for x, _ in pairs]), np.concatenate([y.ravel() for _, y in pairs]), "%s %s" % (kind, rows))


@pytest.mark.gpu
def test_fast_build_resident_frames_with_joints_deterministic_and_within_tolerance(libs):
    """The fast build (the benchmarked one) through f2 frames of contacts and joints. Two runs of four frames are bitwise equal (run-to-run
    determinism). Held to the oracle one resident frame at a time: a third run stops after three frames and downloads its state; a fourth runs
    the same three frames (bitwise the same, by the determinism above) without any download, its host twin takes the third run's state, and
    both then run one more f2 frame (redistribution, joints warm-starting from the impulses they kept on the device), which must stay within the
    DESIGN §5 one-frame joint tolerances, per quantity (_within_one_frame_tolerances). The fourth run must not download before that frame:
    download_impulses / download_prestep also refresh the device's staging copies of every row, which would hide rows that were rewound
    instead of kept. No velocity kicks here (the strict cases cover the motion upload): the bounds are for the solver's rounding, and from the
    settled third frame single joint type batches already reach 2e-3 relative RMS on their own (measured on an H100); a rewound frame is off
    by 0.4 relative RMS and 2.8 in a body velocity."""
    runs = [resident.resident_frames(_mixed(), strict=False) for _ in range(2)]
    a, b = (util.snapshot(run[1]) for run in runs)
    util.compare(a, b, exact=True)
    _, source, _, _, features = resident.resident_frames(_mixed(), frames=3, strict=False, push=False)
    host, dev, _, _, _ = resident.resident_frames(_mixed(), frames=4, strict=False, take_state=(2, source, features), push=False)
    _within_one_frame_tolerances(util.snapshot(host), util.snapshot(dev))
