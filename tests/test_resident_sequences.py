"""Random sequences of resident calls under the frame protocol of include/bepucuda.h (a frame is solve, changes, then that frame's uploads and
writes): an oracle twin and a resident device twin (strict build) take the same seeded operations, frame by frame, in protocol order.

Changes: body removes with their constraints, body adds with projectile contacts and their feature ids (forwarded with bepuhost_cuda_change), now
and then a whole ragdoll. Uploads and writes: update_contacts of some contact type batches, write_constraints of joint descriptions, write_bodies,
upload_body_motion, accelerations and point gravity set or cleared, set_integrator and set_solve_description (sometimes with the values they
have). The solve: solve_device_only at a dt of its own. Reads: read_constraints, predict_bounding_boxes and find_sleepable_islands. Refused calls:
a body remove while rows are pending, an index out of range, accelerations for another body count; each must raise and change nothing.

Body motion is compared bit for bit after every solve, every read exactly, and every live constraint's record word for word at the end. The
accelerations and shapes are set once and follow the bodies through removes; adds forwarded without them leave the arrays at the old count, so a
frame with adds sets them again. The fast build is held to a device twin that describes again every frame, byte for byte.

A failure names the seed and the operation log up to the failing frame; replay(log, scene, mode) runs a log again, to cut it down by hand."""
import json

import numpy as np
import pytest

import bepuphysics2_b200 as bp
from bepuphysics2_b200 import scenes
from bepuphysics2_b200.native import BODY_ACTIVITY_DTYPE, BODY_SHAPE_DTYPE, ERR_BAD_STATE, ERR_INVALID_ARGUMENT, EXEC_GRAPH, EXEC_STREAM, contact_count
from oracle import binding as ob
from tests import island_checker, util
from tests.resident import body_frame, lane_record, live_handles, narrow_phase_like_update, push_bodies, remove_a_ragdoll, set_description, set_terms
from tests.test_constraint_write import apply_records, changed, records_of

SCENES = {
    "pile_w4": (lambda: scenes.shape_pile(1500, seed=51, nonconvex_fraction=0.3), dict(bundle_width=4)),
    "zoo_fallback_w8": (lambda: scenes.merge(scenes.shape_pile(700, seed=52, nonconvex_fraction=0.4), scenes.joint_zoo(300, per_type=8, seed=53),
                                             scenes.ragdolls(4, seed=54, motor="servo")), dict(bundle_width=8, fallback_batch_threshold=6)),
    "ragdolls_w16": (lambda: scenes.merge(scenes.ragdolls(20, seed=55, motor="motor"), scenes.ragdolls(20, seed=56, motor="servo")), dict(bundle_width=16)),
}
MODES = {"graph": EXEC_GRAPH, "stream": EXEC_STREAM}
SEEDS = range(6)
FRAMES = 11
DTS = (1 / 60, 1 / 144, 1 / 30, 1 / 240, 0.0123)


def make_twin(scene, bundle_width=8, fallback_batch_threshold=64):
    return util.make_sim(scene, bundle_width=bundle_width, fallback_batch_threshold=fallback_batch_threshold, substeps=2, velocity_iterations=2)


# ---- the generator: a log of frames, each a list of operations in protocol order ------------------------------------------------------------------
def generate(seed, scene, fast=False):
    """The operation log of one run: FRAMES frames of (name, arguments...) tuples, JSON-able. `fast`: only operations a twin that describes again
    every frame can mirror (no contact update with device-side redistribution, no refused calls)."""
    rng = np.random.default_rng(seed)
    joints = scene != "pile_w4"
    sub = lambda: int(rng.integers(1 << 31))
    log = []
    for frame in range(FRAMES):
        ops = []
        if frame > 0:
            if rng.random() < 0.5:
                spawn = int(rng.choice([0, 0, 4, 12]))
                ops.append(("change", int(rng.integers(1, 10)), spawn, bool(joints and rng.random() < 0.25), sub()))
            if not fast and rng.random() < 0.6:
                ops.append(("update_contacts", sub()))
            if joints and rng.random() < 0.4:
                ops.append(("write_constraints", sub()))
            if not fast and rng.random() < 0.3:
                ops.append(("refuse", int(rng.integers(3))))
            if rng.random() < 0.4:
                ops.append(("write_bodies", sub()))
            if rng.random() < 0.4:
                ops.append(("upload_body_motion", frame))
        if frame == 0 or rng.random() < 0.3:
            ops.append(("accelerations", bool(rng.random() < 0.6), sub()))
        if rng.random() < 0.3:
            ops.append(("point_gravity", [float(v) for v in rng.uniform(-20, 20, 3)], float(rng.choice([0.0, 300.0])), bool(rng.random() < 0.6)))
        if rng.random() < 0.3:
            unchanged = rng.random() < 0.3
            ops.append(("integrator", None if unchanged else dict(angular_integration_mode=int(rng.integers(3)), allow_substeps_for_unconstrained=int(rng.integers(2)),
                                                                   integrate_velocity_for_kinematics=int(rng.integers(2)), linear_damping=float(rng.choice([0.0, 0.03, 1.0])),
                                                                   angular_damping=float(rng.choice([0.0, 0.5, 1.5])), gravity=[0.0, float(rng.uniform(-15, 0)), 0.0])))
        if rng.random() < 0.3:
            ops.append(("description", None if rng.random() < 0.3 else [int(i) for i in rng.integers(0, 3, size=int(rng.integers(1, 4)))]))
        ops.append(("solve", float(rng.choice(DTS))))
        if rng.random() < 0.5:
            ops.append(("read_constraints", sub()))
        if rng.random() < 0.4:
            ops.append(("bounds", float(rng.choice(DTS)), sub()))
        if rng.random() < 0.3:
            ops.append(("islands", sub()))
        log.append(ops)
    return log


# ---- the twins ----------------------------------------------------------------------------------------------------------------------------------
def random_shapes(rng, n):
    s = np.zeros(n, dtype=BODY_SHAPE_DTYPE)
    s["type"] = rng.choice([0, 1, 2, 4], size=n)
    s["a"], s["b"], s["c"] = rng.uniform(0.1, 1, size=(3, n)).astype(np.float32)
    s["maximum_speculative_margin"] = np.float32(0.2)
    return s


class World:
    """What both twins share: the per-handle records a host keeps (shapes, accelerations, contact feature ids) and the velocity terms in force."""

    def __init__(self, sim, seed):
        rng = np.random.default_rng(seed + 1000)
        self.shape_of = {int(h): s for h, s in zip(sim.body_handles, random_shapes(rng, sim.body_count))}
        self.acc_of = {}
        self.acc_on = False
        self.gravity = None
        self.features = {}  # constraint handle -> its contact feature ids
        for h in live_handles(sim):
            n = contact_count(sim.constraint_location(int(h))[1])
            if n:
                self.features[int(h)] = rng.integers(0, 1 << 20, size=n).astype(np.int32)

    def shapes(self, sim):
        return np.array([self.shape_of[int(h)] for h in sim.body_handles], dtype=BODY_SHAPE_DTYPE)

    def terms(self, sim):
        out = {}
        if self.acc_on:
            out["accelerations"] = np.stack([self.acc_of[int(h)] for h in sim.body_handles])
        if self.gravity is not None:
            out["center"], out["strength"] = self.gravity
        return out


def lane_handles(sim):
    """{(batch, type batch): handle per lane, -1 in holes} of the contact type batches."""
    keys = {(tb.batch_index, tb.type_id): (tb.batch_index, tb.type_batch_index, tb.constraint_count) for tb in sim.type_batches() if contact_count(tb.type_id)}
    out = {(b, t): np.full(n, -1, dtype=np.int64) for b, t, n in keys.values()}
    for h in live_handles(sim):
        b, type_id, i = sim.constraint_location(int(h))
        if (b, type_id) in keys:
            out[keys[(b, type_id)][:2]][i] = h
    return out


def features_by_key(sim, world):
    out = {}
    for key, handles in lane_handles(sim).items():
        tb = next(t for t in sim.type_batches() if (t.batch_index, t.type_batch_index) == key)
        ids = np.zeros((len(handles), contact_count(tb.type_id)), dtype=np.int32)
        for i, h in enumerate(handles):
            if h >= 0:
                ids[i] = world.features[int(h)]
        out[key] = ids
    return out


def locations(sim, handles):
    return np.array([(0,) + sim.constraint_location(int(h)) for h in handles], dtype=np.int32).reshape(-1, 4)


class Run:
    """Both twins and the shared world; `do` applies one operation to both and checks what it reads."""

    def __init__(self, scene, mode, fast=False):
        make, kw = SCENES[scene]
        self.scene_name, self.fast = scene, fast
        s = make()
        self.a, self.b = make_twin(s, **kw), make_twin(s, **kw)  # a: the oracle (or, fast, the describing twin); b: the resident twin
        self.world = World(self.a, 0)
        strict = not fast
        self.ta = bp.CudaTimestepper(self.a, strict_fp=False) if fast else None
        self.tb = bp.CudaTimestepper(self.b, strict_fp=strict, execution_mode=mode)
        self.tb.describe()
        self.tb.set_body_shapes(self.world.shapes(self.b))
        self.tb.set_contact_features(features_by_key(self.b, self.world))
        self.adds_since_arrays = False
        self.pending = False

    def close(self):
        for ts in (self.ta, self.tb):
            if ts is not None:
                ts.close()

    def both(self, fn):
        fn(self.a)
        fn(self.b)

    def do(self, op):
        name, args = op[0], op[1:]
        getattr(self, "op_" + name)(*args)

    # ---- changes
    def op_change(self, removes, spawn, ragdoll, seed):
        """Removes (a ragdoll, then random bodies), then the projectiles and their contacts. Every new contact carries the same feature ids, so
        that they do not depend on the handles the adds were given (freed handles are handed out again)."""
        rng = np.random.default_rng(seed)
        ids = rng.integers(0, 1 << 20, size=4).astype(np.int32)
        for sim in (self.a, self.b):
            if ragdoll:
                remove_a_ragdoll(sim, seed, None)
            frame_rng = np.random.default_rng(seed)
            body_frame(sim, frame_rng, 0, removes)
            bodies_before, constraints_before = set(sim.body_handles.tolist()), set(live_handles(sim).tolist())
            body_frame(sim, frame_rng, spawn, 0)  # the same draws as one body_frame(sim, rng, spawn, removes)
        new_bodies = sorted(set(self.b.body_handles.tolist()) - bodies_before)
        new_constraints = sorted(set(live_handles(self.b).tolist()) - constraints_before)
        assert len(new_bodies) == len(new_constraints) == spawn
        for h in new_constraints:
            self.world.features[h] = ids[:contact_count(4)].copy()
        for h in new_bodies:
            self.world.shape_of[h] = random_shapes(rng, 1)[0]
            self.world.acc_of[h] = rng.normal(size=8).astype(np.float32)
        self.tb.change(np.tile(ids, (spawn, 1)))
        if new_bodies:  # forwarded without shapes and accelerations: both arrays are set again for the new count
            self.tb.set_body_shapes(self.world.shapes(self.b))
            if self.world.acc_on:
                self.tb.set_body_accelerations(self.world.terms(self.b)["accelerations"])

    # ---- uploads and writes
    def op_update_contacts(self, seed):
        keys = sorted(lane_handles(self.a))
        rng = np.random.default_rng(seed)
        chosen = [k for k in keys if rng.random() < 0.6]
        old = features_by_key(self.a, self.world)
        new_a = narrow_phase_like_update(self.a, {k: old[k] for k in chosen}, np.random.default_rng(seed + 1))
        new_b = narrow_phase_like_update(self.b, {k: old[k] for k in chosen}, np.random.default_rng(seed + 1))
        for tb in self.a.type_batches():
            key = (tb.batch_index, tb.type_batch_index)
            if key in new_a:
                ob.update_contact_impulses(tb, old[key], new_a[key])
        self.tb.update_contacts(new_b)
        self.pending = True
        handles = lane_handles(self.a)
        for key, ids in new_a.items():
            for i, h in enumerate(handles[key]):
                if h >= 0:
                    self.world.features[int(h)] = ids[i].copy()

    def op_write_constraints(self, seed):
        rng = np.random.default_rng(seed)
        joints = [int(h) for h in live_handles(self.a) if not contact_count(self.a.constraint_location(int(h))[1])]
        if not joints:
            return
        pick = rng.choice(joints, size=min(len(joints), 12), replace=False)
        loc = locations(self.a, pick)[:, 1:]
        records = changed(records_of(self.a, loc), rng)
        apply_records(self.a, loc, records)
        apply_records(self.b, loc, records)  # the resident twin's host keeps the description it sent
        self.tb.write_constraints(loc, records)  # the describing twin uploads them with its next describe
        self.pending = True

    def op_refuse(self, which):
        """A call the header refuses: a body remove while rows are pending (uploads or writes since the last solve), otherwise one out of range
        or listing a body twice; or accelerations for another body count."""
        n = self.b.body_count
        calls = (lambda: self.tb.remove_bodies([n]), lambda: self.tb.remove_bodies([n - 1, n - 1]),
                 lambda: self.tb.set_body_accelerations(np.zeros((n + 1, 8), dtype=np.float32)))
        code = ERR_BAD_STATE if self.pending and which < 2 else ERR_INVALID_ARGUMENT
        with pytest.raises(bp.BepuCudaError) as e:
            calls[which]()
        assert e.value.code == code

    def op_write_bodies(self, seed):
        rng = np.random.default_rng(seed)
        idx = rng.integers(0, self.b.body_count, size=int(rng.integers(1, 20)))
        kick = rng.normal(size=(len(idx), 3)).astype(np.float32)
        lift = np.float32(rng.uniform(0, 0.5))
        for sim in (self.a, self.b):
            sim.bodies[idx, 8:11] += kick  # duplicates: the kick of the last one counts, as on the device
            sim.bodies[idx[:1], 5] += lift  # one teleport
        self.tb.write_bodies(idx)

    def op_upload_body_motion(self, frame):
        self.both(lambda sim: push_bodies(sim, frame))
        self.tb.upload_body_motion()

    def op_accelerations(self, on, seed):
        rng = np.random.default_rng(seed)
        self.world.acc_on = on
        if on:
            self.world.acc_of = {int(h): rng.normal(size=8).astype(np.float32) for h in self.b.body_handles}
        self.tb.set_body_accelerations(self.world.terms(self.b).get("accelerations"))

    def op_point_gravity(self, center, strength, on):
        self.world.gravity = (center, strength) if on else None
        terms = self.world.terms(self.b)
        self.tb.set_point_gravity(terms.get("center"), terms.get("strength", 0.0))

    def op_integrator(self, fields):
        integ = self.b.integrator if fields is None else util.integrator(**fields)
        for sim in (self.a, self.b):
            sim.set_integrator(bp.IntegratorDesc.from_buffer_copy(integ))
        set_description(self.tb, self.b)

    def op_description(self, iterations):
        its = self.b.velocity_iterations if iterations is None else iterations
        self.both(lambda sim: sim.set_solve_description(len(its), list(its)))
        set_description(self.tb, self.b)

    # ---- the solve
    def op_solve(self, dt):
        terms = self.world.terms(self.a)
        if self.fast:
            self.ta.describe()
            self.ta.set_body_shapes(self.world.shapes(self.a))
            set_terms(self.ta, terms)
            self.ta.solve(dt, download=True)
            self.ta.download_prestep()
        else:
            ob.solve(self.a, dt, **terms)
        self.tb.solve_device_only(dt)
        self.tb.download_bodies()
        self.pending = False
        assert np.array_equal(util.bits(self.a.bodies[:, util.MEANINGFUL]), util.bits(self.b.bodies[:, util.MEANINGFUL])), "bodies after the solve"

    # ---- reads
    def records_a(self, handles):
        if self.fast:
            return self.ta.read_constraints(locations(self.a, handles))
        return np.stack([lane_record(self.a, int(h)) for h in handles]) if len(handles) else np.zeros((0, 64), dtype=np.int32)

    def op_read_constraints(self, seed):
        live = live_handles(self.a)
        assert np.array_equal(live, live_handles(self.b))
        pick = np.random.default_rng(seed).choice(live, size=min(len(live), 40), replace=False)
        assert np.array_equal(self.records_a(pick), self.tb.read_constraints(locations(self.b, pick))), "read_constraints"

    def activities(self, rng, sim):
        act = np.zeros(sim.body_count, dtype=BODY_ACTIVITY_DTYPE)
        energy = (sim.bodies[:, 8:11].astype(np.float64) ** 2).sum(1) + (sim.bodies[:, 12:15].astype(np.float64) ** 2).sum(1)
        act["sleep_threshold"] = (energy * rng.choice([0.5, 2.0], size=sim.body_count)).astype(np.float32)
        act["minimum_timesteps_under_threshold"] = rng.choice([0, 1, 3], size=sim.body_count)
        act["timesteps_under_threshold_count"] = rng.choice([0, 2, 255], size=sim.body_count)
        return act

    def op_bounds(self, dt, seed):
        act_a = self.activities(np.random.default_rng(seed), self.a)
        act_b = act_a.copy()
        terms = self.world.terms(self.a)
        if self.fast:
            want = self.ta.predict_bounding_boxes(dt, act_a)
        else:
            want = ob.predict_bounding_boxes(self.a.bodies, self.world.shapes(self.a), act_a, dt, self.a.integrator, **terms)
        got = self.tb.predict_bounding_boxes(dt, act_b)
        assert np.array_equal(util.bits(want), util.bits(got)), "bounds"
        assert np.array_equal(act_a.view(np.uint8), act_b.view(np.uint8)), "activities"

    def op_islands(self, seed):
        candidates = np.random.default_rng(seed).random(self.b.body_count) < 0.7
        act = np.zeros(self.b.body_count, dtype=BODY_ACTIVITY_DTYPE)
        act["sleep_candidate"] = candidates
        if self.fast:
            want = self.ta.find_sleepable_islands(act)[:3]
        else:
            want = island_checker.find_sleepable_islands(self.a.type_batches(), self.a.body_count, self.a.bundle_width, candidates)
        got = self.tb.find_sleepable_islands(act)[:3]
        for x, y, what in zip(want, got, ("island of body", "roots", "counts")):
            assert np.array_equal(x, y), "islands: " + what

    def finish(self):
        """Every live constraint's record, word for word."""
        live = live_handles(self.b)
        assert np.array_equal(live, live_handles(self.a))
        assert np.array_equal(self.records_a(live), self.tb.read_constraints(locations(self.b, live))), "records at the end"


def replay(log, scene, mode=EXEC_GRAPH, fast=False):
    """Runs an operation log (generate's, or one cut down by hand) on fresh twins. Raises AssertionError naming the frame and operation that
    failed, with the log up to that frame."""
    run = Run(scene, mode, fast)
    try:
        for frame, ops in enumerate(log):
            for op in ops:
                try:
                    run.do(op)
                except AssertionError as e:
                    raise AssertionError("%s: frame %d, operation %s: %s\nlog up to here: %s" % (scene, frame, json.dumps(op), e, json.dumps(log[:frame + 1]))) from None
        run.finish()
        return run
    finally:
        run.close()


def _ops(log):
    return {op[0] for ops in log for op in ops}


def test_the_generated_logs_reach_every_operation():
    """Over the seeds, every scene's logs hold every operation; the ones with joints write joint descriptions and remove whole ragdolls."""
    for scene in SCENES:
        logs = [generate(seed, scene) for seed in SEEDS]
        names = set().union(*map(_ops, logs))
        want = {"change", "update_contacts", "refuse", "write_bodies", "upload_body_motion", "accelerations", "point_gravity", "integrator", "description",
                "solve", "read_constraints", "bounds", "islands"}
        assert want <= names, (scene, want - names)
        if scene != "pile_w4":
            assert "write_constraints" in names
            assert any(op[0] == "change" and op[3] for log in logs for ops in log for op in ops)
        assert any(op[0] == "change" and op[2] == 0 for log in logs for ops in log for op in ops)  # removes alone: the arrays follow the bodies
        assert "update_contacts" not in set().union(*(_ops(generate(seed, scene, fast=True)) for seed in SEEDS))
        log = generate(3, scene)
        assert json.loads(json.dumps(log)) == [[list(op) for op in ops] for ops in log]  # a log is plain data: printed, it replays


@pytest.mark.gpu
@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("seed", SEEDS)
@pytest.mark.parametrize("scene", sorted(SCENES))
def test_a_random_sequence_stays_on_the_oracle(libs, scene, seed, mode):
    try:
        replay(generate(seed, scene), scene, MODES[mode])
    except AssertionError as e:
        raise AssertionError("seed %d, %s mode: %s" % (seed, mode, e)) from None


@pytest.mark.gpu
@pytest.mark.parametrize("scene", sorted(SCENES))
def test_the_fast_build_resident_twin_equals_a_describing_twin(libs, scene):
    try:
        replay(generate(100, scene, fast=True), scene, EXEC_GRAPH, fast=True)
    except AssertionError as e:
        raise AssertionError("seed 100, fast build: %s" % e) from None
