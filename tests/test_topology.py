"""The constraint topology plan without a GPU: csrc/bepu_topology.cpp (which device batch every constraint runs in, the work list, the stage
program and how each of its stages is launched) compiled for the host with g++ behind tests/topology/topology_shim.cpp, fed with the type batches of the host mirror.
Every property is stated from the uploaded data: coverage of the work list, the fallback levelisation of DESIGN §2 and its minimality, the stage
order of Solver_Solve.cs:L1419-1479, the exchange sequence of a sharded graph, the launch rules of resolve_stage_launch and the prologue prefetch
rule of DESIGN §3.
TEST INFRASTRUCTURE: the product never loads the shim."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from bepuphysics2_b200 import _build, scenes, sharding
from tests import util

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.join(ROOT, "tests", "topology")
CSRC = os.path.join(ROOT, "bepuphysics2_b200", "csrc")

# BatchTypeId of the reference's contact constraints: convex manifolds 0-7, nonconvex 8-10 and 15-17
CONTACT_TYPES = set(range(11)) | {15, 16, 17}
WS_FIRST, WS, SOLVE, INCREMENTAL, KIN_FIRST, KIN, FINAL = range(7)
NO_EXCHANGE, RANK_BARRIER = -1, -2
ROWS_FREE, CONTACTS_ONLY, BODIES_FREE, INTEGRABLE = 2, 8, 16, 32  # facts of a program op (kOp*)
KERNEL_FULL, KERNEL_CONTACTS, KERNEL_DEEP = range(3)  # StageKernel
PDL, ROWS, EXT, EARLY_WORLD, EARLY_OWNED, BODIES_INTEGRATED = 1, 2, 4, 8, 16, 32  # launch flags (kLaunch*)
KINEMATIC_BIT, INDEX_MASK = 1 << 30, 0x0FFFFFFF
ERR_INVALID_ARGUMENT, ERR_BATCH_INVARIANT, ERR_BAD_STATE = -1, -5, -6


@pytest.fixture(scope="module")
def shim():
    lib = os.path.join(HERE, "libtopology_shim.so")
    srcs = [os.path.join(HERE, "topology_shim.cpp"), os.path.join(CSRC, "bepu_topology.cpp")]
    deps = srcs + [os.path.join(CSRC, f) for f in ("bepu_topology.h", "bepu_device_types.h", "bepu_layout_kernels.h", "bepu_joint_registry.inc")]
    if not os.path.exists(lib) or any(os.path.getmtime(s) > os.path.getmtime(lib) for s in deps):
        cuda_include = os.path.join(os.path.dirname(os.path.dirname(_build.NVCC)), "include")
        subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-Wall", "-shared", "-fPIC", "-I", CSRC, "-I", cuda_include, "-o", lib] + srcs)
    dll = C.CDLL(lib)
    vp, i32 = C.c_void_p, C.c_int32
    dll.topology_plan.restype = vp
    dll.topology_plan.argtypes = [i32, vp, vp, i32, i32, i32, i32, i32]
    dll.topology_plan_error.argtypes = [vp, C.c_char_p, i32]
    for name in ("sizes", "tbs", "maps", "work", "batches", "source_live"):
        getattr(dll, "topology_plan_" + name).argtypes = [vp, vp]
    dll.topology_plan_free.argtypes = [vp]
    dll.topology_program.restype = vp
    dll.topology_program.argtypes = [vp, i32, vp, i32, i32, i32, i32]
    dll.topology_program_sizes.argtypes = [vp, vp]
    dll.topology_program_ops.argtypes = [vp, vp]
    dll.topology_program_free.argtypes = [vp]
    dll.topology_resolve.argtypes = [vp, i32, i32, i32, i32, vp]
    dll.topology_same_launches.argtypes = [i32] * 6
    return dll


class Plan:
    def __init__(self, dll, handle):
        self.dll, self.handle = dll, handle
        s = np.zeros(11, dtype=np.int64)
        dll.topology_plan_sizes(handle, s.ctypes.data)
        n_tbs, n_maps, n_work, n_batches, n_sources = (int(v) for v in s[:5])
        self.all_work_count, self.sync_batch_count, self.fallback_levels, self.constraint_count, self.inc_begin, self.inc_count = (int(v) for v in s[5:])
        self.tbs = np.zeros((n_tbs, 5), dtype=np.int64)  # type id, bundle count, device batch, source, map offset
        self.maps = np.zeros(n_maps, dtype=np.int32)
        self.work = np.zeros((n_work, 3), dtype=np.int32)  # type batch, bundle, live lanes
        self.batches = np.zeros((n_batches, 3), dtype=np.int32)  # begin, count, contacts only
        self.source_live = np.zeros(n_sources, dtype=np.int32)
        for name, a in (("tbs", self.tbs), ("maps", self.maps), ("work", self.work), ("batches", self.batches), ("source_live", self.source_live)):
            getattr(dll, "topology_plan_" + name)(handle, a.ctypes.data)

    def __del__(self):
        self.dll.topology_plan_free(self.handle)

    def program(self, iterations, kinematic_count, integrate_velocity_for_kinematics, peer_mode, body_count):
        """ops[n, 7]: stage, work begin, work count, exchange, exchange index, facts, algorithmic bytes; and the per-solve totals."""
        its = np.asarray(iterations, dtype=np.int32)
        h = self.dll.topology_program(self.handle, its.size, its.ctypes.data, kinematic_count, int(integrate_velocity_for_kinematics), int(peer_mode), body_count)
        s = np.zeros(5, dtype=np.int64)
        self.dll.topology_program_sizes(h, s.ctypes.data)
        ops = np.zeros((int(s[0]), 7), dtype=np.int64)
        self.dll.topology_program_ops(h, ops.ctypes.data)
        self.dll.topology_program_free(h)
        return ops, dict(exchange_count=int(s[1]), stage_count=int(s[2]), constraint_iterations=int(s[3]), algorithmic_bytes=int(s[4]))


def plan(dll, sources, W, threshold, batch_count, body_count, peer_mode=False):
    """sources: (batch, type batch, type id, count, references[bundles, bodies, W]). A Plan, or (error code, message)."""
    n = len(sources)
    meta = np.array([s[:4] for s in sources], dtype=np.int32).reshape(n, 4)
    refs = [np.ascontiguousarray(s[4], dtype=np.int32) for s in sources]
    ptrs = (C.c_void_p * max(n, 1))(*[r.ctypes.data for r in refs])
    h = dll.topology_plan(n, meta.ctypes.data, ptrs, W, threshold, batch_count, body_count, int(peer_mode))
    message = C.create_string_buffer(256)
    rc = dll.topology_plan_error(h, message, 256)
    if rc != 0:
        dll.topology_plan_free(h)
        return rc, message.value.decode()
    return Plan(dll, h)


def resolve(dll, ops, extensions, angular_mode, profile):
    """resolve_stage_launch for every op: [n, 2] kernel, launch flags."""
    ops = np.ascontiguousarray(ops, dtype=np.int64)
    out = np.zeros((len(ops), 2), dtype=np.int32)
    dll.topology_resolve(ops.ctypes.data, len(ops), int(extensions), angular_mode, int(profile), out.ctypes.data)
    return out


LAUNCH_CONTEXTS = [(ext, mode, profile) for ext in (False, True) for mode in (0, 1, 2) for profile in (False, True)]


def check_launches(dll, ops, peer_mode):
    """The launch rules of DESIGN §3 for every op of a program, in every context (integrator extensions, angular mode, profile)."""
    stage, count, facts = ops[:, 0], ops[:, 2], ops[:, 5]
    sharded = (stage <= SOLVE) & (ops[:, 3] != NO_EXCHANGE)
    deep = (stage <= SOLVE) & (count >= dll.topology_deep_batch_bundles())
    integrating = (stage == WS_FIRST) | (stage == WS)
    has_contacts = bool((stage == INCREMENTAL).any())
    for ext, mode, profile in LAUNCH_CONTEXTS:
        kernel, flags = resolve(dll, ops, ext, mode, profile).T
        early = (flags & (EARLY_WORLD | EARLY_OWNED)) != 0
        integrated = (flags & BODIES_INTEGRATED) != 0
        contacts_kernel = kernel == KERNEL_CONTACTS
        assert ((kernel == KERNEL_DEEP) == deep).all(), "deep iff a WarmStart / Solve op at or above the threshold"
        assert (contacts_kernel == ((stage <= SOLVE) & ((facts & CONTACTS_ONLY) != 0) & ~sharded & ~deep)).all()
        assert (((flags & EXT) != 0) == (ext & (integrating | (stage >= KIN_FIRST)))).all(), "kExt on the integrating stages only"
        assert not (early & (deep | sharded)).any() and not (profile and early.any()), "no body record before the wait on deep, sharded or profile launches"
        assert (((flags & PDL) != 0) == (not profile) & (stage <= INCREMENTAL)).all()
        assert (((flags & ROWS) != 0) == (not profile) & ((facts & ROWS_FREE) != 0)).all()
        assert (integrated == (((facts & INTEGRABLE) != 0) & (mode == 0) & (not ext))).all()
        assert not integrated.any() or (has_contacts and not peer_mode and mode == 0 and not ext)
        assert not (integrated & (stage != INCREMENTAL) & (stage != WS)).any(), "the incremental op and later WarmStart ops only"
        # what each instantiation compiles: owned loads in WarmStartFirst / WarmStart, world loads in Solve and the contact-only WarmStart
        world, owned = (flags & EARLY_WORLD) != 0, (flags & EARLY_OWNED) != 0
        assert not (world & owned).any() and not (owned & ~integrating).any() and not (world & (stage == WS_FIRST)).any()
        assert (integrated & contacts_kernel & ((flags & ROWS) != 0))[world & (stage == WS)].all(), "world loads on a WarmStart only behind a flagged one"
        # and every load the program allows is made (the prologue rule test below checks that each is sound)
        allowed = ((facts & BODIES_FREE) != 0) & ~deep & ~sharded & (not profile)
        assert (owned == allowed & integrating & ~integrated).all()
        assert (world == allowed & ((stage == SOLVE) | ((stage == WS) & integrated & contacts_kernel & ((flags & ROWS) != 0)))).all()


def sim_sources(sim):
    return [(tb.batch_index, tb.type_batch_index, tb.type_id, tb.constraint_count, tb.body_references) for tb in sim.type_batches()]


def constraints_of(p, sources, tb):
    """Source constraint of every lane of planned type batch tb (-1 = padding)."""
    type_id, bundles, _, source, map_offset = (int(v) for v in p.tbs[tb])
    if map_offset >= 0:
        return p.maps[map_offset:map_offset + 32 * bundles]
    lanes = np.arange(32 * bundles)
    return np.where(lanes < sources[source][3], lanes, -1)


def mixed_scene(seed=3):
    return scenes.merge(scenes.shape_pile(1200, seed=seed, nonconvex_fraction=0.3), scenes.ragdolls(4, seed=seed + 1), scenes.joint_zoo(400, per_type=8, seed=seed + 2, kinematic_fraction=0.1))


@pytest.mark.parametrize("W", [4, 8, 16])
def test_plan_covers_every_bundle_and_live_constraint_once(libs, shim, W):
    threshold = 6
    sim = util.make_sim(mixed_scene(), bundle_width=W, fallback_batch_threshold=threshold)
    sources = sim_sources(sim)
    p = plan(shim, sources, W, threshold, sim.batch_count, sim.body_count)
    assert p.fallback_levels > 0 and p.sync_batch_count == threshold
    live = {(i, c) for i, (b, _, _, count, refs) in enumerate(sources) for c in range(count) if b < threshold or refs[c // W, 0, c % W] >= 0}
    placed, bundles = [], []
    for tb in range(len(p.tbs)):
        placed += [(int(p.tbs[tb, 3]), int(c)) for c in constraints_of(p, sources, tb) if c >= 0]
        bundles += [(tb, k) for k in range(p.tbs[tb, 1])]
    assert len(placed) == len(set(placed)) and set(placed) == live, "every live constraint exactly once, holes never"
    assert p.constraint_count == len(live) and p.source_live.tolist() == [sum(1 for s, _ in live if s == i) for i in range(len(sources))]
    everything = [tuple(w) for w in p.work[:p.all_work_count, :2].tolist()]
    assert len(everything) == len(set(everything)) and set(everything) == set(bundles)
    assert p.inc_begin == p.all_work_count and p.inc_begin + p.inc_count == len(p.work)
    incremental = [tuple(w) for w in p.work[p.inc_begin:, :2].tolist()]
    assert sorted(incremental) == sorted((tb, k) for tb, k in bundles if p.tbs[tb, 0] in CONTACT_TYPES)
    for tb, k, lanes in p.work.tolist():
        assert lanes == int((constraints_of(p, sources, tb)[32 * k:32 * k + 32] >= 0).sum())
    assert p.work[:p.all_work_count, 2].sum() == p.constraint_count
    begin = 0
    for d, (b0, count, contacts_only) in enumerate(p.batches.tolist()):
        assert b0 == begin
        begin += count
        tbs = {int(t) for t in p.work[b0:b0 + count, 0]}
        assert all(p.tbs[t, 2] == d for t in tbs)
        assert contacts_only == int(all(p.tbs[t, 0] in CONTACT_TYPES for t in tbs))
    assert begin == p.all_work_count and len(p.batches) == p.sync_batch_count + p.fallback_levels


@pytest.mark.parametrize("case", ["fallback_stress", "pile", "kinematic_zoo"])
def test_fallback_levels_keep_the_sequential_order_and_are_minimal(libs, shim, case):
    W = 8
    scene, threshold = {"fallback_stress": (lambda: scenes.fallback_stress(3000, hubs=6, seed=7), 4), "pile": (lambda: scenes.shape_pile(2000, seed=9), 2),
                        "kinematic_zoo": (lambda: scenes.joint_zoo(600, per_type=12, seed=11, kinematic_fraction=0.2), 1)}[case]
    sim = util.make_sim(scene(), bundle_width=W, fallback_batch_threshold=threshold)
    sources = sim_sources(sim)
    p = plan(shim, sources, W, threshold, sim.batch_count, sim.body_count)
    level = {}
    for tb in range(len(p.tbs)):
        if p.tbs[tb, 4] >= 0:
            for c in constraints_of(p, sources, tb):
                if c >= 0:
                    level[(int(p.tbs[tb, 3]), int(c))] = int(p.tbs[tb, 2]) - p.sync_batch_count + 1
    # the reference's sequential fallback loop: sources in (batch, type batch) order, bundle after bundle, all lanes of a bundle at once
    latest, per_level, kinematic_refs, checked = {}, {}, 0, 0
    for i, (b, _, _, count, refs) in enumerate(sources):
        if b < threshold:
            continue
        for k in range(refs.shape[0]):
            bundle = []
            for c in range(k * W, min(count, k * W + W)):
                r = [int(x) for x in refs[k, :, c % W]]
                if r[0] < 0:
                    assert (i, c) not in level, "a hole is never planned"
                    continue
                dynamic = [x & INDEX_MASK for x in r if x >= 0 and not x & KINEMATIC_BIT]
                kinematic_refs += sum(1 for x in r if x >= 0 and x & KINEMATIC_BIT)
                earlier = [latest[x] for x in dynamic if x in latest]
                lv = level[(i, c)]
                assert all(e < lv for e in earlier), "an earlier constraint on the same dynamic body runs in a strictly lower level"
                assert lv == 1 + max(earlier, default=0), "the level is the lowest the sequential order allows"
                for x in dynamic:
                    assert x not in per_level.setdefault(lv, set()), "no level holds a dynamic body twice"
                    per_level[lv].add(x)
                bundle.append((dynamic, lv))
                checked += 1
            for dynamic, lv in bundle:
                for x in dynamic:
                    latest[x] = lv
    assert checked == len(level) > 100
    assert p.fallback_levels == max(level.values()) > 1
    if case == "kinematic_zoo":
        assert kinematic_refs > 0  # and the minimality above counted only dynamic bodies


def test_plan_refuses_what_the_device_cannot_run(libs, shim):
    W = 4

    def contact1(*lanes):  # one bundle of Contact1 (type 4, two bodies) in batch 1, the fallback batch at threshold 1
        refs = np.full((1, 2, W), -1, dtype=np.int32)
        for lane, pair in enumerate(lanes):
            refs[0, :, lane] = pair
        return [(1, 0, 4, len(lanes), refs)]

    assert plan(shim, contact1((0, 1), (2, 1)), W, 1, 2, 4) == (ERR_BATCH_INVARIANT, "end_constraints: a fallback bundle references the same dynamic body more than once")
    assert plan(shim, contact1((0, 4)), W, 1, 2, 4) == (ERR_INVALID_ARGUMENT, "end_constraints: body reference out of range")
    assert plan(shim, contact1((0, 1)), W, 1, 2, 4, peer_mode=True) == (ERR_BAD_STATE, "end_constraints: the sequential fallback batch is not supported across ranks")
    shared_kinematic = plan(shim, contact1((0, 1 | KINEMATIC_BIT), (2, 1 | KINEMATIC_BIT)), W, 1, 2, 4)
    assert shared_kinematic.fallback_levels == 1 and shared_kinematic.constraint_count == 2


def expected_program(p, iterations, kinematic_count, integrate_velocity_for_kinematics, peer_mode, body_count):
    """Solver_Solve.cs:L1419-1479: per substep the incremental contact update and the kinematic integration (substeps > 0) or the first-substep
    kinematic velocity integration, WarmStart of every batch, then the velocity iterations over every batch; the final pose pass last. Peer mode: rank
    barriers around the incremental update and before the final pose, and every synchronized batch is an exchange point on every rank.
    Rows: stage, work begin, work count, exchange, contacts only."""
    ops = []
    barrier = [KIN, 0, 0, RANK_BARRIER, 0]
    for s, its in enumerate(iterations):
        if s > 0:
            if peer_mode:
                ops.append(barrier)
            if p.inc_count:
                ops.append([INCREMENTAL, p.inc_begin, p.inc_count, NO_EXCHANGE, 0])
            if kinematic_count:
                ops.append([KIN, 0, kinematic_count, NO_EXCHANGE, 0])
        elif integrate_velocity_for_kinematics and kinematic_count:
            ops.append([KIN_FIRST, 0, kinematic_count, NO_EXCHANGE, 0])
        if peer_mode:
            ops.append(barrier)
        for stage in [WS_FIRST if s == 0 else WS] + [SOLVE] * its:
            for b, (begin, count, contacts_only) in enumerate(p.batches.tolist()):
                if count or (peer_mode and b < p.sync_batch_count):
                    ops.append([stage, begin, count, b if peer_mode else NO_EXCHANGE, contacts_only])
    if peer_mode:
        ops.append(barrier)
    ops.append([FINAL, 0, body_count, NO_EXCHANGE, 0])
    return np.array(ops, dtype=np.int64)


def check_program(p, ops, totals, iterations, body_count, *args):
    want = expected_program(p, iterations, *args[:3], body_count)
    assert np.array_equal(ops[:, :4], want[:, :4])
    assert ((ops[:, 5] & CONTACTS_ONLY) != 0).tolist() == (want[:, 4] != 0).tolist()
    exchange = ops[:, 3] != NO_EXCHANGE
    assert ops[:, 4].tolist() == (np.cumsum(exchange) - exchange).tolist() and totals["exchange_count"] == exchange.sum()
    assert totals["stage_count"] == int(((ops[:, 2] > 0) | (ops[:, 0] == FINAL)).sum())
    assert totals["constraint_iterations"] == p.constraint_count * sum(iterations)
    assert totals["algorithmic_bytes"] == int(ops[(ops[:, 0] != KIN_FIRST) & (ops[:, 0] != KIN), 6].sum())
    assert ops[-1, 6] == 108 * body_count


@pytest.mark.parametrize("iterations", [[1], [2, 2], [3, 0, 1], [1, 2, 3, 4], [0]])
@pytest.mark.parametrize("integrate_velocity_for_kinematics", [False, True])
def test_stage_program_follows_the_reference_solve_order(libs, shim, iterations, integrate_velocity_for_kinematics):
    sim = util.make_sim(mixed_scene(5), fallback_batch_threshold=6)
    kinematic_count = len(sim.constrained_kinematics)
    assert kinematic_count > 0
    p = plan(shim, sim_sources(sim), 8, 6, sim.batch_count, sim.body_count)
    ops, totals = p.program(iterations, kinematic_count, integrate_velocity_for_kinematics, False, sim.body_count)
    check_program(p, ops, totals, iterations, sim.body_count, kinematic_count, integrate_velocity_for_kinematics, False)
    assert ops[-1, 0] == FINAL


@pytest.mark.parametrize("ranks", [2, 3])
def test_every_rank_of_a_partition_runs_the_same_exchange_sequence(libs, shim, ranks):
    sim = util.make_sim(scenes.merge(scenes.shape_pile(1500, seed=13), scenes.ragdolls(4, seed=14)))
    shards, _, _, _ = sharding.partition(sim, ranks)
    kinematic_count = len(sim.constrained_kinematics)
    for iterations in ([1], [2, 1, 3]):
        sequences = []
        for r in range(ranks):
            sources = [(d["batch_index"], d["type_batch_index"], d["type_id"], d["count"], d["refs"]) for d in shards[r]]
            p = plan(shim, sources, sim.bundle_width, sim.fallback_batch_threshold, sim.batch_count, sim.body_count, peer_mode=True)
            ops, totals = p.program(iterations, kinematic_count, True, True, sim.body_count)
            check_program(p, ops, totals, iterations, sim.body_count, kinematic_count, True, True)
            sequences.append(ops[ops[:, 3] != NO_EXCHANGE][:, [0, 3, 4]].tolist())
        assert all(s == sequences[0] for s in sequences) and len(sequences[0]) > 2 * sim.batch_count


@pytest.mark.parametrize("case", ["mixed", "single_batch", "joints_only", "peer"])
def test_every_launch_follows_the_rules(libs, shim, case):
    """resolve_stage_launch on every op of the programs of these scenes, with iteration schedules that contain zeros, in every launch context."""
    if case == "peer":
        sim = util.make_sim(scenes.merge(scenes.shape_pile(1500, seed=13), scenes.ragdolls(4, seed=14)))
        shards, _, _, _ = sharding.partition(sim, 2)
        plans = [plan(shim, [(d["batch_index"], d["type_batch_index"], d["type_id"], d["count"], d["refs"]) for d in shard], sim.bundle_width,
                      sim.fallback_batch_threshold, sim.batch_count, sim.body_count, peer_mode=True) for shard in shards]
    else:
        scene = {"mixed": lambda: mixed_scene(7), "single_batch": lambda: single_batch(scenes.shape_pile(800, seed=17)),
                 "joints_only": lambda: scenes.joint_zoo(600, 20, seed=4, kinematic_fraction=0.1)}[case]()
        sim = util.make_sim(scene, fallback_batch_threshold=6)
        plans = [plan(shim, sim_sources(sim), 8, 6, sim.batch_count, sim.body_count)]
    assert (plans[0].inc_count == 0) == (case == "joints_only")
    for p in plans:
        for iterations in ([1], [2, 2], [0, 3, 1], [0, 0], [3, 0, 1, 2]):
            for ivk in (False, True):
                ops, _ = p.program(iterations, len(sim.constrained_kinematics), ivk, case == "peer", sim.body_count)
                check_launches(shim, ops, case == "peer")


def test_same_launches_holds_exactly_when_every_op_launches_the_same(libs, shim):
    """same_launches, which decides when a captured graph is re-captured, against resolve_stage_launch on a program with every op kind: for every
    pair of launch contexts it holds exactly when every op resolves to the same launch in both."""
    sim = util.make_sim(mixed_scene(7), fallback_batch_threshold=6)
    p = plan(shim, sim_sources(sim), 8, 6, sim.batch_count, sim.body_count)
    ops, _ = p.program([2, 1], len(sim.constrained_kinematics), True, False, sim.body_count)
    assert set(ops[:, 0].tolist()) == {WS_FIRST, WS, SOLVE, INCREMENTAL, KIN_FIRST, KIN, FINAL} and ((ops[:, 5] & INTEGRABLE) != 0).any()
    launches = {lc: resolve(shim, ops, *lc) for lc in LAUNCH_CONTEXTS}
    for a in LAUNCH_CONTEXTS:
        for b in LAUNCH_CONTEXTS:
            same = shim.topology_same_launches(*(int(v) for v in a + b)) != 0
            assert same == np.array_equal(launches[a], launches[b]), (a, b)


def single_batch(scene):
    """The constraints of `scene` that share no body with an earlier one: the whole scene is one batch."""
    used, kept = set(), []
    for type_id, handles, prestep in scene["constraints"]:
        keep = []
        for i, row in enumerate(handles.tolist()):
            if not used.intersection(row):
                used.update(row)
                keep.append(i)
        if keep:
            kept.append((type_id, handles[keep], prestep[keep]))
    return {"bodies": scene["bodies"], "constraints": kept}


@pytest.mark.parametrize("case", ["mixed", "single_batch"])
def test_prologue_prefetch_only_reads_what_the_previous_stage_does_not_write(libs, shim, case):
    """DESIGN §3: a stage's prologue runs while its immediate predecessor is still running, so it may load only what that predecessor does not write.
    What each stage writes: WarmStart(b) the velocities of b's bodies, and the pose and world inertia of those it integrates (the lowest batch that
    references a body integrates it) unless its launch has kLaunchBodiesIntegrated; WarmStartFirst(b) the velocities of b's bodies and the world
    inertia of those it integrates (IntegrateVelocity moves no pose); Solve(b) velocities and b's impulses; the incremental update the prestep of
    every contact bundle, and with kLaunchBodiesIntegrated the pose and world inertia of every integrated body; the kinematic passes the velocities
    and (substeps > 0) poses of the kinematic bodies. Nothing writes local inertia. The program's facts are checked against the writes of unflagged
    launches. What a resolved launch loads before its wait: rows = b's prestep and impulses; world = world inertia of the bodies in slots 0 and 1,
    and their pose unless the kernel is contact-only; owned = the local inertia and pose of the bodies b integrates; the incremental update with
    kLaunchBodiesIntegrated (integrate_body_pose, launched with PDL) the local inertia and pose of every integrated body. Nothing is known about what
    ran before the first stage."""
    W = 8
    scene = mixed_scene(7) if case == "mixed" else single_batch(scenes.shape_pile(800, seed=17))
    sim = util.make_sim(scene, bundle_width=W, fallback_batch_threshold=6)
    sources = sim_sources(sim)
    p = plan(shim, sources, W, 6, sim.batch_count, sim.body_count)
    assert (len(p.batches) == 1) == (case == "single_batch")
    kinematics = set(int(k) for k in sim.constrained_kinematics)
    slot01, dynamic = [], []  # per device batch: bodies in slots 0 and 1, dynamic bodies
    for d in range(len(p.batches)):
        near, dyn = set(), set()
        for tb in np.flatnonzero(p.tbs[:, 2] == d):
            refs = sources[int(p.tbs[tb, 3])][4]
            for c in constraints_of(p, sources, tb):
                if c >= 0:
                    r = [int(x) for x in refs[c // W, :, c % W]]
                    near.update(x & INDEX_MASK for x in r[:2] if x >= 0)
                    dyn.update(x & INDEX_MASK for x in r if x >= 0 and not x & KINEMATIC_BIT)
        slot01.append(near)
        dynamic.append(dyn)
    integrator = {}
    for d in range(len(p.batches)):
        for x in dynamic[d]:
            integrator.setdefault(x, d)
    integrated = [{x for x in dynamic[d] if integrator[x] == d} for d in range(len(p.batches))]
    contact_batches = {int(p.tbs[t, 2]) for t in p.work[p.inc_begin:, 0]}
    batch_of = {int(b): d for d, b in enumerate(p.batches[:, 0]) if p.batches[d, 1] > 0}

    every_integrated = set().union(*integrated)
    world_loads_on_ws = 0
    body_loads_behind = {WS_FIRST: 0, WS: 0, SOLVE: 0}  # incremental launches with pre-wait body loads, by the stage of their predecessor

    def writes(op, flags=0):
        stage, d = int(op[0]), batch_of.get(int(op[1]))
        if stage == WS_FIRST:
            return {("velocity", x) for x in dynamic[d]} | {("inertia", x) for x in integrated[d]}
        if stage == WS:
            return {("velocity", x) for x in dynamic[d]} | ({(what, x) for x in integrated[d] for what in ("pose", "inertia")} if not flags & BODIES_INTEGRATED else set())
        if stage == SOLVE:
            return {("velocity", x) for x in dynamic[d]} | {("impulses", d)}
        if stage == INCREMENTAL:
            return {("prestep", c) for c in contact_batches} | ({(what, x) for x in every_integrated for what in ("pose", "inertia")} if flags & BODIES_INTEGRATED else set())
        return {(what, x) for x in kinematics for what in (("velocity", "pose") if stage == KIN else ("velocity",))}

    def loads(op, kernel, flags):
        if int(op[0]) == INCREMENTAL:
            return {(what, x) for x in every_integrated for what in ("local", "pose")} if flags & BODIES_INTEGRATED and flags & PDL else set()
        d = batch_of[int(op[1])]
        got = {("prestep", d), ("impulses", d)} if flags & ROWS else set()
        if flags & EARLY_WORLD:
            got |= {(what, x) for x in slot01[d] for what in (("inertia",) if kernel == KERNEL_CONTACTS else ("inertia", "pose"))}
        if flags & EARLY_OWNED:
            got |= {(what, x) for x in integrated[d] for what in ("local", "pose")}
        return got

    for iterations in ([1], [2, 2], [0, 3, 1], [0, 0], [2, 0, 2]):
        for ivk in (False, True):
            ops, _ = p.program(iterations, len(kinematics), ivk, False, sim.body_count)
            previous = None
            for op in ops:
                stage, count = int(op[0]), int(op[2])
                if count == 0:
                    continue
                if stage in (WS_FIRST, WS, SOLVE):
                    d = batch_of[int(op[1])]
                    rows_ok = previous is not None and not writes(previous) & {("prestep", d), ("impulses", d)}
                    bodies_ok = previous is not None and not writes(previous) & {("pose", x) for x in integrated[d]} if stage != SOLVE else \
                        previous is not None and not writes(previous) & {(what, x) for x in slot01[d] for what in ("pose", "inertia")}
                    rows, bodies = bool(op[5] & ROWS_FREE), bool(op[5] & BODIES_FREE)
                    assert rows_ok or not rows, "row prefetch behind a stage that writes the rows"
                    assert bodies_ok or not bodies, "body prefetch behind a stage that writes the records"
                    assert bodies == bodies_ok, "a body prefetch the rule allows is missing"
                    if rows_ok and not rows:
                        # the program is coarser than the rule in two places: behind the incremental update (which it does not track per batch) and
                        # behind a WarmStart of the same batch (single-batch scenes)
                        assert int(previous[0]) == INCREMENTAL or (int(previous[0]) in (WS_FIRST, WS) and previous[1] == op[1]), "a row prefetch the rule allows is missing"
                elif stage == INCREMENTAL:
                    assert op[5] & (ROWS_FREE | BODIES_FREE) == 0, "the incremental update reads its rows after the wait"
                previous = op
            assert ops[0, 5] & (ROWS_FREE | BODIES_FREE) == 0
            # every load of every resolved launch avoids what the resolved launch before it writes
            live = ops[(ops[:, 2] > 0) & (ops[:, 3] != RANK_BARRIER)]
            for ext, mode, profile in LAUNCH_CONTEXTS:
                resolved = resolve(shim, live, ext, mode, profile)
                world_on_ws = 0
                for i, op in enumerate(live):
                    if int(op[0]) not in (WS_FIRST, WS, SOLVE, INCREMENTAL):
                        continue
                    kernel, flags = (int(v) for v in resolved[i])
                    got = loads(op, kernel, flags)
                    assert i > 0 or not got, "a prologue load before the first stage of the solve"
                    clash = got & writes(live[i - 1], int(resolved[i - 1, 1])) if i > 0 else set()
                    assert not clash, "op %d (%s) loads %s that its predecessor writes" % (i, op.tolist(), sorted(clash)[:4])
                    world_on_ws += int(op[0]) == WS and bool(flags & EARLY_WORLD)
                    if got and int(op[0]) == INCREMENTAL:
                        body_loads_behind[int(live[i - 1, 0])] += 1
                world_loads_on_ws += world_on_ws
    assert (world_loads_on_ws > 0) == (case == "mixed"), "the world-inertia load of a flagged WarmStart behind an earlier batch's is covered"
    # the incremental update's body CTAs were checked behind a Solve and, in the substeps without iterations, behind a WarmStart and a WarmStartFirst
    assert body_loads_behind[SOLVE] > 0 and body_loads_behind[WS] > 0 and body_loads_behind[WS_FIRST] > 0, body_loads_behind
