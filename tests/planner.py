"""The constraint topology planner without a GPU: csrc/bepu_topology.cpp (which device batch every constraint runs in, the work list, the stage
program and how each of its stages is launched) compiled for the host with g++ behind tests/topology/topology_shim.cpp, and what the planner tests
share: its constants, the plan and program readers, the launch rules and the scenes. TEST INFRASTRUCTURE: the product never loads the shim."""
import ctypes as C
import json
import os
import re

import numpy as np

from bepuphysics2_b200 import _build, scenes
from tests import harness

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "bepuphysics2_b200", "csrc")

# The reference's constraint layouts by BatchTypeId (tests/golden/type_layouts.json, generated from its C# sources): bodies and the names of the
# prestep and accumulated-impulse rows. The contact facts below are read from the row names.
with open(os.path.join(ROOT, "tests", "golden", "type_layouts.json")) as f:
    TYPE_LAYOUTS = {int(k): v for k, v in json.load(f)["types"].items()}


def depth_rows(type_id):
    """Prestep rows of a type's contact depths (Contact<i>.Depth) in contact order; [] for joints."""
    return [r for r, name in enumerate(TYPE_LAYOUTS[type_id]["prestep_rows"]) if re.fullmatch(r"Contact\d\.Depth", name)]


def penetration_rows(type_id):
    """Accumulated-impulse rows of a type's penetration impulses (Penetration<i>, Contact<i>.Penetration) in contact order; [] for joints."""
    return [r for r, name in enumerate(TYPE_LAYOUTS[type_id]["impulse_rows"]) if re.fullmatch(r"Penetration\d|Contact\d\.Penetration", name)]


def contacts(type_id):
    """Contacts per constraint of a type id; 0 for joints and ids without a type."""
    return len(depth_rows(type_id)) if type_id in TYPE_LAYOUTS else 0


CONTACT_TYPES = {t for t in TYPE_LAYOUTS if contacts(t)}
WS_FIRST, WS, SOLVE, INCREMENTAL, KIN_FIRST, KIN, FINAL = range(7)
NO_EXCHANGE, RANK_BARRIER = -1, -2
ROWS_FREE, CONTACTS_ONLY, BODIES_FREE, INTEGRABLE = 2, 8, 16, 32  # facts of a program op (kOp*)
KERNEL_FULL, KERNEL_CONTACTS, KERNEL_DEEP = range(3)  # StageKernel
PDL, ROWS, EXT, EARLY_WORLD, EARLY_OWNED, BODIES_INTEGRATED = 1, 2, 4, 8, 16, 32  # launch flags (kLaunch*)
KINEMATIC_BIT, INDEX_MASK = 1 << 30, 0x0FFFFFFF
ERR_INVALID_ARGUMENT, ERR_BATCH_INVARIANT, ERR_BAD_STATE = -1, -5, -6


def read_source(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def source_int(name, pattern):
    m = re.search(pattern, read_source(name), re.M)
    assert m, pattern
    return int(m.group(1))


DEEP_BUNDLES = source_int("bepu_topology.h", r"^constexpr int32_t kDeepBatchBundles = (\d+);")


_SHIM = None


def shim():
    """The topology shim, built and loaded once per process."""
    global _SHIM
    if _SHIM is not None:
        return _SHIM
    cuda_include = os.path.join(os.path.dirname(os.path.dirname(_build.NVCC)), "include")
    dll = harness.load("topology_shim", [os.path.join(ROOT, "tests", "topology", "topology_shim.cpp"), os.path.join(CSRC, "bepu_topology.cpp")],
                       ["-O2", "-std=c++17", "-Wall", "-shared", "-fPIC", "-I", cuda_include], includes=[CSRC, os.path.join(ROOT, "include")])
    vp, i32 = C.c_void_p, C.c_int32
    dll.topology_plan.restype = vp
    dll.topology_plan.argtypes = [i32, vp, vp, i32, i32, i32, i32, i32, i32, i32]
    dll.topology_plan_error.argtypes = [vp, C.c_char_p, i32]
    for name in ("sizes", "tbs", "maps", "work", "batches", "source_live"):
        getattr(dll, "topology_plan_" + name).argtypes = [vp, vp]
    dll.topology_plan_inverse_size.restype = C.c_int64
    dll.topology_plan_inverse_size.argtypes = [vp]
    dll.topology_plan_inverse.argtypes = [vp, vp, vp, vp]
    dll.topology_plan_free.argtypes = [vp]
    dll.topology_program.restype = vp
    dll.topology_program.argtypes = [vp, i32, vp, i32, i32, i32, i32]
    dll.topology_program_sizes.argtypes = [vp, vp]
    dll.topology_program_ops.argtypes = [vp, vp]
    dll.topology_program_free.argtypes = [vp]
    dll.topology_exchange_targets.argtypes = [vp, i32, vp, i32, i32, i32, vp, vp]
    dll.topology_resolve.argtypes = [vp, i32, i32, i32, i32, vp]
    dll.topology_same_launches.argtypes = [i32] * 6
    dll.topology_integrated_warm_start_launch.argtypes = [i32] * 3
    dll.topology_type_info.restype = C.c_char_p
    dll.topology_type_info.argtypes = [i32, vp]
    _SHIM = dll
    return dll


def type_info(type_id):
    """The planner's get_type_info of a type id and the access-filter float counts of its type table row, by name; None for an id without a type."""
    out = np.zeros(11, dtype=np.int64)
    name = shim().topology_type_info(type_id, out.ctypes.data)
    fields = "bodies prestep_rows impulse_rows contacts solve_bytes warm_start_bytes incremental_bytes solve_read solve_written warm_start_read warm_start_written"
    return None if name is None else dict(zip(fields.split(), out.tolist()), name=name.decode())


class Plan:
    def __init__(self, handle):
        self.dll, self.handle = shim(), handle
        s = np.zeros(11, dtype=np.int64)
        self.dll.topology_plan_sizes(handle, s.ctypes.data)
        n_tbs, n_maps, n_work, n_batches, n_sources = (int(v) for v in s[:5])
        self.all_work_count, self.sync_batch_count, self.fallback_levels, self.constraint_count, self.inc_begin, self.inc_count = (int(v) for v in s[5:])
        self.tbs = np.zeros((n_tbs, 5), dtype=np.int64)  # type id, bundle count, device batch, source, map offset
        self.maps = np.zeros(n_maps, dtype=np.int32)
        self.work = np.zeros((n_work, 3), dtype=np.int32)  # type batch, bundle, live lanes
        self.batches = np.zeros((n_batches, 3), dtype=np.int32)  # begin, count, contacts only
        self.source_live = np.zeros(n_sources, dtype=np.int32)
        for name, a in (("tbs", self.tbs), ("maps", self.maps), ("work", self.work), ("batches", self.batches), ("source_live", self.source_live)):
            getattr(self.dll, "topology_plan_" + name)(handle, a.ctypes.data)

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


def plan(sources, W, threshold, batch_count, body_count, peer_mode=False, rank=0, fallback_rank=-1):
    """sources: (batch, type batch, type id, count, references[bundles, bodies, W]). In peer mode the plan of `rank`, with `fallback_rank` the
    rank that owns the fallback batch (-1 = none). A Plan, or (error code, message)."""
    dll = shim()
    n = len(sources)
    meta = np.array([s[:4] for s in sources], dtype=np.int32).reshape(n, 4)
    refs = [np.ascontiguousarray(s[4], dtype=np.int32) for s in sources]
    ptrs = (C.c_void_p * max(n, 1))(*[r.ctypes.data for r in refs])
    h = dll.topology_plan(n, meta.ctypes.data, ptrs, W, threshold, batch_count, body_count, int(peer_mode), rank, fallback_rank)
    message = C.create_string_buffer(256)
    rc = dll.topology_plan_error(h, message, 256)
    if rc != 0:
        dll.topology_plan_free(h)
        return rc, message.value.decode()
    return Plan(h)


def inverse_of(p):
    """The inverse slot map of a plan: per source its device type batch (synchronized) and its first inverse entry (fallback); per inverse entry
    its device type batch and slot."""
    n_sources = len(p.source_live)
    source_tb = np.zeros(n_sources, dtype=np.int32)
    offsets = np.zeros(n_sources, dtype=np.int64)
    size = int(p.dll.topology_plan_inverse_size(p.handle))
    inverse = np.zeros((max(size, 1), 2), dtype=np.int32)
    p.dll.topology_plan_inverse(p.handle, source_tb.ctypes.data, offsets.ctypes.data, inverse.ctypes.data)
    return source_tb, offsets, inverse[:size]


def resolve(ops, extensions, angular_mode, profile):
    """resolve_stage_launch for every op: [n, 2] kernel, launch flags."""
    ops = np.ascontiguousarray(ops, dtype=np.int64)
    out = np.zeros((len(ops), 2), dtype=np.int32)
    shim().topology_resolve(ops.ctypes.data, len(ops), int(extensions), angular_mode, int(profile), out.ctypes.data)
    return out


LAUNCH_CONTEXTS = [(ext, mode, profile) for ext in (False, True) for mode in (0, 1, 2) for profile in (False, True)]


def check_launches(ops, peer_mode):
    """The launch rules of DESIGN §3 for every op of a program, in every context (integrator extensions, angular mode, profile)."""
    stage, count, facts = ops[:, 0], ops[:, 2], ops[:, 5]
    sharded = (stage <= SOLVE) & (ops[:, 3] != NO_EXCHANGE)
    deep = (stage <= SOLVE) & (count >= shim().topology_deep_batch_bundles())
    integrating = (stage == WS_FIRST) | (stage == WS)
    has_contacts = bool((stage == INCREMENTAL).any())
    for ext, mode, profile in LAUNCH_CONTEXTS:
        kernel, flags = resolve(ops, ext, mode, profile).T
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
        # and every load the program allows is made (the prologue rule test of tests/test_topology.py checks that each is sound)
        allowed = ((facts & BODIES_FREE) != 0) & ~deep & ~sharded & (not profile)
        assert (owned == allowed & integrating & ~integrated).all()
        assert (world == allowed & ((stage == SOLVE) | ((stage == WS) & integrated & contacts_kernel & ((flags & ROWS) != 0)))).all()


def sim_sources(sim):
    return [(tb.batch_index, tb.type_batch_index, tb.type_id, tb.constraint_count, tb.body_references) for tb in sim.type_batches()]


def shard_sources(shard):
    return [(d["batch_index"], d["type_batch_index"], d["type_id"], d["count"], d["refs"]) for d in shard]


def constraints_of(p, sources, tb):
    """Source constraint of every lane of planned type batch tb (-1 = padding)."""
    type_id, bundles, _, source, map_offset = (int(v) for v in p.tbs[tb])
    if map_offset >= 0:
        return p.maps[map_offset:map_offset + 32 * bundles]
    lanes = np.arange(32 * bundles)
    return np.where(lanes < sources[source][3], lanes, -1)


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


# ---- scenes ---------------------------------------------------------------------------------------------------------------------------------------

def mixed_scene(seed=3):
    return scenes.merge(scenes.shape_pile(1200, seed=seed, nonconvex_fraction=0.3), scenes.ragdolls(4, seed=seed + 1), scenes.joint_zoo(400, per_type=8, seed=seed + 2, kinematic_fraction=0.1))


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


def in_first_batches(scene, batches):
    """The constraints of `scene` that Solver.Add's first fit (insertion order, dynamic bodies only) places in batches 0..batches-1. Dropping
    the others moves none of these: where a constraint lands depends only on the constraints in the batches below it."""
    dynamic = scene["bodies"][:, 22] != 0
    used = [set() for _ in range(batches)]
    kept = []
    for type_id, handles, prestep in scene["constraints"]:
        keep = []
        for i, row in enumerate(handles.tolist()):
            bodies = [h for h in row if dynamic[h]]
            for b in range(batches):
                if not used[b].intersection(bodies):
                    used[b].update(bodies)
                    keep.append(i)
                    break
        if keep:
            kept.append((type_id, handles[keep], prestep[keep]))
    return {"bodies": scene["bodies"], "constraints": kept}
