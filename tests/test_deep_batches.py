"""Deep batches: a device batch of kDeepBatchBundles bundles or more runs its WarmStartFirst / WarmStart / Solve stages in the deep register budget
(constraint_stage_kernel<S, BEPU_DEEP_MINB, kExt, false> in csrc/bepu_solver_kernels.cu: the full type switch at 80 registers, every body record
gathered after the grid-dependency wait). The 100 k-body pile never gets there; the 1 M-body pile of BASELINE C4 does in its first ten batches.
CPU: the threshold and the budget read from the source, the topology plan (the shim of tests/test_topology.py) of every scene the GPU tests below
solve, and the registers and stack frames of the deep kernels in the built library. GPU: the strict build against the oracle, bit for bit, on a
mixed deep scene with every registered type and on the C4 pile; the fast build within the suite's tolerances (max abs taken at the 99.9th
percentile at this scale, see CONTACT_TOLERANCE) and run-to-run deterministic there.
Peer-sharded deep stages are not covered here: their ranks must be co-resident at thousands of CTAs per stage, which needs one GPU per rank."""
import os
import re

import numpy as np
import pytest

from bepuphysics2_b200 import native, scenes
from tests import test_topology as topo
from tests import util
from tests.test_stage_kernel_resources import resident_warps, resource_usage

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "bepuphysics2_b200", "csrc")
DT = 1.0 / 60.0
f32 = np.float32
BODIES_INTEGRATED = 32
WS_FIRST, WS, SOLVE = topo.WS_FIRST, topo.WS, topo.SOLVE

shim = topo.shim


def _read(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _source_int(pattern):
    m = re.search(pattern, _read("bepu_solver_kernels.cu"), re.M)
    assert m, pattern
    return int(m.group(1))


DEEP_BUNDLES = _source_int(r"^constexpr int kDeepBatchBundles = (\d+);")
DEEP_MINB = _source_int(r"^#define BEPU_DEEP_MINB (\d+)$")


def registered_type_ids():
    """The type ids the device registers: the contact types of bepu_topology.cpp and the joints of bepu_joint_registry.inc."""
    ids = {int(t) for t in re.findall(r"add\((\d+), make_contact\(", _read("bepu_topology.cpp"))}
    return ids | {int(t) for t in re.findall(r"^add\((\d+), make_joint\(", _read("bepu_joint_registry.inc"), re.M)}


# ---- the scenes --------------------------------------------------------------------------------------------------------------------------------------

def _in_first_batches(scene, batches):
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


PILE_BODIES = 230_000


def deep_scene():
    """A 230 k-body pile (convex and nonconvex manifolds; its first six batches are deep) merged with every joint type: the zoo, and ragdolls with
    motors and with servos. The joints are added in reverse order, so that the ragdolls' hinges and swivel hinges (added last by scenes.ragdolls)
    find room in the first batches, and only those in the first five batches are kept: batches 0-4 are deep and mixed, batch 5 deep and all
    contacts. The constrained kinematic bodies (zoo partners, the ragdoll tubes) move and spin."""
    joints = scenes.merge(scenes.joint_zoo(12_000, per_type=300, seed=22), scenes.ragdolls(150, seed=23), scenes.ragdolls(150, seed=24, motor="servo"))
    joints["constraints"] = joints["constraints"][::-1]
    scene = scenes.merge(scenes.shape_pile(PILE_BODIES, seed=21, nonconvex_fraction=0.3), _in_first_batches(joints, 5))
    kin = np.flatnonzero(scene["bodies"][:, 22] == 0)
    rng = np.random.default_rng(25)
    scene["bodies"][kin, 8:11] = rng.uniform(-0.3, 0.3, size=(kin.size, 3)).astype(f32)
    scene["bodies"][kin, 12:15] = rng.uniform(-0.2, 0.2, size=(kin.size, 3)).astype(f32)
    return scene


def _integrator(kinematics=1, angular_mode=0):
    d = native.IntegratorDesc.default()
    d.integrate_velocity_for_kinematics = kinematics
    d.angular_integration_mode = angular_mode
    return d


ITERATIONS = [2, 0, 1]


def deep_kw(angular_mode=0):
    return dict(substeps=len(ITERATIONS), velocity_iterations=ITERATIONS, integrator=_integrator(angular_mode=angular_mode))


C4_KW = dict(substeps=4, velocity_iterations=2)


@pytest.fixture(scope="module")
def mixed():
    return deep_scene()


@pytest.fixture(scope="module")
def c4_pile():
    return scenes.shape_pile(1_000_000, seed=5)


def _plan(shim, sim):
    return topo.plan(shim, topo.sim_sources(sim), sim.bundle_width, sim.fallback_batch_threshold, sim.batch_count, sim.body_count)


def _deep(p):
    return [d for d, (_, count, _) in enumerate(p.batches.tolist()) if count >= DEEP_BUNDLES]


# ---- CPU: the threshold, the plans, the budget --------------------------------------------------------------------------------------------------------

def test_threshold_and_budget_come_from_the_source():
    assert DEEP_BUNDLES > 0 and DEEP_MINB > 1
    # every WarmStartFirst / WarmStart / Solve launch at or above the threshold takes the deep budget, contact-only or not
    assert re.search(r"if \(work_count >= kDeepBatchBundles\) return launch_stage_variant<STAGE, BEPU_DEEP_MINB, false>", _read("bepu_solver_kernels.cu"))
    assert len(registered_type_ids()) == 44


def test_mixed_scene_runs_every_type_in_deep_batches(libs, shim, mixed):
    sim = util.make_sim(mixed, **deep_kw())
    p = _plan(shim, sim)
    deep = _deep(p)
    assert deep, p.batches[:, 1].tolist()
    types = {int(t) for t in p.tbs[np.isin(p.tbs[:, 2], deep), 0]}
    assert types == registered_type_ids(), sorted(registered_type_ids() - types)
    contacts_only = [bool(p.batches[d, 2]) for d in deep]
    assert any(contacts_only) and not all(contacts_only), contacts_only
    assert len(sim.constrained_kinematics) > 0
    # substeps > 0 flag every WarmStart of a deep batch: its integrating lanes find pose and world inertia written by the incremental update
    ops, _ = p.program(ITERATIONS, len(sim.constrained_kinematics), True, False, sim.body_count)
    begins = {int(p.batches[d, 0]) for d in deep}
    for stage in (WS_FIRST, WS, SOLVE):
        on_deep = ops[(ops[:, 0] == stage) & np.isin(ops[:, 1], list(begins)) & (ops[:, 2] >= DEEP_BUNDLES)]
        assert len(on_deep) == len(deep) * {WS_FIRST: 1, WS: len(ITERATIONS) - 1, SOLVE: sum(ITERATIONS)}[stage]
        flagged = (on_deep[:, 5] & BODIES_INTEGRATED) != 0
        assert flagged.all() if stage == WS else not flagged.any(), stage
        contacts = (on_deep[:, 5] & topo.CONTACTS_ONLY) != 0
        assert contacts.any() and not contacts.all(), stage


def test_c4_pile_has_deep_batches_and_the_100k_pile_none(libs, shim, c4_pile):
    big = _plan(shim, util.make_sim(c4_pile, **C4_KW))
    assert len(_deep(big)) >= 2, big.batches[:, 1].tolist()
    # the benchmark-scale test of tests/test_gpu_parity.py therefore never runs a deep kernel
    small = _plan(shim, util.make_sim(scenes.shape_pile(100_000, seed=5), substeps=8, velocity_iterations=2))
    assert not _deep(small) and small.batches[:, 1].max() > 0, small.batches[:, 1].tolist()


DEEP_KERNEL = re.compile(r"_ZN\d+(bepu_fast|bepu_strict)23constraint_stage_kernelILi(\d)ELi(\d+)ELb([01])ELb0EE")
# Stack frames of the deep kernels as built today (cuobjdump --dump-resource-usage), observed, not chosen. The out-of-line angular-momentum calls
# take 48 B; the rest is spill of the full switch at 80 registers. An upper bound, so that a growth of the spill fails here.
DEEP_STACK = {("bepu_fast", 0, False): 176, ("bepu_fast", 0, True): 176, ("bepu_fast", 1, False): 304, ("bepu_fast", 1, True): 288, ("bepu_fast", 2, False): 80,
              ("bepu_strict", 0, False): 208, ("bepu_strict", 0, True): 176, ("bepu_strict", 1, False): 288, ("bepu_strict", 1, True): 272, ("bepu_strict", 2, False): 64}


def deep_kernels():
    """(flavour, stage, kExt) -> resources of the deep instantiations: MINB == BEPU_DEEP_MINB and kContacts false (the contact-only Solve has
    the same MINB)."""
    found = {}
    for name, res in resource_usage().items():
        m = DEEP_KERNEL.match(name)
        if m and int(m.group(3)) == DEEP_MINB:
            found[(m.group(1), int(m.group(2)), m.group(4) == "1")] = res
    return found


def test_deep_stage_kernels_exist_for_both_flavours_plain_and_with_extensions():
    # per-body accelerations and point gravity only change the integrating WarmStart stages: Solve has no kExt instantiation
    assert set(deep_kernels()) == set(DEEP_STACK)


def test_deep_stage_kernels_keep_24_warps_resident_without_local_memory_and_with_the_observed_stack():
    found = deep_kernels()
    assert found
    for key, res in found.items():
        assert res["REG"] <= 80 and resident_warps(res["REG"], res["SHARED"]) >= 2 * DEEP_MINB, (key, res)
        assert res["LOCAL"] == 0 and res["STACK"] <= DEEP_STACK[key], (key, res)


# ---- GPU: the strict build against the oracle ---------------------------------------------------------------------------------------------------------

def _oracle(scene, kw, frames, terms=None):
    sim = util.make_sim(scene, **kw)
    acc, center, strength = terms or (None, None, 0.0)
    return util.run_oracle(sim, DT, frames=frames, threads=16, simd=True, accelerations=acc, center=center, strength=strength)


def _device(scene, kw, frames, strict=True, mode=native.EXEC_GRAPH, terms=None, profile=False):
    """Runs `frames` frames (refresh between them) on the device; returns the snapshot and, with profile, the launch count of the last frame."""
    sim = util.make_sim(scene, **kw)
    ts = native.CudaTimestepper(sim, strict_fp=strict, execution_mode=mode)
    launches = None
    try:
        ts.describe()
        if terms:
            ts.set_body_accelerations(terms[0])
            ts.set_point_gravity(terms[1], terms[2])
        for f in range(frames):
            if f > 0:
                ts.refresh()
            if profile:
                launches = sum(ts.profile_stages(DT).launches)
                ts.download_bodies()
                ts.download_impulses()
            else:
                ts.solve(DT, download=True)
            ts.download_prestep()
        if not profile:
            launches = ts.timings().kernel_launches
    finally:
        ts.close()
    return util.snapshot(sim), launches


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [native.EXEC_GRAPH, native.EXEC_STREAM])
def test_mixed_deep_scene_bit_exact(libs, mixed, mode):
    """Deep WarmStartFirst, deep WarmStart with the bodies-integrated flag (pose and world inertia from the incremental update's per-body CTAs),
    deep Solve, a substep without iterations, and constrained kinematics with IntegrateVelocityForKinematics, over three refreshed frames."""
    kw = deep_kw()
    got, _ = _device(mixed, kw, 3, mode=mode)
    util.compare(_oracle(mixed, kw, 3), got, exact=True)


@pytest.mark.gpu
@pytest.mark.parametrize("angular_mode", [1, 2])
def test_mixed_deep_scene_momentum_conserving_modes_bit_exact(libs, mixed, angular_mode):
    """The owning lane keeps the whole integration in the deep WarmStart, including the first-substep bundle quirk."""
    kw = deep_kw(angular_mode)
    got, _ = _device(mixed, kw, 2)
    util.compare(_oracle(mixed, kw, 2), got, exact=True)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [native.EXEC_GRAPH, native.EXEC_STREAM])
def test_mixed_deep_scene_accelerations_and_point_gravity_bit_exact(libs, mixed, mode):
    """Per-body accelerations and point gravity: the deep kExt WarmStart instantiations, which integrate the pose themselves."""
    kw = deep_kw()
    n = mixed["bodies"].shape[0]
    terms = (np.random.default_rng(31).uniform(-5, 5, size=(n, 8)).astype(f32), (1.0, -40.0, 2.0), 800.0)
    got, _ = _device(mixed, kw, 2, mode=mode, terms=terms)
    util.compare(_oracle(mixed, kw, 2, terms=terms), got, exact=True)


@pytest.mark.gpu
def test_mixed_deep_scene_profile_stages_advances_like_solve(libs, mixed):
    kw = deep_kw()
    got, launches = _device(mixed, kw, 2, profile=True)
    util.compare(_oracle(mixed, kw, 2), got, exact=True)
    _, graph_launches = _device(mixed, kw, 1)
    assert launches == graph_launches > 0


@pytest.fixture(scope="module")
def c4_reference(c4_pile):
    """The oracle's state after frame 1 and after frame 2 of the C4 pile at 4 x 2."""
    sim = util.make_sim(c4_pile, **C4_KW)
    first = util.run_oracle(sim, DT, frames=1, threads=16, simd=True)
    return first, util.run_oracle(sim, DT, frames=1, threads=16, simd=True)


@pytest.mark.gpu
def test_c4_pile_bit_exact(libs, c4_pile, c4_reference):
    """BASELINE C4 itself: the 1 M-body pile, 4 substeps x 2 iterations, two frames, graph mode; its first ten batches run the deep kernels."""
    for _ in range(2):  # a race would not show every time
        got, _ = _device(c4_pile, C4_KW, 2)
        util.compare(c4_reference[1], got, exact=True)


# ---- GPU: the fast build ------------------------------------------------------------------------------------------------------------------------------

# The one-frame tolerances of test_fast_build_within_tolerance (contacts: relative RMS 1e-5, max abs 1e-4) and of
# test_joint_zoo_fast_build_within_tolerance (joints: 1e-3, 5e-2) were set on scenes of a few thousand bodies. With hundreds of thousands of
# manifolds a handful of contacts sit at a clamp, where a last-bit difference switches an impulse on or off: one frame of the C4 pile differs by
# up to 4e-3 in a velocity while 99.9 % of the values differ by less than 2e-6, and a build without the deep budget (BEPU_DEEP_MINB=1: the
# uncapped kernels on every batch) gives the same fast-build errors, bit for bit, on both scenes here. So at this scale the max-abs bound holds for
# the 99.9th percentile, and the relative RMS is taken over each quantity as a whole: contacts 5e-5 (measured on an H100: at most 1.2e-5), joints
# 1e-3 (measured 1.1e-5).
CONTACT_TOLERANCE = dict(rel_rms=5e-5, p999=1e-4)
JOINT_TOLERANCE = dict(rel_rms=1e-3, p999=5e-2)


def _contacts_only(snap, bodies):
    """The pile's bodies (which only contacts touch) and the contact type batches of a snapshot."""
    return {"bodies": snap["bodies"][:bodies], "type_batches": [t for t in snap["type_batches"] if t["key"][2] in topo.CONTACT_TYPES]}


def _check_fast(ref, got, label, rel_rms, p999):
    """Relative RMS error and 99.9th percentile of the absolute error of body poses, linear and angular velocities and the accumulated impulses of
    every valid lane, the fast build against the oracle."""
    quantities = {name: (ref["bodies"][:, cols], got["bodies"][:, cols]) for name, cols in (("poses", util.MOTION[:7]), ("linear", util.MOTION[7:10]),
                                                                                             ("angular", util.MOTION[10:]))}
    impulses = [(np.where(v, ta["impulses"], 0).ravel(), np.where(v, tb["impulses"], 0).ravel())
                for ta, tb in zip(ref["type_batches"], got["type_batches"]) for v in [np.broadcast_to(ta["valid"][:, None, :], ta["impulses"].shape)]]
    quantities["impulses"] = (np.concatenate([x for x, _ in impulses]), np.concatenate([y for _, y in impulses]))
    for name, (x, y) in quantities.items():
        x, y = x.astype(np.float64), y.astype(np.float64)
        assert np.isfinite(y).all(), (label, name)
        d = np.abs(x - y)
        rms, q = np.sqrt((d ** 2).sum() / (x ** 2).sum()), np.quantile(d, 0.999)
        print("fast build, %s, %s: relative RMS %.2e, 99.9th percentile %.2e, max abs %.2e" % (label, name, rms, q, d.max()))
        assert rms <= rel_rms and q <= p999, (label, name, rms, q)


@pytest.mark.gpu
def test_mixed_deep_scene_fast_build_within_tolerance(libs, mixed):
    kw = deep_kw()
    ref, (got, _) = _oracle(mixed, kw, 1), _device(mixed, kw, 1, strict=False)
    _check_fast(ref, got, "mixed deep scene", **JOINT_TOLERANCE)
    _check_fast(_contacts_only(ref, PILE_BODIES), _contacts_only(got, PILE_BODIES), "mixed deep scene, pile", **CONTACT_TOLERANCE)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [native.EXEC_GRAPH, native.EXEC_STREAM])
def test_mixed_deep_scene_fast_build_is_run_to_run_deterministic(libs, mixed, mode):
    """A deep batch is several waves of CTAs: no result may depend on which of them runs first."""
    runs = [_device(mixed, deep_kw(), 2, strict=False, mode=mode)[0] for _ in range(3)]
    for other in runs[1:]:
        util.compare(runs[0], other, exact=True)


@pytest.mark.gpu
def test_c4_pile_fast_build_within_tolerance(libs, c4_pile, c4_reference):
    got, _ = _device(c4_pile, C4_KW, 1, strict=False)
    _check_fast(c4_reference[0], got, "C4 pile", **CONTACT_TOLERANCE)
