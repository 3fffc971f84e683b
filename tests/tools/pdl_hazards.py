"""PDL hazard harness: the stage kernels of libbepucuda_hazard.so (-DBEPU_HAZARD) against the oracle.

Each stage kernel runs a prologue before its grid-dependency wait while its predecessor is still running, and that prologue may load only what the
predecessor does not write (DESIGN §3). Whether a wrong load shows up in an ordinary run depends on timing. The hazard build makes it show every
time: every thread of every PDL kernel spends a delay after its trigger and before any post-wait load or store (pdl_wait_then_trigger), so the
next grid's prologue loads run before any store of its predecessor, provided both grids are resident together (the residency precondition,
tests/test_pdl_hazards.py). With the delay on and no canary, the strict build must equal the oracle bit for bit on every configuration below; with a
canary (a load planted on the wrong side of the wait, bepu_device_types.h) it must differ on the canary's scene.

    BEPUCUDA_VARIANT=hazard python tests/tools/pdl_hazards.py --check   prints one JSON line

The variant library is chosen when the process loads it, and each context reads BEPUCUDA_HAZARD ("delay_us=<n>,canary=<k>") when it is created.
TEST INFRASTRUCTURE: the product never loads the hazard build."""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bepuphysics2_b200 import native, scenes  # noqa: E402
from tests import planner, resident, util  # noqa: E402

DT = 1.0 / 60.0
DELAY_US = 50  # the delay of the checked runs; the residency precondition says what it has to cover
f32 = np.float32
MODES = {"graph": native.EXEC_GRAPH, "stream": native.EXEC_STREAM}
CANARY_SOLVE_VELOCITY, CANARY_ROW_PREFETCH, CANARY_EARLY_WORLD_BEHIND_INCREMENTAL, CANARY_INCREMENTAL_VELOCITY, CANARY_SKIP_SHARD_WAIT = 1, 2, 3, 4, 5


def with_kinematics(scene, fraction, seed):
    """`scene` with a random `fraction` of its bodies kinematic and moving. Constraints whose slot 0 is kinematic, or that hold more than one
    kinematic body, are dropped, so kinematic bodies sit in slot 1 of two-body contacts only."""
    bodies = scene["bodies"].copy()
    rng = np.random.default_rng(seed)
    kin = rng.random(bodies.shape[0]) < fraction
    bodies[kin, 16:23] = 0.0
    bodies[kin, 8:11] = rng.uniform(-0.3, 0.3, size=(int(kin.sum()), 3)).astype(f32)
    bodies[kin, 12:15] = rng.uniform(-0.2, 0.2, size=(int(kin.sum()), 3)).astype(f32)
    kept = []
    for type_id, handles, prestep in scene["constraints"]:
        keep = ~kin[handles[:, 0]] & (kin[handles].sum(axis=1) <= 1)
        if keep.any():
            kept.append((type_id, handles[keep], prestep[keep]))
    return {"bodies": bodies, "constraints": kept}


def pile():
    return scenes.shape_pile(2500, seed=6)


def mixed(seed=7):
    return scenes.merge(scenes.shape_pile(1200, seed=seed, nonconvex_fraction=0.3), scenes.ragdolls(4, seed=seed + 1),
                        scenes.joint_zoo(400, per_type=8, seed=seed + 2, kinematic_fraction=0.1))


def single_batch_pile():
    return planner.single_batch(scenes.shape_pile(800, seed=17))


def deep():
    """A reduced copy of the deep-batch scene of tests/test_deep_batches.py: a 160 k-body pile whose head batches are deep, with every joint type
    in its first two batches and moving constrained kinematics."""
    joints = scenes.merge(scenes.joint_zoo(3000, per_type=60, seed=22), scenes.ragdolls(30, seed=23))
    joints["constraints"] = joints["constraints"][::-1]
    scene = scenes.merge(scenes.shape_pile(DEEP_PILE_BODIES, seed=21, nonconvex_fraction=0.3), planner.in_first_batches(joints, 2))
    kin = np.flatnonzero(scene["bodies"][:, 22] == 0)
    rng = np.random.default_rng(25)
    scene["bodies"][kin, 8:11] = rng.uniform(-0.3, 0.3, size=(kin.size, 3)).astype(f32)
    scene["bodies"][kin, 12:15] = rng.uniform(-0.2, 0.2, size=(kin.size, 3)).astype(f32)
    return scene


DEEP_PILE_BODIES = 160_000


def terms(n):
    return np.random.default_rng(31).uniform(-5, 5, size=(n, 8)).astype(f32), (1.0, -40.0, 2.0), 800.0


# name: (scene, keyword arguments of util.make_sim, kind, extra). kind: "single" (one context, frames with refresh), "terms" (one context with
# per-body accelerations and point gravity), "resident" (two resident frames through set_contact_features / update_contacts), "ranks" (extra =
# rank count, contexts of one process wired as peers), "fallback_ranks" (the same with a sequential fallback batch on one rank).
CONFIGS = {
    "pile_kinematics_4x2": (lambda: with_kinematics(pile(), 0.03, 8), dict(substeps=4, velocity_iterations=2), "single", None),
    "pile_4x2": (pile, dict(substeps=4, velocity_iterations=2), "single", None),
    "single_batch_pile_1x3": (single_batch_pile, dict(substeps=1, velocity_iterations=3), "single", None),
    "mixed_fallback": (mixed, dict(substeps=2, velocity_iterations=2, fallback_batch_threshold=6), "single", None),
    "joint_zoo": (lambda: scenes.joint_zoo(600, 20, seed=4, kinematic_fraction=0.1), dict(substeps=2, velocity_iterations=2), "single", None),
    "schedule_0_3_1": (lambda: mixed(5), dict(substeps=3, velocity_iterations=[0, 3, 1], fallback_batch_threshold=6), "single", None),
    "schedule_2_0_2": (lambda: with_kinematics(pile(), 0.03, 8), dict(substeps=3, velocity_iterations=[2, 0, 2]), "single", None),
    "angular_mode_1": (mixed, dict(substeps=2, velocity_iterations=2, integrator=util.integrator(angular_integration_mode=1)), "single", None),
    "accelerations_point_gravity": (mixed, dict(substeps=2, velocity_iterations=2), "terms", None),
    "resident_frames": (lambda: scenes.shape_pile(3000, seed=31, nonconvex_fraction=0.3), {}, "resident", None),
    "ranks_2": (lambda: scenes.shape_pile(2500, seed=6), dict(substeps=4, velocity_iterations=2), "ranks", 2),
    "ranks_3_fallback": (lambda: scenes.fallback_stress(3000, hubs=6, seed=7), dict(fallback_batch_threshold=4, substeps=2, velocity_iterations=2),
                         "fallback_ranks", 3),
    "deep": (deep, dict(substeps=3, velocity_iterations=[2, 0, 1], integrator=util.integrator()), "single", None),
}
# canary: (name, the configurations it must be caught on). Row prefetch is caught twice: behind a stage of the same batch (Solve after Solve in a
# single-batch pile) and behind the incremental update (the first WarmStart's depth rows, in a pile without kinematic passes).
CANARIES = {
    CANARY_SOLVE_VELOCITY: ("solve_velocity_before_wait", ["pile_4x2"]),
    CANARY_ROW_PREFETCH: ("row_prefetch_without_flag", ["single_batch_pile_1x3", "pile_4x2"]),
    CANARY_EARLY_WORLD_BEHIND_INCREMENTAL: ("early_world_behind_incremental", ["pile_4x2"]),
    CANARY_INCREMENTAL_VELOCITY: ("incremental_velocity_before_wait", ["pile_4x2"]),
    CANARY_SKIP_SHARD_WAIT: ("boundary_warps_skip_shard_wait", ["ranks_2"]),
}


def make_sim(name):
    make, kw, _, _ = CONFIGS[name]
    return util.make_sim(make(), **kw)


_ORACLE = {}


def _oracle(name, scene, kw, frames, with_terms):
    if name not in _ORACLE:
        sim = util.make_sim(scene, **kw)
        acc, center, strength = terms(sim.body_count) if with_terms else (None, None, 0.0)
        _ORACLE[name] = util.run_oracle(sim, DT, frames=frames, threads=16, simd=True, accelerations=acc, center=center, strength=strength)
    return _ORACLE[name]


def run(name, mode, hazard):
    """One run of configuration `name` in execution mode `mode` under BEPUCUDA_HAZARD=`hazard`: None when it equals the oracle bit for bit, the
    first difference otherwise."""
    make, kw, kind, extra = CONFIGS[name]
    os.environ["BEPUCUDA_HAZARD"] = hazard
    scene = make()
    try:
        if kind in ("single", "terms"):
            frames = 1 if name == "deep" else 2
            sim = util.make_sim(scene, **kw)
            got = util.run_gpu(sim, DT, frames=frames, mode=MODES[mode], terms=terms(sim.body_count) if kind == "terms" else None)
            util.compare(_oracle(name, scene, kw, frames, kind == "terms"), got, exact=True)
        elif kind == "resident":
            host, dev, _, _, _ = resident.resident_frames(scene, frames=2, mode=MODES[mode])
            util.compare(util.snapshot(host), util.snapshot(dev), exact=True)
        else:
            util.run_ranks(scene, extra, frames=2, mode=mode, **kw)
    except AssertionError as e:
        return str(e).split("\n")[0][:300]
    finally:
        os.environ.pop("BEPUCUDA_HAZARD", None)
    return None


def check():
    import torch

    assert os.environ.get("BEPUCUDA_VARIANT") == "hazard", "run with BEPUCUDA_VARIANT=hazard"
    props = torch.cuda.get_device_properties(0)
    out = {"device": props.name, "sm_count": props.multi_processor_count, "delay_us": DELAY_US, "scenes": {}, "canaries": {}}
    for name in CONFIGS:
        for mode in MODES:
            t0 = time.time()
            out["scenes"]["%s/%s" % (name, mode)] = {"difference": run(name, mode, "delay_us=%d" % DELAY_US), "seconds": round(time.time() - t0, 2)}
    for canary, (label, names) in CANARIES.items():
        for name in names:
            key = "%d_%s/%s" % (canary, label, name)
            delayed = run(name, "stream", "delay_us=%d,canary=%d" % (DELAY_US, canary))
            plain = run(name, "stream", "delay_us=0,canary=%d" % canary)
            out["canaries"][key] = {"caught_with_delay": delayed is not None, "caught_without_delay": plain is not None, "difference": delayed}
    return out


if __name__ == "__main__":
    if "--check" not in sys.argv:
        sys.exit(__doc__)
    print(json.dumps(check()))
