"""Which contact-only WarmStart instantiation each resolved launch runs, without a GPU. A contact-only WarmStart launch with kLaunchBodiesIntegrated
runs integrated_constraint_stage_kernel, which has no pose integration; every other one runs constraint_stage_kernel, which integrates. Each
instantiation compiles only the prologue loads its launches can ask for (DESIGN §3): the integrated one world inertia, the other one local inertia
and pose of the integrating slots, so resolve_stage_launch must never ask an instantiation for a load it does not have.
TEST INFRASTRUCTURE: the shim (tests/topology/launch_instance_shim.cpp) is built into a temporary directory; the product never loads it."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from bepuphysics2_b200 import _build, scenes
from tests import util
from tests.test_topology import (BODIES_INTEGRATED, EARLY_OWNED, EARLY_WORLD, EXT, HERE, KERNEL_CONTACTS, LAUNCH_CONTEXTS, CSRC, WS, mixed_scene, plan,
                                 resolve, sim_sources, single_batch)
from tests.test_topology import shim  # noqa: F401  (fixture)


@pytest.fixture(scope="module")
def instance(tmp_path_factory):
    lib = str(tmp_path_factory.mktemp("launch_instance") / "liblaunch_instance_shim.so")
    cuda_include = os.path.join(os.path.dirname(os.path.dirname(_build.NVCC)), "include")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-Wall", "-shared", "-fPIC", "-I", CSRC, "-I", cuda_include, "-o", lib,
                           os.path.join(HERE, "launch_instance_shim.cpp")])
    dll = C.CDLL(lib)
    dll.topology_integrated_warm_start_launch.argtypes = [C.c_int, C.c_int, C.c_int]
    return dll


@pytest.mark.parametrize("case", ["mixed", "single_batch"])
def test_contact_only_warm_start_launches_run_the_instantiation_that_has_their_loads(libs, shim, instance, case):  # noqa: F811
    scene = mixed_scene(7) if case == "mixed" else single_batch(scenes.shape_pile(800, seed=17))
    sim = util.make_sim(scene, fallback_batch_threshold=6)
    p = plan(shim, sim_sources(sim), 8, 6, sim.batch_count, sim.body_count)
    seen = set()
    for iterations in ([1], [2, 2], [0, 3, 1], [3, 0, 1, 2]):
        ops, _ = p.program(iterations, len(sim.constrained_kinematics), False, False, sim.body_count)
        for ext, mode, profile in LAUNCH_CONTEXTS:
            kernel, flags = resolve(shim, ops, ext, mode, profile).T
            integrated = np.array([instance.topology_integrated_warm_start_launch(int(s), int(k), int(f)) for s, k, f in zip(ops[:, 0], kernel, flags)], dtype=bool)
            contact_ws = (ops[:, 0] == WS) & (kernel == KERNEL_CONTACTS)
            assert (integrated == (contact_ws & ((flags & BODIES_INTEGRATED) != 0))).all()
            assert not (integrated & ((flags & (EXT | EARLY_OWNED)) != 0)).any(), "the integrated instantiation has no kExt and no owned loads"
            assert not (contact_ws & ~integrated & ((flags & EARLY_WORLD) != 0)).any(), "the integrating instantiation has no world loads"
            seen.update(zip(integrated[contact_ws].tolist(), ((flags[contact_ws] & EARLY_WORLD) != 0).tolist()))
    # both instantiations run; the integrated one also with its prologue loads where a WarmStart follows another WarmStart
    assert {(True, False), (False, False)} | ({(True, True)} if case == "mixed" else set()) <= seen, seen
