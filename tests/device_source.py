"""tests/device_on_host/device_on_host.cpp: the device headers (csrc/bepu_device_math.cuh, bepu_contacts.cuh, bepu_joints.cuh,
bepu_joints_more.cuh, bepu_integration.cuh, bepu_bounds_math.cuh, bepu_redistribute.cuh) compiled for the host with the arithmetic of the strict
-fmad=false build, one constraint lane of one stage per call, and the inputs the tests feed it. TEST INFRASTRUCTURE: the product never loads it."""
import ctypes as C
import os

import numpy as np

from bepuphysics2_b200 import scenes
from oracle import binding as ob
from tests import harness

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.join(ROOT, "tests", "device_on_host")
CSRC = os.path.join(ROOT, "bepuphysics2_b200", "csrc")
SOURCE = os.path.join(HERE, "device_on_host.cpp")
INCLUDES = (os.path.join(HERE, "stubs"), HERE, CSRC)
LANES = 32


def flags(optimisation=("-O2",)):
    """The harness's g++ flags; `optimisation` replaces -O2 (the coverage build)."""
    return list(optimisation) + ["-std=c++17", *harness.STRICT_FLAGS, "-Wall", "-Wno-unused-function", "-Wno-unknown-pragmas", "-pthread", "-shared", "-fPIC"]


def load():
    """(the harness, the oracle), each with the argument types of its lane, integration and bounds entry points."""
    dev = harness.load("device_on_host", [SOURCE], flags(), INCLUDES)
    fp = C.POINTER(C.c_float)
    dev.device_on_host_eval_lane.argtypes = [C.c_int32, C.c_int32, fp, C.c_float, fp, fp, fp]
    dev.device_on_host_type_info.argtypes = [C.c_int32] + [C.POINTER(C.c_int32)] * 4
    orc = ob.load()
    orc.oracle_eval_lane.argtypes = [C.c_int32, C.c_int32, fp, C.c_float, fp, fp, fp, C.c_int32]
    dev.device_on_host_eval_integration.argtypes = [C.c_int32, fp, fp]
    orc.oracle_eval_integration.argtypes = [C.c_int32, fp, fp]
    return dev, orc


def random_states(rng, bodies):
    """Per body: position, unit orientation, a symmetric positive definite world inverse inertia, inverse mass."""
    out = np.zeros((bodies, 14), dtype=np.float32)
    out[:, 0:3] = rng.normal(0, 2, (bodies, 3))
    q = rng.normal(0, 1, (bodies, 4))
    out[:, 3:7] = q / np.linalg.norm(q, axis=1, keepdims=True)
    for b in range(bodies):
        r = np.linalg.qr(rng.normal(0, 1, (3, 3)))[0]
        m = r @ np.diag(rng.uniform(0.5, 4.0, 3)) @ r.T
        out[b, 7:13] = (m[0, 0], m[1, 0], m[1, 1], m[2, 0], m[2, 1], m[2, 2])
    out[:, 13] = rng.uniform(0.3, 2.0, bodies)
    return out


def prestep_samples():
    """type id -> float32[samples, prestep rows] of valid prestep data, from the same generators the GPU tests and the bench use."""
    samples = {}
    for scene in (scenes.shape_pile(1500, seed=21, nonconvex_fraction=0.5), scenes.joint_zoo(600, per_type=24, seed=21), scenes.ragdolls(6, seed=21), scenes.ragdolls(6, seed=22, motor="servo")):
        for type_id, _, prestep in scene["constraints"]:
            samples.setdefault(int(type_id), []).append(np.asarray(prestep, dtype=np.float32)[:24])
    return {k: np.concatenate(v)[:32] for k, v in samples.items()}
