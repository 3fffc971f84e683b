"""Pins the hand-written oracle (oracle/*.h) to the REFERENCE'S OWN C# TEXT.

The reference cannot be built here (no .NET). Its constraint functions, wide math and pose integration are straight-line code, so
oracle/ref_transpile/cs2cpp.py transpiles those sources mechanically (syntax only; every operator and call is the C# text's, in its order) into
oracle/_ref/libbepu_ref.so, compiled without FMA contraction like RyuJIT's Vector<float> code. Two layers of checks, all BIT FOR BIT:

  * committed known-answer vectors (tests/golden/reference_vectors.npz, generated from the transpiled reference by
    tests/golden/make_reference_vectors.py): every one of the 44 constraint types x {WarmStart, Solve, IncrementallyUpdateForSubstep}, the four
    PoseIntegration functions, and 38 chains of 1000 x (WarmStart; Solve) on the reference's constraint micro-benchmark inputs
    (DemoBenchmarks/*ConstraintBenchmarks*.cs);
  * fresh random inputs (other seeds), generated here, against the transpiled reference's answers on them (tests/golden/reference_fresh_vectors.npz,
    made by tests/golden/make_reference_fresh_vectors.py where a checkout of the reference is at hand).
All of it runs from the committed files alone.

What this file leaves to others: the solver driver (substep loop, batch order, integration responsibilities, gather/scatter, the TypeProcessor bundle
loops, the final pose pass, PredictBoundingBoxes' per-body glue, impulse redistribution) is generic / unsafe C# the transpiler does not cover.
tests/reference_frame.py restates it a second time from the C# text on top of the transpiled library, and
tests/test_oracle_driver_pinned_to_reference.py holds the oracle to that restatement bit for bit; tests/test_oracle.py adds closed-form answers.
TEST INFRASTRUCTURE: nothing in the product loads either library."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from oracle import binding as ob
from tests import util

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
FP = C.POINTER(C.c_float)
DT = 1.0 / 240.0


@pytest.fixture(scope="module")
def oracle(libs):
    lib = ob.load()
    lib.oracle_eval_lane.argtypes = [C.c_int32, C.c_int32, FP, C.c_float, FP, FP, FP, C.c_int32]
    lib.oracle_eval_integration.argtypes = [C.c_int32, FP, FP]
    return lib


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "reference_vectors.npz"))


def test_golden_vectors_cover_every_registered_type(oracle, golden):
    registered = sorted(t for t in range(64) if ob.type_info(t) is not None)
    in_file = sorted(int(k[5:7]) for k in golden.files if k.startswith("lane_") and k.endswith("_states"))
    assert registered == in_file and len(registered) == 44


def test_oracle_reproduces_the_reference_constraint_functions_bit_for_bit(oracle, golden):
    checked = 0
    for type_id in sorted(t for t in range(64) if ob.type_info(t) is not None):
        key = "lane_%02d_" % type_id
        states, vel, imp, pre = (golden[key + n] for n in ("states", "velocities", "impulses", "prestep"))
        bodies, prestep_rows, impulse_rows = ob.type_info(type_id)
        assert states.shape[1:] == (bodies, 14) and imp.shape[1] == impulse_rows and pre.shape[1] == prestep_rows
        for i in range(states.shape[0]):
            for stage in (0, 1, 2):
                v, a, p = vel[i].copy(), imp[i].copy(), pre[i].copy()
                st = np.ascontiguousarray(states[i])
                assert oracle.oracle_eval_lane(type_id, stage, util.float_ptr(st), DT, util.float_ptr(p), util.float_ptr(a), util.float_ptr(v), 1) == 0
                what = "type %d stage %d sample %d" % (type_id, stage, i)
                assert np.array_equal(util.bits(v), util.bits(golden[key + "out%d_velocities" % stage][i])), what + ": velocities"
                assert np.array_equal(util.bits(a), util.bits(golden[key + "out%d_impulses" % stage][i])), what + ": accumulated impulses"
                assert np.array_equal(util.bits(p), util.bits(golden[key + "out%d_prestep" % stage][i])), what + ": prestep"
                checked += 1
        # the vectors exercise the functions: WarmStart and Solve moved the velocities
        assert not np.array_equal(golden[key + "out1_velocities"], vel)
    assert checked == 44 * 3 * 6


def test_oracle_reproduces_the_reference_pose_integration_bit_for_bit(oracle, golden):
    """PoseIntegration.Integrate (custom Sin/Cos, normalisation, |w| <= 1e-15 fallback), RotateInverseInertia, IntegrateAngularVelocityConserveMomentum,
    ...WithGyroscopicTorque (BepuPhysics/PoseIntegrator.cs:L146-253)."""
    for op in range(4):
        ins, outs = golden["integration_%d_in" % op], golden["integration_%d_out" % op]
        for i in range(ins.shape[0]):
            got = np.zeros(outs.shape[1], dtype=np.float32)
            assert oracle.oracle_eval_integration(op, util.float_ptr(np.ascontiguousarray(ins[i])), util.float_ptr(got)) == 0
            assert np.array_equal(util.bits(got), util.bits(outs[i])), "integration function %d sample %d" % (op, i)


def test_oracle_reproduces_the_reference_benchmark_chains_bit_for_bit(oracle, golden):
    """DemoBenchmarks/{One,Two,Three,Four}BodyConstraintBenchmarks[Deep].cs: 1000 x (WarmStart; Solve) at dt = 1/60 from rest on the benchmark's own
    prestep data; a chain amplifies any difference in a single evaluation, and exercises warm starting with the solver's own accumulated impulses."""
    names = list(golden["bench_names"])
    assert len(names) >= 30
    for n, name in enumerate(names):
        k = "bench_%02d_" % n
        tid = int(golden[k + "type"])
        st, p = np.ascontiguousarray(golden[k + "states"]), golden[k + "prestep"].copy()
        v, a = np.zeros_like(golden[k + "out_velocities"]), np.zeros_like(golden[k + "out_impulses"])
        for _ in range(1000):
            oracle.oracle_eval_lane(tid, 0, util.float_ptr(st), 1.0 / 60.0, util.float_ptr(p), util.float_ptr(a), util.float_ptr(v), 1)
            oracle.oracle_eval_lane(tid, 1, util.float_ptr(st), 1.0 / 60.0, util.float_ptr(p), util.float_ptr(a), util.float_ptr(v), 1)
        assert np.isfinite(v).all(), name
        assert np.array_equal(util.bits(v), util.bits(golden[k + "out_velocities"])), name + ": velocities after 1000 iterations"
        assert np.array_equal(util.bits(a), util.bits(golden[k + "out_impulses"])), name + ": accumulated impulses after 1000 iterations"


@pytest.fixture(scope="module")
def fresh():
    """The transpiled reference's answers on the fresh inputs, stored by tests/golden/make_reference_fresh_vectors.py."""
    return np.load(os.path.join(ROOT, "tests", "golden", "reference_fresh_vectors.npz"))


def test_transpiled_reference_covers_all_types_and_reproduces_the_committed_vectors(oracle, golden, fresh):
    assert sorted(fresh["covered_types"].tolist()) == sorted(t for t in range(64) if ob.type_info(t) is not None)
    # both committed files come from the same transpiled library: its Solve on the first type-7 sample, stored with the fresh answers, is the vector
    assert np.array_equal(util.bits(fresh["lane07_out1_velocities"]), util.bits(golden["lane_07_out1_velocities"][0]))


def test_oracle_matches_the_transpiled_reference_on_fresh_inputs(oracle, fresh):
    """Every type, every stage, 32 fresh samples per type (other seeds than the committed vectors), plus degenerate lanes: zero velocities and
    impulses, identical poses, a kinematic partner (zero inverse mass and inertia). The reference's outputs are stored as one SHA-256 per type and
    stage over the bits of every sample's velocities, accumulated impulses and prestep, next to a digest of the inputs they were computed from."""
    import make_reference_fresh_vectors as gen

    got, got_inputs = gen.lane_digests(oracle.oracle_eval_lane)
    types = fresh["lane_types"].tolist()
    assert sorted(got_inputs) == types
    for i, type_id in enumerate(types):
        assert got_inputs[type_id] == fresh["lane_input_digests"][i], "type %d: the seeded inputs are not those the stored answers were computed from" % type_id
        for stage in (0, 1, 2):
            assert got[(type_id, stage)] == fresh["lane_digests"][i, stage], "type %d stage %d: the oracle differs from the transpiled reference" % (type_id, stage)
