"""Generates tests/golden/reference_fresh_vectors.npz: what the transpiled reference (oracle/_ref/libbepu_ref.so, built by
oracle/ref_transpile/build_ref.py from a checkout of the reference's C# sources) computes on the "fresh" inputs of
tests/test_oracle_pinned_to_reference.py and tests/test_bounds.py, so that those comparisons run without the reference:

  * covered_types: the constraint type ids the transpiled library implements;
  * lane07_out1_velocities: its Solve on sample 0 of type 7 in reference_vectors.npz (ties this file to that one);
  * lane_types / lane_digests / lane_input_digests: per type id and stage (0 WarmStart, 1 Solve, 2 IncrementallyUpdateForSubstep), SHA-256 of the
    bits of its outputs (velocities, accumulated impulses, prestep, sample after sample) on the seeded inputs of fresh_lane_cases(), and of
    those inputs, so that a change of the input generators is told apart from a change of the oracle;
  * bounds_out: its convex bounds (min.xyz, margin, max.xyz) on the 400 seeded inputs of fresh_bounds_inputs().

    BEPU_REFERENCE_ROOT=<reference checkout> python tests/golden/make_reference_fresh_vectors.py
"""
import ctypes as C
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
for p in (ROOT, os.path.join(ROOT, "tests", "golden"), os.path.join(ROOT, "oracle", "ref_transpile")):
    if p not in sys.path:
        sys.path.insert(0, p)

FP = C.POINTER(C.c_float)
DT_LANE = 1.0 / 240.0
DT_BOUNDS = 1.0 / 60.0
PATH = os.path.join(ROOT, "tests", "golden", "reference_fresh_vectors.npz")


def _ptr(a):
    return a.ctypes.data_as(FP)


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def fresh_lane_cases():
    """(type id, states, velocities, impulses, prestep) per sample: 32 samples per type, prestep rows from the scene generators, random body
    states, velocities and impulses, plus degenerate lanes (zero velocities and impulses, a kinematic partner, identity orientations)."""
    from oracle import binding as ob
    from tests.device_source import prestep_samples, random_states

    samples = prestep_samples()
    rng = np.random.default_rng(991)
    for type_id in sorted(samples):
        bodies, _, impulse_rows = ob.type_info(type_id)
        for n, prestep in enumerate(samples[type_id]):
            states = random_states(rng, bodies)
            vel = rng.normal(0, 1.5, (bodies, 6)).astype(np.float32)
            imp = np.abs(rng.normal(0, 0.2, impulse_rows)).astype(np.float32)
            if n % 8 == 5:
                vel[:] = 0
                imp[:] = 0
            if n % 8 == 6 and bodies > 1:
                states[1, 7:14] = 0  # kinematic partner
            if n % 8 == 7:
                states[:, 3:7] = (0, 0, 0, 1)
            yield type_id, states, vel, imp, prestep


def lane_digests(eval_lane):
    """eval_lane(type_id, stage, states, dt, prestep, impulses, velocities, row stride) -> rc, in place. Returns ({(type, stage): output digest}, {type: input digest})."""
    outputs, inputs = {}, {}
    for type_id, states, vel, imp, prestep in fresh_lane_cases():
        h_in = inputs.setdefault(type_id, hashlib.sha256())
        for a in (states, vel, imp, prestep):
            h_in.update(_bits(a).tobytes())
        for stage in (0, 1, 2):
            p, a, v = prestep.copy(), imp.copy(), vel.copy()
            assert eval_lane(type_id, stage, _ptr(states), DT_LANE, _ptr(p), _ptr(a), _ptr(v), 1) == 0
            h = outputs.setdefault((type_id, stage), hashlib.sha256())
            for x in (v, a, p):
                h.update(_bits(x).tobytes())
    return {k: h.hexdigest() for k, h in outputs.items()}, {k: h.hexdigest() for k, h in inputs.items()}


def fresh_bounds_inputs():
    import make_reference_bounds_vectors as gen

    return gen.make_inputs(np.random.default_rng(77), 400)


def main():
    import build_ref
    import make_reference_bounds_vectors as gen

    if build_ref.build() is None:
        raise SystemExit("no reference checkout at %s (set BEPU_REFERENCE_ROOT)" % build_ref.REFERENCE)
    lib = C.CDLL(build_ref.LIB)
    lib.ref_eval_lane.argtypes = [C.c_int32, C.c_int32, FP, C.c_float, FP, FP, FP, C.c_int32]
    lib.ref_covered_types.argtypes = [C.POINTER(C.c_int32), C.c_int32]
    ids = (C.c_int32 * 64)()
    covered = np.array(sorted(ids[:lib.ref_covered_types(ids, 64)]), dtype=np.int32)

    golden = np.load(os.path.join(ROOT, "tests", "golden", "reference_vectors.npz"))
    key = "lane_07_"
    v, a, p = golden[key + "velocities"][0].copy(), golden[key + "impulses"][0].copy(), golden[key + "prestep"][0].copy()
    assert lib.ref_eval_lane(7, 1, _ptr(np.ascontiguousarray(golden[key + "states"][0])), DT_LANE, _ptr(p), _ptr(a), _ptr(v), 1) == 0

    digests, input_digests = lane_digests(lib.ref_eval_lane)
    types = np.array(sorted(input_digests), dtype=np.int32)
    out = {
        "covered_types": covered,
        "lane07_out1_velocities": v,
        "lane_types": types,
        "lane_digests": np.array([[digests[(t, s)] for s in (0, 1, 2)] for t in types.tolist()]),
        "lane_input_digests": np.array([input_digests[t] for t in types.tolist()]),
        "bounds_out": gen.evaluate(gen.load_ref(), *fresh_bounds_inputs(), DT_BOUNDS),
    }
    np.savez_compressed(PATH, **out)
    print("wrote", PATH, {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
