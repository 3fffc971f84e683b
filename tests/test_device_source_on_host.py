"""Holds the CUDA constraint SOURCE to the oracle without a GPU. tests/device_on_host/device_on_host.cpp compiles the device headers
(csrc/bepu_device_math.cuh, bepu_contacts.cuh, bepu_joints.cuh, bepu_joints_more.cuh) for the host with g++ -ffp-contract=off -- the arithmetic
of the strict -fmad=false build -- and evaluates one constraint lane of one stage per call; the oracle does the same through oracle_eval_lane.
For every one of the 44 types and each of WarmStart / Solve / IncrementallyUpdateForSubstep the outputs (body velocities, accumulated impulses,
prestep) must agree BIT FOR BIT on prestep data taken from the seeded scene generators, random body states, velocities and impulses.
The GPU parity tests remain the check of the binary that ships (kernels, gather/scatter, integration, scheduling); this one lets the constraint
math be changed and re-verified on a machine without a GPU. TEST INFRASTRUCTURE: the product never loads either library."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from bepuphysics2_b200 import scenes
from oracle import binding as ob
from tests import util

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.join(ROOT, "tests", "device_on_host")
CSRC = os.path.join(ROOT, "bepuphysics2_b200", "csrc")
LANES = 32
DT = 1.0 / 240.0  # a substep of the 8 x 2 configuration at 1/30 s


def compile_device_on_host(lib, optimisation=("-O2",)):
    """The build recipe of the harness: g++ with the arithmetic of the strict build; `optimisation` replaces -O2 (the coverage build)."""
    src = os.path.join(HERE, "device_on_host.cpp")
    subprocess.check_call(["/usr/bin/g++"] + list(optimisation) + ["-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-march=x86-64-v3", "-Wall", "-Wno-unused-function", "-Wno-unknown-pragmas", "-pthread",
                                                                   "-I", os.path.join(HERE, "stubs"), "-I", HERE, "-I", CSRC, "-shared", "-fPIC", "-o", lib, src])


@pytest.fixture(scope="module")
def device_on_host():
    lib = os.path.join(HERE, "libdevice_on_host.so")
    srcs = [os.path.join(HERE, "device_on_host.cpp"), os.path.join(HERE, "stubs", "cuda_runtime.h")] + [os.path.join(CSRC, f) for f in ("bepu_device_math.cuh", "bepu_contacts.cuh", "bepu_joints.cuh", "bepu_joints_more.cuh", "bepu_integration.cuh", "bepu_bounds_math.cuh", "bepu_redistribute.cuh")]
    if not os.path.exists(lib) or any(os.path.getmtime(s) > os.path.getmtime(lib) for s in srcs):
        compile_device_on_host(lib)
    dev = C.CDLL(lib)
    fp = C.POINTER(C.c_float)
    dev.device_on_host_eval_lane.argtypes = [C.c_int32, C.c_int32, fp, C.c_float, fp, fp, fp]
    dev.device_on_host_type_info.argtypes = [C.c_int32] + [C.POINTER(C.c_int32)] * 4
    orc = ob.load()
    orc.oracle_eval_lane.argtypes = [C.c_int32, C.c_int32, fp, C.c_float, fp, fp, fp, C.c_int32]
    dev.device_on_host_eval_integration.argtypes = [C.c_int32, fp, fp]
    orc.oracle_eval_integration.argtypes = [C.c_int32, fp, fp]
    return dev, orc


def _ptr(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def _random_states(rng, bodies):
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


def _prestep_samples():
    """type id -> float32[samples, prestep rows] of valid prestep data, from the same generators the GPU tests and the bench use."""
    samples = {}
    for scene in (scenes.shape_pile(1500, seed=21, nonconvex_fraction=0.5), scenes.joint_zoo(600, per_type=24, seed=21), scenes.ragdolls(6, seed=21), scenes.ragdolls(6, seed=22, motor="servo")):
        for type_id, _, prestep in scene["constraints"]:
            samples.setdefault(int(type_id), []).append(np.asarray(prestep, dtype=np.float32)[:24])
    return {k: np.concatenate(v)[:32] for k, v in samples.items()}


def test_device_constraint_source_matches_the_oracle_bit_for_bit(libs, device_on_host):
    dev, orc = device_on_host
    samples = _prestep_samples()
    supported = sorted(t for t in range(64) if ob.type_info(t) is not None)
    assert sorted(samples) == supported, "the scene generators cover every registered type"
    rng = np.random.default_rng(7)
    checked = 0
    for type_id in supported:
        bodies, prestep_rows, impulse_rows = ob.type_info(type_id)
        info = [C.c_int32() for _ in range(4)]
        assert dev.device_on_host_type_info(type_id, *[C.byref(i) for i in info]) == 0
        assert (info[0].value, info[1].value, info[2].value) == (bodies, prestep_rows, impulse_rows)
        for prestep in samples[type_id]:
            assert prestep.shape == (prestep_rows,)
            states = _random_states(rng, bodies)
            velocities = rng.normal(0, 1.5, (bodies, 6)).astype(np.float32)
            impulses = np.abs(rng.normal(0, 0.2, impulse_rows)).astype(np.float32)
            for stage in (0, 1, 2):
                if stage == 2 and not info[3].value:
                    continue
                # device layout: row r of the lane at [r * 32]; the oracle reads the same buffers with that row stride
                p_dev = np.zeros(prestep_rows * LANES, dtype=np.float32)
                p_dev[::LANES] = prestep
                a_dev = np.zeros(impulse_rows * LANES, dtype=np.float32)
                a_dev[::LANES] = impulses
                v_dev = velocities.copy()
                p_orc, a_orc, v_orc = p_dev.copy(), a_dev.copy(), v_dev.copy()
                assert dev.device_on_host_eval_lane(type_id, stage, _ptr(states), DT, _ptr(p_dev), _ptr(a_dev), _ptr(v_dev)) == 0
                assert orc.oracle_eval_lane(type_id, stage, _ptr(states), DT, _ptr(p_orc), _ptr(a_orc), _ptr(v_orc), LANES) == 0
                what = "type %d stage %d" % (type_id, stage)
                assert np.isfinite(v_orc).all() and np.isfinite(a_orc).all(), what
                assert np.array_equal(v_dev.view(np.uint32), v_orc.view(np.uint32)), what + ": velocities"
                assert np.array_equal(a_dev.view(np.uint32), a_orc.view(np.uint32)), what + ": accumulated impulses"
                assert np.array_equal(p_dev.view(np.uint32), p_orc.view(np.uint32)), what + ": prestep"
                if stage < 2:
                    assert not np.array_equal(v_dev, velocities) or not impulses.any(), what + ": the stage did something"
                checked += 1
    assert checked > 44 * 2 * 16


def test_device_integration_source_matches_the_oracle_bit_for_bit(libs, device_on_host):
    """csrc/bepu_integration.cuh (orientation integration through the custom sin / cos, inertia rotation, both momentum-conserving angular
    updates, the velocity callback, the optional per-body acceleration and point-gravity terms) against the oracle's restatement of
    PoseIntegrator.cs:L146-253, DemoCallbacks.cs, PerBodyGravityDemo.cs and PlanetDemo.cs, function by function."""
    dev, orc = device_on_host
    rng = np.random.default_rng(11)

    def unit_q():
        q = rng.normal(0, 1, 4)
        return q / np.linalg.norm(q)

    def spd():
        r = np.linalg.qr(rng.normal(0, 1, (3, 3)))[0]
        m = r @ np.diag(rng.uniform(0.3, 5.0, 3)) @ r.T
        return np.array([m[0, 0], m[1, 0], m[1, 1], m[2, 0], m[2, 1], m[2, 2]])

    for trial in range(400):
        w = rng.normal(0, 1, 3) * 10.0 ** rng.uniform(-3, 1.5)
        if trial % 50 == 0:
            w = w * 0.0  # |w| <= 1e-15: the identity branch
        q, local = unit_q(), spd()
        world = spd()
        cases = {
            0: np.r_[q, w, rng.choice([1, -1]) * 0.5 / rng.choice([60.0, 240.0, 480.0])],
            1: np.r_[local, q],
            2: np.r_[q, local, world, w],
            3: np.r_[q, local, w, 1.0 / rng.choice([60.0, 240.0])],
            4: np.r_[rng.normal(0, 3, 6), 0.0, -10.0 / 240.0, 0.0, 0.97 ** (1 / 240.0), 0.97 ** (1 / 240.0)],
        }
        for op, operands in cases.items():
            operands = np.ascontiguousarray(operands, dtype=np.float32)
            a, b = np.zeros(6, dtype=np.float32), np.zeros(6, dtype=np.float32)
            assert dev.device_on_host_eval_integration(op, _ptr(operands), _ptr(a)) == 0
            assert orc.oracle_eval_integration(op, _ptr(operands), _ptr(b)) == 0
            assert np.isfinite(b).all()
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), "integration op %d, trial %d: %s vs %s" % (op, trial, a, b)

    # op 5, the optional terms: neither, point gravity alone and both; positions and center close together (|offset| <= 1 clamps) and far apart
    rng = np.random.default_rng(17)
    for trial in range(4000):
        operands = np.zeros(22, dtype=np.float32)
        operands[0:12] = rng.normal(0, 5, size=12)
        operands[12] = rng.uniform(1e-3, 0.05)
        operands[13:19] = rng.normal(0, 3 if trial % 2 else 50, size=6)
        operands[19] = rng.uniform(-100, 100)
        operands[20], operands[21] = (trial >> 1) & 1, 1 if trial % 4 != 1 else 0
        a, b = np.zeros(6, dtype=np.float32), np.zeros(6, dtype=np.float32)
        assert dev.device_on_host_eval_integration(5, _ptr(operands), _ptr(a)) == 0
        assert orc.oracle_eval_integration(5, _ptr(operands), _ptr(b)) == 0
        assert np.isfinite(b).all()
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), "integration op 5, trial %d: %s -> %s vs %s" % (trial, operands, a, b)


def test_bounds_source_reproduces_the_reference_vectors_bit_for_bit(device_on_host):
    """csrc/bepu_bounds_math.cuh (the arithmetic of bepucuda_predict_bounding_boxes) compiled for the host against the known-answer vectors generated
    from the reference's own C# text (tests/golden/reference_bounds_vectors.npz): the CUDA source of f4 is pinned to the reference without a GPU."""
    dev, _ = device_on_host
    fp = C.POINTER(C.c_float)
    dev.device_on_host_convex_bounds.argtypes = [C.c_int32, fp, fp, C.c_int32, fp, fp, fp, fp, C.c_float, fp]
    golden = np.load(os.path.join(ROOT, "tests", "golden", "reference_bounds_vectors.npz"))
    checked = 0
    for k in (0, 1):
        types, dims, margins, allow, q, pos, lin, ang = (np.ascontiguousarray(golden["set%d_%s" % (k, n)]) for n in ("types", "dims", "margins", "allow", "q", "pos", "lin", "ang"))
        dt, want = float(golden["set%d_dt" % k]), golden["set%d_out" % k]
        for i in range(types.shape[0]):
            out = np.zeros(7, dtype=np.float32)
            assert dev.device_on_host_convex_bounds(int(types[i]), _ptr(dims[i]), _ptr(margins[i]), int(allow[i]), _ptr(q[i]), _ptr(pos[i]), _ptr(lin[i]), _ptr(ang[i]), dt, _ptr(out)) == 0
            assert np.array_equal(out.view(np.uint32), want[i].view(np.uint32)), "set %d sample %d (shape type %d)" % (k, i, types[i])
            checked += 1
    assert checked == 96


def _redistribute_case_ids(n):
    """Every id-equality pattern of n old and n new feature ids: (old, new) drawn from an alphabet of n + 1 symbols, (n + 1)^(2n) cases. The symbols
    are the int32 edges and negative ids, so that the comparison is held at the values where a signed / unsigned mix-up would show."""
    alphabet = np.array([np.iinfo(np.int32).min, -1, 0, np.iinfo(np.int32).max, -7][:n + 1], dtype=np.int32)
    k = n + 1
    digits = (np.arange(k ** (2 * n), dtype=np.int64)[:, None] // (k ** np.arange(2 * n, dtype=np.int64))[None, :]) % k
    ids = alphabet[digits]
    return np.ascontiguousarray(ids[:, :n]), np.ascontiguousarray(ids[:, n:])


def _redistribute_float64(old_ids, old_imp, new_ids):
    """RedistributeImpulses restated in float64 over many constraints at once: (new impulses where matched, NaN where unmatched; the float64
    remainder per unmatched contact, NaN when nothing is unmatched; the float64 remainder)."""
    cases, n = old_ids.shape
    remaining = old_imp.astype(np.float64)
    new = np.full((cases, n), np.nan)
    rows = np.arange(cases)
    for i in range(n):
        eq = old_ids == new_ids[:, i:i + 1]
        matched = eq.any(axis=1)
        j = np.argmax(eq, axis=1)  # the first old contact with the id
        new[matched, i] = remaining[rows[matched], j[matched]]
        remaining[rows[matched], j[matched]] = 0.0
    unmatched = np.isnan(new).sum(axis=1)
    remainder = remaining.sum(axis=1)
    with np.errstate(invalid="ignore", divide="ignore"):
        share = np.where(unmatched > 0, remainder / np.maximum(unmatched, 1), np.nan)
    return new, share, remainder


def test_redistribution_source_matches_the_oracle_on_every_id_pattern(libs, device_on_host):
    """csrc/bepu_redistribute.cuh (the per-constraint body of redistribute_impulses_kernel) against oracle_update_contact_impulses bit for bit, for
    every id-equality pattern at n = 1-4 contacts (duplicates in old, in new and in both, nothing matched, all matched and permuted), with impulses
    of 0, subnormals, ordinary values and values near FLT_MAX (remainders that overflow to inf). Then against float64: a matched contact carries
    its old impulse exactly (0 included: it stays matched), an unmatched one the remainder / unmatched count to within fp32 rounding."""
    dev, orc = device_on_host
    i32p = C.POINTER(C.c_int32)
    for lib, name in ((dev, "device_on_host_update_contact_impulses"), (orc, "oracle_update_contact_impulses")):
        getattr(lib, name).argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    fmax = np.finfo(np.float32).max
    pool = np.array([0.0, 0.0, 1e-45, 3e-39, 1.1754942e-38, 0.25, 1.5, 7.0, 1234.5, fmax * 0.3, fmax * 0.6, fmax], dtype=np.float32)
    rng = np.random.default_rng(5)
    checked = 0
    for n in (1, 2, 3, 4):
        old_ids, new_ids = _redistribute_case_ids(n)
        cases = old_ids.shape[0]
        assert cases == (n + 1) ** (2 * n)
        # the type ids with n contacts: convex one- and two-body, nonconvex (2-4 contacts) one- and two-body
        types = [n - 1, n + 3] + ([n + 6, n + 13] if n >= 2 else [])
        for trial, type_id in enumerate(types):
            bodies, _, impulse_rows = ob.type_info(type_id)
            W = (1, 8, 16, 4)[trial]
            bundles = (cases + W - 1) // W
            old_imp = pool[rng.integers(0, pool.size, size=(cases, n))]
            if trial == 0:
                old_imp[:] = pool[rng.integers(0, 6, size=(cases, n))]  # zeros, subnormals and small values only: no overflow anywhere
            else:
                old_imp[::3] = pool[rng.integers(pool.size - 3, pool.size, size=old_imp[::3].shape)]  # near FLT_MAX only: remainders overflow
            acc = rng.normal(0, 1, size=(bundles, impulse_rows, W)).astype(np.float32)  # tangent / twist rows: must come out untouched
            penetration = [2 + i for i in range(n)] if type_id < 8 else [3 * i + 2 for i in range(n)]
            c = np.arange(cases)
            for i, r in enumerate(penetration):
                acc[c // W, r, c % W] = old_imp[:, i]
            a_dev, a_orc = acc.copy(), acc.copy()
            assert dev.device_on_host_update_contact_impulses(type_id, cases, W, a_dev.ctypes.data, old_ids.ctypes.data, new_ids.ctypes.data) == 0
            assert orc.oracle_update_contact_impulses(type_id, cases, W, a_orc.ctypes.data, old_ids.ctypes.data, new_ids.ctypes.data) == 0
            what = "n = %d, type %d, W = %d" % (n, type_id, W)
            assert np.array_equal(a_dev.view(np.uint32), a_orc.view(np.uint32)), what + ": device source differs from the oracle"
            others = [r for r in range(impulse_rows) if r not in penetration]
            assert np.array_equal(a_dev[:, others, :].view(np.uint32), acc[:, others, :].view(np.uint32)), what + ": a friction / twist row changed"
            out = np.stack([a_dev[c // W, r, c % W] for r in penetration], axis=1)
            new64, share64, remainder64 = _redistribute_float64(old_ids, old_imp, new_ids)
            matched = ~np.isnan(new64)
            assert np.array_equal(out[matched].astype(np.float64), new64[matched]), what + ": a matched contact did not carry its old impulse exactly"
            unmatched = ~matched
            share = np.broadcast_to(share64[:, None], out.shape)[unmatched]
            got = out[unmatched].astype(np.float64)
            finite = np.isfinite(got)
            # n fp32 additions and one division, all of non-negative values: relative error <= (n + 1) 2^-24, plus n subnormal quanta
            tol = (n + 1) * 2.0 ** -24 * share[finite] + n * 2.0 ** -149
            assert (np.abs(got[finite] - share[finite]) <= tol).all(), what + ": remainder share off by more than fp32 rounding"
            rem = np.broadcast_to(remainder64[:, None], out.shape)[unmatched]
            assert (rem[~finite] > float(fmax) * (1 - 2.0 ** -23)).all(), what + ": an unmatched share overflowed although the remainder fits fp32"
            if trial > 0 and n > 1:
                assert (~finite).any(), what + ": no remainder overflowed to inf"
            if n > 1:  # (a single contact has only four cases)
                assert ((out == 0) & matched).any() and (unmatched.sum(axis=1) == n).any() and (unmatched.sum(axis=1) == 0).any(), what
            checked += cases
    assert checked == sum(((n + 1) ** (2 * n)) * (2 if n == 1 else 4) for n in (1, 2, 3, 4))
