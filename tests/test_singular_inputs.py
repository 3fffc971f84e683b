"""Singular inputs: the fallback jacobians, fallback axes and clamped denominators of the constraint functions, held to the reference.

tests/golden/reference_singular_vectors.npz (tests/golden/make_reference_singular_vectors.py) holds hand-made singular lanes -- coincident
anchors and centres, parallel and antiparallel axes, opposed twist bases, servos at their target, collinear / coplanar / coincident Area and
Volume bodies, contact and body edges -- with the transpiled reference's outputs. On the CPU: the oracle and the CUDA constraint source (compiled
for the host, tests/device_on_host) reproduce every case bit for bit; a coverage build of that source proves that both outcomes of every guard
(every comparison with a non-zero float literal in the device headers, SITES below) run on these inputs; the scalar and the 8-wide oracle agree
on scenes made of the cases. On the GPU: the same scenes, in which every case is one constraint on its own bodies posed exactly in the case's
state (so that substep 0 evaluates the guarded branch on the device), against the oracle -- bit for bit in the strict build, through the
full-switch, the contact-only and the deep stage kernels, and within the joint tolerances in the fast build."""
import ctypes as C
import gzip
import json
import os
import re
import subprocess
import sys
import textwrap

import numpy as np
import pytest

from bepuphysics2_b200 import native, scenes
from bepuphysics2_b200.native import EXEC_GRAPH, EXEC_STREAM
from oracle import binding as ob
from tests import test_topology as topo
from tests import util
from tests.test_deep_batches import DEEP_BUNDLES
from tests.test_device_source_on_host import CSRC, LANES, _ptr, compile_device_on_host, device_on_host  # noqa: F401 (device_on_host: fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "reference_singular_vectors.npz")
DT_LANE = 1.0 / 240.0  # the generator's dt
DT = 1.0 / 60.0
HEADERS = ("bepu_device_math.cuh", "bepu_contacts.cuh", "bepu_joints.cuh", "bepu_joints_more.cuh", "bepu_integration.cuh")
CONTACT_TYPES = (0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 15, 16, 17)
ONE_BODY_CONTACTS, TWO_BODY_CONTACTS = (0, 1, 2, 3, 8, 9, 10), (4, 5, 6, 7, 15, 16, 17)
shim = topo.shim


@pytest.fixture(scope="module")
def golden():
    g = np.load(GOLDEN)
    return {k: g[k] for k in g.files}


def _cases(g):
    return range(g["type"].size)


def _eval(fn, g, i, stage, stride, takes_stride):
    """One stage of case i through fn(type, stage, states, dt, prestep, impulses, velocities[, stride]); rows laid out with `stride`."""
    type_id = int(g["type"][i])
    _, prestep_rows, impulse_rows = ob.type_info(type_id)
    p = np.zeros(prestep_rows * stride, dtype=np.float32)
    p[::stride] = g["prestep"][i][:prestep_rows]
    a = np.zeros(impulse_rows * stride, dtype=np.float32)
    a[::stride] = g["impulses"][i][:impulse_rows]
    v = g["velocities"][i].copy()
    states = np.ascontiguousarray(g["states"][i])
    args = [type_id, stage, _ptr(states), DT_LANE, _ptr(p), _ptr(a), _ptr(v)]
    assert (fn(*args, stride) if takes_stride else fn(*args)) == 0
    return v, a[::stride], p[::stride]


def _check_against_golden(fn, g, stride, takes_stride):
    checked = 0
    for i in _cases(g):
        type_id = int(g["type"][i])
        _, prestep_rows, impulse_rows = ob.type_info(type_id)
        for stage in range(int(g["stages"][i])):
            v, a, p = _eval(fn, g, i, stage, stride, takes_stride)
            what = "case %d (type %d, %s) stage %d" % (i, type_id, g["label"][i], stage)
            assert np.array_equal(v.view(np.uint32), g["out_velocities"][i, stage].view(np.uint32)), what + ": velocities"
            assert np.array_equal(a.view(np.uint32), g["out_impulses"][i, stage, :impulse_rows].view(np.uint32)), what + ": accumulated impulses"
            assert np.array_equal(p.view(np.uint32), g["out_prestep"][i, stage, :prestep_rows].view(np.uint32)), what + ": prestep"
            checked += 1
    return checked


def test_golden_cases_cover_every_type_and_both_states(golden):
    g = golden
    assert set(g["type"].tolist()) >= set(CONTACT_TYPES) | {22, 23, 24, 25, 26, 27, 28, 29, 30, 31, 32, 33, 34, 35, 36, 37, 38, 42, 43, 44, 45, 46, 47, 52, 53, 55}
    rest = ~g["velocities"].any(axis=(1, 2)) & ~g["impulses"].any(axis=1)
    assert rest.sum() * 2 == g["type"].size and (g["impulses"][~rest].any(axis=1)).all(), "every case from rest and moving with non-zero impulses"
    for k in ("out_velocities", "out_impulses", "out_prestep"):
        assert np.isfinite(g[k]).all(), k
    assert (g["stages"] == np.where(np.isin(g["type"], CONTACT_TYPES), 3, 2)).all()


def test_oracle_reproduces_the_reference_on_singular_inputs(libs, golden):
    orc = ob.load()
    fp = C.POINTER(C.c_float)
    orc.oracle_eval_lane.argtypes = [C.c_int32, C.c_int32, fp, C.c_float, fp, fp, fp, C.c_int32]
    assert _check_against_golden(orc.oracle_eval_lane, golden, LANES, True) > 1000


def test_device_source_reproduces_the_reference_on_singular_inputs(libs, golden, device_on_host):
    dev, _ = device_on_host
    assert _check_against_golden(dev.device_on_host_eval_lane, golden, LANES, False) > 1000


# ---- both outcomes of every guard ---------------------------------------------------------------------------------------------------------------
#
# A site: the header, a substring of its text that occurs once there (it may span lines), the text of the threshold on the guard's line, the cases
# (generator site names) meant to reach it and the type ids that reach it. check "branches": gcov records branches on the guard's line (one pair
# per inlined copy: per type and stage), and every one must be taken. "consumer": the comparison only sets a bool; `consumer` names the line that
# branches on it. "predicate": the branch lives inside fmax_ps (whose copies gcov cannot tell apart), so float64 predicates over the inputs show
# that some case of the site lies on each side. "integration": reached through device_on_host_eval_integration op 0 with w = 0 and w != 0.

def _area_terms(x):
    """float64 AreaConstraint jacobians (AreaConstraint.cs:L93-138) of body positions x: negated A, B, C."""
    ab, ac = x[1] - x[0], x[2] - x[0]
    n = np.cross(ab, ac)
    length = np.linalg.norm(n)
    n = n / length if length > 1e-10 else n * 0.0
    jb, jc = np.cross(ac, n), np.cross(n, ab)
    return [jb + jc, jb, jc]


def _volume_terms(x):
    """float64 VolumeConstraint jacobians (VolumeConstraint.cs:L96-123): negated A, B, C, D."""
    ab, ac, ad = x[1] - x[0], x[2] - x[0], x[3] - x[0]
    jb, jc, jd = np.cross(ac, ad), np.cross(ad, ab), np.cross(ab, ac)
    return [jb + jc + jd, jb, jc, jd]


def _jacobian_length_squared(terms):
    return lambda g, i: sum(float(j @ j) for j in terms(g["states"][i, :, 0:3].astype(np.float64)))


def _inverse_effective_mass(terms):
    def f(g, i):
        js = terms(g["states"][i, :, 0:3].astype(np.float64))
        squared = max(1e-14, sum(float(j @ j) for j in js))
        return sum(float(j @ j) * float(g["states"][i, k, 13]) for k, j in enumerate(js)) / squared
    return f


def _at_rest(g, i):
    return not g["velocities"][i].any() and not g["impulses"][i].any()


def _friction_site(types):
    # from rest the tangent csv and accumulated impulse are zero, so the friction magnitude is exactly 0 < 1e-16; moving, the accumulated tangent
    # impulse is >= 0.125 per axis and the csi of one Solve cannot cancel it exactly on these inputs (the Solve output shows a non-zero tangent)
    def tangent_out(g, i):
        n = ob.type_info(int(g["type"][i]))[2]
        rows = [r for r in range(n) if (int(g["type"][i]) < 8 and r < 2) or (int(g["type"][i]) >= 8 and r % 3 != 2)]
        return np.abs(g["out_impulses"][i, 1, rows]).max()
    return dict(check="predicate", cases={"friction_clamp"}, types=types,
                fallback=lambda g, i: _at_rest(g, i), normal=lambda g, i: not _at_rest(g, i) and tangent_out(g, i) > 1e-16)


SITES = {
    "quaternion_between_antiparallel": dict(file="bepu_device_math.cuh", text="bool useNormalCase = d > -0.999999f;", threshold="-0.999999f", check="consumer",
                                            consumer="q.x = useNormalCase ? c.x : (xIsSmallest ? 0.0f : (yIsSmaller ? -v1.z : -v1.y));", cases={"twist_opposed_z"}, types={26, 27}),
    "axis_angle_fallback": dict(file="bepu_device_math.cuh", text="bool useFallback = axisLength < 1e-14f;", threshold="1e-14f", check="consumer",
                                consumer="axis.x = useFallback ? 1.0f : axis.x;", cases={"axis_angle_fallback"}, types={29, 31, 42}),
    "friction_two_body": dict(file="bepu_contacts.cuh", text="accumulated = accumulated + csi;\n    float magnitude = length(accumulated);\n    float scl = fmin_ps(1.0f, maximumImpulse / fmax_ps(1e-16f, magnitude));",
                              threshold="1e-16f", **_friction_site(set(TWO_BODY_CONTACTS))),
    "friction_one_body": dict(file="bepu_contacts.cuh", text="accumulated = accumulated - negativeCSI;\n    float magnitude = length(accumulated);\n    float scl = fmin_ps(1.0f, maximumImpulse / fmax_ps(1e-16f, magnitude));",
                              threshold="1e-16f", **_friction_site(set(ONE_BODY_CONTACTS))),
    "servo_target_speed_3": dict(file="bepu_joints.cuh", text="scl = targetSpeed < 1e-10f ? 1.0f : scl;", threshold="1e-10f", check="branches",
                                 cases={"axis_angle_fallback", "servo_error_length"}, types={29, 42, 44, 53}),
    "servo_impulse_magnitude_3": dict(file="bepu_joints.cuh", text="float impulseScale = fabsf(magnitude) < 1e-10f ? 1.0f : fmin_ps(maximumImpulse / magnitude, 1.0f);\n    accumulated = accumulated * impulseScale;",
                                      threshold="1e-10f", check="branches", cases={"axis_angle_fallback", "servo_error_length", "servo_impulse_magnitude"}, types={29, 30, 42, 43, 44, 45, 52, 53}),
    "swing_limit_fallback": dict(file="bepu_joints.cuh", text="return dot(j, j) < 1e-7f ? fallback : j;", threshold="1e-7f", check="branches", cases={"swing_limit_fallback"}, types={25}),
    "twist_jacobian_full": dict(file="bepu_joints.cuh", text="return len < 1e-10f ? basisA.z : j;", threshold="1e-10f", check="branches", cases={"twist_opposed_z"}, types={26, 27}),
    "twist_jacobian_only": dict(file="bepu_joints.cuh", text="return len < 1e-10f ? basisAZ : j;", threshold="1e-10f", check="branches", cases={"twist_opposed_z"}, types={26, 27}),
    "hinge_on_plane_x": dict(file="bepu_joints.cuh", text="onPlaneX = xLength < 1e-7f ? hingeAxisA : onPlaneX;", threshold="1e-7f", check="branches", cases={"hinge_on_plane_x"}, types={23, 47}),
    "hinge_on_plane_y": dict(file="bepu_joints.cuh", text="onPlaneY = yLength < 1e-7f ? hingeAxisA : onPlaneY;", threshold="1e-7f", check="branches", cases={"hinge_on_plane_y"}, types={23, 47}),
    "swivel_hinge_fallback": dict(file="bepu_joints.cuh", text="return length_squared(j) < 1e-3f ? hingeAxis : j;", threshold="1e-3f", check="branches", cases={"swivel_hinge_fallback"}, types={46}),
    "servo_error_length_3": dict(file="bepu_joints_more.cuh", text="errorAxis = errorLength < 1e-10f ? V3{0.0f, 0.0f, 0.0f} : errorAxis;", threshold="1e-10f", check="branches",
                                 cases={"servo_error_length"}, types={44, 53}),
    "servo_error_length_2": dict(file="bepu_joints_more.cuh", text="if (errorLength < 1e-10f) errorAxis = V2{0.0f, 0.0f};", threshold="1e-10f", check="branches",
                                 cases={"servo_error_length_2"}, types={37}),
    "servo_target_speed_2": dict(file="bepu_joints_more.cuh", text="scl = targetSpeed < 1e-10f ? 1.0f : scl;", threshold="1e-10f", check="branches", cases={"servo_error_length_2"}, types={37}),
    "servo_impulse_magnitude_2": dict(file="bepu_joints_more.cuh", text="float impulseScale = fabsf(magnitude) < 1e-10f ? 1.0f : fmin_ps(maximumImpulse / magnitude, 1.0f);\n    accumulated = unclamped * impulseScale;",
                                      threshold="1e-10f", check="branches", cases={"servo_error_length_2"}, types={37}),
    "angular_swivel_hinge_fallback": dict(file="bepu_joints_more.cuh", text="return dot(j, j) < 1e-3f ? fallbackJacobian : j;", threshold="1e-3f", check="branches",
                                          cases={"angular_swivel_hinge_fallback"}, types={24}),
    "twist_motor_fallback": dict(file="bepu_joints_more.cuh", text="return len < 1e-10f ? axisA : j;", threshold="1e-10f", check="branches", cases={"twist_motor_fallback"}, types={28}),
    "distance_servo_coincident": dict(file="bepu_joints_more.cuh", text="f.direction = anchorOffset * (1.0f / f.distance);\n        if (f.distance < 1e-9f)", threshold="1e-9f", check="branches",
                                      cases={"distance_coincident"}, types={33}),
    "distance_limit_coincident": dict(file="bepu_joints_more.cuh", text="f.direction = anchorOffset * (sign / f.distance);\n        if (f.distance < 1e-9f)", threshold="1e-9f", check="branches",
                                      cases={"distance_coincident"}, types={34}),
    "center_distance_warm_start": dict(file="bepu_joints_more.cuh", text="if (lengthSquared < 1e-10f) jacobianA", threshold="1e-10f", check="branches", cases={"center_distance_coincident"}, types={35}),
    "center_distance_solve": dict(file="bepu_joints_more.cuh", text="if (distance < 1e-5f) jacobianA = V3{1.0f, 0.0f, 0.0f};\n        Springiness", threshold="1e-5f", check="branches",
                                  cases={"center_distance_coincident"}, types={35}),
    "center_distance_limit": dict(file="bepu_joints_more.cuh", text="if (distance < 1e-5f) jacobianA = V3{1.0f, 0.0f, 0.0f};\n        useMinimum", threshold="1e-5f", check="branches",
                                  cases={"center_distance_coincident"}, types={55}),
    "area_normal": dict(file="bepu_joints_more.cuh", text="j.normalLength > 1e-10f ?", threshold="1e-10f", check="branches", cases={"area_normal", "area_clamp"}, types={36}),
    "area_jacobian_clamp": dict(file="bepu_joints_more.cuh", text="j.contributionC;\n        jacobianLengthSquared = fmax_ps(1e-14f, jacobianLengthSquared);", threshold="1e-14f", check="predicate",
                                cases={"area_clamp", "area_normal"}, types={36}, value=_jacobian_length_squared(_area_terms)),
    "area_effective_mass_clamp": dict(file="bepu_joints_more.cuh", text="fmax_ps(\n            1e-14f, inverseJacobianLengthSquared", threshold="1e-14f", check="predicate",
                                      cases={"area_clamp", "area_normal"}, types={36}, value=_inverse_effective_mass(_area_terms)),
    "volume_jacobian_clamp": dict(file="bepu_joints_more.cuh", text="j.contributionD;\n        jacobianLengthSquared = fmax_ps(1e-14f, jacobianLengthSquared);", threshold="1e-14f", check="predicate",
                                  cases={"volume_clamp"}, types={32}, value=_jacobian_length_squared(_volume_terms)),
    "volume_effective_mass_clamp": dict(file="bepu_joints_more.cuh", text="float inverseEffectiveMass = fmax_ps(1e-14f, inverseJacobianLengthSquared", threshold="1e-14f", check="predicate",
                                        cases={"volume_clamp"}, types={32}, value=_inverse_effective_mass(_volume_terms)),
    "integrate_orientation_speed": dict(file="bepu_integration.cuh", text="return speed > 1e-15f ? end : start;", threshold="1e-15f", check="integration", cases=set(), types=set()),
}


def _read(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _line_of(name, text, threshold):
    """1-based line of `threshold` inside the one occurrence of `text` in header `name`."""
    src = _read(name)
    assert src.count(text) == 1, "%s: %r occurs %d times" % (name, text, src.count(text))
    start = src.index(text)
    offset = text.index(threshold)
    return src.count("\n", 0, start + offset) + 1


def test_every_float_threshold_of_the_device_headers_is_a_listed_site():
    """Every comparison with a non-zero float literal and every fmax_ps clamp by one in the device headers is a site above, so a guard added later
    cannot go untested. (Comparisons with 0.0f select a sign, not a fallback.)"""
    listed = {(s["file"], _line_of(s["file"], s["text"], s["threshold"])) for s in SITES.values()}
    assert len(listed) == len(SITES)
    literal = r"-?(?:\d+\.\d*|\.\d+|\d+)(?:e-?\d+)?f\b"
    pattern = re.compile(r"(?:[<>]=?\s*(%s))|(?:(%s)\s*[<>]=?(?!>))|(?:fmax_ps\(\s*(%s))" % (literal, literal, literal))
    found = set()
    for name in HEADERS:
        src = _read(name)
        for m in pattern.finditer(src):
            value = next(v for v in m.groups() if v is not None)
            if float(value.rstrip("f")) == 0.0:
                continue
            at = m.start(m.lastindex)
            found.add((name, src.count("\n", 0, at) + 1))
    assert found - listed == set(), "unlisted guards: %s" % sorted(found - listed)
    assert listed - found == set(), "listed sites that are no guard: %s" % sorted(listed - found)


CHILD = textwrap.dedent("""
    import ctypes as C, sys
    import numpy as np
    lib_path, golden, lanes = sys.argv[1], sys.argv[2], int(sys.argv[3])
    lib = C.CDLL(lib_path)
    fp = C.POINTER(C.c_float)
    lib.device_on_host_eval_lane.argtypes = [C.c_int32, C.c_int32, fp, C.c_float, fp, fp, fp]
    lib.device_on_host_type_info.argtypes = [C.c_int32] + [C.POINTER(C.c_int32)] * 4
    lib.device_on_host_eval_integration.argtypes = [C.c_int32, fp, fp]
    ptr = lambda a: a.ctypes.data_as(fp)
    g = np.load(golden)
    bad = []
    for i in range(g["type"].size):
        t = int(g["type"][i])
        info = [C.c_int32() for _ in range(4)]
        assert lib.device_on_host_type_info(t, *[C.byref(x) for x in info]) == 0
        prows, irows = info[1].value, info[2].value
        for stage in range(int(g["stages"][i])):
            p = np.zeros(prows * lanes, np.float32); p[::lanes] = g["prestep"][i][:prows]
            a = np.zeros(irows * lanes, np.float32); a[::lanes] = g["impulses"][i][:irows]
            v = g["velocities"][i].copy()
            s = np.ascontiguousarray(g["states"][i])
            assert lib.device_on_host_eval_lane(t, stage, ptr(s), np.float32(1.0 / 240.0), ptr(p), ptr(a), ptr(v)) == 0
            for got, want in ((v, g["out_velocities"][i, stage]), (a[::lanes], g["out_impulses"][i, stage, :irows]), (p[::lanes], g["out_prestep"][i, stage, :prows])):
                if not np.array_equal(got.view(np.uint32), want.view(np.uint32)):
                    bad.append("case %d (%s) stage %d" % (i, g["label"][i], stage))
    for w in ((0.0, 0.0, 0.0), (0.5, -1.0, 2.0)):  # integrate_orientation: |w| = 0 keeps the orientation, |w| > 0 rotates it
        operands = np.array((0.0, 0.0, 0.0, 1.0) + w + (1.0 / 480.0,), np.float32)
        out = np.zeros(4, np.float32)
        assert lib.device_on_host_eval_integration(0, ptr(operands), ptr(out)) == 0
    if bad:
        sys.exit("the coverage build differs from the reference: " + "; ".join(bad[:10]))
""")


@pytest.fixture(scope="module")
def coverage(tmp_path_factory, golden):
    """gcov's per-line branch counts {(header, line): [taken counts]} of the -O0 --coverage build after evaluating every singular case."""
    d = tmp_path_factory.mktemp("coverage")
    lib = str(d / "libdevice_on_host_cov.so")
    compile_device_on_host(lib, ("-O0", "--coverage"))
    # the counters are written when the process that ran the code exits
    subprocess.run([sys.executable, "-c", CHILD, lib, GOLDEN, str(LANES)], cwd=str(d), check=True)
    gcda = [f for f in os.listdir(d) if f.endswith(".gcda")]
    assert len(gcda) == 1, os.listdir(d)
    subprocess.run(["/usr/bin/gcov", "-b", "-j", gcda[0]], cwd=str(d), check=True, stdout=subprocess.DEVNULL)
    report = [f for f in os.listdir(d) if f.endswith(".gcov.json.gz")]
    assert len(report) == 1, os.listdir(d)
    with gzip.open(str(d / report[0])) as f:
        data = json.load(f)
    branches = {}
    for entry in data["files"]:
        name = os.path.basename(entry["file"])
        if name in HEADERS:
            for line in entry["lines"]:
                branches.setdefault((name, line["line_number"]), []).extend(b["count"] for b in line["branches"])
    return branches


def _site_cases(g, site):
    return [i for i in _cases(g) if str(g["site"][i]) in site["cases"] and int(g["type"][i]) in site["types"]]


def test_both_outcomes_of_every_guard_run_on_the_singular_inputs(golden, coverage):
    g = golden
    failures = []
    for name, site in SITES.items():
        cases = _site_cases(g, site)
        missing = sorted(t for t in site["types"] if not any(int(g["type"][i]) == t for i in cases))
        if missing:
            failures.append("%s: no case for type(s) %s" % (name, missing))
            continue
        if site["check"] in ("branches", "consumer", "integration"):
            line = _line_of(site["file"], site["consumer"], site["consumer"][:8]) if site["check"] == "consumer" else _line_of(site["file"], site["text"], site["threshold"])
            counts = coverage.get((site["file"], line), [])
            if not counts:
                failures.append("%s: gcov records no branch on %s:%d" % (name, site["file"], line))
            elif min(counts) == 0:
                failures.append("%s: %d of %d branch outcomes on %s:%d never taken" % (name, counts.count(0), len(counts), site["file"], line))
        elif site["check"] == "predicate":
            if "value" in site:
                values = [site["value"](g, i) for i in cases]
                clamped, free = any(v < 1e-14 for v in values), any(v > 1e-14 for v in values)
            else:
                clamped, free = any(site["fallback"](g, i) for i in cases), any(site["normal"](g, i) for i in cases)
            if not (clamped and free):
                failures.append("%s: the cases reach only the %s side" % (name, "clamped" if clamped else "unclamped"))
    assert not failures, "\n".join(failures)


# ---- scenes of the cases: one constraint per case on its own bodies ------------------------------------------------------------------------------

def singular_scene(g, which, replicas=1):
    """(scene, {first body handle: case}) of the cases selected by `which` (a boolean mask), `replicas` times on disjoint bodies. Bodies carry
    the case's pose, local inverse inertia, inverse mass and velocities."""
    bodies, groups, first = [], [], {}
    handle = 0
    for _ in range(replicas):
        for i in np.flatnonzero(which):
            type_id = int(g["type"][i])
            nb = ob.type_info(type_id)[0]
            s, v = g["states"][i, :nb], g["velocities"][i, :nb]
            bodies.append(scenes.make_bodies(s[:, 0:3], orientation=s[:, 3:7], linear=v[:, 0:3], angular=v[:, 3:6], inverse_mass=s[:, 13], inverse_inertia=g["local_inertia"][i, :nb]))
            row = np.arange(handle, handle + nb, dtype=np.int32)[None, :]
            prestep = g["prestep"][i][None, :ob.type_info(type_id)[1]]
            if groups and groups[-1][0] == type_id:
                groups[-1] = (type_id, np.concatenate([groups[-1][1], row]), np.concatenate([groups[-1][2], prestep]))
            else:
                groups.append((type_id, row, prestep))
            first[handle] = i
            handle += nb
    return {"bodies": np.concatenate(bodies), "constraints": groups, "description": "singular cases"}, first


def _no_gravity():
    d = native.IntegratorDesc.default()
    d.gravity[0] = d.gravity[1] = d.gravity[2] = 0.0
    return d


def make_singular_sim(g, scene, first, **kw):
    """A host simulation of the scene with every constraint's accumulated impulses set to its case's (the moving cases start warm)."""
    sim = util.make_sim(scene, integrator=_no_gravity(), **kw)
    for tb in sim.type_batches():
        refs = tb.body_references[:, 0, :] & topo.INDEX_MASK
        for bundle, lane in zip(*np.nonzero(tb.body_references[:, 0, :] >= 0)):
            i = first[int(refs[bundle, lane])]
            tb.accumulated_impulses[bundle, :, lane] = g["impulses"][i][:tb.impulse_rows]
    return sim


def clamped_jacobian(g):
    """Area / Volume lanes whose jacobian length is clamped (coincident or collinear bodies): the clamp makes the effective mass ~1e14 and the
    accumulated impulse ~1e22. From a moving state their bodies leave the finite range within two frames (and x86 and the GPU write different
    NaN payloads), and the fast build's approximate square root is off by ~1e15 in absolute terms there, relatively by ~1e-7."""
    terms = {36: _area_terms, 32: _volume_terms}
    return np.array([int(g["type"][i]) in terms and _jacobian_length_squared(terms[int(g["type"][i])])(g, i) < 1e-14 for i in _cases(g)])


def _scene(g, kind):
    """The cases of one scene: "mixed" every case, "contacts" the contact cases, "deep" the mixed scene replicated until its one batch holds
    DEEP_BUNDLES device bundles, "clamped" the clamped Area / Volume lanes from rest alone, "unclamped" every other case. The clamped lanes from a moving state are in none."""
    contact = np.isin(g["type"], CONTACT_TYPES)
    rest = np.array([_at_rest(g, i) for i in _cases(g)])
    runaway = clamped_jacobian(g) & ~rest
    if kind == "mixed":
        return singular_scene(g, ~runaway)
    if kind == "contacts":
        return singular_scene(g, contact)
    if kind == "clamped":
        return singular_scene(g, clamped_jacobian(g) & rest)
    if kind == "unclamped":
        return singular_scene(g, ~clamped_jacobian(g))
    counts = [int(((g["type"] == t) & ~runaway).sum()) for t in set(g["type"].tolist())]
    replicas = 1
    while sum(-(-replicas * n // LANES) for n in counts) < DEEP_BUNDLES:  # device bundles are LANES wide
        replicas += 1
    return singular_scene(g, ~runaway, replicas=replicas)


KW = dict(substeps=2, velocity_iterations=2)


@pytest.fixture(scope="module")
def scenes_of_cases(golden):
    return {kind: _scene(golden, kind) for kind in ("mixed", "contacts", "deep", "clamped", "unclamped")}


def test_scenes_reach_the_full_the_contact_only_and_the_deep_kernels(libs, shim, golden, scenes_of_cases):
    """The mixed scene runs in full-switch launches, the contact-only scene in contact-only launches, the replicated one in deep launches."""
    for kind, (scene, first) in scenes_of_cases.items():
        if kind in ("clamped", "unclamped"):
            continue
        sim = make_singular_sim(golden, scene, first, **KW)
        assert sim.batch_count == 1, kind  # every constraint has bodies of its own
        p = topo.plan(shim, topo.sim_sources(sim), sim.bundle_width, sim.fallback_batch_threshold, sim.batch_count, sim.body_count)
        ops, _ = p.program(sim.velocity_iterations, len(sim.constrained_kinematics), True, False, sim.body_count)
        stages = ops[ops[:, 0] <= topo.SOLVE]
        for ext, mode, profile in topo.LAUNCH_CONTEXTS:
            kernel = topo.resolve(shim, stages, ext, mode, profile)[:, 0]
            want = {"mixed": topo.KERNEL_FULL, "contacts": topo.KERNEL_CONTACTS, "deep": topo.KERNEL_DEEP}[kind]
            assert (kernel == want).all(), (kind, ext, mode, profile, kernel.tolist())
        count = int(p.batches[0, 1])
        assert (count >= DEEP_BUNDLES) == (kind == "deep"), (kind, count)


@pytest.mark.parametrize("kind", ["mixed", "contacts", "clamped"])
def test_scalar_and_simd_oracle_agree_on_singular_scenes(libs, golden, scenes_of_cases, kind):
    scene, first = scenes_of_cases[kind]
    a = util.run_oracle(make_singular_sim(golden, scene, first, **KW), DT, frames=2, simd=False)
    b = util.run_oracle(make_singular_sim(golden, scene, first, **KW), DT, frames=2, simd=True)
    util.compare(a, b, exact=True)


# ---- GPU -----------------------------------------------------------------------------------------------------------------------------------------

def _gpu_parity(g, scene, first, exact, mode=EXEC_GRAPH, frames=1, **kw):
    ref = util.run_oracle(make_singular_sim(g, scene, first, **kw), DT, frames=frames)
    got = util.run_gpu(make_singular_sim(g, scene, first, **kw), DT, frames=frames, strict=exact, mode=mode)
    return ref, got


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [EXEC_GRAPH, EXEC_STREAM])
@pytest.mark.parametrize("kind", ["mixed", "contacts", "deep", "clamped"])
def test_strict_build_matches_the_oracle_bit_for_bit_on_singular_scenes(libs, golden, scenes_of_cases, kind, mode):
    scene, first = scenes_of_cases[kind]
    ref, got = _gpu_parity(golden, scene, first, True, mode=mode, frames=1 if kind == "deep" else 2, **KW)
    util.compare(ref, got, exact=True)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["unclamped", "contacts", "clamped"])
def test_fast_build_on_singular_scenes(libs, golden, scenes_of_cases, kind):
    """One substep of one iteration: both builds see the exactly singular input and take the same side of every guard, so the joint tolerances of
    test_joint_zoo_fast_build_within_tolerance hold -- except at the clamped Area / Volume lanes, where the same side is taken but the clamp
    magnifies the approximate square root to an absolute error of ~1e15 on impulses of ~1e22: those are held to the relative bound alone. Over
    2 x 2 and several frames the geometry is only near-singular and a threshold may flip between the builds: finite outputs only."""
    scene, first = scenes_of_cases[kind]
    ref, got = _gpu_parity(golden, scene, first, False, substeps=1, velocity_iterations=1)
    util.compare(ref, got, exact=False, rel_rms=1e-3, max_abs=np.inf if kind == "clamped" else 5e-2)
    _, got = _gpu_parity(golden, scene, first, False, frames=3, **KW)
    assert np.isfinite(got["bodies"][:, util.MEANINGFUL]).all()
    for tb in got["type_batches"]:
        assert np.isfinite(np.where(tb["valid"][:, None, :], tb["impulses"], 0)).all() and np.isfinite(np.where(tb["valid"][:, None, :], tb["prestep"], 0)).all(), tb["key"]
