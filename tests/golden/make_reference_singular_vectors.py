"""Generates tests/golden/reference_singular_vectors.npz: what the transpiled reference (oracle/_ref/libbepu_ref.so, built by
oracle/ref_transpile/build_ref.py from a checkout of the reference's C# sources) computes on hand-made SINGULAR constraint lanes, the inputs on
which the constraint functions leave their generic path for a fallback jacobian or axis, or clamp a denominator:

  * coincident anchors or centres (Distance*, CenterDistance*, BallSocketServo, OneBodyLinearServo, PointOnLineServo);
  * parallel and antiparallel axes (SwingLimit, AngularSwivelHinge, SwivelHinge, TwistMotor), hinge axes on a jacobian axis (Hinge, AngularHinge);
  * twist bases whose Z axes oppose each other (TwistServo, TwistLimit), along each world axis and along a direction whose |x| is smallest, so that
    every sub-branch of the antiparallel case of QuaternionWide.GetQuaternionBetweenNormalizedVectors runs (ties of |v1.x|, |v1.y|, |v1.z| included);
  * servos already at their target, and servos with zero speed and force (every servo and one-body servo form), motors at rest;
  * collinear and coincident Area bodies, coplanar, collinear and coincident Volume bodies;
  * contact edges: friction 0, depth exactly 0, MaximumRecoveryVelocity 0, all contact offsets equal, nonconvex manifolds with identical normals;
  * body edges on two-body types: a rotation-locked dynamic body (zero inverse inertia, non-zero inverse mass) and a kinematic partner.

Orientations are the identity or exactly representable axis-permuting quaternions (components 0, +-0.5, +-1), so the world inverse inertia equals
the rotated local one bit for bit and a singularity is exact rather than merely close. Every case runs from rest (zero velocities and accumulated
impulses) and from a moving state with non-zero impulses. A case is one lane; `site` names the guard it targets (see SITES in
tests/test_singular_inputs.py), "" for the contact and body edges that target no guard of their own.

Every stored output is finite. A body variant on which the reference itself yields inf or NaN is user error in bepuphysics2 and is left out: an
angular-only joint between a rotation-locked body and a kinematic one has no angular effective mass, and a linear one between a kinematic body and
another kinematic or locked body along a locked axis none either. NaN payloads differ between x86 and the GPU and cannot be compared bit for bit.

Arrays (N cases, bodies padded to 4, prestep rows to 35, impulse rows to 12, stages 0 WarmStart, 1 Solve, 2 IncrementallyUpdateForSubstep; stage 2
is evaluated for the contact types only, `stages` says how many stages a case has):
  type, site, label, stages, states [N, 4, 14] (lane body states: position, orientation xyzw, world inverse inertia, inverse mass),
  local_inertia [N, 4, 6], velocities [N, 4, 6], impulses [N, 12], prestep [N, 35], out_velocities [N, 3, 4, 6], out_impulses [N, 3, 12],
  out_prestep [N, 3, 35].

    BEPU_REFERENCE_ROOT=<reference checkout> python tests/golden/make_reference_singular_vectors.py
"""
import ctypes as C
import itertools
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
for p in (ROOT, os.path.join(ROOT, "oracle", "ref_transpile")):
    if p not in sys.path:
        sys.path.insert(0, p)

FP = C.POINTER(C.c_float)
DT = 1.0 / 240.0
PATH = os.path.join(ROOT, "tests", "golden", "reference_singular_vectors.npz")
MAX_BODIES, MAX_PRESTEP, MAX_IMPULSES = 4, 35, 12
CONTACT_TYPES = (0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 15, 16, 17)
FMAX = float(np.finfo(np.float32).max)
SPRING = (30.0 * 6.283185307179586477, 2.0)  # SpringSettings(30, 1)
SERVO = (2.0, 0.5, 100.0)  # MaximumSpeed, BaseSpeed, MaximumForce
SERVO_DEFAULT = (FMAX, 0.0, FMAX)  # ServoSettings.Default
SERVO_ZERO = (0.0, 0.0, 0.0)
MOTOR = (100.0, 1.0)  # MaximumForce, Damping
INERTIA = (1.0, 0.5, 2.0)  # diagonal local inverse inertia of an ordinary dynamic body


def layouts():
    with open(os.path.join(ROOT, "tests", "golden", "type_layouts.json")) as f:
        return {int(k): v for k, v in json.load(f)["types"].items()}


# ---- exact rotations ----------------------------------------------------------------------------------------------------------------------------

def matrix(q):
    x, y, z, w = (float(c) for c in q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


IDENTITY = (0.0, 0.0, 0.0, 1.0)
PERMUTE = (0.5, 0.5, 0.5, 0.5)  # x -> y -> z -> x
# the twelve rotations with components in {0, +-0.5, +-1}: every one maps the coordinate axes onto signed coordinate axes, exactly
EXACT = [q for q in itertools.product((-1.0, -0.5, 0.0, 0.5, 1.0), repeat=4) if abs(sum(c * c for c in q) - 1) < 1e-12 and q[3] >= 0
         and (q[3] > 0 or next(c for c in q if c != 0) > 0) and len({abs(c) for c in q} - {0.0}) == 1]
assert len(EXACT) == 12


def rotation_taking(z_from, z_to):
    """An exact rotation that maps z_from onto z_to (both signed coordinate axes)."""
    for q in EXACT:
        if np.array_equal(matrix(q) @ np.asarray(z_from, dtype=np.float64), np.asarray(z_to, dtype=np.float64)):
            return q
    raise ValueError((z_from, z_to))


def qmul(a, b):
    """Hamilton product a * b (apply b, then a): bepu's Concatenate(b, a)."""
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return (aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx, aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz)


def to_local(v, q):
    """World direction v expressed in the frame of orientation q."""
    return tuple(matrix(q).T @ np.asarray(v, dtype=np.float64))


# ---- cases --------------------------------------------------------------------------------------------------------------------------------------

def body(pos, q=IDENTITY, inertia=INERTIA, inv_mass=1.0):
    return {"pos": tuple(float(c) for c in pos), "q": q, "inertia": tuple(inertia), "inv_mass": inv_mass}


def locked(b):
    return dict(b, inertia=(0.0, 0.0, 0.0))


def kinematic(b):
    return dict(b, inertia=(0.0, 0.0, 0.0), inv_mass=0.0)


def prestep(layout, fields):
    rows = layout["prestep_rows"]
    out = np.full(len(rows), np.nan)
    for name, vals in fields.items():
        vals = np.atleast_1d(np.asarray(vals, dtype=np.float64))
        idx = [i for i, r in enumerate(rows) if r == name or r.startswith(name + ".")]
        assert len(idx) == vals.size, (name, rows)
        out[idx] = vals
    assert not np.isnan(out).any(), (fields, [r for r, v in zip(rows, out) if np.isnan(v)])
    return out.astype(np.float32)


def contact_cases(L):
    """Contact edges for every contact type: friction 0, depth 0, recovery 0, all offsets equal, identical nonconvex normals; for two-body
    manifolds also a rotation-locked body A and a kinematic body B. The rest state runs the friction clamps at zero magnitude."""
    out = []
    for t in CONTACT_TYPES:
        nonconvex = t >= 8
        two = t in (4, 5, 6, 7, 15, 16, 17)
        n = (t % 4 + 1) if t < 8 else (t - 6 if t < 15 else t - 13)
        corners = [(-0.5, -0.5, -0.5), (0.5, -0.5, -0.5), (0.5, -0.5, 0.5), (-0.5, -0.5, 0.5)][:n]
        normals = [(0.0, 1.0, 0.0), (0.0, 0.0, 1.0), (1.0, 0.0, 0.0), (0.0, -1.0, 0.0)][:n]

        def make(label, friction=1.0, depth=0.01, recovery=2.0, offsets=corners, normal_list=normals, bodies=None):
            f = {"MaterialProperties.FrictionCoefficient": friction, "MaterialProperties.SpringSettings": SPRING, "MaterialProperties.MaximumRecoveryVelocity": recovery}
            for i in range(n):
                if nonconvex:
                    f["Contact%d.Offset" % i] = offsets[i]
                    f["Contact%d.Normal" % i] = normal_list[i]
                else:
                    f["Contact%d.OffsetA" % i] = offsets[i]
                f["Contact%d.Depth" % i] = depth
            if not nonconvex:
                f["Normal"] = (0.0, 1.0, 0.0)
            if two:
                f["OffsetB"] = (0.0, -1.0, 0.0)
            bs = bodies or ([body((0, 1, 0)), body((0, 0, 0), q=PERMUTE)] if two else [body((0, 1, 0), q=PERMUTE)])
            out.append((t, "friction_clamp", "contact %d: %s" % (t, label), bs, prestep(L[t], f)))

        make("generic")
        make("friction 0", friction=0.0)
        make("depth exactly 0", depth=0.0)
        make("MaximumRecoveryVelocity 0", recovery=0.0)
        make("all offsets equal", offsets=[(0.25, -0.5, 0.125)] * n)
        if nonconvex:
            make("identical normals", normal_list=[(0.0, 1.0, 0.0)] * n)
        if two:
            make("rotation-locked body A", bodies=[locked(body((0, 1, 0))), body((0, 0, 0))])
            make("kinematic body B", bodies=[body((0, 1, 0)), kinematic(body((0, 0, 0)))])
    return out


def joint_cases(L):
    out = []

    def add(t, site, label, bodies, **fields):
        out.append((t, site, label, bodies, prestep(L[t], fields)))

    A, B = body((0, 0, 0)), body((0, 1, 0))
    PA, PB = body((0, 0, 0), q=PERMUTE), body((0, 1, 0), q=PERMUTE)
    Z, NZ = (0.0, 0.0, 1.0), (0.0, 0.0, -1.0)
    two_body_edges = lambda a, b: [("", [a, b]), (" (A rotation-locked)", [locked(a), b]), (" (B kinematic)", [a, kinematic(b)]), (" (A locked, B kinematic)", [locked(a), kinematic(b)])]

    # -- parallel / antiparallel axes, per body orientation: the local axes are the world axis expressed in each body's frame
    for a, b, how in ((A, B, "identity"), (PA, B, "A permuted"), (PA, PB, "both permuted")):
        for wb, rel in ((Z, "parallel"), (NZ, "antiparallel"), ((1.0, 0.0, 0.0), "perpendicular")):
            la, lb = to_local(Z, a["q"]), to_local(wb, b["q"])
            for suffix, bs in (two_body_edges(a, b) if rel != "perpendicular" else [("", [a, b])]):
                add(25, "swing_limit_fallback", "SwingLimit %s axes, %s%s" % (rel, how, suffix), bs, AxisLocalA=la, AxisLocalB=lb, MinimumDot=0.5, SpringSettings=SPRING)
                add(24, "angular_swivel_hinge_fallback", "AngularSwivelHinge %s axes, %s%s" % (rel, how, suffix), bs, LocalSwivelAxisA=la, LocalHingeAxisB=lb, SpringSettings=SPRING)
                add(46, "swivel_hinge_fallback", "SwivelHinge %s axes, %s%s" % (rel, how, suffix), bs, LocalOffsetA=(0, 0.5, 0), LocalSwivelAxisA=la, LocalOffsetB=to_local((0, -0.5, 0), b["q"]),
                    LocalHingeAxisB=lb, SpringSettings=SPRING)
            if rel == "antiparallel":
                for suffix, bs in two_body_edges(a, b):
                    add(28, "twist_motor_fallback", "TwistMotor opposed axes, %s%s" % (how, suffix), bs, LocalAxisA=la, LocalAxisB=lb, TargetVelocity=0.5, Settings=MOTOR)
            else:  # the generic side of the guard
                add(28, "twist_motor_fallback", "TwistMotor %s axes, %s" % (rel, how), [a, b], LocalAxisA=la, LocalAxisB=lb, TargetVelocity=0.5, Settings=MOTOR)
        # hinge axis B on jacobian axis X, then on Y, of hinge axis A = z: both on-plane fallbacks
        for wb, which in (((0.0, 1.0, 0.0), "x"), ((1.0, 0.0, 0.0), "y")):
            la, lb = to_local(Z, a["q"]), to_local(wb, b["q"])
            add(23, "hinge_on_plane_" + which, "AngularHinge axis B on the %s jacobian axis, %s" % (which, how), [a, b], LocalHingeAxisA=la, LocalHingeAxisB=lb, SpringSettings=SPRING)
            add(47, "hinge_on_plane_" + which, "Hinge axis B on the %s jacobian axis, %s" % (which, how), [a, b], LocalOffsetA=(0, 0.5, 0), LocalHingeAxisA=la,
                LocalOffsetB=to_local((0, -0.5, 0), b["q"]), LocalHingeAxisB=lb, SpringSettings=SPRING)

    # -- twist bases with opposed Z axes: along z (|x| = |y| tie, y smaller than z), along y (tie, y not smaller), along x, and along (0, 0.6, 0.8)
    for axis in ((0.0, 0.0, 1.0), (0.0, 1.0, 0.0), (1.0, 0.0, 0.0)):
        qa = rotation_taking(Z, axis)
        qb = rotation_taking(Z, tuple(-c for c in axis))
        for suffix, bs in two_body_edges(A, B):
            add(26, "twist_opposed_z", "TwistServo opposed Z along %s%s" % (axis, suffix), bs, LocalBasisA=qa, LocalBasisB=qb, TargetAngle=0.25, SpringSettings=SPRING, ServoSettings=SERVO)
            add(27, "twist_opposed_z", "TwistLimit opposed Z along %s%s" % (axis, suffix), bs, LocalBasisA=qa, LocalBasisB=qb, MinimumAngle=-0.5, MaximumAngle=0.5, SpringSettings=SPRING)
    c, s = np.sqrt(0.9), np.sqrt(0.1)  # rotation about x taking z to (0, -0.6, 0.8); then half a turn about its own x axis
    qa = (float(np.float32(s)), 0.0, 0.0, float(np.float32(c)))
    qb = qmul(qa, (1.0, 0.0, 0.0, 0.0))
    add(26, "twist_opposed_z", "TwistServo opposed Z, |x| smallest", [A, B], LocalBasisA=qa, LocalBasisB=qb, TargetAngle=0.25, SpringSettings=SPRING, ServoSettings=SERVO)
    add(27, "twist_opposed_z", "TwistLimit opposed Z, |x| smallest", [A, B], LocalBasisA=qa, LocalBasisB=qb, MinimumAngle=-0.5, MaximumAngle=0.5, SpringSettings=SPRING)
    # nearly opposed: dot(Z_A, Z_B) = -cos(1e-3) ~ -0.9999995, between -1 and the -0.999999 threshold (still the antiparallel case)
    qn = (float(np.float32(np.cos(5e-4))), 0.0, 0.0, float(np.float32(np.sin(5e-4))))
    add(26, "twist_opposed_z", "TwistServo nearly opposed Z, dot -0.9999995", [A, B], LocalBasisA=IDENTITY, LocalBasisB=qn, TargetAngle=0.25, SpringSettings=SPRING, ServoSettings=SERVO)
    add(27, "twist_opposed_z", "TwistLimit nearly opposed Z, dot -0.9999995", [A, B], LocalBasisA=IDENTITY, LocalBasisB=qn, MinimumAngle=-0.5, MaximumAngle=0.5, SpringSettings=SPRING)
    add(26, "twist_opposed_z", "TwistServo at its target (aligned Z axes)", [A, B], LocalBasisA=IDENTITY, LocalBasisB=IDENTITY, TargetAngle=0.0, SpringSettings=SPRING, ServoSettings=SERVO)
    add(27, "twist_opposed_z", "TwistLimit aligned Z axes", [A, B], LocalBasisA=IDENTITY, LocalBasisB=PERMUTE, MinimumAngle=-0.5, MaximumAngle=0.5, SpringSettings=SPRING)

    # -- angular servos at their target (the error rotation is the identity: the axis-angle fallback), with every servo setting
    for servo, how in ((SERVO, "servo"), (SERVO_DEFAULT, "default servo"), (SERVO_ZERO, "zero speed and force")):
        for a, b, orient in ((A, B, "identity"), (PA, PB, "both permuted")):
            for suffix, bs in two_body_edges(a, b):
                add(29, "axis_angle_fallback", "AngularServo at target, %s, %s%s" % (how, orient, suffix), bs, TargetRelativeRotationLocalA=IDENTITY, SpringSettings=SPRING, ServoSettings=servo)
            add(42, "axis_angle_fallback", "OneBodyAngularServo at target, %s, %s" % (how, orient), [a], TargetOrientation=a["q"], SpringSettings=SPRING, ServoSettings=servo)
        # off target: the generic side of the same guards
        add(29, "axis_angle_fallback", "AngularServo off target, %s" % how, [A, B], TargetRelativeRotationLocalA=PERMUTE, SpringSettings=SPRING, ServoSettings=servo)
        add(42, "axis_angle_fallback", "OneBodyAngularServo off target, %s" % how, [A], TargetOrientation=PERMUTE, SpringSettings=SPRING, ServoSettings=servo)
        add(53, "servo_error_length", "BallSocketServo separated anchors, %s" % how, [A, B], LocalOffsetA=(0, 0.25, 0), LocalOffsetB=(0, -0.25, 0), SpringSettings=SPRING, ServoSettings=servo)
        add(44, "servo_error_length", "OneBodyLinearServo off its target, %s" % how, [PB], LocalOffset=(0.5, 0, 0), Target=(0.5, 1.0, 0.0), SpringSettings=SPRING, ServoSettings=servo)
        add(37, "servo_error_length_2", "PointOnLineServo anchor off the line, %s" % how, [A, B], LocalOffsetA=(0, 0.5, 0), LocalOffsetB=(0.75, -0.25, 0), LocalDirection=(1.0, 0.0, 0.0),
            ServoSettings=servo, SpringSettings=SPRING)
        add(53, "servo_error_length", "BallSocketServo coincident anchors, %s" % how, [A, B], LocalOffsetA=(0, 0.5, 0), LocalOffsetB=(0, -0.5, 0), SpringSettings=SPRING, ServoSettings=servo)
        add(53, "servo_error_length", "BallSocketServo coincident anchors, permuted, %s" % how, [PA, PB], LocalOffsetA=to_local((0, 0.5, 0), PERMUTE), LocalOffsetB=to_local((0, -0.5, 0), PERMUTE),
            SpringSettings=SPRING, ServoSettings=servo)
        add(44, "servo_error_length", "OneBodyLinearServo at its target, %s" % how, [PB], LocalOffset=to_local((0.5, 0, 0), PERMUTE), Target=(0.5, 1.0, 0.0), SpringSettings=SPRING, ServoSettings=servo)
        add(37, "servo_error_length_2", "PointOnLineServo anchor on the line, %s" % how, [A, B], LocalOffsetA=(0, 0.5, 0), LocalOffsetB=(0, -0.5, 0), LocalDirection=(1.0, 0.0, 0.0),
            ServoSettings=servo, SpringSettings=SPRING)
        add(37, "servo_error_length_2", "PointOnLineServo anchor on the line away from A, %s" % how, [A, B], LocalOffsetA=(0, 0.5, 0), LocalOffsetB=(0.75, -0.5, 0), LocalDirection=(1.0, 0.0, 0.0),
            ServoSettings=servo, SpringSettings=SPRING)
        add(33, "distance_coincident", "DistanceServo coincident anchors, %s" % how, [A, B], LocalOffsetA=(0, 0.5, 0), LocalOffsetB=(0, -0.5, 0), TargetDistance=0.5, ServoSettings=servo,
            SpringSettings=SPRING)
        add(33, "", "DistanceServo at its target distance, %s" % how, [A, B], LocalOffsetA=(0, 0.25, 0), LocalOffsetB=(0, -0.25, 0), TargetDistance=0.5, ServoSettings=servo, SpringSettings=SPRING)
        add(38, "", "LinearAxisServo at its target offset, %s" % how, [A, B], LocalOffsetA=(0, 0, 0), LocalOffsetB=(0, 0, 0), LocalPlaneNormal=(0.0, 1.0, 0.0), TargetOffset=1.0,
            ServoSettings=servo, SpringSettings=SPRING)
    for suffix, bs in two_body_edges(A, B):
        add(31, "axis_angle_fallback", "Weld at its target pose" + suffix, bs, LocalOffset=(0, 1, 0), LocalOrientation=IDENTITY, SpringSettings=SPRING)
        add(53, "servo_error_length", "BallSocketServo coincident anchors" + suffix, bs, LocalOffsetA=(0.5, 0.5, 0), LocalOffsetB=(0.5, -0.5, 0), SpringSettings=SPRING, ServoSettings=SERVO)
        add(30, "servo_impulse_magnitude", "AngularMotor, target velocity 0" + suffix, bs, TargetVelocityLocalA=(0, 0, 0), Settings=MOTOR)
        add(52, "servo_impulse_magnitude", "BallSocketMotor, target velocity 0" + suffix, bs, LocalOffsetB=(0, -0.5, 0), TargetVelocityLocalA=(0, 0, 0), Settings=MOTOR)
        add(22, "", "BallSocket coincident anchors" + suffix, bs, LocalOffsetA=(0, 0.5, 0), LocalOffsetB=(0, -0.5, 0), SpringSettings=SPRING)
    add(31, "axis_angle_fallback", "Weld off its target orientation", [A, B], LocalOffset=(0, 1, 0), LocalOrientation=PERMUTE, SpringSettings=SPRING)
    add(31, "axis_angle_fallback", "Weld at its target pose, permuted", [PA, PB], LocalOffset=to_local((0, 1, 0), PERMUTE), LocalOrientation=IDENTITY, SpringSettings=SPRING)
    add(43, "servo_impulse_magnitude", "OneBodyAngularMotor, target velocity 0", [PA], TargetVelocity=(0, 0, 0), Settings=MOTOR)
    add(45, "servo_impulse_magnitude", "OneBodyLinearMotor, target velocity 0", [PA], LocalOffset=(0.5, 0, 0), TargetVelocity=(0, 0, 0), Settings=MOTOR)
    add(30, "servo_impulse_magnitude", "AngularMotor, zero force", [A, B], TargetVelocityLocalA=(0, 0, 0), Settings=(0.0, 1.0))
    add(43, "servo_impulse_magnitude", "OneBodyAngularMotor, zero force", [A], TargetVelocity=(0, 0, 0), Settings=(0.0, 1.0))
    add(45, "servo_impulse_magnitude", "OneBodyLinearMotor, zero force", [A], LocalOffset=(0.5, 0, 0), TargetVelocity=(0, 0, 0), Settings=(0.0, 1.0))
    add(52, "servo_impulse_magnitude", "BallSocketMotor, zero force", [A, B], LocalOffsetB=(0, -0.5, 0), TargetVelocityLocalA=(0, 0, 0), Settings=(0.0, 1.0))

    # -- coincident anchors and centres
    for suffix, bs in two_body_edges(A, B):
        add(34, "distance_coincident", "DistanceLimit coincident anchors" + suffix, bs, LocalOffsetA=(0, 0.5, 0), LocalOffsetB=(0, -0.5, 0), MinimumDistance=0.25, MaximumDistance=1.0, SpringSettings=SPRING)
        add(33, "distance_coincident", "DistanceServo coincident anchors" + suffix, bs, LocalOffsetA=(0, 0.5, 0), LocalOffsetB=(0, -0.5, 0), TargetDistance=0.5, ServoSettings=SERVO, SpringSettings=SPRING)
    add(34, "distance_coincident", "DistanceLimit separated anchors", [A, B], LocalOffsetA=(0, 0.25, 0), LocalOffsetB=(0, -0.25, 0), MinimumDistance=0.25, MaximumDistance=1.0, SpringSettings=SPRING)
    add(55, "center_distance_coincident", "CenterDistanceLimit separated centres", [A, B], MinimumDistance=0.5, MaximumDistance=2.0, SpringSettings=SPRING)
    # anchors 1e-10 apart: below the 1e-9 threshold, yet not coincident
    for t, extra in ((33, dict(TargetDistance=0.5, ServoSettings=SERVO)), (34, dict(MinimumDistance=0.25, MaximumDistance=1.0))):
        add(t, "distance_coincident", "%s anchors 1e-10 apart" % ("DistanceServo" if t == 33 else "DistanceLimit"), [A, body((0, 1e-10, 0))], LocalOffsetA=(0, 0, 0),
            LocalOffsetB=(0, 0, 0), SpringSettings=SPRING, **extra)
    C0, C1 = body((0.5, 0.25, -1)), body((0.5, 0.25, -1), q=PERMUTE)
    for suffix, bs in (("", [C0, C1]), (" (A rotation-locked)", [locked(C0), C1]), (" (B kinematic)", [C0, kinematic(C1)])):
        add(35, "center_distance_coincident", "CenterDistance coincident centres" + suffix, bs, TargetDistance=1.0, SpringSettings=SPRING)
        add(55, "center_distance_coincident", "CenterDistanceLimit coincident centres" + suffix, bs, MinimumDistance=0.5, MaximumDistance=2.0, SpringSettings=SPRING)
    add(35, "center_distance_coincident", "CenterDistance at its target", [A, B], TargetDistance=1.0, SpringSettings=SPRING)

    # -- Area and Volume: collinear, coplanar and coincident bodies
    line = [body((0, 0, 0)), body((1, 0, 0)), body((2, 0, 0))]
    point = [body((1, 1, 1)), body((1, 1, 1)), body((1, 1, 1)), body((1, 1, 1))]
    add(36, "area_normal", "Area collinear bodies", line, TargetScaledArea=1.0, SpringSettings=SPRING)
    add(36, "area_normal", "Area two coincident bodies", [body((0, 0, 0)), body((0, 0, 0)), body((0, 1, 0))], TargetScaledArea=1.0, SpringSettings=SPRING)
    add(36, "area_clamp", "Area coincident bodies", point[:3], TargetScaledArea=1.0, SpringSettings=SPRING)
    add(36, "area_clamp", "Area unit triangle", [body((0, 0, 0)), body((1, 0, 0)), body((0, 1, 0))], TargetScaledArea=1.0, SpringSettings=SPRING)
    add(32, "volume_clamp", "Volume coincident bodies", point, TargetScaledVolume=1.0, SpringSettings=SPRING)
    add(32, "", "Volume coplanar bodies", [body((0, 0, 0)), body((1, 0, 0)), body((0, 1, 0)), body((1, 1, 0))], TargetScaledVolume=1.0, SpringSettings=SPRING)
    add(32, "", "Volume collinear bodies", line + [body((3, 0, 0))], TargetScaledVolume=1.0, SpringSettings=SPRING)
    add(32, "volume_clamp", "Volume unit tetrahedron", [body((0, 0, 0)), body((1, 0, 0)), body((0, 1, 0)), body((0, 0, 1))], TargetScaledVolume=1.0, SpringSettings=SPRING)
    return out


def lane_inputs(bodies, moving, impulse_rows):
    n = len(bodies)
    states = np.zeros((MAX_BODIES, 14), dtype=np.float32)
    local = np.zeros((MAX_BODIES, 6), dtype=np.float32)
    for k, b in enumerate(bodies):
        d = np.diag(np.asarray(b["inertia"], dtype=np.float64))
        R = matrix(b["q"])
        w = R @ d @ R.T  # exact: R permutes and signs axes
        states[k, 0:3] = b["pos"]
        states[k, 3:7] = b["q"]
        states[k, 7:13] = (w[0, 0], w[1, 0], w[1, 1], w[2, 0], w[2, 1], w[2, 2])
        states[k, 13] = b["inv_mass"]
        local[k] = (d[0, 0], 0, d[1, 1], 0, 0, d[2, 2])
    vel = np.zeros((MAX_BODIES, 6), dtype=np.float32)
    imp = np.zeros(MAX_IMPULSES, dtype=np.float32)
    if moving:
        for k in range(n):
            vel[k] = np.array([0.5, -0.25, 0.75, -0.375, 0.625, 0.25]) * (1 + 0.5 * k)
        imp[:impulse_rows] = 0.125 * (1 + np.arange(impulse_rows) % 3)
    return states, local, vel, imp


def make_cases():
    """The singular cases as (type, site, label, bodies, prestep) tuples."""
    L = layouts()
    return contact_cases(L) + joint_cases(L)


def evaluate(eval_lane, type_id, states, vel, imp, pre, stages):
    """One case through eval_lane(type, stage, states, dt, prestep, impulses, velocities, row stride 1): per stage (velocities, impulses, prestep)."""
    outs = []
    for stage in range(stages):
        p, a, v = pre.copy(), imp.copy(), vel.copy()
        assert eval_lane(type_id, stage, states.ctypes.data_as(FP), DT, p.ctypes.data_as(FP), a.ctypes.data_as(FP), v.ctypes.data_as(FP), 1) == 0
        outs.append((v, a, p))
    return outs


def generate(eval_lane):
    L = layouts()
    rows = {"dropped": []}
    cols = {k: [] for k in ("type", "site", "label", "stages", "states", "local_inertia", "velocities", "impulses", "prestep", "out_velocities", "out_impulses", "out_prestep")}
    for type_id, site, label, bodies, pre in make_cases():
        nb, ni = L[type_id]["bodies"], len(L[type_id]["impulse_rows"])
        assert len(bodies) == nb, label
        stages = 3 if type_id in CONTACT_TYPES else 2
        for moving in (False, True):
            states, local, vel, imp = lane_inputs(bodies, moving, ni)
            p = np.zeros(MAX_PRESTEP, dtype=np.float32)
            p[:pre.size] = pre
            outs = evaluate(eval_lane, type_id, states, vel, imp, p, stages)
            if not all(np.isfinite(x).all() for o in outs for x in o):
                rows["dropped"].append(label)
                continue
            ov = np.zeros((3, MAX_BODIES, 6), dtype=np.float32)
            oi = np.zeros((3, MAX_IMPULSES), dtype=np.float32)
            op = np.zeros((3, MAX_PRESTEP), dtype=np.float32)
            for s, (v, a, q) in enumerate(outs):
                ov[s], oi[s], op[s] = v, a, q
            for k, x in (("type", type_id), ("site", site), ("label", label + (", moving" if moving else ", from rest")), ("stages", stages), ("states", states),
                         ("local_inertia", local), ("velocities", vel), ("impulses", imp), ("prestep", p), ("out_velocities", ov), ("out_impulses", oi), ("out_prestep", op)):
                cols[k].append(x)
    out = {k: np.array(v) for k, v in cols.items()}
    out["type"] = out["type"].astype(np.int32)
    out["stages"] = out["stages"].astype(np.int32)
    for k in ("out_velocities", "out_impulses", "out_prestep"):
        assert np.isfinite(out[k]).all(), k
    return out, sorted(set(rows["dropped"]))


def main():
    import build_ref

    if build_ref.build() is None:
        raise SystemExit("no reference checkout at %s (set BEPU_REFERENCE_ROOT)" % build_ref.REFERENCE)
    lib = C.CDLL(build_ref.LIB)
    lib.ref_eval_lane.argtypes = [C.c_int32, C.c_int32, FP, C.c_float, FP, FP, FP, C.c_int32]
    out, dropped = generate(lib.ref_eval_lane)
    np.savez_compressed(PATH, **out)
    print("wrote", PATH, "%d cases" % out["type"].size, "; left out (the reference is not finite there):", dropped)


if __name__ == "__main__":
    main()
