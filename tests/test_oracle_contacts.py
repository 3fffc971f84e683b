"""CPU tests pinning the oracle's restatement of all 14 contact manifold types (Constraints/Contact/ContactConvexTypes.cs,
ContactNonconvexCommon.cs) on analytic known answers that do not come from the oracle: a resting body's penetration impulses carry its
weight; friction decelerates a sliding body at mu * g for the per-contact friction of the nonconvex types and at (mu / N) * g for the
N-contact convex types (the reference bounds the manifold's tangent impulse by `(1/N) * FrictionCoefficient * sum(penetration impulses)`,
ContactConvexTypes.cs:L1502-1503 for Contact4, likewise L475, L639, L813, L1138, L1315 — reproduced as written); twist friction decelerates a
spinning body by (mu / N) * sum(N_i * r_i) / I; and a penetrating contact separates at no more than MaximumRecoveryVelocity. One-body
types act against the static world, two-body types against a kinematic ground body."""
import numpy as np
import pytest

from bepuphysics2_b200 import scenes
from tests import util

DT = 1.0 / 60.0
G = 10.0

FOOTPRINTS = {
    1: [[0.0, -0.5, 0.0]],
    2: [[-0.5, -0.5, 0.0], [0.5, -0.5, 0.0]],
    3: [[-0.5, -0.5, -0.4], [0.5, -0.5, -0.4], [0.0, -0.5, 0.8]],  # centroid under the centre of mass
    4: [[-0.5, -0.5, -0.5], [0.5, -0.5, -0.5], [-0.5, -0.5, 0.5], [0.5, -0.5, 0.5]],
}
CONTACT_TYPES = (
    [(scenes.CONVEX_ONE_BODY[n], n, "convex", 1) for n in (1, 2, 3, 4)]
    + [(scenes.CONVEX_TWO_BODY[n], n, "convex", 2) for n in (1, 2, 3, 4)]
    + [(scenes.NONCONVEX_ONE_BODY[n], n, "nonconvex", 1) for n in (2, 3, 4)]
    + [(scenes.NONCONVEX_TWO_BODY[n], n, "nonconvex", 2) for n in (2, 3, 4)]
)
IDS = ["type%d" % t[0] for t in CONTACT_TYPES]


def _scene(type_id, contacts, family, body_count, friction, depth=0.0, linear=(0, 0, 0), angular=(0, 0, 0), inverse_inertia=(6.0, 0, 6.0, 0, 0, 6.0), max_recovery=2.0):
    """One unit-mass body at the origin resting through `contacts` contacts with normal +y on the world / on kinematic body 1."""
    pos = np.array([[0, 0, 0], [0, -1.0, 0]], dtype=np.float32)[:body_count]
    inv_mass = np.array([1.0, 0.0], dtype=np.float32)[:body_count]
    inertia = np.zeros((body_count, 6), dtype=np.float32)
    inertia[0] = inverse_inertia
    lin = np.zeros((body_count, 3), dtype=np.float32)
    ang = np.zeros((body_count, 3), dtype=np.float32)
    lin[0], ang[0] = linear, angular
    bodies = scenes.make_bodies(pos, linear=lin, angular=ang, inverse_mass=inv_mass, inverse_inertia=inertia)
    offsets = np.asarray([FOOTPRINTS[contacts]], dtype=np.float32)
    depths = np.full((1, contacts), depth, dtype=np.float32)
    offset_b = (pos[1] - pos[0])[None, :] if body_count == 2 else None
    if family == "convex":
        pre = scenes.convex_prestep(offsets, depths, np.array([[0, 1, 0]], dtype=np.float32), offset_b, friction=friction, max_recovery=max_recovery)
    else:
        normals = np.tile(np.array([[[0, 1, 0]]], dtype=np.float32), (1, contacts, 1))
        pre = scenes.nonconvex_prestep(offsets, depths, normals, offset_b, friction=friction, max_recovery=max_recovery)
    handles = np.arange(body_count, dtype=np.int32)[None, :]
    return {"bodies": bodies, "constraints": [(type_id, handles, pre)]}


def _penetration_impulses(sim, contacts, family):
    (tb,) = list(sim.type_batches())
    rows = tb.accumulated_impulses[0, :, 0].astype(np.float64)
    # convex: Tangent.X, Tangent.Y, Penetration0..N-1, Twist; nonconvex: (Tangent.X, Tangent.Y, Penetration) per contact (tests/golden/type_layouts.json)
    return rows[2 : 2 + contacts] if family == "convex" else rows[2::3]


@pytest.mark.parametrize("type_id,contacts,family,body_count", CONTACT_TYPES, ids=IDS)
def test_resting_contact_carries_the_weight(libs, type_id, contacts, family, body_count):
    sim = util.make_sim(_scene(type_id, contacts, family, body_count, friction=1.0), substeps=1, velocity_iterations=4, integrator=util.integrator(gravity=(0.0, -G, 0.0), linear_damping=0.0, angular_damping=0.0))
    for _ in range(120):
        util.ob.solve(sim, DT)
    pen = _penetration_impulses(sim, contacts, family)
    assert (pen >= 0).all()
    assert pen.sum() == pytest.approx(G * DT, rel=1e-3)
    # the footprints are balanced about the centre of mass: no net torque, so the body does not start to rotate (an unbalanced contact
    # would add 6 * 0.5 * g * dt = 0.5 rad/s per frame; the soft contacts of the asymmetric 3-point footprint settle with a few mrad/s)
    assert np.abs(sim.bodies[0, 12:15]).max() < 1e-2
    # a rigid-ish contact (30 Hz, critically damped) lets the body sink only slowly under its weight
    assert -0.05 < float(sim.bodies[0, 9]) <= 1e-6


@pytest.mark.parametrize("type_id,contacts,family,body_count", CONTACT_TYPES, ids=IDS)
def test_sliding_friction_decelerates_at_mu_g(libs, type_id, contacts, family, body_count):
    mu = 0.4
    cone = mu / contacts if family == "convex" else mu  # see the module docstring
    # rotation locked (zero inverse inertia) so that the friction force acting below the centre of mass does not tip the body
    scene = _scene(type_id, contacts, family, body_count, friction=mu, linear=(3.0, 0, 1.0), inverse_inertia=(0, 0, 0, 0, 0, 0))
    sim = util.make_sim(scene, substeps=1, velocity_iterations=4, integrator=util.integrator(gravity=(0.0, -G, 0.0), linear_damping=0.0, angular_damping=0.0))
    speeds = []
    for _ in range(40):
        util.ob.solve(sim, DT)
        speeds.append(np.hypot(float(sim.bodies[0, 8]), float(sim.bodies[0, 10])))
    direction = sim.bodies[0, [8, 10]].astype(np.float64) / speeds[-1]
    assert direction == pytest.approx(np.array([3.0, 1.0]) / np.hypot(3.0, 1.0), abs=1e-3)  # friction opposes the motion, it does not steer it
    assert speeds[15] - speeds[35] == pytest.approx(20 * cone * G * DT, rel=2e-2)


@pytest.mark.parametrize("type_id,contacts,family,body_count", [t for t in CONTACT_TYPES if t[2] == "convex" and t[1] > 1], ids=[i for i, t in zip(IDS, CONTACT_TYPES) if t[2] == "convex" and t[1] > 1])
def test_twist_friction_decelerates_the_spin(libs, type_id, contacts, family, body_count):
    """TwistFriction: |impulse| <= mu / N * sum(penetration impulses) ... * distances (ContactConvexTypes.cs, premultiplied friction coefficient)."""
    mu, inverse_inertia_y = 0.3, 6.0
    scene = _scene(type_id, contacts, family, body_count, friction=mu, angular=(0, 6.0, 0))
    sim = util.make_sim(scene, substeps=1, velocity_iterations=4, integrator=util.integrator(gravity=(0.0, -G, 0.0), linear_damping=0.0, angular_damping=0.0))
    spin = []
    for _ in range(30):
        util.ob.solve(sim, DT)
        spin.append(float(sim.bodies[0, 13]))
    pts = np.asarray(FOOTPRINTS[contacts], dtype=np.float64)
    lever = np.linalg.norm(pts - pts.mean(axis=0), axis=1)
    pen = _penetration_impulses(sim, contacts, family)
    # each contact carries N_i; the reference bounds the twist impulse by (mu / N) * sum_i(N_i * r_i) — N here is the contact count
    expected_per_frame = inverse_inertia_y * (mu / contacts) * float((pen * lever).sum())
    assert spin[10] - spin[25] == pytest.approx(15 * expected_per_frame, rel=3e-2)
    assert spin[25] > 0


@pytest.mark.parametrize("type_id,contacts,family,body_count", CONTACT_TYPES, ids=IDS)
def test_penetration_recovery_is_speed_limited(libs, type_id, contacts, family, body_count):
    """A deep contact pushes out at MaximumRecoveryVelocity at most (PenetrationLimit.cs:L78-131: bias = min(depth * ERP, maxRecovery))."""
    integ = util.integrator(gravity=(0.0, -G, 0.0), linear_damping=0.0, angular_damping=0.0)
    integ.gravity[1] = 0.0
    scene = _scene(type_id, contacts, family, body_count, friction=1.0, depth=0.5, max_recovery=0.75)
    sim = util.make_sim(scene, substeps=1, velocity_iterations=8, integrator=integ)
    for _ in range(10):
        util.ob.solve(sim, DT)
    assert float(sim.bodies[0, 9]) == pytest.approx(0.75, rel=2e-2)
    # and a separated contact (negative depth beyond what the body can close in a step) applies nothing
    scene = _scene(type_id, contacts, family, body_count, friction=1.0, depth=-1.0)
    sim = util.make_sim(scene, substeps=1, velocity_iterations=4, integrator=util.integrator(gravity=(0.0, -G, 0.0), linear_damping=0.0, angular_damping=0.0))
    util.ob.solve(sim, DT)
    assert float(sim.bodies[0, 9]) == pytest.approx(-G * DT, rel=1e-6)
    assert np.abs(_penetration_impulses(sim, contacts, family)).max() == 0.0


@pytest.mark.parametrize("type_id,contacts,family,body_count", CONTACT_TYPES, ids=IDS)
def test_speculative_contact_only_removes_the_velocity_that_would_penetrate(libs, type_id, contacts, family, body_count):
    """Negative depth passes through the bias unclamped: bias = depth / dt (PenetrationLimit.cs:L124-127), so a body approaching a contact
    that is still `gap` away is slowed towards the approach speed gap / dt that just closes the gap this step, and a slower one is left
    alone. Each contact is a soft row (SpringSettings.cs:L37-55: softness = extra / (1 + extra) per unit effective mass, extra =
    1 / (w dt (w dt + 2 zeta))): the converged impulses of one step are the solution of a small linear system, solved here in float64."""
    integ = util.integrator(gravity=(0.0, -G, 0.0), linear_damping=0.0, angular_damping=0.0)
    integ.gravity[1] = 0.0
    gap = 0.01
    sim = util.make_sim(_scene(type_id, contacts, family, body_count, friction=0.0, depth=-gap, linear=(0, -1.0, 0)), substeps=1, velocity_iterations=30, integrator=integ)
    util.ob.solve(sim, DT)
    # float64 fixed point of the N soft rows: (J M^-1 J^T + extra * diag(K)) lambda = bias - J v0, K_i = (J M^-1 J^T)_ii, v = v0 + M^-1 J^T lambda
    w_dt = 2 * np.pi * 30 * DT
    extra = 1.0 / (w_dt * (w_dt + 2.0))
    normal = np.array([0.0, 1.0, 0.0])
    jac = np.array([np.r_[normal, np.cross(r, normal)] for r in np.asarray(FOOTPRINTS[contacts], dtype=np.float64)])
    inverse_mass = np.diag([1.0, 1.0, 1.0, 6.0, 6.0, 6.0])
    v0 = np.array([0, -1.0, 0, 0, 0, 0])
    a = jac @ inverse_mass @ jac.T
    lam = np.linalg.solve(a + extra * np.diag(np.diag(a)), -gap / DT - jac @ v0)
    assert (lam > 0).all()
    expected = v0 + inverse_mass @ jac.T @ lam
    assert sim.bodies[0, 8:11].astype(np.float64) == pytest.approx(expected[:3], abs=2e-5)
    assert sim.bodies[0, 12:15].astype(np.float64) == pytest.approx(expected[3:], abs=2e-5)
    assert _penetration_impulses(sim, contacts, family) == pytest.approx(lam, rel=1e-3)
    sim = util.make_sim(_scene(type_id, contacts, family, body_count, friction=0.0, depth=-gap, linear=(0, -0.5, 0)), substeps=1, velocity_iterations=8, integrator=integ)
    util.ob.solve(sim, DT)
    assert float(sim.bodies[0, 9]) == pytest.approx(-0.5, rel=1e-6)
    assert np.abs(_penetration_impulses(sim, contacts, family)).max() == 0.0
