// Pose / velocity integration arithmetic of the solver kernels (no memory access): PoseIntegrator.cs:L99-261, TypeProcessor.cs:L1204-1283,
// Demos/DemoCallbacks.cs:L99-102. Kept apart from the kernels so that tests/device_on_host can compile it for the host.
#pragma once
#include "bepu_device_math.cuh"

namespace BEPU_NS {

// ---- integration (PoseIntegrator.cs:L99-261, TypeProcessor.cs:L1204-1283, Demos/DemoCallbacks.cs:L99-102) -----------
BEPU_DI Q4 integrate_orientation(Q4 start, V3 w, float halfDt) {  // PoseIntegrator.cs:L146-164
    float speed = length(w);
    float halfAngle = speed * halfDt;
    float s = sin_approx(halfAngle);
    float scl = s / speed;
    Q4 q{w.x * scl, w.y * scl, w.z * scl, cos_approx(halfAngle)};
    Q4 end = normalize(concatenate(start, q));
    return speed > 1e-15f ? end : start;
}
BEPU_DI Sym3 rotate_inverse_inertia(Sym3 local, Q4 q) { return rotation_sandwich(matrix_from_quaternion(q), local); }  // L166-175
// The pose half of IntegratePoseAndVelocity (TypeProcessor.cs:L1204-1248): position and orientation advance by the velocity over dt, and the
// local inverse inertia is rotated into the new orientation. Shared by the WarmStart stages and the body part of the incremental contact update.
BEPU_DI void integrate_pose_and_inertia(V3 lin, V3 ang, float dt, Sym3 local, V3& pos, Q4& q, Sym3& world) {
    pos = pos + lin * dt;
    q = integrate_orientation(q, ang, dt * 0.5f);
    world = rotate_inverse_inertia(local, q);
}
BEPU_DI void callback_integrate_velocity(Velocity& v, float gx, float gy, float gz, float linearDampingDt, float angularDampingDt) {
    v.lin = (v.lin + V3{gx, gy, gz}) * linearDampingDt;
    v.ang = v.ang * angularDampingDt;
}
// The two optional terms of bepucuda_set_body_accelerations / bepucuda_set_point_gravity, applied after callback_integrate_velocity wherever its
// result is kept. Per-body accelerations (PerBodyGravityDemo.cs:L57-88): v += a * dt, not damped. Point gravity (PlanetDemo.cs:L36-47), in its
// operation order: offset = position - center, v.lin -= (attractorDt * offset) * (1 / max(1, |offset|^3)), with attractorDt = dt * strength from
// PrepareForIntegration; Vector3Wide / Vector<float> multiplies by the reciprocal (Vector3Wide.cs:L357-363).
BEPU_DI void integrate_velocity_extensions(Velocity& v, bool accelerations, V3 linearAcceleration, V3 angularAcceleration, float dt, bool pointGravity, V3 position,
                                           V3 center, float attractorDt) {
    if (accelerations) {
        v.lin = v.lin + linearAcceleration * dt;
        v.ang = v.ang + angularAcceleration * dt;
    }
    if (pointGravity) {
        const V3 offset = position - center;
        const float distance = length(offset);
        const float inverse = 1.0f / fmaxf(1.0f, distance * distance * distance);
        v.lin = v.lin - (offset * attractorDt) * inverse;
    }
}
BEPU_DI void fallback_if_inertia_incompatible(V3 previous, V3& w) {  // L180-190
    const float inf = __int_as_float(0x7f800000);
    bool useNew = fabsf(w.x) < inf && fabsf(w.y) < inf && fabsf(w.z) < inf;
    w = useNew ? w : previous;
}
// The two momentum-conserving modes are rare (AngularIntegrationMode.Nonconserving is the default everywhere in the
// reference's demos/benchmarks); keeping them out of line keeps their registers out of the hot WarmStart path.
static __device__ __noinline__ void integrate_angular_conserve_momentum(Q4 previousOrientation, Sym3 localInverseInertia, Sym3 worldInverseInertia, V3& w) {  // L192-206
    M33 prevR = matrix_from_quaternion(previousOrientation);
    V3 localPrevW = transform_by_transposed(w, prevR);
    Sym3 localInertiaTensor = invert(localInverseInertia);
    V3 angularMomentum = transform(transform(localPrevW, localInertiaTensor), prevR);
    V3 previous = w;
    w = transform(angularMomentum, worldInverseInertia);
    fallback_if_inertia_incompatible(previous, w);
}
static __device__ __noinline__ void integrate_angular_gyroscopic(Q4 orientation, Sym3 localInverseInertia, V3& w, float dt) {  // L208-253
    M33 R = matrix_from_quaternion(orientation);
    V3 localW = transform_by_transposed(w, R);
    Sym3 I = invert(localInverseInertia);
    V3 localMomentum = transform(localW, I);
    V3 residual = cross(localMomentum, localW) * dt;
    M33 skewMomentum{{0.0f, -localMomentum.z, localMomentum.y}, {localMomentum.z, 0.0f, -localMomentum.x}, {-localMomentum.y, localMomentum.x, 0.0f}};
    M33 skewVelocity{{0.0f, -localW.z, localW.y}, {localW.z, 0.0f, -localW.x}, {-localW.y, localW.x, 0.0f}};
    M33 tsv = multiply(skewVelocity, I);
    M33 J;
    V3 cx = (tsv.x - skewMomentum.x) * dt, cy = (tsv.y - skewMomentum.y) * dt, cz = (tsv.z - skewMomentum.z) * dt;
    J.x = {I.xx + cx.x, I.yx + cx.y, I.zx + cx.z};
    J.y = {I.yx + cy.x, I.yy + cy.y, I.zy + cy.z};
    J.z = {I.zx + cz.x, I.zy + cz.y, I.zz + cz.z};
    V3 newtonStep = transform(residual, invert(J));
    localW = localW - newtonStep;
    V3 previous = w;
    w = transform(localW, R);
    fallback_if_inertia_incompatible(previous, w);
}

}  // namespace BEPU_NS
