// The remaining joint / motor / servo / limit constraint functions of the reference's default type set (DefaultTypes.cs) for the sm_90a
// solver kernels (one thread = one constraint). Same call shape as bepu_joints.cuh:
//   warm_start(const BodyState* b, const float* p, const float* a, Velocity* v)
//   solve(const BodyState* b, float dt, float inverseDt, const float* p, float* a, Velocity* v)
// with b / v holding kBodies entries (1, 2, 3 or 4).
//
// MathHelper.FastReciprocal / FastReciprocalSquareRoot (MathHelper.cs:L380-413) are rcpps / rsqrtps hardware approximations on x86 whose
// error differs between CPU vendors; the portable definition the reference carries for other targets (1/v, 1/sqrt(v)) is what is used here.
#pragma once
#include "bepu_joints.cuh"
#include "bepu_type_table.h"

namespace BEPU_NS {

// ---- more settings helpers ----
BEPU_DI void servo_clamp_impulse1(float maximumImpulse, float& accumulated, float& csi) {  // ServoSettings.cs:L145-151
    float previous = accumulated;
    accumulated = fmax_ps(-maximumImpulse, fmin_ps(maximumImpulse, accumulated + csi));
    csi = accumulated - previous;
}
BEPU_DI V3 servo_clamped_bias_velocity3e(V3 error, float positionErrorToBiasVelocity, float maximumSpeed, float baseSpeedSetting, float inverseDt) {  // ServoSettings.cs:L132-142
    float errorLength = length(error);
    V3 errorAxis = error * (1.0f / errorLength);
    errorAxis = errorLength < 1e-10f ? V3{0.0f, 0.0f, 0.0f} : errorAxis;
    return servo_clamped_bias_velocity3(errorAxis, errorLength, positionErrorToBiasVelocity, maximumSpeed, baseSpeedSetting, inverseDt);
}
BEPU_DI V2 servo_clamped_bias_velocity2e(V2 error, float positionErrorToBiasVelocity, float maximumSpeed, float baseSpeedSetting, float inverseDt) {  // ServoSettings.cs:L88-113
    float errorLength = length(error);
    V2 errorAxis = error * (1.0f / errorLength);
    if (errorLength < 1e-10f) errorAxis = V2{0.0f, 0.0f};
    float baseSpeed = fmin_ps(baseSpeedSetting, errorLength * inverseDt);
    float unclampedBiasSpeed = errorLength * positionErrorToBiasVelocity;
    float targetSpeed = fmax_ps(baseSpeed, unclampedBiasSpeed);
    float scl = fmin_ps(1.0f, maximumSpeed / targetSpeed);
    scl = targetSpeed < 1e-10f ? 1.0f : scl;
    return errorAxis * (scl * unclampedBiasSpeed);
}
BEPU_DI void servo_clamp_impulse2(float maximumImpulse, V2& accumulated, V2& csi) {  // ServoSettings.cs:L153-164
    V2 previous = accumulated;
    V2 unclamped = accumulated + csi;
    float magnitude = length(unclamped);
    float impulseScale = fabsf(magnitude) < 1e-10f ? 1.0f : fmin_ps(maximumImpulse / magnitude, 1.0f);
    accumulated = unclamped * impulseScale;
    csi = accumulated - previous;
}
BEPU_DI float inequality_bias_velocity(float error, float positionErrorToVelocity, float inverseDt) { return fmin_ps(error * inverseDt, error * positionErrorToVelocity); }  // InequalityHelpers.cs:L9-12

// ---- Weld (31): Weld.cs:L83-221; Symmetric6x6Wide.cs:L84-129 ----
// prestep: LocalOffset xyz, LocalOrientation xyzw, AngularFrequency, TwiceDampingRatio | impulses: Orientation xyz, Offset xyz
BEPU_DI M33 cross_product_matrix(V3 v) { return M33{V3{0.0f, -v.z, v.y}, V3{v.z, 0.0f, -v.x}, V3{-v.y, v.x, 0.0f}}; }  // Matrix3x3Wide.cs:L169-180
BEPU_DI M33 multiply_sym_matrix(Sym3 a, const M33& b) {  // Symmetric3x3Wide.cs:L343-356
    M33 r;
    r.x.x = a.xx * b.x.x + a.yx * b.y.x + a.zx * b.z.x;
    r.x.y = a.xx * b.x.y + a.yx * b.y.y + a.zx * b.z.y;
    r.x.z = a.xx * b.x.z + a.yx * b.y.z + a.zx * b.z.z;
    r.y.x = a.yx * b.x.x + a.yy * b.y.x + a.zy * b.z.x;
    r.y.y = a.yx * b.x.y + a.yy * b.y.y + a.zy * b.z.y;
    r.y.z = a.yx * b.x.z + a.yy * b.y.z + a.zy * b.z.z;
    r.z.x = a.zx * b.x.x + a.zy * b.y.x + a.zz * b.z.x;
    r.z.y = a.zx * b.x.y + a.zy * b.y.y + a.zz * b.z.y;
    r.z.z = a.zx * b.x.z + a.zy * b.y.z + a.zz * b.z.z;
    return r;
}
BEPU_DI Sym3 complete_matrix_sandwich_transpose(const M33& a, const M33& b) {  // Symmetric3x3Wide.cs:L508-518
    Sym3 r;
    r.xx = a.x.x * b.x.x + a.y.x * b.y.x + a.z.x * b.z.x;
    r.yx = a.x.y * b.x.x + a.y.y * b.y.x + a.z.y * b.z.x;
    r.yy = a.x.y * b.x.y + a.y.y * b.y.y + a.z.y * b.z.y;
    r.zx = a.x.z * b.x.x + a.y.z * b.y.x + a.z.z * b.z.x;
    r.zy = a.x.z * b.x.y + a.y.z * b.y.y + a.z.z * b.z.y;
    r.zz = a.x.z * b.x.z + a.y.z * b.y.z + a.z.z * b.z.z;
    return r;
}
BEPU_DI void ldlt_solve6(V3 v0, V3 v1, Sym3 a, const M33& b, Sym3 d, V3& result0, V3& result1) {
    float d1 = a.xx;
    float inverseD1 = 1.0f / d1;
    float l21 = inverseD1 * a.yx, l31 = inverseD1 * a.zx, l41 = inverseD1 * b.x.x, l51 = inverseD1 * b.x.y, l61 = inverseD1 * b.x.z;
    float d2 = a.yy - l21 * l21 * d1;
    float inverseD2 = 1.0f / d2;
    float l32 = inverseD2 * (a.zy - l31 * l21 * d1);
    float l42 = inverseD2 * (b.y.x - l41 * l21 * d1);
    float l52 = inverseD2 * (b.y.y - l51 * l21 * d1);
    float l62 = inverseD2 * (b.y.z - l61 * l21 * d1);
    float d3 = a.zz - l31 * l31 * d1 - l32 * l32 * d2;
    float inverseD3 = 1.0f / d3;
    float l43 = inverseD3 * (b.z.x - l41 * l31 * d1 - l42 * l32 * d2);
    float l53 = inverseD3 * (b.z.y - l51 * l31 * d1 - l52 * l32 * d2);
    float l63 = inverseD3 * (b.z.z - l61 * l31 * d1 - l62 * l32 * d2);
    float d4 = d.xx - l41 * l41 * d1 - l42 * l42 * d2 - l43 * l43 * d3;
    float inverseD4 = 1.0f / d4;
    float l54 = inverseD4 * (d.yx - l51 * l41 * d1 - l52 * l42 * d2 - l53 * l43 * d3);
    float l64 = inverseD4 * (d.zx - l61 * l41 * d1 - l62 * l42 * d2 - l63 * l43 * d3);
    float d5 = d.yy - l51 * l51 * d1 - l52 * l52 * d2 - l53 * l53 * d3 - l54 * l54 * d4;
    float inverseD5 = 1.0f / d5;
    float l65 = inverseD5 * (d.zy - l61 * l51 * d1 - l62 * l52 * d2 - l63 * l53 * d3 - l64 * l54 * d4);
    float d6 = d.zz - l61 * l61 * d1 - l62 * l62 * d2 - l63 * l63 * d3 - l64 * l64 * d4 - l65 * l65 * d5;
    float inverseD6 = 1.0f / d6;
    result0.x = v0.x;
    result0.y = v0.y - l21 * result0.x;
    result0.z = v0.z - l31 * result0.x - l32 * result0.y;
    result1.x = v1.x - l41 * result0.x - l42 * result0.y - l43 * result0.z;
    result1.y = v1.y - l51 * result0.x - l52 * result0.y - l53 * result0.z - l54 * result1.x;
    result1.z = v1.z - l61 * result0.x - l62 * result0.y - l63 * result0.z - l64 * result1.x - l65 * result1.y;
    result1.z = result1.z * inverseD6;
    result1.y = result1.y * inverseD5 - l65 * result1.z;
    result1.x = result1.x * inverseD4 - l64 * result1.z - l54 * result1.y;
    result0.z = result0.z * inverseD3 - l63 * result1.z - l53 * result1.y - l43 * result1.x;
    result0.y = result0.y * inverseD2 - l62 * result1.z - l52 * result1.y - l42 * result1.x - l32 * result0.z;
    result0.x = result0.x * inverseD1 - l61 * result1.z - l51 * result1.y - l41 * result1.x - l31 * result0.z - l21 * result0.y;
}
struct Weld {
    static constexpr int kBodies = 2, kPrestepRows = 9, kImpulseRows = 6;
    static constexpr bool kIncremental = false, kNeedsPose = true;
    BEPU_DI static void apply(const Inertia& iA, const Inertia& iB, V3 offset, V3 orientationCSI, V3 offsetCSI, Velocity& vA, Velocity& vB) {  // L85-114
        vA.lin = vA.lin + offsetCSI * iA.inv_mass;
        V3 angularImpulseA = cross(offset, offsetCSI) + orientationCSI;
        vA.ang = vA.ang + transform(angularImpulseA, iA.t);
        vB.lin = vB.lin - offsetCSI * iB.inv_mass;
        vB.ang = vB.ang - transform(orientationCSI, iB.t);
    }
    template <class PR, class AR> BEPU_DI static void warm_start(const BodyState* b, PR p, AR a, Velocity* v) {
        V3 offset = transform(ldrow3(p, 0), b[0].q);
        apply(b[0].inertia, b[1].inertia, offset, V3{ldacc(a, 0), ldacc(a, 1), ldacc(a, 2)}, V3{ldacc(a, 3), ldacc(a, 4), ldacc(a, 5)}, v[0], v[1]);
    }
    template <class PR, class AR> BEPU_DI static void solve(const BodyState* b, float dt, float, PR p, AR a, Velocity* v) {
        const Inertia& iA = b[0].inertia;
        const Inertia& iB = b[1].inertia;
        V3 offset = transform(ldrow3(p, 0), b[0].q);
        Sym3 jmjtA = iA.t + iB.t;
        M33 xAB = cross_product_matrix(offset);
        M33 jmjtB = multiply_sym_matrix(iA.t, xAB);
        Sym3 jmjtD = complete_matrix_sandwich_transpose(xAB, jmjtB);
        float diagonalAdd = iA.inv_mass + iB.inv_mass;
        jmjtD.xx += diagonalAdd;
        jmjtD.yy += diagonalAdd;
        jmjtD.zz += diagonalAdd;
        V3 positionError = (b[1].pos - b[0].pos) - offset;
        Q4 targetOrientationB = concatenate(ldrow4(p, 3), b[0].q);
        Q4 rotationError = concatenate(conjugate(targetOrientationB), b[1].q);
        V3 rotationErrorAxis;
        float rotationErrorLength;
        axis_angle_from_quaternion(rotationError, rotationErrorAxis, rotationErrorLength);
        Springiness sp = compute_springiness(ldrow(p, 7), ldrow(p, 8), dt);
        const float pe2v = sp.position_error_to_velocity, cfm = sp.effective_mass_cfm_scale, soft = sp.softness_impulse_scale;
        V3 orientationBiasVelocity = rotationErrorAxis * (rotationErrorLength * pe2v);
        V3 offsetBiasVelocity = positionError * pe2v;
        const V3 wA = v[0].ang, wB = v[1].ang, lA = v[0].lin, lB = v[1].lin;
        V3 orientationCSV, offsetCSV;
        orientationCSV.x = orientationBiasVelocity.x - wA.x + wB.x;
        orientationCSV.y = orientationBiasVelocity.y - wA.y + wB.y;
        orientationCSV.z = orientationBiasVelocity.z - wA.z + wB.z;
        offsetCSV.x = offsetBiasVelocity.x - lA.x + lB.x - (wA.y * offset.z - wA.z * offset.y);
        offsetCSV.y = offsetBiasVelocity.y - lA.y + lB.y - (wA.z * offset.x - wA.x * offset.z);
        offsetCSV.z = offsetBiasVelocity.z - lA.z + lB.z - (wA.x * offset.y - wA.y * offset.x);
        V3 orientationCSI, offsetCSI;
        ldlt_solve6(orientationCSV, offsetCSV, jmjtA, jmjtB, jmjtD, orientationCSI, offsetCSI);
        V3 accOrientation{ldacc(a, 0), ldacc(a, 1), ldacc(a, 2)}, accOffset{ldacc(a, 3), ldacc(a, 4), ldacc(a, 5)};
        orientationCSI.x = orientationCSI.x * cfm - accOrientation.x * soft;
        orientationCSI.y = orientationCSI.y * cfm - accOrientation.y * soft;
        orientationCSI.z = orientationCSI.z * cfm - accOrientation.z * soft;
        accOrientation = accOrientation + orientationCSI;
        offsetCSI.x = offsetCSI.x * cfm - accOffset.x * soft;
        offsetCSI.y = offsetCSI.y * cfm - accOffset.y * soft;
        offsetCSI.z = offsetCSI.z * cfm - accOffset.z * soft;
        accOffset = accOffset + offsetCSI;
        apply(iA, iB, offset, orientationCSI, offsetCSI, v[0], v[1]);
        stacc(a, 0, accOrientation.x); stacc(a, 1, accOrientation.y); stacc(a, 2, accOrientation.z);
        stacc(a, 3, accOffset.x); stacc(a, 4, accOffset.y); stacc(a, 5, accOffset.z);
    }
};

// ---- AngularHinge (23): AngularHinge.cs:L71-223 ----
// prestep: LocalHingeAxisA xyz, LocalHingeAxisB xyz, AngularFrequency, TwiceDampingRatio | impulses: xy
struct AngularHinge {
    static constexpr int kBodies = 2, kPrestepRows = 8, kImpulseRows = 2;
    static constexpr bool kIncremental = false, kNeedsPose = true;
    BEPU_DI static void apply(const M23& i2vA, const M23& ni2vB, V2 csi, V3& wA, V3& wB) {  // L114-120
        wA = wA + transform(csi, i2vA);
        wB = wB - transform(csi, ni2vB);
    }
    BEPU_DI static M23 jacobians(V3 localHingeAxisA, Q4 qA, V3& hingeAxisA) {  // L122-131
        V3 localAX, localAY;
        build_orthonormal_basis(localHingeAxisA, localAX, localAY);
        M33 mA = matrix_from_quaternion(qA);
        hingeAxisA = transform(localHingeAxisA, mA);
        return M23{transform(localAX, mA), transform(localAY, mA)};
    }
    template <class PR, class AR> BEPU_DI static void warm_start(const BodyState* b, PR p, AR a, Velocity* v) {
        V3 hingeAxisA;
        M23 jacobianA = jacobians(ldrow3(p, 0), b[0].q, hingeAxisA);
        apply(multiply(jacobianA, b[0].inertia.t), multiply(jacobianA, b[1].inertia.t), V2{ldacc(a, 0), ldacc(a, 1)}, v[0].ang, v[1].ang);
    }
    template <class PR, class AR> BEPU_DI static void solve(const BodyState* b, float dt, float, PR p, AR a, Velocity* v) {
        V3 hingeAxisA;
        M23 jacobianA = jacobians(ldrow3(p, 0), b[0].q, hingeAxisA);
        V3 hingeAxisB = transform(ldrow3(p, 3), b[1].q);
        M23 i2vA = multiply(jacobianA, b[0].inertia.t), ni2vB = multiply(jacobianA, b[1].inertia.t);
        Sym2 inverseEffectiveMass = complete_matrix_sandwich(i2vA, jacobianA) + complete_matrix_sandwich(ni2vB, jacobianA);
        Sym2 effectiveMass = invert(inverseEffectiveMass);
        Springiness sp = compute_springiness(ldrow(p, 6), ldrow(p, 7), dt);
        V2 errorAngle = hinge_error_angles(hingeAxisA, hingeAxisB, jacobianA);
        V2 biasVelocity = errorAngle * (-sp.position_error_to_velocity);
        V2 biasImpulse = transform(biasVelocity, effectiveMass);
        V3 difference = v[0].ang - v[1].ang;
        V2 csv = transform_by_transpose(difference, jacobianA);
        V2 csi = transform(csv, effectiveMass);
        csi = csi * sp.effective_mass_cfm_scale;
        V2 acc{ldacc(a, 0), ldacc(a, 1)};
        V2 softnessContribution = acc * sp.softness_impulse_scale;
        csi = softnessContribution + csi;
        csi = biasImpulse - csi;
        acc = acc + csi;
        apply(i2vA, ni2vB, csi, v[0].ang, v[1].ang);
        stacc(a, 0, acc.x); stacc(a, 1, acc.y);
    }
};

// ---- AngularSwivelHinge (24): AngularSwivelHinge.cs:L71-148 ----
// prestep: LocalSwivelAxisA xyz, LocalHingeAxisB xyz, AngularFrequency, TwiceDampingRatio | impulse: 1
struct AngularSwivelHinge {
    static constexpr int kBodies = 2, kPrestepRows = 8, kImpulseRows = 1;
    static constexpr bool kIncremental = false, kNeedsPose = true;
    template <class PR> BEPU_DI static V3 jacobian(PR p, Q4 qA, Q4 qB, V3& swivelAxis, V3& hingeAxis) {  // L82-94
        swivelAxis = transform(ldrow3(p, 0), qA);
        hingeAxis = transform(ldrow3(p, 3), qB);
        V3 j = cross(swivelAxis, hingeAxis);
        V3 fallbackJacobian = find_perpendicular(swivelAxis);
        return dot(j, j) < 1e-3f ? fallbackJacobian : j;
    }
    template <class PR, class AR> BEPU_DI static void warm_start(const BodyState* b, PR p, AR a, Velocity* v) {
        V3 swivelAxis, hingeAxis;
        V3 j = jacobian(p, b[0].q, b[1].q, swivelAxis, hingeAxis);
        angular1_apply(transform(j, b[0].inertia.t), transform(j, b[1].inertia.t), ldacc(a, 0), v[0].ang, v[1].ang);
    }
    template <class PR, class AR> BEPU_DI static void solve(const BodyState* b, float dt, float, PR p, AR a, Velocity* v) {
        V3 swivelAxis, hingeAxis;
        V3 j = jacobian(p, b[0].q, b[1].q, swivelAxis, hingeAxis);
        V3 i2vA = transform(j, b[0].inertia.t), ni2vB = transform(j, b[1].inertia.t);
        float angularA = dot(i2vA, j), angularB = dot(ni2vB, j);
        Springiness sp = compute_springiness(ldrow(p, 6), ldrow(p, 7), dt);
        float effectiveMass = sp.effective_mass_cfm_scale / (angularA + angularB);
        float error = dot(hingeAxis, swivelAxis);
        float biasVelocity = -(sp.position_error_to_velocity * error);
        float csv = dot(v[0].ang - v[1].ang, j);
        float acc = ldacc(a, 0);
        float csi = effectiveMass * (biasVelocity - csv) - acc * sp.softness_impulse_scale;
        acc = acc + csi;
        angular1_apply(i2vA, ni2vB, csi, v[0].ang, v[1].ang);
        stacc(a, 0, acc);
    }
};

// ---- TwistMotor (28): TwistMotor.cs:L77-126 ----
// prestep: LocalAxisA xyz, LocalAxisB xyz, TargetVelocity, MaximumForce, Damping | impulse: 1
struct TwistMotor {
    static constexpr int kBodies = 2, kPrestepRows = 9, kImpulseRows = 1;
    static constexpr bool kIncremental = false, kNeedsPose = true;
    BEPU_DI static V3 jacobian(Q4 qA, Q4 qB, V3 localAxisA, V3 localAxisB) {  // L79-89
        V3 axisA = transform(localAxisA, qA), axisB = transform(localAxisB, qB);
        V3 j = axisA + axisB;
        float len = length(j);
        j = j * (1.0f / len);
        return len < 1e-10f ? axisA : j;
    }
    template <class PR, class AR> BEPU_DI static void warm_start(const BodyState* b, PR p, AR a, Velocity* v) {
        V3 j = jacobian(b[0].q, b[1].q, ldrow3(p, 0), ldrow3(p, 3));
        angular1_apply(transform(j, b[0].inertia.t), transform(j, b[1].inertia.t), ldacc(a, 0), v[0].ang, v[1].ang);
    }
    template <class PR, class AR> BEPU_DI static void solve(const BodyState* b, float dt, float, PR p, AR a, Velocity* v) {
        V3 j = jacobian(b[0].q, b[1].q, ldrow3(p, 0), ldrow3(p, 3));
        V3 i2vA = transform(j, b[0].inertia.t), ni2vB = transform(j, b[1].inertia.t);  // TwistServo.cs:L133-144
        float unsoftenedInverseEffectiveMass = dot(i2vA, j) + dot(ni2vB, j);
        MotorSoftness m = motor_softness(ldrow(p, 7), ldrow(p, 8), dt);
        float effectiveMass = m.effective_mass_cfm_scale / unsoftenedInverseEffectiveMass;
        V3 velocityToImpulseA = j * effectiveMass;
        float biasImpulse = ldrow(p, 6) * effectiveMass;
        float csiVelocityComponent = dot(v[0].ang - v[1].ang, velocityToImpulseA);
        float acc = ldacc(a, 0);
        float csi = biasImpulse - acc * m.softness_impulse_scale - csiVelocityComponent;
        float previous = acc;
        acc = fmax_ps(fmin_ps(acc + csi, m.maximum_impulse), -m.maximum_impulse);
        csi = acc - previous;
        angular1_apply(i2vA, ni2vB, csi, v[0].ang, v[1].ang);
        stacc(a, 0, acc);
    }
};

// ---- AngularAxisMotor (41): AngularAxisMotor.cs:L69-106 ----
// prestep: LocalAxisA xyz, TargetVelocity, MaximumForce, Damping | impulse: 1
struct AngularAxisMotor {
    static constexpr int kBodies = 2, kPrestepRows = 6, kImpulseRows = 1;
    static constexpr bool kIncremental = false, kNeedsPose = true;
    template <class PR, class AR> BEPU_DI static void warm_start(const BodyState* b, PR p, AR a, Velocity* v) {
        V3 axis = transform(ldrow3(p, 0), b[0].q);
        angular1_apply(transform(axis, b[0].inertia.t), transform(axis, b[1].inertia.t), ldacc(a, 0), v[0].ang, v[1].ang);
    }
    template <class PR, class AR> BEPU_DI static void solve(const BodyState* b, float dt, float, PR p, AR a, Velocity* v) {
        V3 jA = transform(ldrow3(p, 0), b[0].q);
        V3 jIA = transform(jA, b[0].inertia.t);
        float contributionA = dot(jA, jIA);
        V3 jIB = transform(jA, b[1].inertia.t);
        float contributionB = dot(jA, jIB);
        MotorSoftness m = motor_softness(ldrow(p, 4), ldrow(p, 5), dt);
        float acc = ldacc(a, 0);
        float csi = (ldrow(p, 3) + dot(v[1].ang, jA) - dot(v[0].ang, jA)) * m.effective_mass_cfm_scale / (contributionA + contributionB) - acc * m.softness_impulse_scale;
        servo_clamp_impulse1(m.maximum_impulse, acc, csi);
        angular1_apply(jIA, jIB, csi, v[0].ang, v[1].ang);
        stacc(a, 0, acc);
    }
};

// ---- AngularAxisGearMotor (54): AngularAxisGearMotor.cs:L70-114 ----
// prestep: LocalAxisA xyz, VelocityScale, MaximumForce, Damping | impulse: 1
// Reference behaviour reproduced as written: Solve's final ApplyImpulse (L112) is given the clamped ACCUMULATED impulse, not the corrective impulse.
struct AngularAxisGearMotor {
    static constexpr int kBodies = 2, kPrestepRows = 6, kImpulseRows = 1;
    static constexpr bool kIncremental = false, kNeedsPose = true;
    template <class PR, class AR> BEPU_DI static void warm_start(const BodyState* b, PR p, AR a, Velocity* v) {
        V3 axis = transform(ldrow3(p, 0), b[0].q);
        V3 jA = axis * ldrow(p, 3);
        angular1_apply(transform(jA, b[0].inertia.t), transform(axis, b[1].inertia.t), ldacc(a, 0), v[0].ang, v[1].ang);
    }
    template <class PR, class AR> BEPU_DI static void solve(const BodyState* b, float dt, float, PR p, AR a, Velocity* v) {
        V3 axis = transform(ldrow3(p, 0), b[0].q);
        V3 jA = axis * ldrow(p, 3);
        V3 i2vA = transform(jA, b[0].inertia.t);
        float contributionA = dot(jA, i2vA);
        V3 ni2vB = transform(axis, b[1].inertia.t);
        float contributionB = dot(axis, ni2vB);
        MotorSoftness m = motor_softness(ldrow(p, 4), ldrow(p, 5), dt);
        float effectiveMass = m.effective_mass_cfm_scale / (contributionA + contributionB);
        float unscaledCSVA = dot(v[0].ang, jA);
        float negatedCSVB = dot(v[1].ang, axis);
        float acc = ldacc(a, 0);
        float csi = (negatedCSVB - unscaledCSVA) * effectiveMass - acc * m.softness_impulse_scale;
        servo_clamp_impulse1(m.maximum_impulse, acc, csi);
        angular1_apply(i2vA, ni2vB, acc, v[0].ang, v[1].ang);
        stacc(a, 0, acc);
    }
};

// ---- BallSocketMotor (52) / BallSocketServo (53): BallSocketMotor.cs:L68-97, BallSocketServo.cs:L75-107, BallSocketShared.cs ----
BEPU_DI Sym3 ball_socket_effective_mass(const Inertia& iA, const Inertia& iB, V3 offsetA, V3 offsetB, float effectiveMassCFMScale) {  // BallSocketShared.cs:L10-26
    Sym3 inverseEffectiveMass = skew_sandwich(offsetA, iA.t) + skew_sandwich(offsetB, iB.t);
    float linearContribution = iA.inv_mass + iB.inv_mass;
    inverseEffectiveMass.xx += linearContribution;
    inverseEffectiveMass.yy += linearContribution;
    inverseEffectiveMass.zz += linearContribution;
    return invert(inverseEffectiveMass) * effectiveMassCFMScale;
}
BEPU_DI void ball_socket_solve_clamped(Velocity& vA, Velocity& vB, V3 offsetA, V3 offsetB, V3 biasVelocity, Sym3 effectiveMass, float soft, float maximumImpulse, V3& acc,
                                       const Inertia& iA, const Inertia& iB) {  // BallSocketShared.cs:L47-62, L126-134
    V3 csv = vA.lin - vB.lin;
    csv = csv + cross(vA.ang, offsetA);
    csv = csv + cross(offsetB, vB.ang);
    csv = biasVelocity - csv;
    V3 corrective = transform(csv, effectiveMass) - acc * soft;
    servo_clamp_impulse3(maximumImpulse, acc, corrective);
    ball_socket_apply(vA, vB, offsetA, offsetB, iA, iB, corrective);
}
// prestep: LocalOffsetB xyz, TargetVelocityLocalA xyz, MaximumForce, Damping | impulses: xyz
struct BallSocketMotor {
    static constexpr int kBodies = 2, kPrestepRows = 8, kImpulseRows = 3;
    static constexpr bool kIncremental = false, kNeedsPose = true;
    template <class PR, class AR> BEPU_DI static void warm_start(const BodyState* b, PR p, AR a, Velocity* v) {
        V3 targetOffsetB = transform(ldrow3(p, 0), b[1].q);
        ball_socket_apply(v[0], v[1], (b[1].pos - b[0].pos) + targetOffsetB, targetOffsetB, b[0].inertia, b[1].inertia, V3{ldacc(a, 0), ldacc(a, 1), ldacc(a, 2)});
    }
    template <class PR, class AR> BEPU_DI static void solve(const BodyState* b, float dt, float, PR p, AR a, Velocity* v) {
        V3 targetOffsetB = transform(ldrow3(p, 0), b[1].q);
        V3 offsetA = (b[1].pos - b[0].pos) + targetOffsetB;
        MotorSoftness m = motor_softness(ldrow(p, 6), ldrow(p, 7), dt);
        Sym3 effectiveMass = ball_socket_effective_mass(b[0].inertia, b[1].inertia, offsetA, targetOffsetB, m.effective_mass_cfm_scale);
        V3 biasVelocity = -transform(ldrow3(p, 3), b[0].q);
        V3 acc{ldacc(a, 0), ldacc(a, 1), ldacc(a, 2)};
        ball_socket_solve_clamped(v[0], v[1], offsetA, targetOffsetB, biasVelocity, effectiveMass, m.softness_impulse_scale, m.maximum_impulse, acc, b[0].inertia, b[1].inertia);
        stacc(a, 0, acc.x); stacc(a, 1, acc.y); stacc(a, 2, acc.z);
    }
};
// prestep: LocalOffsetA xyz, LocalOffsetB xyz, AngularFrequency, TwiceDampingRatio, MaximumSpeed, BaseSpeed, MaximumForce | impulses: xyz
struct BallSocketServo {
    static constexpr int kBodies = 2, kPrestepRows = 11, kImpulseRows = 3;
    static constexpr bool kIncremental = false, kNeedsPose = true;
    template <class PR, class AR> BEPU_DI static void warm_start(const BodyState* b, PR p, AR a, Velocity* v) {
        V3 offsetA = transform(ldrow3(p, 0), b[0].q), offsetB = transform(ldrow3(p, 3), b[1].q);
        ball_socket_apply(v[0], v[1], offsetA, offsetB, b[0].inertia, b[1].inertia, V3{ldacc(a, 0), ldacc(a, 1), ldacc(a, 2)});
    }
    template <class PR, class AR> BEPU_DI static void solve(const BodyState* b, float dt, float inverseDt, PR p, AR a, Velocity* v) {
        V3 offsetA = transform(ldrow3(p, 0), b[0].q), offsetB = transform(ldrow3(p, 3), b[1].q);
        Springiness sp = compute_springiness(ldrow(p, 6), ldrow(p, 7), dt);
        Sym3 effectiveMass = ball_socket_effective_mass(b[0].inertia, b[1].inertia, offsetA, offsetB, sp.effective_mass_cfm_scale);
        V3 error = ((b[1].pos - b[0].pos) + offsetB) - offsetA;
        V3 biasVelocity = servo_clamped_bias_velocity3e(error, sp.position_error_to_velocity, ldrow(p, 8), ldrow(p, 9), inverseDt);
        float maximumImpulse = ldrow(p, 10) * dt;
        V3 acc{ldacc(a, 0), ldacc(a, 1), ldacc(a, 2)};
        ball_socket_solve_clamped(v[0], v[1], offsetA, offsetB, biasVelocity, effectiveMass, sp.softness_impulse_scale, maximumImpulse, acc, b[0].inertia, b[1].inertia);
        stacc(a, 0, acc.x); stacc(a, 1, acc.y); stacc(a, 2, acc.z);
    }
};

// ---- DistanceServo (33): DistanceServo.cs:L107-226 ----
// prestep: LocalOffsetA xyz, LocalOffsetB xyz, TargetDistance, MaximumSpeed, BaseSpeed, MaximumForce, AngularFrequency, TwiceDampingRatio | impulse: 1
struct DistanceServo {
    static constexpr int kBodies = 2, kPrestepRows = 12, kImpulseRows = 1;
    static constexpr bool kIncremental = false, kNeedsPose = true;
    struct Frame { V3 anchorOffsetA, anchorOffsetB, direction, angularJA, angularJB; float distance; };
    template <class PR> BEPU_DI static Frame frame(const BodyState* b, PR p) {  // GetDistance L109-117 + ComputeJacobian L119-130
        Frame f;
        f.anchorOffsetA = transform(ldrow3(p, 0), b[0].q);
        f.anchorOffsetB = transform(ldrow3(p, 3), b[1].q);
        V3 anchorB = f.anchorOffsetB + (b[1].pos - b[0].pos);
        V3 anchorOffset = anchorB - f.anchorOffsetA;
        f.distance = length(anchorOffset);
        f.direction = anchorOffset * (1.0f / f.distance);
        if (f.distance < 1e-9f) f.direction = V3{1.0f, 0.0f, 0.0f};
        f.angularJA = cross(f.anchorOffsetA, f.direction);
        f.angularJB = cross(f.direction, f.anchorOffsetB);
        return f;
    }
    BEPU_DI static void apply(float imA, float imB, V3 direction, V3 ai2vA, V3 ai2vB, float csi, Velocity& vA, Velocity& vB) {  // L160-183
        vA.lin = direction * (csi * imA) + vA.lin;
        vA.ang = ai2vA * csi + vA.ang;
        vB.lin = vB.lin - direction * (csi * imB);
        vB.ang = ai2vB * csi + vB.ang;
    }
    template <class PR, class AR> BEPU_DI static void warm_start(const BodyState* b, PR p, AR a, Velocity* v) {
        Frame f = frame(b, p);
        apply(b[0].inertia.inv_mass, b[1].inertia.inv_mass, f.direction, transform(f.angularJA, b[0].inertia.t), transform(f.angularJB, b[1].inertia.t), ldacc(a, 0), v[0], v[1]);
    }
    template <class PR, class AR> BEPU_DI static void solve(const BodyState* b, float dt, float inverseDt, PR p, AR a, Velocity* v) {
        Frame f = frame(b, p);
        V3 ai2vA = transform(f.angularJA, b[0].inertia.t), ai2vB = transform(f.angularJB, b[1].inertia.t);  // ComputeTransforms L132-158
        float angularContributionA = dot(f.angularJA, ai2vA), angularContributionB = dot(f.angularJB, ai2vB);
        float inverseEffectiveMass = b[0].inertia.inv_mass + b[1].inertia.inv_mass + angularContributionA + angularContributionB;
        Springiness sp = compute_springiness(ldrow(p, 10), ldrow(p, 11), dt);
        float effectiveMass = sp.effective_mass_cfm_scale / inverseEffectiveMass;
        float error = f.distance - ldrow(p, 6);
        float clampedBiasVelocity = servo_clamped_bias_velocity(error, sp.position_error_to_velocity, ldrow(p, 7), ldrow(p, 8), inverseDt);
        float maximumImpulse = ldrow(p, 9) * dt;
        float linearCSVA = dot(v[0].lin, f.direction), negatedLinearCSVB = dot(v[1].lin, f.direction);
        float angularCSVA = dot(v[0].ang, f.angularJA), angularCSVB = dot(v[1].ang, f.angularJB);
        float acc = ldacc(a, 0);
        float csi = (clampedBiasVelocity - linearCSVA - angularCSVA + negatedLinearCSVB - angularCSVB) * effectiveMass - acc * sp.softness_impulse_scale;
        servo_clamp_impulse1(maximumImpulse, acc, csi);
        apply(b[0].inertia.inv_mass, b[1].inertia.inv_mass, f.direction, ai2vA, ai2vB, csi, v[0], v[1]);
        stacc(a, 0, acc);
    }
};

// ---- DistanceLimit (34): DistanceLimit.cs:L103-181 ----
// prestep: LocalOffsetA xyz, LocalOffsetB xyz, MinimumDistance, MaximumDistance, AngularFrequency, TwiceDampingRatio | impulse: 1
struct DistanceLimit {
    static constexpr int kBodies = 2, kPrestepRows = 10, kImpulseRows = 1;
    static constexpr bool kIncremental = false, kNeedsPose = true;
    struct Frame { V3 direction, angularJA, angularJB; float distance; bool useMinimum; };
    template <class PR> BEPU_DI static Frame frame(const BodyState* b, PR p) {  // L116-139
        Frame f;
        V3 offsetA = transform(ldrow3(p, 0), b[0].q), offsetB = transform(ldrow3(p, 3), b[1].q);
        V3 anchorOffset = (offsetB - offsetA) + (b[1].pos - b[0].pos);
        f.distance = length(anchorOffset);
        f.useMinimum = fabsf(f.distance - ldrow(p, 6)) < fabsf(f.distance - ldrow(p, 7));
        float sign = f.useMinimum ? -1.0f : 1.0f;
        f.direction = anchorOffset * (sign / f.distance);
        if (f.distance < 1e-9f) f.direction = V3{1.0f, 0.0f, 0.0f};
        f.angularJA = cross(offsetA, f.direction);
        f.angularJB = cross(f.direction, offsetB);
        return f;
    }
    BEPU_DI static void apply(V3 linearJA, V3 angularJA, V3 angularJB, const Inertia& iA, const Inertia& iB, float csi, Velocity& vA, Velocity& vB) {  // L105-114
        V3 impulseScaledLinearJacobian = linearJA * csi;
        vA.lin = vA.lin + impulseScaledLinearJacobian * iA.inv_mass;
        vB.lin = vB.lin - impulseScaledLinearJacobian * iB.inv_mass;
        vA.ang = vA.ang + transform(angularJA * csi, iA.t);
        vB.ang = vB.ang + transform(angularJB * csi, iB.t);
    }
    template <class PR, class AR> BEPU_DI static void warm_start(const BodyState* b, PR p, AR a, Velocity* v) {
        Frame f = frame(b, p);
        apply(f.direction, f.angularJA, f.angularJB, b[0].inertia, b[1].inertia, ldacc(a, 0), v[0], v[1]);
    }
    template <class PR, class AR> BEPU_DI static void solve(const BodyState* b, float dt, float inverseDt, PR p, AR a, Velocity* v) {
        Frame f = frame(b, p);
        float linearCSVA = dot(v[0].lin, f.direction), negatedLinearCSVB = dot(v[1].lin, f.direction);
        float angularCSVA = dot(v[0].ang, f.angularJA), angularCSVB = dot(v[1].ang, f.angularJB);
        float csv = linearCSVA - negatedLinearCSVB + angularCSVA + angularCSVB;
        float angularContributionA = vector_sandwich(f.angularJA, b[0].inertia.t), angularContributionB = vector_sandwich(f.angularJB, b[1].inertia.t);
        float inverseEffectiveMass = b[0].inertia.inv_mass + b[1].inertia.inv_mass + angularContributionA + angularContributionB;
        Springiness sp = compute_springiness(ldrow(p, 8), ldrow(p, 9), dt);
        float effectiveMass = sp.effective_mass_cfm_scale / inverseEffectiveMass;
        float error = f.useMinimum ? ldrow(p, 6) - f.distance : f.distance - ldrow(p, 7);
        float biasVelocity = inequality_bias_velocity(error, sp.position_error_to_velocity, inverseDt);
        float acc = ldacc(a, 0);
        float csi = -acc * sp.softness_impulse_scale - effectiveMass * (csv - biasVelocity);
        clamp_positive(acc, csi);
        apply(f.direction, f.angularJA, f.angularJB, b[0].inertia, b[1].inertia, csi, v[0], v[1]);
        stacc(a, 0, acc);
    }
};

// ---- PointOnLineServo (37): PointOnLineServo.cs:L82-193 ----
// prestep: LocalOffsetA xyz, LocalOffsetB xyz, LocalDirection xyz, MaximumSpeed, BaseSpeed, MaximumForce, AngularFrequency, TwiceDampingRatio | impulses: xy
struct PointOnLineServo {
    static constexpr int kBodies = 2, kPrestepRows = 14, kImpulseRows = 2;
    static constexpr bool kIncremental = false, kNeedsPose = true;
    struct Frame { V3 anchorOffset; M23 linearJacobian, angularJA, angularJB; };
    BEPU_DI static void apply(Velocity& vA, Velocity& vB, const Frame& f, const Inertia& iA, const Inertia& iB, V2 csi) {  // L84-101
        V3 linearImpulseA = transform(csi, f.linearJacobian);
        V3 angularImpulseA = transform(csi, f.angularJA);
        V3 angularImpulseB = transform(csi, f.angularJB);
        V3 angularChangeA = transform(angularImpulseA, iA.t), angularChangeB = transform(angularImpulseB, iB.t);
        V3 linearChangeA = linearImpulseA * iA.inv_mass, negatedLinearChangeB = linearImpulseA * iB.inv_mass;
        vA.lin = linearChangeA + vA.lin;
        vA.ang = angularChangeA + vA.ang;
        vB.lin = vB.lin - negatedLinearChangeB;
        vB.ang = angularChangeB + vB.ang;
    }
    template <class PR> BEPU_DI static Frame frame(const BodyState* b, PR p) {  // L103-126
        Frame f;
        V3 localDirection = ldrow3(p, 6);
        V3 localTangentX, localTangentY;
        build_orthonormal_basis(localDirection, localTangentX, localTangentY);
        M33 mA = matrix_from_quaternion(b[0].q);
        V3 anchorA = transform(ldrow3(p, 0), mA);
        V3 offsetB = transform(ldrow3(p, 3), b[1].q);
        V3 direction = transform(localDirection, mA);
        V3 anchorB = offsetB + (b[1].pos - b[0].pos);
        f.anchorOffset = anchorB - anchorA;
        float d = dot(f.anchorOffset, direction);
        V3 offsetA = direction * d + anchorA;
        f.linearJacobian.x = transform(localTangentX, mA);
        f.linearJacobian.y = transform(localTangentY, mA);
        f.angularJA.x = cross(offsetA, f.linearJacobian.x);
        f.angularJA.y = cross(offsetA, f.linearJacobian.y);
        f.angularJB.x = cross(f.linearJacobian.x, offsetB);
        f.angularJB.y = cross(f.linearJacobian.y, offsetB);
        return f;
    }
    template <class PR, class AR> BEPU_DI static void warm_start(const BodyState* b, PR p, AR a, Velocity* v) {
        Frame f = frame(b, p);
        apply(v[0], v[1], f, b[0].inertia, b[1].inertia, V2{ldacc(a, 0), ldacc(a, 1)});
    }
    template <class PR, class AR> BEPU_DI static void solve(const BodyState* b, float dt, float inverseDt, PR p, AR a, Velocity* v) {
        Frame f = frame(b, p);
        Sym2 linearContribution = sandwich_scale(f.linearJacobian, b[0].inertia.inv_mass + b[1].inertia.inv_mass);
        Sym2 inverseEffectiveMass = matrix_sandwich(f.angularJA, b[0].inertia.t) + matrix_sandwich(f.angularJB, b[1].inertia.t);
        inverseEffectiveMass = inverseEffectiveMass + linearContribution;
        Sym2 effectiveMass = invert(inverseEffectiveMass);
        Springiness sp = compute_springiness(ldrow(p, 12), ldrow(p, 13), dt);
        const float cfm = sp.effective_mass_cfm_scale;
        effectiveMass = Sym2{effectiveMass.xx * cfm, effectiveMass.yx * cfm, effectiveMass.yy * cfm};
        V2 linearCSV = transform_by_transpose(v[0].lin, f.linearJacobian) - transform_by_transpose(v[1].lin, f.linearJacobian);
        V2 angularCSV = transform_by_transpose(v[0].ang, f.angularJA) + transform_by_transpose(v[1].ang, f.angularJB);
        V2 csv = linearCSV + angularCSV;
        V2 error{dot(f.anchorOffset, f.linearJacobian.x), dot(f.anchorOffset, f.linearJacobian.y)};
        V2 biasVelocity = servo_clamped_bias_velocity2e(error, sp.position_error_to_velocity, ldrow(p, 9), ldrow(p, 10), inverseDt);
        float maximumImpulse = ldrow(p, 11) * dt;
        csv = biasVelocity - csv;
        V2 csi = transform(csv, effectiveMass);
        V2 acc{ldacc(a, 0), ldacc(a, 1)};
        csi = csi - acc * sp.softness_impulse_scale;
        servo_clamp_impulse2(maximumImpulse, acc, csi);
        apply(v[0], v[1], f, b[0].inertia, b[1].inertia, csi);
        stacc(a, 0, acc.x); stacc(a, 1, acc.y);
    }
};

// ---- LinearAxis family: LinearAxisServo.cs:L173-248, LinearAxisMotor.cs:L82-110, LinearAxisLimit.cs:L90-151 ----
struct LinearAxisFrame { V3 normal, angularJA, angularJB; float planeNormalDot; };
BEPU_DI void linear_axis_apply(V3 linearJA, V3 ai2vA, V3 ai2vB, const Inertia& iA, const Inertia& iB, float csi, Velocity& vA, Velocity& vB) {  // LinearAxisServo.cs:L173-180
    vA.lin = vA.lin + linearJA * (csi * iA.inv_mass);
    vB.lin = vB.lin - linearJA * (csi * iB.inv_mass);
    vA.ang = vA.ang + ai2vA * csi;
    vB.ang = vB.ang + ai2vB * csi;
}
template <class PR> BEPU_DI LinearAxisFrame linear_axis_frame(const BodyState* b, PR p) {  // LinearAxisServo.cs:L182-197
    LinearAxisFrame f;
    M33 mA = matrix_from_quaternion(b[0].q);
    f.normal = transform(ldrow3(p, 6), mA);
    V3 anchorA = transform(ldrow3(p, 0), mA);
    V3 offsetB = transform(ldrow3(p, 3), b[1].q);
    V3 anchorB = (b[1].pos - b[0].pos) + offsetB;
    f.planeNormalDot = dot(anchorB - anchorA, f.normal);
    V3 offsetFromAToClosestPointOnPlaneToB = anchorB - f.normal * f.planeNormalDot;
    f.angularJA = cross(offsetFromAToClosestPointOnPlaneToB, f.normal);
    f.angularJB = cross(f.normal, offsetB);
    return f;
}
BEPU_DI float linear_axis_effective_mass(const LinearAxisFrame& f, const Inertia& iA, const Inertia& iB, float cfm, V3& ai2vA, V3& ai2vB) {  // L199-209
    ai2vA = transform(f.angularJA, iA.t);
    ai2vB = transform(f.angularJB, iB.t);
    float angularContributionA = dot(f.angularJA, ai2vA), angularContributionB = dot(f.angularJB, ai2vB);
    return cfm / (iA.inv_mass + iB.inv_mass + angularContributionA + angularContributionB);
}
BEPU_DI float linear_axis_csv(const Velocity* v, const LinearAxisFrame& f) { return dot(v[0].lin - v[1].lin, f.normal) + dot(v[0].ang, f.angularJA) + dot(v[1].ang, f.angularJB); }
template <class AR> BEPU_DI void linear_axis_warm_start(const LinearAxisFrame& f, const BodyState* b, AR a, Velocity* v) {
    linear_axis_apply(f.normal, transform(f.angularJA, b[0].inertia.t), transform(f.angularJB, b[1].inertia.t), b[0].inertia, b[1].inertia, ldacc(a, 0), v[0], v[1]);
}
// prestep: LocalOffsetA xyz, LocalOffsetB xyz, LocalPlaneNormal xyz, TargetOffset, MaximumSpeed, BaseSpeed, MaximumForce, AngularFrequency, TwiceDampingRatio | impulse: 1
struct LinearAxisServo {
    static constexpr int kBodies = 2, kPrestepRows = 15, kImpulseRows = 1;
    static constexpr bool kIncremental = false, kNeedsPose = true;
    template <class PR, class AR> BEPU_DI static void warm_start(const BodyState* b, PR p, AR a, Velocity* v) { linear_axis_warm_start(linear_axis_frame(b, p), b, a, v); }
    template <class PR, class AR> BEPU_DI static void solve(const BodyState* b, float dt, float inverseDt, PR p, AR a, Velocity* v) {
        LinearAxisFrame f = linear_axis_frame(b, p);
        Springiness sp = compute_springiness(ldrow(p, 13), ldrow(p, 14), dt);
        V3 ai2vA, ai2vB;
        float effectiveMass = linear_axis_effective_mass(f, b[0].inertia, b[1].inertia, sp.effective_mass_cfm_scale, ai2vA, ai2vB);
        float biasVelocity = servo_clamped_bias_velocity(f.planeNormalDot - ldrow(p, 9), sp.position_error_to_velocity, ldrow(p, 10), ldrow(p, 11), inverseDt);
        float maximumImpulse = ldrow(p, 12) * dt;
        float csv = linear_axis_csv(v, f);
        float acc = ldacc(a, 0);
        float csi = effectiveMass * (biasVelocity - csv) - acc * sp.softness_impulse_scale;
        servo_clamp_impulse1(maximumImpulse, acc, csi);
        linear_axis_apply(f.normal, ai2vA, ai2vB, b[0].inertia, b[1].inertia, csi, v[0], v[1]);
        stacc(a, 0, acc);
    }
};
// prestep: LocalOffsetA xyz, LocalOffsetB xyz, LocalPlaneNormal xyz, TargetVelocity, MaximumForce, Damping | impulse: 1
struct LinearAxisMotor {
    static constexpr int kBodies = 2, kPrestepRows = 12, kImpulseRows = 1;
    static constexpr bool kIncremental = false, kNeedsPose = true;
    template <class PR, class AR> BEPU_DI static void warm_start(const BodyState* b, PR p, AR a, Velocity* v) { linear_axis_warm_start(linear_axis_frame(b, p), b, a, v); }
    template <class PR, class AR> BEPU_DI static void solve(const BodyState* b, float dt, float, PR p, AR a, Velocity* v) {
        LinearAxisFrame f = linear_axis_frame(b, p);
        MotorSoftness m = motor_softness(ldrow(p, 10), ldrow(p, 11), dt);
        V3 ai2vA, ai2vB;
        float effectiveMass = linear_axis_effective_mass(f, b[0].inertia, b[1].inertia, m.effective_mass_cfm_scale, ai2vA, ai2vB);
        float csv = linear_axis_csv(v, f);
        float acc = ldacc(a, 0);
        float csi = effectiveMass * (-ldrow(p, 9) - csv) - acc * m.softness_impulse_scale;
        servo_clamp_impulse1(m.maximum_impulse, acc, csi);
        linear_axis_apply(f.normal, ai2vA, ai2vB, b[0].inertia, b[1].inertia, csi, v[0], v[1]);
        stacc(a, 0, acc);
    }
};
// prestep: LocalOffsetA xyz, LocalOffsetB xyz, LocalPlaneNormal xyz, MinimumOffset, MaximumOffset, AngularFrequency, TwiceDampingRatio | impulse: 1
struct LinearAxisLimit {
    static constexpr int kBodies = 2, kPrestepRows = 13, kImpulseRows = 1;
    static constexpr bool kIncremental = false, kNeedsPose = true;
    template <class PR> BEPU_DI static LinearAxisFrame frame(const BodyState* b, PR p, float& error) {  // LinearAxisLimit.cs:L92-119
        LinearAxisFrame f;
        M33 mA = matrix_from_quaternion(b[0].q);
        f.normal = transform(ldrow3(p, 6), mA);
        V3 anchorA = transform(ldrow3(p, 0), mA);
        V3 offsetB = transform(ldrow3(p, 3), b[1].q);
        V3 anchorB = (b[1].pos - b[0].pos) + offsetB;
        f.planeNormalDot = dot(anchorB - anchorA, f.normal);
        float minimumError = ldrow(p, 9) - f.planeNormalDot;
        float maximumError = f.planeNormalDot - ldrow(p, 10);
        bool useMin = fabsf(minimumError) < fabsf(maximumError);
        error = useMin ? minimumError : maximumError;
        if (useMin) f.normal = -f.normal;
        V3 offsetFromAToClosestPointOnPlaneToB = anchorB - f.normal * f.planeNormalDot;
        f.angularJA = cross(offsetFromAToClosestPointOnPlaneToB, f.normal);
        f.angularJB = cross(f.normal, offsetB);
        return f;
    }
    template <class PR, class AR> BEPU_DI static void warm_start(const BodyState* b, PR p, AR a, Velocity* v) {
        float error;
        linear_axis_warm_start(frame(b, p, error), b, a, v);
    }
    template <class PR, class AR> BEPU_DI static void solve(const BodyState* b, float dt, float inverseDt, PR p, AR a, Velocity* v) {
        float error;
        LinearAxisFrame f = frame(b, p, error);
        Springiness sp = compute_springiness(ldrow(p, 11), ldrow(p, 12), dt);
        V3 ai2vA, ai2vB;
        float effectiveMass = linear_axis_effective_mass(f, b[0].inertia, b[1].inertia, sp.effective_mass_cfm_scale, ai2vA, ai2vB);
        float biasVelocity = inequality_bias_velocity(error, sp.position_error_to_velocity, inverseDt);
        float csv = linear_axis_csv(v, f);
        float acc = ldacc(a, 0);
        float csi = effectiveMass * (biasVelocity - csv) - acc * sp.softness_impulse_scale;
        clamp_positive(acc, csi);
        linear_axis_apply(f.normal, ai2vA, ai2vB, b[0].inertia, b[1].inertia, csi, v[0], v[1]);
        stacc(a, 0, acc);
    }
};

// ---- CenterDistanceConstraint (35) / CenterDistanceLimit (55): CenterDistanceConstraint.cs:L69-133, CenterDistanceLimit.cs:L78-132 ----
BEPU_DI void center_distance_apply(V3 jacobianA, float imA, float imB, float impulse, Velocity& a, Velocity& b) {  // L71-80
    a.lin = a.lin + jacobianA * (impulse * imA);
    b.lin = b.lin - jacobianA * (impulse * imB);
}
// prestep: TargetDistance, AngularFrequency, TwiceDampingRatio | impulse: 1
struct CenterDistanceConstraint {
    static constexpr int kBodies = 2, kPrestepRows = 3, kImpulseRows = 1;
    static constexpr bool kIncremental = false, kNeedsPose = true;
    template <class PR, class AR> BEPU_DI static void warm_start(const BodyState* b, PR, AR a, Velocity* v) {
        V3 ab = b[1].pos - b[0].pos;
        float lengthSquared = length_squared(ab);
        float inverseDistance = 1.0f / sqrtf(lengthSquared);
        V3 jacobianA = ab * inverseDistance;
        if (lengthSquared < 1e-10f) jacobianA = V3{1.0f, 0.0f, 0.0f};
        center_distance_apply(jacobianA, b[0].inertia.inv_mass, b[1].inertia.inv_mass, ldacc(a, 0), v[0], v[1]);
    }
    template <class PR, class AR> BEPU_DI static void solve(const BodyState* b, float dt, float, PR p, AR a, Velocity* v) {
        V3 ab = b[1].pos - b[0].pos;
        float distance = length(ab);
        float inverseDistance = 1.0f / distance;
        V3 jacobianA = ab * inverseDistance;
        if (distance < 1e-5f) jacobianA = V3{1.0f, 0.0f, 0.0f};
        Springiness sp = compute_springiness(ldrow(p, 1), ldrow(p, 2), dt);
        float effectiveMass = sp.effective_mass_cfm_scale / (b[0].inertia.inv_mass + b[1].inertia.inv_mass);
        float biasVelocity = (distance - ldrow(p, 0)) * sp.position_error_to_velocity;
        float linearCSVA = dot(v[0].lin, jacobianA), negatedCSVB = dot(v[1].lin, jacobianA);
        float acc = ldacc(a, 0);
        float csi = (biasVelocity - (linearCSVA - negatedCSVB)) * effectiveMass - acc * sp.softness_impulse_scale;
        acc = acc + csi;
        center_distance_apply(jacobianA, b[0].inertia.inv_mass, b[1].inertia.inv_mass, csi, v[0], v[1]);
        stacc(a, 0, acc);
    }
};
// prestep: MinimumDistance, MaximumDistance, AngularFrequency, TwiceDampingRatio | impulse: 1
struct CenterDistanceLimit {
    static constexpr int kBodies = 2, kPrestepRows = 4, kImpulseRows = 1;
    static constexpr bool kIncremental = false, kNeedsPose = true;
    BEPU_DI static V3 jacobian(float minimumDistance, float maximumDistance, V3 pA, V3 pB, float& distance, bool& useMinimum) {  // L80-96
        V3 ab = pB - pA;
        distance = length(ab);
        float inverseDistance = 1.0f / distance;
        V3 jacobianA = ab * inverseDistance;
        if (distance < 1e-5f) jacobianA = V3{1.0f, 0.0f, 0.0f};
        useMinimum = fabsf(distance - minimumDistance) < fabsf(distance - maximumDistance);
        return useMinimum ? -jacobianA : jacobianA;
    }
    template <class PR, class AR> BEPU_DI static void warm_start(const BodyState* b, PR p, AR a, Velocity* v) {
        float distance;
        bool useMinimum;
        V3 jacobianA = jacobian(ldrow(p, 0), ldrow(p, 1), b[0].pos, b[1].pos, distance, useMinimum);
        center_distance_apply(jacobianA, b[0].inertia.inv_mass, b[1].inertia.inv_mass, ldacc(a, 0), v[0], v[1]);
    }
    template <class PR, class AR> BEPU_DI static void solve(const BodyState* b, float dt, float inverseDt, PR p, AR a, Velocity* v) {
        float distance;
        bool useMinimum;
        const float minimumDistance = ldrow(p, 0), maximumDistance = ldrow(p, 1);
        V3 jacobianA = jacobian(minimumDistance, maximumDistance, b[0].pos, b[1].pos, distance, useMinimum);
        Springiness sp = compute_springiness(ldrow(p, 2), ldrow(p, 3), dt);
        float effectiveMass = sp.effective_mass_cfm_scale / (b[0].inertia.inv_mass + b[1].inertia.inv_mass);
        float error = useMinimum ? minimumDistance - distance : distance - maximumDistance;
        float biasVelocity = inequality_bias_velocity(error, sp.position_error_to_velocity, inverseDt);
        float csv = dot(v[0].lin, jacobianA) - dot(v[1].lin, jacobianA);
        float acc = ldacc(a, 0);
        float csi = -acc * sp.softness_impulse_scale - effectiveMass * (csv - biasVelocity);
        clamp_positive(acc, csi);
        center_distance_apply(jacobianA, b[0].inertia.inv_mass, b[1].inertia.inv_mass, csi, v[0], v[1]);
        stacc(a, 0, acc);
    }
};

// ---- one-body joints ----
// OneBodyAngularServo (42): OneBodyAngularServo.cs:L69-109
// prestep: TargetOrientation xyzw, AngularFrequency, TwiceDampingRatio, MaximumSpeed, BaseSpeed, MaximumForce | impulses: xyz
struct OneBodyAngularServo {
    static constexpr int kBodies = 1, kPrestepRows = 9, kImpulseRows = 3;
    static constexpr bool kIncremental = false, kNeedsPose = true;
    template <class PR, class AR> BEPU_DI static void warm_start(const BodyState* b, PR, AR a, Velocity* v) {
        v[0].ang = v[0].ang + transform(V3{ldacc(a, 0), ldacc(a, 1), ldacc(a, 2)}, b[0].inertia.t);
    }
    template <class PR, class AR> BEPU_DI static void solve(const BodyState* b, float dt, float inverseDt, PR p, AR a, Velocity* v) {
        Q4 errorRotation = concatenate(conjugate(b[0].q), ldrow4(p, 0));
        V3 errorAxis;
        float errorLength;
        axis_angle_from_quaternion(errorRotation, errorAxis, errorLength);
        Springiness sp = compute_springiness(ldrow(p, 4), ldrow(p, 5), dt);
        Sym3 effectiveMass = invert(b[0].inertia.t);
        V3 clampedBiasVelocity = servo_clamped_bias_velocity3(errorAxis, errorLength, sp.position_error_to_velocity, ldrow(p, 6), ldrow(p, 7), inverseDt);
        float maximumImpulse = ldrow(p, 8) * dt;
        V3 csv = clampedBiasVelocity - v[0].ang;
        V3 csi = transform(csv, effectiveMass);
        V3 acc{ldacc(a, 0), ldacc(a, 1), ldacc(a, 2)};
        csi = csi * sp.effective_mass_cfm_scale - acc * sp.softness_impulse_scale;
        servo_clamp_impulse3(maximumImpulse, acc, csi);
        v[0].ang = v[0].ang + transform(csi, b[0].inertia.t);
        stacc(a, 0, acc.x); stacc(a, 1, acc.y); stacc(a, 2, acc.z);
    }
};
// OneBodyAngularMotor (43): OneBodyAngularMotor.cs:L61-93
// prestep: TargetVelocity xyz, MaximumForce, Damping | impulses: xyz
struct OneBodyAngularMotor {
    static constexpr int kBodies = 1, kPrestepRows = 5, kImpulseRows = 3;
    static constexpr bool kIncremental = false, kNeedsPose = true;
    template <class PR, class AR> BEPU_DI static void warm_start(const BodyState* b, PR, AR a, Velocity* v) {
        v[0].ang = v[0].ang + transform(V3{ldacc(a, 0), ldacc(a, 1), ldacc(a, 2)}, b[0].inertia.t);
    }
    template <class PR, class AR> BEPU_DI static void solve(const BodyState* b, float dt, float, PR p, AR a, Velocity* v) {
        MotorSoftness m = motor_softness(ldrow(p, 3), ldrow(p, 4), dt);
        Sym3 unsoftenedEffectiveMass = invert(b[0].inertia.t);
        V3 csi = transform(ldrow3(p, 0) - v[0].ang, unsoftenedEffectiveMass);
        V3 acc{ldacc(a, 0), ldacc(a, 1), ldacc(a, 2)};
        csi = csi * m.effective_mass_cfm_scale - acc * m.softness_impulse_scale;
        servo_clamp_impulse3(m.maximum_impulse, acc, csi);
        v[0].ang = v[0].ang + transform(csi, b[0].inertia.t);
        stacc(a, 0, acc.x); stacc(a, 1, acc.y); stacc(a, 2, acc.z);
    }
};
BEPU_DI void one_body_linear_apply(V3 offset, const Inertia& inertia, Velocity& vA, V3 csi) {  // OneBodyLinearServo.cs:L93-105
    vA.ang = vA.ang + transform(cross(offset, csi), inertia.t);
    vA.lin = vA.lin + csi * inertia.inv_mass;
}
BEPU_DI Sym3 one_body_linear_effective_mass(V3 offset, const Inertia& inertia) {
    Sym3 inverseEffectiveMass = skew_sandwich(offset, inertia.t);
    inverseEffectiveMass.xx += inertia.inv_mass;
    inverseEffectiveMass.yy += inertia.inv_mass;
    inverseEffectiveMass.zz += inertia.inv_mass;
    return invert(inverseEffectiveMass);
}
// OneBodyLinearServo (44): OneBodyLinearServo.cs:L77-146
// prestep: LocalOffset xyz, Target xyz, AngularFrequency, TwiceDampingRatio, MaximumSpeed, BaseSpeed, MaximumForce | impulses: xyz
struct OneBodyLinearServo {
    static constexpr int kBodies = 1, kPrestepRows = 11, kImpulseRows = 3;
    static constexpr bool kIncremental = false, kNeedsPose = true;
    template <class PR, class AR> BEPU_DI static void warm_start(const BodyState* b, PR p, AR a, Velocity* v) {
        one_body_linear_apply(transform(ldrow3(p, 0), b[0].q), b[0].inertia, v[0], V3{ldacc(a, 0), ldacc(a, 1), ldacc(a, 2)});
    }
    template <class PR, class AR> BEPU_DI static void solve(const BodyState* b, float dt, float inverseDt, PR p, AR a, Velocity* v) {
        V3 offset = transform(ldrow3(p, 0), b[0].q);
        Springiness sp = compute_springiness(ldrow(p, 6), ldrow(p, 7), dt);
        V3 worldGrabPoint = offset + b[0].pos;
        V3 error = ldrow3(p, 3) - worldGrabPoint;
        V3 biasVelocity = servo_clamped_bias_velocity3e(error, sp.position_error_to_velocity, ldrow(p, 8), ldrow(p, 9), inverseDt);
        float maximumImpulse = ldrow(p, 10) * dt;
        V3 csv = (biasVelocity - cross(v[0].ang, offset)) - v[0].lin;
        Sym3 effectiveMass = one_body_linear_effective_mass(offset, b[0].inertia);
        V3 csi = transform(csv, effectiveMass);
        V3 acc{ldacc(a, 0), ldacc(a, 1), ldacc(a, 2)};
        csi = csi * sp.effective_mass_cfm_scale - acc * sp.softness_impulse_scale;
        servo_clamp_impulse3(maximumImpulse, acc, csi);
        one_body_linear_apply(offset, b[0].inertia, v[0], csi);
        stacc(a, 0, acc.x); stacc(a, 1, acc.y); stacc(a, 2, acc.z);
    }
};
// OneBodyLinearMotor (45): OneBodyLinearMotor.cs:L67-100
// prestep: LocalOffset xyz, TargetVelocity xyz, MaximumForce, Damping | impulses: xyz
struct OneBodyLinearMotor {
    static constexpr int kBodies = 1, kPrestepRows = 8, kImpulseRows = 3;
    static constexpr bool kIncremental = false, kNeedsPose = true;
    template <class PR, class AR> BEPU_DI static void warm_start(const BodyState* b, PR p, AR a, Velocity* v) {
        one_body_linear_apply(transform(ldrow3(p, 0), b[0].q), b[0].inertia, v[0], V3{ldacc(a, 0), ldacc(a, 1), ldacc(a, 2)});
    }
    template <class PR, class AR> BEPU_DI static void solve(const BodyState* b, float dt, float, PR p, AR a, Velocity* v) {
        V3 offset = transform(ldrow3(p, 0), b[0].q);
        MotorSoftness m = motor_softness(ldrow(p, 6), ldrow(p, 7), dt);
        V3 csv = (ldrow3(p, 3) - cross(v[0].ang, offset)) - v[0].lin;
        Sym3 effectiveMass = one_body_linear_effective_mass(offset, b[0].inertia);
        V3 csi = transform(csv, effectiveMass);
        V3 acc{ldacc(a, 0), ldacc(a, 1), ldacc(a, 2)};
        csi = csi * m.effective_mass_cfm_scale - acc * m.softness_impulse_scale;
        servo_clamp_impulse3(m.maximum_impulse, acc, csi);
        one_body_linear_apply(offset, b[0].inertia, v[0], csi);
        stacc(a, 0, acc.x); stacc(a, 1, acc.y); stacc(a, 2, acc.z);
    }
};

// ---- three / four body constraints ----
// AreaConstraint (36): AreaConstraint.cs:L76-197
// prestep: TargetScaledArea, AngularFrequency, TwiceDampingRatio | impulse: 1
struct AreaConstraint {
    static constexpr int kBodies = 3, kPrestepRows = 3, kImpulseRows = 1;
    static constexpr bool kIncremental = false, kNeedsPose = true;
    struct Jacobian { float normalLength, contributionA, contributionB, contributionC, inverseJacobianLength; V3 negatedJacobianA, jacobianB, jacobianC; };
    BEPU_DI static void apply(const BodyState* b, const Jacobian& j, float impulse, Velocity* v) {  // L78-91
        v[0].lin = v[0].lin - j.negatedJacobianA * (b[0].inertia.inv_mass * impulse);
        v[1].lin = v[1].lin + j.jacobianB * (b[1].inertia.inv_mass * impulse);
        v[2].lin = v[2].lin + j.jacobianC * (b[2].inertia.inv_mass * impulse);
    }
    BEPU_DI static Jacobian jacobian(const BodyState* b) {  // L93-138
        Jacobian j;
        V3 ab = b[1].pos - b[0].pos, ac = b[2].pos - b[0].pos;
        V3 abxac = cross(ab, ac);
        j.normalLength = length(abxac);
        V3 normal = abxac * (j.normalLength > 1e-10f ? 1.0f / j.normalLength : 0.0f);
        j.jacobianB = cross(ac, normal);
        j.jacobianC = cross(normal, ab);
        j.negatedJacobianA = j.jacobianB + j.jacobianC;
        j.contributionA = dot(j.negatedJacobianA, j.negatedJacobianA);
        j.contributionB = dot(j.jacobianB, j.jacobianB);
        j.contributionC = dot(j.jacobianC, j.jacobianC);
        float jacobianLengthSquared = j.contributionA + j.contributionB + j.contributionC;
        jacobianLengthSquared = fmax_ps(1e-14f, jacobianLengthSquared);
        j.inverseJacobianLength = 1.0f / sqrtf(jacobianLengthSquared);
        return j;
    }
    template <class PR, class AR> BEPU_DI static void warm_start(const BodyState* b, PR, AR a, Velocity* v) {
        Jacobian j = jacobian(b);
        apply(b, j, j.inverseJacobianLength * ldacc(a, 0), v);
    }
    template <class PR, class AR> BEPU_DI static void solve(const BodyState* b, float dt, float, PR p, AR a, Velocity* v) {
        Jacobian j = jacobian(b);
        float inverseJacobianLengthSquared = j.inverseJacobianLength * j.inverseJacobianLength;
        float inverseEffectiveMass = fmax_ps(
            1e-14f, inverseJacobianLengthSquared * (j.contributionA * b[0].inertia.inv_mass + j.contributionB * b[1].inertia.inv_mass + j.contributionC * b[2].inertia.inv_mass));
        Springiness sp = compute_springiness(ldrow(p, 1), ldrow(p, 2), dt);
        float effectiveMass = sp.effective_mass_cfm_scale / inverseEffectiveMass;
        float biasVelocity = (ldrow(p, 0) - j.normalLength) * j.inverseJacobianLength * sp.position_error_to_velocity;
        float negatedVelocityContributionA = dot(j.negatedJacobianA, v[0].lin);
        float velocityContributionB = dot(j.jacobianB, v[1].lin);
        float velocityContributionC = dot(j.jacobianC, v[2].lin);
        float csv = j.inverseJacobianLength * (velocityContributionB + velocityContributionC - negatedVelocityContributionA);
        float acc = ldacc(a, 0);
        float csi = (biasVelocity - csv) * effectiveMass - acc * sp.softness_impulse_scale;
        acc = acc + csi;
        apply(b, j, j.inverseJacobianLength * csi, v);
        stacc(a, 0, acc);
    }
};
// VolumeConstraint (32): VolumeConstraint.cs:L76-186
// prestep: TargetScaledVolume, AngularFrequency, TwiceDampingRatio | impulse: 1
struct VolumeConstraint {
    static constexpr int kBodies = 4, kPrestepRows = 3, kImpulseRows = 1;
    static constexpr bool kIncremental = false, kNeedsPose = true;
    struct Jacobian { float contributionA, contributionB, contributionC, contributionD, inverseJacobianLength; V3 ad, negatedJA, jacobianB, jacobianC, jacobianD; };
    BEPU_DI static void apply(const BodyState* b, const Jacobian& j, float impulse, Velocity* v) {  // L78-94
        v[0].lin = v[0].lin - j.negatedJA * (b[0].inertia.inv_mass * impulse);
        v[1].lin = v[1].lin + j.jacobianB * (b[1].inertia.inv_mass * impulse);
        v[2].lin = v[2].lin + j.jacobianC * (b[2].inertia.inv_mass * impulse);
        v[3].lin = v[3].lin + j.jacobianD * (b[3].inertia.inv_mass * impulse);
    }
    BEPU_DI static Jacobian jacobian(const BodyState* b) {  // L96-123
        Jacobian j;
        V3 ab = b[1].pos - b[0].pos, ac = b[2].pos - b[0].pos;
        j.ad = b[3].pos - b[0].pos;
        j.jacobianB = cross(ac, j.ad);
        j.jacobianC = cross(j.ad, ab);
        j.jacobianD = cross(ab, ac);
        j.negatedJA = j.jacobianB + j.jacobianC;
        j.negatedJA = j.jacobianD + j.negatedJA;
        j.contributionA = dot(j.negatedJA, j.negatedJA);
        j.contributionB = dot(j.jacobianB, j.jacobianB);
        j.contributionC = dot(j.jacobianC, j.jacobianC);
        j.contributionD = dot(j.jacobianD, j.jacobianD);
        float jacobianLengthSquared = j.contributionA + j.contributionB + j.contributionC + j.contributionD;
        jacobianLengthSquared = fmax_ps(1e-14f, jacobianLengthSquared);
        j.inverseJacobianLength = 1.0f / sqrtf(jacobianLengthSquared);
        return j;
    }
    template <class PR, class AR> BEPU_DI static void warm_start(const BodyState* b, PR, AR a, Velocity* v) {
        Jacobian j = jacobian(b);
        apply(b, j, j.inverseJacobianLength * ldacc(a, 0), v);
    }
    template <class PR, class AR> BEPU_DI static void solve(const BodyState* b, float dt, float, PR p, AR a, Velocity* v) {
        Jacobian j = jacobian(b);
        float inverseJacobianLengthSquared = j.inverseJacobianLength * j.inverseJacobianLength;
        float inverseEffectiveMass = fmax_ps(1e-14f, inverseJacobianLengthSquared * (j.contributionA * b[0].inertia.inv_mass + j.contributionB * b[1].inertia.inv_mass +
                                                                                      j.contributionC * b[2].inertia.inv_mass + j.contributionD * b[3].inertia.inv_mass));
        Springiness sp = compute_springiness(ldrow(p, 1), ldrow(p, 2), dt);
        float effectiveMass = sp.effective_mass_cfm_scale / inverseEffectiveMass;
        float volume = dot(j.jacobianD, j.ad);
        float biasVelocity = (ldrow(p, 0) - volume) * j.inverseJacobianLength * sp.position_error_to_velocity;
        float negatedVelocityContributionA = dot(j.negatedJA, v[0].lin);
        float velocityContributionB = dot(j.jacobianB, v[1].lin);
        float velocityContributionC = dot(j.jacobianC, v[2].lin);
        float velocityContributionD = dot(j.jacobianD, v[3].lin);
        float csv = j.inverseJacobianLength * (velocityContributionB + velocityContributionC + velocityContributionD - negatedVelocityContributionA);
        float acc = ldacc(a, 0);
        float csi = (biasVelocity - csv) * effectiveMass - acc * sp.softness_impulse_scale;
        acc = acc + csi;
        apply(b, j, j.inverseJacobianLength * csi, v);
        stacc(a, 0, acc);
    }
};

#define BEPU_JOINT_TYPES_MORE(X)                                                                                                                     \
    X(23, AngularHinge) X(24, AngularSwivelHinge) X(28, TwistMotor) X(31, Weld) X(32, VolumeConstraint) X(33, DistanceServo) X(34, DistanceLimit)      \
    X(35, CenterDistanceConstraint) X(36, AreaConstraint) X(37, PointOnLineServo) X(38, LinearAxisServo) X(39, LinearAxisMotor) X(40, LinearAxisLimit) \
    X(41, AngularAxisMotor) X(42, OneBodyAngularServo) X(43, OneBodyAngularMotor) X(44, OneBodyLinearServo) X(45, OneBodyLinearMotor)                  \
    X(52, BallSocketMotor) X(53, BallSocketServo) X(54, AngularAxisGearMotor) X(55, CenterDistanceLimit)

// Every build of the device types holds them to the type table the planner sizes the arenas from: each listed struct has its id's bodies and
// rows, and the lists name exactly the table's ids (a duplicate id in the lists is a duplicate case of the type switch).
#define BEPU_CHECK_TYPE(ID, T)                                                                                                                       \
    static_assert(bepucuda::type_row(ID) && bepucuda::type_row(ID)->bodies == T::kBodies && bepucuda::type_row(ID)->prestep_rows == T::kPrestepRows && \
                      bepucuda::type_row(ID)->impulse_rows == T::kImpulseRows,                                                                       \
                  "type " #ID " (" #T "): kBodies, kPrestepRows, kImpulseRows differ from its row of bepu_type_table.h");
BEPU_CONTACT_TYPES(BEPU_CHECK_TYPE)
BEPU_JOINT_TYPES(BEPU_CHECK_TYPE)
BEPU_JOINT_TYPES_MORE(BEPU_CHECK_TYPE)
#undef BEPU_CHECK_TYPE
#define BEPU_COUNT_TYPE(ID, T) +1
static_assert(0 BEPU_CONTACT_TYPES(BEPU_COUNT_TYPE) BEPU_JOINT_TYPES(BEPU_COUNT_TYPE) BEPU_JOINT_TYPES_MORE(BEPU_COUNT_TYPE) == bepucuda::kTypeCount,
              "the device type lists and bepu_type_table.h name different type ids");
#undef BEPU_COUNT_TYPE

}  // namespace BEPU_NS
