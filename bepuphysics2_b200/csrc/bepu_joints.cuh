// Joint / motor / servo / limit constraint functions for the sm_90a solver kernels (one thread = one constraint).
// Every type exposes: kBodies, kPrestepRows, kImpulseRows, kIncremental=false, kNeedsPose=true and
//   warm_start(const BodyState* b, const float* p, const float* a, Velocity* v)
//   solve(const BodyState* b, float dt, float inverseDt, const float* p, float* a, Velocity* v)
// where p / a address this lane's element of prestep / impulse row 0 (row r at [r * 32]).
#pragma once
#include "bepu_contacts.cuh"
#include "bepu_device_math.cuh"

namespace BEPU_NS {

struct V4 { float x, y, z, w; };

// ---- settings helpers ----
struct MotorSoftness { float effective_mass_cfm_scale, softness_impulse_scale, maximum_impulse; };
BEPU_DI MotorSoftness motor_softness(float maximumForce, float damping, float dt) {  // MotorSettings.cs:L70-98
    float dtd = dt * damping;
    MotorSoftness m;
    m.maximum_impulse = maximumForce * dt;
    m.softness_impulse_scale = 1.0f / (dtd + 1.0f);
    m.effective_mass_cfm_scale = dtd * m.softness_impulse_scale;
    return m;
}
BEPU_DI float servo_clamped_bias_velocity(float error, float positionErrorToVelocity, float maximumSpeed, float baseSpeedSetting, float inverseDt) {  // ServoSettings.cs:L75-85
    float baseSpeed = fmin_ps(baseSpeedSetting, fabsf(error) * inverseDt);
    float biasVelocity = error * positionErrorToVelocity;
    return biasVelocity < 0.0f ? fmax_ps(-maximumSpeed, fmin_ps(-baseSpeed, biasVelocity)) : fmin_ps(maximumSpeed, fmax_ps(baseSpeed, biasVelocity));
}
BEPU_DI V3 servo_clamped_bias_velocity3(V3 errorAxis, float errorLength, float positionErrorToBiasVelocity, float maximumSpeed, float baseSpeedSetting, float inverseDt) {  // L116-128
    float baseSpeed = fmin_ps(baseSpeedSetting, errorLength * inverseDt);
    float unclampedBiasSpeed = errorLength * positionErrorToBiasVelocity;
    float targetSpeed = fmax_ps(baseSpeed, unclampedBiasSpeed);
    float scl = fmin_ps(1.0f, maximumSpeed / targetSpeed);
    scl = targetSpeed < 1e-10f ? 1.0f : scl;
    return errorAxis * (scl * unclampedBiasSpeed);
}
BEPU_DI void servo_clamp_impulse3(float maximumImpulse, V3& accumulated, V3& csi) {  // ServoSettings.cs:L167-178
    V3 previous = accumulated;
    accumulated = accumulated + csi;
    float magnitude = length(accumulated);
    float impulseScale = fabsf(magnitude) < 1e-10f ? 1.0f : fmin_ps(maximumImpulse / magnitude, 1.0f);
    accumulated = accumulated * impulseScale;
    csi = accumulated - previous;
}
BEPU_DI void clamp_positive(float& accumulated, float& impulse) {  // InequalityHelpers.cs:L16-21
    float previous = accumulated;
    accumulated = fmax_ps(0.0f, accumulated + impulse);
    impulse = accumulated - previous;
}
BEPU_DI void angular1_apply(V3 impulseToVelocityA, V3 negatedImpulseToVelocityB, float csi, V3& wA, V3& wB) {
    wA = wA + impulseToVelocityA * csi;
    wB = wB - negatedImpulseToVelocityB * csi;
}
BEPU_DI void angular3_apply(V3& wA, V3& wB, Sym3 i2vA, Sym3 ni2vB, V3 csi) {  // AngularServo.cs:L60-66
    wA = wA + transform(csi, i2vA);
    wB = wB - transform(csi, ni2vB);
}


// ---- BallSocket (22): BallSocket.cs:L57-90, BallSocketShared.cs ----
// prestep: LocalOffsetA xyz, LocalOffsetB xyz, AngularFrequency, TwiceDampingRatio | impulses: xyz
BEPU_DI void ball_socket_apply(Velocity& vA, Velocity& vB, V3 offsetA, V3 offsetB, const Inertia& iA, const Inertia& iB, V3 csi) {  // BallSocketShared.cs:L29-45
    vA.ang = vA.ang + transform(cross(offsetA, csi), iA.t);
    vA.lin = vA.lin + csi * iA.inv_mass;
    vB.ang = vB.ang + transform(cross(csi, offsetB), iB.t);
    vB.lin = vB.lin - csi * iB.inv_mass;
}
struct BallSocket {
    static constexpr int kBodies = 2, kPrestepRows = 8, kImpulseRows = 3;
    static constexpr bool kIncremental = false, kNeedsPose = true;
    template <class PR, class AR> BEPU_DI static void warm_start(const BodyState* b, PR p, AR a, Velocity* v) {
        V3 offsetA = transform(ldrow3(p, 0), b[0].q), offsetB = transform(ldrow3(p, 3), b[1].q);
        ball_socket_apply(v[0], v[1], offsetA, offsetB, b[0].inertia, b[1].inertia, V3{ldacc(a, 0), ldacc(a, 1), ldacc(a, 2)});
    }
    template <class PR, class AR> BEPU_DI static void solve(const BodyState* b, float dt, float, PR p, AR a, Velocity* v) {
        V3 offsetA = transform(ldrow3(p, 0), b[0].q), offsetB = transform(ldrow3(p, 3), b[1].q);
        Springiness sp = compute_springiness(ldrow(p, 6), ldrow(p, 7), dt);
        // ComputeEffectiveMass, BallSocketShared.cs:L10-26
        Sym3 inverseEffectiveMass = skew_sandwich(offsetA, b[0].inertia.t) + skew_sandwich(offsetB, b[1].inertia.t);
        float linearContribution = b[0].inertia.inv_mass + b[1].inertia.inv_mass;
        inverseEffectiveMass.xx += linearContribution;
        inverseEffectiveMass.yy += linearContribution;
        inverseEffectiveMass.zz += linearContribution;
        Sym3 effectiveMass = invert(inverseEffectiveMass) * sp.effective_mass_cfm_scale;
        V3 error = ((b[1].pos - b[0].pos) + offsetB) - offsetA;
        V3 biasVelocity = error * sp.position_error_to_velocity;
        // ComputeCorrectiveImpulse, L47-62
        V3 csv = v[0].lin - v[1].lin;
        csv = csv + cross(v[0].ang, offsetA);
        csv = csv + cross(offsetB, v[1].ang);
        csv = biasVelocity - csv;
        V3 acc{ldacc(a, 0), ldacc(a, 1), ldacc(a, 2)};
        V3 corrective = transform(csv, effectiveMass) - acc * sp.softness_impulse_scale;
        acc = acc + corrective;
        ball_socket_apply(v[0], v[1], offsetA, offsetB, b[0].inertia, b[1].inertia, corrective);
        stacc(a, 0, acc.x); stacc(a, 1, acc.y); stacc(a, 2, acc.z);
    }
};

// ---- SwingLimit (25): SwingLimit.cs:L86-149 ----
// prestep: AxisLocalA xyz, AxisLocalB xyz, MinimumDot, AngularFrequency, TwiceDampingRatio | impulse: 1
struct SwingLimit {
    static constexpr int kBodies = 2, kPrestepRows = 9, kImpulseRows = 1;
    static constexpr bool kIncremental = false, kNeedsPose = true;
    template <class PR> BEPU_DI static V3 jacobian(PR p, Q4 qA, Q4 qB, V3& axisA, V3& axisB) {
        axisA = transform(ldrow3(p, 0), qA);
        axisB = transform(ldrow3(p, 3), qB);
        V3 j = cross(axisA, axisB);
        V3 fallback = find_perpendicular(axisA);
        return dot(j, j) < 1e-7f ? fallback : j;
    }
    template <class PR, class AR> BEPU_DI static void warm_start(const BodyState* b, PR p, AR a, Velocity* v) {
        V3 axisA, axisB;
        V3 j = jacobian(p, b[0].q, b[1].q, axisA, axisB);
        angular1_apply(transform(j, b[0].inertia.t), transform(j, b[1].inertia.t), ldacc(a, 0), v[0].ang, v[1].ang);
    }
    template <class PR, class AR> BEPU_DI static void solve(const BodyState* b, float dt, float inverseDt, PR p, AR a, Velocity* v) {
        V3 axisA, axisB;
        V3 j = jacobian(p, b[0].q, b[1].q, axisA, axisB);
        V3 i2vA = transform(j, b[0].inertia.t), ni2vB = transform(j, b[1].inertia.t);
        float angularContributionA = dot(i2vA, j), angularContributionB = dot(ni2vB, j);
        Springiness sp = compute_springiness(ldrow(p, 7), ldrow(p, 8), dt);
        float effectiveMass = sp.effective_mass_cfm_scale / (angularContributionA + angularContributionB);
        float error = dot(axisA, axisB) - ldrow(p, 6);
        float biasVelocity = -fmin_ps(error * inverseDt, error * sp.position_error_to_velocity);
        float csv = dot(v[0].ang - v[1].ang, j);
        float acc = ldacc(a, 0);
        float csi = effectiveMass * (biasVelocity - csv) - acc * sp.softness_impulse_scale;
        clamp_positive(acc, csi);
        angular1_apply(i2vA, ni2vB, csi, v[0].ang, v[1].ang);
        stacc(a, 0, acc);
    }
};

// ---- twist family: TwistServo.cs:L69-151 ----
BEPU_DI void transform_unit_xz(Q4 r, V3& x, V3& z) {  // QuaternionWide.cs:L467-492
    float qX2 = r.x + r.x, qY2 = r.y + r.y, qZ2 = r.z + r.z;
    float YY = qY2 * r.y, ZZ = qZ2 * r.z;
    x.x = 1.0f - YY - ZZ;
    float XY = qX2 * r.y, ZW = qZ2 * r.w;
    x.y = XY + ZW;
    float XZ = qX2 * r.z, YW = qY2 * r.w;
    x.z = XZ - YW;
    float XX = qX2 * r.x, XW = qX2 * r.w, YZ = qY2 * r.z;
    z.x = XZ + YW;
    z.y = YZ - XW;
    z.z = 1.0f - XX - YY;
}
BEPU_DI V3 twist_jacobian_full(Q4 qA, Q4 qB, Q4 localBasisA, Q4 localBasisB, V3& basisBX, V3& basisBZ, M33& basisA) {  // L69-84
    Q4 basisQuaternionA = concatenate(localBasisA, qA);
    Q4 basisQuaternionB = concatenate(localBasisB, qB);
    transform_unit_xz(basisQuaternionB, basisBX, basisBZ);
    basisA = matrix_from_quaternion(basisQuaternionA);
    V3 j = basisA.z + basisBZ;
    float len = length(j);
    j = j * (1.0f / len);
    return len < 1e-10f ? basisA.z : j;
}
BEPU_DI V3 twist_jacobian_only(Q4 qA, Q4 qB, Q4 localBasisA, Q4 localBasisB) {  // L139-151
    V3 basisAZ = transform_unit_z(concatenate(localBasisA, qA)), basisBZ = transform_unit_z(concatenate(localBasisB, qB));
    V3 j = basisAZ + basisBZ;
    float len = length(j);
    j = j * (1.0f / len);
    return len < 1e-10f ? basisAZ : j;
}
BEPU_DI float twist_current_angle(V3 basisBX, V3 basisBZ, const M33& basisA) {  // L86-96
    Q4 aligningRotation = quaternion_between_normalized(basisBZ, basisA.z);
    V3 alignedBasisBX = transform(basisBX, aligningRotation);
    float x = dot(alignedBasisBX, basisA.x), y = dot(alignedBasisBX, basisA.y);
    float absAngle = acos_approx(x);
    return y < 0.0f ? -absAngle : absAngle;
}
struct TwistEffectiveMass { V3 i2vA, ni2vB, v2iA; float position_error_to_velocity, softness_impulse_scale, effective_mass; };
BEPU_DI TwistEffectiveMass twist_effective_mass(float dt, float angularFrequency, float twiceDampingRatio, Sym3 iA, Sym3 iB, V3 j) {  // L98-126
    TwistEffectiveMass r;
    r.i2vA = transform(j, iA);
    r.ni2vB = transform(j, iB);
    float unsoftenedInverseEffectiveMass = dot(r.i2vA, j) + dot(r.ni2vB, j);
    Springiness sp = compute_springiness(angularFrequency, twiceDampingRatio, dt);
    r.position_error_to_velocity = sp.position_error_to_velocity;
    r.softness_impulse_scale = sp.softness_impulse_scale;
    r.effective_mass = sp.effective_mass_cfm_scale / unsoftenedInverseEffectiveMass;
    r.v2iA = j * r.effective_mass;
    return r;
}

// ---- TwistLimit (27): TwistLimit.cs:L68-123 ----
// prestep: LocalBasisA xyzw, LocalBasisB xyzw, MinimumAngle, MaximumAngle, AngularFrequency, TwiceDampingRatio | impulse: 1
struct TwistLimit {
    static constexpr int kBodies = 2, kPrestepRows = 12, kImpulseRows = 1;
    static constexpr bool kIncremental = false, kNeedsPose = true;
    template <class PR> BEPU_DI static V3 jacobian(PR p, Q4 qA, Q4 qB, float& error) {
        V3 basisBX, basisBZ;
        M33 basisA;
        V3 j = twist_jacobian_full(qA, qB, ldrow4(p, 0), ldrow4(p, 4), basisBX, basisBZ, basisA);
        float angle = twist_current_angle(basisBX, basisBZ, basisA);
        float minError = signed_angle_difference(ldrow(p, 8), angle);
        float maxError = signed_angle_difference(ldrow(p, 9), angle);
        bool useMin = fabsf(minError) < fabsf(maxError);
        error = useMin ? -minError : maxError;
        return useMin ? -j : j;
    }
    template <class PR, class AR> BEPU_DI static void warm_start(const BodyState* b, PR p, AR a, Velocity* v) {
        float error;
        V3 j = jacobian(p, b[0].q, b[1].q, error);
        angular1_apply(transform(j, b[0].inertia.t), transform(j, b[1].inertia.t), ldacc(a, 0), v[0].ang, v[1].ang);
    }
    template <class PR, class AR> BEPU_DI static void solve(const BodyState* b, float dt, float inverseDt, PR p, AR a, Velocity* v) {
        float error;
        V3 j = jacobian(p, b[0].q, b[1].q, error);
        TwistEffectiveMass m = twist_effective_mass(dt, ldrow(p, 10), ldrow(p, 11), b[0].inertia.t, b[1].inertia.t, j);
        float biasVelocity = error < 0.0f ? error * inverseDt : error * m.position_error_to_velocity;
        float biasImpulse = biasVelocity * m.effective_mass;
        float csiVelocityComponent = dot(v[0].ang - v[1].ang, m.v2iA);
        float acc = ldacc(a, 0);
        float csi = biasImpulse - acc * m.softness_impulse_scale - csiVelocityComponent;
        clamp_positive(acc, csi);
        angular1_apply(m.i2vA, m.ni2vB, csi, v[0].ang, v[1].ang);
        stacc(a, 0, acc);
    }
};

// ---- TwistServo (26): TwistServo.cs:L153-192 ----
// prestep: LocalBasisA xyzw, LocalBasisB xyzw, TargetAngle, AngularFrequency, TwiceDampingRatio, MaximumSpeed, BaseSpeed, MaximumForce | impulse: 1
struct TwistServo {
    static constexpr int kBodies = 2, kPrestepRows = 14, kImpulseRows = 1;
    static constexpr bool kIncremental = false, kNeedsPose = true;
    template <class PR, class AR> BEPU_DI static void warm_start(const BodyState* b, PR p, AR a, Velocity* v) {
        V3 j = twist_jacobian_only(b[0].q, b[1].q, ldrow4(p, 0), ldrow4(p, 4));
        angular1_apply(transform(j, b[0].inertia.t), transform(j, b[1].inertia.t), ldacc(a, 0), v[0].ang, v[1].ang);
    }
    template <class PR, class AR> BEPU_DI static void solve(const BodyState* b, float dt, float inverseDt, PR p, AR a, Velocity* v) {
        V3 basisBX, basisBZ;
        M33 basisA;
        V3 j = twist_jacobian_full(b[0].q, b[1].q, ldrow4(p, 0), ldrow4(p, 4), basisBX, basisBZ, basisA);
        TwistEffectiveMass m = twist_effective_mass(dt, ldrow(p, 9), ldrow(p, 10), b[0].inertia.t, b[1].inertia.t, j);
        float angle = twist_current_angle(basisBX, basisBZ, basisA);
        float error = signed_angle_difference(ldrow(p, 8), angle);
        float clampedBiasVelocity = servo_clamped_bias_velocity(error, m.position_error_to_velocity, ldrow(p, 11), ldrow(p, 12), inverseDt);
        float maximumImpulse = ldrow(p, 13) * dt;
        float biasImpulse = clampedBiasVelocity * m.effective_mass;
        float csiVelocityComponent = dot(v[0].ang - v[1].ang, m.v2iA);
        float acc = ldacc(a, 0);
        float csi = biasImpulse - acc * m.softness_impulse_scale - csiVelocityComponent;
        float previous = acc;
        acc = fmin_ps(fmax_ps(acc + csi, -maximumImpulse), maximumImpulse);
        csi = acc - previous;
        angular1_apply(m.i2vA, m.ni2vB, csi, v[0].ang, v[1].ang);
        stacc(a, 0, acc);
    }
};

// ---- AngularMotor (30): AngularMotor.cs:L52-79 ----
// prestep: TargetVelocityLocalA xyz, MaximumForce, Damping | impulses: xyz
struct AngularMotor {
    static constexpr int kBodies = 2, kPrestepRows = 5, kImpulseRows = 3;
    static constexpr bool kIncremental = false, kNeedsPose = true;
    template <class PR, class AR> BEPU_DI static void warm_start(const BodyState* b, PR, AR a, Velocity* v) {
        angular3_apply(v[0].ang, v[1].ang, b[0].inertia.t, b[1].inertia.t, V3{ldacc(a, 0), ldacc(a, 1), ldacc(a, 2)});
    }
    template <class PR, class AR> BEPU_DI static void solve(const BodyState* b, float dt, float, PR p, AR a, Velocity* v) {
        MotorSoftness ms = motor_softness(ldrow(p, 3), ldrow(p, 4), dt);
        Sym3 unsoftenedEffectiveMass = invert(b[0].inertia.t + b[1].inertia.t);
        V3 biasVelocity = transform(ldrow3(p, 0), b[0].q);
        V3 csv = biasVelocity - (v[0].ang - v[1].ang);
        V3 csi = transform(csv, unsoftenedEffectiveMass) * ms.effective_mass_cfm_scale;
        V3 acc{ldacc(a, 0), ldacc(a, 1), ldacc(a, 2)};
        csi = csi - acc * ms.softness_impulse_scale;
        servo_clamp_impulse3(ms.maximum_impulse, acc, csi);
        angular3_apply(v[0].ang, v[1].ang, b[0].inertia.t, b[1].inertia.t, csi);
        stacc(a, 0, acc.x); stacc(a, 1, acc.y); stacc(a, 2, acc.z);
    }
};

// ---- AngularServo (29): AngularServo.cs:L58-109 ----
// prestep: TargetRelativeRotationLocalA xyzw, AngularFrequency, TwiceDampingRatio, MaximumSpeed, BaseSpeed, MaximumForce | impulses: xyz
struct AngularServo {
    static constexpr int kBodies = 2, kPrestepRows = 9, kImpulseRows = 3;
    static constexpr bool kIncremental = false, kNeedsPose = true;
    template <class PR, class AR> BEPU_DI static void warm_start(const BodyState* b, PR, AR a, Velocity* v) {
        angular3_apply(v[0].ang, v[1].ang, b[0].inertia.t, b[1].inertia.t, V3{ldacc(a, 0), ldacc(a, 1), ldacc(a, 2)});
    }
    template <class PR, class AR> BEPU_DI static void solve(const BodyState* b, float dt, float inverseDt, PR p, AR a, Velocity* v) {
        Q4 targetOrientationB = concatenate(ldrow4(p, 0), b[0].q);
        Q4 errorRotation = concatenate(conjugate(targetOrientationB), b[1].q);
        V3 errorAxis;
        float errorLength;
        axis_angle_from_quaternion(errorRotation, errorAxis, errorLength);
        Springiness sp = compute_springiness(ldrow(p, 4), ldrow(p, 5), dt);
        Sym3 unsoftenedEffectiveMass = invert(b[0].inertia.t + b[1].inertia.t);
        V3 clampedBiasVelocity = servo_clamped_bias_velocity3(errorAxis, errorLength, sp.position_error_to_velocity, ldrow(p, 6), ldrow(p, 7), inverseDt);
        float maximumImpulse = ldrow(p, 8) * dt;
        V3 csv = clampedBiasVelocity - (v[0].ang - v[1].ang);
        V3 csi = transform(csv, unsoftenedEffectiveMass) * sp.effective_mass_cfm_scale;
        V3 acc{ldacc(a, 0), ldacc(a, 1), ldacc(a, 2)};
        csi = csi - acc * sp.softness_impulse_scale;
        servo_clamp_impulse3(maximumImpulse, acc, csi);
        angular3_apply(v[0].ang, v[1].ang, b[0].inertia.t, b[1].inertia.t, csi);
        stacc(a, 0, acc.x); stacc(a, 1, acc.y); stacc(a, 2, acc.z);
    }
};

// ---- Hinge (47): Hinge.cs:L89-222; AngularHinge.cs:L74-112; Symmetric5x5Wide.cs:L21-51 ----
// prestep: LocalOffsetA xyz, LocalHingeAxisA xyz, LocalOffsetB xyz, LocalHingeAxisB xyz, AngularFrequency, TwiceDampingRatio | impulses: BallSocket xyz, Hinge xy
BEPU_DI V2 hinge_error_angles(V3 hingeAxisA, V3 hingeAxisB, const M23& jacobianA) {
    V3 onPlaneX = hingeAxisB - jacobianA.x * dot(hingeAxisB, jacobianA.x);
    V3 onPlaneY = hingeAxisB - jacobianA.y * dot(hingeAxisB, jacobianA.y);
    float xLength = length(onPlaneX), yLength = length(onPlaneY);
    onPlaneX = onPlaneX * (1.0f / xLength);
    onPlaneY = onPlaneY * (1.0f / yLength);
    onPlaneX = xLength < 1e-7f ? hingeAxisA : onPlaneX;
    onPlaneY = yLength < 1e-7f ? hingeAxisA : onPlaneY;
    V2 e{acos_approx(dot(onPlaneX, hingeAxisA)), acos_approx(dot(onPlaneY, hingeAxisA))};
    float hbxay = dot(onPlaneX, jacobianA.y), hbyax = dot(onPlaneY, jacobianA.x);
    e.x = hbxay < 0.0f ? e.x : -e.x;
    e.y = hbyax < 0.0f ? -e.y : e.y;
    return e;
}
struct Sym5 { Sym3 A; M23 B; Sym2 D; };
BEPU_DI Sym5 invert5(Sym3 a, const M23& b, Sym2 d) {
    Sym2 invD = invert(d);
    M23 bTInvD;  // Symmetric2x2Wide.MultiplyTransposed(b, invD)
    bTInvD.x = {b.x.x * invD.xx + b.y.x * invD.yx, b.x.y * invD.xx + b.y.y * invD.yx, b.x.z * invD.xx + b.y.z * invD.yx};
    bTInvD.y = {b.x.x * invD.yx + b.y.x * invD.yy, b.x.y * invD.yx + b.y.y * invD.yy, b.x.z * invD.yx + b.y.z * invD.yy};
    Sym3 s = complete_matrix_sandwich_t(bTInvD, b);
    Sym5 r;
    r.A = invert(Sym3{a.xx - s.xx, a.yx - s.yx, a.yy - s.yy, a.zx - s.zx, a.zy - s.zy, a.zz - s.zz});
    M23 n;  // Symmetric3x3Wide.MultiplyByTransposed(result.A, bTInvD)
    n.x.x = r.A.xx * bTInvD.x.x + r.A.yx * bTInvD.x.y + r.A.zx * bTInvD.x.z;
    n.y.x = r.A.xx * bTInvD.y.x + r.A.yx * bTInvD.y.y + r.A.zx * bTInvD.y.z;
    n.x.y = r.A.yx * bTInvD.x.x + r.A.yy * bTInvD.x.y + r.A.zy * bTInvD.x.z;
    n.y.y = r.A.yx * bTInvD.y.x + r.A.yy * bTInvD.y.y + r.A.zy * bTInvD.y.z;
    n.x.z = r.A.zx * bTInvD.x.x + r.A.zy * bTInvD.x.y + r.A.zz * bTInvD.x.z;
    n.y.z = r.A.zx * bTInvD.y.x + r.A.zy * bTInvD.y.y + r.A.zz * bTInvD.y.z;
    r.B = {-n.x, -n.y};
    r.D = complete_matrix_sandwich(bTInvD, n) + invD;
    return r;
}
struct Hinge {
    static constexpr int kBodies = 2, kPrestepRows = 14, kImpulseRows = 5;
    static constexpr bool kIncremental = false, kNeedsPose = true;
    BEPU_DI static void apply(V3 offsetA, V3 offsetB, const M23& hingeJacobian, const Inertia& iA, const Inertia& iB, V3 ballSocket, V2 hinge, Velocity& vA, Velocity& vB) {  // L70-92
        vA.lin = vA.lin + ballSocket * iA.inv_mass;
        V3 hingeAngularImpulseA = transform(hinge, hingeJacobian);
        vA.ang = vA.ang + transform(cross(offsetA, ballSocket) + hingeAngularImpulseA, iA.t);
        vB.lin = vB.lin - ballSocket * iB.inv_mass;
        vB.ang = vB.ang + transform(cross(ballSocket, offsetB) - hingeAngularImpulseA, iB.t);
    }
    template <class PR, class AR> BEPU_DI static void warm_start(const BodyState* b, PR p, AR a, Velocity* v) {
        M33 mA = matrix_from_quaternion(b[0].q);
        V3 offsetA = transform(ldrow3(p, 0), mA);
        V3 offsetB = transform(ldrow3(p, 6), b[1].q);
        V3 localAX, localAY;
        build_orthonormal_basis(ldrow3(p, 3), localAX, localAY);
        M23 hingeJacobian{transform(localAX, mA), transform(localAY, mA)};
        apply(offsetA, offsetB, hingeJacobian, b[0].inertia, b[1].inertia, V3{ldacc(a, 0), ldacc(a, 1), ldacc(a, 2)}, V2{ldacc(a, 3), ldacc(a, 4)}, v[0], v[1]);
    }
    template <class PR, class AR> BEPU_DI static void solve(const BodyState* b, float dt, float, PR p, AR a, Velocity* v) {
        const Inertia& iA = b[0].inertia;
        const Inertia& iB = b[1].inertia;
        M33 mA = matrix_from_quaternion(b[0].q), mB = matrix_from_quaternion(b[1].q);
        V3 localHingeAxisA = ldrow3(p, 3);
        V3 offsetA = transform(ldrow3(p, 0), mA), hingeAxisA = transform(localHingeAxisA, mA);
        V3 offsetB = transform(ldrow3(p, 6), mB), hingeAxisB = transform(ldrow3(p, 9), mB);
        V3 localAX, localAY;
        build_orthonormal_basis(localHingeAxisA, localAX, localAY);
        M23 hingeJacobian{transform(localAX, mA), transform(localAY, mA)};
        Sym3 A = skew_sandwich(offsetA, iA.t) + skew_sandwich(offsetB, iB.t);
        float linearContribution = iA.inv_mass + iB.inv_mass;
        A.xx += linearContribution;
        A.yy += linearContribution;
        A.zz += linearContribution;
        M23 hingeInertiaA = multiply(hingeJacobian, iA.t), hingeInertiaB = multiply(hingeJacobian, iB.t);
        Sym2 D = complete_matrix_sandwich(hingeInertiaA, hingeJacobian) + complete_matrix_sandwich(hingeInertiaB, hingeJacobian);
        M23 B{cross(hingeInertiaA.x, offsetA) + cross(hingeInertiaB.x, offsetB), cross(hingeInertiaA.y, offsetA) + cross(hingeInertiaB.y, offsetB)};
        Sym5 m = invert5(A, B, D);
        Springiness sp = compute_springiness(ldrow(p, 12), ldrow(p, 13), dt);
        V3 ballSocketError = ((b[1].pos - b[0].pos) + offsetB) - offsetA;
        V3 ballSocketBiasVelocity = ballSocketError * sp.position_error_to_velocity;
        V2 hingeBiasVelocity = hinge_error_angles(hingeAxisA, hingeAxisB, hingeJacobian) * (-sp.position_error_to_velocity);
        V3 ballSocketAngularCSV = cross(v[0].ang, offsetA) + cross(offsetB, v[1].ang);
        V3 v0 = ballSocketBiasVelocity - (ballSocketAngularCSV + (v[0].lin - v[1].lin));
        V2 v1 = hingeBiasVelocity - (transform_by_transpose(v[0].ang, hingeJacobian) - transform_by_transpose(v[1].ang, hingeJacobian));
        V3 csiBall;  // Symmetric5x5Wide.TransformWithoutOverlap
        V2 csiHinge;
        csiBall.x = v0.x * m.A.xx + v0.y * m.A.yx + v0.z * m.A.zx + v1.x * m.B.x.x + v1.y * m.B.y.x;
        csiBall.y = v0.x * m.A.yx + v0.y * m.A.yy + v0.z * m.A.zy + v1.x * m.B.x.y + v1.y * m.B.y.y;
        csiBall.z = v0.x * m.A.zx + v0.y * m.A.zy + v0.z * m.A.zz + v1.x * m.B.x.z + v1.y * m.B.y.z;
        csiHinge.x = v0.x * m.B.x.x + v0.y * m.B.x.y + v0.z * m.B.x.z + v1.x * m.D.xx + v1.y * m.D.yx;
        csiHinge.y = v0.x * m.B.y.x + v0.y * m.B.y.y + v0.z * m.B.y.z + v1.x * m.D.yx + v1.y * m.D.yy;
        csiBall = csiBall * sp.effective_mass_cfm_scale;
        csiHinge = csiHinge * sp.effective_mass_cfm_scale;
        V3 accBall{ldacc(a, 0), ldacc(a, 1), ldacc(a, 2)};
        V2 accHinge{ldacc(a, 3), ldacc(a, 4)};
        csiBall = csiBall - accBall * sp.softness_impulse_scale;
        csiHinge = csiHinge - accHinge * sp.softness_impulse_scale;
        accBall = accBall + csiBall;
        accHinge = accHinge + csiHinge;
        apply(offsetA, offsetB, hingeJacobian, iA, iB, csiBall, csiHinge, v[0], v[1]);
        stacc(a, 0, accBall.x); stacc(a, 1, accBall.y); stacc(a, 2, accBall.z); stacc(a, 3, accHinge.x); stacc(a, 4, accHinge.y);
    }
};

// ---- SwivelHinge (46): SwivelHinge.cs:L86-215; Symmetric4x4Wide.cs:L46-80 ----
// prestep: LocalOffsetA xyz, LocalSwivelAxisA xyz, LocalOffsetB xyz, LocalHingeAxisB xyz, AngularFrequency, TwiceDampingRatio | impulses: xyzw
struct Sym4 { float xx, yx, yy, zx, zy, zz, wx, wy, wz, ww; };
BEPU_DI Sym4 invert4(const Sym4& m) {
    float s0 = m.xx * m.yy - m.yx * m.yx;
    float s1 = m.xx * m.zy - m.yx * m.zx;
    float s2 = m.xx * m.wy - m.yx * m.wx;
    float s3 = m.yx * m.zy - m.yy * m.zx;
    float s4 = m.yx * m.wy - m.yy * m.wx;
    float s5 = m.zx * m.wy - m.zy * m.wx;
    float c5 = m.zz * m.ww - m.wz * m.wz;
    float c4 = m.zy * m.ww - m.wy * m.wz;
    float c3 = m.zy * m.wz - m.wy * m.zz;
    float c2 = m.zx * m.ww - m.wx * m.wz;
    float c1 = m.zx * m.wz - m.wx * m.zz;
    float id = 1.0f / (s0 * c5 - s1 * c4 + s2 * c3 + s3 * c2 - s4 * c1 + s5 * s5);
    Sym4 r;
    r.xx = (m.yy * c5 - m.zy * c4 + m.wy * c3) * id;
    r.yx = (-m.yx * c5 + m.zy * c2 - m.wy * c1) * id;
    r.yy = (m.xx * c5 - m.zx * c2 + m.wx * c1) * id;
    r.zx = (m.yx * c4 - m.yy * c2 + m.wy * s5) * id;
    r.zy = (-m.xx * c4 + m.yx * c2 - m.wx * s5) * id;
    r.zz = (m.wx * s4 - m.wy * s2 + m.ww * s0) * id;
    r.wx = (-m.yx * c3 + m.yy * c1 - m.zy * s5) * id;
    r.wy = (m.xx * c3 - m.yx * c1 + m.zx * s5) * id;
    r.wz = (-m.wx * s3 + m.wy * s1 - m.wz * s0) * id;
    r.ww = (m.zx * s3 - m.zy * s1 + m.zz * s0) * id;
    return r;
}
struct SwivelHinge {
    static constexpr int kBodies = 2, kPrestepRows = 14, kImpulseRows = 4;
    static constexpr bool kIncremental = false, kNeedsPose = true;
    BEPU_DI static void apply(V3 offsetA, V3 offsetB, V3 j, const Inertia& iA, const Inertia& iB, V4 csi, Velocity& vA, Velocity& vB) {  // L66-84
        V3 ballSocketCSI{csi.x, csi.y, csi.z};
        vA.lin = vA.lin + ballSocketCSI * iA.inv_mass;
        V3 swivelHingeAngularImpulseA = j * csi.w;
        vA.ang = vA.ang + transform(cross(offsetA, ballSocketCSI) + swivelHingeAngularImpulseA, iA.t);
        vB.lin = vB.lin - ballSocketCSI * iB.inv_mass;
        vB.ang = vB.ang + transform(cross(ballSocketCSI, offsetB) - swivelHingeAngularImpulseA, iB.t);
    }
    template <class PR> BEPU_DI static V3 jacobian(PR p, Q4 qA, Q4 qB, V3& swivelAxis, V3& hingeAxis, V3& offsetA, V3& offsetB) {  // L86-101
        M33 mA = matrix_from_quaternion(qA), mB = matrix_from_quaternion(qB);
        offsetA = transform(ldrow3(p, 0), mA);
        swivelAxis = transform(ldrow3(p, 3), mA);
        offsetB = transform(ldrow3(p, 6), mB);
        hingeAxis = transform(ldrow3(p, 9), mB);
        V3 j = cross(swivelAxis, hingeAxis);
        return length_squared(j) < 1e-3f ? hingeAxis : j;
    }
    template <class PR, class AR> BEPU_DI static void warm_start(const BodyState* b, PR p, AR a, Velocity* v) {
        V3 swivelAxis, hingeAxis, offsetA, offsetB;
        V3 j = jacobian(p, b[0].q, b[1].q, swivelAxis, hingeAxis, offsetA, offsetB);
        apply(offsetA, offsetB, j, b[0].inertia, b[1].inertia, V4{ldacc(a, 0), ldacc(a, 1), ldacc(a, 2), ldacc(a, 3)}, v[0], v[1]);
    }
    template <class PR, class AR> BEPU_DI static void solve(const BodyState* b, float dt, float, PR p, AR a, Velocity* v) {
        const Inertia& iA = b[0].inertia;
        const Inertia& iB = b[1].inertia;
        V3 swivelAxis, hingeAxis, offsetA, offsetB;
        V3 j = jacobian(p, b[0].q, b[1].q, swivelAxis, hingeAxis, offsetA, offsetB);
        Sym3 upperLeft = skew_sandwich(offsetA, iA.t) + skew_sandwich(offsetB, iB.t);
        float linearContribution = iA.inv_mass + iB.inv_mass;
        Sym4 m;
        m.xx = upperLeft.xx + linearContribution; m.yx = upperLeft.yx; m.yy = upperLeft.yy + linearContribution;
        m.zx = upperLeft.zx; m.zy = upperLeft.zy; m.zz = upperLeft.zz + linearContribution;
        V3 swivelHingeInertiaA = transform(j, iA.t), swivelHingeInertiaB = transform(j, iB.t);
        m.ww = dot(swivelHingeInertiaA, j) + dot(swivelHingeInertiaB, j);
        V3 upperRight = cross(swivelHingeInertiaA, offsetA) + cross(swivelHingeInertiaB, offsetB);
        m.wx = upperRight.x; m.wy = upperRight.y; m.wz = upperRight.z;
        Sym4 e = invert4(m);
        Springiness sp = compute_springiness(ldrow(p, 12), ldrow(p, 13), dt);
        V3 ballSocketError = ((b[1].pos - b[0].pos) + offsetB) - offsetA;
        float pe2v = sp.position_error_to_velocity;
        V4 bias{ballSocketError.x * pe2v, ballSocketError.y * pe2v, ballSocketError.z * pe2v, pe2v * -dot(hingeAxis, swivelAxis)};
        V3 ballSocketAngularCSV = cross(v[0].ang, offsetA) + cross(offsetB, v[1].ang);
        V3 ballSocketLinearCSV = v[0].lin - v[1].lin;
        V4 csv{bias.x - (ballSocketAngularCSV.x + ballSocketLinearCSV.x), bias.y - (ballSocketAngularCSV.y + ballSocketLinearCSV.y),
               bias.z - (ballSocketAngularCSV.z + ballSocketLinearCSV.z), bias.w - (dot(j, v[0].ang) - dot(j, v[1].ang))};
        V4 csi;
        csi.x = csv.x * e.xx + csv.y * e.yx + csv.z * e.zx + csv.w * e.wx;
        csi.y = csv.x * e.yx + csv.y * e.yy + csv.z * e.zy + csv.w * e.wy;
        csi.z = csv.x * e.zx + csv.y * e.zy + csv.z * e.zz + csv.w * e.wz;
        csi.w = csv.x * e.wx + csv.y * e.wy + csv.z * e.wz + csv.w * e.ww;
        const float cfm = sp.effective_mass_cfm_scale, soft = sp.softness_impulse_scale;
        V4 acc{ldacc(a, 0), ldacc(a, 1), ldacc(a, 2), ldacc(a, 3)};
        csi = {csi.x * cfm - acc.x * soft, csi.y * cfm - acc.y * soft, csi.z * cfm - acc.z * soft, csi.w * cfm - acc.w * soft};
        acc = {acc.x + csi.x, acc.y + csi.y, acc.z + csi.z, acc.w + csi.w};
        apply(offsetA, offsetB, j, iA, iB, csi, v[0], v[1]);
        stacc(a, 0, acc.x); stacc(a, 1, acc.y); stacc(a, 2, acc.z); stacc(a, 3, acc.w);
    }
};

#define BEPU_JOINT_TYPES(X) X(22, BallSocket) X(25, SwingLimit) X(26, TwistServo) X(27, TwistLimit) X(29, AngularServo) X(30, AngularMotor) X(46, SwivelHinge) X(47, Hinge)

}  // namespace BEPU_NS
