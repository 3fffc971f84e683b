// ORACLE — test infrastructure only (see bepu_math.h header). Convex and nonconvex contact constraint functions.
// Restates BepuPhysics/Constraints/Contact/{PenetrationLimit,PenetrationLimitOneBody,TangentFriction,
// TangentFrictionOneBody,TwistFriction,TwistFrictionOneBody,ContactConvexTypes,ContactNonconvexCommon}.cs.
#pragma once
#include "bepu_math.h"

namespace bepu_oracle {

// A view of one AOSOA bundle chunk: row r of the bundle starts at base + r * stride elements (float, or double for the float64 lane).
template <class F> struct Rows {
    typename LaneTraits<F>::Scalar* base;
    int stride;
    inline F get(int r) const {
        F v;
        std::memcpy(&v, base + (size_t)r * stride, sizeof(F));
        return v;
    }
    inline void set(int r, const F& v) const { std::memcpy(base + (size_t)r * stride, &v, sizeof(F)); }
    inline V3<F> get3(int r) const { return {get(r), get(r + 1), get(r + 2)}; }
    inline V2<F> get2(int r) const { return {get(r), get(r + 1)}; }
    inline void set3(int r, const V3<F>& v) const { set(r, v.x); set(r + 1, v.y); set(r + 2, v.z); }
    inline void set2(int r, const V2<F>& v) const { set(r, v.x); set(r + 1, v.y); }
    inline Q4<F> get4(int r) const { return {get(r), get(r + 1), get(r + 2), get(r + 3)}; }
};

// ---- PenetrationLimit (two body) : Contact/PenetrationLimit.cs ---------------------------------------------------
// L45-65 ApplyImpulse
template <class F>
inline void penetration_apply_impulse(const Inertia<F>& iA, const Inertia<F>& iB, const V3<F>& normal, const V3<F>& angularA, const V3<F>& angularB,
                                      const F& impulse, Velocity<F>& vA, Velocity<F>& vB) {
    F linearVelocityChangeA = impulse * iA.inv_mass;
    V3<F> dLinA = scale(normal, linearVelocityChangeA);
    V3<F> angImpA = scale(angularA, impulse);
    V3<F> dAngA = transform(angImpA, iA.t);
    F linearVelocityChangeB = impulse * iB.inv_mass;
    V3<F> dLinB = scale(normal, linearVelocityChangeB);
    V3<F> angImpB = scale(angularB, impulse);
    V3<F> dAngB = transform(angImpB, iB.t);
    vA.lin = add(vA.lin, dLinA);
    vA.ang = add(vA.ang, dAngA);
    vB.lin = sub(vB.lin, dLinB);
    vB.ang = add(vB.ang, dAngB);
}
// L67-75 WarmStart
template <class F>
inline void penetration_warm_start(const Inertia<F>& iA, const Inertia<F>& iB, const V3<F>& normal, const V3<F>& offsetA, const V3<F>& offsetB,
                                   const F& accumulated, Velocity<F>& vA, Velocity<F>& vB) {
    V3<F> angularA = cross(offsetA, normal);
    V3<F> angularB = cross(normal, offsetB);
    penetration_apply_impulse(iA, iB, normal, angularA, angularB, accumulated, vA, vB);
}
// L78-131 Solve (+ L10-26 ComputeCorrectiveImpulse)
template <class F>
inline void penetration_solve(const Inertia<F>& iA, const Inertia<F>& iB, const V3<F>& normal, const V3<F>& offsetA, const V3<F>& offsetB,
                              const F& depth, const F& positionErrorToVelocity, const F& effectiveMassCFMScale, const F& maximumRecoveryVelocity,
                              const F& inverseDt, const F& softnessImpulseScale, F& accumulated, Velocity<F>& vA, Velocity<F>& vB) {
    V3<F> angularA = cross(offsetA, normal);
    V3<F> angularB = cross(normal, offsetB);
    F angularA0 = vector_sandwich(angularA, iA.t);
    F angularB0 = vector_sandwich(angularB, iB.t);
    F linear = iA.inv_mass + iB.inv_mass;
    F effectiveMass = effectiveMassCFMScale / (linear + angularA0 + angularB0);
    F biasVelocity = vmin(depth * inverseDt, vmin(depth * positionErrorToVelocity, maximumRecoveryVelocity));
    // ComputeCorrectiveImpulse
    F csvaLinear = dot(vA.lin, normal);
    F csvaAngular = dot(vA.ang, angularA);
    F negatedCSVBLinear = dot(vB.lin, normal);
    F csvbAngular = dot(vB.ang, angularB);
    F negatedCSI = accumulated * softnessImpulseScale + (csvaLinear - negatedCSVBLinear + csvaAngular + csvbAngular - biasVelocity) * effectiveMass;
    F previous = accumulated;
    accumulated = vmax(bc<F>(0.0f), accumulated - negatedCSI);
    F csi = accumulated - previous;
    penetration_apply_impulse(iA, iB, normal, angularA, angularB, csi, vA, vB);
}
// L28-43 UpdatePenetrationDepth
template <class F>
inline void update_penetration_depth(const F& dt, const V3<F>& contactOffsetA, const V3<F>& offsetB, const V3<F>& normal,
                                     const Velocity<F>& vA, const Velocity<F>& vB, F& depth) {
    V3<F> wxra = cross(vA.ang, contactOffsetA);
    V3<F> contactVelocityA = add(wxra, vA.lin);
    V3<F> contactOffsetB = sub(contactOffsetA, offsetB);
    V3<F> wxrb = cross(vB.ang, contactOffsetB);
    V3<F> contactVelocityB = add(wxrb, vB.lin);
    V3<F> diff = sub(contactVelocityA, contactVelocityB);
    F estimatedDepthChangeVelocity = dot(normal, diff);
    depth = depth - estimatedDepthChangeVelocity * dt;
}

// ---- PenetrationLimitOneBody : Contact/PenetrationLimitOneBody.cs ------------------------------------------------
template <class F>
inline void penetration1_apply_impulse(const Inertia<F>& iA, const V3<F>& normal, const V3<F>& angularA, const F& impulse, Velocity<F>& vA) {
    F linearVelocityChangeA = impulse * iA.inv_mass;
    V3<F> dLinA = scale(normal, linearVelocityChangeA);
    V3<F> angImpA = scale(angularA, impulse);
    V3<F> dAngA = transform(angImpA, iA.t);
    vA.lin = add(vA.lin, dLinA);
    vA.ang = add(vA.ang, dAngA);
}
template <class F>
inline void penetration1_warm_start(const Inertia<F>& iA, const V3<F>& normal, const V3<F>& offsetA, const F& accumulated, Velocity<F>& vA) {
    V3<F> angularA = cross(offsetA, normal);
    penetration1_apply_impulse(iA, normal, angularA, accumulated, vA);
}
template <class F>
inline void penetration1_solve(const Inertia<F>& iA, const V3<F>& normal, const V3<F>& offsetA, const F& depth, const F& positionErrorToVelocity,
                               const F& effectiveMassCFMScale, const F& maximumRecoveryVelocity, const F& inverseDt, const F& softnessImpulseScale,
                               F& accumulated, Velocity<F>& vA) {
    V3<F> angularA = cross(offsetA, normal);
    F angularA0 = vector_sandwich(angularA, iA.t);
    F effectiveMass = effectiveMassCFMScale / (iA.inv_mass + angularA0);
    F biasVelocity = vmin(depth * inverseDt, vmin(depth * positionErrorToVelocity, maximumRecoveryVelocity));
    F csvaLinear = dot(vA.lin, normal);
    F csvaAngular = dot(vA.ang, angularA);
    F negatedCSI = accumulated * softnessImpulseScale + (csvaLinear + csvaAngular - biasVelocity) * effectiveMass;
    F previous = accumulated;
    accumulated = vmax(bc<F>(0.0f), accumulated - negatedCSI);
    F csi = accumulated - previous;
    penetration1_apply_impulse(iA, normal, angularA, csi, vA);
}
template <class F>
inline void update_penetration_depth1(const F& dt, const V3<F>& contactOffset, const V3<F>& normal, const Velocity<F>& v, F& depth) {
    V3<F> wxr = cross(v.ang, contactOffset);
    V3<F> contactVelocity = add(wxr, v.lin);
    F estimatedDepthChange = dot(normal, contactVelocity);
    depth = depth - estimatedDepthChange * dt;
}

// ---- TangentFriction (two body) : Contact/TangentFriction.cs -----------------------------------------------------
template <class F> struct TangentJacobians { M23<F> linearA, angularA, angularB; };
// L17-27
template <class F>
inline TangentJacobians<F> tangent_jacobians(const V3<F>& tX, const V3<F>& tY, const V3<F>& offsetA, const V3<F>& offsetB) {
    TangentJacobians<F> j;
    j.linearA.x = tX; j.linearA.y = tY;
    j.angularA.x = cross(offsetA, tX);
    j.angularA.y = cross(offsetA, tY);
    j.angularB.x = cross(tX, offsetB);
    j.angularB.y = cross(tY, offsetB);
    return j;
}
// L29-46
template <class F>
inline void tangent_apply_impulse(const TangentJacobians<F>& j, const Inertia<F>& iA, const Inertia<F>& iB, const V2<F>& impulse, Velocity<F>& vA, Velocity<F>& vB) {
    V3<F> linearImpulseA = transform(impulse, j.linearA);
    V3<F> angularImpulseA = transform(impulse, j.angularA);
    V3<F> angularImpulseB = transform(impulse, j.angularB);
    V3<F> cvALin = scale(linearImpulseA, iA.inv_mass);
    V3<F> cvAAng = transform(angularImpulseA, iA.t);
    V3<F> cvBLin = scale(linearImpulseA, iB.inv_mass);
    V3<F> cvBAng = transform(angularImpulseB, iB.t);
    vA.lin = add(vA.lin, cvALin);
    vA.ang = add(vA.ang, cvAAng);
    vB.lin = sub(vB.lin, cvBLin);
    vB.ang = add(vB.ang, cvBAng);
}
template <class F>
inline void tangent_warm_start(const V3<F>& tX, const V3<F>& tY, const V3<F>& offsetA, const V3<F>& offsetB, const Inertia<F>& iA, const Inertia<F>& iB,
                               const V2<F>& accumulated, Velocity<F>& vA, Velocity<F>& vB) {
    TangentJacobians<F> j = tangent_jacobians(tX, tY, offsetA, offsetB);
    tangent_apply_impulse(j, iA, iB, accumulated, vA, vB);
}
// L82-100 Solve (+ L48-70 ComputeCorrectiveImpulse)
template <class F>
inline void tangent_solve(const V3<F>& tX, const V3<F>& tY, const V3<F>& offsetA, const V3<F>& offsetB, const Inertia<F>& iA, const Inertia<F>& iB,
                          const F& maximumImpulse, V2<F>& accumulated, Velocity<F>& vA, Velocity<F>& vB) {
    TangentJacobians<F> j = tangent_jacobians(tX, tY, offsetA, offsetB);
    Sym2<F> linearContributionA = sandwich_scale(j.linearA, iA.inv_mass);
    Sym2<F> linearContributionB = sandwich_scale(j.linearA, iB.inv_mass);
    Sym2<F> angularContributionA = matrix_sandwich(j.angularA, iA.t);
    Sym2<F> angularContributionB = matrix_sandwich(j.angularB, iB.t);
    Sym2<F> linear = add(linearContributionA, linearContributionB);
    Sym2<F> angular = add(angularContributionA, angularContributionB);
    Sym2<F> inverseEffectiveMass = add(linear, angular);
    Sym2<F> effectiveMass = invert(inverseEffectiveMass);
    // ComputeCorrectiveImpulse
    V2<F> csvaLinear = transform_by_transpose(vA.lin, j.linearA);
    V2<F> csvaAngular = transform_by_transpose(vA.ang, j.angularA);
    V2<F> csvbLinear = transform_by_transpose(vB.lin, j.linearA);
    V2<F> csvbAngular = transform_by_transpose(vB.ang, j.angularB);
    V2<F> csvLinear = sub(csvbLinear, csvaLinear);
    V2<F> csvAngular = add(csvaAngular, csvbAngular);
    V2<F> csv = sub(csvLinear, csvAngular);
    V2<F> csi = transform(csv, effectiveMass);
    V2<F> previous = accumulated;
    accumulated = add(accumulated, csi);
    F magnitude = length(accumulated);
    F scl = vmin(bc<F>(1.0f), maximumImpulse / vmax(bc<F>(1e-16f), magnitude));
    accumulated = scale(accumulated, scl);
    V2<F> corrective = sub(accumulated, previous);
    tangent_apply_impulse(j, iA, iB, corrective, vA, vB);
}

// ---- TangentFrictionOneBody : Contact/TangentFrictionOneBody.cs --------------------------------------------------
template <class F>
inline void tangent1_apply_impulse(const M23<F>& linearA, const M23<F>& angularA, const Inertia<F>& iA, const V2<F>& impulse, Velocity<F>& vA) {
    V3<F> linearImpulseA = transform(impulse, linearA);
    V3<F> angularImpulseA = transform(impulse, angularA);
    V3<F> cvALin = scale(linearImpulseA, iA.inv_mass);
    V3<F> cvAAng = transform(angularImpulseA, iA.t);
    vA.lin = add(vA.lin, cvALin);
    vA.ang = add(vA.ang, cvAAng);
}
template <class F>
inline void tangent1_warm_start(const V3<F>& tX, const V3<F>& tY, const V3<F>& offsetA, const Inertia<F>& iA, const V2<F>& accumulated, Velocity<F>& vA) {
    M23<F> linearA{tX, tY};
    M23<F> angularA{cross(offsetA, tX), cross(offsetA, tY)};
    tangent1_apply_impulse(linearA, angularA, iA, accumulated, vA);
}
template <class F>
inline void tangent1_solve(const V3<F>& tX, const V3<F>& tY, const V3<F>& offsetA, const Inertia<F>& iA, const F& maximumImpulse, V2<F>& accumulated, Velocity<F>& vA) {
    M23<F> linearA{tX, tY};
    M23<F> angularA{cross(offsetA, tX), cross(offsetA, tY)};
    Sym2<F> linearContributionA = sandwich_scale(linearA, iA.inv_mass);
    Sym2<F> angularContributionA = matrix_sandwich(angularA, iA.t);
    Sym2<F> inverseEffectiveMass = add(linearContributionA, angularContributionA);
    Sym2<F> effectiveMass = invert(inverseEffectiveMass);
    V2<F> csvaLinear = transform_by_transpose(vA.lin, linearA);
    V2<F> csvaAngular = transform_by_transpose(vA.ang, angularA);
    V2<F> csv = add(csvaLinear, csvaAngular);
    V2<F> negativeCSI = transform(csv, effectiveMass);
    V2<F> previous = accumulated;
    accumulated = sub(accumulated, negativeCSI);
    F magnitude = length(accumulated);
    F scl = vmin(bc<F>(1.0f), maximumImpulse / vmax(bc<F>(1e-16f), magnitude));
    accumulated = scale(accumulated, scl);
    V2<F> corrective = sub(accumulated, previous);
    tangent1_apply_impulse(linearA, angularA, iA, corrective, vA);
}

// ---- TwistFriction : Contact/TwistFriction.cs, TwistFrictionOneBody.cs -------------------------------------------
template <class F>
inline void twist_apply_impulse(const V3<F>& angularJacobianA, const Inertia<F>& iA, const Inertia<F>& iB, const F& impulse, Velocity<F>& vA, Velocity<F>& vB) {
    V3<F> worldImpulseA = scale(angularJacobianA, impulse);
    V3<F> dA = transform(worldImpulseA, iA.t);
    V3<F> dB = transform(worldImpulseA, iB.t);
    vA.ang = add(vA.ang, dA);
    vB.ang = sub(vB.ang, dB);
}
template <class F>
inline void twist_solve(const V3<F>& angularJacobianA, const Inertia<F>& iA, const Inertia<F>& iB, const F& maximumImpulse, F& accumulated, Velocity<F>& vA, Velocity<F>& vB) {
    F angularA = vector_sandwich(angularJacobianA, iA.t);
    F angularB = vector_sandwich(angularJacobianA, iB.t);
    F inverseEffectiveMass = angularA + angularB;
    MaskOf<F> inverseIsZero = eq(bc<F>(0.0f), inverseEffectiveMass);
    F effectiveMass = sel(inverseIsZero, bc<F>(0.0f), bc<F>(1.0f) / inverseEffectiveMass);
    F csvA = dot(vA.ang, angularJacobianA);
    F negatedCSVB = dot(vB.ang, angularJacobianA);
    F negatedCSI = (csvA - negatedCSVB) * effectiveMass;
    F previous = accumulated;
    accumulated = vmin(maximumImpulse, vmax(-maximumImpulse, accumulated - negatedCSI));
    F csi = accumulated - previous;
    twist_apply_impulse(angularJacobianA, iA, iB, csi, vA, vB);
}
template <class F>
inline void twist1_apply_impulse(const V3<F>& angularJacobianA, const Inertia<F>& iA, const F& impulse, Velocity<F>& vA) {
    V3<F> worldImpulseA = scale(angularJacobianA, impulse);
    V3<F> dA = transform(worldImpulseA, iA.t);
    vA.ang = add(vA.ang, dA);
}
template <class F>
inline void twist1_solve(const V3<F>& angularJacobianA, const Inertia<F>& iA, const F& maximumImpulse, F& accumulated, Velocity<F>& vA) {
    F angularA = vector_sandwich(angularJacobianA, iA.t);
    MaskOf<F> inverseIsZero = eq(bc<F>(0.0f), angularA);
    F effectiveMass = sel(inverseIsZero, bc<F>(0.0f), bc<F>(1.0f) / angularA);
    F csvA = dot(vA.ang, angularJacobianA);
    F negativeCSI = csvA * effectiveMass;
    F previous = accumulated;
    accumulated = vmin(maximumImpulse, vmax(-maximumImpulse, accumulated - negativeCSI));
    F csi = accumulated - previous;
    twist1_apply_impulse(angularJacobianA, iA, csi, vA);
}

// ---- FrictionHelpers.ComputeFrictionCenter : Contact/ContactConvexTypes.cs:L124-196 ------------------------------
template <class F, int N>
inline V3<F> friction_center(const V3<F>* offsets, const F* depths) {
    F zero = bc<F>(0.0f), one = bc<F>(1.0f);
    F w[N];
    for (int i = 0; i < N; ++i) w[i] = sel(lt(depths[i], zero), zero, one);
    F weightSum = w[0];
    for (int i = 1; i < N; ++i) weightSum = weightSum + w[i];
    MaskOf<F> useFallback = eq(weightSum, zero);
    weightSum = sel(useFallback, bc<F>((float)N), weightSum);
    F inverseWeightSum = one / weightSum;
    V3<F> c[N];
    for (int i = 0; i < N; ++i) {
        F wi = sel(useFallback, inverseWeightSum, w[i] * inverseWeightSum);
        c[i] = scale(offsets[i], wi);
    }
    if (N == 2) return add(c[0], c[1]);
    if (N == 3) return add(add(c[0], c[1]), c[2]);
    return add(add(c[0], c[1]), add(c[2 % N], c[3 % N]));
}

// ---- Convex manifold constraints : Contact/ContactConvexTypes.cs -------------------------------------------------
// Prestep row layout (ConvexContactWide = OffsetA xyz + Depth; MaterialPropertiesWide = FrictionCoefficient, SpringSettings{AngularFrequency,
// TwiceDampingRatio}, MaximumRecoveryVelocity; ContactConvexCommon.cs:L6-17):
//   one body : [contact i: 4i..4i+3] [normal 4N..4N+2] [material 4N+3..4N+6]                      -> 4N+7 rows
//   two body : [contact i: 4i..4i+3] [offsetB 4N..4N+2] [normal 4N+3..4N+5] [material 4N+6..4N+9]  -> 4N+10 rows
// Accumulated impulses: [tangent 0..1] [penetration 2..N+1] [twist N+2]                               -> N+3 rows
template <int N, bool TwoBody> struct ConvexLayout {
    static constexpr int kOffsetB = 4 * N;
    static constexpr int kNormal = TwoBody ? 4 * N + 3 : 4 * N;
    static constexpr int kFriction = kNormal + 3;
    static constexpr int kAngularFrequency = kNormal + 4;
    static constexpr int kTwiceDampingRatio = kNormal + 5;
    static constexpr int kMaxRecovery = kNormal + 6;
    static constexpr int kPrestepRows = kNormal + 7;
    static constexpr int kImpulseRows = N + 3;
};

// Two-body convex: e.g. Contact4Functions, ContactConvexTypes.cs:L1461-1514 (N=1: L941-980).
template <class F, int N> struct ConvexTwoBody {
    typedef ConvexLayout<N, true> L;
    static void warm_start(const Inertia<F>& iA, const Inertia<F>& iB, const Rows<F>& p, const Rows<F>& a, Velocity<F>& vA, Velocity<F>& vB) {
        V3<F> normal = p.get3(L::kNormal), offsetB = p.get3(L::kOffsetB);
        V3<F> x, z;
        build_orthonormal_basis(normal, x, z);
        V3<F> offs[N]; F depths[N];
        for (int i = 0; i < N; ++i) { offs[i] = p.get3(4 * i); depths[i] = p.get(4 * i + 3); }
        V3<F> centerA = (N == 1) ? offs[0] : friction_center<F, N>(offs, depths);
        V3<F> centerB = sub(centerA, offsetB);
        tangent_warm_start(x, z, centerA, centerB, iA, iB, a.get2(0), vA, vB);
        for (int i = 0; i < N; ++i) penetration_warm_start(iA, iB, normal, offs[i], sub(offs[i], offsetB), a.get(2 + i), vA, vB);
        twist_apply_impulse(normal, iA, iB, a.get(N + 2), vA, vB);
    }
    static void solve(const Inertia<F>& iA, const Inertia<F>& iB, float dt, float inverseDt, const Rows<F>& p, const Rows<F>& a, Velocity<F>& vA, Velocity<F>& vB) {
        V3<F> normal = p.get3(L::kNormal), offsetB = p.get3(L::kOffsetB);
        F friction = p.get(L::kFriction), maxRecovery = p.get(L::kMaxRecovery);
        F positionErrorToVelocity, effectiveMassCFMScale, softnessImpulseScale;
        compute_springiness(p.get(L::kAngularFrequency), p.get(L::kTwiceDampingRatio), dt, positionErrorToVelocity, effectiveMassCFMScale, softnessImpulseScale);
        F inverseDtWide = bc<F>(inverseDt);
        V3<F> offs[N]; F depths[N]; F pen[N];
        for (int i = 0; i < N; ++i) { offs[i] = p.get3(4 * i); depths[i] = p.get(4 * i + 3); pen[i] = a.get(2 + i); }
        for (int i = 0; i < N; ++i)
            penetration_solve(iA, iB, normal, offs[i], sub(offs[i], offsetB), depths[i], positionErrorToVelocity, effectiveMassCFMScale, maxRecovery, inverseDtWide,
                              softnessImpulseScale, pen[i], vA, vB);
        V3<F> x, z;
        build_orthonormal_basis(normal, x, z);
        V2<F> tangent = a.get2(0);
        F twist = a.get(N + 2);
        if (N == 1) {
            F maximumTangentImpulse = friction * pen[0];
            V3<F> centerB = sub(offs[0], offsetB);
            tangent_solve(x, z, offs[0], centerB, iA, iB, maximumTangentImpulse, tangent, vA, vB);
            F maximumTwistImpulse = friction * pen[0] * vmax(bc<F>(0.0f), depths[0]);
            twist_solve(normal, iA, iB, maximumTwistImpulse, twist, vA, vB);
        } else {
            F premultiplied = bc<F>(1.0f / N) * friction;
            F penSum = pen[0];
            for (int i = 1; i < N; ++i) penSum = penSum + pen[i];
            F maximumTangentImpulse = premultiplied * penSum;
            V3<F> centerA = friction_center<F, N>(offs, depths);
            V3<F> centerB = sub(centerA, offsetB);
            tangent_solve(x, z, centerA, centerB, iA, iB, maximumTangentImpulse, tangent, vA, vB);
            F twistSum = pen[0] * distance(centerA, offs[0]);
            for (int i = 1; i < N; ++i) twistSum = twistSum + pen[i] * distance(centerA, offs[i]);
            F maximumTwistImpulse = premultiplied * twistSum;
            twist_solve(normal, iA, iB, maximumTwistImpulse, twist, vA, vB);
        }
        a.set2(0, tangent);
        for (int i = 0; i < N; ++i) a.set(2 + i, pen[i]);
        a.set(N + 2, twist);
    }
    static void incremental_update(float dt, const Velocity<F>& vA, const Velocity<F>& vB, const Rows<F>& p) {
        V3<F> normal = p.get3(L::kNormal), offsetB = p.get3(L::kOffsetB);
        F dtw = bc<F>(dt);
        for (int i = 0; i < N; ++i) {
            F depth = p.get(4 * i + 3);
            update_penetration_depth(dtw, p.get3(4 * i), offsetB, normal, vA, vB, depth);
            p.set(4 * i + 3, depth);
        }
    }
};

// One-body convex: e.g. Contact1OneBodyFunctions, ContactConvexTypes.cs:L292-329 (N=2: L441-486).
template <class F, int N> struct ConvexOneBody {
    typedef ConvexLayout<N, false> L;
    static void warm_start(const Inertia<F>& iA, const Rows<F>& p, const Rows<F>& a, Velocity<F>& vA) {
        V3<F> normal = p.get3(L::kNormal);
        V3<F> x, z;
        build_orthonormal_basis(normal, x, z);
        V3<F> offs[N]; F depths[N];
        for (int i = 0; i < N; ++i) { offs[i] = p.get3(4 * i); depths[i] = p.get(4 * i + 3); }
        V3<F> centerA = (N == 1) ? offs[0] : friction_center<F, N>(offs, depths);
        tangent1_warm_start(x, z, centerA, iA, a.get2(0), vA);
        for (int i = 0; i < N; ++i) penetration1_warm_start(iA, normal, offs[i], a.get(2 + i), vA);
        twist1_apply_impulse(normal, iA, a.get(N + 2), vA);
    }
    static void solve(const Inertia<F>& iA, float dt, float inverseDt, const Rows<F>& p, const Rows<F>& a, Velocity<F>& vA) {
        V3<F> normal = p.get3(L::kNormal);
        F friction = p.get(L::kFriction), maxRecovery = p.get(L::kMaxRecovery);
        F positionErrorToVelocity, effectiveMassCFMScale, softnessImpulseScale;
        compute_springiness(p.get(L::kAngularFrequency), p.get(L::kTwiceDampingRatio), dt, positionErrorToVelocity, effectiveMassCFMScale, softnessImpulseScale);
        F inverseDtWide = bc<F>(inverseDt);
        V3<F> offs[N]; F depths[N]; F pen[N];
        for (int i = 0; i < N; ++i) { offs[i] = p.get3(4 * i); depths[i] = p.get(4 * i + 3); pen[i] = a.get(2 + i); }
        for (int i = 0; i < N; ++i)
            penetration1_solve(iA, normal, offs[i], depths[i], positionErrorToVelocity, effectiveMassCFMScale, maxRecovery, inverseDtWide, softnessImpulseScale, pen[i], vA);
        V3<F> x, z;
        build_orthonormal_basis(normal, x, z);
        V2<F> tangent = a.get2(0);
        F twist = a.get(N + 2);
        if (N == 1) {
            F maximumTangentImpulse = friction * pen[0];
            tangent1_solve(x, z, offs[0], iA, maximumTangentImpulse, tangent, vA);
            F maximumTwistImpulse = friction * pen[0] * vmax(bc<F>(0.0f), depths[0]);
            twist1_solve(normal, iA, maximumTwistImpulse, twist, vA);
        } else {
            F premultiplied = bc<F>(1.0f / N) * friction;
            F penSum = pen[0];
            for (int i = 1; i < N; ++i) penSum = penSum + pen[i];
            F maximumTangentImpulse = premultiplied * penSum;
            V3<F> centerA = friction_center<F, N>(offs, depths);
            tangent1_solve(x, z, centerA, iA, maximumTangentImpulse, tangent, vA);
            F twistSum = pen[0] * distance(centerA, offs[0]);
            for (int i = 1; i < N; ++i) twistSum = twistSum + pen[i] * distance(centerA, offs[i]);
            F maximumTwistImpulse = premultiplied * twistSum;
            twist1_solve(normal, iA, maximumTwistImpulse, twist, vA);
        }
        a.set2(0, tangent);
        for (int i = 0; i < N; ++i) a.set(2 + i, pen[i]);
        a.set(N + 2, twist);
    }
    static void incremental_update(float dt, const Velocity<F>& vA, const Rows<F>& p) {
        V3<F> normal = p.get3(L::kNormal);
        F dtw = bc<F>(dt);
        for (int i = 0; i < N; ++i) {
            F depth = p.get(4 * i + 3);
            update_penetration_depth1(dtw, p.get3(4 * i), normal, vA, depth);
            p.set(4 * i + 3, depth);
        }
    }
};

// ---- Nonconvex manifold constraints : Contact/ContactNonconvexCommon.cs:L171-299, ContactNonconvexTypes.cs -------
// Prestep rows: [material 0..3 = FrictionCoefficient, AngularFrequency, TwiceDampingRatio, MaximumRecoveryVelocity]
//               [offsetB 4..6 (two body only)] [contact i: Offset xyz, Depth, Normal xyz] (7 rows each)
// Accumulated impulses: per contact [tangent xy, penetration] (3 rows each)
template <int N, bool TwoBody> struct NonconvexLayout {
    static constexpr int kOffsetB = 4;
    static constexpr int kContacts = TwoBody ? 7 : 4;
    static constexpr int kPrestepRows = kContacts + 7 * N;
    static constexpr int kImpulseRows = 3 * N;
};

template <class F, int N> struct NonconvexTwoBody {
    typedef NonconvexLayout<N, true> L;
    // ContactNonconvexCommon.cs:L246-261
    static void warm_start(const Inertia<F>& iA, const Inertia<F>& iB, const Rows<F>& p, const Rows<F>& a, Velocity<F>& vA, Velocity<F>& vB) {
        V3<F> offsetB = p.get3(L::kOffsetB);
        for (int i = 0; i < N; ++i) {
            int c = L::kContacts + 7 * i;
            V3<F> offset = p.get3(c), normal = p.get3(c + 4);
            V3<F> x, z;
            build_orthonormal_basis(normal, x, z);
            V3<F> contactOffsetB = sub(offset, offsetB);
            tangent_warm_start(x, z, offset, contactOffsetB, iA, iB, a.get2(3 * i), vA, vB);
            penetration_warm_start(iA, iB, normal, offset, contactOffsetB, a.get(3 * i + 2), vA, vB);
        }
    }
    // L263-283
    static void solve(const Inertia<F>& iA, const Inertia<F>& iB, float dt, float inverseDt, const Rows<F>& p, const Rows<F>& a, Velocity<F>& vA, Velocity<F>& vB) {
        V3<F> offsetB = p.get3(L::kOffsetB);
        F friction = p.get(0), maxRecovery = p.get(3);
        F positionErrorToVelocity, effectiveMassCFMScale, softnessImpulseScale;
        compute_springiness(p.get(1), p.get(2), dt, positionErrorToVelocity, effectiveMassCFMScale, softnessImpulseScale);
        F inverseDtWide = bc<F>(inverseDt);
        for (int i = 0; i < N; ++i) {
            int c = L::kContacts + 7 * i;
            V3<F> offset = p.get3(c), normal = p.get3(c + 4);
            F depth = p.get(c + 3);
            V2<F> tangent = a.get2(3 * i);
            F pen = a.get(3 * i + 2);
            V3<F> contactOffsetB = sub(offset, offsetB);
            penetration_solve(iA, iB, normal, offset, contactOffsetB, depth, positionErrorToVelocity, effectiveMassCFMScale, maxRecovery, inverseDtWide, softnessImpulseScale, pen, vA, vB);
            V3<F> x, z;
            build_orthonormal_basis(normal, x, z);
            F maximumTangentImpulse = friction * pen;
            tangent_solve(x, z, offset, contactOffsetB, iA, iB, maximumTangentImpulse, tangent, vA, vB);
            a.set2(3 * i, tangent);
            a.set(3 * i + 2, pen);
        }
    }
    // L287-297
    static void incremental_update(float dt, const Velocity<F>& vA, const Velocity<F>& vB, const Rows<F>& p) {
        V3<F> offsetB = p.get3(L::kOffsetB);
        F dtw = bc<F>(dt);
        for (int i = 0; i < N; ++i) {
            int c = L::kContacts + 7 * i;
            F depth = p.get(c + 3);
            update_penetration_depth(dtw, p.get3(c), offsetB, p.get3(c + 4), vA, vB, depth);
            p.set(c + 3, depth);
        }
    }
};

template <class F, int N> struct NonconvexOneBody {
    typedef NonconvexLayout<N, false> L;
    // ContactNonconvexCommon.cs:L186-199
    static void warm_start(const Inertia<F>& iA, const Rows<F>& p, const Rows<F>& a, Velocity<F>& vA) {
        for (int i = 0; i < N; ++i) {
            int c = L::kContacts + 7 * i;
            V3<F> offset = p.get3(c), normal = p.get3(c + 4);
            V3<F> x, z;
            build_orthonormal_basis(normal, x, z);
            tangent1_warm_start(x, z, offset, iA, a.get2(3 * i), vA);
            penetration1_warm_start(iA, normal, offset, a.get(3 * i + 2), vA);
        }
    }
    // L201-219
    static void solve(const Inertia<F>& iA, float dt, float inverseDt, const Rows<F>& p, const Rows<F>& a, Velocity<F>& vA) {
        F friction = p.get(0), maxRecovery = p.get(3);
        F positionErrorToVelocity, effectiveMassCFMScale, softnessImpulseScale;
        compute_springiness(p.get(1), p.get(2), dt, positionErrorToVelocity, effectiveMassCFMScale, softnessImpulseScale);
        F inverseDtWide = bc<F>(inverseDt);
        for (int i = 0; i < N; ++i) {
            int c = L::kContacts + 7 * i;
            V3<F> offset = p.get3(c), normal = p.get3(c + 4);
            F depth = p.get(c + 3);
            V2<F> tangent = a.get2(3 * i);
            F pen = a.get(3 * i + 2);
            penetration1_solve(iA, normal, offset, depth, positionErrorToVelocity, effectiveMassCFMScale, maxRecovery, inverseDtWide, softnessImpulseScale, pen, vA);
            V3<F> x, z;
            build_orthonormal_basis(normal, x, z);
            F maximumTangentImpulse = friction * pen;
            tangent1_solve(x, z, offset, iA, maximumTangentImpulse, tangent, vA);
            a.set2(3 * i, tangent);
            a.set(3 * i + 2, pen);
        }
    }
    // L231-239
    static void incremental_update(float dt, const Velocity<F>& vA, const Rows<F>& p) {
        F dtw = bc<F>(dt);
        for (int i = 0; i < N; ++i) {
            int c = L::kContacts + 7 * i;
            F depth = p.get(c + 3);
            update_penetration_depth1(dtw, p.get3(c), p.get3(c + 4), vA, depth);
            p.set(c + 3, depth);
        }
    }
};

}  // namespace bepu_oracle
