// Contact constraint functions for the sm_90a solver kernels: convex manifolds with 1-4 contacts and nonconvex
// manifolds with 2-4 contacts, one- and two-body (type ids 0-10, 15-17).
// Reference behaviour: BepuPhysics/Constraints/Contact/{PenetrationLimit,PenetrationLimitOneBody,TangentFriction,
// TangentFrictionOneBody,TwistFriction,TwistFrictionOneBody,ContactConvexTypes,ContactNonconvexCommon}.cs.
//
// Data access: one thread = one constraint. `p` / `a` point at this lane's element of row 0 of the bundle's prestep /
// accumulated-impulse block in the device AOSOA-32 layout; row r of the lane is p[r * 32] (a 128-B coalesced line per
// warp per row).
#pragma once
#include "bepu_device_math.cuh"

namespace BEPU_NS {

constexpr int kLanes = 32;

// Row accessors. A constraint function sees its prestep rows through `P` and its accumulated impulses through `A`:
//   GlobalRows / GlobalAcc : straight from the AOSOA-32 arrays in HBM. Prestep rows are read once per stage: load through L2 only
//                            (ld.global.cg): an L1 line filled
//                            before IncrementallyUpdateForSubstep rewrote a depth row would be stale.
//   StagedRows / StagedAcc : the bundle's prestep + impulse block was bulk-copied (cp.async.bulk, one transaction per block) into this
//                            warp's shared-memory slab; reads are conflict-free LDS (lane stride 4 B, row stride 128 B), impulse writes go
//                            straight back to HBM.
struct GlobalRows { const float* ptr; };
struct GlobalAcc { float* ptr; };
struct StagedRows { uint32_t addr, bar, parity; };    // shared-space byte address of this lane's element of row 0; the mbarrier the bulk copies complete on and the phase parity to wait for (0 for a single-use barrier)
struct StagedAcc { uint32_t addr; float* ptr; };      // read staged copy, write global
BEPU_DI float lds_f32(uint32_t addr) {
    float v;
    asm("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr));
    return v;
}
// Blocks until the rows behind an accessor may be read: the staged block lands asynchronously (phase 0 of the slab's single-use mbarrier).
BEPU_DI void rows_ready(GlobalRows) {}
BEPU_DI void rows_ready(StagedRows p) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "MBAR_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra MBAR_DONE;\n"
        "bra MBAR_WAIT;\n"
        "MBAR_DONE:\n"
        "}\n" ::"r"(p.bar), "r"(p.parity)
        : "memory");
}
BEPU_DI float ldrow(const float* p, int r) { return __ldcg(p + r * kLanes); }  // raw pointer form (IncrementallyUpdateForSubstep rewrites rows in place)
BEPU_DI float ldrow(GlobalRows p, int r) { return __ldcg(p.ptr + r * kLanes); }
BEPU_DI float ldrow(StagedRows p, int r) { return lds_f32(p.addr + r * (kLanes * 4)); }
template <class PR> BEPU_DI V3 ldrow3(PR p, int r) { return {ldrow(p, r), ldrow(p, r + 1), ldrow(p, r + 2)}; }
template <class PR> BEPU_DI Q4 ldrow4(PR p, int r) { return {ldrow(p, r), ldrow(p, r + 1), ldrow(p, r + 2), ldrow(p, r + 3)}; }
BEPU_DI float ldacc(GlobalAcc a, int r) { return a.ptr[r * kLanes]; }
BEPU_DI void stacc(GlobalAcc a, int r, float v) { a.ptr[r * kLanes] = v; }
BEPU_DI float ldacc(StagedAcc a, int r) { return lds_f32(a.addr + r * (kLanes * 4)); }
BEPU_DI void stacc(StagedAcc a, int r, float v) { __stcs(a.ptr + r * kLanes, v); }  // streaming store: read again only after the whole set went by

// ---- two-body penetration limit: PenetrationLimit.cs ----
BEPU_DI void penetration_apply(const Inertia& iA, const Inertia& iB, V3 normal, V3 angularA, V3 angularB, float impulse, Velocity& vA, Velocity& vB) {  // L45-65
    V3 dLinA = normal * (impulse * iA.inv_mass);
    V3 dAngA = transform(angularA * impulse, iA.t);
    V3 dLinB = normal * (impulse * iB.inv_mass);
    V3 dAngB = transform(angularB * impulse, iB.t);
    vA.lin = vA.lin + dLinA;
    vA.ang = vA.ang + dAngA;
    vB.lin = vB.lin - dLinB;
    vB.ang = vB.ang + dAngB;
}
BEPU_DI void penetration_warm_start(const Inertia& iA, const Inertia& iB, V3 normal, V3 offsetA, V3 offsetB, float accumulated, Velocity& vA, Velocity& vB) {  // L67-75
    penetration_apply(iA, iB, normal, cross(offsetA, normal), cross(normal, offsetB), accumulated, vA, vB);
}
BEPU_DI void penetration_solve(const Inertia& iA, const Inertia& iB, V3 normal, V3 offsetA, V3 offsetB, float depth, const Springiness& sp, float maxRecovery,
                               float inverseDt, float& accumulated, Velocity& vA, Velocity& vB) {  // L78-131, L10-26
    V3 angularA = cross(offsetA, normal);
    V3 angularB = cross(normal, offsetB);
    float angularA0 = vector_sandwich(angularA, iA.t);
    float angularB0 = vector_sandwich(angularB, iB.t);
    float linear = iA.inv_mass + iB.inv_mass;
    float effectiveMass = sp.effective_mass_cfm_scale / (linear + angularA0 + angularB0);
    float biasVelocity = fmin_ps(depth * inverseDt, fmin_ps(depth * sp.position_error_to_velocity, maxRecovery));
    float csvaLinear = dot(vA.lin, normal);
    float csvaAngular = dot(vA.ang, angularA);
    float negatedCSVBLinear = dot(vB.lin, normal);
    float csvbAngular = dot(vB.ang, angularB);
    float negatedCSI = accumulated * sp.softness_impulse_scale + (csvaLinear - negatedCSVBLinear + csvaAngular + csvbAngular - biasVelocity) * effectiveMass;
    float previous = accumulated;
    accumulated = fmax_ps(0.0f, accumulated - negatedCSI);
    penetration_apply(iA, iB, normal, angularA, angularB, accumulated - previous, vA, vB);
}
BEPU_DI float updated_depth(float dt, V3 contactOffsetA, V3 offsetB, V3 normal, const Velocity& vA, const Velocity& vB, float depth) {  // L28-43
    V3 contactVelocityA = cross(vA.ang, contactOffsetA) + vA.lin;
    V3 contactOffsetB = contactOffsetA - offsetB;
    V3 contactVelocityB = cross(vB.ang, contactOffsetB) + vB.lin;
    float estimatedDepthChangeVelocity = dot(normal, contactVelocityA - contactVelocityB);
    return depth - estimatedDepthChangeVelocity * dt;
}

// ---- one-body penetration limit: PenetrationLimitOneBody.cs ----
BEPU_DI void penetration1_apply(const Inertia& iA, V3 normal, V3 angularA, float impulse, Velocity& vA) {
    V3 dLinA = normal * (impulse * iA.inv_mass);
    V3 dAngA = transform(angularA * impulse, iA.t);
    vA.lin = vA.lin + dLinA;
    vA.ang = vA.ang + dAngA;
}
BEPU_DI void penetration1_solve(const Inertia& iA, V3 normal, V3 offsetA, float depth, const Springiness& sp, float maxRecovery, float inverseDt, float& accumulated,
                                Velocity& vA) {
    V3 angularA = cross(offsetA, normal);
    float angularA0 = vector_sandwich(angularA, iA.t);
    float effectiveMass = sp.effective_mass_cfm_scale / (iA.inv_mass + angularA0);
    float biasVelocity = fmin_ps(depth * inverseDt, fmin_ps(depth * sp.position_error_to_velocity, maxRecovery));
    float csvaLinear = dot(vA.lin, normal);
    float csvaAngular = dot(vA.ang, angularA);
    float negatedCSI = accumulated * sp.softness_impulse_scale + (csvaLinear + csvaAngular - biasVelocity) * effectiveMass;
    float previous = accumulated;
    accumulated = fmax_ps(0.0f, accumulated - negatedCSI);
    penetration1_apply(iA, normal, angularA, accumulated - previous, vA);
}
BEPU_DI float updated_depth1(float dt, V3 contactOffset, V3 normal, const Velocity& v, float depth) {
    V3 contactVelocity = cross(v.ang, contactOffset) + v.lin;
    return depth - dot(normal, contactVelocity) * dt;
}

// ---- tangent friction: TangentFriction.cs, TangentFrictionOneBody.cs ----
struct TangentJacobians { M23 linearA, angularA, angularB; };
BEPU_DI TangentJacobians tangent_jacobians(V3 tX, V3 tY, V3 offsetA, V3 offsetB) {  // L17-27
    TangentJacobians j;
    j.linearA = {tX, tY};
    j.angularA = {cross(offsetA, tX), cross(offsetA, tY)};
    j.angularB = {cross(tX, offsetB), cross(tY, offsetB)};
    return j;
}
BEPU_DI void tangent_apply(const TangentJacobians& j, const Inertia& iA, const Inertia& iB, V2 impulse, Velocity& vA, Velocity& vB) {  // L29-46
    V3 linearImpulseA = transform(impulse, j.linearA);
    V3 angularImpulseA = transform(impulse, j.angularA);
    V3 angularImpulseB = transform(impulse, j.angularB);
    vA.lin = vA.lin + linearImpulseA * iA.inv_mass;
    vA.ang = vA.ang + transform(angularImpulseA, iA.t);
    vB.lin = vB.lin - linearImpulseA * iB.inv_mass;
    vB.ang = vB.ang + transform(angularImpulseB, iB.t);
}
BEPU_DI void tangent_solve(V3 tX, V3 tY, V3 offsetA, V3 offsetB, const Inertia& iA, const Inertia& iB, float maximumImpulse, V2& accumulated, Velocity& vA, Velocity& vB) {  // L82-100, L48-70
    TangentJacobians j = tangent_jacobians(tX, tY, offsetA, offsetB);
    Sym2 linear = sandwich_scale(j.linearA, iA.inv_mass) + sandwich_scale(j.linearA, iB.inv_mass);
    Sym2 angular = matrix_sandwich(j.angularA, iA.t) + matrix_sandwich(j.angularB, iB.t);
    Sym2 effectiveMass = invert(linear + angular);
    V2 csvaLinear = transform_by_transpose(vA.lin, j.linearA);
    V2 csvaAngular = transform_by_transpose(vA.ang, j.angularA);
    V2 csvbLinear = transform_by_transpose(vB.lin, j.linearA);
    V2 csvbAngular = transform_by_transpose(vB.ang, j.angularB);
    V2 csv = (csvbLinear - csvaLinear) - (csvaAngular + csvbAngular);
    V2 csi = transform(csv, effectiveMass);
    V2 previous = accumulated;
    accumulated = accumulated + csi;
    float magnitude = length(accumulated);
    float scl = fmin_ps(1.0f, maximumImpulse / fmax_ps(1e-16f, magnitude));
    accumulated = accumulated * scl;
    tangent_apply(j, iA, iB, accumulated - previous, vA, vB);
}
BEPU_DI void tangent1_apply(const M23& linearA, const M23& angularA, const Inertia& iA, V2 impulse, Velocity& vA) {
    V3 linearImpulseA = transform(impulse, linearA);
    V3 angularImpulseA = transform(impulse, angularA);
    vA.lin = vA.lin + linearImpulseA * iA.inv_mass;
    vA.ang = vA.ang + transform(angularImpulseA, iA.t);
}
BEPU_DI void tangent1_solve(V3 tX, V3 tY, V3 offsetA, const Inertia& iA, float maximumImpulse, V2& accumulated, Velocity& vA) {
    M23 linearA{tX, tY};
    M23 angularA{cross(offsetA, tX), cross(offsetA, tY)};
    Sym2 effectiveMass = invert(sandwich_scale(linearA, iA.inv_mass) + matrix_sandwich(angularA, iA.t));
    V2 csv = transform_by_transpose(vA.lin, linearA) + transform_by_transpose(vA.ang, angularA);
    V2 negativeCSI = transform(csv, effectiveMass);
    V2 previous = accumulated;
    accumulated = accumulated - negativeCSI;
    float magnitude = length(accumulated);
    float scl = fmin_ps(1.0f, maximumImpulse / fmax_ps(1e-16f, magnitude));
    accumulated = accumulated * scl;
    tangent1_apply(linearA, angularA, iA, accumulated - previous, vA);
}

// ---- twist friction: TwistFriction.cs, TwistFrictionOneBody.cs ----
BEPU_DI void twist_apply(V3 axis, const Inertia& iA, const Inertia& iB, float impulse, Velocity& vA, Velocity& vB) {
    V3 worldImpulseA = axis * impulse;
    vA.ang = vA.ang + transform(worldImpulseA, iA.t);
    vB.ang = vB.ang - transform(worldImpulseA, iB.t);
}
BEPU_DI void twist_solve(V3 axis, const Inertia& iA, const Inertia& iB, float maximumImpulse, float& accumulated, Velocity& vA, Velocity& vB) {
    float inverseEffectiveMass = vector_sandwich(axis, iA.t) + vector_sandwich(axis, iB.t);
    float effectiveMass = (0.0f == inverseEffectiveMass) ? 0.0f : 1.0f / inverseEffectiveMass;
    float negatedCSI = (dot(vA.ang, axis) - dot(vB.ang, axis)) * effectiveMass;
    float previous = accumulated;
    accumulated = fmin_ps(maximumImpulse, fmax_ps(-maximumImpulse, accumulated - negatedCSI));
    twist_apply(axis, iA, iB, accumulated - previous, vA, vB);
}
BEPU_DI void twist1_apply(V3 axis, const Inertia& iA, float impulse, Velocity& vA) { vA.ang = vA.ang + transform(axis * impulse, iA.t); }
BEPU_DI void twist1_solve(V3 axis, const Inertia& iA, float maximumImpulse, float& accumulated, Velocity& vA) {
    float angularA = vector_sandwich(axis, iA.t);
    float effectiveMass = (0.0f == angularA) ? 0.0f : 1.0f / angularA;
    float negativeCSI = dot(vA.ang, axis) * effectiveMass;
    float previous = accumulated;
    accumulated = fmin_ps(maximumImpulse, fmax_ps(-maximumImpulse, accumulated - negativeCSI));
    twist1_apply(axis, iA, accumulated - previous, vA);
}

// ---- convex manifolds: ContactConvexTypes.cs (generated per contact count; here one template) ----
// prestep rows  one body: [contact i: OffsetA xyz, Depth]x N, Normal xyz, Friction, AngularFrequency, TwiceDampingRatio, MaxRecovery
//               two body: [contact i]x N, OffsetB xyz, Normal xyz, Friction, AngularFrequency, TwiceDampingRatio, MaxRecovery
// impulse rows: Tangent xy, Penetration[N], Twist
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

// FrictionHelpers.ComputeFrictionCenter, ContactConvexTypes.cs:L124-196
template <int N> BEPU_DI V3 friction_center(const V3 (&offs)[N], const float (&depths)[N]) {
    float w[N];
#pragma unroll
    for (int i = 0; i < N; ++i) w[i] = depths[i] < 0.0f ? 0.0f : 1.0f;
    float weightSum = w[0];
#pragma unroll
    for (int i = 1; i < N; ++i) weightSum = weightSum + w[i];
    bool useFallback = weightSum == 0.0f;
    weightSum = useFallback ? (float)N : weightSum;
    float inverseWeightSum = 1.0f / weightSum;
    V3 c[N];
#pragma unroll
    for (int i = 0; i < N; ++i) c[i] = offs[i] * (useFallback ? inverseWeightSum : w[i] * inverseWeightSum);
    if constexpr (N == 2) return c[0] + c[1];
    else if constexpr (N == 3) return (c[0] + c[1]) + c[2];
    else return (c[0] + c[1]) + (c[2] + c[3]);
}

template <int N> struct ConvexTwoBody {
    typedef ConvexLayout<N, true> L;
    static constexpr int kBodies = 2;
    static constexpr int kPrestepRows = L::kPrestepRows;
    static constexpr int kImpulseRows = L::kImpulseRows;
    static constexpr bool kIncremental = true;
    static constexpr bool kNeedsPose = false;

    template <class PR, class AR> BEPU_DI static void warm_start(const Inertia& iA, const Inertia& iB, PR p, AR a, Velocity& vA, Velocity& vB) {  // e.g. L1473-1486
        V3 normal = ldrow3(p, L::kNormal), offsetB = ldrow3(p, L::kOffsetB);
        V3 x, z;
        build_orthonormal_basis(normal, x, z);
        V3 offs[N];
        float depths[N];
#pragma unroll
        for (int i = 0; i < N; ++i) { offs[i] = ldrow3(p, 4 * i); depths[i] = ldrow(p, 4 * i + 3); }
        V3 centerA;
        if constexpr (N == 1) centerA = offs[0]; else centerA = friction_center<N>(offs, depths);
        V3 centerB = centerA - offsetB;
        tangent_apply(tangent_jacobians(x, z, centerA, centerB), iA, iB, V2{ldacc(a, 0), ldacc(a, 1)}, vA, vB);
        // the per-contact rows as a real loop (smaller instruction footprint) -- rows re-read by index, same operations in the same order
#pragma unroll 1
        for (int i = 0; i < N; ++i) {
            V3 offset = ldrow3(p, 4 * i);
            penetration_warm_start(iA, iB, normal, offset, offset - offsetB, ldacc(a, 2 + i), vA, vB);
        }
        twist_apply(normal, iA, iB, ldacc(a, N + 2), vA, vB);
    }
    template <class PR, class AR> BEPU_DI static void solve(const Inertia& iA, const Inertia& iB, float dt, float inverseDt, PR p, AR a, Velocity& vA, Velocity& vB) {  // e.g. L1488-1513
        V3 normal = ldrow3(p, L::kNormal), offsetB = ldrow3(p, L::kOffsetB);
        float friction = ldrow(p, L::kFriction), maxRecovery = ldrow(p, L::kMaxRecovery);
        Springiness sp = compute_springiness(ldrow(p, L::kAngularFrequency), ldrow(p, L::kTwiceDampingRatio), dt);
        if constexpr (N > 1) {
            // The N penetration rows as a real loop (measured -4 % per step: the straight-line version paced the warp by instruction fetch). The friction centre is a pure function of the prestep rows, so
            // it moves in front; the two friction sums accumulate left to right exactly like the unrolled expressions below.
            V3 offs[N];
            float depths[N];
#pragma unroll
            for (int i = 0; i < N; ++i) { offs[i] = ldrow3(p, 4 * i); depths[i] = ldrow(p, 4 * i + 3); }
            const V3 centerA = friction_center<N>(offs, depths);
            float penSum = 0.0f, twistSum = 0.0f;
#pragma unroll 1
            for (int i = 0; i < N; ++i) {
                V3 offset = ldrow3(p, 4 * i);
                float pen = ldacc(a, 2 + i);
                penetration_solve(iA, iB, normal, offset, offset - offsetB, ldrow(p, 4 * i + 3), sp, maxRecovery, inverseDt, pen, vA, vB);
                stacc(a, 2 + i, pen);
                const float lever = pen * distance(centerA, offset);
                penSum = i == 0 ? pen : penSum + pen;  // (not 0 + pen: the sign of a zero impulse must survive)
                twistSum = i == 0 ? lever : twistSum + lever;
            }
            V3 x, z;
            build_orthonormal_basis(normal, x, z);
            V2 tangent{ldacc(a, 0), ldacc(a, 1)};
            float twist = ldacc(a, N + 2);
            const float premultiplied = (1.0f / N) * friction;
            tangent_solve(x, z, centerA, centerA - offsetB, iA, iB, premultiplied * penSum, tangent, vA, vB);
            twist_solve(normal, iA, iB, premultiplied * twistSum, twist, vA, vB);
            stacc(a, 0, tangent.x);
            stacc(a, 1, tangent.y);
            stacc(a, N + 2, twist);
        } else
        {
        V3 offs[N];
        float depths[N], pen[N];
#pragma unroll
        for (int i = 0; i < N; ++i) { offs[i] = ldrow3(p, 4 * i); depths[i] = ldrow(p, 4 * i + 3); pen[i] = ldacc(a, 2 + i); }
#pragma unroll
        for (int i = 0; i < N; ++i) penetration_solve(iA, iB, normal, offs[i], offs[i] - offsetB, depths[i], sp, maxRecovery, inverseDt, pen[i], vA, vB);
        V3 x, z;
        build_orthonormal_basis(normal, x, z);
        V2 tangent{ldacc(a, 0), ldacc(a, 1)};
        float twist = ldacc(a, N + 2);
        if constexpr (N == 1) {
            float maximumTangentImpulse = friction * pen[0];
            tangent_solve(x, z, offs[0], offs[0] - offsetB, iA, iB, maximumTangentImpulse, tangent, vA, vB);
            float maximumTwistImpulse = friction * pen[0] * fmax_ps(0.0f, depths[0]);
            twist_solve(normal, iA, iB, maximumTwistImpulse, twist, vA, vB);
        } else {
            float premultiplied = (1.0f / N) * friction;
            float penSum = pen[0];
#pragma unroll
            for (int i = 1; i < N; ++i) penSum = penSum + pen[i];
            V3 centerA = friction_center<N>(offs, depths);
            tangent_solve(x, z, centerA, centerA - offsetB, iA, iB, premultiplied * penSum, tangent, vA, vB);
            float twistSum = pen[0] * distance(centerA, offs[0]);
#pragma unroll
            for (int i = 1; i < N; ++i) twistSum = twistSum + pen[i] * distance(centerA, offs[i]);
            twist_solve(normal, iA, iB, premultiplied * twistSum, twist, vA, vB);
        }
        stacc(a, 0, tangent.x);
        stacc(a, 1, tangent.y);
#pragma unroll
        for (int i = 0; i < N; ++i) stacc(a, 2 + i, pen[i]);
        stacc(a, N + 2, twist);
        }
    }
    BEPU_DI static void incremental_update(float dt, const Velocity& vA, const Velocity& vB, float* p) {  // e.g. L1464-1471
        V3 normal = ldrow3(p, L::kNormal), offsetB = ldrow3(p, L::kOffsetB);
#pragma unroll
        for (int i = 0; i < N; ++i) p[(4 * i + 3) * kLanes] = updated_depth(dt, ldrow3(p, 4 * i), offsetB, normal, vA, vB, ldrow(p, 4 * i + 3));
    }
};

template <int N> struct ConvexOneBody {
    typedef ConvexLayout<N, false> L;
    static constexpr int kBodies = 1;
    static constexpr int kPrestepRows = L::kPrestepRows;
    static constexpr int kImpulseRows = L::kImpulseRows;
    static constexpr bool kIncremental = true;
    static constexpr bool kNeedsPose = false;

    template <class PR, class AR> BEPU_DI static void warm_start(const Inertia& iA, PR p, AR a, Velocity& vA) {  // e.g. L303-309
        V3 normal = ldrow3(p, L::kNormal);
        V3 x, z;
        build_orthonormal_basis(normal, x, z);
        V3 offs[N];
        float depths[N];
#pragma unroll
        for (int i = 0; i < N; ++i) { offs[i] = ldrow3(p, 4 * i); depths[i] = ldrow(p, 4 * i + 3); }
        V3 centerA;
        if constexpr (N == 1) centerA = offs[0]; else centerA = friction_center<N>(offs, depths);
        tangent1_apply(M23{x, z}, M23{cross(centerA, x), cross(centerA, z)}, iA, V2{ldacc(a, 0), ldacc(a, 1)}, vA);
#pragma unroll 1
        for (int i = 0; i < N; ++i) penetration1_apply(iA, normal, cross(ldrow3(p, 4 * i), normal), ldacc(a, 2 + i), vA);
        twist1_apply(normal, iA, ldacc(a, N + 2), vA);
    }
    template <class PR, class AR> BEPU_DI static void solve(const Inertia& iA, float dt, float inverseDt, PR p, AR a, Velocity& vA) {  // e.g. L311-328
        V3 normal = ldrow3(p, L::kNormal);
        float friction = ldrow(p, L::kFriction), maxRecovery = ldrow(p, L::kMaxRecovery);
        Springiness sp = compute_springiness(ldrow(p, L::kAngularFrequency), ldrow(p, L::kTwiceDampingRatio), dt);
        if constexpr (N > 1) {  // see ConvexTwoBody::solve
            V3 offs[N];
            float depths[N];
#pragma unroll
            for (int i = 0; i < N; ++i) { offs[i] = ldrow3(p, 4 * i); depths[i] = ldrow(p, 4 * i + 3); }
            const V3 centerA = friction_center<N>(offs, depths);
            float penSum = 0.0f, twistSum = 0.0f;
#pragma unroll 1
            for (int i = 0; i < N; ++i) {
                V3 offset = ldrow3(p, 4 * i);
                float pen = ldacc(a, 2 + i);
                penetration1_solve(iA, normal, offset, ldrow(p, 4 * i + 3), sp, maxRecovery, inverseDt, pen, vA);
                stacc(a, 2 + i, pen);
                const float lever = pen * distance(centerA, offset);
                penSum = i == 0 ? pen : penSum + pen;
                twistSum = i == 0 ? lever : twistSum + lever;
            }
            V3 x, z;
            build_orthonormal_basis(normal, x, z);
            V2 tangent{ldacc(a, 0), ldacc(a, 1)};
            float twist = ldacc(a, N + 2);
            const float premultiplied = (1.0f / N) * friction;
            tangent1_solve(x, z, centerA, iA, premultiplied * penSum, tangent, vA);
            twist1_solve(normal, iA, premultiplied * twistSum, twist, vA);
            stacc(a, 0, tangent.x);
            stacc(a, 1, tangent.y);
            stacc(a, N + 2, twist);
        } else
        {
        V3 offs[N];
        float depths[N], pen[N];
#pragma unroll
        for (int i = 0; i < N; ++i) { offs[i] = ldrow3(p, 4 * i); depths[i] = ldrow(p, 4 * i + 3); pen[i] = ldacc(a, 2 + i); }
#pragma unroll
        for (int i = 0; i < N; ++i) penetration1_solve(iA, normal, offs[i], depths[i], sp, maxRecovery, inverseDt, pen[i], vA);
        V3 x, z;
        build_orthonormal_basis(normal, x, z);
        V2 tangent{ldacc(a, 0), ldacc(a, 1)};
        float twist = ldacc(a, N + 2);
        if constexpr (N == 1) {
            tangent1_solve(x, z, offs[0], iA, friction * pen[0], tangent, vA);
            twist1_solve(normal, iA, friction * pen[0] * fmax_ps(0.0f, depths[0]), twist, vA);
        } else {
            float premultiplied = (1.0f / N) * friction;
            float penSum = pen[0];
#pragma unroll
            for (int i = 1; i < N; ++i) penSum = penSum + pen[i];
            V3 centerA = friction_center<N>(offs, depths);
            tangent1_solve(x, z, centerA, iA, premultiplied * penSum, tangent, vA);
            float twistSum = pen[0] * distance(centerA, offs[0]);
#pragma unroll
            for (int i = 1; i < N; ++i) twistSum = twistSum + pen[i] * distance(centerA, offs[i]);
            twist1_solve(normal, iA, premultiplied * twistSum, twist, vA);
        }
        stacc(a, 0, tangent.x);
        stacc(a, 1, tangent.y);
#pragma unroll
        for (int i = 0; i < N; ++i) stacc(a, 2 + i, pen[i]);
        stacc(a, N + 2, twist);
        }
    }
    BEPU_DI static void incremental_update(float dt, const Velocity& vA, float* p) {
        V3 normal = ldrow3(p, L::kNormal);
#pragma unroll
        for (int i = 0; i < N; ++i) p[(4 * i + 3) * kLanes] = updated_depth1(dt, ldrow3(p, 4 * i), normal, vA, ldrow(p, 4 * i + 3));
    }
};

// ---- nonconvex manifolds: ContactNonconvexCommon.cs:L171-299 ----
// Every contact of a nonconvex manifold is a self-contained block (own normal, penetration row and friction), so its loops can run rolled.
#define BEPU_CONTACT_LOOP _Pragma("unroll 1")
// prestep rows: Friction, AngularFrequency, TwiceDampingRatio, MaxRecovery, [OffsetB xyz (two body)], [contact i: Offset xyz, Depth, Normal xyz]x N
// impulse rows: [contact i: Tangent xy, Penetration]x N
template <int N, bool TwoBody> struct NonconvexLayout {
    static constexpr int kOffsetB = 4;
    static constexpr int kContacts = TwoBody ? 7 : 4;
    static constexpr int kPrestepRows = kContacts + 7 * N;
    static constexpr int kImpulseRows = 3 * N;
};
template <int N> struct NonconvexTwoBody {
    typedef NonconvexLayout<N, true> L;
    static constexpr int kBodies = 2;
    static constexpr int kPrestepRows = L::kPrestepRows;
    static constexpr int kImpulseRows = L::kImpulseRows;
    static constexpr bool kIncremental = true;
    static constexpr bool kNeedsPose = false;
    template <class PR, class AR> BEPU_DI static void warm_start(const Inertia& iA, const Inertia& iB, PR p, AR a, Velocity& vA, Velocity& vB) {  // L246-261
        V3 offsetB = ldrow3(p, L::kOffsetB);
BEPU_CONTACT_LOOP
        for (int i = 0; i < N; ++i) {
            const int c = L::kContacts + 7 * i;
            V3 offset = ldrow3(p, c), normal = ldrow3(p, c + 4);
            V3 x, z;
            build_orthonormal_basis(normal, x, z);
            V3 contactOffsetB = offset - offsetB;
            tangent_apply(tangent_jacobians(x, z, offset, contactOffsetB), iA, iB, V2{ldacc(a, 3 * i), ldacc(a, 3 * i + 1)}, vA, vB);
            penetration_warm_start(iA, iB, normal, offset, contactOffsetB, ldacc(a, 3 * i + 2), vA, vB);
        }
    }
    template <class PR, class AR> BEPU_DI static void solve(const Inertia& iA, const Inertia& iB, float dt, float inverseDt, PR p, AR a, Velocity& vA, Velocity& vB) {  // L263-283
        V3 offsetB = ldrow3(p, L::kOffsetB);
        float friction = ldrow(p, 0), maxRecovery = ldrow(p, 3);
        Springiness sp = compute_springiness(ldrow(p, 1), ldrow(p, 2), dt);
BEPU_CONTACT_LOOP
        for (int i = 0; i < N; ++i) {
            const int c = L::kContacts + 7 * i;
            V3 offset = ldrow3(p, c), normal = ldrow3(p, c + 4);
            float depth = ldrow(p, c + 3);
            V2 tangent{ldacc(a, 3 * i), ldacc(a, 3 * i + 1)};
            float pen = ldacc(a, 3 * i + 2);
            V3 contactOffsetB = offset - offsetB;
            penetration_solve(iA, iB, normal, offset, contactOffsetB, depth, sp, maxRecovery, inverseDt, pen, vA, vB);
            V3 x, z;
            build_orthonormal_basis(normal, x, z);
            tangent_solve(x, z, offset, contactOffsetB, iA, iB, friction * pen, tangent, vA, vB);
            stacc(a, 3 * i, tangent.x);
            stacc(a, 3 * i + 1, tangent.y);
            stacc(a, 3 * i + 2, pen);
        }
    }
    BEPU_DI static void incremental_update(float dt, const Velocity& vA, const Velocity& vB, float* p) {  // L287-297
        V3 offsetB = ldrow3(p, L::kOffsetB);
#pragma unroll
        for (int i = 0; i < N; ++i) {
            const int c = L::kContacts + 7 * i;
            p[(c + 3) * kLanes] = updated_depth(dt, ldrow3(p, c), offsetB, ldrow3(p, c + 4), vA, vB, ldrow(p, c + 3));
        }
    }
};
template <int N> struct NonconvexOneBody {
    typedef NonconvexLayout<N, false> L;
    static constexpr int kBodies = 1;
    static constexpr int kPrestepRows = L::kPrestepRows;
    static constexpr int kImpulseRows = L::kImpulseRows;
    static constexpr bool kIncremental = true;
    static constexpr bool kNeedsPose = false;
    template <class PR, class AR> BEPU_DI static void warm_start(const Inertia& iA, PR p, AR a, Velocity& vA) {  // L186-199
BEPU_CONTACT_LOOP
        for (int i = 0; i < N; ++i) {
            const int c = L::kContacts + 7 * i;
            V3 offset = ldrow3(p, c), normal = ldrow3(p, c + 4);
            V3 x, z;
            build_orthonormal_basis(normal, x, z);
            tangent1_apply(M23{x, z}, M23{cross(offset, x), cross(offset, z)}, iA, V2{ldacc(a, 3 * i), ldacc(a, 3 * i + 1)}, vA);
            penetration1_apply(iA, normal, cross(offset, normal), ldacc(a, 3 * i + 2), vA);
        }
    }
    template <class PR, class AR> BEPU_DI static void solve(const Inertia& iA, float dt, float inverseDt, PR p, AR a, Velocity& vA) {  // L201-219
        float friction = ldrow(p, 0), maxRecovery = ldrow(p, 3);
        Springiness sp = compute_springiness(ldrow(p, 1), ldrow(p, 2), dt);
BEPU_CONTACT_LOOP
        for (int i = 0; i < N; ++i) {
            const int c = L::kContacts + 7 * i;
            V3 offset = ldrow3(p, c), normal = ldrow3(p, c + 4);
            float depth = ldrow(p, c + 3);
            V2 tangent{ldacc(a, 3 * i), ldacc(a, 3 * i + 1)};
            float pen = ldacc(a, 3 * i + 2);
            penetration1_solve(iA, normal, offset, depth, sp, maxRecovery, inverseDt, pen, vA);
            V3 x, z;
            build_orthonormal_basis(normal, x, z);
            tangent1_solve(x, z, offset, iA, friction * pen, tangent, vA);
            stacc(a, 3 * i, tangent.x);
            stacc(a, 3 * i + 1, tangent.y);
            stacc(a, 3 * i + 2, pen);
        }
    }
    BEPU_DI static void incremental_update(float dt, const Velocity& vA, float* p) {  // L231-239
#pragma unroll
        for (int i = 0; i < N; ++i) {
            const int c = L::kContacts + 7 * i;
            p[(c + 3) * kLanes] = updated_depth1(dt, ldrow3(p, c), ldrow3(p, c + 4), vA, ldrow(p, c + 3));
        }
    }
};

// BatchTypeId -> contact type (Contact/ContactConvexTypes.cs, ContactNonconvexTypes.cs)
#define BEPU_CONTACT_TYPES(X)                                                                                                     \
    X(0, ConvexOneBody<1>) X(1, ConvexOneBody<2>) X(2, ConvexOneBody<3>) X(3, ConvexOneBody<4>)                                   \
    X(4, ConvexTwoBody<1>) X(5, ConvexTwoBody<2>) X(6, ConvexTwoBody<3>) X(7, ConvexTwoBody<4>)                                   \
    X(8, NonconvexOneBody<2>) X(9, NonconvexOneBody<3>) X(10, NonconvexOneBody<4>)                                                \
    X(15, NonconvexTwoBody<2>) X(16, NonconvexTwoBody<3>) X(17, NonconvexTwoBody<4>)

}  // namespace BEPU_NS
