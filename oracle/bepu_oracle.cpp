// ORACLE — test infrastructure only (see bepu_math.h). Driver: body gather/scatter, embedded integration, the substep loop,
// integration responsibilities and the final pose pass, restated from the reference's single-threaded executable spec.
// Parity: the constraint / math / integration functions called from here are pinned to the reference's C# text (oracle/ref_transpile). THIS file's
// driver logic (stage order, integration responsibilities, gather/scatter, bundle loops, the final pose pass, PredictBoundingBoxes' per-body glue,
// impulse redistribution) is pinned to a second, independent restatement of the reference's single-threaded frame that runs on the transpiled
// reference's own arithmetic (tests/reference_frame.py, tests/test_oracle_driver_pinned_to_reference.py), bit for bit on a scene matrix.
#include "bepu_oracle.h"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <vector>
#ifdef _OPENMP
#include <omp.h>
#include <sched.h>
#include <atomic>
#endif

#include "bepu_contacts.h"
#include "bepu_joints.h"
#include "bepu_joints_more.h"

namespace bepu_oracle {

// BepuPhysics/Bodies_GatherScatter.cs:L107-139
static constexpr uint32_t kDynamicLimit = 1u << 30;
static constexpr int32_t kBodyReferenceMask = (int32_t)~((1u << 31) | (1u << 30));

template <class F> struct BodyIn {
    V3<F> pos;
    Q4<F> q;
    Inertia<F> inertia;
};

template <class F> struct TypeOps {
    int bodies = 0, prestep_rows = 0, impulse_rows = 0;
    void (*warm_start)(const BodyIn<F>*, const Rows<F>&, const Rows<F>&, Velocity<F>*) = nullptr;
    void (*solve)(const BodyIn<F>*, float, float, const Rows<F>&, const Rows<F>&, Velocity<F>*) = nullptr;
    void (*incremental)(float, const Velocity<F>*, const Rows<F>&) = nullptr;
};

// ---- adapters from the typed functions to the uniform table -----------------------------------------------------
template <class F, class T> struct Adapt2 {  // two-body contact style: only inertias needed
    static void ws(const BodyIn<F>* b, const Rows<F>& p, const Rows<F>& a, Velocity<F>* v) { T::warm_start(b[0].inertia, b[1].inertia, p, a, v[0], v[1]); }
    static void sv(const BodyIn<F>* b, float dt, float idt, const Rows<F>& p, const Rows<F>& a, Velocity<F>* v) { T::solve(b[0].inertia, b[1].inertia, dt, idt, p, a, v[0], v[1]); }
    static void inc(float dt, const Velocity<F>* v, const Rows<F>& p) { T::incremental_update(dt, v[0], v[1], p); }
};
template <class F, class T> struct Adapt1 {
    static void ws(const BodyIn<F>* b, const Rows<F>& p, const Rows<F>& a, Velocity<F>* v) { T::warm_start(b[0].inertia, p, a, v[0]); }
    static void sv(const BodyIn<F>* b, float dt, float idt, const Rows<F>& p, const Rows<F>& a, Velocity<F>* v) { T::solve(b[0].inertia, dt, idt, p, a, v[0]); }
    static void inc(float dt, const Velocity<F>* v, const Rows<F>& p) { T::incremental_update(dt, v[0], p); }
};
// joint style: full pose + inertia per body; T::warm_start(const BodyIn<F>*, p, a, v), T::solve(const BodyIn<F>*, dt, idt, p, a, v)
template <class F, class T> struct AdaptJ {
    static void ws(const BodyIn<F>* b, const Rows<F>& p, const Rows<F>& a, Velocity<F>* v) {
        T::warm_start(b[0].pos, b[0].q, b[0].inertia, b[1].pos, b[1].q, b[1].inertia, p, a, v[0], v[1]);
    }
    static void sv(const BodyIn<F>* b, float dt, float idt, const Rows<F>& p, const Rows<F>& a, Velocity<F>* v) {
        T::solve(b[0].pos, b[0].q, b[0].inertia, b[1].pos, b[1].q, b[1].inertia, dt, idt, p, a, v[0], v[1]);
    }
};
template <class F, class T> struct AdaptJ1 {
    static void ws(const BodyIn<F>* b, const Rows<F>& p, const Rows<F>& a, Velocity<F>* v) { T::warm_start(b[0].pos, b[0].q, b[0].inertia, p, a, v[0]); }
    static void sv(const BodyIn<F>* b, float dt, float idt, const Rows<F>& p, const Rows<F>& a, Velocity<F>* v) {
        T::solve(b[0].pos, b[0].q, b[0].inertia, dt, idt, p, a, v[0]);
    }
};

// three / four body constraints (AreaConstraint, VolumeConstraint) only touch positions, inverse masses and linear velocities
template <class F, class T> struct AdaptJN {
    static void ws(const BodyIn<F>* b, const Rows<F>& p, const Rows<F>& a, Velocity<F>* v) {
        V3<F> pos[T::kBodies];
        F im[T::kBodies];
        for (int i = 0; i < T::kBodies; ++i) { pos[i] = b[i].pos; im[i] = b[i].inertia.inv_mass; }
        T::warm_start(pos, im, p, a, v);
    }
    static void sv(const BodyIn<F>* b, float dt, float idt, const Rows<F>& p, const Rows<F>& a, Velocity<F>* v) {
        V3<F> pos[T::kBodies];
        F im[T::kBodies];
        for (int i = 0; i < T::kBodies; ++i) { pos[i] = b[i].pos; im[i] = b[i].inertia.inv_mass; }
        T::solve(pos, im, dt, idt, p, a, v);
    }
};
template <class F> struct Registry {
    typedef F Lane;
    TypeOps<F> ops[64];
    template <class T> void contact2(int id) {
        ops[id].bodies = 2; ops[id].prestep_rows = T::L::kPrestepRows; ops[id].impulse_rows = T::L::kImpulseRows;
        ops[id].warm_start = &Adapt2<F, T>::ws; ops[id].solve = &Adapt2<F, T>::sv; ops[id].incremental = &Adapt2<F, T>::inc;
    }
    template <class T> void contact1(int id) {
        ops[id].bodies = 1; ops[id].prestep_rows = T::L::kPrestepRows; ops[id].impulse_rows = T::L::kImpulseRows;
        ops[id].warm_start = &Adapt1<F, T>::ws; ops[id].solve = &Adapt1<F, T>::sv; ops[id].incremental = &Adapt1<F, T>::inc;
    }
    template <class T> void joint2(int id) {
        ops[id].bodies = 2; ops[id].prestep_rows = T::kPrestepRows; ops[id].impulse_rows = T::kImpulseRows;
        ops[id].warm_start = &AdaptJ<F, T>::ws; ops[id].solve = &AdaptJ<F, T>::sv; ops[id].incremental = nullptr;
    }
    template <class T> void joint1(int id) {
        ops[id].bodies = 1; ops[id].prestep_rows = T::kPrestepRows; ops[id].impulse_rows = T::kImpulseRows;
        ops[id].warm_start = &AdaptJ1<F, T>::ws; ops[id].solve = &AdaptJ1<F, T>::sv; ops[id].incremental = nullptr;
    }
    template <class T> void jointN(int id) {
        ops[id].bodies = T::kBodies; ops[id].prestep_rows = T::kPrestepRows; ops[id].impulse_rows = T::kImpulseRows;
        ops[id].warm_start = &AdaptJN<F, T>::ws; ops[id].solve = &AdaptJN<F, T>::sv; ops[id].incremental = nullptr;
    }
    Registry() {
        // BatchTypeId constants: Contact/ContactConvexTypes.cs, ContactNonconvexTypes.cs and each joint file.
        contact1<ConvexOneBody<F, 1>>(0); contact1<ConvexOneBody<F, 2>>(1); contact1<ConvexOneBody<F, 3>>(2); contact1<ConvexOneBody<F, 4>>(3);
        contact2<ConvexTwoBody<F, 1>>(4); contact2<ConvexTwoBody<F, 2>>(5); contact2<ConvexTwoBody<F, 3>>(6); contact2<ConvexTwoBody<F, 4>>(7);
        contact1<NonconvexOneBody<F, 2>>(8); contact1<NonconvexOneBody<F, 3>>(9); contact1<NonconvexOneBody<F, 4>>(10);
        contact2<NonconvexTwoBody<F, 2>>(15); contact2<NonconvexTwoBody<F, 3>>(16); contact2<NonconvexTwoBody<F, 4>>(17);
        register_joints(*this);
        register_joints_more(*this);
    }
};
template <class F> static const Registry<F>& registry() {
    static Registry<F> r;
    return r;
}

// ---- gather / scatter: Bodies_GatherScatter.cs:L267-478 (gather), L484-549 (pose), L553-622 (inertia), L626-753 (velocity) ----
template <class F>
static inline void gather_state(const float* bodies, const int32_t* refs, bool worldInertia, BodyIn<F>& b, Velocity<F>& v) {
    constexpr int PW = LaneTraits<F>::Width;
    for (int l = 0; l < PW; ++l) {
        int32_t enc = refs[l];
        if (enc < 0) {  // empty lane -> zeros
            set_lane(b.q.x, l, 0.f); set_lane(b.q.y, l, 0.f); set_lane(b.q.z, l, 0.f); set_lane(b.q.w, l, 0.f);
            set_lane(b.pos.x, l, 0.f); set_lane(b.pos.y, l, 0.f); set_lane(b.pos.z, l, 0.f);
            set_lane(v.lin.x, l, 0.f); set_lane(v.lin.y, l, 0.f); set_lane(v.lin.z, l, 0.f);
            set_lane(v.ang.x, l, 0.f); set_lane(v.ang.y, l, 0.f); set_lane(v.ang.z, l, 0.f);
            set_lane(b.inertia.t.xx, l, 0.f); set_lane(b.inertia.t.yx, l, 0.f); set_lane(b.inertia.t.yy, l, 0.f);
            set_lane(b.inertia.t.zx, l, 0.f); set_lane(b.inertia.t.zy, l, 0.f); set_lane(b.inertia.t.zz, l, 0.f);
            set_lane(b.inertia.inv_mass, l, 0.f);
            continue;
        }
        const float* s = bodies + (size_t)(enc & kBodyReferenceMask) * 32;
        set_lane(b.q.x, l, s[0]); set_lane(b.q.y, l, s[1]); set_lane(b.q.z, l, s[2]); set_lane(b.q.w, l, s[3]);
        set_lane(b.pos.x, l, s[4]); set_lane(b.pos.y, l, s[5]); set_lane(b.pos.z, l, s[6]);
        set_lane(v.lin.x, l, s[8]); set_lane(v.lin.y, l, s[9]); set_lane(v.lin.z, l, s[10]);
        set_lane(v.ang.x, l, s[12]); set_lane(v.ang.y, l, s[13]); set_lane(v.ang.z, l, s[14]);
        const float* in = s + (worldInertia ? 24 : 16);
        set_lane(b.inertia.t.xx, l, in[0]); set_lane(b.inertia.t.yx, l, in[1]); set_lane(b.inertia.t.yy, l, in[2]);
        set_lane(b.inertia.t.zx, l, in[3]); set_lane(b.inertia.t.zy, l, in[4]); set_lane(b.inertia.t.zz, l, in[5]);
        set_lane(b.inertia.inv_mass, l, in[6]);
    }
}
template <class F> static inline void scatter_velocities(float* bodies, const int32_t* refs, const Velocity<F>& v) {
    constexpr int PW = LaneTraits<F>::Width;
    for (int l = 0; l < PW; ++l) {
        uint32_t enc = (uint32_t)refs[l];
        if (enc >= kDynamicLimit) continue;  // kinematic or empty
        float* s = bodies + (size_t)enc * 32;
        s[8] = get_lane(v.lin.x, l); s[9] = get_lane(v.lin.y, l); s[10] = get_lane(v.lin.z, l);
        s[12] = get_lane(v.ang.x, l); s[13] = get_lane(v.ang.y, l); s[14] = get_lane(v.ang.z, l);
    }
}
template <class F> static inline void scatter_pose(float* bodies, const int32_t* refs, const bool* mask, const V3<F>& pos, const Q4<F>& q) {
    constexpr int PW = LaneTraits<F>::Width;
    for (int l = 0; l < PW; ++l) {
        if (!mask[l]) continue;
        float* s = bodies + (size_t)(refs[l] & kBodyReferenceMask) * 32;
        s[0] = get_lane(q.x, l); s[1] = get_lane(q.y, l); s[2] = get_lane(q.z, l); s[3] = get_lane(q.w, l);
        s[4] = get_lane(pos.x, l); s[5] = get_lane(pos.y, l); s[6] = get_lane(pos.z, l);
    }
}
template <class F> static inline void scatter_world_inertia(float* bodies, const int32_t* refs, const bool* mask, const Inertia<F>& in) {
    constexpr int PW = LaneTraits<F>::Width;
    for (int l = 0; l < PW; ++l) {
        if (!mask[l]) continue;
        float* s = bodies + (size_t)(refs[l] & kBodyReferenceMask) * 32 + 24;
        s[0] = get_lane(in.t.xx, l); s[1] = get_lane(in.t.yx, l); s[2] = get_lane(in.t.yy, l);
        s[3] = get_lane(in.t.zx, l); s[4] = get_lane(in.t.zy, l); s[5] = get_lane(in.t.zz, l);
        s[6] = get_lane(in.inv_mass, l);
    }
}
template <class F> static inline MaskOf<F> make_mask(const bool* m);
template <> inline bool make_mask<float>(const bool* m) { return m[0]; }
template <> inline i8 make_mask<f8>(const bool* m) {
    i8 r = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int i = 0; i < 8; ++i) r[i] = m[i] ? -1 : 0;
    return r;
}

// ---- integration: PoseIntegrator.cs:L99-261, Demos/DemoCallbacks.cs:L79-105 ----------------------------------------
// The optional terms, integrate_velocity_extensions of csrc/bepu_integration.cuh (PerBodyGravityDemo.cs:L57-88: v += a * dt, not damped;
// PlanetDemo.cs:L44-46 in its operation order, with Vector3Wide.Length and Vector3Wide / Vector<float> = multiply by the reciprocal,
// Vector3Wide.cs:L357-363, L573-576).
template <class F>
static inline void apply_velocity_terms(Velocity<F>& v, bool accelerations, const V3<F>& linearAcceleration, const V3<F>& angularAcceleration, float dt, bool pointGravity,
                                        const V3<F>& position, const V3<F>& center, float attractorDt) {
    if (accelerations) {
        v.lin = add(v.lin, scale(linearAcceleration, bc<F>(dt)));
        v.ang = add(v.ang, scale(angularAcceleration, bc<F>(dt)));
    }
    if (pointGravity) {
        V3<F> offset = sub(position, center);
        F distance = length(offset);
        F inverse = bc<F>(1.0f) / vmax(bc<F>(1.0f), distance * distance * distance);
        v.lin = sub(v.lin, scale(scale(offset, bc<F>(attractorDt)), inverse));
    }
}

struct Callbacks {
    float gravity[3];
    float linear_damping, angular_damping;
    int angular_mode;
    bool allow_substeps_unconstrained, integrate_kinematic_velocity;
    oracle_integrator_terms terms{};  // zeroed: no terms
    // PrepareForIntegration products
    float gravity_dt[3];
    float linear_damping_dt, angular_damping_dt;
    float dt, attractor_dt;
    void prepare(float dt) {  // DemoCallbacks.cs:L79-86, PlanetDemo.cs:L36-40
        auto clamp01 = [](float v) { return v < 0.f ? 0.f : (v > 1.f ? 1.f : v); };
        linear_damping_dt = powf(clamp01(1 - linear_damping), dt);
        angular_damping_dt = powf(clamp01(1 - angular_damping), dt);
        for (int i = 0; i < 3; ++i) gravity_dt[i] = gravity[i] * dt;
        this->dt = dt;
        attractor_dt = dt * terms.strength;
    }
    template <class F> void integrate_velocity(Velocity<F>& v) const {  // DemoCallbacks.cs:L99-102
        V3<F> g{bc<F>(gravity_dt[0]), bc<F>(gravity_dt[1]), bc<F>(gravity_dt[2])};
        v.lin = scale(add(v.lin, g), bc<F>(linear_damping_dt));
        v.ang = scale(v.ang, bc<F>(angular_damping_dt));
    }
    // The declarative callback, then the terms of the lanes' bodies at the position the reference hands the callback. refs: the encoded body
    // references of the lanes (negative = empty lane).
    template <class F> void integrate_velocity(Velocity<F>& v, const V3<F>& position, const int32_t* refs) const {
        integrate_velocity(v);
        if (terms.accelerations || terms.point_gravity) integrate_velocity_terms(v, position, refs);
    }
    template <class F> void integrate_velocity_terms(Velocity<F>& v, const V3<F>& position, const int32_t* refs) const {
        constexpr int PW = LaneTraits<F>::Width;
        V3<F> al{bc<F>(0.0f), bc<F>(0.0f), bc<F>(0.0f)}, aa = al;
        if (terms.accelerations)
            for (int l = 0; l < PW; ++l) {
                if (refs[l] < 0) continue;
                const float* a = terms.accelerations + (size_t)(refs[l] & kBodyReferenceMask) * 8;
                set_lane(al.x, l, a[0]); set_lane(al.y, l, a[1]); set_lane(al.z, l, a[2]);
                set_lane(aa.x, l, a[4]); set_lane(aa.y, l, a[5]); set_lane(aa.z, l, a[6]);
            }
        const float* c = terms.center;
        apply_velocity_terms<F>(v, terms.accelerations != nullptr, al, aa, dt, terms.point_gravity != 0, position, V3<F>{bc<F>(c[0]), bc<F>(c[1]), bc<F>(c[2])}, attractor_dt);
    }
};

// PoseIntegrator.cs:L146-164 Integrate(QuaternionWide)
template <class F> static inline Q4<F> integrate_orientation(const Q4<F>& start, const V3<F>& angularVelocity, const F& halfDt) {
    F speed = length(angularVelocity);
    F halfAngle = speed * halfDt;
    F s = sin_approx(halfAngle);
    F scl = s / speed;
    Q4<F> q{angularVelocity.x * scl, angularVelocity.y * scl, angularVelocity.z * scl, cos_approx(halfAngle)};
    Q4<F> end = normalize(concatenate(start, q));
    MaskOf<F> speedValid = gt(speed, bc<F>(1e-15f));
    return sel4<F>(speedValid, end, start);
}
// PoseIntegrator.cs:L166-175
template <class F> static inline Sym3<F> rotate_inverse_inertia(const Sym3<F>& local, const Q4<F>& q) {
    M33<F> r = matrix_from_quaternion(q);
    return rotation_sandwich(r, local);
}
// Matrix3x3Wide.cs Invert (general 3x3, adjugate form), used by the gyroscopic mode.
template <class F> static inline M33<F> invert33(const M33<F>& m) {
    F m11 = m.y.y * m.z.z - m.z.y * m.y.z;
    F m21 = m.y.z * m.z.x - m.z.z * m.y.x;
    F m31 = m.y.x * m.z.y - m.z.x * m.y.y;
    F determinantInverse = bc<F>(1.0f) / (m11 * m.x.x + m21 * m.x.y + m31 * m.x.z);
    F m12 = m.z.y * m.x.z - m.x.y * m.z.z;
    F m22 = m.z.z * m.x.x - m.x.z * m.z.x;
    F m32 = m.z.x * m.x.y - m.x.x * m.z.y;
    F m13 = m.x.y * m.y.z - m.y.y * m.x.z;
    F m23 = m.x.z * m.y.x - m.y.z * m.x.x;
    F m33 = m.x.x * m.y.y - m.y.x * m.x.y;
    M33<F> r;
    r.x.x = m11 * determinantInverse; r.y.x = m21 * determinantInverse; r.z.x = m31 * determinantInverse;
    r.x.y = m12 * determinantInverse; r.y.y = m22 * determinantInverse; r.z.y = m32 * determinantInverse;
    r.x.z = m13 * determinantInverse; r.y.z = m23 * determinantInverse; r.z.z = m33 * determinantInverse;
    return r;
}
// PoseIntegrator.cs:L180-190
template <class F> static inline void fallback_if_inertia_incompatible(const V3<F>& previous, V3<F>& w) {
    F inf = bc<F>(INFINITY);
    MaskOf<F> useNew = mand(lt(vabs(w.x), inf), mand(lt(vabs(w.y), inf), lt(vabs(w.z), inf)));
    w = sel3<F>(useNew, w, previous);
}
// PoseIntegrator.cs:L192-206
template <class F>
static inline void integrate_angular_conserve_momentum(const Q4<F>& previousOrientation, const Sym3<F>& localInverseInertia, const Sym3<F>& worldInverseInertia, V3<F>& w) {
    M33<F> prevR = matrix_from_quaternion(previousOrientation);
    V3<F> localPrevW = transform_by_transposed(w, prevR);
    Sym3<F> localInertiaTensor = invert(localInverseInertia);
    V3<F> localAngularMomentum = transform(localPrevW, localInertiaTensor);
    V3<F> angularMomentum = transform(localAngularMomentum, prevR);
    V3<F> previous = w;
    w = transform(angularMomentum, worldInverseInertia);
    fallback_if_inertia_incompatible(previous, w);
}
// PoseIntegrator.cs:L208-253
template <class F>
static inline void integrate_angular_gyroscopic(const Q4<F>& orientation, const Sym3<F>& localInverseInertia, V3<F>& w, const F& dt) {
    M33<F> R = matrix_from_quaternion(orientation);
    V3<F> localW = transform_by_transposed(w, R);
    Sym3<F> I = invert(localInverseInertia);
    V3<F> localMomentum = transform(localW, I);
    V3<F> residual = scale(cross(localMomentum, localW), dt);
    // Matrix3x3Wide.CreateCrossProduct: X = (0, -v.Z, v.Y), Y = (v.Z, 0, -v.X), Z = (-v.Y, v.X, 0)
    F zero = bc<F>(0.0f);
    M33<F> skewMomentum{{zero, -localMomentum.z, localMomentum.y}, {localMomentum.z, zero, -localMomentum.x}, {-localMomentum.y, localMomentum.x, zero}};
    M33<F> skewVelocity{{zero, -localW.z, localW.y}, {localW.z, zero, -localW.x}, {-localW.y, localW.x, zero}};
    M33<F> transformedSkewVelocity = multiply(skewVelocity, I);
    M33<F> change;
    change.x = scale(sub(transformedSkewVelocity.x, skewMomentum.x), dt);
    change.y = scale(sub(transformedSkewVelocity.y, skewMomentum.y), dt);
    change.z = scale(sub(transformedSkewVelocity.z, skewMomentum.z), dt);
    // jacobian = localInertiaTensor + change (Symmetric3x3Wide + Matrix3x3Wide)
    M33<F> J;
    J.x = {I.xx + change.x.x, I.yx + change.x.y, I.zx + change.x.z};
    J.y = {I.yx + change.y.x, I.yy + change.y.y, I.zy + change.y.z};
    J.z = {I.zx + change.z.x, I.zy + change.z.y, I.zz + change.z.z};
    M33<F> invJ = invert33(J);
    V3<F> newtonStep = transform(residual, invJ);
    localW = sub(localW, newtonStep);
    V3<F> previous = w;
    w = transform(localW, R);
    fallback_if_inertia_incompatible(previous, w);
}

// TypeProcessor.cs:L1204-1248 IntegratePoseAndVelocity; the callback sees the integrated pose (L1244). refs: the lanes' body references.
template <class F>
static inline void integrate_pose_and_velocity(const Callbacks& cb, const Inertia<F>& local, float dt, const MaskOf<F>& mask, V3<F>& pos, Q4<F>& q, Velocity<F>& v, Inertia<F>& world,
                                               const int32_t* refs) {
    F dtWide = bc<F>(dt);
    V3<F> newPosition = add(pos, scale(v.lin, dtWide));
    pos = sel3<F>(mask, newPosition, pos);
    world.inv_mass = local.inv_mass;
    Velocity<F> previousVelocity = v;
    F halfDt = dtWide * bc<F>(0.5f);
    if (cb.angular_mode == 1) {
        Q4<F> previousOrientation = q;
        Q4<F> newOrientation = integrate_orientation(q, v.ang, halfDt);
        q = sel4<F>(mask, newOrientation, q);
        world.t = rotate_inverse_inertia(local.t, q);
        integrate_angular_conserve_momentum(previousOrientation, local.t, world.t, v.ang);
    } else if (cb.angular_mode == 2) {
        Q4<F> newOrientation = integrate_orientation(q, v.ang, halfDt);
        q = sel4<F>(mask, newOrientation, q);
        world.t = rotate_inverse_inertia(local.t, q);
        integrate_angular_gyroscopic(q, local.t, v.ang, dtWide);
    } else {
        Q4<F> newOrientation = integrate_orientation(q, v.ang, halfDt);
        q = sel4<F>(mask, newOrientation, q);
        world.t = rotate_inverse_inertia(local.t, q);
    }
    cb.integrate_velocity(v, pos, refs);
    v.lin = sel3<F>(mask, v.lin, previousVelocity.lin);
    v.ang = sel3<F>(mask, v.ang, previousVelocity.ang);
}
// TypeProcessor.cs:L1251-1283 IntegrateVelocity; the callback sees the current pose (L1276).
template <class F>
static inline void integrate_velocity_only(const Callbacks& cb, const Inertia<F>& local, float dt, const MaskOf<F>& mask, bool conditional, const V3<F>& pos, const Q4<F>& q,
                                           Velocity<F>& v, Inertia<F>& world, const int32_t* refs) {
    world.inv_mass = local.inv_mass;
    world.t = rotate_inverse_inertia(local.t, q);
    if (cb.angular_mode == 1) {
        Q4<F> previousOrientation = integrate_orientation(q, v.ang, bc<F>(dt * -0.5f));
        integrate_angular_conserve_momentum(previousOrientation, local.t, world.t, v.ang);
    } else if (cb.angular_mode == 2) {
        integrate_angular_gyroscopic(q, local.t, v.ang, bc<F>(dt));
    }
    if (conditional) {
        Velocity<F> previousVelocity = v;
        cb.integrate_velocity(v, pos, refs);
        v.lin = sel3<F>(mask, v.lin, previousVelocity.lin);
        v.ang = sel3<F>(mask, v.ang, previousVelocity.ang);
    } else {
        cb.integrate_velocity(v, pos, refs);
    }
}

// ---- solver state ---------------------------------------------------------------------------------------------------
struct Bitset {
    std::vector<uint64_t> w;
    void resize(size_t bits) { w.assign((bits + 63) / 64, 0); }
    bool get(size_t i) const { return (w[i >> 6] >> (i & 63)) & 1; }
    void set(size_t i) { w[i >> 6] |= (uint64_t)1 << (i & 63); }
    bool any() const {
        for (auto x : w) if (x) return true;
        return false;
    }
};

struct TypeBatchFlags {
    Bitset slot[4];
    bool coarse = false;
};

struct Solver {
    oracle_scene* sc;
    Callbacks cb;
    std::vector<std::vector<TypeBatchFlags>> flags;  // [batch][typeBatch], batch 0 unused
    Bitset constrained;                              // merged constrained body set (+ constrained kinematics)
};

enum BundleMode { kNone = 0, kPartial = 1, kAll = 2 };
// TypeProcessor.cs:L1155-1202 BundleShouldIntegrate
static inline BundleMode bundle_should_integrate(const Bitset& f, int bundleIndex, int W, int constraintCount, bool* laneMask) {
    int start = bundleIndex * W;
    int set = 0;
    for (int i = 0; i < W; ++i) {
        int idx = start + i;
        bool b = idx < constraintCount && f.get(idx);
        laneMask[i] = b;
        set += b;
    }
    if (set == W) return kAll;
    if (set > 0) return kPartial;
    return kNone;
}

// Solver_Solve.cs:L1072-1388 PrepareConstraintIntegrationResponsibilities (+ L951-1044)
static void prepare_integration_responsibilities(Solver& s) {
    oracle_scene& sc = *s.sc;
    const int W = sc.bundle_width;
    s.constrained.resize(sc.body_count);
    s.flags.assign(sc.batch_count, {});
    Bitset merged;
    merged.resize(sc.body_count);
    for (int b = 0; b < sc.batch_count; ++b) {
        oracle_batch& batch = sc.batches[b];
        // batchReferencedHandles[b]: dynamic bodies referenced by this batch
        Bitset referenced;
        referenced.resize(sc.body_count);
        for (int t = 0; t < batch.type_batch_count; ++t) {
            oracle_type_batch& tb = batch.type_batches[t];
            int nb = registry<float>().ops[tb.type_id].bodies;
            int bundles = (tb.constraint_count + W - 1) / W;
            for (int k = 0; k < bundles; ++k)
                for (int slot = 0; slot < nb; ++slot)
                    for (int l = 0; l < W; ++l) {
                        int32_t enc = tb.body_references[((size_t)k * nb + slot) * W + l];
                        if ((uint32_t)enc < kDynamicLimit) referenced.set(enc);
                    }
        }
        if (b > 0) {
            // bodiesFirstObservedInBatches[b] = referenced & ~merged
            Bitset first;
            first.resize(sc.body_count);
            for (size_t i = 0; i < first.w.size(); ++i) first.w[i] = referenced.w[i] & ~merged.w[i];
            const bool isFallback = b == sc.fallback_batch_threshold;
            // For the fallback: earliest (typeBatchIndex, indexInTypeBatch) among each body's constraints (L996-1019).
            std::vector<uint64_t> earliest;
            if (isFallback) {
                earliest.assign(sc.body_count, UINT64_MAX);
                for (int t = 0; t < batch.type_batch_count; ++t) {
                    oracle_type_batch& tb = batch.type_batches[t];
                    int nb = registry<float>().ops[tb.type_id].bodies;
                    for (int c = 0; c < tb.constraint_count; ++c)
                        for (int slot = 0; slot < nb; ++slot) {
                            int32_t enc = tb.body_references[((size_t)(c / W) * nb + slot) * W + (c % W)];
                            if (enc == -1) continue;
                            int idx = enc & kBodyReferenceMask;
                            uint64_t cand = ((uint64_t)t << 32) | (uint32_t)c;
                            if (cand < earliest[idx]) earliest[idx] = cand;
                        }
                }
            }
            s.flags[b].resize(batch.type_batch_count);
            for (int t = 0; t < batch.type_batch_count; ++t) {
                oracle_type_batch& tb = batch.type_batches[t];
                int nb = registry<float>().ops[tb.type_id].bodies;
                TypeBatchFlags& tf = s.flags[b][t];
                for (int slot = 0; slot < nb; ++slot) tf.slot[slot].resize(tb.constraint_count);
                for (int c = 0; c < tb.constraint_count; ++c)
                    for (int slot = 0; slot < nb; ++slot) {
                        int32_t enc = tb.body_references[((size_t)(c / W) * nb + slot) * W + (c % W)];
                        if (enc == -1) continue;
                        int idx = enc & kBodyReferenceMask;
                        if (!first.get(idx)) continue;
                        if (isFallback) {
                            uint64_t slotKey = ((uint64_t)t << 32) | (uint32_t)c;
                            if (slotKey == earliest[idx]) tf.slot[slot].set(c);
                        } else {
                            tf.slot[slot].set(c);
                        }
                    }
                tf.coarse = false;
                for (int slot = 0; slot < nb; ++slot) tf.coarse = tf.coarse || tf.slot[slot].any();
            }
        }
        for (size_t i = 0; i < merged.w.size(); ++i) merged.w[i] |= referenced.w[i];
    }
    s.constrained = merged;
    for (int i = 0; i < sc.constrained_kinematic_count; ++i) s.constrained.set(sc.constrained_kinematics[i]);  // L1372-1381
}

// ---- per-bundle stage evaluation -----------------------------------------------------------------------------------
// WarmStart: {One,Two,...}BodyTypeProcessor.WarmStart (TwoBodyTypeProcessor.cs:L168-203) + GatherAndIntegrate (TypeProcessor.cs:L1298-1397)
template <class F>
static void warm_start_bundle(Solver& s, const TypeOps<F>& ops, oracle_type_batch& tb, int bundle, int batchIndex, const TypeBatchFlags* tf, bool allowPose, float dt) {
    oracle_scene& sc = *s.sc;
    const int W = sc.bundle_width;
    constexpr int PW = LaneTraits<F>::Width;
    const int nb = ops.bodies;
    BundleMode mode[4];
    bool laneMask[4][32];
    for (int slot = 0; slot < nb; ++slot) {
        const int32_t* refs = tb.body_references + ((size_t)bundle * nb + slot) * W;
        if (batchIndex == 0) {
            mode[slot] = kAll;  // BatchShouldAlwaysIntegrate: mask = dynamic lanes
            for (int l = 0; l < W; ++l) laneMask[slot][l] = (uint32_t)refs[l] < kDynamicLimit;
        } else if (!tf->coarse) {
            mode[slot] = kNone;  // BatchShouldNeverIntegrate
        } else {
            mode[slot] = bundle_should_integrate(tf->slot[slot], bundle, W, tb.constraint_count, laneMask[slot]);
        }
    }
    for (int chunk = 0; chunk < W / PW; ++chunk) {
        BodyIn<F> body[4];
        Velocity<F> vel[4];
        for (int slot = 0; slot < nb; ++slot) {
            const int32_t* refs = tb.body_references + ((size_t)bundle * nb + slot) * W + chunk * PW;
            if (mode[slot] == kNone) {
                gather_state<F>(sc.bodies, refs, true, body[slot], vel[slot]);
                continue;
            }
            BodyIn<F> g;
            gather_state<F>(sc.bodies, refs, false, g, vel[slot]);
            const bool* m = laneMask[slot] + chunk * PW;
            MaskOf<F> mask = make_mask<F>(m);
            body[slot].pos = g.pos;
            body[slot].q = g.q;
            if (allowPose) {
                integrate_pose_and_velocity<F>(s.cb, g.inertia, dt, mask, body[slot].pos, body[slot].q, vel[slot], body[slot].inertia, refs);
                scatter_pose<F>(sc.bodies, refs, m, body[slot].pos, body[slot].q);
                scatter_world_inertia<F>(sc.bodies, refs, m, body[slot].inertia);
            } else {
                integrate_velocity_only<F>(s.cb, g.inertia, dt, mask, batchIndex != 0, body[slot].pos, body[slot].q, vel[slot], body[slot].inertia, refs);
                scatter_world_inertia<F>(sc.bodies, refs, m, body[slot].inertia);
            }
        }
        Rows<F> p{tb.prestep + (size_t)bundle * ops.prestep_rows * W + chunk * PW, W};
        Rows<F> a{tb.accumulated_impulses + (size_t)bundle * ops.impulse_rows * W + chunk * PW, W};
        ops.warm_start(body, p, a, vel);
        for (int slot = 0; slot < nb; ++slot) {
            const int32_t* refs = tb.body_references + ((size_t)bundle * nb + slot) * W + chunk * PW;
            scatter_velocities<F>(sc.bodies, refs, vel[slot]);
        }
    }
}
// Solve: TwoBodyTypeProcessor.cs:L205-225
template <class F> static void solve_bundle(Solver& s, const TypeOps<F>& ops, oracle_type_batch& tb, int bundle, float dt, float inverseDt) {
    oracle_scene& sc = *s.sc;
    const int W = sc.bundle_width;
    constexpr int PW = LaneTraits<F>::Width;
    const int nb = ops.bodies;
    for (int chunk = 0; chunk < W / PW; ++chunk) {
        BodyIn<F> body[4];
        Velocity<F> vel[4];
        for (int slot = 0; slot < nb; ++slot)
            gather_state<F>(sc.bodies, tb.body_references + ((size_t)bundle * nb + slot) * W + chunk * PW, true, body[slot], vel[slot]);
        Rows<F> p{tb.prestep + (size_t)bundle * ops.prestep_rows * W + chunk * PW, W};
        Rows<F> a{tb.accumulated_impulses + (size_t)bundle * ops.impulse_rows * W + chunk * PW, W};
        ops.solve(body, dt, inverseDt, p, a, vel);
        for (int slot = 0; slot < nb; ++slot)
            scatter_velocities<F>(sc.bodies, tb.body_references + ((size_t)bundle * nb + slot) * W + chunk * PW, vel[slot]);
    }
}
// IncrementallyUpdateForSubstep: TwoBodyTypeProcessor.cs:L228-241
template <class F> static void incremental_bundle(Solver& s, const TypeOps<F>& ops, oracle_type_batch& tb, int bundle, float dt) {
    oracle_scene& sc = *s.sc;
    const int W = sc.bundle_width;
    constexpr int PW = LaneTraits<F>::Width;
    const int nb = ops.bodies;
    for (int chunk = 0; chunk < W / PW; ++chunk) {
        BodyIn<F> body[4];
        Velocity<F> vel[4];
        for (int slot = 0; slot < nb; ++slot)
            gather_state<F>(sc.bodies, tb.body_references + ((size_t)bundle * nb + slot) * W + chunk * PW, true, body[slot], vel[slot]);
        Rows<F> p{tb.prestep + (size_t)bundle * ops.prestep_rows * W + chunk * PW, W};
        ops.incremental(dt, vel, p);
    }
}

// ---- kinematic prepasses: PoseIntegrator.cs:L451-487 (the gathered pose, L480), L493-535 (the integrated pose, L529) ------------------------
static void integrate_kinematic_velocities(Solver& s) {
    oracle_scene& sc = *s.sc;
    for (int i = 0; i < sc.constrained_kinematic_count; ++i) {
        int32_t idx = sc.constrained_kinematics[i];
        BodyIn<float> b;
        Velocity<float> v;
        gather_state<float>(sc.bodies, &idx, false, b, v);
        s.cb.integrate_velocity(v, b.pos, &idx);
        scatter_velocities<float>(sc.bodies, &idx, v);
    }
}
static void integrate_kinematic_poses_and_velocities(Solver& s, float dt) {
    oracle_scene& sc = *s.sc;
    for (int i = 0; i < sc.constrained_kinematic_count; ++i) {
        int32_t idx = sc.constrained_kinematics[i];
        BodyIn<float> b;
        Velocity<float> v;
        gather_state<float>(sc.bodies, &idx, false, b, v);
        b.pos = add(b.pos, scale(v.lin, dt));
        b.q = integrate_orientation<float>(b.q, v.ang, dt * 0.5f);
        bool m = true;
        scatter_pose<float>(sc.bodies, &idx, &m, b.pos, b.q);
        if (s.cb.integrate_kinematic_velocity) {
            s.cb.integrate_velocity(v, b.pos, &idx);
            scatter_velocities<float>(sc.bodies, &idx, v);
        }
    }
}

// ---- final pass: PoseIntegrator.cs:L537-693 IntegrateBundlesAfterSubstepping; the callback sees the position before each step's update ------
static void integrate_after_substepping(Solver& s, float dt, int substepCount) {
    oracle_scene& sc = *s.sc;
    float substepDt = dt / substepCount;
    float velocityIntegrationTimestep = s.cb.allow_substeps_unconstrained ? substepDt : dt;
    s.cb.prepare(velocityIntegrationTimestep);  // L710-712
#pragma omp parallel for schedule(static) num_threads(sc.threads > 0 ? sc.threads : 1)
    for (int i = 0; i < sc.body_count; ++i) {
        int32_t idx = i;
        bool unconstrained = !s.constrained.get(i);
        float effectiveDt = s.cb.allow_substeps_unconstrained ? substepDt : (unconstrained ? dt : substepDt);
        float halfDt = effectiveDt * 0.5f;
        BodyIn<float> b;
        Velocity<float> v;
        gather_state<float>(sc.bodies, &idx, false, b, v);
        bool m = true;
        if (!unconstrained) {
            // Constrained bodies take one pose step of substep length (L684-691 and the masked first step of L632-682).
            Q4<float> q = integrate_orientation<float>(b.q, v.ang, halfDt);
            V3<float> p = add(b.pos, scale(v.lin, effectiveDt));
            scatter_pose<float>(sc.bodies, &idx, &m, p, q);
            continue;
        }
        bool kinematic = b.inertia.inv_mass == 0 && b.inertia.t.xx == 0 && b.inertia.t.yx == 0 && b.inertia.t.yy == 0 && b.inertia.t.zx == 0 && b.inertia.t.zy == 0 &&
                         b.inertia.t.zz == 0;
        bool integrateVelocity = s.cb.integrate_kinematic_velocity || !kinematic;
        int steps = s.cb.allow_substeps_unconstrained ? substepCount : 1;
        for (int step = 0; step < steps; ++step) {
            if (integrateVelocity) s.cb.integrate_velocity(v, b.pos, &idx);
            b.pos = add(b.pos, scale(v.lin, effectiveDt));
            if (s.cb.angular_mode == 1) {
                Q4<float> previousOrientation = b.q;
                b.q = integrate_orientation<float>(b.q, v.ang, halfDt);
                Sym3<float> world = rotate_inverse_inertia(b.inertia.t, b.q);
                V3<float> w = v.ang;
                integrate_angular_conserve_momentum(previousOrientation, b.inertia.t, world, w);
                v.ang = w;
            } else if (s.cb.angular_mode == 2) {
                b.q = integrate_orientation<float>(b.q, v.ang, halfDt);
                V3<float> w = v.ang;
                integrate_angular_gyroscopic(b.q, b.inertia.t, w, effectiveDt);
                v.ang = w;
            } else {
                b.q = integrate_orientation<float>(b.q, v.ang, halfDt);
            }
            scatter_pose<float>(sc.bodies, &idx, &m, b.pos, b.q);
            if (integrateVelocity) scatter_velocities<float>(sc.bodies, &idx, v);
        }
    }
}

// ---- the substep loop: Solver_Solve.cs:L1415-1479 ------------------------------------------------------------------
// Multithreaded shape = the reference's SolveWorker (Solver_Solve.cs:L458-654): every worker walks the same stage list, takes its share of
// the stage's bundles and meets the others at a spinning sync point between stages; the fallback batch runs on worker 0 (L546-583).
struct StageBarrier {
    std::atomic<int> arrived{0};
    std::atomic<int> epoch{0};
    int count = 1;
    void wait() {
        if (count == 1) return;
        const int e = epoch.load(std::memory_order_acquire);
        if (arrived.fetch_add(1, std::memory_order_acq_rel) == count - 1) {
            arrived.store(0, std::memory_order_relaxed);
            epoch.store(e + 1, std::memory_order_release);
            return;
        }
        for (int spins = 0; epoch.load(std::memory_order_acquire) == e; ++spins) {
            if (spins < 4096)
                __builtin_ia32_pause();
            else
                sched_yield();  // oversubscribed host: let the thread we are waiting for run
        }
    }
};

template <class F> static void run_solve(Solver& s, float totalDt) {
    oracle_scene& sc = *s.sc;
    const int W = sc.bundle_width;
    const auto& reg = registry<F>();
    const int substepCount = sc.substep_count;
    float substepDt = totalDt / substepCount;
    s.cb.prepare(substepDt);
    float inverseDt = 1.0f / substepDt;
    // team size the OpenMP runtime really grants (OMP_THREAD_LIMIT, nesting)
    int workers = sc.threads > 0 ? sc.threads : 1;
    if (workers > 1) {
        int granted = 1;
#pragma omp parallel num_threads(workers)
        {
#pragma omp single
            granted = omp_get_num_threads();
        }
        workers = granted;
    }

    // flattened (typeBatch, bundle) work lists per batch
    struct Work { int t, bundle; };
    std::vector<std::vector<Work>> work(sc.batch_count);
    for (int b = 0; b < sc.batch_count; ++b)
        for (int t = 0; t < sc.batches[b].type_batch_count; ++t) {
            int bundles = (sc.batches[b].type_batches[t].constraint_count + W - 1) / W;
            for (int k = 0; k < bundles; ++k) work[b].push_back({t, k});
        }

    StageBarrier barrier;
    barrier.count = workers;
    auto worker = [&](const int worker_index) {
        // this worker's share of batch b: a contiguous block of bundles; the sequential fallback batch belongs to worker 0
        auto share = [&](int b, int& begin, int& end) {
            const int n = (int)work[b].size();
            if (b >= sc.fallback_batch_threshold) {
                begin = 0;
                end = worker_index == 0 ? n : 0;
            } else {
                begin = (int)((int64_t)n * worker_index / workers);
                end = (int)((int64_t)n * (worker_index + 1) / workers);
            }
        };
        int begin, end;
        for (int substep = 0; substep < substepCount; ++substep) {
            if (substep > 0) {
                for (int b = 0; b < sc.batch_count; ++b) {  // contact depths only read velocities: no sync between batches
                    const int n = (int)work[b].size();
                    begin = (int)((int64_t)n * worker_index / workers);
                    end = (int)((int64_t)n * (worker_index + 1) / workers);
                    for (int i = begin; i < end; ++i) {
                        oracle_type_batch& tb = sc.batches[b].type_batches[work[b][i].t];
                        const TypeOps<F>& ops = reg.ops[tb.type_id];
                        if (ops.incremental) incremental_bundle<F>(s, ops, tb, work[b][i].bundle, substepDt);
                    }
                }
                barrier.wait();
                if (worker_index == 0) integrate_kinematic_poses_and_velocities(s, substepDt);
                barrier.wait();
            } else if (s.cb.integrate_kinematic_velocity) {
                if (worker_index == 0) integrate_kinematic_velocities(s);
                barrier.wait();
            }
            for (int b = 0; b < sc.batch_count; ++b) {
                share(b, begin, end);
                for (int i = begin; i < end; ++i) {
                    oracle_type_batch& tb = sc.batches[b].type_batches[work[b][i].t];
                    warm_start_bundle<F>(s, reg.ops[tb.type_id], tb, work[b][i].bundle, b, b > 0 ? &s.flags[b][work[b][i].t] : nullptr, substep > 0, substepDt);
                }
                barrier.wait();
            }
            const int iterations = sc.velocity_iterations[substep];
            for (int it = 0; it < iterations; ++it)
                for (int b = 0; b < sc.batch_count; ++b) {
                    share(b, begin, end);
                    for (int i = begin; i < end; ++i) {
                        oracle_type_batch& tb = sc.batches[b].type_batches[work[b][i].t];
                        solve_bundle<F>(s, reg.ops[tb.type_id], tb, work[b][i].bundle, substepDt, inverseDt);
                    }
                    barrier.wait();
                }
        }
    };
    if (workers == 1) {
        worker(0);
        return;
    }
    bool ran = false;
#pragma omp parallel num_threads(workers)
    {
        // every member sees the same team size: either all of them walk the stage list or none does (a short team would hang the sync points)
        if (omp_get_num_threads() == workers) {
            worker(omp_get_thread_num());
#pragma omp master
            ran = true;
        }
    }
    if (!ran) {
        workers = 1;
        barrier.count = 1;
        worker(0);
    }
}

}  // namespace bepu_oracle

using namespace bepu_oracle;

extern "C" int32_t oracle_type_info(int32_t type_id, int32_t* bodies, int32_t* prestep_floats, int32_t* impulse_floats) {
    if (type_id < 0 || type_id >= 64) return -1;
    const TypeOps<float>& o = registry<float>().ops[type_id];
    if (!o.solve) return -1;
    if (bodies) *bodies = o.bodies;
    if (prestep_floats) *prestep_floats = o.prestep_rows;
    if (impulse_floats) *impulse_floats = o.impulse_rows;
    return 0;
}

// One constraint lane of one stage through the typed functions (stage 0 WarmStart, 1 Solve, 2 IncrementallyUpdateForSubstep): the hook that lets
// the CPU suite compare a host compilation of the CUDA constraint SOURCE against this restatement (tests/test_device_source_on_host.py).
// body_states: per body 14 floats (position 3, orientation xyzw, world inverse inertia XX YX YY ZX ZY ZZ, inverse mass); velocities: per body 6;
// row r of the lane is prestep[r * row_stride] / impulses[r * row_stride].
extern "C" int32_t oracle_eval_lane(int32_t type_id, int32_t stage, const float* body_states, float dt, float* prestep, float* impulses, float* velocities, int32_t row_stride) {
    if (type_id < 0 || type_id >= 64) return -1;
    const TypeOps<float>& o = registry<float>().ops[type_id];
    if (!o.solve) return -1;
    BodyIn<float> b[4];
    Velocity<float> v[4];
    for (int s = 0; s < o.bodies; ++s) {
        const float* f = body_states + 14 * s;
        b[s].pos = {f[0], f[1], f[2]};
        b[s].q = {f[3], f[4], f[5], f[6]};
        b[s].inertia.t = {f[7], f[8], f[9], f[10], f[11], f[12]};
        b[s].inertia.inv_mass = f[13];
        const float* w = velocities + 6 * s;
        v[s].lin = {w[0], w[1], w[2]};
        v[s].ang = {w[3], w[4], w[5]};
    }
    Rows<float> p{prestep, row_stride}, a{impulses, row_stride};
    if (stage == 0) o.warm_start(b, p, a, v);
    else if (stage == 1) o.solve(b, dt, 1.0f / dt, p, a, v);
    else if (o.incremental) o.incremental(dt, v, p);
    for (int s = 0; s < o.bodies; ++s) {
        float* w = velocities + 6 * s;
        w[0] = v[s].lin.x; w[1] = v[s].lin.y; w[2] = v[s].lin.z;
        w[3] = v[s].ang.x; w[4] = v[s].ang.y; w[5] = v[s].ang.z;
    }
    return 0;
}

// The integration arithmetic, one call per function (same ops and operand layout as device_on_host_eval_integration in tests/device_on_host).
extern "C" int32_t oracle_eval_integration(int32_t op, const float* in, float* out) {
    auto sym = [&](int i) { return Sym3<float>{in[i], in[i + 1], in[i + 2], in[i + 3], in[i + 4], in[i + 5]}; };
    if (op == 0) {
        Q4<float> q = integrate_orientation<float>(Q4<float>{in[0], in[1], in[2], in[3]}, V3<float>{in[4], in[5], in[6]}, in[7]);
        out[0] = q.x; out[1] = q.y; out[2] = q.z; out[3] = q.w;
    } else if (op == 1) {
        Sym3<float> r = rotate_inverse_inertia<float>(sym(0), Q4<float>{in[6], in[7], in[8], in[9]});
        out[0] = r.xx; out[1] = r.yx; out[2] = r.yy; out[3] = r.zx; out[4] = r.zy; out[5] = r.zz;
    } else if (op == 2) {
        V3<float> w{in[16], in[17], in[18]};
        integrate_angular_conserve_momentum<float>(Q4<float>{in[0], in[1], in[2], in[3]}, sym(4), sym(10), w);
        out[0] = w.x; out[1] = w.y; out[2] = w.z;
    } else if (op == 3) {
        V3<float> w{in[10], in[11], in[12]};
        integrate_angular_gyroscopic<float>(Q4<float>{in[0], in[1], in[2], in[3]}, sym(4), w, in[13]);
        out[0] = w.x; out[1] = w.y; out[2] = w.z;
    } else if (op == 4) {
        Callbacks cb{};
        cb.gravity_dt[0] = in[6]; cb.gravity_dt[1] = in[7]; cb.gravity_dt[2] = in[8];
        cb.linear_damping_dt = in[9]; cb.angular_damping_dt = in[10];
        Velocity<float> v{{in[0], in[1], in[2]}, {in[3], in[4], in[5]}};
        cb.integrate_velocity(v);
        out[0] = v.lin.x; out[1] = v.lin.y; out[2] = v.lin.z; out[3] = v.ang.x; out[4] = v.ang.y; out[5] = v.ang.z;
    } else if (op == 5) {
        Velocity<float> v{{in[0], in[1], in[2]}, {in[3], in[4], in[5]}};
        apply_velocity_terms<float>(v, in[20] != 0.0f, V3<float>{in[6], in[7], in[8]}, V3<float>{in[9], in[10], in[11]}, in[12], in[21] != 0.0f,
                                    V3<float>{in[13], in[14], in[15]}, V3<float>{in[16], in[17], in[18]}, in[19]);
        out[0] = v.lin.x; out[1] = v.lin.y; out[2] = v.lin.z; out[3] = v.ang.x; out[4] = v.ang.y; out[5] = v.ang.z;
    } else {
        return -1;
    }
    return 0;
}

// ---- narrow-phase impulse carry-over for a contact constraint whose type did not change ---------------------------------------------------------
// NarrowPhase.RedistributeImpulses, CollisionDetection/NarrowPhaseConstraintUpdate.cs:L81-135.
extern "C" void oracle_redistribute_impulses(int32_t oldContactCount, const int32_t* oldFeatureIds, float* oldImpulses, int32_t newContactCount, const int32_t* newFeatureIds,
                                             float* newImpulses) {
    int unmatchedCount = 0;
    for (int i = 0; i < newContactCount; ++i) {
        newImpulses[i] = -1;  // accumulated impulses cannot be negative: a negative value flags 'unmatched' (L92-93)
        for (int j = 0; j < oldContactCount; ++j) {
            if (oldFeatureIds[j] == newFeatureIds[i]) {
                newImpulses[i] = oldImpulses[j];
                oldImpulses[j] = 0;  // will not be distributed to the unmatched contacts (L98-100)
                break;
            }
        }
        if (newImpulses[i] < 0) ++unmatchedCount;
    }
    if (unmatchedCount > 0) {  // L110-131: the remaining impulse is shared evenly by the unmatched contacts
        float unmatchedImpulse = 0;
        for (int i = 0; i < oldContactCount; ++i) unmatchedImpulse += oldImpulses[i];
        float impulsePerUnmatched = unmatchedImpulse / unmatchedCount;
        for (int i = 0; i < newContactCount; ++i)
            if (newImpulses[i] < 0) newImpulses[i] = impulsePerUnmatched;
    }
}
// UpdateConstraint, same-type branch (L147-183), for a whole type batch in the reference AOSOA-W layout: GatherOldImpulses / ScatterNewImpulses
// address the penetration rows of the accumulated impulses (ContactConstraintAccessor.cs:L36-78: after the Vector2Wide tangent for convex types,
// NonconvexAccumulatedImpulses.Penetration of contact i otherwise).
extern "C" int32_t oracle_update_contact_impulses(int32_t type_id, int32_t constraint_count, int32_t W, float* accumulated_impulses, const int32_t* old_feature_ids,
                                                  const int32_t* new_feature_ids) {
    const bool convex = type_id >= 0 && type_id <= 7;
    int n;
    if (convex) n = (type_id & 3) + 1;
    else if (type_id >= 8 && type_id <= 10) n = type_id - 6;
    else if (type_id >= 15 && type_id <= 17) n = type_id - 13;
    else return -1;
    const int rows = convex ? n + 3 : 3 * n;
    for (int c = 0; c < constraint_count; ++c) {
        float* bundle = accumulated_impulses + (size_t)(c / W) * rows * W + (c % W);
        float oldImpulses[8], newImpulses[8];
        for (int i = 0; i < n; ++i) oldImpulses[i] = bundle[(convex ? 2 + i : 3 * i + 2) * W];
        oracle_redistribute_impulses(n, old_feature_ids + (size_t)c * n, oldImpulses, n, new_feature_ids + (size_t)c * n, newImpulses);
        for (int i = 0; i < n; ++i) bundle[(convex ? 2 + i : 3 * i + 2) * W] = newImpulses[i];
    }
    return 0;
}

// Batch assignment of Solver.Add (Solver.cs:L1182-1199) for a whole constraint list: every constraint, in ascending key order, goes to the first
// batch whose referenced-handle set holds none of its dynamic bodies (GetBlockingBodyHandles L1058-1078: kinematic references never block); batch
// index == fallback_threshold is the fallback batch and takes whatever no synchronized batch could (TryAllocateInBatch L1093-1140). The key is the
// one include/bepucuda.h documents for bepucuda_color_constraints: order 0 = index (the reference's own add sequence), 1 = hashed, 2 = priorities.
static uint32_t oracle_color_hash(uint32_t c) {
    uint32_t h = c * 0x9E3779B1u;
    h ^= h >> 15;
    h *= 0x85EBCA77u;
    h ^= h >> 13;
    h *= 0xC2B2AE3Du;
    h ^= h >> 16;
    return h;
}
extern "C" int32_t oracle_first_fit_batches(int32_t constraint_count, int32_t bodies_per_constraint, const int32_t* encoded_body_references, int32_t body_count,
                                            int32_t fallback_threshold, int32_t order, const uint32_t* priorities, int32_t* batch_indices_out) {
    if (constraint_count < 0 || bodies_per_constraint < 1 || bodies_per_constraint > 4 || order < 0 || order > 2 || (order == 2 && !priorities)) return -1;
    std::vector<uint64_t> keys((size_t)constraint_count);
    for (int c = 0; c < constraint_count; ++c) keys[c] = ((uint64_t)(order == 0 ? 0u : (order == 1 ? oracle_color_hash((uint32_t)c) : priorities[c])) << 32) | (uint32_t)c;
    std::sort(keys.begin(), keys.end());
    const size_t words = ((size_t)body_count + 63) / 64;
    std::vector<std::vector<uint64_t>> batchReferencedHandles;  // Solver.cs:L33, one IndexSet per batch
    for (uint64_t key : keys) {
        const int c = (int)(uint32_t)key;
        int blocking[4], blockingCount = 0;
        for (int s = 0; s < bodies_per_constraint; ++s) {
            const int32_t enc = encoded_body_references[(size_t)c * bodies_per_constraint + s];
            if (enc < 0 || ((uint32_t)enc & 0x40000000u)) continue;
            if (enc >= body_count) return -2;
            blocking[blockingCount++] = enc;
        }
        for (int target = 0;; ++target) {
            if (target == (int)batchReferencedHandles.size()) batchReferencedHandles.emplace_back(words, 0ull);
            else if (target < fallback_threshold) {
                bool fits = true;
                for (int i = 0; i < blockingCount; ++i) fits = fits && !((batchReferencedHandles[target][blocking[i] >> 6] >> (blocking[i] & 63)) & 1);
                if (!fits) continue;
            }
            if (target < fallback_threshold)
                for (int i = 0; i < blockingCount; ++i) batchReferencedHandles[target][blocking[i] >> 6] |= 1ull << (blocking[i] & 63);
            batch_indices_out[c] = target;
            break;
        }
    }
    return (int32_t)batchReferencedHandles.size();
}

// ---- PredictBoundingBoxes (SURVEY.md §8 f4), one body at a time in scalar fp32 (this file is compiled -ffp-contract=off) --------------------------------
// PoseIntegrator.PredictBoundingBoxes (PoseIntegrator.cs:L307-370), UpdateSleepCandidacy (L286-304), BoundingBoxBatcher.ExecuteConvexBatch
// (Collidables/BoundingBoxBatcher.cs:L176-197), IConvexShape.GetBounds of Sphere.cs:L149-160, Capsule.cs:L226-239, Box.cs:L211-222,
// Cylinder.cs:L222-235, BoundingBoxHelpers.GetAngularBoundsExpansion / GetBoundsExpansion (BoundingBoxHelpers.cs:L12-58).
struct oracle_body_shape { int32_t type; float a, b, c, minimum_speculative_margin, maximum_speculative_margin; int32_t allow_expansion_beyond_speculative_margin, reserved; };
struct oracle_body_activity { float sleep_threshold; uint8_t minimum_timesteps_under_threshold, timesteps_under_threshold_count, sleep_candidate, reserved; };
// terms: the optional velocity terms, or NULL (the default) for none.
extern "C" int32_t oracle_predict_bounding_boxes(int32_t body_count, const float* bodies, const oracle_body_shape* shapes, oracle_body_activity* activities, float dt,
                                                 const float* gravity, float linear_damping, float angular_damping, int32_t integrate_velocity_for_kinematics,
                                                 float* bounds_out, const oracle_integrator_terms* terms = nullptr) {
    Callbacks cb{};
    std::copy(gravity, gravity + 3, cb.gravity);
    cb.linear_damping = linear_damping;
    cb.angular_damping = angular_damping;
    if (terms) cb.terms = *terms;
    cb.prepare(dt);  // PoseIntegrator.cs:L428: PrepareForIntegration with the frame dt
    for (int32_t i = 0; i < body_count; ++i) {
        const float* b = bodies + (size_t)i * 32;
        const Q4<float> orientation = {b[0], b[1], b[2], b[3]};
        const V3<float> position = {b[4], b[5], b[6]};
        V3<float> linear = {b[8], b[9], b[10]}, angular = {b[12], b[13], b[14]};
        // Bodies.IsKinematic (Bodies.cs:L326-331) compares the OR of the seven floats' bits with 0.0f as a FLOAT: any mix of +0 and -0 is kinematic
        bool kinematic = true;
        for (int k = 16; k < 23; ++k) kinematic = kinematic && b[k] == 0.0f;
        const bool integrate = integrate_velocity_for_kinematics != 0 || !kinematic;
        const float sleepEnergy = length_squared(linear) + length_squared(angular);
        if (integrate) {  // IntegrateVelocity at the current pose (PoseIntegrator.cs:L339-341); the result is not stored
            Velocity<float> v{linear, angular};
            cb.integrate_velocity(v, position, &i);
            linear = v.lin;
            angular = v.ang;
        }
        oracle_body_activity& activity = activities[i];
        if (sleepEnergy > activity.sleep_threshold) {
            activity.timesteps_under_threshold_count = 0;
            activity.sleep_candidate = 0;
        } else if (activity.timesteps_under_threshold_count < 255) {
            ++activity.timesteps_under_threshold_count;
            if (activity.timesteps_under_threshold_count >= activity.minimum_timesteps_under_threshold) activity.sleep_candidate = 1;
        }
        float* out = bounds_out + (size_t)i * 8;
        const oracle_body_shape& s = shapes[i];
        V3<float> max;
        float maximumRadius, maximumAngularExpansion;
        if (s.type == 0) {
            max = {s.a, s.a, s.a};
            maximumRadius = 0.0f;
            maximumAngularExpansion = 0.0f;
        } else if (s.type == 1) {
            const float radius = s.a, halfLength = s.b;
            V3<float> segmentOffset = scale(transform_unit_y(orientation), halfLength);
            segmentOffset = {vabs(segmentOffset.x), vabs(segmentOffset.y), vabs(segmentOffset.z)};
            max = {segmentOffset.x + radius, segmentOffset.y + radius, segmentOffset.z + radius};
            maximumRadius = halfLength + radius;
            maximumAngularExpansion = halfLength;
        } else if (s.type == 2) {
            const float HalfWidth = s.a, HalfHeight = s.b, HalfLength = s.c;
            const M33<float> basis = matrix_from_quaternion(orientation);
            max.x = vabs(HalfWidth * basis.x.x) + vabs(HalfHeight * basis.y.x) + vabs(HalfLength * basis.z.x);
            max.y = vabs(HalfWidth * basis.x.y) + vabs(HalfHeight * basis.y.y) + vabs(HalfLength * basis.z.y);
            max.z = vabs(HalfWidth * basis.x.z) + vabs(HalfHeight * basis.y.z) + vabs(HalfLength * basis.z.z);
            maximumRadius = vsqrt(HalfWidth * HalfWidth + HalfHeight * HalfHeight + HalfLength * HalfLength);
            maximumAngularExpansion = maximumRadius - vmin(HalfLength, vmin(HalfHeight, HalfLength));  // Box.cs:L221 as written
        } else if (s.type == 4) {
            const float Radius = s.a, HalfLength = s.b;
            const V3<float> y = transform_unit_y(orientation);
            const V3<float> squared = {1.0f - y.x * y.x, 1.0f - y.y * y.y, 1.0f - y.z * y.z};
            max.x = vabs(HalfLength * y.x) + vsqrt(vmax(0.0f, squared.x)) * Radius;
            max.y = vabs(HalfLength * y.y) + vsqrt(vmax(0.0f, squared.y)) * Radius;
            max.z = vabs(HalfLength * y.z) + vsqrt(vmax(0.0f, squared.z)) * Radius;
            maximumRadius = vsqrt(HalfLength * HalfLength + Radius * Radius);
            maximumAngularExpansion = maximumRadius - vmin(HalfLength, Radius);
        } else {
            for (int k = 0; k < 8; ++k) out[k] = 0.0f;
            continue;
        }
        // GetAngularBoundsExpansion
        const float a = vmin(length(angular) * dt, 3.14159274f / 3.0f);
        const float a2 = a * a, a4 = a2 * a2, a6 = a4 * a2;
        const float cosAngleMinusOne = a2 * (-1.0f / 2.0f) + a4 * (1.0f / 24.0f) - a6 * (1.0f / 720.0f);
        const float angularBoundsExpansion = vmin(maximumAngularExpansion, vsqrt(-2.0f * maximumRadius * maximumRadius * cosAngleMinusOne));
        float speculativeMargin = length(linear) * dt + angularBoundsExpansion;
        speculativeMargin = vmax(s.minimum_speculative_margin, vmin(s.maximum_speculative_margin, speculativeMargin));
        const float maximumBoundsExpansion = s.allow_expansion_beyond_speculative_margin ? 3.40282347e+38f : speculativeMargin;
        // GetBoundsExpansion
        const V3<float> linearDisplacement = scale(linear, dt);
        V3<float> minExpansion = {vmin(0.0f, linearDisplacement.x) - angularBoundsExpansion, vmin(0.0f, linearDisplacement.y) - angularBoundsExpansion, vmin(0.0f, linearDisplacement.z) - angularBoundsExpansion};
        V3<float> maxExpansion = {vmax(0.0f, linearDisplacement.x) + angularBoundsExpansion, vmax(0.0f, linearDisplacement.y) + angularBoundsExpansion, vmax(0.0f, linearDisplacement.z) + angularBoundsExpansion};
        minExpansion = {vmax(-maximumBoundsExpansion, minExpansion.x), vmax(-maximumBoundsExpansion, minExpansion.y), vmax(-maximumBoundsExpansion, minExpansion.z)};
        maxExpansion = {vmin(maximumBoundsExpansion, maxExpansion.x), vmin(maximumBoundsExpansion, maxExpansion.y), vmin(maximumBoundsExpansion, maxExpansion.z)};
        const V3<float> bundleMin = add(position, add(neg(max), minExpansion));
        const V3<float> bundleMax = add(position, add(max, maxExpansion));
        out[0] = bundleMin.x; out[1] = bundleMin.y; out[2] = bundleMin.z; out[3] = speculativeMargin;
        out[4] = bundleMax.x; out[5] = bundleMax.y; out[6] = bundleMax.z; out[7] = 1.0f;
    }
    return 0;
}

extern "C" int32_t oracle_max_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}

extern "C" int32_t oracle_solve(oracle_scene* sc, float dt) {
    if (!sc || sc->substep_count < 1 || sc->bundle_width < 1 || sc->bundle_width > 32) return -1;
    if (sc->simd && sc->bundle_width != 8) return -2;
    for (int b = 0; b < sc->batch_count; ++b)
        for (int t = 0; t < sc->batches[b].type_batch_count; ++t) {
            int id = sc->batches[b].type_batches[t].type_id;
            if (id < 0 || id >= 64 || !registry<float>().ops[id].solve) return -3;
        }
    Solver s;
    s.sc = sc;
    std::copy(sc->gravity, sc->gravity + 3, s.cb.gravity);
    s.cb.linear_damping = sc->linear_damping;
    s.cb.angular_damping = sc->angular_damping;
    s.cb.angular_mode = sc->angular_integration_mode;
    s.cb.allow_substeps_unconstrained = sc->allow_substeps_for_unconstrained != 0;
    s.cb.integrate_kinematic_velocity = sc->integrate_velocity_for_kinematics != 0;
    s.cb.terms = sc->terms;
    // Simulation.Solve: Simulation.cs:L278-290
    prepare_integration_responsibilities(s);
    if (sc->simd)
        run_solve<f8>(s, dt);
    else
        run_solve<float>(s, dt);
    integrate_after_substepping(s, dt, sc->substep_count);
    return 0;
}
