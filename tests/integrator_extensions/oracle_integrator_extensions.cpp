// TEST INFRASTRUCTURE. The CPU oracle of the optional velocity terms of bepucuda_set_body_accelerations / bepucuda_set_point_gravity
// (include/bepucuda.h): the oracle's own translation unit (oracle/bepu_oracle.cpp, unchanged) is compiled in, and the driver functions that call
// IntegrateVelocity are restated here with the terms applied after the declarative callback. Everything else -- the constraint registry,
// gather/scatter, the pose integration arithmetic, the integration responsibilities, the Solve and IncrementallyUpdateForSubstep bundles -- is the
// oracle's, unchanged. Single-threaded (the batch order of the oracle's one-worker path); scalar and 8-wide like the oracle.
// Build: g++ -O2 -std=c++17 -fPIC -fopenmp -ffp-contract=off -fno-fast-math -march=x86-64-v3 -I oracle -shared (tests/test_integrator_extensions.py)
#include "bepu_oracle.cpp"

namespace bepu_oracle {
namespace ext {

struct Terms {
    const float* accelerations;  // body_count x 8 {a.xyz 0 | alpha.xyz 0}, or nullptr
    int32_t point_gravity;
    float center[3];
    float strength;
};

// The two terms (PerBodyGravityDemo.cs:L57-88: v += a * dt; PlanetDemo.cs:L44-46 in its operation order, with Vector3Wide.Length and
// Vector3Wide / Vector<float> = multiply by the reciprocal, Vector3Wide.cs:L357-363, L573-576).
template <class F>
static inline void integrate_velocity_extensions(Velocity<F>& v, bool accelerations, const V3<F>& linearAcceleration, const V3<F>& angularAcceleration, float dt, bool pointGravity,
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

// The declarative callback (Callbacks::integrate_velocity) followed by the terms of the lanes' bodies at the position the reference hands the
// callback. refs: the PW encoded body references of the lanes (-1 = empty lane); dt: the dt of the last PrepareForIntegration.
struct ExtSolver {
    Solver s;
    Terms terms;
    float prepared_dt = 0.0f;
    void prepare(float dt) {
        s.cb.prepare(dt);
        prepared_dt = dt;
    }
    template <class F> void integrate_velocity(Velocity<F>& v, const V3<F>& position, const int32_t* refs) const {
        s.cb.integrate_velocity(v);
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
        integrate_velocity_extensions<F>(v, terms.accelerations != nullptr, al, aa, prepared_dt, terms.point_gravity != 0, position, V3<F>{bc<F>(c[0]), bc<F>(c[1]), bc<F>(c[2])},
                                         prepared_dt * terms.strength);  // gravityDt = dt * Gravity (PlanetDemo.cs:L36-40)
    }
};

// integrate_pose_and_velocity of the oracle (TypeProcessor.cs:L1204-1248); the callback sees the integrated pose (L1244).
template <class F>
static void integrate_pose_and_velocity(const ExtSolver& e, const Inertia<F>& local, float dt, const MaskOf<F>& mask, V3<F>& pos, Q4<F>& q, Velocity<F>& v, Inertia<F>& world,
                                        const int32_t* refs) {
    const Callbacks& cb = e.s.cb;
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
    e.integrate_velocity(v, pos, refs);
    v.lin = sel3<F>(mask, v.lin, previousVelocity.lin);
    v.ang = sel3<F>(mask, v.ang, previousVelocity.ang);
}
// integrate_velocity_only of the oracle (TypeProcessor.cs:L1251-1283); the callback sees the current pose.
template <class F>
static void integrate_velocity_only(const ExtSolver& e, const Inertia<F>& local, float dt, const MaskOf<F>& mask, bool conditional, const V3<F>& pos, const Q4<F>& q, Velocity<F>& v,
                                    Inertia<F>& world, const int32_t* refs) {
    const Callbacks& cb = e.s.cb;
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
        e.integrate_velocity(v, pos, refs);
        v.lin = sel3<F>(mask, v.lin, previousVelocity.lin);
        v.ang = sel3<F>(mask, v.ang, previousVelocity.ang);
    } else {
        e.integrate_velocity(v, pos, refs);
    }
}

// warm_start_bundle of the oracle with the two integration calls above.
template <class F>
static void warm_start_bundle(ExtSolver& e, const TypeOps<F>& ops, oracle_type_batch& tb, int bundle, int batchIndex, const TypeBatchFlags* tf, bool allowPose, float dt) {
    oracle_scene& sc = *e.s.sc;
    const int W = sc.bundle_width;
    constexpr int PW = LaneTraits<F>::Width;
    const int nb = ops.bodies;
    BundleMode mode[4];
    bool laneMask[4][32];
    for (int slot = 0; slot < nb; ++slot) {
        const int32_t* refs = tb.body_references + ((size_t)bundle * nb + slot) * W;
        if (batchIndex == 0) {
            mode[slot] = kAll;
            for (int l = 0; l < W; ++l) laneMask[slot][l] = (uint32_t)refs[l] < kDynamicLimit;
        } else if (!tf->coarse) {
            mode[slot] = kNone;
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
                integrate_pose_and_velocity<F>(e, g.inertia, dt, mask, body[slot].pos, body[slot].q, vel[slot], body[slot].inertia, refs);
                scatter_pose<F>(sc.bodies, refs, m, body[slot].pos, body[slot].q);
                scatter_world_inertia<F>(sc.bodies, refs, m, body[slot].inertia);
            } else {
                integrate_velocity_only<F>(e, g.inertia, dt, mask, batchIndex != 0, body[slot].pos, body[slot].q, vel[slot], body[slot].inertia, refs);
                scatter_world_inertia<F>(sc.bodies, refs, m, body[slot].inertia);
            }
        }
        Rows<F> p{tb.prestep + (size_t)bundle * ops.prestep_rows * W + chunk * PW, W};
        Rows<F> a{tb.accumulated_impulses + (size_t)bundle * ops.impulse_rows * W + chunk * PW, W};
        ops.warm_start(body, p, a, vel);
        for (int slot = 0; slot < nb; ++slot) scatter_velocities<F>(sc.bodies, tb.body_references + ((size_t)bundle * nb + slot) * W + chunk * PW, vel[slot]);
    }
}

// Kinematic prepasses (PoseIntegrator.cs:L451-487: the gathered pose, L480; L493-535: the integrated pose, L529).
static void integrate_kinematic_velocities(ExtSolver& e) {
    oracle_scene& sc = *e.s.sc;
    for (int i = 0; i < sc.constrained_kinematic_count; ++i) {
        int32_t idx = sc.constrained_kinematics[i];
        BodyIn<float> b;
        Velocity<float> v;
        gather_state<float>(sc.bodies, &idx, false, b, v);
        e.integrate_velocity(v, b.pos, &idx);
        scatter_velocities<float>(sc.bodies, &idx, v);
    }
}
static void integrate_kinematic_poses_and_velocities(ExtSolver& e, float dt) {
    oracle_scene& sc = *e.s.sc;
    for (int i = 0; i < sc.constrained_kinematic_count; ++i) {
        int32_t idx = sc.constrained_kinematics[i];
        BodyIn<float> b;
        Velocity<float> v;
        gather_state<float>(sc.bodies, &idx, false, b, v);
        b.pos = add(b.pos, scale(v.lin, dt));
        b.q = integrate_orientation<float>(b.q, v.ang, dt * 0.5f);
        bool m = true;
        scatter_pose<float>(sc.bodies, &idx, &m, b.pos, b.q);
        if (e.s.cb.integrate_kinematic_velocity) {
            e.integrate_velocity(v, b.pos, &idx);
            scatter_velocities<float>(sc.bodies, &idx, v);
        }
    }
}

// Final pass (PoseIntegrator.cs:L537-693, L707-712); the callback sees the position before each step's pose update.
static void integrate_after_substepping(ExtSolver& e, float dt, int substepCount) {
    oracle_scene& sc = *e.s.sc;
    const Callbacks& cb = e.s.cb;
    float substepDt = dt / substepCount;
    float velocityIntegrationTimestep = cb.allow_substeps_unconstrained ? substepDt : dt;
    e.prepare(velocityIntegrationTimestep);
    for (int i = 0; i < sc.body_count; ++i) {
        int32_t idx = i;
        bool unconstrained = !e.s.constrained.get(i);
        float effectiveDt = cb.allow_substeps_unconstrained ? substepDt : (unconstrained ? dt : substepDt);
        float halfDt = effectiveDt * 0.5f;
        BodyIn<float> b;
        Velocity<float> v;
        gather_state<float>(sc.bodies, &idx, false, b, v);
        bool m = true;
        if (!unconstrained) {
            Q4<float> q = integrate_orientation<float>(b.q, v.ang, halfDt);
            V3<float> p = add(b.pos, scale(v.lin, effectiveDt));
            scatter_pose<float>(sc.bodies, &idx, &m, p, q);
            continue;
        }
        bool kinematic = b.inertia.inv_mass == 0 && b.inertia.t.xx == 0 && b.inertia.t.yx == 0 && b.inertia.t.yy == 0 && b.inertia.t.zx == 0 && b.inertia.t.zy == 0 &&
                         b.inertia.t.zz == 0;
        bool integrateVelocity = cb.integrate_kinematic_velocity || !kinematic;
        int steps = cb.allow_substeps_unconstrained ? substepCount : 1;
        for (int step = 0; step < steps; ++step) {
            if (integrateVelocity) e.integrate_velocity(v, b.pos, &idx);
            b.pos = add(b.pos, scale(v.lin, effectiveDt));
            if (cb.angular_mode == 1) {
                Q4<float> previousOrientation = b.q;
                b.q = integrate_orientation<float>(b.q, v.ang, halfDt);
                Sym3<float> world = rotate_inverse_inertia(b.inertia.t, b.q);
                V3<float> w = v.ang;
                integrate_angular_conserve_momentum(previousOrientation, b.inertia.t, world, w);
                v.ang = w;
            } else if (cb.angular_mode == 2) {
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

// The substep loop of the oracle (Solver_Solve.cs:L1415-1479) on one worker.
template <class F> static void run_solve(ExtSolver& e, float totalDt) {
    oracle_scene& sc = *e.s.sc;
    const int W = sc.bundle_width;
    const auto& reg = registry<F>();
    const int substepCount = sc.substep_count;
    const float substepDt = totalDt / substepCount;
    e.prepare(substepDt);
    const float inverseDt = 1.0f / substepDt;
    auto bundles = [&](int b, int t) { return (sc.batches[b].type_batches[t].constraint_count + W - 1) / W; };
    for (int substep = 0; substep < substepCount; ++substep) {
        if (substep > 0) {
            for (int b = 0; b < sc.batch_count; ++b)
                for (int t = 0; t < sc.batches[b].type_batch_count; ++t) {
                    oracle_type_batch& tb = sc.batches[b].type_batches[t];
                    const TypeOps<F>& ops = reg.ops[tb.type_id];
                    if (ops.incremental)
                        for (int k = 0; k < bundles(b, t); ++k) incremental_bundle<F>(e.s, ops, tb, k, substepDt);
                }
            integrate_kinematic_poses_and_velocities(e, substepDt);
        } else if (e.s.cb.integrate_kinematic_velocity) {
            integrate_kinematic_velocities(e);
        }
        for (int b = 0; b < sc.batch_count; ++b)
            for (int t = 0; t < sc.batches[b].type_batch_count; ++t) {
                oracle_type_batch& tb = sc.batches[b].type_batches[t];
                for (int k = 0; k < bundles(b, t); ++k) warm_start_bundle<F>(e, reg.ops[tb.type_id], tb, k, b, b > 0 ? &e.s.flags[b][t] : nullptr, substep > 0, substepDt);
            }
        for (int it = 0; it < sc.velocity_iterations[substep]; ++it)
            for (int b = 0; b < sc.batch_count; ++b)
                for (int t = 0; t < sc.batches[b].type_batch_count; ++t) {
                    oracle_type_batch& tb = sc.batches[b].type_batches[t];
                    for (int k = 0; k < bundles(b, t); ++k) solve_bundle<F>(e.s, reg.ops[tb.type_id], tb, k, substepDt, inverseDt);
                }
    }
}

}  // namespace ext
}  // namespace bepu_oracle

// oracle_solve with the terms (scene->threads is ignored: one worker). 0 on success.
extern "C" int32_t oracle_ext_solve(oracle_scene* sc, const bepu_oracle::ext::Terms* terms, float dt) {
    using namespace bepu_oracle;
    if (!sc || !terms || sc->substep_count < 1 || sc->bundle_width < 1 || sc->bundle_width > 32) return -1;
    if (sc->simd && sc->bundle_width != 8) return -2;
    for (int b = 0; b < sc->batch_count; ++b)
        for (int t = 0; t < sc->batches[b].type_batch_count; ++t) {
            int id = sc->batches[b].type_batches[t].type_id;
            if (id < 0 || id >= 64 || !registry<float>().ops[id].solve) return -3;
        }
    ext::ExtSolver e;
    e.s.sc = sc;
    e.terms = *terms;
    std::copy(sc->gravity, sc->gravity + 3, e.s.cb.gravity);
    e.s.cb.linear_damping = sc->linear_damping;
    e.s.cb.angular_damping = sc->angular_damping;
    e.s.cb.angular_mode = sc->angular_integration_mode;
    e.s.cb.allow_substeps_unconstrained = sc->allow_substeps_for_unconstrained != 0;
    e.s.cb.integrate_kinematic_velocity = sc->integrate_velocity_for_kinematics != 0;
    prepare_integration_responsibilities(e.s);
    if (sc->simd)
        ext::run_solve<f8>(e, dt);
    else
        ext::run_solve<float>(e, dt);
    ext::integrate_after_substepping(e, dt, sc->substep_count);
    return 0;
}

// PredictBoundingBoxes with the terms (PoseIntegrator.cs:L339-341, L428: the current pose, PrepareForIntegration with the frame dt). The
// oracle's routine runs twice: on the bodies as they are, for the sleep candidacy (it reads the velocity before the callback), and on a copy
// whose velocities already hold callback + terms, with a neutral callback (gravity 0, damping 0: v -> (v + 0) * 1), for the bounds.
extern "C" int32_t oracle_ext_predict_bounding_boxes(int32_t body_count, const float* bodies, const oracle_body_shape* shapes, oracle_body_activity* activities, float dt,
                                                     const float* gravity, float linear_damping, float angular_damping, int32_t integrate_velocity_for_kinematics,
                                                     const bepu_oracle::ext::Terms* terms, float* bounds_out) {
    using namespace bepu_oracle;
    if (body_count < 0 || !terms) return -1;
    std::vector<float> integrated(bodies, bodies + (size_t)body_count * 32);
    Callbacks cb{};
    std::copy(gravity, gravity + 3, cb.gravity);
    cb.linear_damping = linear_damping;
    cb.angular_damping = angular_damping;
    ext::ExtSolver e;
    e.s.cb = cb;
    e.terms = *terms;
    e.prepare(dt);
    for (int32_t i = 0; i < body_count; ++i) {
        float* b = integrated.data() + (size_t)i * 32;
        bool kinematic = true;  // Bodies.IsKinematic, Bodies.cs:L326-331
        for (int k = 16; k < 23; ++k) { uint32_t bits; std::memcpy(&bits, b + k, 4); kinematic = kinematic && bits == 0u; }
        if (!(integrate_velocity_for_kinematics != 0 || !kinematic)) continue;
        Velocity<float> v{{b[8], b[9], b[10]}, {b[12], b[13], b[14]}};
        e.integrate_velocity(v, V3<float>{b[4], b[5], b[6]}, &i);
        b[8] = v.lin.x; b[9] = v.lin.y; b[10] = v.lin.z;
        b[12] = v.ang.x; b[13] = v.ang.y; b[14] = v.ang.z;
    }
    std::vector<oracle_body_activity> scratch(activities, activities + body_count);
    int32_t rc = oracle_predict_bounding_boxes(body_count, bodies, shapes, activities, dt, gravity, linear_damping, angular_damping, integrate_velocity_for_kinematics, bounds_out);
    if (rc != 0) return rc;
    const float none[3] = {0.0f, 0.0f, 0.0f};
    return oracle_predict_bounding_boxes(body_count, integrated.data(), shapes, scratch.data(), dt, none, 0.0f, 0.0f, integrate_velocity_for_kinematics, bounds_out);
}

// The arithmetic of the terms alone, same operand layout as device_integrator_extensions_on_host_eval: v[0..5], linear acceleration[6..8], angular
// acceleration[9..11], dt[12], position[13..15], center[16..18], attractorDt[19], accelerations on[20] != 0, point gravity on[21] != 0 -> v.
extern "C" int32_t oracle_ext_eval(const float* in, float* out) {
    using namespace bepu_oracle;
    Velocity<float> v{{in[0], in[1], in[2]}, {in[3], in[4], in[5]}};
    ext::integrate_velocity_extensions<float>(v, in[20] != 0.0f, V3<float>{in[6], in[7], in[8]}, V3<float>{in[9], in[10], in[11]}, in[12], in[21] != 0.0f,
                                              V3<float>{in[13], in[14], in[15]}, V3<float>{in[16], in[17], in[18]}, in[19]);
    out[0] = v.lin.x; out[1] = v.lin.y; out[2] = v.lin.z; out[3] = v.ang.x; out[4] = v.ang.y; out[5] = v.ang.z;
    return 0;
}
