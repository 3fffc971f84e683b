// TEST INFRASTRUCTURE. One frame of the oracle's solve on a scene in which every constraint has bodies of its own, evaluated with the oracle's
// templated functions at a lane type F: float (the arithmetic of the strict CUDA build) or double (the same operations in float64, the
// yardstick that tests/test_fast_build_precision.py holds both GPU builds to). Nothing here is part of the product.
//
// Such a scene has one batch and every lane owns its dynamic bodies, so the driver follows run_solve's order for batch 0 alone: substeps > 0
// run the incremental contact update and the kinematic pose pass; WarmStart integrates each lane's bodies (integrate_pose_and_velocity or
// integrate_velocity_only) before the warm start; then the Solve iterations; after the last substep integrate_after_substepping's pose step of
// the constrained bodies. It calls the oracle's functions only and restates none of their arithmetic. The inputs are the scene's fp32 values in
// both entry points, and so are dt and the Callbacks::prepare products; in the double entry point body state, rows and impulses stay double.
//
// Build: g++ <oracle/Makefile CXXFLAGS> -Werror=float-conversion -I oracle -shared (a float64 value reaching a float overload fails the build).
#include "bepu_oracle.cpp"

namespace bepu_oracle {

// A body record of the driver: the floats of BodyDynamics (BodyProperties.cs:L318-338) as Scalar, the same layout as oracle_scene.bodies.
template <class F> struct IsolatedState {
    typedef typename LaneTraits<F>::Scalar S;
    S* bodies;         // body_count x 32
    S** prestep;       // per type batch of batch 0, AOSOA [bundle][row][W]
    S** impulses;
    static void load(const S* s, bool worldInertia, BodyIn<F>& b, Velocity<F>& v) {
        b.q = {s[0], s[1], s[2], s[3]};
        b.pos = {s[4], s[5], s[6]};
        v.lin = {s[8], s[9], s[10]};
        v.ang = {s[12], s[13], s[14]};
        const S* in = s + (worldInertia ? 24 : 16);
        b.inertia.t = {in[0], in[1], in[2], in[3], in[4], in[5]};
        b.inertia.inv_mass = in[6];
    }
    static void store_velocity(S* s, const Velocity<F>& v) {
        s[8] = v.lin.x; s[9] = v.lin.y; s[10] = v.lin.z;
        s[12] = v.ang.x; s[13] = v.ang.y; s[14] = v.ang.z;
    }
    static void store_pose(S* s, const V3<F>& pos, const Q4<F>& q) {
        s[0] = q.x; s[1] = q.y; s[2] = q.z; s[3] = q.w;
        s[4] = pos.x; s[5] = pos.y; s[6] = pos.z;
    }
    static void store_world_inertia(S* s, const Inertia<F>& in) {
        S* w = s + 24;
        w[0] = in.t.xx; w[1] = in.t.yx; w[2] = in.t.yy; w[3] = in.t.zx; w[4] = in.t.zy; w[5] = in.t.zz; w[6] = in.inv_mass;
    }
    S* body(int32_t encoded) const { return bodies + (size_t)(encoded & kBodyReferenceMask) * 32; }
};

static Callbacks callbacks_of(const oracle_scene& sc) {  // as oracle_solve sets them
    Callbacks cb{};
    std::copy(sc.gravity, sc.gravity + 3, cb.gravity);
    cb.linear_damping = sc.linear_damping;
    cb.angular_damping = sc.angular_damping;
    cb.angular_mode = sc.angular_integration_mode;
    cb.allow_substeps_unconstrained = sc.allow_substeps_for_unconstrained != 0;
    cb.integrate_kinematic_velocity = sc.integrate_velocity_for_kinematics != 0;
    cb.terms = sc.terms;
    return cb;
}

// 0, or negative when the scene is not one batch of constraints on bodies of their own with every body constrained.
static int32_t check_isolated(const oracle_scene& sc) {
    if (sc.batch_count != 1 || sc.substep_count < 1 || sc.bundle_width < 1 || sc.bundle_width > 32) return -1;
    std::vector<int> uses(sc.body_count, 0);
    const int W = sc.bundle_width;
    for (int t = 0; t < sc.batches[0].type_batch_count; ++t) {
        const oracle_type_batch& tb = sc.batches[0].type_batches[t];
        if (tb.type_id < 0 || tb.type_id >= 64 || !registry<float>().ops[tb.type_id].solve) return -2;
        const int nb = registry<float>().ops[tb.type_id].bodies;
        for (int c = 0; c < tb.constraint_count; ++c)
            for (int slot = 0; slot < nb; ++slot) {
                const int32_t enc = tb.body_references[((size_t)(c / W) * nb + slot) * W + (c % W)];
                if (enc < 0) return -3;  // a hole: the scene was not built by adds alone
                const int idx = enc & kBodyReferenceMask;
                if (idx >= sc.body_count || ++uses[idx] > 1) return -4;  // shared body
            }
    }
    for (int i = 0; i < sc.body_count; ++i)
        if (!uses[i]) return -5;  // an unconstrained body takes the other branch of integrate_after_substepping
    return 0;
}

template <class F> static void isolated_solve(const oracle_scene& sc, float dt, const IsolatedState<F>& st) {
    typedef IsolatedState<F> St;
    const int W = sc.bundle_width;
    const oracle_batch& batch = sc.batches[0];
    const auto& reg = registry<F>();
    Callbacks cb = callbacks_of(sc);
    const int substepCount = sc.substep_count;
    const float substepDt = dt / substepCount;
    cb.prepare(substepDt);
    const float inverseDt = 1.0f / substepDt;
    // every live lane of batch 0 once: (type batch, bundle, lane)
    struct Lane { int t, bundle, lane; };
    std::vector<Lane> lanes;
    for (int t = 0; t < batch.type_batch_count; ++t)
        for (int c = 0; c < batch.type_batches[t].constraint_count; ++c) lanes.push_back({t, c / W, c % W});
    auto rows = [&](const Lane& l, typename St::S* const* base, int count) {
        return Rows<F>{base[l.t] + (size_t)l.bundle * count * W + l.lane, W};
    };
    auto ref_of = [&](const Lane& l, int slot, int nb) { return batch.type_batches[l.t].body_references[((size_t)l.bundle * nb + slot) * W + l.lane]; };

    for (int substep = 0; substep < substepCount; ++substep) {
        if (substep > 0) {
            for (const Lane& l : lanes) {  // incremental_bundle
                const TypeOps<F>& ops = reg.ops[batch.type_batches[l.t].type_id];
                if (!ops.incremental) continue;
                BodyIn<F> body[4];
                Velocity<F> vel[4];
                for (int slot = 0; slot < ops.bodies; ++slot) St::load(st.body(ref_of(l, slot, ops.bodies)), true, body[slot], vel[slot]);
                ops.incremental(substepDt, vel, rows(l, st.prestep, ops.prestep_rows));
            }
            for (int i = 0; i < sc.constrained_kinematic_count; ++i) {  // integrate_kinematic_poses_and_velocities
                int32_t idx = sc.constrained_kinematics[i];
                BodyIn<F> b;
                Velocity<F> v;
                St::load(st.body(idx), false, b, v);
                b.pos = add(b.pos, scale(v.lin, bc<F>(substepDt)));
                b.q = integrate_orientation<F>(b.q, v.ang, bc<F>(substepDt * 0.5f));
                St::store_pose(st.body(idx), b.pos, b.q);
                if (cb.integrate_kinematic_velocity) {
                    cb.integrate_velocity(v, b.pos, &idx);
                    St::store_velocity(st.body(idx), v);
                }
            }
        } else if (cb.integrate_kinematic_velocity) {
            for (int i = 0; i < sc.constrained_kinematic_count; ++i) {  // integrate_kinematic_velocities
                int32_t idx = sc.constrained_kinematics[i];
                BodyIn<F> b;
                Velocity<F> v;
                St::load(st.body(idx), false, b, v);
                cb.integrate_velocity(v, b.pos, &idx);
                St::store_velocity(st.body(idx), v);
            }
        }
        for (const Lane& l : lanes) {  // warm_start_bundle, batch 0: every dynamic body of the lane is integrated here
            const TypeOps<F>& ops = reg.ops[batch.type_batches[l.t].type_id];
            BodyIn<F> body[4];
            Velocity<F> vel[4];
            int32_t refs[4];
            for (int slot = 0; slot < ops.bodies; ++slot) {
                refs[slot] = ref_of(l, slot, ops.bodies);
                const bool dynamic = (uint32_t)refs[slot] < kDynamicLimit;
                BodyIn<F> g;
                St::load(st.body(refs[slot]), false, g, vel[slot]);
                body[slot].pos = g.pos;
                body[slot].q = g.q;
                if (substep > 0) {
                    integrate_pose_and_velocity<F>(cb, g.inertia, substepDt, dynamic, body[slot].pos, body[slot].q, vel[slot], body[slot].inertia, &refs[slot]);
                    if (dynamic) St::store_pose(st.body(refs[slot]), body[slot].pos, body[slot].q);
                } else {
                    integrate_velocity_only<F>(cb, g.inertia, substepDt, dynamic, false, body[slot].pos, body[slot].q, vel[slot], body[slot].inertia, &refs[slot]);
                }
                if (dynamic) St::store_world_inertia(st.body(refs[slot]), body[slot].inertia);
            }
            ops.warm_start(body, rows(l, st.prestep, ops.prestep_rows), rows(l, st.impulses, ops.impulse_rows), vel);
            for (int slot = 0; slot < ops.bodies; ++slot)
                if ((uint32_t)refs[slot] < kDynamicLimit) St::store_velocity(st.body(refs[slot]), vel[slot]);
        }
        for (int it = 0; it < sc.velocity_iterations[substep]; ++it)
            for (const Lane& l : lanes) {  // solve_bundle
                const TypeOps<F>& ops = reg.ops[batch.type_batches[l.t].type_id];
                BodyIn<F> body[4];
                Velocity<F> vel[4];
                for (int slot = 0; slot < ops.bodies; ++slot) St::load(st.body(ref_of(l, slot, ops.bodies)), true, body[slot], vel[slot]);
                ops.solve(body, substepDt, inverseDt, rows(l, st.prestep, ops.prestep_rows), rows(l, st.impulses, ops.impulse_rows), vel);
                for (int slot = 0; slot < ops.bodies; ++slot) {
                    const int32_t enc = ref_of(l, slot, ops.bodies);
                    if ((uint32_t)enc < kDynamicLimit) St::store_velocity(st.body(enc), vel[slot]);
                }
            }
    }
    // integrate_after_substepping: every body is constrained (check_isolated) and takes one pose step of substep length
    const float effectiveDt = substepDt;
    const float halfDt = effectiveDt * 0.5f;
    for (int i = 0; i < sc.body_count; ++i) {
        BodyIn<F> b;
        Velocity<F> v;
        St::load(st.bodies + (size_t)i * 32, false, b, v);
        Q4<F> q = integrate_orientation<F>(b.q, v.ang, bc<F>(halfDt));
        V3<F> p = add(b.pos, scale(v.lin, bc<F>(effectiveDt)));
        St::store_pose(st.bodies + (size_t)i * 32, p, q);
    }
}

}  // namespace bepu_oracle

// In place on the scene's own fp32 buffers, like oracle_solve.
extern "C" int32_t isolated_solve_f32(const oracle_scene* sc, float dt) {
    if (!sc) return -1;
    int32_t rc = check_isolated(*sc);
    if (rc != 0) return rc;
    const oracle_batch& batch = sc->batches[0];
    std::vector<float*> prestep(batch.type_batch_count), impulses(batch.type_batch_count);
    for (int t = 0; t < batch.type_batch_count; ++t) {
        prestep[t] = batch.type_batches[t].prestep;
        impulses[t] = batch.type_batches[t].accumulated_impulses;
    }
    isolated_solve<float>(*sc, dt, IsolatedState<float>{sc->bodies, prestep.data(), impulses.data()});
    return 0;
}

// In place on float64 copies of the scene's buffers (same layouts); the scene's own fp32 buffers supply the references and are not written.
extern "C" int32_t isolated_solve_f64(const oracle_scene* sc, float dt, double* bodies, double** prestep, double** impulses) {
    if (!sc) return -1;
    int32_t rc = check_isolated(*sc);
    if (rc != 0) return rc;
    isolated_solve<double>(*sc, dt, IsolatedState<double>{bodies, prestep, impulses});
    return 0;
}
