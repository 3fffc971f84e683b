// TEST INFRASTRUCTURE. Compiles the device constraint functions of bepuphysics2_b200/csrc/{bepu_device_math,bepu_contacts,bepu_joints,
// bepu_joints_more}.cuh for the HOST (g++, -ffp-contract=off: the arithmetic of the strict -fmad=false CUDA build) and exposes one lane of one
// stage per call, so that the CPU test-suite can hold the CUDA source itself -- not only the GPU binary -- to the oracle bit for bit
// (tests/test_device_source_on_host.py). Nothing here is part of the product; the product never falls back to it.
//
// Build: g++ -O2 -std=c++17 -ffp-contract=off -fno-fast-math -march=x86-64-v3 -I tests/device_on_host/stubs -I bepuphysics2_b200/csrc -shared -fPIC
#define BEPU_NS bepu_device_on_host
#include "bepu_joints_more.cuh"  // pulls in bepu_joints.cuh, bepu_contacts.cuh, bepu_device_math.cuh (with the stub cuda_runtime.h)
#include "bepu_integration.cuh"

#include <atomic>
#include <thread>

namespace BEPU_NS {

// The per-body-count call adaptors of csrc/bepu_solver_kernels.cuh (call_warm_start / call_solve / call_incremental), restated: that header
// also holds the kernels proper (PTX, shared memory) and cannot be compiled for the host.
template <class T> static void call_warm_start(const BodyState* b, GlobalRows p, GlobalAcc a, Velocity* v) {
    if constexpr (T::kNeedsPose) T::warm_start(b, p, a, v);
    else if constexpr (T::kBodies == 2) T::warm_start(b[0].inertia, b[1].inertia, p, a, v[0], v[1]);
    else T::warm_start(b[0].inertia, p, a, v[0]);
}
template <class T> static void call_solve(const BodyState* b, float dt, float inverseDt, GlobalRows p, GlobalAcc a, Velocity* v) {
    if constexpr (T::kNeedsPose) T::solve(b, dt, inverseDt, p, a, v);
    else if constexpr (T::kBodies == 2) T::solve(b[0].inertia, b[1].inertia, dt, inverseDt, p, a, v[0], v[1]);
    else T::solve(b[0].inertia, dt, inverseDt, p, a, v[0]);
}
template <class T> static void call_incremental(float dt, const Velocity* v, float* p) {
    if constexpr (T::kIncremental) {
        if constexpr (T::kBodies == 2) T::incremental_update(dt, v[0], v[1], p);
        else T::incremental_update(dt, v[0], p);
    }
}

template <class T> static int eval(int stage, const float* body_states, float dt, float* prestep, float* impulses, float* velocities) {
    constexpr int NB = T::kBodies;
    BodyState b[NB];
    Velocity v[NB];
    for (int s = 0; s < NB; ++s) {
        const float* f = body_states + 14 * s;
        b[s].pos = {f[0], f[1], f[2]};
        b[s].q = {f[3], f[4], f[5], f[6]};
        b[s].inertia.t = {f[7], f[8], f[9], f[10], f[11], f[12]};
        b[s].inertia.inv_mass = f[13];
        const float* w = velocities + 6 * s;
        v[s].lin = {w[0], w[1], w[2]};
        v[s].ang = {w[3], w[4], w[5]};
    }
    if (stage == 0) call_warm_start<T>(b, GlobalRows{prestep}, GlobalAcc{impulses}, v);
    else if (stage == 1) call_solve<T>(b, dt, 1.0f / dt, GlobalRows{prestep}, GlobalAcc{impulses}, v);
    else call_incremental<T>(dt, v, prestep);
    for (int s = 0; s < NB; ++s) {
        float* w = velocities + 6 * s;
        w[0] = v[s].lin.x; w[1] = v[s].lin.y; w[2] = v[s].lin.z;
        w[3] = v[s].ang.x; w[4] = v[s].ang.y; w[5] = v[s].ang.z;
    }
    return 0;
}

}  // namespace BEPU_NS

using namespace BEPU_NS;

// Rows are laid out like one lane of a device bundle: row r of the lane is prestep[r * 32] (kLanes), same for impulses.
// body_states: per body 14 floats (position 3, orientation xyzw, world inverse inertia XX YX YY ZX ZY ZZ, inverse mass); velocities: per body 6.
// stage: 0 WarmStart, 1 Solve, 2 IncrementallyUpdateForSubstep. Returns -1 for an id without a type.
extern "C" int32_t device_on_host_eval_lane(int32_t type_id, int32_t stage, const float* body_states, float dt, float* prestep, float* impulses, float* velocities) {
    switch (type_id) {
#define CASE(ID, T) \
    case ID: return eval<T>(stage, body_states, dt, prestep, impulses, velocities);
        BEPU_CONTACT_TYPES(CASE)
        BEPU_JOINT_TYPES(CASE)
        BEPU_JOINT_TYPES_MORE(CASE)
#undef CASE
        default: return -1;
    }
}
extern "C" int32_t device_on_host_type_info(int32_t type_id, int32_t* bodies, int32_t* prestep_rows, int32_t* impulse_rows, int32_t* incremental) {
    switch (type_id) {
#define CASE(ID, T) \
    case ID: *bodies = T::kBodies; *prestep_rows = T::kPrestepRows; *impulse_rows = T::kImpulseRows; *incremental = T::kIncremental ? 1 : 0; return 0;
        BEPU_CONTACT_TYPES(CASE)
        BEPU_JOINT_TYPES(CASE)
        BEPU_JOINT_TYPES_MORE(CASE)
#undef CASE
        default: return -1;
    }
}

// The integration arithmetic of csrc/bepu_integration.cuh. op 0: integrate_orientation(q[0..3], w[4..6], halfDt[7]) -> q; 1: rotate_inverse_inertia(
// local[0..5], q[6..9]) -> 6 floats; 2: integrate_angular_conserve_momentum(previous q[0..3], local[4..9], world[10..15], w[16..18]) -> w;
// 3: integrate_angular_gyroscopic(q[0..3], local[4..9], w[10..12], dt[13]) -> w; 4: callback_integrate_velocity(v[0..5], gravity dt[6..8],
// linear damping dt[9], angular damping dt[10]) -> v; 5: integrate_velocity_extensions(v[0..5], linear acceleration[6..8], angular acceleration[9..11],
// dt[12], position[13..15], center[16..18], attractorDt[19], accelerations on[20] != 0, point gravity on[21] != 0) -> v.
extern "C" int32_t device_on_host_eval_integration(int32_t op, const float* in, float* out) {
    auto sym = [&](int i) { return Sym3{in[i], in[i + 1], in[i + 2], in[i + 3], in[i + 4], in[i + 5]}; };
    if (op == 0) {
        Q4 q = integrate_orientation(Q4{in[0], in[1], in[2], in[3]}, V3{in[4], in[5], in[6]}, in[7]);
        out[0] = q.x; out[1] = q.y; out[2] = q.z; out[3] = q.w;
    } else if (op == 1) {
        Sym3 r = rotate_inverse_inertia(sym(0), Q4{in[6], in[7], in[8], in[9]});
        out[0] = r.xx; out[1] = r.yx; out[2] = r.yy; out[3] = r.zx; out[4] = r.zy; out[5] = r.zz;
    } else if (op == 2) {
        V3 w{in[16], in[17], in[18]};
        integrate_angular_conserve_momentum(Q4{in[0], in[1], in[2], in[3]}, sym(4), sym(10), w);
        out[0] = w.x; out[1] = w.y; out[2] = w.z;
    } else if (op == 3) {
        V3 w{in[10], in[11], in[12]};
        integrate_angular_gyroscopic(Q4{in[0], in[1], in[2], in[3]}, sym(4), w, in[13]);
        out[0] = w.x; out[1] = w.y; out[2] = w.z;
    } else if (op == 4) {
        Velocity v{{in[0], in[1], in[2]}, {in[3], in[4], in[5]}};
        callback_integrate_velocity(v, in[6], in[7], in[8], in[9], in[10]);
        out[0] = v.lin.x; out[1] = v.lin.y; out[2] = v.lin.z; out[3] = v.ang.x; out[4] = v.ang.y; out[5] = v.ang.z;
    } else if (op == 5) {
        Velocity v{{in[0], in[1], in[2]}, {in[3], in[4], in[5]}};
        integrate_velocity_extensions(v, in[20] != 0.0f, V3{in[6], in[7], in[8]}, V3{in[9], in[10], in[11]}, in[12], in[21] != 0.0f, V3{in[13], in[14], in[15]},
                                      V3{in[16], in[17], in[18]}, in[19]);
        out[0] = v.lin.x; out[1] = v.lin.y; out[2] = v.lin.z; out[3] = v.ang.x; out[4] = v.ang.y; out[5] = v.ang.z;
    } else {
        return -1;
    }
    return 0;
}

// Impulse carry-over of the device-side contact update (csrc/bepu_redistribute.cuh, what redistribute_impulses_kernel runs per constraint) over a
// whole type batch in the reference AOSOA-W layout, with the operands of oracle_update_contact_impulses. Returns -1 for a type without contacts.
#include "bepu_redistribute.cuh"
extern "C" int32_t device_on_host_update_contact_impulses(int32_t type_id, int32_t constraint_count, int32_t W, float* accumulated_impulses, const int32_t* old_feature_ids,
                                                          const int32_t* new_feature_ids) {
    const int n = bepucuda::contact_count_of_type(type_id);
    if (n == 0) return -1;
    const int rows = bepucuda::type_row(type_id)->impulse_rows;
    for (int c = 0; c < constraint_count; ++c) {
        float* bundle = accumulated_impulses + (size_t)(c / W) * rows * W + (c % W);
        float oldImpulses[4], newImpulses[4];
        for (int i = 0; i < n; ++i) oldImpulses[i] = bundle[bepucuda::penetration_impulse_row(type_id, i) * W];
        bepucuda::redistribute_impulses(n, old_feature_ids + (size_t)c * n, oldImpulses, new_feature_ids + (size_t)c * n, newImpulses);
        for (int i = 0; i < n; ++i) bundle[bepucuda::penetration_impulse_row(type_id, i) * W] = newImpulses[i];
    }
    return 0;
}
// The row of contact i's penetration impulse that redistribute_impulses_kernel reads and writes.
extern "C" int32_t device_on_host_penetration_impulse_row(int32_t type_id, int32_t i) { return bepucuda::penetration_impulse_row(type_id, i); }

// PredictBoundingBoxes arithmetic of csrc/bepu_bounds_math.cuh (same operand layout as ref_convex_bounds of the transpiled reference's harness).
#include "bepu_bounds_math.cuh"
extern "C" int32_t device_on_host_convex_bounds(int32_t type, const float* dims, const float* margins, int32_t allow, const float* q, const float* pos, const float* lin, const float* ang,
                                                float dt, float* out) {
    using namespace BEPU_NS;
    if (!(type == 0 || type == 1 || type == 2 || type == 4)) return -1;
    const ConvexShape shape = {type, dims[0], dims[1], dims[2], margins[0], margins[1], allow};
    V3 mn, mx;
    float margin;
    convex_bounds(shape, Q4{q[0], q[1], q[2], q[3]}, V3{pos[0], pos[1], pos[2]}, Velocity{{lin[0], lin[1], lin[2]}, {ang[0], ang[1], ang[2]}}, dt, mn, mx, margin);
    out[0] = mn.x; out[1] = mn.y; out[2] = mn.z; out[3] = margin; out[4] = mx.x; out[5] = mx.y; out[6] = mx.z;
    return 0;
}
