// PredictBoundingBoxes kernel (sm_90a), compiled -fmad=false with IEEE sqrt: the results are bit-identical to a non-contracting CPU evaluation of
// the reference's expressions (tests/test_bounds.py). One thread per body, fully coalesced: reads the 32-B pose / velocity / local inertia records
// the solver keeps resident (96 B), the 32-B shape record and the 8-B activity; writes 32 B of bounds + margin and the activity. HBM-bound
// (168 B per body); the bounding boxes of every body are independent, so there is nothing to order.
#define BEPU_NS bepu_bounds_math
#include "bepu_bounds_math.cuh"
#include "bepu_integration.cuh"
#include "bepu_bounds.h"

namespace bepucuda {

namespace {

using namespace bepu_bounds_math;

__global__ void predict_bounding_boxes_kernel(BodyBuffers B, const BodyShape* __restrict__ shapes, BodyActivityRecord* __restrict__ activities, float4* __restrict__ bounds,
                                              const __grid_constant__ PredictParams p) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B.count) return;
    const float4 q4 = B.pose[2 * (size_t)i], p4 = B.pose[2 * (size_t)i + 1];
    const float4 l4 = B.velocity[2 * (size_t)i], w4 = B.velocity[2 * (size_t)i + 1];
    const float4 i0 = B.inertia_local[2 * (size_t)i], i1 = B.inertia_local[2 * (size_t)i + 1];
    const Q4 orientation = {q4.x, q4.y, q4.z, q4.w};
    const V3 position = {p4.x, p4.y, p4.z};
    Velocity velocity = {{l4.x, l4.y, l4.z}, {w4.x, w4.y, w4.z}};
    // Bodies.IsKinematic (Bodies.cs:L326-331) compares the OR of the seven floats' bits with 0.0f as a float: inverse mass and inverse inertia
    // are all +0 or -0, in any mix
    const bool kinematic = i1.z == 0.0f && i0.x == 0.0f && i0.y == 0.0f && i0.z == 0.0f && i0.w == 0.0f && i1.x == 0.0f && i1.y == 0.0f;
    const bool integrate = p.integrate_velocity_for_kinematics != 0 || !kinematic;
    const float sleepEnergy = length_squared(velocity.lin) + length_squared(velocity.ang);
    // the integrated velocity is only used for the prediction; it is not stored (PoseIntegrator.cs:L339)
    if (integrate) {
        velocity.lin = (velocity.lin + V3{p.gravity_dt[0], p.gravity_dt[1], p.gravity_dt[2]}) * p.linear_damping_dt;
        velocity.ang = velocity.ang * p.angular_damping_dt;
        if (p.integrate_extensions) {
            V3 linearAcceleration{0.0f, 0.0f, 0.0f}, angularAcceleration{0.0f, 0.0f, 0.0f};
            if (p.integrate_extensions & kIntegrateAccelerations) {
                const float4 a0 = p.accelerations[2 * (size_t)i], a1 = p.accelerations[2 * (size_t)i + 1];
                linearAcceleration = {a0.x, a0.y, a0.z};
                angularAcceleration = {a1.x, a1.y, a1.z};
            }
            integrate_velocity_extensions(velocity, (p.integrate_extensions & kIntegrateAccelerations) != 0, linearAcceleration, angularAcceleration, p.dt,
                                          (p.integrate_extensions & kIntegratePointGravity) != 0, position,
                                          V3{p.attractor_center[0], p.attractor_center[1], p.attractor_center[2]}, p.attractor_dt);
        }
    }
    // UpdateSleepCandidacy (PoseIntegrator.cs:L286-304)
    BodyActivityRecord activity = activities[i];
    if (sleepEnergy > activity.sleep_threshold) {
        activity.timesteps_under_threshold_count = 0;
        activity.sleep_candidate = 0;
    } else if (activity.timesteps_under_threshold_count < 255) {
        ++activity.timesteps_under_threshold_count;
        if (activity.timesteps_under_threshold_count >= activity.minimum_timesteps_under_threshold) activity.sleep_candidate = 1;
    }
    activities[i] = activity;

    const BodyShape shape = shapes[i];
    if (!(shape.type == 0 || shape.type == 1 || shape.type == 2 || shape.type == 4)) {
        bounds[2 * (size_t)i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        bounds[2 * (size_t)i + 1] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        return;
    }
    const ConvexShape convex = {shape.type, shape.a, shape.b, shape.c, shape.minimum_speculative_margin, shape.maximum_speculative_margin, shape.allow_expansion_beyond_speculative_margin};
    V3 bundleMin, bundleMax;
    float speculativeMargin;
    convex_bounds(convex, orientation, position, velocity, p.dt, bundleMin, bundleMax, speculativeMargin);
    bounds[2 * (size_t)i] = make_float4(bundleMin.x, bundleMin.y, bundleMin.z, speculativeMargin);
    bounds[2 * (size_t)i + 1] = make_float4(bundleMax.x, bundleMax.y, bundleMax.z, 1.0f);
}

}  // namespace

void launch_predict_bounding_boxes(const BodyBuffers& B, const BodyShape* shapes, BodyActivityRecord* activities, float4* bounds, const PredictParams& params, cudaStream_t s) {
    if (B.count <= 0) return;
    predict_bounding_boxes_kernel<<<(unsigned)((B.count + 255) / 256), 256, 0, s>>>(B, shapes, activities, bounds, params);
}

}  // namespace bepucuda
