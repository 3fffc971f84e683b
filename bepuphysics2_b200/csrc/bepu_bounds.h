// PredictBoundingBoxes on the device (SURVEY.md §8 f4): PoseIntegrator.PredictBoundingBoxes (PoseIntegrator.cs:L307-370), UpdateSleepCandidacy
// (L286-304) and the convex-primitive path of BoundingBoxBatcher.ExecuteConvexBatch (Collidables/BoundingBoxBatcher.cs:L142-222) over the body
// arrays the solver keeps resident.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

#include "bepu_device_types.h"

namespace bepucuda {

// One record per body (32 bytes), uploaded by bepucuda_set_body_shapes. type = the reference's shape type id (Sphere.Id 0, Capsule.Id 1, Box.Id 2,
// Cylinder.Id 4); anything else (no shape, or a type whose bounds stay on the host) produces no bounds.
struct BodyShape {
    int32_t type;
    float a, b, c;                        // sphere: radius; capsule: radius, half length; box: half width, half height, half length; cylinder: radius, half length
    float minimum_speculative_margin, maximum_speculative_margin;
    int32_t allow_expansion_beyond_speculative_margin;
    int32_t pad;
};
// BodyActivity (BodyProperties.cs:L386-416), 8 bytes, updated in place.
struct BodyActivityRecord {
    float sleep_threshold;
    uint8_t minimum_timesteps_under_threshold, timesteps_under_threshold_count, sleep_candidate, pad;
};
struct PredictParams {
    float dt;
    float gravity_dt[3];           // PrepareForIntegration(dt) of the declarative callback (Demos/DemoCallbacks.cs:L79-86), with the FULL frame dt
    float linear_damping_dt, angular_damping_dt;
    int32_t integrate_velocity_for_kinematics;
    // bepucuda_set_body_accelerations / bepucuda_set_point_gravity, as in FrameParams (with the frame dt)
    const float4* accelerations;
    uint32_t integrate_extensions;
    float attractor_center[3];
    float attractor_dt;
};
// bounds: 8 floats per body {min.xyz, speculative margin, max.xyz, 1 if bounds were produced else 0}
void launch_predict_bounding_boxes(const BodyBuffers& B, const BodyShape* shapes, BodyActivityRecord* activities, float4* bounds, const PredictParams& params, cudaStream_t s);

}  // namespace bepucuda
