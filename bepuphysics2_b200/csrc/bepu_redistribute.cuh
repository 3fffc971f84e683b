// Per-constraint arithmetic of the device-side contact update (redistribute_impulses_kernel, bepu_layout_kernels.cu): plain scalar fp32 behind
// __host__ __device__, in its own header so that tests/device_on_host can compile it for the host and check it without a GPU.
#pragma once
#include <cstdint>

namespace bepucuda {

// Row of contact i's penetration impulse among a contact constraint's accumulated impulses: convex types [2 + i] (after the two tangent rows,
// ContactConstraintAccessor.cs:L58-66), nonconvex types [3 i + 2] (L70-76).
__host__ __device__ __forceinline__ int penetration_impulse_row(int type_id, int i) { return type_id < 8 ? 2 + i : 3 * i + 2; }

// NarrowPhase.RedistributeImpulses (CollisionDetection/NarrowPhaseConstraintUpdate.cs:L81-135) for one constraint of n (<= 4) contacts, old and
// new counts equal (the same-type update, L172-183): a new contact whose feature id matches an old one takes that contact's accumulated impulse
// (the first old contact with the id, whose impulse is then zeroed); the impulse left on unmatched old contacts is shared equally among the
// unmatched new contacts. oldImpulses is consumed.
__host__ __device__ __forceinline__ void redistribute_impulses(int n, const int32_t* oldIds, float* oldImpulses, const int32_t* newIds, float* newImpulses) {
    int unmatchedCount = 0;
    for (int i = 0; i < n; ++i) {
        newImpulses[i] = -1.0f;  // accumulated impulses cannot be negative: negative = unmatched
        for (int j = 0; j < n; ++j) {
            if (oldIds[j] == newIds[i]) {
                newImpulses[i] = oldImpulses[j];
                oldImpulses[j] = 0.0f;  // not distributed to the unmatched contacts
                break;
            }
        }
        if (newImpulses[i] < 0.0f) ++unmatchedCount;
    }
    if (unmatchedCount > 0) {
        float unmatchedImpulse = 0.0f;
        for (int i = 0; i < n; ++i) unmatchedImpulse += oldImpulses[i];
        const float impulsePerUnmatched = unmatchedImpulse / (float)unmatchedCount;
        for (int i = 0; i < n; ++i)
            if (newImpulses[i] < 0.0f) newImpulses[i] = impulsePerUnmatched;
    }
}

}  // namespace bepucuda
