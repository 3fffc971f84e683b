// TEST INFRASTRUCTURE. Compiles integrate_pose_and_inertia of bepuphysics2_b200/csrc/bepu_integration.cuh -- the pose half of
// IntegratePoseAndVelocity that the WarmStart stages and the body part of the incremental contact update share -- for the HOST (g++,
// -ffp-contract=off: the arithmetic of the strict -fmad=false CUDA build), so that tests/test_body_integration_in_incremental.py can hold it to
// the oracle bit for bit without a GPU. Nothing here is part of the product.
#define BEPU_NS bepu_device_on_host
#include "bepu_integration.cuh"

// in: linear velocity [0..2], angular velocity [3..5], dt [6], local inverse inertia [7..12] (xx yx yy zx zy zz), position [13..15],
// orientation [16..19] (x y z w). out: position [0..2], orientation [3..6], world inverse inertia [7..12].
extern "C" int32_t pose_integration_on_host(const float* in, float* out) {
    using namespace BEPU_NS;
    V3 pos{in[13], in[14], in[15]};
    Q4 q{in[16], in[17], in[18], in[19]};
    Sym3 world;
    integrate_pose_and_inertia(V3{in[0], in[1], in[2]}, V3{in[3], in[4], in[5]}, in[6], Sym3{in[7], in[8], in[9], in[10], in[11], in[12]}, pos, q, world);
    const float r[13] = {pos.x, pos.y, pos.z, q.x, q.y, q.z, q.w, world.xx, world.yx, world.yy, world.zx, world.zy, world.zz};
    for (int i = 0; i < 13; ++i) out[i] = r[i];
    return 0;
}
