// TEST INFRASTRUCTURE. Compiles integrate_velocity_extensions of bepuphysics2_b200/csrc/bepu_integration.cuh for the HOST (g++ -ffp-contract=off:
// the arithmetic of the strict -fmad=false CUDA build), like tests/device_on_host does for the rest of that header, so that the CPU test-suite can
// hold the CUDA source of the optional velocity terms to the oracle bit for bit (tests/test_integrator_extensions.py).
// Build: g++ -O2 -std=c++17 -ffp-contract=off -fno-fast-math -march=x86-64-v3 -I tests/device_on_host/stubs -I bepuphysics2_b200/csrc -shared -fPIC
#define BEPU_NS bepu_device_on_host
#include "bepu_integration.cuh"

using namespace BEPU_NS;

// Same operand layout as oracle_ext_eval: v[0..5], linear acceleration[6..8], angular acceleration[9..11], dt[12], position[13..15], center[16..18],
// attractorDt[19], accelerations on[20] != 0, point gravity on[21] != 0 -> v.
extern "C" int32_t device_integrator_extensions_on_host_eval(const float* in, float* out) {
    Velocity v{{in[0], in[1], in[2]}, {in[3], in[4], in[5]}};
    integrate_velocity_extensions(v, in[20] != 0.0f, V3{in[6], in[7], in[8]}, V3{in[9], in[10], in[11]}, in[12], in[21] != 0.0f, V3{in[13], in[14], in[15]},
                                  V3{in[16], in[17], in[18]}, in[19]);
    out[0] = v.lin.x; out[1] = v.lin.y; out[2] = v.lin.z; out[3] = v.ang.x; out[4] = v.ang.y; out[5] = v.ang.z;
    return 0;
}
