// Test shim for tests/test_integrated_warm_start_launch.py: which contact-only WarmStart instantiation launch_stage (csrc/bepu_solver_kernels.cu)
// runs for a resolved launch, as csrc/bepu_topology.h decides it. TEST INFRASTRUCTURE: the product never loads the shim.
#include "bepu_topology.h"

extern "C" int topology_integrated_warm_start_launch(int stage, int kernel, int flags) {
    return bepucuda::integrated_warm_start_launch(stage, bepucuda::StageLaunch{kernel, flags}) ? 1 : 0;
}
