// Test shim of tests/test_body_write.py: check_body_write and gather_motion_halves of bepuphysics2_b200/csrc/bepu_topology.h behind a
// ctypes-friendly C interface. Built with g++ together with bepu_topology.cpp; the product never loads it.
#include "bepu_topology.h"

using namespace bepucuda;

extern "C" {

// The status of bepucuda_write_bodies' host check.
int body_write_check(int bodies_uploaded, int body_count, const void* body_dynamics, int count, const int32_t* body_indices) {
    const char* why = "";
    return check_body_write(bodies_uploaded != 0, body_count, body_dynamics, count, body_indices, &why);
}

// out: float[count][16], the staged motion halves.
void body_write_gather(const void* body_dynamics, const int32_t* body_indices, int count, float* out) {
    gather_motion_halves(body_dynamics, body_indices, count, out);
}

}  // extern "C"
