// Test shim of tests/test_body_changes.py: replay_body_removes of bepuphysics2_b200/csrc/bepu_topology.h behind a ctypes-friendly C interface.
// Built with g++ together with bepu_topology.cpp; the product never loads it.
#include <cstring>

#include "bepu_topology.h"

using namespace bepucuda;

extern "C" {

// On success: *final_count and moved_to_out[count]; on failure neither is written. Returns the replay's code.
int body_removes(int body_count, int count, const int32_t* indices, int32_t* final_count, int32_t* moved_to_out) {
    int32_t n = 0;
    std::vector<int32_t> moved_to;
    std::string error;
    const int rc = replay_body_removes(body_count, count, indices, &n, &moved_to, &error);
    if (rc != 0) return rc;
    *final_count = n;
    if (!moved_to.empty()) std::memcpy(moved_to_out, moved_to.data(), moved_to.size() * sizeof(int32_t));
    return 0;
}

}  // extern "C"
