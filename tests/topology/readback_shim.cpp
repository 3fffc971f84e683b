// Test shim for tests/test_constraint_readback.py: the inverse slot map of plan_topology (bepuphysics2_b200/csrc/bepu_topology.h) that
// topology_shim.cpp does not reach. Built with g++ together with topology_shim.cpp and bepu_topology.cpp, whose plan handles and accessors it
// shares; the product never loads it.
#include <cstring>

#include "bepu_topology.h"

using namespace bepucuda;

// the plan handle of topology_shim.cpp
struct PlanHandle {
    TopologyPlan plan;
    int rc;
    std::string error;
};

extern "C" {

int64_t topology_plan_inverse_size(void* h) { return (int64_t)((PlanHandle*)h)->plan.inverse.size(); }
// per source: its device type batch (synchronized) and its first inverse entry (fallback); per entry: device type batch, slot
void topology_plan_inverse(void* h, int32_t* source_type_batch, int64_t* source_inverse_offset, int32_t* inverse) {
    const TopologyPlan& p = ((PlanHandle*)h)->plan;
    std::memcpy(source_type_batch, p.source_type_batch.data(), p.source_type_batch.size() * 4);
    std::memcpy(source_inverse_offset, p.source_inverse_offset.data(), p.source_inverse_offset.size() * 8);
    for (size_t i = 0; i < p.inverse.size(); ++i) {
        inverse[2 * i] = p.inverse[i].type_batch;
        inverse[2 * i + 1] = p.inverse[i].slot;
    }
}

}  // extern "C"
