// Test shim for tests/test_sharded_fallback.py: the peer-sharding entry points of bepuphysics2_b200/csrc/bepu_topology.h that
// topology_shim.cpp does not reach (plan_topology with a rank and a fallback rank, exchange_targets). Built with g++ together with
// topology_shim.cpp and bepu_topology.cpp, whose plan handles and accessors it shares; the product never loads it.
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

// topology_plan in peer mode, for `rank` with `fallback_rank` (-1 = none)
void* topology_plan_peer(int n, const int32_t* meta, const int32_t* const* refs, int W, int fallback_threshold, int batch_count, int body_count, int rank,
                         int fallback_rank) {
    std::vector<SourceView> sources;
    for (int i = 0; i < n; ++i) sources.push_back({meta[4 * i], meta[4 * i + 1], meta[4 * i + 2], meta[4 * i + 3], refs[i]});
    PlanHandle* h = new PlanHandle;
    h->rc = plan_topology(sources, W, fallback_threshold, batch_count, body_count, true, &h->plan, &h->error, rank, fallback_rank);
    return h;
}

// exchange_targets of the peer-mode program of `plan` with per-device-batch boundary counts; out: kShardMaxExchanges cumulative targets
int topology_exchange_targets(void* plan, int substeps, const int32_t* iterations, int kinematic_count, int integrate_velocity_for_kinematics, int body_count,
                              const int32_t* boundary_count, unsigned long long* out) {
    const TopologyPlan& p = ((PlanHandle*)plan)->plan;
    const StageProgram prog = build_stage_program(p, std::vector<int32_t>(iterations, iterations + substeps), kinematic_count, integrate_velocity_for_kinematics != 0, true,
                                                  body_count);
    std::vector<unsigned long long> targets;
    std::string error;
    const int rc = exchange_targets(prog, std::vector<int32_t>(boundary_count, boundary_count + p.batches.size()), &targets, &error);
    if (rc == 0) std::memcpy(out, targets.data(), targets.size() * sizeof(unsigned long long));
    return rc;
}
int topology_max_exchanges() { return kShardMaxExchanges; }

}  // extern "C"
