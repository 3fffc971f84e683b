// Sleepable islands on the device: the question IslandSleeper asks with CollectIsland and its SleepPredicate (IslandSleeper.cs:L85-223), answered
// for every island of the resident constraint graph at once. An island is a connected component of the graph whose vertices are the active-set
// bodies and whose edges are the constraints the device holds (every batch, the fallback levels included); kinematic references connect like any
// other, as Solver.EnumerateConnectedBodyReferences reports decoded references (Solver.cs:L1781-1784).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

#include "bepu_device_types.h"
#include "bepu_layout_kernels.h"

namespace bepucuda {

struct IslandBuffers {
    const DeviceTypeBatch* tbs;            // the resident type batches, read through the work list (work[0 .. work_count) covers every bundle once)
    const WorkItem* work;
    int32_t work_count;
    const uint8_t* activities;             // bepucuda_body_activity records, 8 bytes per body; only sleep_candidate (byte 6) is read
    int32_t* label;                        // per body: a body of the same island with a smaller index, or itself for the island's root
    int32_t* blocked;                      // per root: nonzero when a body of its island is not a sleep candidate
    int32_t* count;                        // per root: bodies in its island
    unsigned int* changed;                 // set by a hook pass that joined two trees
    int32_t body_count;
};

// Min-label connected components. label[b] = b at first; a round hooks, for every live constraint lane, the roots of its bodies onto the smallest
// of them (atomicMin), then points every body at its root. A parent always has a smaller index than its child, so the label forest stays acyclic
// and the root of a finished island is its smallest body index. Rounds repeat until a hook pass changes nothing (*changed == 0).
void launch_island_init(const IslandBuffers& ib, cudaStream_t s);
void launch_island_round(const IslandBuffers& ib, cudaStream_t s);
// Per body, into its root: count[root] += 1, blocked[root] |= !sleep_candidate.
void launch_island_verdict(const IslandBuffers& ib, cudaStream_t s);
// roots_out[0 .. *selected) = the roots r with blocked[r] == 0 in ascending order, counts_out[i] = count[roots_out[i]]. temp / temp_bytes: CUB
// scratch (temp == nullptr: *temp_bytes receives the size needed and nothing is launched). flags: body_count bytes of scratch.
cudaError_t launch_island_select(const IslandBuffers& ib, uint8_t* flags, int32_t* roots_out, int32_t* counts_out, int32_t* selected, void* temp, size_t* temp_bytes,
                                 cudaStream_t s);

}  // namespace bepucuda
