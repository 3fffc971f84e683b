// Sleepable-island search kernels (sm_90a). See bepu_islands.h.
//
// Why the result does not depend on the order of atomics: every label a pass writes is a body of the same island with a smaller index than the
// body it is written to (hooks join two trees through a constraint both touch; the shortcut and the path splitting of find_root only move a pointer
// up its own tree). The forest is therefore acyclic and every tree is inside one island. The loop ends after a round in which no constraint lane
// saw two different roots, so every constraint then lies inside one tree and every tree is a whole island, rooted at its smallest body index.
// Integer work, bound by L2 atomics and dependent loads; no ordering between passes other than the kernel boundary.
#include <cub/device/device_select.cuh>
#include <thrust/iterator/counting_iterator.h>

#include "bepu_islands.h"

namespace bepucuda {

namespace {

// Root of x's tree. Path splitting: every visited body is pointed at its grandparent (atomicMin, so a concurrent hook that moved it higher up is
// kept). Loads bypass L1: a value another SM wrote during this pass shortens the walk, and a stale one is still a valid ancestor.
__device__ __forceinline__ int32_t find_root(int32_t* label, int32_t x) {
    int32_t p = __ldcg(label + x);
    while (p != x) {
        const int32_t gp = __ldcg(label + p);
        if (gp != p) atomicMin(label + x, gp);
        x = p;
        p = gp;
    }
    return x;
}

__global__ void island_init_kernel(IslandBuffers ib) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= ib.body_count) return;
    ib.label[i] = i;
    ib.blocked[i] = 0;
    ib.count[i] = 0;
}

// One warp per work item (32-lane bundle), one lane per constraint: hook the roots of the lane's bodies onto the smallest of them.
__global__ void island_hook_kernel(IslandBuffers ib) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= ib.work_count) return;
    const WorkItem w = ib.work[warp];
    const DeviceTypeBatch tb = ib.tbs[w.type_batch];
    const int nb = tb.bodies;
    const int32_t* refs = tb.refs + (size_t)w.bundle * nb * 32 + lane;
    int32_t roots[4];
    int32_t lowest = 0x7fffffff;
#pragma unroll
    for (int s = 0; s < 4; ++s) {
        roots[s] = -1;
        if (s >= nb) continue;
        const int32_t enc = refs[s * 32];
        if (enc < 0) continue;  // empty lane
        // drops the kinematic bit and the device's integration-ownership bits: a kinematic body joins islands like any other
        roots[s] = find_root(ib.label, (int32_t)((uint32_t)enc & kRefIndexMask));
        lowest = min(lowest, roots[s]);
    }
    bool hooked = false;
#pragma unroll
    for (int s = 0; s < 4; ++s) {
        if (roots[s] >= 0 && roots[s] != lowest) {
            atomicMin(ib.label + roots[s], lowest);
            hooked = true;
        }
    }
    if (__any_sync(0xFFFFFFFFu, hooked) && lane == 0) *ib.changed = 1u;
}

// One thread per body: point it at its root.
__global__ void island_shortcut_kernel(IslandBuffers ib) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= ib.body_count) return;
    const int32_t root = find_root(ib.label, i);
    if (__ldcg(ib.label + i) != root) ib.label[i] = root;  // nothing writes a label below its root: a plain store keeps the minimum
}

// One thread per body; the lanes of a warp that share a root add into it once.
__global__ void island_verdict_kernel(IslandBuffers ib) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= ib.body_count) return;
    const int32_t root = ib.label[i];
    const bool candidate = ib.activities[(size_t)i * 8 + 6] != 0;  // BodyActivity.SleepCandidate
    const unsigned active = __activemask();
    const unsigned peers = __match_any_sync(active, root);
    const bool any_blocked = (__ballot_sync(active, !candidate) & peers) != 0u;
    if ((threadIdx.x & 31) == (unsigned)(__ffs((int)peers) - 1)) {
        atomicAdd(ib.count + root, __popc(peers));
        if (any_blocked) ib.blocked[root] = 1;
    }
}

__global__ void island_flags_kernel(IslandBuffers ib, uint8_t* flags) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= ib.body_count) return;
    flags[i] = ib.label[i] == i && ib.blocked[i] == 0;
}

__global__ void island_gather_counts_kernel(IslandBuffers ib, const int32_t* roots, const int32_t* selected, int32_t* counts_out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= *selected) return;
    counts_out[i] = ib.count[roots[i]];
}

inline unsigned blocks_for(size_t threads) { return (unsigned)((threads + 255) / 256); }

}  // namespace

void launch_island_init(const IslandBuffers& ib, cudaStream_t s) { island_init_kernel<<<blocks_for((size_t)ib.body_count), 256, 0, s>>>(ib); }

void launch_island_round(const IslandBuffers& ib, cudaStream_t s) {
    island_hook_kernel<<<blocks_for((size_t)ib.work_count * 32), 256, 0, s>>>(ib);
    island_shortcut_kernel<<<blocks_for((size_t)ib.body_count), 256, 0, s>>>(ib);
}

void launch_island_verdict(const IslandBuffers& ib, cudaStream_t s) { island_verdict_kernel<<<blocks_for((size_t)ib.body_count), 256, 0, s>>>(ib); }

cudaError_t launch_island_select(const IslandBuffers& ib, uint8_t* flags, int32_t* roots_out, int32_t* counts_out, int32_t* selected, void* temp, size_t* temp_bytes,
                                 cudaStream_t s) {
    const thrust::counting_iterator<int32_t> indices(0);
    if (!temp) return cub::DeviceSelect::Flagged(nullptr, *temp_bytes, indices, flags, roots_out, selected, ib.body_count, s);
    island_flags_kernel<<<blocks_for((size_t)ib.body_count), 256, 0, s>>>(ib, flags);
    cudaError_t e = cub::DeviceSelect::Flagged(temp, *temp_bytes, indices, flags, roots_out, selected, ib.body_count, s);
    if (e != cudaSuccess) return e;
    island_gather_counts_kernel<<<blocks_for((size_t)ib.body_count), 256, 0, s>>>(ib, roots_out, selected, counts_out);
    return cudaGetLastError();
}

}  // namespace bepucuda
