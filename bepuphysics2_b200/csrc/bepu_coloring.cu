// Device-side batch colouring kernels (sm_90a). See bepu_coloring.h.
//
// Why this reproduces sequential first fit exactly: Solver.Add gives constraint c the first batch that holds none of the constraints added before c
// which share a dynamic body with c. Here c is assigned in the round in which it holds the lowest key on every one of its dynamic bodies, i.e. when
// all lower-key constraints on those bodies have been assigned and no higher-key one has (a higher-key neighbour is not the minimum on the shared
// body while c is unassigned). The per-body masks then hold exactly the batches of c's lower-key neighbours, so the lowest free bit is the batch
// sequential first fit in key order would have chosen. Integer work, HBM/atomic-bound; no ordering between rounds other than the kernel boundary.
#include "bepu_coloring.h"

namespace bepucuda {

namespace {

constexpr unsigned long long kNoKey = ~0ull;
constexpr uint32_t kKinematicBit = 1u << 30;

__device__ __forceinline__ unsigned long long key_of(const ColoringBuffers& cb, int c) {
    const uint32_t hi = cb.order == 0 ? 0u : (cb.order == 1 ? color_hash((uint32_t)c) : cb.priorities[c]);
    return ((unsigned long long)hi << 32) | (uint32_t)c;
}

__global__ void color_init_kernel(ColoringBuffers cb) {
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < (size_t)cb.body_count; i += stride) {
        cb.body_min[i] = kNoKey;
        cb.body_mask[i] = 0ull;
    }
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < (size_t)cb.constraint_count; i += stride) {
        cb.batch_out[i] = -1;
        cb.list[0][i] = (int32_t)i;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) cb.counts[0] = (unsigned int)cb.constraint_count;
}

// Per body: the lowest key among its uncoloured constraints.
__global__ void color_min_kernel(ColoringBuffers cb, int round) {
    const unsigned int n = cb.counts[round];
    const int32_t* list = cb.list[round & 1];
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const int c = list[i];
        const unsigned long long key = key_of(cb, c);
        for (int s = 0; s < cb.bodies_per_constraint; ++s) {
            const int32_t enc = cb.refs[(size_t)c * cb.bodies_per_constraint + s];
            if (enc < 0 || ((uint32_t)enc & kKinematicBit)) continue;
            atomicMin(cb.body_min + ((uint32_t)enc & (kKinematicBit - 1u)), key);
        }
    }
}

__global__ void color_assign_kernel(ColoringBuffers cb, int round) {
    const unsigned int n = cb.counts[round];
    const int32_t* list = cb.list[round & 1];
    int32_t* next = cb.list[(round + 1) & 1];
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    const size_t first = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    // whole warps iterate together so that the appends can be aggregated
    for (size_t base = first - (threadIdx.x & 31); base < n; base += stride) {
        const size_t i = base + (threadIdx.x & 31);
        bool pending = false;
        int c = -1;
        if (i < n) {
            c = list[i];
            const unsigned long long key = key_of(cb, c);
            bool ready = true;
            unsigned long long used = 0ull;
            for (int s = 0; s < cb.bodies_per_constraint; ++s) {
                const int32_t enc = cb.refs[(size_t)c * cb.bodies_per_constraint + s];
                if (enc < 0 || ((uint32_t)enc & kKinematicBit)) continue;
                const uint32_t b = (uint32_t)enc & (kKinematicBit - 1u);
                ready = ready && cb.body_min[b] == key;
                used |= cb.body_mask[b];  // only meaningful when ready: then nobody else writes these masks in this round
            }
            if (ready) {
                const int T = cb.fallback_threshold;
                const unsigned long long candidates = ~used & (T >= 64 ? ~0ull : ((1ull << T) - 1ull));
                const int batch = candidates ? __ffsll((long long)candidates) - 1 : T;  // TryAllocateInBatch: index == threshold accepts everything
                for (int s = 0; s < cb.bodies_per_constraint; ++s) {
                    const int32_t enc = cb.refs[(size_t)c * cb.bodies_per_constraint + s];
                    if (enc < 0 || ((uint32_t)enc & kKinematicBit)) continue;
                    const uint32_t b = (uint32_t)enc & (kKinematicBit - 1u);
                    if (batch < T) cb.body_mask[b] |= 1ull << batch;
                    cb.body_min[b] = kNoKey;  // the next round recomputes this body's minimum over what is left
                }
                cb.batch_out[c] = batch;
            } else {
                pending = true;
            }
        }
        const unsigned int ballot = __ballot_sync(0xFFFFFFFFu, pending);
        if (ballot) {
            unsigned int offset = 0;
            const int leader = __ffs((int)ballot) - 1;
            if ((threadIdx.x & 31) == leader) offset = atomicAdd(cb.counts + round + 1, (unsigned int)__popc(ballot));
            offset = __shfl_sync(0xFFFFFFFFu, offset, leader);
            if (pending) next[offset + __popc(ballot & ((1u << (threadIdx.x & 31)) - 1u))] = c;
        }
    }
}

inline unsigned grid_for(size_t n) {
    const size_t blocks = (n + 255) / 256;
    return (unsigned)(blocks < 1 ? 1 : (blocks > 132 * 8 ? 132 * 8 : blocks));  // grid-stride: at most 8 CTAs per SM of an H100 SXM (132 SMs)
}

}  // namespace

void launch_color_init(const ColoringBuffers& cb, cudaStream_t s) {
    const size_t n = (size_t)(cb.constraint_count > cb.body_count ? cb.constraint_count : cb.body_count);
    color_init_kernel<<<grid_for(n), 256, 0, s>>>(cb);
}
void launch_color_round(const ColoringBuffers& cb, int round, cudaStream_t s) {
    const unsigned grid = grid_for((size_t)cb.constraint_count);
    color_min_kernel<<<grid, 256, 0, s>>>(cb, round);
    color_assign_kernel<<<grid, 256, 0, s>>>(cb, round);
}

}  // namespace bepucuda
