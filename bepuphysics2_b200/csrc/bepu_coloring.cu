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

// Stages the references (and the priorities, given for order 2 only), runs rounds in chunks until every constraint has a batch, and copies the batch
// indices to batch_indices_out (host). *rounds: the rounds run, or -1 if a round assigned nothing (an internal error). A failing CUDA call
// returns its error, and its text in *failed.
#define CHECK(call) do { const cudaError_t _e = (call); if (_e != cudaSuccess) { *failed = #call; return _e; } } while (0)
cudaError_t color_constraints(ColoringScratch& scratch, int32_t constraint_count, int32_t bodies_per_constraint, const int32_t* encoded_body_references, int32_t body_count,
                              int32_t fallback_threshold, int32_t order, const uint32_t* priorities, int32_t* batch_indices_out, int64_t* rounds, const char** failed, cudaStream_t s) {
    constexpr int kRoundsPerChunk = 32;  // even: the ping-pong lists return to their starting roles after every chunk
    const size_t words = (size_t)constraint_count * bodies_per_constraint, nb = (size_t)std::max(body_count, 1), nc = (size_t)constraint_count;
    CHECK(scratch.refs.reserve(words * 4));
    CHECK(scratch.priorities.reserve(nc * 4));
    CHECK(scratch.body_min.reserve(nb * 8));
    CHECK(scratch.body_mask.reserve(nb * 8));
    CHECK(scratch.out.reserve(nc * 4));
    CHECK(scratch.lists.reserve(nc * 8));
    CHECK(scratch.counts.reserve((kRoundsPerChunk + 1) * 4));
    CHECK(cudaMemcpyAsync(scratch.refs.ptr, encoded_body_references, words * 4, cudaMemcpyHostToDevice, s));
    if (priorities) CHECK(cudaMemcpyAsync(scratch.priorities.ptr, priorities, nc * 4, cudaMemcpyHostToDevice, s));
    const ColoringBuffers cb{scratch.refs.as<int32_t>(), scratch.priorities.as<uint32_t>(), scratch.body_min.as<unsigned long long>(), scratch.body_mask.as<unsigned long long>(),
                             scratch.out.as<int32_t>(), {scratch.lists.as<int32_t>(), scratch.lists.as<int32_t>() + nc}, scratch.counts.as<unsigned int>(), constraint_count,
                             bodies_per_constraint, body_count, fallback_threshold, order};
    CHECK(cudaMemsetAsync(scratch.counts.ptr, 0, (kRoundsPerChunk + 1) * 4, s));
    launch_color_init(cb, s);
    unsigned int counts[kRoundsPerChunk + 1];
    *rounds = 0;
    for (;;) {
        for (int r = 0; r < kRoundsPerChunk; ++r) launch_color_round(cb, r, s);
        CHECK(cudaMemcpyAsync(counts, scratch.counts.ptr, sizeof(counts), cudaMemcpyDeviceToHost, s));
        CHECK(cudaStreamSynchronize(s));
        CHECK(cudaGetLastError());
        int used = kRoundsPerChunk;
        for (int r = 0; r < kRoundsPerChunk; ++r)
            if (counts[r + 1] == 0) { used = r + 1; break; }
        *rounds += used;
        if (counts[used] == 0) break;
        // every round assigns at least the constraint with the globally lowest key, so the list shrinks: the loop ends after at most constraint_count rounds
        if (counts[kRoundsPerChunk] >= counts[0]) { *rounds = -1; return cudaSuccess; }
        counts[0] = counts[kRoundsPerChunk];
        for (int r = 1; r <= kRoundsPerChunk; ++r) counts[r] = 0;
        CHECK(cudaMemcpyAsync(scratch.counts.ptr, counts, sizeof(counts), cudaMemcpyHostToDevice, s));
        CHECK(cudaStreamSynchronize(s));  // `counts` is a stack array: the copy must have read it before the next chunk's download overwrites it
    }
    CHECK(cudaMemcpyAsync(batch_indices_out, scratch.out.ptr, nc * 4, cudaMemcpyDeviceToHost, s));
    CHECK(cudaStreamSynchronize(s));
    return cudaSuccess;
}

}  // namespace bepucuda
