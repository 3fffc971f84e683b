// Device-side batch colouring (SURVEY.md §8 f3): the batch search of Solver.Add / FindCandidateBatch (Solver.cs:L984-1014, L1182-1199) for a whole
// constraint set at once, and the fixed point BatchCompressor works towards (BatchCompressor.cs:L233) when fed the current batch indices as priorities.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

#include "bepu_cuda_handles.h"

namespace bepucuda {

// Priority key of constraint c: constraints are assigned in ascending key order; ties cannot occur (the low word is the constraint index).
//   order 0 (insertion order): key = c                       -- exactly the sequence of Solver.Add calls
//   order 1 (hashed order)   : key = color_hash(c) << 32 | c -- a fixed pseudo-random permutation: O(log n) dependent rounds on bounded-degree graphs
//   order 2 (by priority)    : key = priorities[c] << 32 | c -- caller-defined (current batch index: compression)
__host__ __device__ inline uint32_t color_hash(uint32_t c) {
    uint32_t h = c * 0x9E3779B1u;
    h ^= h >> 15;
    h *= 0x85EBCA77u;
    h ^= h >> 13;
    h *= 0xC2B2AE3Du;
    h ^= h >> 16;
    return h;
}

struct ColoringBuffers {
    const int32_t* refs;             // [constraint][slot], slot stride = bodies_per_constraint; -1 = unused slot, bit 30 = kinematic (never blocks)
    const uint32_t* priorities;      // order 2 only
    unsigned long long* body_min;    // per body: lowest key among its uncoloured constraints (all ones = none)
    unsigned long long* body_mask;   // per body: synchronized batches already holding one of its constraints (batchReferencedHandles, transposed)
    int32_t* batch_out;              // per constraint: assigned batch index, -1 while uncoloured
    int32_t* list[2];                // uncoloured constraints, ping-pong
    unsigned int* counts;            // counts[r] = length of the list round r reads
    int32_t constraint_count, bodies_per_constraint, body_count, fallback_threshold, order;
};
// One round = launch_color_round: every uncoloured constraint that holds the lowest key on each of its dynamic bodies takes the lowest batch
// none of those bodies is in yet (first fit; the fallback batch when all synchronized batches are blocked). Reads list[round & 1] (counts[round]
// entries), appends the rest to list[(round + 1) & 1] / counts[round + 1], which must be zero beforehand.
void launch_color_init(const ColoringBuffers& cb, cudaStream_t s);
void launch_color_round(const ColoringBuffers& cb, int round, cudaStream_t s);

// bepucuda_color_constraints for checked arguments (bepu_coloring.cu). `scratch` keeps its device buffers from call to call.
struct ColoringScratch { DeviceBuffer refs, priorities, body_min, body_mask, out, lists, counts; };
cudaError_t color_constraints(ColoringScratch& scratch, int32_t constraint_count, int32_t bodies_per_constraint, const int32_t* encoded_body_references, int32_t body_count,
                              int32_t fallback_threshold, int32_t order, const uint32_t* priorities, int32_t* batch_indices_out, int64_t* rounds, const char** failed, cudaStream_t s);

}  // namespace bepucuda
