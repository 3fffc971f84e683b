// Layout conversion and topology analysis kernels of libbepucuda (no constraint numerics here, compiled once):
//   - BodyDynamics 128-B AOS (BepuPhysics/BodyProperties.cs:L318-338)  <->  four arrays of 32-B records
//   - reference AOSOA-W type batch buffers (Constraints/TypeBatch.cs:L10-27)  <->  device AOSOA-32
//   - integration ownership (Solver_Solve.cs:L951-1044,L1072-1388) and the batch invariant check
#include "bepu_layout_kernels.h"
#include "bepu_redistribute.cuh"

namespace bepucuda {

// One thread per float4 of the AOS record: fully coalesced 128-B-per-body reads.
//   float4 0,1 -> pose | 2,3 -> velocity | 4,5 -> local inertia | 6,7 -> world inertia
__global__ void split_bodies_kernel(const float4* __restrict__ raw, int body_count, BodyBuffers B) {
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (size_t)body_count * 8) return;
    const size_t body = t >> 3;
    const int part = (int)(t & 7);
    float4 v = raw[t];
    if (part == 1 || part == 2 || part == 3) v.w = 0.0f;  // padding floats carry no meaning
    if (part == 5) v.w = 0.0f;
    if (part == 7) v.w = 0.0f;
    float4* dst = part < 2 ? B.pose : part < 4 ? B.velocity : part < 6 ? B.inertia_local : B.inertia_world;
    dst[body * 2 + (part & 1)] = v;
}

// Writes pose, velocity and world inertia back into the retained raw AOS image; local inertia and padding stay as uploaded.
__global__ void merge_bodies_kernel(float4* __restrict__ raw, int body_count, BodyBuffers B) {
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (size_t)body_count * 8) return;
    const size_t body = t >> 3;
    const int part = (int)(t & 7);
    if (part == 4 || part == 5) return;
    const float4* src = part < 2 ? B.pose : part < 4 ? B.velocity : B.inertia_world;
    float4 v = src[body * 2 + (part & 1)];
    float4 old = raw[t];
    if (part == 1 || part == 2 || part == 3 || part == 7) v.w = old.w;  // keep the host's padding bits
    raw[t] = v;
}

// Row 0 of lane `lane` of bundle `bundle` of an AOSOA-32 array with `rows` rows per bundle (a device type batch's body references, prestep or
// accumulated impulses); row r is at [r * 32]. A macro: as an inline function it changed the instructions nvcc selects for transpose_in_all_kernel.
#define SLOT_ROW0(base, rows, bundle, lane) ((base) + (size_t)(bundle) * (rows) * 32 + (lane))

// AOSOA-W (reference layout: [bundleW][row][W]) <-> AOSOA-32 for every device type batch in one launch.
// One warp per destination bundle; lane = destination constraint slot. `map` (fallback levels only) gives the source
// constraint index of each destination slot, -1 = padding; without a map slot i is source constraint i.
// For W = 8 a warp reads four 32-B sectors per row (sector-efficient) and writes one 128-B line per row.
__global__ void transpose_in_all_kernel(const DeviceTypeBatch* __restrict__ tbs, const TransposeDesc* __restrict__ descs, const WorkItem* __restrict__ work, int work_count,
                                        int W, int what) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= work_count) return;
    const WorkItem w = work[warp];
    const TransposeDesc d = descs[w.type_batch];
    if (what & kTransposePending) what &= d.flags;
    if (!(what & (kTransposeRefs | kTransposePrestep | kTransposeImpulses))) return;
    const DeviceTypeBatch tb = tbs[w.type_batch];
    const int slot = w.bundle * 32 + lane;
    int c = d.map ? d.map[slot] : slot;
    if (c >= d.src_count) c = -1;
    const size_t sb = c < 0 ? 0 : (size_t)(c / W), sl = c < 0 ? 0 : (size_t)(c % W);
    if (what & kTransposeRefs) {
        int32_t* dst = SLOT_ROW0(tb.refs, d.bodies, w.bundle, lane);
        for (int r = 0; r < d.bodies; ++r) {
            int32_t v = kRefEmpty;
            if (c >= 0) {
                v = d.src_refs[(sb * d.bodies + r) * W + sl];
                v = v < 0 ? kRefEmpty : (int32_t)(((uint32_t)v & kRefIndexMask) | ((uint32_t)v & kRefKinematicBit));
            }
            dst[r * 32] = v;
        }
    }
    if (what & kTransposePrestep) {
        float* dst = SLOT_ROW0(tb.prestep, d.prestep_rows, w.bundle, lane);
        for (int r = 0; r < d.prestep_rows; ++r) dst[r * 32] = c < 0 ? 0.0f : d.src_prestep[(sb * d.prestep_rows + r) * W + sl];
    }
    if (what & kTransposeImpulses) {
        float* dst = SLOT_ROW0(tb.impulses, d.impulse_rows, w.bundle, lane);
        for (int r = 0; r < d.impulse_rows; ++r) dst[r * 32] = c < 0 ? 0.0f : d.src_impulses[(sb * d.impulse_rows + r) * W + sl];
    }
}

// NarrowPhase.RedistributeImpulses on the device-resident penetration impulses, one constraint per lane (bepu_redistribute.cuh).
__global__ void redistribute_impulses_kernel(const DeviceTypeBatch* __restrict__ tbs, const TransposeDesc* __restrict__ descs, const WorkItem* __restrict__ work, int work_count) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= work_count) return;
    const WorkItem w = work[warp];
    const TransposeDesc d = descs[w.type_batch];
    if (!(d.flags & kDescRedistribute)) return;
    const DeviceTypeBatch tb = tbs[w.type_batch];
    const int slot = w.bundle * 32 + lane;
    const int c = d.map ? d.map[slot] : slot;
    if (c < 0 || c >= d.src_count) return;
    const int n = d.contacts;
    float* acc = tb.impulses + (size_t)w.bundle * d.impulse_rows * 32 + lane;
    float oldImpulses[4], newImpulses[4];
    for (int i = 0; i < n; ++i) oldImpulses[i] = acc[penetration_impulse_row(tb.type_id, i) * 32];
    redistribute_impulses(n, d.features_old + (size_t)c * n, oldImpulses, d.features_new + (size_t)c * n, newImpulses);
    for (int i = 0; i < n; ++i) acc[penetration_impulse_row(tb.type_id, i) * 32] = newImpulses[i];
}

// One thread per float4 of the motion half of a BodyDynamics record (float4 0,1 -> pose, 2,3 -> velocity).
__global__ void scatter_body_motion_kernel(const float4* __restrict__ raw, int body_count, BodyBuffers B) {
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (size_t)body_count * 4) return;
    const size_t body = t >> 2;
    const int part = (int)(t & 3);
    float4 v = raw[body * 8 + part];
    if (part != 0) v.w = 0.0f;  // padding floats carry no meaning (and hold versions / stamps on the device)
    (part < 2 ? B.pose : B.velocity)[body * 2 + (part & 1)] = v;
}
__global__ void gather_body_motion_kernel(float4* __restrict__ raw, int body_count, BodyBuffers B) {
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (size_t)body_count * 4) return;
    const size_t body = t >> 2;
    const int part = (int)(t & 3);
    float4 v = (part < 2 ? B.pose : B.velocity)[body * 2 + (part & 1)];
    if (part != 0) v.w = 0.0f;
    raw[body * 8 + part] = v;
}
__global__ void transpose_out_all_kernel(const DeviceTypeBatch* __restrict__ tbs, const TransposeDesc* __restrict__ descs, const WorkItem* __restrict__ work, int work_count,
                                         int W, int what) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= work_count) return;
    const WorkItem w = work[warp];
    const DeviceTypeBatch tb = tbs[w.type_batch];
    const TransposeDesc d = descs[w.type_batch];
    const int slot = w.bundle * 32 + lane;
    const int c = d.map ? d.map[slot] : slot;
    if (c < 0 || c >= d.src_count) return;
    const size_t sb = (size_t)(c / W), sl = (size_t)(c % W);
    if (what & kTransposePrestep) {
        const float* src = SLOT_ROW0(tb.prestep, d.prestep_rows, w.bundle, lane);
        for (int r = 0; r < d.prestep_rows; ++r) d.src_prestep[(sb * d.prestep_rows + r) * W + sl] = src[r * 32];
    }
    if (what & kTransposeImpulses) {
        const float* src = SLOT_ROW0(tb.impulses, d.impulse_rows, w.bundle, lane);
        for (int r = 0; r < d.impulse_rows; ++r) d.src_impulses[(sb * d.impulse_rows + r) * W + sl] = src[r * 32];
    }
}

// bepucuda_read_constraints: one warp per request. Lane l gathers words l and l + 32 of the request's record from the rows of its slot, so the
// warp stores the 256-B record as two coalesced 128-B rows; the only rows read are those of the requested constraints.
// Record words: kRecord* (bepu_layout_kernels.h).
__global__ void read_constraints_kernel(const DeviceTypeBatch* __restrict__ tbs, const TransposeDesc* __restrict__ descs, const DeviceSlot* __restrict__ inverse,
                                        const ReadRequest* __restrict__ requests, int count, int32_t* __restrict__ records) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= count) return;
    const ReadRequest q = requests[warp];
    const DeviceSlot at = q.at.type_batch < 0 ? inverse[q.at.slot] : q.at;
    int32_t out[2] = {lane == 0 ? q.type_id : 0, 0};
    if (at.type_batch >= 0) {
        const TransposeDesc d = descs[at.type_batch];
        const DeviceTypeBatch tb = tbs[at.type_batch];
        const int bundle = at.slot >> 5, l = at.slot & 31;
        for (int k = 0; k < 2; ++k) {
            const int w = lane + 32 * k;
            if (w == 1) {
                out[k] = 1;
            } else if (w >= kRecordRefs && w < kRecordImpulses) {
                // the host's encoding: the device-only ownership bits (DESIGN §2) cleared, empty slots -1
                const int r = w - kRecordRefs;
                const int32_t v = r < d.bodies ? SLOT_ROW0(tb.refs, d.bodies, bundle, l)[r * 32] : kRefEmpty;
                out[k] = v < 0 ? kRefEmpty : (int32_t)((uint32_t)v & (kRefIndexMask | kRefKinematicBit));
            } else if (w >= kRecordImpulses && w < kRecordPrestep) {
                if (w - kRecordImpulses < d.impulse_rows) out[k] = __float_as_int(SLOT_ROW0(tb.impulses, d.impulse_rows, bundle, l)[(w - kRecordImpulses) * 32]);
            } else if (w >= kRecordPrestep && w < kRecordEnd) {
                if (w - kRecordPrestep < d.prestep_rows) out[k] = __float_as_int(SLOT_ROW0(tb.prestep, d.prestep_rows, bundle, l)[(w - kRecordPrestep) * 32]);
            }
        }
    }
    int32_t* record = records + (size_t)warp * 64;
    record[lane] = out[0];
    record[lane + 32] = out[1];
}

// bepucuda_write_constraints: one warp per queued write; lane r writes prestep rows r and r + 32 of the write's slot. Only the written constraints'
// prestep rows are touched: their accumulated impulses and body references stay as they are.
__global__ void write_constraints_kernel(const DeviceTypeBatch* __restrict__ tbs, const TransposeDesc* __restrict__ descs, const PrestepWrite* __restrict__ writes,
                                         const float* __restrict__ rows, int count) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= count) return;
    const PrestepWrite q = writes[warp];
    const int n = descs[q.at.type_batch].prestep_rows;
    float* dst = SLOT_ROW0(tbs[q.at.type_batch].prestep, n, q.at.slot >> 5, q.at.slot & 31);
    for (int r = lane; r < n; r += 32) dst[r * 32] = rows[q.row0 + r];
}

// Pass 1 over every (constraint, body slot): first_batch[body] = min device batch referencing it as a dynamic body;
// per-body reference count and bitmask of synchronized batches for the batch-invariant check.
__global__ void ownership_pass1_kernel(const DeviceTypeBatch* __restrict__ tbs, const WorkItem* __restrict__ work, int work_count, int sync_batch_count, int body_count,
                                       int32_t* first_batch, int32_t* sync_refcount, unsigned long long* sync_mask, int32_t* error_flag) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= work_count) return;
    const WorkItem w = work[warp];
    const DeviceTypeBatch tb = tbs[w.type_batch];
    const int nb = tb.bodies;
    for (int s = 0; s < nb; ++s) {
        const int32_t enc = tb.refs[((size_t)w.bundle * nb + s) * 32 + lane];
        if (enc < 0 || (enc & kRefKinematicBit)) continue;
        const int idx = enc & kRefIndexMask;
        if (idx >= body_count) { atomicExch(error_flag, 2); continue; }
        atomicMin(first_batch + idx, tb.device_batch);
        if (tb.device_batch < sync_batch_count && tb.device_batch < 64) {
            atomicAdd(sync_refcount + idx, 1);
            atomicOr(sync_mask + idx, 1ull << tb.device_batch);
        }
    }
}
// Pass 2: set the integrate bit on the owning lane, mark constrained bodies.
__global__ void ownership_pass2_kernel(const DeviceTypeBatch* __restrict__ tbs, const WorkItem* __restrict__ work, int work_count, int body_count,
                                       const int32_t* __restrict__ first_batch, uint8_t* constrained) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= work_count) return;
    const WorkItem w = work[warp];
    const DeviceTypeBatch tb = tbs[w.type_batch];
    const int nb = tb.bodies;
    for (int s = 0; s < nb; ++s) {
        int32_t* r = tb.refs + ((size_t)w.bundle * nb + s) * 32 + lane;
        const int32_t enc = *r;
        if (enc < 0) continue;
        const int idx = enc & kRefIndexMask;
        if (idx >= body_count) continue;
        constrained[idx] = 1;  // kinematics referenced by constraints count as constrained too (Solver_Solve.cs:L1372-1381)
        if (enc & kRefKinematicBit) continue;
        if (first_batch[idx] == tb.device_batch) *r = (int32_t)((uint32_t)enc | kRefIntegrateBit);
    }
}
// Pass 3: per SOURCE bundle and body slot, "does any lane integrate"; then broadcast that to every lane of the source bundle.
__global__ void bundle_flags_pass_kernel(const DeviceTypeBatch* __restrict__ tbs, const TransposeDesc* __restrict__ descs, const WorkItem* __restrict__ work, int work_count,
                                         int W, int32_t* source_bundle_flags, int phase) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= work_count) return;
    const WorkItem w = work[warp];
    const DeviceTypeBatch tb = tbs[w.type_batch];
    const TransposeDesc d = descs[w.type_batch];
    const int slot_index = w.bundle * 32 + lane;
    const int c = d.map ? d.map[slot_index] : slot_index;
    if (c < 0 || c >= d.src_count) return;
    int32_t* flags = source_bundle_flags + ((size_t)d.src_bundle_base + (size_t)(c / W)) * 4;
    for (int s = 0; s < d.bodies; ++s) {
        int32_t* r = tb.refs + ((size_t)w.bundle * d.bodies + s) * 32 + lane;
        const int32_t enc = *r;
        if (enc < 0) continue;
        if (phase == 0) {
            if ((uint32_t)enc & kRefIntegrateBit) flags[s] = 1;
        } else if (flags[s]) {
            *r = (int32_t)((uint32_t)enc | kRefBundleIntegratesBit);
        }
    }
}
__global__ void check_invariant_kernel(int body_count, const int32_t* __restrict__ sync_refcount, const unsigned long long* __restrict__ sync_mask, int32_t* error_flag) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= body_count) return;
    if (__popcll(sync_mask[i]) != sync_refcount[i]) atomicExch(error_flag, 1);
}
__global__ void mark_kinematics_kernel(const int32_t* __restrict__ kinematics, int count, int body_count, uint8_t* constrained, int32_t* error_flag) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const int idx = kinematics[i];
    if (idx < 0 || idx >= body_count) { atomicExch(error_flag, 2); return; }
    constrained[idx] = 1;
}
// Peer sharding: the integration owner of a body is the lowest batch referencing it on any rank. `global` holds host batch indices, which are the
// device batch indices of the synchronized batches on every rank. A body the whole graph first references in the fallback batch (global index at
// or above the threshold) keeps the device batch pass 1 found: only the fallback rank has lanes there, and it numbers its levels itself.
__global__ void merge_first_batch_kernel(int32_t* __restrict__ first_batch, const int32_t* __restrict__ global, int body_count, int fallback_threshold) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= body_count) return;
    const int32_t g = global[i];
    if (g < fallback_threshold) first_batch[i] = g;
}
__global__ void fill_i32_kernel(int32_t* p, size_t n, int32_t v) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}

// Batched copy: ONE launch moves every (page-locked, device-mapped) host buffer of a frame across PCIe/C2C in either direction, replacing hundreds of
// small cudaMemcpyAsync calls (one per type batch buffer). Chunks are <= 64 KiB; a CTA streams a chunk with 16-byte accesses, fully coalesced, so the
// link sees maximum-size read/write requests and many of them in flight.
__global__ void batched_copy_kernel(const CopyChunk* __restrict__ chunks, int chunk_count) {
    for (int c = blockIdx.x; c < chunk_count; c += gridDim.x) {
        const CopyChunk ch = chunks[c];
        if ((((size_t)ch.dst | (size_t)ch.src | ch.bytes) & 15) == 0) {
            const uint4* s = reinterpret_cast<const uint4*>(ch.src);
            uint4* d = reinterpret_cast<uint4*>(ch.dst);
            const size_t n = ch.bytes >> 4;
            for (size_t i = threadIdx.x; i < n; i += blockDim.x) d[i] = s[i];
        } else {
            const uint32_t* s = reinterpret_cast<const uint32_t*>(ch.src);
            uint32_t* d = reinterpret_cast<uint32_t*>(ch.dst);
            const size_t n = ch.bytes >> 2;
            for (size_t i = threadIdx.x; i < n; i += blockDim.x) d[i] = s[i];
        }
    }
}
void launch_batched_copy(const CopyChunk* chunks, int chunk_count, cudaStream_t s) {
    if (chunk_count <= 0) return;
    const int grid = chunk_count < 1184 ? chunk_count : 1184;  // 8 CTAs per SM at most; each keeps 256 x 16 B in flight
    batched_copy_kernel<<<grid, 256, 0, s>>>(chunks, chunk_count);
}

static inline unsigned blocks_for(size_t n, int threads) { return (unsigned)((n + threads - 1) / threads); }

void launch_split_bodies(const void* raw, int body_count, const BodyBuffers& B, cudaStream_t s) {
    if (body_count <= 0) return;
    split_bodies_kernel<<<blocks_for((size_t)body_count * 8, 256), 256, 0, s>>>((const float4*)raw, body_count, B);
}
void launch_merge_bodies(void* raw, int body_count, const BodyBuffers& B, cudaStream_t s) {
    if (body_count <= 0) return;
    merge_bodies_kernel<<<blocks_for((size_t)body_count * 8, 256), 256, 0, s>>>((float4*)raw, body_count, B);
}
void launch_transpose_in_all(const DeviceTypeBatch* tbs, const TransposeDesc* descs, const WorkItem* work, int work_count, int W, int what, cudaStream_t s) {
    if (work_count <= 0) return;
    transpose_in_all_kernel<<<blocks_for((size_t)work_count * 32, 128), 128, 0, s>>>(tbs, descs, work, work_count, W, what);
}
void launch_transpose_out_all(const DeviceTypeBatch* tbs, const TransposeDesc* descs, const WorkItem* work, int work_count, int W, int what, cudaStream_t s) {
    if (work_count <= 0) return;
    transpose_out_all_kernel<<<blocks_for((size_t)work_count * 32, 128), 128, 0, s>>>(tbs, descs, work, work_count, W, what);
}
void launch_read_constraints(const DeviceTypeBatch* tbs, const TransposeDesc* descs, const DeviceSlot* inverse, const ReadRequest* requests, int count, int32_t* records,
                             cudaStream_t s) {
    if (count <= 0) return;
    read_constraints_kernel<<<blocks_for((size_t)count * 32, 128), 128, 0, s>>>(tbs, descs, inverse, requests, count, records);
}
void launch_write_constraints(const DeviceTypeBatch* tbs, const TransposeDesc* descs, const PrestepWrite* writes, const float* rows, int count, cudaStream_t s) {
    if (count <= 0) return;
    write_constraints_kernel<<<blocks_for((size_t)count * 32, 128), 128, 0, s>>>(tbs, descs, writes, rows, count);
}
void launch_redistribute_impulses(const DeviceTypeBatch* tbs, const TransposeDesc* descs, const WorkItem* work, int work_count, cudaStream_t s) {
    if (work_count <= 0) return;
    redistribute_impulses_kernel<<<blocks_for((size_t)work_count * 32, 128), 128, 0, s>>>(tbs, descs, work, work_count);
}
void launch_scatter_body_motion(const void* raw, int body_count, const BodyBuffers& B, cudaStream_t s) {
    if (body_count <= 0) return;
    scatter_body_motion_kernel<<<blocks_for((size_t)body_count * 4, 256), 256, 0, s>>>((const float4*)raw, body_count, B);
}
void launch_gather_body_motion(void* raw, int body_count, const BodyBuffers& B, cudaStream_t s) {
    if (body_count <= 0) return;
    gather_body_motion_kernel<<<blocks_for((size_t)body_count * 4, 256), 256, 0, s>>>((float4*)raw, body_count, B);
}
// ---- peer sharding ------------------------------------------------------------------------------------------------------------------------
// Rank barrier. Launched with programmatic stream serialization like the stage kernels: it may start while the stage before it is still running,
// waits for that stage to complete, and only then lets the NEXT stage's grid start its prologue (work record, body references, row prefetch),
// which overlaps with the barrier below.
__global__ void __launch_bounds__(256, 1)
shard_barrier_kernel(ShardPeers peers, const FrameParams* __restrict__ fpp, uint32_t exchange_index, int32_t* error_flag) {
    pdl_wait_then_trigger((int32_t)exchange_index);  // the hazard build's delay field rides in the high bits of the exchange index
#ifdef BEPU_HAZARD
    exchange_index &= 0xffffu;
#endif
    const unsigned long long seq = (unsigned long long)fpp->exchange_base + exchange_index + 1ull;
    const int p = threadIdx.x;
    if (p < peers.rank_count && p != peers.rank) {
        asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(peers.flags[p] + peers.rank), "l"(seq) : "memory");
        unsigned long long seen;
        unsigned int spins = 0;
        do {
            asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(seen) : "l"(peers.flags[peers.rank] + p) : "memory");
        } while (seen < seq && ++spins < 200000000u);
        if (seen < seq) atomicExch(error_flag, 5);  // a peer never arrived: results are void
    }
}
void launch_shard_barrier(const ShardPeers& peers, const FrameParams* fp, uint32_t exchange_index, int32_t* error_flag, cudaStream_t s) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(1);
    cfg.blockDim = dim3(256);
    cfg.stream = s;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    cudaLaunchKernelEx(&cfg, shard_barrier_kernel, peers, fp, exchange_index, error_flag);
}
__global__ void fill_peer_masks_kernel(const int32_t* __restrict__ refs, uint32_t* __restrict__ peer_masks, size_t count, const uint8_t* __restrict__ body_masks, int rank) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const int32_t enc = refs[i];
    uint32_t m = 0;
    if (enc >= 0 && !((uint32_t)enc & kRefKinematicBit)) m = (uint32_t)body_masks[(uint32_t)enc & kRefIndexMask] & ~(1u << rank);
    peer_masks[i] = m;
}
void launch_fill_peer_masks(const int32_t* refs, uint32_t* peer_masks, size_t count, const uint8_t* body_masks, int rank, cudaStream_t s) {
    if (count == 0) return;
    fill_peer_masks_kernel<<<blocks_for(count, 256), 256, 0, s>>>(refs, peer_masks, count, body_masks, rank);
}
__global__ void boundary_flags_kernel(const DeviceTypeBatch* __restrict__ tbs, const WorkItem* __restrict__ work, int work_count, long long peer_delta,
                                      uint8_t* __restrict__ flags) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= work_count) return;
    const WorkItem w = work[warp];
    const DeviceTypeBatch tb = tbs[w.type_batch];
    const int32_t* refs = tb.refs + (size_t)w.bundle * tb.bodies * 32 + lane;
    uint32_t m = 0;
    for (int s = 0; s < tb.bodies; ++s) m |= (uint32_t)refs[peer_delta + s * 32];
    const bool any = __any_sync(0xFFFFFFFFu, m != 0);
    if (lane == 0) flags[warp] = any ? 1 : 0;
}
__global__ void pack_ref_rows_kernel(const WorkRecord* __restrict__ records, int count, int32_t* __restrict__ rows) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)count * 64) return;
    // the reference arena is padded: the second row of a one-body type batch is in bounds (and ignored by the kernels)
    rows[i] = records[i >> 6].refs[i & 63];
}
void launch_pack_ref_rows(const WorkRecord* records, int count, int32_t* rows, cudaStream_t s) {
    if (count <= 0) return;
    pack_ref_rows_kernel<<<blocks_for((size_t)count * 64, 256), 256, 0, s>>>(records, count, rows);
}
void launch_boundary_flags(const DeviceTypeBatch* tbs, const WorkItem* work, int work_count, long long peer_delta, uint8_t* flags, cudaStream_t s) {
    if (work_count <= 0) return;
    boundary_flags_kernel<<<blocks_for((size_t)work_count * 32, 128), 128, 0, s>>>(tbs, work, work_count, peer_delta, flags);
}
void launch_fill_i32(int32_t* p, size_t n, int32_t v, cudaStream_t s) {
    if (n == 0) return;
    fill_i32_kernel<<<blocks_for(n, 256), 256, 0, s>>>(p, n, v);
}
void launch_ownership_pass1(const DeviceTypeBatch* tbs, const WorkItem* work, int work_count, int sync_batch_count, int body_count,
                            int32_t* first_batch, int32_t* sync_refcount, unsigned long long* sync_mask, int32_t* error_flag, cudaStream_t s) {
    if (work_count > 0)
        ownership_pass1_kernel<<<blocks_for((size_t)work_count * 32, 128), 128, 0, s>>>(tbs, work, work_count, sync_batch_count, body_count, first_batch,
                                                                                         sync_refcount, sync_mask, error_flag);
}
void launch_merge_first_batch(int32_t* first_batch, const int32_t* global_first_batch, int body_count, int fallback_threshold, cudaStream_t s) {
    if (body_count > 0) merge_first_batch_kernel<<<blocks_for(body_count, 256), 256, 0, s>>>(first_batch, global_first_batch, body_count, fallback_threshold);
}
void launch_ownership_rest(const DeviceTypeBatch* tbs, const WorkItem* work, int work_count, int body_count, const int32_t* first_batch,
                           const int32_t* sync_refcount, const unsigned long long* sync_mask, uint8_t* constrained, const int32_t* kinematics, int kinematic_count,
                           int32_t* error_flag, const TransposeDesc* descs, int W, int32_t* source_bundle_flags, cudaStream_t s) {
    if (work_count > 0) {
        ownership_pass2_kernel<<<blocks_for((size_t)work_count * 32, 128), 128, 0, s>>>(tbs, work, work_count, body_count, first_batch, constrained);
        bundle_flags_pass_kernel<<<blocks_for((size_t)work_count * 32, 128), 128, 0, s>>>(tbs, descs, work, work_count, W, source_bundle_flags, 0);
        bundle_flags_pass_kernel<<<blocks_for((size_t)work_count * 32, 128), 128, 0, s>>>(tbs, descs, work, work_count, W, source_bundle_flags, 1);
    }
    if (body_count > 0) check_invariant_kernel<<<blocks_for(body_count, 256), 256, 0, s>>>(body_count, sync_refcount, sync_mask, error_flag);
    if (kinematic_count > 0) mark_kinematics_kernel<<<blocks_for(kinematic_count, 128), 128, 0, s>>>(kinematics, kinematic_count, body_count, constrained, error_flag);
}

}  // namespace bepucuda
