// Launchers of the layout / topology kernels (bepu_layout_kernels.cu).
#pragma once
#include "bepu_device_types.h"
#include "bepu_type_table.h"

namespace bepucuda {

void launch_split_bodies(const void* raw, int body_count, const BodyBuffers& B, cudaStream_t s);
void launch_merge_bodies(void* raw, int body_count, const BodyBuffers& B, cudaStream_t s);
// Per device type batch: where its data lives in the uploaded reference-layout (AOSOA-W) image.
struct TransposeDesc {
    int32_t* src_refs;
    float* src_prestep;
    float* src_impulses;
    const int32_t* map;   // destination slot -> source constraint index (fallback levels), or nullptr for identity
    int32_t src_count;    // TypeBatch.ConstraintCount of the source
    int32_t bodies, prestep_rows, impulse_rows;
    int32_t src_bundle_base;  // index of the source type batch's first host-width bundle in the per-bundle flag array
    int32_t flags;            // kTransposePrestep / kTransposeImpulses: rows uploaded since the last transposition; kDescRedistribute
    int32_t contacts;         // per manifold; 0 for joints
    const int32_t* features_old;  // contact feature ids the resident impulses belong to / the frame's new ids ([constraint][contact]); null = none
    const int32_t* features_new;
};
// what: the rows to transpose. kTransposePending restricts them, per type batch, to those its descriptor marks as uploaded; the other type batches
// keep their device rows (accumulated impulses left by the last solve, depths the incremental update moved).
enum { kTransposeRefs = 1, kTransposePrestep = 2, kTransposeImpulses = 4, kTransposePending = 8 };
constexpr int32_t kDescRedistribute = 16;
void launch_transpose_in_all(const DeviceTypeBatch* tbs, const TransposeDesc* descs, const WorkItem* work, int work_count, int W, int what, cudaStream_t s);
void launch_transpose_out_all(const DeviceTypeBatch* tbs, const TransposeDesc* descs, const WorkItem* work, int work_count, int W, int what, cudaStream_t s);
// Lane `slot % 32` of bundle `slot / 32` of device type batch `type_batch`.
struct DeviceSlot {
    int32_t type_batch, slot;
};
// One location of bepucuda_read_constraints, resolved on the host. A constraint of a synchronized type batch is its device slot (identity slots); one
// of a fallback type batch is found on the device through the planner's inverse map: at = {-1, entry}, and the entry is {-1, -1} for a hole.
struct ReadRequest {
    int32_t type_id;
    DeviceSlot at;
};
// bepucuda_read_constraints: the 64-word record of every request (include/bepucuda.h), read from the AOSOA-32 rows, into records[count][64].
void launch_read_constraints(const DeviceTypeBatch* tbs, const TransposeDesc* descs, const DeviceSlot* inverse, const ReadRequest* requests, int count, int32_t* records,
                             cudaStream_t s);
// Words of the 64-word record of bepucuda_read_constraints / bepucuda_write_constraints (include/bepucuda.h): 0 type id, 1 live, 2-5 body references,
// 6-17 accumulated impulses, 18-52 prestep, 53-63 zero.
constexpr int kRecordRefs = 2, kRecordImpulses = 6, kRecordPrestep = 18, kRecordEnd = 53;
constexpr int kRecordPrestepWords = kRecordEnd - kRecordPrestep;
static_assert(kRecordImpulses - kRecordRefs >= max_over_types([](const TypeRow& r) { return r.bodies; }), "record: body references of every type");
static_assert(kRecordPrestep - kRecordImpulses >= max_over_types([](const TypeRow& r) { return r.impulse_rows; }), "record: impulse rows of every type");
static_assert(kRecordPrestepWords >= max_over_types([](const TypeRow& r) { return r.prestep_rows; }), "record: prestep rows of every type");
// One queued write of bepucuda_write_constraints: the constraint at `at` takes the prestep rows rows[row0 .. row0 + its type's prestep_rows).
struct PrestepWrite {
    DeviceSlot at;
    int32_t row0;
};
// bepucuda_write_constraints: the prestep rows of every write into the AOSOA-32 rows of its slot (impulses and body references untouched).
void launch_write_constraints(const DeviceTypeBatch* tbs, const TransposeDesc* descs, const PrestepWrite* writes, const float* rows, int count, cudaStream_t s);
void launch_fill_i32(int32_t* p, size_t n, int32_t v, cudaStream_t s);
// RedistributeImpulses (NarrowPhaseConstraintUpdate.cs:L81-135) for every device type batch whose descriptor has kDescRedistribute, on the AOSOA-32 impulses.
void launch_redistribute_impulses(const DeviceTypeBatch* tbs, const TransposeDesc* descs, const WorkItem* work, int work_count, cudaStream_t s);
// Motion half (floats 0-15) of 128-B BodyDynamics records <-> pose / velocity records. `raw` may be mapped host memory.
void launch_scatter_body_motion(const void* raw, int body_count, const BodyBuffers& B, cudaStream_t s);
void launch_gather_body_motion(void* raw, int body_count, const BodyBuffers& B, cudaStream_t s);
// One chunk (<= 64 KiB, sizes multiple of 4 bytes) of a batched host<->device copy through mapped pinned memory.
struct CopyChunk {
    void* dst;
    const void* src;
    size_t bytes;
};
void launch_batched_copy(const CopyChunk* chunks, int chunk_count, cudaStream_t s);
void launch_ownership_pass1(const DeviceTypeBatch* tbs, const WorkItem* work, int work_count, int sync_batch_count, int body_count,
                            int32_t* first_batch, int32_t* sync_refcount, unsigned long long* sync_mask, int32_t* error_flag, cudaStream_t s);
// Peer sharding, between the ownership passes: first_batch[i] = global_first_batch[i] (host batch indices, lowest over every rank) unless that is
// at or above fallback_threshold, where the device batch of pass 1 (a fallback level of the fallback rank) stays.
void launch_merge_first_batch(int32_t* first_batch, const int32_t* global_first_batch, int body_count, int fallback_threshold, cudaStream_t s);
void launch_ownership_rest(const DeviceTypeBatch* tbs, const WorkItem* work, int work_count, int body_count, const int32_t* first_batch,
                           const int32_t* sync_refcount, const unsigned long long* sync_mask, uint8_t* constrained, const int32_t* kinematics, int kinematic_count,
                           int32_t* error_flag, const TransposeDesc* descs, int W, int32_t* source_bundle_flags, cudaStream_t s);
// Peer sharding, rank barrier: one CTA signals every peer and waits for every peer's signal of the same exchange point (flag barrier in peer
// memory). Sets *error_flag to 5 when a peer does not arrive before the timeout.
void launch_shard_barrier(const ShardPeers& peers, const FrameParams* fp, uint32_t exchange_index, int32_t* error_flag, cudaStream_t s);

// Peer sharding: peer_masks[i] = ranks other than `rank` that reference the dynamic body of device reference refs[i] (0 for empty and
// kinematic slots); body_masks[b] has bit r set when rank r references body b.
void launch_fill_peer_masks(const int32_t* refs, uint32_t* peer_masks, size_t count, const uint8_t* body_masks, int rank, cudaStream_t s);
// flags[i] = 1 when any lane of work item i has a non-empty destination mask (a "boundary" bundle, see ShardStage).
void launch_boundary_flags(const DeviceTypeBatch* tbs, const WorkItem* work, int work_count, long long peer_delta, uint8_t* flags, cudaStream_t s);

// Reference rows next to the work list: rows[i][0..1][lane] = the first two body-reference rows of work record i (64 words per record), so that a
// solver warp fetches its work record and its body references with independent loads (one DRAM round trip instead of two).
void launch_pack_ref_rows(const WorkRecord* records, int count, int32_t* rows, cudaStream_t s);

// Numerics flavours (bepu_solver_kernels.cu, compiled twice).
// Peer-sharded stage (bepucuda_shard_*): every written body record also goes to the ranks named by the per-(lane, slot) destination masks at
// refs + peer_delta (launch_fill_peer_masks).
struct ShardLaunch {
    ShardPeers peers;
    long long peer_delta;
    ShardStage stage;
};
struct SolverLaunchers {
    // Launches one constraint stage (kStageWarmStartFirst / kStageWarmStart / kStageSolve / kStageIncremental) over `work_count` bundles, in the
    // instantiation `kernel` (StageKernel) with the launch flags that resolve_stage_launch (bepu_topology.h) chose for it.
    // ref_rows: the packed reference rows of records[0 .. work_count) (launch_pack_ref_rows).
    // shard: nullptr on a single GPU; a WarmStartFirst / WarmStart / Solve stage of a peer-sharded solve otherwise.
    void (*constraint_stage)(int stage, int kernel, const WorkRecord* records, const int32_t* ref_rows, int work_count, const BodyBuffers& B, const FrameParams* fp,
                             int launch_flags, const ShardLaunch* shard, cudaStream_t s);
    // launch_flags: kLaunchIntegratorExtensions or 0
    void (*kinematic_stage)(int stage, const int32_t* kinematics, int count, const BodyBuffers& B, const FrameParams* fp, int launch_flags, cudaStream_t s);
    void (*final_pose)(const BodyBuffers& B, const FrameParams* fp, int launch_flags, cudaStream_t s);
};
const SolverLaunchers* get_launchers_bepu_fast();
const SolverLaunchers* get_launchers_bepu_strict();

}  // namespace bepucuda
