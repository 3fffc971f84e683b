// Launchers of the layout / topology kernels (bepu_layout_kernels.cu).
#pragma once
#include "bepu_device_types.h"

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
    int32_t flags;            // kDescResidentImpulses: the accumulated impulses live on the device (bepucuda_update_contacts), transpose_in skips them
    const int32_t* features_old;  // contact feature ids the resident impulses belong to / the frame's new ids ([constraint][contact]); null = none
    const int32_t* features_new;
};
constexpr int32_t kDescResidentImpulses = 1, kDescRedistribute = 2;
enum { kTransposeRefs = 1, kTransposePrestep = 2, kTransposeImpulses = 4 };
void launch_transpose_in_all(const DeviceTypeBatch* tbs, const TransposeDesc* descs, const WorkItem* work, int work_count, int W, int what, cudaStream_t s);
void launch_transpose_out_all(const DeviceTypeBatch* tbs, const TransposeDesc* descs, const WorkItem* work, int work_count, int W, int what, cudaStream_t s);
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
void launch_ownership_pass1(const DeviceTypeBatch* tbs, const WorkItem* work, int work_count, const int32_t* bodies_per_type, int sync_batch_count, int body_count,
                            int32_t* first_batch, int32_t* sync_refcount, unsigned long long* sync_mask, int32_t* error_flag, cudaStream_t s);
void launch_ownership_rest(const DeviceTypeBatch* tbs, const WorkItem* work, int work_count, const int32_t* bodies_per_type, int body_count, const int32_t* first_batch,
                           const int32_t* sync_refcount, const unsigned long long* sync_mask, uint8_t* constrained, const int32_t* kinematics, int kinematic_count,
                           int32_t* error_flag, const TransposeDesc* descs, int W, int32_t* source_bundle_flags, cudaStream_t s);
// Peer sharding, rank barrier: one CTA signals every peer and waits for every peer's signal of the same exchange point (flag barrier in peer
// memory). Sets *error_flag to 5 when a peer does not arrive before the timeout.
void launch_shard_barrier(const ShardPeers& peers, const FrameParams* fp, uint32_t exchange_index, int32_t* error_flag, cudaStream_t s);

// Peer sharding: peer_masks[i] = ranks other than `rank` that reference the dynamic body of device reference refs[i] (0 for empty and
// kinematic slots); body_masks[b] has bit r set when rank r references body b.
void launch_fill_peer_masks(const int32_t* refs, uint32_t* peer_masks, size_t count, const uint8_t* body_masks, int rank, cudaStream_t s);
// flags[i] = 1 when any lane of work record i has a non-empty destination mask (a "boundary" bundle, see ShardStage).
void launch_boundary_flags(const WorkRecord* records, int count, const int32_t* bodies_per_type, long long peer_delta, uint8_t* flags, cudaStream_t s);

// Reference rows next to the work list: rows[i][0..1][lane] = the first two body-reference rows of work record i (64 words per record), so that a
// solver warp fetches its work record and its body references with independent loads (one DRAM round trip instead of two).
void launch_pack_ref_rows(const WorkRecord* records, int count, int32_t* rows, cudaStream_t s);

// Numerics flavours (bepu_solver_kernels.cu, compiled twice).
constexpr int kLaunchPdl = 1, kLaunchPrefetchRows = 2, kLaunchIntegratorExtensions = 4, kLaunchContactsOnly = 8, kLaunchPrefetchBodies = 16, kLaunchBodiesIntegrated = 32;
// Peer-sharded stage (bepucuda_shard_*): every written body record also goes to the ranks named by the per-(lane, slot) destination masks at
// refs + peer_delta (launch_fill_peer_masks).
struct ShardLaunch {
    ShardPeers peers;
    long long peer_delta;
    ShardStage stage;
};
struct SolverLaunchers {
    // Launches one constraint stage (kStageWarmStartFirst / kStageWarmStart / kStageSolve / kStageIncremental) over `work_count` bundles.
    // launch_flags: kLaunchPdl = launch with programmatic stream serialization (the kernel overlaps its prologue with the previous stage);
    // kLaunchPrefetchRows = the kernel launched just before this one writes neither this batch's prestep nor its impulses, so the prologue may fetch them.
    // kLaunchIntegratorExtensions = per-body accelerations or point gravity are set: the WarmStart stages run the instantiation that applies them.
    // kLaunchContactsOnly = every bundle of the batch is a contact: the WarmStart / Solve stage runs the contact-only instantiation (not sharded).
    // kLaunchPrefetchBodies = the kernel launched just before this one is a stage of this solve and not the WarmStart of this batch, so the prologue
    // may load the body records it does not write (constraint_stage_body).
    // kLaunchBodiesIntegrated (substeps > 0, FrameParams::angular_mode 0): the incremental contact update also integrates the pose and rotates the
    // world inertia of every body a constraint lane integrates, one thread per body, and the WarmStart stages leave that part to it.
    // ref_rows: the packed reference rows of records[0 .. work_count) (launch_pack_ref_rows).
    // shard: nullptr on a single GPU; a WarmStartFirst / WarmStart / Solve stage of a peer-sharded solve otherwise.
    void (*constraint_stage)(int stage, const WorkRecord* records, const int32_t* ref_rows, int work_count, const BodyBuffers& B, const FrameParams* fp, int launch_flags,
                             const ShardLaunch* shard, cudaStream_t s);
    // launch_flags: kLaunchIntegratorExtensions or 0 (the other bits do not apply to the per-body passes)
    void (*kinematic_stage)(int stage, const int32_t* kinematics, int count, const BodyBuffers& B, const FrameParams* fp, int launch_flags, cudaStream_t s);
    void (*final_pose)(const BodyBuffers& B, const FrameParams* fp, int launch_flags, cudaStream_t s);
};
const SolverLaunchers* get_launchers_bepu_fast();
const SolverLaunchers* get_launchers_bepu_strict();

}  // namespace bepucuda
