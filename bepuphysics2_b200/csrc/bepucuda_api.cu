// libbepucuda host side: context, device memory, uploads/downloads, device tables of the topology plan (bepu_topology.h), stage launches, CUDA graph.
// C ABI declared in include/bepucuda.h. No CPU fallback lives here: without a usable CUDA device bepucuda_create fails.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/bepucuda.h"
#include "bepu_layout_kernels.h"
#include "bepu_coloring.h"
#include "bepu_islands.h"
#include "bepu_bounds.h"
#include "bepu_cuda_handles.h"
#include "bepu_topology.h"

using namespace bepucuda;

namespace bepucuda {

// Raw rows of a source type batch on the device, in the reference's AOSOA-W layout: body references, prestep and impulses, and for the
// device-side contact update (bepucuda_update_contacts) the feature ids of the resident impulses (old) and of the frame being uploaded (new).
struct RawRows {
    int32_t* refs = nullptr;
    float* prestep = nullptr;
    float* impulses = nullptr;
    int32_t* features_old = nullptr;
    int32_t* features_new = nullptr;
};
enum RowKind { kRowRefs, kRowPrestep, kRowImpulses, kRowFeatures };
// Bytes of one kind of row for `count` constraints of type t: whole bundles of W for body references, prestep and impulses; exactly `count`
// constraints for feature ids, which are [constraint][contact] and not bundled.
static size_t row_bytes(const TypeInfo* t, RowKind k, int count, int W) {
    const int per_constraint[4] = {t->bodies, t->prestep_rows, t->impulse_rows, t->contacts};
    const size_t lanes = k == kRowFeatures ? (size_t)count : ((size_t)count + W - 1) / W * W;
    return lanes * per_constraint[k] * 4;
}

struct SourceTypeBatch {
    ChangeSource host;     // the host's type batch: batch, type batch, type id, count, and body references retained only for fallback batches (levelisation)
    int capacity = 0;      // constraints the rows hold (whole bundles); bepucuda_add_constraints grows them
    RawRows rows;          // feature ids once bepucuda_set_contact_features set them or an add brought them
    float* host_impulses = nullptr;  // the host's AccumulatedImpulses (bepucuda_download_impulses); null after an add until the host passes it again
    // rows uploaded since the last transposition (kTransposePrestep / kTransposeImpulses): refresh_device_rows transposes only these, so the rows
    // of every other type batch, the accumulated impulses in particular, stay as the last solve left them on the device
    int32_t pending = 0;
    bool redistribute = false;
    const TypeInfo* type() const { return get_type_info(host.type_id); }
    size_t bytes(RowKind k, int W) const { return row_bytes(type(), k, host.count, W); }
    // the rows as the lane copies of bepucuda_add_constraints / bepucuda_remove_constraints and the reference remap of bepucuda_remove_bodies see them
    SourceRows lane_rows() const {
        const TypeInfo* t = type();
        return {rows.refs, rows.prestep, rows.impulses, rows.features_old, t->bodies, t->prestep_rows, t->impulse_rows, t->contacts};
    }
    RefSpan ref_span(int W) const { return {rows.refs, (int64_t)(bytes(kRowRefs, W) / 4)}; }
};

// The per-body device arrays: the 128-B records that uploads and downloads pass through, and the arrays the kernels read through BodyBuffers.
struct BodyArrays {
    DeviceBuffer raw, pose, velocity, inertia_local, inertia_world, constrained, first_batch;
    // Room for n bodies, contents dropped; constrained flags reallocated here start cleared. first_batch is sized and filled by the plan.
    cudaError_t reserve(size_t n, cudaStream_t s) {
        cudaError_t e = raw.reserve(n * 128);
        for (DeviceBuffer* b : {&pose, &velocity, &inertia_local, &inertia_world})
            if (e == cudaSuccess) e = b->reserve(n * 32);
        const size_t old_constrained_capacity = constrained.capacity;
        if (e == cudaSuccess) e = constrained.reserve(n + 1);
        if (e == cudaSuccess && constrained.capacity != old_constrained_capacity) e = cudaMemsetAsync(constrained.ptr, 0, constrained.capacity, s);
        return e;
    }
    // Room for n bodies, the records of the first `keep` kept. A failure leaves the arrays grown so far grown, records and all.
    cudaError_t grow(size_t n, size_t keep, cudaStream_t s) {
        cudaError_t e = raw.grow(n * 128, keep * 128, s);
        for (DeviceBuffer* b : {&pose, &velocity, &inertia_local, &inertia_world})
            if (e == cudaSuccess) e = b->grow(n * 32, keep * 32, s);
        if (e == cudaSuccess) e = constrained.grow(n + 1, keep, s);
        if (e == cudaSuccess) e = first_batch.grow(n * 4, keep * 4, s);
        return e;
    }
    BodyBuffers view(int count) const {
        return {pose.as<float4>(), velocity.as<float4>(), inertia_local.as<float4>(), inertia_world.as<float4>(), constrained.as<uint8_t>(), first_batch.as<int32_t>(), count};
    }
};
inline bool operator==(const BodyBuffers& a, const BodyBuffers& b) {
    return a.pose == b.pose && a.velocity == b.velocity && a.inertia_local == b.inertia_local && a.inertia_world == b.inertia_world && a.constrained == b.constrained &&
           a.first_batch == b.first_batch && a.count == b.count;
}

// The stage sequence of the program captured as a graph (dropped when the program is replaced), and the body buffers and launch context its
// launches bake in besides the program: matches() says whether a frame can replay it.
struct StageGraph {
    Graph graph;
    GraphExec exec;  // destroyed before the graph it was instantiated from
    BodyBuffers bodies{};
    LaunchContext launch{};
    void reset() { exec.reset(); graph.reset(); }
    bool matches(const BodyBuffers& b, const LaunchContext& lc) const { return exec && bodies == b && same_launches(launch, lc); }
};

}  // namespace bepucuda

struct bepucuda_ctx {
    bepucuda_config cfg{};
    int device = 0;
    Stream stream;  // declared before every other handle, so that it is destroyed after them
    TimingWindow solve_window, upload_window, download_window;
    std::string error;
    const SolverLaunchers* launchers = nullptr;

    // solve description / integrator
    std::vector<int32_t> iterations{1};
    int fallback_threshold = 64;
    bepucuda_integrator_desc integ{};
    bool integ_set = false;
    // bepucuda_set_body_accelerations: device copy, the body count it was set for (-1: not set), and the pinned staging of the last upload
    DeviceBuffer accelerations;
    int accelerations_count = -1;
    StagedUpload accelerations_stage;
    // bepucuda_set_point_gravity
    bool point_gravity = false;
    float attractor_center[3] = {0.0f, 0.0f, 0.0f};
    float attractor_strength = 0.0f;

    // bodies
    int body_count = 0;
    bool bodies_uploaded = false;  // a bepucuda_upload_bodies has succeeded
    BodyArrays bodies;
    DeviceBuffer sync_refcount, sync_mask;
    BodyBuffers B{};  // bodies.view(body_count), set by refresh_body_buffers

    // constraints
    int W = 8;
    int batch_count = 0;
    bool constraints_open = false, constraints_ready = false, data_dirty = false;
    std::vector<SourceTypeBatch> sources;
    ChunkArena raw_arena, pinned_arena;
    DeviceBuffer record_table, ref_rows, source_bundle_flags, refs32, prestep32, impulses32, tb_table, tdesc_table, work_table, map_table, kinematics_dev, frame_params_dev, error_dev;
    TopologyPlan topo;                          // device batches and work list of the last successful end_constraints
    std::vector<TransposeDesc> tdescs;          // per planned type batch
    std::vector<WorkRecord> records;            // what the solver kernels read (parallel to topo.work)
    // peer sharding (bepucuda_shard_*): one constraint graph over several GPUs with NVLink peer stores from the stage kernels
    bool peer_mode = false;
    ShardPeers peers{};
    DeviceBuffer shard_flags, peer32, body_masks_dev, boundary_flags_dev;
    uint32_t shard_solve_index = 0;                                 // solves since the arrival targets were last published
    std::vector<int> boundary_count;                                // per device batch: bundles that touch a body another rank references
    std::vector<uint8_t> body_masks;                                // bepucuda_shard_set_body_masks: per body, the ranks that reference it
    std::vector<IpcMapping> opened_ipc;
    std::vector<int32_t> global_first_batch;
    DeviceBuffer global_first_batch_dev;
    std::vector<uint8_t> global_constrained;
    int32_t fallback_rank = -1;                                     // bepucuda_shard_set_fallback_rank: the rank that runs the fallback batch
    uint32_t exchange_counter = 0;                                  // exchange points executed so far (flag barrier sequence)
    std::vector<int32_t> kinematics;
    StageProgram program;
    PinnedBuffer frame_params_host;             // FrameParams
#ifdef BEPU_HAZARD
    int32_t hazard_canary = 0, hazard_delay_us = 0;  // BEPUCUDA_HAZARD at bepucuda_create (hazard build only, see hazard_launch_bits)
#endif

    StageGraph stage_graph;

    bepucuda_timings timings{};
    int64_t h2d_accum = 0;
    struct HostRange { char* host; size_t bytes; char* dev; };
    std::vector<HostRange> host_ranges;    // page-locked + device-mapped host memory registered through bepucuda_host_register
    std::vector<CopyChunk> pending_h2d;    // batched copies waiting for the next flush
    DeviceBuffer chunk_table;
    StagedUpload chunk_stage[4];           // pinned ring for chunk tables
    int chunk_stage_next = 0;
    Event user_events[16];
    DeviceBuffer body_shapes, body_activities, body_bounds;  // bepucuda_set_body_shapes / bepucuda_predict_bounding_boxes
    int shape_count = -1;
    ColoringScratch coloring;  // bepucuda_color_constraints
    IslandScratch islands;     // bepucuda_find_sleepable_islands
    DeviceBuffer inverse_table, read_requests, read_records;  // bepucuda_read_constraints: the plan's inverse slot map, one call's requests and records
    PrestepWriteQueue prestep_writes;  // bepucuda_write_constraints since the last solve, applied by refresh_device_rows
    DeviceBuffer write_table, write_rows;
    StagedUpload write_stage, write_rows_stage;
    DeviceBuffer body_writes;         // bepucuda_write_bodies: one call's staged motion halves (unregistered buffers) and body indices
    StagedUpload body_write_stage;
    std::vector<Event> profile_events;
    DeviceBuffer change_sources, change_copies, change_records, change_features;  // bepucuda_add_constraints / bepucuda_remove_constraints
    std::vector<std::pair<void*, size_t>> spare_rows;  // raw-arena blocks of grown and removed sources, taken again by later growth (until a describe)
    DeviceBuffer moved_to, removed_marks, ref_spans;  // bepucuda_remove_bodies
};

namespace {

int fail(bepucuda_ctx* c, int code, const std::string& msg) {
    if (c) c->error = msg;
    return code;
}
int cuda_fail(bepucuda_ctx* c, cudaError_t e, const char* what) {
    return fail(c, e == cudaErrorMemoryAllocation ? BEPUCUDA_ERR_OUT_OF_MEMORY : BEPUCUDA_ERR_CUDA, std::string(what) + ": " + cudaGetErrorString(e));
}
#define CK(call)                                                  \
    do {                                                          \
        cudaError_t _e = (call);                                  \
        if (_e != cudaSuccess) return cuda_fail(ctx, _e, #call);  \
    } while (0)
// Returns a status other than BEPUCUDA_OK to the caller.
#define TRY(expr)                                \
    do {                                         \
        const int _rc = (expr);                  \
        if (_rc != BEPUCUDA_OK) return _rc;      \
    } while (0)

// Device alias of a host pointer if [ptr, ptr + bytes) lies inside a registered (mapped) range, else nullptr.
char* map_host(bepucuda_ctx* ctx, const void* ptr, size_t bytes) {
    const char* p = (const char*)ptr;
    for (auto& r : ctx->host_ranges)
        if (p >= r.host && p + bytes <= r.host + r.bytes) return r.dev + (p - r.host);
    return nullptr;
}
void queue_chunks(std::vector<CopyChunk>& list, void* dst, const void* src, size_t bytes) {
    const size_t kChunk = (size_t)64 << 10;
    for (size_t off = 0; off < bytes; off += kChunk) list.push_back({(char*)dst + off, (const char*)src + off, std::min(kChunk, bytes - off)});
}
// Room for `bytes` in the pinned staging buffer of `st`, once the previous upload has left it.
int reserve_staging(bepucuda_ctx* ctx, StagedUpload& st, size_t bytes) {
    CK(st.done.create(cudaEventDisableTiming));
    CK(cudaEventSynchronize(st.done));
    CK(st.host.reserve(bytes));
    return BEPUCUDA_OK;
}
// H2D copy of the first `bytes` of the staging buffer of `st`.
int send_staging(bepucuda_ctx* ctx, StagedUpload& st, void* dst, size_t bytes) {
    CK(cudaMemcpyAsync(dst, st.host.ptr, bytes, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaEventRecord(st.done, ctx->stream));
    return BEPUCUDA_OK;
}
// H2D copy of `bytes` at `src` through the pinned staging buffer of `st`.
int upload_staged(bepucuda_ctx* ctx, StagedUpload& st, void* dst, const void* src, size_t bytes) {
    TRY(reserve_staging(ctx, st, bytes));
    std::memcpy(st.host.ptr, src, bytes);
    return send_staging(ctx, st, dst, bytes);
}

// Runs the queued chunks as one kernel. The chunk table travels through a ring of pinned staging buffers.
int flush_chunks(bepucuda_ctx* ctx, std::vector<CopyChunk>& list) {
    if (list.empty()) return BEPUCUDA_OK;
    const size_t bytes = list.size() * sizeof(CopyChunk);
    CK(ctx->chunk_table.reserve(bytes));
    StagedUpload& st = ctx->chunk_stage[ctx->chunk_stage_next];
    ctx->chunk_stage_next = (ctx->chunk_stage_next + 1) & 3;
    // The device-side table is reused by every flush: stream order keeps the previous batched copy ahead of this overwrite.
    TRY(upload_staged(ctx, st, ctx->chunk_table.ptr, list.data(), bytes));
    launch_batched_copy(ctx->chunk_table.as<CopyChunk>(), (int)list.size(), ctx->stream);
    CK(cudaGetLastError());
    list.clear();
    return BEPUCUDA_OK;
}

// The H2D copy of constraint rows and contact feature ids. A registered (mapped) host buffer is read by the batched copy kernel at the next flush.
// While the constraints are being described, small buffers are packed through the pinned staging arena, so that hundreds of tiny type batches do
// not each pay a pageable-memory DMA setup; begin_constraints recycles that arena, so after end_constraints every other copy goes directly.
int copy_in(bepucuda_ctx* ctx, void* dst, const void* src, size_t bytes) {
    if (bytes == 0) return BEPUCUDA_OK;
    if (char* alias = map_host(ctx, src, bytes)) {
        queue_chunks(ctx->pending_h2d, dst, alias, bytes);
    } else if (ctx->constraints_open && bytes < ((size_t)256 << 10)) {
        cudaError_t e = cudaSuccess;
        void* stage = ctx->pinned_arena.alloc(bytes, &e);
        if (!stage) return cuda_fail(ctx, e, "pinned staging");
        std::memcpy(stage, src, bytes);
        CK(cudaMemcpyAsync(dst, stage, bytes, cudaMemcpyHostToDevice, ctx->stream));
    } else {
        CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, ctx->stream));
    }
    ctx->h2d_accum += (int64_t)bytes;
    return BEPUCUDA_OK;
}

// Reserves the device table `name` for the elements of `v` plus `slack` bytes, and queues their copy if there are any.
template <class T> int upload_table(bepucuda_ctx* ctx, const char* name, DeviceBuffer& table, const std::vector<T>& v, size_t slack) {
    cudaError_t e = table.reserve(v.size() * sizeof(T) + slack);
    if (e == cudaSuccess && !v.empty()) e = cudaMemcpyAsync(table.ptr, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice, ctx->stream);
    return e == cudaSuccess ? BEPUCUDA_OK : cuda_fail(ctx, e, name);
}

SourceTypeBatch* find_source(bepucuda_ctx* ctx, int32_t batch_index, int32_t type_batch_index) {
    for (auto& s : ctx->sources)
        if (s.host.batch_index == batch_index && s.host.type_batch_index == type_batch_index) return &s;
    return nullptr;
}

// A block of `bytes` for source rows: a spare block of the arena between `bytes` and twice that, or a new one. Spare blocks are what grown and
// removed sources left, so a run that stays on the change calls reuses them instead of growing the arena with every re-created type batch.
void* take_rows(bepucuda_ctx* ctx, size_t bytes, cudaError_t* e) {
    size_t best = ctx->spare_rows.size();
    for (size_t i = 0; i < ctx->spare_rows.size(); ++i) {
        const size_t have = ctx->spare_rows[i].second;
        if (have >= bytes && have <= 2 * bytes && (best == ctx->spare_rows.size() || have < ctx->spare_rows[best].second)) best = i;
    }
    if (best == ctx->spare_rows.size()) return ctx->raw_arena.alloc(bytes, e);
    void* p = ctx->spare_rows[best].first;
    ctx->spare_rows[best] = ctx->spare_rows.back();
    ctx->spare_rows.pop_back();
    return p;
}
void give_rows(bepucuda_ctx* ctx, void* p, size_t bytes) {
    if (p && bytes) ctx->spare_rows.push_back({p, bytes});
}
void give_source_rows(bepucuda_ctx* ctx, const TypeInfo* t, int capacity, const RawRows& r) {
    auto give = [&](void* p, RowKind k) { give_rows(ctx, p, row_bytes(t, k, capacity, ctx->W)); };
    give(r.refs, kRowRefs);
    give(r.prestep, kRowPrestep);
    give(r.impulses, kRowImpulses);
    give(r.features_old, kRowFeatures);
    give(r.features_new, kRowFeatures);
}
// The feature-id rows of `capacity` constraints into *r; on failure the block taken goes back and *r keeps none.
cudaError_t take_feature_rows(bepucuda_ctx* ctx, const TypeInfo* t, int capacity, RawRows* r) {
    cudaError_t e = cudaSuccess;
    const size_t bytes = row_bytes(t, kRowFeatures, capacity, ctx->W);
    r->features_old = (int32_t*)take_rows(ctx, bytes, &e);
    if (r->features_old) r->features_new = (int32_t*)take_rows(ctx, bytes, &e);
    if (r->features_new) return cudaSuccess;
    give_rows(ctx, r->features_old, bytes);
    r->features_old = nullptr;
    return e == cudaSuccess ? cudaErrorMemoryAllocation : e;
}
// The rows of `capacity` constraints, with feature ids when `features` and t is a contact type; on failure every block taken goes back and the
// error is returned. In a describe there are no spare blocks, so the rows are new arena blocks, taken in row order.
cudaError_t take_source_rows(bepucuda_ctx* ctx, const TypeInfo* t, int capacity, bool features, RawRows* out) {
    cudaError_t e = cudaSuccess;
    auto take = [&](RowKind k) { return take_rows(ctx, row_bytes(t, k, capacity, ctx->W), &e); };
    RawRows r;
    r.refs = (int32_t*)take(kRowRefs);
    if (r.refs) r.prestep = (float*)take(kRowPrestep);
    if (r.prestep) r.impulses = (float*)take(kRowImpulses);
    if (!r.impulses) e = e == cudaSuccess ? cudaErrorMemoryAllocation : e;
    else if (features && t->contacts > 0) e = take_feature_rows(ctx, t, capacity, &r);
    if (e != cudaSuccess) {
        give_source_rows(ctx, t, capacity, r);
        return e;
    }
    *out = r;
    return cudaSuccess;
}

void refresh_body_buffers(bepucuda_ctx* ctx) { ctx->B = ctx->bodies.view(ctx->body_count); }

// The device's AOSOA-32 rows of `what` (kTransposePrestep / kTransposeImpulses) back into the sources' raw rows.
int transpose_out(bepucuda_ctx* ctx, int what) {
    launch_transpose_out_all(ctx->tb_table.as<DeviceTypeBatch>(), ctx->tdesc_table.as<TransposeDesc>(), ctx->work_table.as<WorkItem>(), ctx->topo.all_work_count, ctx->W,
                             what, ctx->stream);
    CK(cudaGetLastError());
    return BEPUCUDA_OK;
}

// The optional velocity terms that are set (bepucuda_set_body_accelerations / bepucuda_set_point_gravity): kIntegrateAccelerations |
// kIntegratePointGravity. Whether any is set is an input of resolve_stage_launch; their values are frame parameters.
uint32_t integrate_extensions(const bepucuda_ctx* ctx) {
    return (ctx->accelerations_count >= 0 ? kIntegrateAccelerations : 0u) | (ctx->point_gravity ? kIntegratePointGravity : 0u);
}
#ifdef BEPU_HAZARD
// The hazard fields of every launch of this context (bepu_device_types.h): its canary, and its delay, which grows with the rank in peer mode so that
// the ranks drift apart by one delay per stage wherever boundary warps do not wait for their peers.
int32_t hazard_launch_bits(const bepucuda_ctx* ctx) {
    const int delay_units = std::min(255, ctx->hazard_delay_us * (1 + (ctx->peer_mode ? ctx->peers.rank : 0)) / 10);
    return (ctx->hazard_canary << kLaunchHazardCanaryShift) | (delay_units << kLaunchHazardDelayShift);
}
// BEPUCUDA_HAZARD="delay_us=<n>,canary=<k>" (either part optional)
void read_hazard_environment(bepucuda_ctx* ctx) {
    const char* env = std::getenv("BEPUCUDA_HAZARD");
    if (!env) return;
    const char* d = std::strstr(env, "delay_us=");
    const char* c = std::strstr(env, "canary=");
    if (d) ctx->hazard_delay_us = std::max(0, std::atoi(d + 9));
    if (c) ctx->hazard_canary = std::atoi(c + 7) & 7;
}
#endif
LaunchContext launch_context(const bepucuda_ctx* ctx, bool profile) { return {integrate_extensions(ctx) != 0, ctx->integ.angular_integration_mode, profile}; }

// Profiling sink of issue_stage_sequence: the launch of program op i sets launched[i] and is bracketed by events[2i] and events[2i + 1].
struct StageEvents {
    const std::vector<Event>& events;
    std::vector<int>& launched;
};

// Issues the whole stage sequence of one frame as individual launches on `s` (used directly in STREAM mode and under capture in GRAPH mode), each
// as resolve_stage_launch says. With `profile`, each event pair times one kernel alone.
void issue_stage_sequence(bepucuda_ctx* ctx, cudaStream_t s, int64_t* launches, const StageEvents* profile = nullptr) {
    const WorkRecord* records = ctx->record_table.as<WorkRecord>();
    const int32_t* ref_rows = ctx->ref_rows.as<int32_t>();
    const FrameParams* fp = ctx->frame_params_dev.as<FrameParams>();
    const int32_t* kin = ctx->kinematics_dev.as<int32_t>();
    ShardLaunch shard{ctx->peers, (long long)(ctx->peer32.as<int32_t>() - ctx->refs32.as<int32_t>()), {0, ctx->error_dev.as<int32_t>()}};
    int64_t n = 0;
    const LaunchContext lc = launch_context(ctx, profile != nullptr);
#ifdef BEPU_HAZARD
    const int32_t hazard = hazard_launch_bits(ctx);
#else
    constexpr int32_t hazard = 0;
#endif
    for (size_t i = 0; i < ctx->program.ops.size(); ++i) {
        const StageOp& op = ctx->program.ops[i];
        const bool barrier = op.exchange == kRankBarrier;
        // A sharded stage without constraints on this rank launches nothing but still counts as an exchange point: nothing arrives from this
        // rank there, and its arrival targets say so.
        if (barrier || (op.stage == kStageFinalPose ? ctx->B.count > 0 : op.work_count > 0)) {
            const StageLaunch launch = resolve_stage_launch(op, lc);
            if (profile) cudaEventRecord(profile->events[2 * i], s);
            if (barrier) {
                // all ranks meet: before the first stage of a solve; around the incremental contact update, which reads the velocities of shared
                // bodies; and before the final pose pass
                launch_shard_barrier(ctx->peers, fp, op.exchange_index | (uint32_t)hazard, ctx->error_dev.as<int32_t>(), s);
            } else if (op.stage <= kStageIncremental) {
                // a sharded stage stores the records it writes for shared bodies into the ranks that reference them, and its boundary bundles wait
                // for and announce arrivals themselves (ShardStage)
                shard.stage.exchange_index = op.exchange_index;
                ctx->launchers->constraint_stage(op.stage, launch.kernel, records + op.work_begin, ref_rows + (size_t)op.work_begin * 64, op.work_count, ctx->B, fp,
                                                 launch.flags | hazard, op.exchange == kNoExchange ? nullptr : &shard, s);
            } else if (op.stage <= kStageKinematic) {
                ctx->launchers->kinematic_stage(op.stage, kin, op.work_count, ctx->B, fp, launch.flags, s);
            } else {
                ctx->launchers->final_pose(ctx->B, fp, launch.flags, s);
            }
            if (profile) {
                cudaEventRecord(profile->events[2 * i + 1], s);
                profile->launched[i] = 1;
            }
            ++n;
        }
    }
    if (launches) *launches = n;
}

// Replaces the stage program and drops the graph captured from the old one. The constraints are ready for a solve only once this succeeds.
int upload_program(bepucuda_ctx* ctx) {
    // Before any early return: a failure below must not leave a graph of the old program, whose launches read tables end_constraints may have
    // reallocated, nor a description that solve takes as ready.
    ctx->constraints_ready = false;
    // work issued under the previous program completes before that program and its graph are replaced
    CK(cudaStreamSynchronize(ctx->stream));
    ctx->stage_graph.reset();
    ctx->program = build_stage_program(ctx->topo, ctx->iterations, (int)ctx->kinematics.size(), ctx->integ.integrate_velocity_for_kinematics != 0, ctx->peer_mode,
                                       ctx->body_count);
    if (ctx->peer_mode) {
        // publish, to every peer, how many boundary bundles of this rank arrive through each exchange point of one solve (ShardStage), and restart
        // the arrival counters other ranks increment here. Every rank does this for the same program, between solves.
        std::vector<unsigned long long> targets;
        std::string error;
        const int rc = exchange_targets(ctx->program, ctx->boundary_count, &targets, &error);
        if (rc != BEPUCUDA_OK) return fail(ctx, rc, error);
        for (int q = 0; q < ctx->peers.rank_count; ++q)
            if (q != ctx->peers.rank)
                CK(cudaMemcpy(ctx->peers.flags[q] + kShardTargetSlot + (size_t)ctx->peers.rank * kShardMaxExchanges, targets.data(), targets.size() * 8, cudaMemcpyDefault));
        CK(cudaMemset((unsigned long long*)ctx->shard_flags.ptr + kShardCounterSlot, 0, kMaxShardRanks * 8));
        ctx->shard_solve_index = 0;
    }
    ctx->timings.stage_count = ctx->program.stage_count;
    ctx->constraints_ready = true;
    return BEPUCUDA_OK;
}

// Callbacks.PrepareForIntegration(dt): Demos/DemoCallbacks.cs:L79-86, and for point gravity gravityDt = dt * Gravity (PlanetDemo.cs:L36-40).
struct IntegrationTerms {
    float gravity_dt[3], linear_damping_dt, angular_damping_dt, attractor_dt;
};
IntegrationTerms prepare_for_integration(const bepucuda_ctx* ctx, float dt) {
    auto clamp01 = [](float v) { return v < 0.f ? 0.f : (v > 1.f ? 1.f : v); };
    IntegrationTerms t;
    for (int i = 0; i < 3; ++i) t.gravity_dt[i] = ctx->integ.gravity[i] * dt;
    t.linear_damping_dt = powf(clamp01(1 - ctx->integ.linear_damping), dt);
    t.angular_damping_dt = powf(clamp01(1 - ctx->integ.angular_damping), dt);
    t.attractor_dt = dt * ctx->attractor_strength;
    return t;
}

void compute_frame_params(bepucuda_ctx* ctx, float dt, FrameParams* fp) {
    const int substeps = (int)ctx->iterations.size();
    const float substepDt = dt / substeps;  // Solver_Solve.cs:L1417
    const bepucuda_integrator_desc& d = ctx->integ;
    const IntegrationTerms sub = prepare_for_integration(ctx, substepDt);
    fp->dt = substepDt;
    fp->inverse_dt = 1.0f / substepDt;
    fp->linear_damping_dt = sub.linear_damping_dt;
    fp->angular_damping_dt = sub.angular_damping_dt;
    for (int i = 0; i < 3; ++i) fp->gravity_dt[i] = sub.gravity_dt[i];
    fp->attractor_dt = sub.attractor_dt;
    // IntegrateAfterSubstepping: PoseIntegrator.cs:L707-712
    const float finalDt = d.allow_substeps_for_unconstrained ? substepDt : dt;
    const IntegrationTerms fin = prepare_for_integration(ctx, finalDt);
    fp->final_dt = finalDt;
    fp->final_linear_damping_dt = fin.linear_damping_dt;
    fp->final_angular_damping_dt = fin.angular_damping_dt;
    for (int i = 0; i < 3; ++i) fp->final_gravity_dt[i] = fin.gravity_dt[i];
    fp->final_attractor_dt = fin.attractor_dt;
    fp->final_steps = d.allow_substeps_for_unconstrained ? substeps : 1;
    fp->angular_mode = d.angular_integration_mode;
    fp->integrate_velocity_for_kinematics = d.integrate_velocity_for_kinematics;
    fp->integrate_extensions = integrate_extensions(ctx);
    const unsigned long long accelerations = (fp->integrate_extensions & kIntegrateAccelerations) ? (unsigned long long)ctx->accelerations.ptr : 0ull;
    fp->accelerations[0] = (uint32_t)accelerations;
    fp->accelerations[1] = (uint32_t)(accelerations >> 32);
    for (int i = 0; i < 3; ++i) fp->attractor_center[i] = ctx->attractor_center[i];
}

// The error message of a location that resolve_location rejects (bepucuda_read_constraints / bepucuda_write_constraints).
std::string no_constraint_at(int32_t i, const bepucuda_constraint_location& l) {
    return "location " + std::to_string(i) + " (set " + std::to_string(l.set_index) + ", batch " + std::to_string(l.batch_index) + ", type " + std::to_string(l.type_id) +
           ", index " + std::to_string(l.index_in_type_batch) + ") names no constraint of the active set";
}

// The prologue of bepucuda_read_constraints / bepucuda_write_constraints (`name`, `write`): the state and argument checks, then every location
// resolved and, for a write, checked against its record. All of it runs before any device work or queueing, so a failing call changes nothing.
int resolve_locations(bepucuda_ctx* ctx, const std::string& name, int32_t count, const bepucuda_constraint_location* locations, const int32_t* records, bool write,
                      std::vector<ResolvedLocation>* resolved) {
    if (ctx->peer_mode) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, name + " in peer mode: a rank holds its constraints compacted, so host locations do not address them");
    if (!ctx->constraints_ready) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, name + " before end_constraints");
    if (count < 0 || (count > 0 && (!locations || !records))) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, name + ": bad arguments");
    resolved->resize((size_t)count);
    for (int32_t i = 0; i < count; ++i) {
        const bepucuda_constraint_location& l = locations[i];
        ResolvedLocation& r = (*resolved)[(size_t)i];
        if (resolve_location(ctx->topo, l, &r) != BEPUCUDA_OK) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, name + ": " + no_constraint_at(i, l));
        if (write && r.at.type_batch < 0) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, name + ": " + no_constraint_at(i, l) + " (a hole of the fallback batch)");
        if (write && records[(size_t)i * 64] != l.type_id)
            return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, name + ": record " + std::to_string(i) + " has type id " + std::to_string(records[(size_t)i * 64]) +
                                                                ", its location type id " + std::to_string(l.type_id));
    }
    return BEPUCUDA_OK;
}

// Accelerations set for another body count than the current one index the wrong bodies: solve, profile_stages and predict_bounding_boxes refuse
// to run before any device work.
int check_accelerations(bepucuda_ctx* ctx, const char* what) {
    if (ctx->accelerations_count >= 0 && ctx->accelerations_count != ctx->body_count)
        return fail(ctx, BEPUCUDA_ERR_BAD_STATE, std::string(what) + ": the body count changed after bepucuda_set_body_accelerations; set them again (or clear them with NULL)");
    return BEPUCUDA_OK;
}

// Brings the device AOSOA-32 rows up to date with what the host queued since the last solve (bepucuda_update_type_batch / bepucuda_update_contacts /
// bepucuda_write_constraints): flushes the batched copies, re-uploads the transposition descriptors when their pending rows, redistribution flags
// or feature ids changed, transposes the pending rows only, redistributes the resident penetration impulses of updated contact type batches from
// the old to the new feature ids, and then writes the queued prestep rows of single constraints, so that they win over a whole-type-batch upload
// of the same frame. A frame that refreshes every type batch in full (bepuhost_cuda_refresh) leaves the descriptors as end_constraints uploaded them.
int refresh_device_rows(bepucuda_ctx* ctx) {
    if (!ctx->data_dirty) return BEPUCUDA_OK;
    TRY(flush_chunks(ctx, ctx->pending_h2d));
    bool any_pending = false, any_redistribute = false, descs_changed = false;
    for (size_t tb = 0; tb < ctx->topo.tbs.size(); ++tb) {
        const SourceTypeBatch& s = ctx->sources[(size_t)ctx->topo.tbs[tb].source];
        TransposeDesc& d = ctx->tdescs[tb];
        const int32_t flags = s.pending | (s.redistribute ? kDescRedistribute : 0);
        if (d.flags != flags || d.features_old != s.rows.features_old || d.features_new != s.rows.features_new) {
            d.flags = flags;
            d.features_old = s.rows.features_old;
            d.features_new = s.rows.features_new;
            descs_changed = true;
        }
        any_pending |= s.pending != 0;
        any_redistribute |= s.redistribute;
    }
    if (descs_changed)
        CK(cudaMemcpyAsync(ctx->tdesc_table.ptr, ctx->tdescs.data(), ctx->tdescs.size() * sizeof(TransposeDesc), cudaMemcpyHostToDevice, ctx->stream));
    if (any_pending)  // a frame whose only change is a constraint write (or a feature-id upload) transposes nothing
        launch_transpose_in_all(ctx->tb_table.as<DeviceTypeBatch>(), ctx->tdesc_table.as<TransposeDesc>(), ctx->work_table.as<WorkItem>(), ctx->topo.all_work_count, ctx->W,
                                kTransposePrestep | kTransposeImpulses | kTransposePending, ctx->stream);
    if (any_redistribute)
        launch_redistribute_impulses(ctx->tb_table.as<DeviceTypeBatch>(), ctx->tdesc_table.as<TransposeDesc>(), ctx->work_table.as<WorkItem>(), ctx->topo.all_work_count, ctx->stream);
    PrestepWriteQueue& q = ctx->prestep_writes;
    if (!q.writes.empty()) {
        const size_t bytes = q.writes.size() * sizeof(PrestepWrite), row_bytes = q.rows.size() * sizeof(float);
        CK(ctx->write_table.reserve(bytes));
        CK(ctx->write_rows.reserve(row_bytes));
        TRY(upload_staged(ctx, ctx->write_stage, ctx->write_table.ptr, q.writes.data(), bytes));
        TRY(upload_staged(ctx, ctx->write_rows_stage, ctx->write_rows.ptr, q.rows.data(), row_bytes));
        ctx->h2d_accum += (int64_t)(bytes + row_bytes);
        launch_write_constraints(ctx->tb_table.as<DeviceTypeBatch>(), ctx->tdesc_table.as<TransposeDesc>(), ctx->write_table.as<PrestepWrite>(), ctx->write_rows.as<float>(),
                                 (int)q.writes.size(), ctx->stream);
        q.clear();
    }
    for (SourceTypeBatch& s : ctx->sources) {
        if (s.redistribute) std::swap(s.rows.features_old, s.rows.features_new);  // the resident impulses now belong to the new ids
        s.redistribute = false;
        s.pending = 0;
    }
    CK(cudaGetLastError());
    ctx->data_dirty = false;
    return BEPUCUDA_OK;
}

// What a frame of length dt needs on the device before its first stage: the refreshed rows, the end of the upload window (bepucuda_timings
// upload_ms / h2d_bytes) and the frame parameters.
int prepare_frame(bepucuda_ctx* ctx, float dt) {
    TRY(refresh_device_rows(ctx));
    if (ctx->upload_window.open) ctx->upload_window.stop(ctx->stream);
    ctx->timings.h2d_bytes = ctx->h2d_accum;
    ctx->h2d_accum = 0;
    // frame parameters (previous solve's copy has completed by stream order only after its graph, a stage profile's before it returned; wait for
    // it before reusing the pinned struct)
    CK(cudaEventSynchronize(ctx->solve_window.end));
    FrameParams* fp = ctx->frame_params_host.as<FrameParams>();
    compute_frame_params(ctx, dt, fp);
    fp->exchange_base = ctx->exchange_counter;
    fp->shard_solve_index = ctx->shard_solve_index;
    CK(cudaMemcpyAsync(ctx->frame_params_dev.ptr, fp, sizeof(FrameParams), cudaMemcpyHostToDevice, ctx->stream));
    return BEPUCUDA_OK;
}

}  // namespace

static int plan_device_rows(bepucuda_ctx* ctx);

extern "C" {

int32_t bepucuda_type_info(int32_t type_id, int32_t* bodies_per_constraint, int32_t* prestep_floats, int32_t* impulse_floats) {
    const TypeInfo* t = get_type_info(type_id);
    if (!t) return BEPUCUDA_ERR_UNSUPPORTED_TYPE;
    if (bodies_per_constraint) *bodies_per_constraint = t->bodies;
    if (prestep_floats) *prestep_floats = t->prestep_rows;
    if (impulse_floats) *impulse_floats = t->impulse_rows;
    return BEPUCUDA_OK;
}

int32_t bepucuda_create(const bepucuda_config* cfg, bepucuda_ctx** out) {
    if (!cfg || !out) return BEPUCUDA_ERR_INVALID_ARGUMENT;
    *out = nullptr;
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count <= 0) return BEPUCUDA_ERR_NO_DEVICE;  // no CPU fallback, by design
    if (cfg->device_ordinal < 0 || cfg->device_ordinal >= count) return BEPUCUDA_ERR_INVALID_ARGUMENT;
    if (cfg->execution_mode != BEPUCUDA_EXEC_GRAPH && cfg->execution_mode != BEPUCUDA_EXEC_STREAM) return BEPUCUDA_ERR_INVALID_ARGUMENT;  // 1 and 3 are retired modes
    bepucuda_ctx* ctx = new bepucuda_ctx();
    ctx->cfg = *cfg;
    ctx->device = cfg->device_ordinal;
    ctx->launchers = cfg->strict_fp ? get_launchers_bepu_strict() : get_launchers_bepu_fast();
    ctx->pinned_arena.pinned_host = true;
    ctx->pinned_arena.min_chunk = (size_t)16 << 20;
#ifdef BEPU_HAZARD
    read_hazard_environment(ctx);
#endif
    cudaError_t e = cudaSetDevice(ctx->device);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(ctx->stream.put(), cudaStreamNonBlocking);
    for (TimingWindow* w : {&ctx->solve_window, &ctx->upload_window, &ctx->download_window})
        for (Event* ev : {&w->begin, &w->end}) e = e == cudaSuccess ? ev->create() : e;
    if (e == cudaSuccess) e = ctx->frame_params_host.reserve(sizeof(FrameParams));
    if (e == cudaSuccess) e = ctx->frame_params_dev.reserve(sizeof(FrameParams));
    if (e == cudaSuccess) e = ctx->error_dev.reserve(8 * sizeof(int32_t));
    if (e != cudaSuccess) {
        bepucuda_destroy(ctx);
        return e == cudaErrorMemoryAllocation ? BEPUCUDA_ERR_OUT_OF_MEMORY : BEPUCUDA_ERR_CUDA;
    }
    // DemoPoseIntegratorCallbacks defaults (Demos/DemoCallbacks.cs:L60)
    ctx->integ.gravity[0] = 0; ctx->integ.gravity[1] = -10; ctx->integ.gravity[2] = 0;
    ctx->integ.linear_damping = 0.03f;
    ctx->integ.angular_damping = 0.03f;
    *out = ctx;
    return BEPUCUDA_OK;
}

int32_t bepucuda_destroy(bepucuda_ctx* ctx) {
    if (!ctx) return BEPUCUDA_OK;
    cudaSetDevice(ctx->device);
    if (ctx->stream) cudaStreamSynchronize(ctx->stream);
    delete ctx;  // every handle and buffer frees itself, on the device set above, the stream last among the handles
    return BEPUCUDA_OK;
}

const char* bepucuda_last_error(bepucuda_ctx* ctx) { return ctx ? ctx->error.c_str() : "null context"; }

int32_t bepucuda_host_register(bepucuda_ctx* ctx, void* ptr, int64_t bytes) {
    if (!ctx || !ptr || bytes <= 0) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "host_register: bad arguments");
    CK(cudaSetDevice(ctx->device));
    CK(cudaHostRegister(ptr, (size_t)bytes, cudaHostRegisterMapped | cudaHostRegisterPortable));
    void* dev = nullptr;
    CK(cudaHostGetDevicePointer(&dev, ptr, 0));
    ctx->host_ranges.push_back({(char*)ptr, (size_t)bytes, (char*)dev});
    return BEPUCUDA_OK;
}
int32_t bepucuda_host_unregister(bepucuda_ctx* ctx, void* ptr) {
    if (!ctx || !ptr) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "host_unregister: bad arguments");
    CK(cudaSetDevice(ctx->device));
    CK(cudaStreamSynchronize(ctx->stream));
    CK(cudaHostUnregister(ptr));
    for (size_t i = 0; i < ctx->host_ranges.size(); ++i)
        if (ctx->host_ranges[i].host == (char*)ptr) { ctx->host_ranges.erase(ctx->host_ranges.begin() + i); break; }
    return BEPUCUDA_OK;
}

int32_t bepucuda_set_solve_description(bepucuda_ctx* ctx, int32_t substep_count, const int32_t* its, int32_t fallback_batch_threshold) {
    if (!ctx || substep_count < 1 || !its || fallback_batch_threshold < 1) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "set_solve_description: bad arguments");
    for (int i = 0; i < substep_count; ++i)
        if (its[i] < 0) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "set_solve_description: negative iteration count");
    std::vector<int32_t> v(its, its + substep_count);
    const bool threshold_changed = fallback_batch_threshold != ctx->fallback_threshold;
    const bool changed = v != ctx->iterations || threshold_changed;
    ctx->iterations = v;
    ctx->fallback_threshold = fallback_batch_threshold;
    if (threshold_changed) ctx->constraints_ready = false;  // fallback split must be redone
    if (changed && ctx->constraints_ready) {
        CK(cudaSetDevice(ctx->device));
        return upload_program(ctx);
    }
    return BEPUCUDA_OK;
}

int32_t bepucuda_set_integrator(bepucuda_ctx* ctx, const bepucuda_integrator_desc* desc) {
    if (!ctx || !desc) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "set_integrator: bad arguments");
    if (desc->angular_integration_mode < 0 || desc->angular_integration_mode > 2) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "set_integrator: unknown AngularIntegrationMode");
    const bool kin_changed = (desc->integrate_velocity_for_kinematics != 0) != (ctx->integ.integrate_velocity_for_kinematics != 0);
    ctx->integ = *desc;
    ctx->integ_set = true;
    if (kin_changed && ctx->constraints_ready) {
        CK(cudaSetDevice(ctx->device));
        return upload_program(ctx);
    }
    return BEPUCUDA_OK;
}

int32_t bepucuda_set_body_accelerations(bepucuda_ctx* ctx, const float* accelerations, int32_t body_count) {
    if (!ctx) return BEPUCUDA_ERR_INVALID_ARGUMENT;
    if (!accelerations) {
        ctx->accelerations_count = -1;
        return BEPUCUDA_OK;
    }
    if (body_count != ctx->body_count) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "set_body_accelerations: the body count must match the last upload_bodies");
    CK(cudaSetDevice(ctx->device));
    ctx->upload_window.start_once(ctx->stream);
    const size_t bytes = (size_t)body_count * 32;
    CK(ctx->accelerations.reserve(std::max(bytes, (size_t)32)));
    if (bytes > 0) {
        // through a pinned staging copy, so that the caller's buffer is free when the call returns without waiting for the device
        TRY(upload_staged(ctx, ctx->accelerations_stage, ctx->accelerations.ptr, accelerations, bytes));
        ctx->h2d_accum += (int64_t)bytes;
    }
    ctx->accelerations_count = body_count;
    return BEPUCUDA_OK;
}

int32_t bepucuda_set_point_gravity(bepucuda_ctx* ctx, int32_t enabled, const float* center, float strength) {
    if (!ctx || (enabled && !center)) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "set_point_gravity: bad arguments");
    ctx->point_gravity = enabled != 0;
    for (int i = 0; i < 3; ++i) ctx->attractor_center[i] = enabled ? center[i] : 0.0f;
    ctx->attractor_strength = enabled ? strength : 0.0f;
    return BEPUCUDA_OK;
}

int32_t bepucuda_upload_bodies(bepucuda_ctx* ctx, const void* body_dynamics, int32_t body_count) {
    if (!ctx || body_count < 0 || (body_count > 0 && !body_dynamics)) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "upload_bodies: bad arguments");
    if ((uint32_t)body_count > kRefIndexMask) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "upload_bodies: too many bodies");
    CK(cudaSetDevice(ctx->device));
    ctx->upload_window.start_once(ctx->stream);
    const size_t n = (size_t)body_count;
    // constrained flags / ownership depend on the body count; force a rebuild of topology products.
    if (body_count != ctx->body_count) ctx->constraints_ready = false;
    if (const cudaError_t e = ctx->bodies.reserve(n, ctx->stream)) return cuda_fail(ctx, e, "upload_bodies: body arrays");
    ctx->body_count = body_count;
    ctx->bodies_uploaded = true;
    refresh_body_buffers(ctx);
    if (body_count > 0) {
        CK(cudaMemcpyAsync(ctx->bodies.raw.ptr, body_dynamics, n * 128, cudaMemcpyHostToDevice, ctx->stream));
        ctx->h2d_accum += (int64_t)n * 128;
        launch_split_bodies(ctx->bodies.raw.ptr, body_count, ctx->B, ctx->stream);
        CK(cudaGetLastError());
    }
    return BEPUCUDA_OK;
}

int32_t bepucuda_begin_constraints(bepucuda_ctx* ctx, int32_t source_bundle_width, int32_t batch_count) {
    if (!ctx || source_bundle_width < 1 || source_bundle_width > 64 || batch_count < 0) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "begin_constraints: bad arguments");
    CK(cudaSetDevice(ctx->device));
    CK(cudaStreamSynchronize(ctx->stream));  // staging arenas are recycled below
    ctx->upload_window.start_once(ctx->stream);
    ctx->W = source_bundle_width;
    ctx->batch_count = batch_count;
    ctx->sources.clear();
    ctx->pending_h2d.clear();  // queued refreshes target raw-arena addresses that are recycled below; a re-describe uploads everything anyway
    ctx->prestep_writes.clear();  // slots of the old plan; the describe uploads the host's prestep, which ApplyDescription already wrote
    ctx->raw_arena.reset();
    ctx->spare_rows.clear();
    ctx->pinned_arena.reset();
    ctx->constraints_open = true;
    ctx->constraints_ready = false;
    return BEPUCUDA_OK;
}

int32_t bepucuda_upload_type_batch(bepucuda_ctx* ctx, int32_t batch_index, int32_t type_batch_index, int32_t type_id, int32_t constraint_count,
                                   const int32_t* body_references, const float* prestep, float* accumulated_impulses) {
    if (!ctx) return BEPUCUDA_ERR_INVALID_ARGUMENT;
    if (!ctx->constraints_open) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "upload_type_batch outside begin/end_constraints");
    if (batch_index < 0 || batch_index >= ctx->batch_count || type_batch_index < 0 || constraint_count < 0)
        return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "upload_type_batch: bad indices");
    const TypeInfo* t = get_type_info(type_id);
    if (!t) return fail(ctx, BEPUCUDA_ERR_UNSUPPORTED_TYPE, "upload_type_batch: unsupported constraint type id " + std::to_string(type_id));
    if (constraint_count == 0) return BEPUCUDA_OK;
    if (!body_references || !prestep || !accumulated_impulses) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "upload_type_batch: null buffer");
    CK(cudaSetDevice(ctx->device));
    const int W = ctx->W;
    SourceTypeBatch s;
    s.host = {batch_index, type_batch_index, type_id, constraint_count, {}};
    s.capacity = (int)(((size_t)constraint_count + W - 1) / W) * W;
    s.host_impulses = accumulated_impulses;
    if (const cudaError_t e = take_source_rows(ctx, t, s.capacity, false, &s.rows)) return cuda_fail(ctx, e, "raw arena");
    TRY(copy_in(ctx, s.rows.refs, body_references, s.bytes(kRowRefs, W)));
    TRY(copy_in(ctx, s.rows.prestep, prestep, s.bytes(kRowPrestep, W)));
    TRY(copy_in(ctx, s.rows.impulses, accumulated_impulses, s.bytes(kRowImpulses, W)));
    if (batch_index >= ctx->fallback_threshold) s.host.refs.assign(body_references, body_references + s.bytes(kRowRefs, W) / 4);
    ctx->sources.push_back(std::move(s));
    return BEPUCUDA_OK;
}

int32_t bepucuda_set_constrained_kinematics(bepucuda_ctx* ctx, const int32_t* body_indices, int32_t count) {
    if (!ctx || count < 0 || (count > 0 && !body_indices)) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "set_constrained_kinematics: bad arguments");
    ctx->kinematics.assign(body_indices, body_indices + count);
    ctx->constraints_ready = false;
    return BEPUCUDA_OK;
}

int32_t bepucuda_end_constraints(bepucuda_ctx* ctx) {
    if (!ctx) return BEPUCUDA_ERR_INVALID_ARGUMENT;
    if (!ctx->constraints_open) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "end_constraints without begin_constraints");
    if (ctx->peer_mode && (int)ctx->body_masks.size() != ctx->body_count)
        return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "end_constraints: peer sharding needs bepucuda_shard_set_body_masks for the current body count");
    CK(cudaSetDevice(ctx->device));
    return plan_device_rows(ctx);
}

}  // extern "C"

// The body of bepucuda_end_constraints, shared with bepucuda_add_constraints / bepucuda_remove_constraints: plans the sources' rows as they are on
// the device (raw arrays), builds the tables, transposes every row in, runs the ownership passes and replaces the stage program.
static int plan_device_rows(bepucuda_ctx* ctx) {
    const int W = ctx->W;
    {
        std::vector<SourceView> views;
        for (const SourceTypeBatch& s : ctx->sources) views.push_back({s.host.batch_index, s.host.type_batch_index, s.host.type_id, s.host.count, s.host.refs.data()});
        TopologyPlan plan;
        std::string error;
        const int rc = plan_topology(views, W, ctx->fallback_threshold, ctx->batch_count, ctx->body_count, ctx->peer_mode, &plan, &error, ctx->peers.rank, ctx->fallback_rank);
        if (rc != BEPUCUDA_OK) return fail(ctx, rc, error);
        ctx->topo = std::move(plan);
        ctx->prestep_writes.plan(ctx->topo);
    }
    const TopologyPlan& topo = ctx->topo;

    // ---- device arenas for the AOSOA-32 image, type batches, transposition descriptors, work records ----
    CK(ctx->refs32.reserve(topo.refs_words * 4 + 1024));  // slack: solver warps always read two body-reference rows
    CK(ctx->prestep32.reserve(topo.prestep_words * 4 + 4));
    CK(ctx->impulses32.reserve(topo.impulse_words * 4 + 4));
    TRY(upload_table(ctx, "map_table", ctx->map_table, topo.maps, 4));
    TRY(upload_table(ctx, "inverse_table", ctx->inverse_table, topo.inverse, 8));
    std::vector<DeviceTypeBatch> tbs(topo.tbs.size());
    ctx->tdescs.resize(topo.tbs.size());
    for (size_t i = 0; i < topo.tbs.size(); ++i) {
        const PlannedTypeBatch& p = topo.tbs[i];
        const SourceTypeBatch& s = ctx->sources[(size_t)p.source];
        const TypeInfo* t = get_type_info(p.type_id);
        tbs[i] = {p.type_id, p.bundle_count, p.device_batch, t->bodies, ctx->refs32.as<int32_t>() + p.refs_offset, ctx->prestep32.as<float>() + p.prestep_offset,
                  ctx->impulses32.as<float>() + p.impulse_offset};
        ctx->tdescs[i] = {s.rows.refs, s.rows.prestep, s.rows.impulses, p.map_offset < 0 ? nullptr : ctx->map_table.as<int32_t>() + p.map_offset, s.host.count, t->bodies, t->prestep_rows,
                          t->impulse_rows, topo.source_bundle_base[(size_t)p.source], kTransposePrestep | kTransposeImpulses, t->contacts, nullptr, nullptr};
    }
    ctx->records = work_records(topo, ctx->refs32.as<int32_t>(), ctx->prestep32.as<float>(), ctx->impulses32.as<float>());

    // ---- upload tables ----
    TRY(upload_table(ctx, "tb_table", ctx->tb_table, tbs, 16));
    TRY(upload_table(ctx, "tdesc_table", ctx->tdesc_table, ctx->tdescs, 16));
    TRY(upload_table(ctx, "work_table", ctx->work_table, topo.work, 16));
    TRY(upload_table(ctx, "record_table", ctx->record_table, ctx->records, 64));
    TRY(upload_table(ctx, "kinematics_dev", ctx->kinematics_dev, ctx->kinematics, 4));

    // ---- transposition into AOSOA-32 + ownership analysis ----
    TRY(flush_chunks(ctx, ctx->pending_h2d));
    launch_transpose_in_all(ctx->tb_table.as<DeviceTypeBatch>(), ctx->tdesc_table.as<TransposeDesc>(), ctx->work_table.as<WorkItem>(), topo.all_work_count, W,
                            kTransposeRefs | kTransposePrestep | kTransposeImpulses, ctx->stream);
    const size_t nb = (size_t)std::max(ctx->body_count, 1);
    CK(ctx->bodies.first_batch.reserve(nb * 4));
    CK(ctx->sync_refcount.reserve(nb * 4));
    CK(ctx->sync_mask.reserve(nb * 8));
    refresh_body_buffers(ctx);
    launch_fill_i32(ctx->bodies.first_batch.as<int32_t>(), nb, 0x7fffffff, ctx->stream);
    CK(cudaMemsetAsync(ctx->sync_refcount.ptr, 0, nb * 4, ctx->stream));
    CK(cudaMemsetAsync(ctx->sync_mask.ptr, 0, nb * 8, ctx->stream));
    CK(cudaMemsetAsync(ctx->bodies.constrained.ptr, 0, nb, ctx->stream));
    CK(cudaMemsetAsync(ctx->error_dev.ptr, 0, 32, ctx->stream));
    CK(ctx->source_bundle_flags.reserve((size_t)std::max(topo.source_bundles, 1) * 16));
    CK(cudaMemsetAsync(ctx->source_bundle_flags.ptr, 0, (size_t)std::max(topo.source_bundles, 1) * 16, ctx->stream));
    launch_ownership_pass1(ctx->tb_table.as<DeviceTypeBatch>(), ctx->work_table.as<WorkItem>(), topo.all_work_count, topo.sync_batch_count,
                           ctx->body_count, ctx->bodies.first_batch.as<int32_t>(), ctx->sync_refcount.as<int32_t>(), (unsigned long long*)ctx->sync_mask.ptr, ctx->error_dev.as<int32_t>(),
                           ctx->stream);
    if (ctx->peer_mode && nb > 0) {
        // peer sharding: the integration owner of a body is the lowest batch referencing it on ANY rank (computed by the host over the whole graph);
        // a body the graph first references in the fallback batch keeps the level this rank, the fallback rank, found for it
        if ((int)ctx->global_first_batch.size() != ctx->body_count) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "end_constraints: bepucuda_shard_set_global was not called for this body count");
        CK(ctx->global_first_batch_dev.reserve(nb * 4));
        CK(cudaMemcpyAsync(ctx->global_first_batch_dev.ptr, ctx->global_first_batch.data(), (size_t)ctx->body_count * 4, cudaMemcpyHostToDevice, ctx->stream));
        launch_merge_first_batch(ctx->bodies.first_batch.as<int32_t>(), ctx->global_first_batch_dev.as<int32_t>(), ctx->body_count, ctx->fallback_threshold, ctx->stream);
    }
    launch_ownership_rest(ctx->tb_table.as<DeviceTypeBatch>(), ctx->work_table.as<WorkItem>(), topo.all_work_count, ctx->body_count,
                          ctx->bodies.first_batch.as<int32_t>(), ctx->sync_refcount.as<int32_t>(), (const unsigned long long*)ctx->sync_mask.ptr, ctx->bodies.constrained.as<uint8_t>(),
                          ctx->kinematics_dev.as<int32_t>(), (int)ctx->kinematics.size(), ctx->error_dev.as<int32_t>(), ctx->tdesc_table.as<TransposeDesc>(), W,
                          ctx->source_bundle_flags.as<int32_t>(), ctx->stream);
    if (ctx->peer_mode) {
        // ... and a body is "constrained" (final pose pass) if any rank constrains it
        CK(cudaMemcpyAsync(ctx->bodies.constrained.ptr, ctx->global_constrained.data(), (size_t)ctx->body_count, cudaMemcpyHostToDevice, ctx->stream));
        // per body reference, the other ranks that need what this rank's constraint writes
        CK(ctx->peer32.reserve(topo.refs_words * 4 + 1024));
        CK(ctx->body_masks_dev.reserve((size_t)ctx->body_count + 16));
        CK(cudaMemcpyAsync(ctx->body_masks_dev.ptr, ctx->body_masks.data(), (size_t)ctx->body_count, cudaMemcpyHostToDevice, ctx->stream));
        launch_fill_peer_masks(ctx->refs32.as<int32_t>(), ctx->peer32.as<uint32_t>(), topo.refs_words, ctx->body_masks_dev.as<uint8_t>(), ctx->peers.rank, ctx->stream);
        // boundary bundles (any lane writes a shared body) go to the front of their batch and carry kRecordBoundaryBit: they are scheduled first, and
        // the flag barrier of the stage involves only them (ShardStage)
        const int n_rec = topo.all_work_count;
        CK(ctx->boundary_flags_dev.reserve((size_t)n_rec + 16));
        launch_boundary_flags(ctx->tb_table.as<DeviceTypeBatch>(), ctx->work_table.as<WorkItem>(), n_rec, (long long)(ctx->peer32.as<int32_t>() - ctx->refs32.as<int32_t>()),
                              ctx->boundary_flags_dev.as<uint8_t>(), ctx->stream);
        std::vector<uint8_t> is_boundary((size_t)n_rec);
        if (n_rec > 0) CK(cudaMemcpyAsync(is_boundary.data(), ctx->boundary_flags_dev.ptr, (size_t)n_rec, cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        ctx->boundary_count = sort_boundary_first(topo, is_boundary.data(), ctx->records);
        if (n_rec > 0) CK(cudaMemcpyAsync(ctx->record_table.ptr, ctx->records.data(), (size_t)n_rec * sizeof(WorkRecord), cudaMemcpyHostToDevice, ctx->stream));
    }
    // the first two body-reference rows of every work record, packed in work-list order (they carry the ownership bits set above)
    CK(ctx->ref_rows.reserve((size_t)std::max<size_t>(ctx->records.size(), 1) * 64 * 4));
    launch_pack_ref_rows(ctx->record_table.as<WorkRecord>(), (int)ctx->records.size(), ctx->ref_rows.as<int32_t>(), ctx->stream);
    CK(cudaGetLastError());
    int32_t err = 0;
    CK(cudaMemcpyAsync(&err, ctx->error_dev.ptr, 4, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));  // also guarantees the std::vector sources of the copies above were consumed
    if (err == 1) return fail(ctx, BEPUCUDA_ERR_BATCH_INVARIANT, "end_constraints: a synchronized batch references the same dynamic body more than once");
    if (err == 2) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "end_constraints: body reference out of range");

    ctx->timings.constraint_count = topo.constraint_count;
    ctx->timings.device_batch_count = (int)topo.batches.size();
    ctx->timings.fallback_level_count = topo.fallback_levels;
    ctx->constraints_open = false;
    ctx->data_dirty = false;
    return upload_program(ctx);
}

extern "C" {

int32_t bepucuda_update_type_batch(bepucuda_ctx* ctx, int32_t batch_index, int32_t type_batch_index, const float* prestep, float* accumulated_impulses) {
    if (!ctx || !prestep || !accumulated_impulses) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "update_type_batch: bad arguments");
    if (!ctx->constraints_ready) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "update_type_batch before end_constraints");
    SourceTypeBatch* s = find_source(ctx, batch_index, type_batch_index);
    if (!s) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "update_type_batch: unknown type batch");
    CK(cudaSetDevice(ctx->device));
    ctx->upload_window.start_once(ctx->stream);
    TRY(copy_in(ctx, s->rows.prestep, prestep, s->bytes(kRowPrestep, ctx->W)));
    TRY(copy_in(ctx, s->rows.impulses, accumulated_impulses, s->bytes(kRowImpulses, ctx->W)));
    s->host_impulses = accumulated_impulses;
    s->pending = kTransposePrestep | kTransposeImpulses;
    s->redistribute = false;  // the host took the impulses back
    ctx->data_dirty = true;
    return BEPUCUDA_OK;
}

int32_t bepucuda_set_contact_features(bepucuda_ctx* ctx, int32_t batch_index, int32_t type_batch_index, const int32_t* feature_ids) {
    if (!ctx || !feature_ids) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "set_contact_features: bad arguments");
    if (!ctx->constraints_open && !ctx->constraints_ready) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "set_contact_features before the type batch was uploaded");
    SourceTypeBatch* s = find_source(ctx, batch_index, type_batch_index);
    if (!s) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "set_contact_features: unknown type batch");
    if (s->type()->contacts == 0) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "set_contact_features: not a contact constraint type");
    CK(cudaSetDevice(ctx->device));
    if (!s->rows.features_old)
        if (const cudaError_t e = take_feature_rows(ctx, s->type(), s->capacity, &s->rows)) return cuda_fail(ctx, e, "raw arena (contact feature ids)");
    // from a mapped buffer the ids are only queued: the next solve copies them, before the host writes the next frame's ids into the same buffer
    if (ctx->constraints_ready) ctx->data_dirty = true;
    return copy_in(ctx, s->rows.features_old, feature_ids, s->bytes(kRowFeatures, ctx->W));
}

int32_t bepucuda_update_contacts(bepucuda_ctx* ctx, int32_t batch_index, int32_t type_batch_index, const float* prestep, const int32_t* new_feature_ids) {
    if (!ctx || !prestep || !new_feature_ids) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "update_contacts: bad arguments");
    if (!ctx->constraints_ready) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "update_contacts before end_constraints");
    SourceTypeBatch* s = find_source(ctx, batch_index, type_batch_index);
    if (!s) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "update_contacts: unknown type batch");
    if (s->type()->contacts == 0) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "update_contacts: not a contact constraint type");
    if (!s->rows.features_old) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "update_contacts: bepucuda_set_contact_features was never called for this type batch");
    if (s->redistribute) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "update_contacts: called twice for the same type batch without a solve in between");
    CK(cudaSetDevice(ctx->device));
    ctx->upload_window.start_once(ctx->stream);
    TRY(copy_in(ctx, s->rows.prestep, prestep, s->bytes(kRowPrestep, ctx->W)));
    TRY(copy_in(ctx, s->rows.features_new, new_feature_ids, s->bytes(kRowFeatures, ctx->W)));
    s->pending |= kTransposePrestep;  // the accumulated impulses stay resident
    s->redistribute = true;
    ctx->data_dirty = true;
    return BEPUCUDA_OK;
}

int32_t bepucuda_upload_body_motion(bepucuda_ctx* ctx, const void* body_dynamics, int32_t body_count) {
    if (!ctx || !body_dynamics || body_count != ctx->body_count) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "upload_body_motion: bad arguments (the body count must match the last upload_bodies)");
    if (body_count == 0) return BEPUCUDA_OK;
    CK(cudaSetDevice(ctx->device));
    ctx->upload_window.start_once(ctx->stream);
    const size_t n = (size_t)body_count;
    if (char* alias = map_host(ctx, body_dynamics, n * 128)) {
        launch_scatter_body_motion(alias, body_count, ctx->B, ctx->stream);  // 64 of every 128 bytes read straight from the mapped host buffer
    } else {
        CK(cudaMemcpy2DAsync(ctx->bodies.raw.ptr, 128, body_dynamics, 128, 64, n, cudaMemcpyHostToDevice, ctx->stream));
        launch_scatter_body_motion(ctx->bodies.raw.ptr, body_count, ctx->B, ctx->stream);
    }
    CK(cudaGetLastError());
    ctx->h2d_accum += (int64_t)n * 64;
    return BEPUCUDA_OK;
}

int32_t bepucuda_write_bodies(bepucuda_ctx* ctx, const void* body_dynamics, int32_t count, const int32_t* body_indices) {
    if (!ctx) return BEPUCUDA_ERR_INVALID_ARGUMENT;
    const char* why = "";
    const int rc = check_body_write(ctx->bodies_uploaded, ctx->body_count, body_dynamics, count, body_indices, &why);
    if (rc != BEPUCUDA_OK) return fail(ctx, rc, std::string("write_bodies: ") + why);
    if (count == 0) return BEPUCUDA_OK;
    CK(cudaSetDevice(ctx->device));
    ctx->upload_window.start_once(ctx->stream);
    const size_t n = (size_t)count, index_bytes = n * sizeof(int32_t);
    // A registered buffer is read by the kernel when the stream reaches it; an unregistered one is gathered here, so it is free on return.
    const char* alias = map_host(ctx, body_dynamics, (size_t)ctx->body_count * 128);
    const size_t motion_bytes = alias ? 0 : n * 64;
    StagedUpload& st = ctx->body_write_stage;
    TRY(reserve_staging(ctx, st, motion_bytes + index_bytes));
    CK(ctx->body_writes.reserve(motion_bytes + index_bytes));
    if (!alias) gather_motion_halves(body_dynamics, body_indices, count, st.host.as<float>());
    std::memcpy(st.host.as<char>() + motion_bytes, body_indices, index_bytes);
    TRY(send_staging(ctx, st, ctx->body_writes.ptr, motion_bytes + index_bytes));
    const int32_t* indices = (const int32_t*)(ctx->body_writes.as<char>() + motion_bytes);
    launch_write_body_motion(alias ? (const void*)alias : ctx->body_writes.ptr, indices, count, !alias, ctx->B, ctx->stream);
    CK(cudaGetLastError());
    ctx->h2d_accum += (int64_t)n * (64 + 4);
    return BEPUCUDA_OK;
}

int32_t bepucuda_download_body_motion(bepucuda_ctx* ctx, void* out, int32_t body_count) {
    if (!ctx || !out || body_count < 0 || body_count > ctx->body_count) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "download_body_motion: bad arguments");
    CK(cudaSetDevice(ctx->device));
    CK(ctx->download_window.start(ctx->stream));
    const size_t n = (size_t)body_count;
    if (char* alias = map_host(ctx, out, n * 128)) {
        launch_gather_body_motion(alias, body_count, ctx->B, ctx->stream);
    } else {
        launch_gather_body_motion(ctx->bodies.raw.ptr, body_count, ctx->B, ctx->stream);
        CK(cudaMemcpy2DAsync(out, 128, ctx->bodies.raw.ptr, 128, 64, n, cudaMemcpyDeviceToHost, ctx->stream));
    }
    CK(cudaGetLastError());
    CK(ctx->download_window.stop(ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    ctx->timings.d2h_bytes = (int64_t)n * 64;
    return BEPUCUDA_OK;
}

int32_t bepucuda_solve(bepucuda_ctx* ctx, float dt) {
    if (!ctx || !(dt > 0)) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "solve: bad arguments");
    TRY(check_accelerations(ctx, "solve"));
    CK(cudaSetDevice(ctx->device));
    if (!ctx->constraints_ready) {
        // No constraints were ever described (or the description was invalidated): only legal when nothing was uploaded.
        if (ctx->constraints_open) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "solve inside begin/end_constraints");
        if (!ctx->sources.empty()) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "solve: constraint description is stale; re-run begin/upload/end_constraints");
        TRY(bepucuda_begin_constraints(ctx, ctx->W, 0));
        TRY(bepucuda_end_constraints(ctx));
    }
    TRY(prepare_frame(ctx, dt));
    CK(ctx->solve_window.start(ctx->stream));
    int64_t launches = 0;
    if (ctx->cfg.execution_mode == BEPUCUDA_EXEC_GRAPH) {
        const LaunchContext lc = launch_context(ctx, false);
        StageGraph& g = ctx->stage_graph;
        if (!g.matches(ctx->B, lc)) {
            g.reset();
            CK(cudaStreamBeginCapture(ctx->stream, cudaStreamCaptureModeThreadLocal));
            int64_t n = 0;
            issue_stage_sequence(ctx, ctx->stream, &n);
            cudaError_t e = cudaStreamEndCapture(ctx->stream, g.graph.put());
            if (e == cudaSuccess) e = cudaGraphInstantiate(g.exec.put(), g.graph, 0);
            if (e != cudaSuccess) return cuda_fail(ctx, e, "graph capture");
            g.bodies = ctx->B;
            g.launch = lc;
            ctx->timings.kernel_launches = n;
            ++ctx->timings.graph_captures;
        }
        CK(cudaGraphLaunch(g.exec, ctx->stream));
        launches = ctx->timings.kernel_launches;
    }
    if (ctx->cfg.execution_mode == BEPUCUDA_EXEC_STREAM) {
        issue_stage_sequence(ctx, ctx->stream, &launches);
        CK(cudaGetLastError());
    }
    CK(ctx->solve_window.stop(ctx->stream));
    if (ctx->peer_mode) { ctx->exchange_counter += ctx->program.exchange_count; ++ctx->shard_solve_index; }  // the flag barrier and the arrival counters keep counting across solves
    ctx->timings.kernel_launches = launches;

    // metric bookkeeping (SURVEY.md §8d)
    ctx->timings.constraint_iterations = ctx->program.constraint_iterations;
    ctx->timings.algorithmic_bytes = ctx->program.algorithmic_bytes;
    // one acceleration record per integrating lane: one per body and substep
    if (ctx->accelerations_count >= 0) ctx->timings.algorithmic_bytes += (int64_t)ctx->body_count * (int64_t)ctx->iterations.size() * 32;
    return BEPUCUDA_OK;
}

static int check_device_error_flag(bepucuda_ctx* ctx) {
    if (ctx->peer_mode) {
        int32_t e = 0;
        CK(cudaMemcpyAsync(&e, ctx->error_dev.ptr, 4, cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        if (e == 5) return fail(ctx, BEPUCUDA_ERR_CUDA, "sharded solve: a peer rank never reached an exchange point (flag barrier timed out); results are invalid");
    }
    return BEPUCUDA_OK;
}

int32_t bepucuda_synchronize(bepucuda_ctx* ctx) {
    if (!ctx) return BEPUCUDA_ERR_INVALID_ARGUMENT;
    CK(cudaSetDevice(ctx->device));
    CK(cudaStreamSynchronize(ctx->stream));
    return check_device_error_flag(ctx);
}

int32_t bepucuda_download_bodies(bepucuda_ctx* ctx, void* out, int32_t body_count) {
    if (!ctx || !out || body_count < 0 || body_count > ctx->body_count) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "download_bodies: bad arguments");
    CK(cudaSetDevice(ctx->device));
    CK(ctx->download_window.start(ctx->stream));
    launch_merge_bodies(ctx->bodies.raw.ptr, body_count, ctx->B, ctx->stream);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(out, ctx->bodies.raw.ptr, (size_t)body_count * 128, cudaMemcpyDeviceToHost, ctx->stream));
    CK(ctx->download_window.stop(ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    ctx->timings.d2h_bytes = (int64_t)body_count * 128;
    return BEPUCUDA_OK;
}

int32_t bepucuda_download_impulses(bepucuda_ctx* ctx) {
    if (!ctx) return BEPUCUDA_ERR_INVALID_ARGUMENT;
    if (!ctx->constraints_ready) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "download_impulses before end_constraints");
    for (const SourceTypeBatch& s : ctx->sources)
        if (!s.host_impulses)
            return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "download_impulses: type batch (" + std::to_string(s.host.batch_index) + ", " + std::to_string(s.host.type_batch_index) +
                                                         ") took constraints through bepucuda_add_constraints; pass its buffers again (update_type_batch or a describe)");
    CK(cudaSetDevice(ctx->device));
    TRY(transpose_out(ctx, kTransposeImpulses));
    int64_t bytes = 0;
    std::vector<CopyChunk> d2h;
    for (auto& s : ctx->sources) {
        const size_t n = s.bytes(kRowImpulses, ctx->W);
        if (char* alias = map_host(ctx, s.host_impulses, n)) queue_chunks(d2h, alias, s.rows.impulses, n);
        else CK(cudaMemcpyAsync(s.host_impulses, s.rows.impulses, n, cudaMemcpyDeviceToHost, ctx->stream));
        bytes += (int64_t)n;
    }
    TRY(flush_chunks(ctx, d2h));
    CK(cudaStreamSynchronize(ctx->stream));
    ctx->timings.d2h_bytes += bytes;
    return BEPUCUDA_OK;
}

int32_t bepucuda_download_prestep(bepucuda_ctx* ctx, int32_t batch_index, int32_t type_batch_index, float* prestep_out) {
    if (!ctx || !prestep_out) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "download_prestep: bad arguments");
    if (!ctx->constraints_ready) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "download_prestep before end_constraints");
    const SourceTypeBatch* s = find_source(ctx, batch_index, type_batch_index);
    if (!s) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "download_prestep: unknown type batch");
    CK(cudaSetDevice(ctx->device));
    TRY(transpose_out(ctx, kTransposePrestep));
    CK(cudaMemcpyAsync(prestep_out, s->rows.prestep, s->bytes(kRowPrestep, ctx->W), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return BEPUCUDA_OK;
}

static_assert(sizeof(bepucuda_constraint_location) == 16, "bepucuda_constraint_location is four int32");

int32_t bepucuda_read_constraints(bepucuda_ctx* ctx, int32_t count, const bepucuda_constraint_location* locations, int32_t* records_out) {
    if (!ctx) return BEPUCUDA_ERR_INVALID_ARGUMENT;
    std::vector<ResolvedLocation> resolved;
    TRY(resolve_locations(ctx, "read_constraints", count, locations, records_out, false, &resolved));
    if (count == 0) return BEPUCUDA_OK;
    std::vector<ReadRequest> requests((size_t)count);
    for (int32_t i = 0; i < count; ++i) {
        const ResolvedLocation& r = resolved[(size_t)i];
        // a fallback constraint, a hole included, is looked up on the device through its inverse entry
        requests[(size_t)i] = {locations[i].type_id, r.inverse_entry < 0 ? r.at : DeviceSlot{-1, (int32_t)r.inverse_entry}};
    }
    CK(cudaSetDevice(ctx->device));
    const size_t n = (size_t)count;
    CK(ctx->read_requests.reserve(n * sizeof(ReadRequest)));
    CK(ctx->read_records.reserve(n * 256));
    CK(cudaMemcpyAsync(ctx->read_requests.ptr, requests.data(), n * sizeof(ReadRequest), cudaMemcpyHostToDevice, ctx->stream));
    launch_read_constraints(ctx->tb_table.as<DeviceTypeBatch>(), ctx->tdesc_table.as<TransposeDesc>(), ctx->inverse_table.as<DeviceSlot>(), ctx->read_requests.as<ReadRequest>(),
                            count, ctx->read_records.as<int32_t>(), ctx->stream);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(records_out, ctx->read_records.ptr, n * 256, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return BEPUCUDA_OK;
}

int32_t bepucuda_write_constraints(bepucuda_ctx* ctx, int32_t count, const bepucuda_constraint_location* locations, const int32_t* records) {
    if (!ctx) return BEPUCUDA_ERR_INVALID_ARGUMENT;
    std::vector<ResolvedLocation> resolved;
    TRY(resolve_locations(ctx, "write_constraints", count, locations, records, true, &resolved));
    if (count == 0) return BEPUCUDA_OK;
    CK(cudaSetDevice(ctx->device));
    ctx->upload_window.start_once(ctx->stream);
    for (int32_t i = 0; i < count; ++i)
        ctx->prestep_writes.put(resolved[(size_t)i].at, (const float*)(records + (size_t)i * 64 + kRecordPrestep), get_type_info(locations[i].type_id)->prestep_rows);
    ctx->data_dirty = true;
    return BEPUCUDA_OK;
}

// ---- graph edits on the resident state: constraint and body adds and removes ----

// The state rules of the four graph edits; `what` names what the call changes.
static int check_graph_edit(bepucuda_ctx* ctx, const std::string& name, const char* what) {
    if (ctx->peer_mode) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, name + " in peer mode");
    if (ctx->constraints_open) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, name + " between begin_constraints and end_constraints");
    if (!ctx->constraints_ready) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, name + " before end_constraints");
    if (ctx->data_dirty)
        return fail(ctx, BEPUCUDA_ERR_BAD_STATE, name + ": rows are pending (uploads or writes since the last solve); change the " + what + " before them");
    return BEPUCUDA_OK;
}

// The device's rows of every constraint back into the sources, where a graph edit changes them and plan_device_rows reads them. From here on a
// failure leaves a context that needs a describe.
static int rows_to_sources(bepucuda_ctx* ctx) {
    TRY(transpose_out(ctx, kTransposePrestep | kTransposeImpulses));
    ctx->constraints_ready = false;
    return BEPUCUDA_OK;
}

// bepucuda_add_constraints (remove = false) and bepucuda_remove_constraints: the dry run of the whole list on the host (replay_changes), then the
// rows brought back to the sources, the lane copies, the new sources and counts, and the plan of the describe over the device rows.
static int change_constraints(bepucuda_ctx* ctx, const std::string& name, bool remove, int32_t count, const bepucuda_constraint_location* locations, const int32_t* records,
                              const int32_t* feature_ids, const int32_t* kinematics, int32_t kinematic_count) {
    TRY(check_graph_edit(ctx, name, "constraints"));
    if (count < 0 || (count > 0 && (!locations || (!remove && !records))) || kinematic_count < 0 || (kinematic_count > 0 && !kinematics))
        return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, name + ": bad arguments");
    for (int32_t i = 0; i < kinematic_count; ++i)
        if (kinematics[i] < 0 || kinematics[i] >= ctx->body_count) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, name + ": constrained kinematic index out of range");
    if (!remove && !feature_ids)
        for (int32_t i = 0; i < count; ++i)
            if (contact_count_of_type(locations[i].type_id) > 0) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, name + ": feature_ids is NULL and entry " + std::to_string(i) + " is a contact");
    const int W = ctx->W;
    ChangeState next;
    next.batch_count = ctx->batch_count;
    for (const SourceTypeBatch& s : ctx->sources) next.sources.push_back(s.host);
    std::vector<LaneCopy> ops;
    std::string error;
    if (replay_changes(&next, remove, W, ctx->fallback_threshold, ctx->body_count, count, locations, records, &ops, &error) != BEPUCUDA_OK)
        return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, name + ": " + error);
    const std::vector<LaneCopy> copies = compose_lane_ops(ops);
    std::vector<char> took_add(next.sources.size(), 0);
    for (const LaneCopy& c : copies) took_add[(size_t)c.dst_source] |= c.src_source == kLaneNew;

    CK(cudaSetDevice(ctx->device));
    // Rows for every source that outgrows its arrays (new sources included), taken before any device work: a failure returns every block taken
    // and leaves the context as it was. A new contact source keeps feature ids when the adds bring them; an existing one keeps them if it had them
    // (one that never had bepucuda_set_contact_features still refuses bepucuda_update_contacts).
    struct Growth { size_t source; int capacity; RawRows rows; };
    std::vector<Growth> growth;
    for (size_t i = 0; i < next.sources.size(); ++i) {
        const ChangeSource& n = next.sources[i];
        const int capacity = i < ctx->sources.size() ? ctx->sources[i].capacity : 0;
        const int needed = (n.count + W - 1) / W * W;
        if (needed <= capacity) continue;
        const bool features = i < ctx->sources.size() ? ctx->sources[i].rows.features_old != nullptr : feature_ids != nullptr;
        Growth g{i, std::max(needed, 2 * capacity), {}};
        if (const cudaError_t e = take_source_rows(ctx, get_type_info(n.type_id), g.capacity, features, &g.rows)) {
            for (const Growth& h : growth) give_source_rows(ctx, get_type_info(next.sources[h.source].type_id), h.capacity, h.rows);
            return cuda_fail(ctx, e, (name + ": raw arena").c_str());
        }
        growth.push_back(g);
    }
    ctx->upload_window.start_once(ctx->stream);
    TRY(rows_to_sources(ctx));
    std::vector<SourceTypeBatch> all = std::move(ctx->sources);
    for (size_t i = all.size(); i < next.sources.size(); ++i) all.emplace_back().host.type_id = next.sources[i].type_id;
    // grown sources: the rows of their old constraints (as transposed out above) into the new arrays; the old arrays become spare
    for (const Growth& g : growth) {
        SourceTypeBatch& s = all[g.source];
        const TypeInfo* t = s.type();
        CK(cudaMemsetAsync(g.rows.refs, 0xff, row_bytes(t, kRowRefs, g.capacity, W), ctx->stream));
        if (g.rows.features_old) CK(cudaMemsetAsync(g.rows.features_old, 0, row_bytes(t, kRowFeatures, g.capacity, W), ctx->stream));
        if (s.host.count > 0) {  // the old count (0 for a new source)
            CK(cudaMemcpyAsync(g.rows.refs, s.rows.refs, s.bytes(kRowRefs, W), cudaMemcpyDeviceToDevice, ctx->stream));
            CK(cudaMemcpyAsync(g.rows.prestep, s.rows.prestep, s.bytes(kRowPrestep, W), cudaMemcpyDeviceToDevice, ctx->stream));
            CK(cudaMemcpyAsync(g.rows.impulses, s.rows.impulses, s.bytes(kRowImpulses, W), cudaMemcpyDeviceToDevice, ctx->stream));
            if (s.rows.features_old) CK(cudaMemcpyAsync(g.rows.features_old, s.rows.features_old, s.bytes(kRowFeatures, W), cudaMemcpyDeviceToDevice, ctx->stream));
        }
        give_source_rows(ctx, t, s.capacity, s.rows);
        s.rows = g.rows;
        s.capacity = g.capacity;
    }
    if (!copies.empty()) {
        std::vector<SourceRows> rows;
        for (const SourceTypeBatch& s : all) rows.push_back(s.lane_rows());
        const size_t n = copies.size();
        TRY(upload_table(ctx, "change_sources", ctx->change_sources, rows, 0));
        TRY(upload_table(ctx, "change_copies", ctx->change_copies, copies, 0));
        CK(ctx->change_records.reserve(n * 256));
        CK(ctx->change_features.reserve(n * 16));
        int64_t bytes = (int64_t)(n * sizeof(LaneCopy));
        const bool features = remove || feature_ids;
        if (remove) {
            launch_gather_lanes(ctx->change_sources.as<SourceRows>(), ctx->change_copies.as<LaneCopy>(), (int)n, W, ctx->change_records.as<int32_t>(),
                                ctx->change_features.as<int32_t>(), ctx->stream);
        } else {
            // an add entry writes one new lane, so copy i is entry copies[i].src_index
            std::vector<int32_t> staged(n * 64), staged_features(feature_ids ? n * 4 : 0);
            for (size_t i = 0; i < n; ++i) {
                const size_t entry = (size_t)copies[i].src_index;
                std::memcpy(staged.data() + i * 64, records + entry * 64, 256);
                if (feature_ids) std::memcpy(staged_features.data() + i * 4, feature_ids + entry * 4, 16);
            }
            CK(cudaMemcpyAsync(ctx->change_records.ptr, staged.data(), n * 256, cudaMemcpyHostToDevice, ctx->stream));
            if (feature_ids) CK(cudaMemcpyAsync(ctx->change_features.ptr, staged_features.data(), n * 16, cudaMemcpyHostToDevice, ctx->stream));
            bytes += (int64_t)n * (256 + (feature_ids ? 16 : 0));
        }
        launch_scatter_lanes(ctx->change_sources.as<SourceRows>(), ctx->change_copies.as<LaneCopy>(), (int)n, W, ctx->change_records.as<int32_t>(),
                             features ? ctx->change_features.as<int32_t>() : nullptr, ctx->stream);
        CK(cudaGetLastError());
        ctx->h2d_accum += bytes;
    }
    // every source takes what the replay left it; an emptied one leaves, and stream order keeps this call's copies ahead of any reuse of its rows
    for (size_t i = 0; i < all.size(); ++i) {
        SourceTypeBatch& s = all[i];
        s.host = std::move(next.sources[i]);
        if (took_add[i]) s.host_impulses = nullptr;
        if (s.host.type_batch_index >= 0) ctx->sources.push_back(std::move(s));
        else give_source_rows(ctx, s.type(), s.capacity, s.rows);
    }
    ctx->batch_count = next.batch_count;
    ctx->kinematics.assign(kinematics, kinematics + kinematic_count);
    ctx->prestep_writes.clear();
    return plan_device_rows(ctx);
}

int32_t bepucuda_add_constraints(bepucuda_ctx* ctx, int32_t count, const bepucuda_constraint_location* locations, const int32_t* records, const int32_t* feature_ids,
                                 const int32_t* constrained_kinematics, int32_t kinematic_count) {
    if (!ctx) return BEPUCUDA_ERR_INVALID_ARGUMENT;
    return change_constraints(ctx, "add_constraints", false, count, locations, records, feature_ids, constrained_kinematics, kinematic_count);
}

int32_t bepucuda_remove_constraints(bepucuda_ctx* ctx, int32_t count, const bepucuda_constraint_location* locations, const int32_t* constrained_kinematics,
                                    int32_t kinematic_count) {
    if (!ctx) return BEPUCUDA_ERR_INVALID_ARGUMENT;
    return change_constraints(ctx, "remove_constraints", true, count, locations, nullptr, nullptr, constrained_kinematics, kinematic_count);
}

int32_t bepucuda_add_bodies(bepucuda_ctx* ctx, const void* body_dynamics, int32_t count, const bepucuda_body_shape* shapes, const float* accelerations) {
    if (!ctx) return BEPUCUDA_ERR_INVALID_ARGUMENT;
    TRY(check_graph_edit(ctx, "add_bodies", "bodies"));
    if (count < 0 || (count > 0 && !body_dynamics)) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "add_bodies: bad arguments");
    if ((int64_t)ctx->body_count + count > (int64_t)kRefIndexMask) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "add_bodies: too many bodies");
    if (count == 0) return BEPUCUDA_OK;
    CK(cudaSetDevice(ctx->device));
    const int first = ctx->body_count;
    const size_t n = (size_t)first + count, added = (size_t)count;
    // Room for n bodies in every per-body array, the accelerations and shapes included when they are set for the current count. B is refreshed
    // whether or not this succeeds: a failed growth leaves the arrays it grew, records and all.
    cudaError_t e = ctx->bodies.grow(n, (size_t)first, ctx->stream);
    if (e == cudaSuccess && ctx->accelerations_count == first) e = ctx->accelerations.grow(n * 32, (size_t)first * 32, ctx->stream);
    if (e == cudaSuccess && ctx->shape_count == first) e = ctx->body_shapes.grow(n * sizeof(BodyShape), (size_t)first * sizeof(BodyShape), ctx->stream);
    refresh_body_buffers(ctx);
    if (e != cudaSuccess) return cuda_fail(ctx, e, "add_bodies: body arrays");
    ctx->upload_window.start_once(ctx->stream);
    int64_t bytes = (int64_t)added * 128;
    CK(cudaMemcpyAsync(ctx->bodies.raw.as<char>() + (size_t)first * 128, body_dynamics, added * 128, cudaMemcpyHostToDevice, ctx->stream));
    // the appended range through the describe's split, and "unconstrained" until a plan says otherwise
    BodyBuffers appended = ctx->B;
    for (float4** p : {&appended.pose, &appended.velocity, &appended.inertia_local, &appended.inertia_world}) *p += (size_t)first * 2;
    launch_split_bodies(ctx->bodies.raw.as<char>() + (size_t)first * 128, count, appended, ctx->stream);
    launch_fill_i32(ctx->bodies.first_batch.as<int32_t>() + first, added, 0x7fffffff, ctx->stream);
    CK(cudaMemsetAsync(ctx->bodies.constrained.as<uint8_t>() + first, 0, added, ctx->stream));
    CK(cudaGetLastError());
    if (ctx->accelerations_count == first && accelerations) {
        CK(cudaMemcpyAsync(ctx->accelerations.as<char>() + (size_t)first * 32, accelerations, added * 32, cudaMemcpyHostToDevice, ctx->stream));
        ctx->accelerations_count = (int)n;
        bytes += (int64_t)added * 32;
    }
    if (ctx->shape_count == first && shapes) {
        CK(cudaMemcpyAsync(ctx->body_shapes.as<char>() + (size_t)first * sizeof(BodyShape), shapes, added * sizeof(BodyShape), cudaMemcpyHostToDevice, ctx->stream));
        ctx->shape_count = (int)n;
        bytes += (int64_t)(added * sizeof(BodyShape));
    }
    ctx->h2d_accum += bytes;
    ctx->body_count = (int)n;
    refresh_body_buffers(ctx);
    return upload_program(ctx);  // the final pose pass covers the new bodies
}

int32_t bepucuda_remove_bodies(bepucuda_ctx* ctx, int32_t count, const int32_t* body_indices) {
    if (!ctx) return BEPUCUDA_ERR_INVALID_ARGUMENT;
    TRY(check_graph_edit(ctx, "remove_bodies", "bodies"));
    const int old = ctx->body_count;
    int32_t final_count = old;
    std::vector<int32_t> moved_to;
    std::string error;
    if (replay_body_removes(old, count, body_indices, &final_count, &moved_to, &error) != BEPUCUDA_OK)
        return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "remove_bodies: " + error);
    if (count == 0) return BEPUCUDA_OK;
    CK(cudaSetDevice(ctx->device));
    CK(ctx->moved_to.reserve((size_t)count * 4));
    CK(ctx->removed_marks.reserve((size_t)old));
    ctx->upload_window.start_once(ctx->stream);
    CK(cudaMemcpyAsync(ctx->moved_to.ptr, moved_to.data(), (size_t)count * 4, cudaMemcpyHostToDevice, ctx->stream));
    ctx->h2d_accum += (int64_t)count * 4;
    // Bodies.RemoveAt forbids orphans: no live constraint may reference a removed body. Checked before anything moves.
    int32_t* flag = ctx->error_dev.as<int32_t>();
    CK(cudaMemsetAsync(ctx->removed_marks.ptr, 0, (size_t)old, ctx->stream));
    CK(cudaMemsetAsync(flag, 0, 4, ctx->stream));
    launch_mark_removed_bodies(ctx->moved_to.as<int32_t>(), count, final_count, ctx->removed_marks.as<uint8_t>(), ctx->stream);
    launch_check_removed_references(ctx->tb_table.as<DeviceTypeBatch>(), ctx->work_table.as<WorkItem>(), ctx->topo.all_work_count, ctx->removed_marks.as<uint8_t>(), old, flag,
                                    ctx->stream);
    CK(cudaGetLastError());
    int32_t referenced = 0;
    CK(cudaMemcpyAsync(&referenced, flag, 4, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    if (referenced) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "remove_bodies: a live constraint references a removed body; remove its constraints first");

    std::vector<RefSpan> spans;
    int64_t max_words = 0;
    for (const SourceTypeBatch& s : ctx->sources) {
        spans.push_back(s.ref_span(ctx->W));
        max_words = std::max(max_words, spans.back().words);
    }
    TRY(upload_table(ctx, "ref_spans", ctx->ref_spans, spans, 0));
    TRY(rows_to_sources(ctx));
    const BodyRecords records{ctx->bodies.raw.as<float4>(), ctx->B, ctx->accelerations_count == old ? ctx->accelerations.as<float4>() : nullptr,
                              ctx->shape_count == old ? ctx->body_shapes.as<float4>() : nullptr};
    launch_move_bodies(records, ctx->moved_to.as<int32_t>(), count, final_count, ctx->stream);
    launch_remap_body_references(ctx->ref_spans.as<RefSpan>(), (int)spans.size(), max_words, ctx->moved_to.as<int32_t>(), count, final_count, ctx->stream);
    CK(cudaGetLastError());
    // the same moves on the host's copies: fallback references (levelisation) and constrained kinematics (a removed one leaves the list)
    auto new_index = [&](int32_t idx) { return idx < final_count || idx >= old ? idx : moved_to[(size_t)(idx - final_count)]; };
    for (SourceTypeBatch& s : ctx->sources)
        for (int32_t& r : s.host.refs)
            if (r >= 0) {
                const int32_t to = new_index((int32_t)((uint32_t)r & kRefIndexMask));
                if (to >= 0) r = (int32_t)(((uint32_t)r & kRefKinematicBit) | (uint32_t)to);
            }
    std::vector<uint8_t> taken((size_t)final_count, 0);  // slots whose body was removed (a moved body took them)
    for (const int32_t to : moved_to)
        if (to >= 0) taken[(size_t)to] = 1;
    std::vector<int32_t> kinematics;
    for (const int32_t k : ctx->kinematics) {
        const int32_t to = k < final_count ? (taken[(size_t)k] ? -1 : k) : new_index(k);
        if (to >= 0) kinematics.push_back(to);
    }
    ctx->kinematics = std::move(kinematics);
    if (ctx->accelerations_count == old) ctx->accelerations_count = final_count;
    if (ctx->shape_count == old) ctx->shape_count = final_count;
    ctx->body_count = final_count;
    refresh_body_buffers(ctx);
    return plan_device_rows(ctx);
}

int32_t bepucuda_get_timings(bepucuda_ctx* ctx, bepucuda_timings* out) {
    if (!ctx || !out) return BEPUCUDA_ERR_INVALID_ARGUMENT;
    CK(cudaSetDevice(ctx->device));
    CK(cudaStreamSynchronize(ctx->stream));
    TRY(check_device_error_flag(ctx));
    ctx->solve_window.measure(&ctx->timings.solve_ms);
    ctx->upload_window.measure(&ctx->timings.upload_ms);
    ctx->download_window.measure(&ctx->timings.download_ms);
    *out = ctx->timings;
    return BEPUCUDA_OK;
}

int32_t bepucuda_event_record(bepucuda_ctx* ctx, int32_t slot) {
    if (!ctx || slot < 0 || slot >= 16) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "event_record: bad slot");
    CK(cudaSetDevice(ctx->device));
    CK(ctx->user_events[slot].create());
    CK(cudaEventRecord(ctx->user_events[slot], ctx->stream));
    return BEPUCUDA_OK;
}
int32_t bepucuda_event_elapsed_ms(bepucuda_ctx* ctx, int32_t a, int32_t b, float* ms) {
    if (!ctx || !ms || a < 0 || a >= 16 || b < 0 || b >= 16 || !ctx->user_events[a] || !ctx->user_events[b]) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "event_elapsed_ms: bad slots");
    CK(cudaSetDevice(ctx->device));
    CK(cudaEventSynchronize(ctx->user_events[b]));
    CK(cudaEventElapsedTime(ms, ctx->user_events[a], ctx->user_events[b]));
    return BEPUCUDA_OK;
}

int32_t bepucuda_profile_stages(bepucuda_ctx* ctx, float dt, bepucuda_stage_profile* out) {
    if (!ctx || !out || !(dt > 0)) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "profile_stages: bad arguments");
    if (!ctx->constraints_ready) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "profile_stages before end_constraints");
    if (ctx->peer_mode) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "profile_stages in peer mode: one rank alone cannot meet its peers at the rank barriers");
    TRY(check_accelerations(ctx, "profile_stages"));
    CK(cudaSetDevice(ctx->device));
    std::memset(out, 0, sizeof(*out));
    ctx->profile_events.resize(std::max(ctx->profile_events.size(), ctx->program.ops.size() * 2));
    for (Event& ev : ctx->profile_events) CK(ev.create());
    TRY(prepare_frame(ctx, dt));
    std::vector<int> launched(ctx->program.ops.size(), 0);
    const StageEvents sink{ctx->profile_events, launched};
    issue_stage_sequence(ctx, ctx->stream, nullptr, &sink);
    CK(cudaStreamSynchronize(ctx->stream));
    CK(cudaGetLastError());
    for (size_t i = 0; i < ctx->program.ops.size(); ++i) {
        if (!launched[i]) continue;
        float ms = 0;
        CK(cudaEventElapsedTime(&ms, ctx->profile_events[2 * i], ctx->profile_events[2 * i + 1]));
        const StageOp& op = ctx->program.ops[i];
        out->ms[op.stage] += ms;
        out->launches[op.stage] += 1;
        out->algorithmic_bytes[op.stage] += op.algorithmic_bytes;
    }
    return BEPUCUDA_OK;
}

static_assert(sizeof(bepucuda_body_shape) == sizeof(BodyShape) && sizeof(bepucuda_body_activity) == sizeof(BodyActivityRecord) && sizeof(BodyActivityRecord) == 8, "ABI structs mirror the device records");

int32_t bepucuda_set_body_shapes(bepucuda_ctx* ctx, const bepucuda_body_shape* shapes, int32_t body_count) {
    if (!ctx || body_count < 0 || (body_count > 0 && !shapes)) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "set_body_shapes: bad arguments");
    CK(cudaSetDevice(ctx->device));
    CK(ctx->body_shapes.reserve((size_t)std::max(body_count, 1) * sizeof(BodyShape)));
    if (body_count > 0) CK(cudaMemcpyAsync(ctx->body_shapes.ptr, shapes, (size_t)body_count * sizeof(BodyShape), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));  // the caller's buffer is only guaranteed for the duration of the call
    ctx->shape_count = body_count;
    return BEPUCUDA_OK;
}

int32_t bepucuda_predict_bounding_boxes(bepucuda_ctx* ctx, float dt, bepucuda_body_activity* activities, float* bounds_out) {
    if (!ctx || !(dt > 0) || !activities || !bounds_out) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "predict_bounding_boxes: bad arguments");
    if (ctx->shape_count != ctx->body_count) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "predict_bounding_boxes: bepucuda_set_body_shapes was not called for the current body count");
    TRY(check_accelerations(ctx, "predict_bounding_boxes"));
    const int n = ctx->body_count;
    if (n == 0) return BEPUCUDA_OK;
    CK(cudaSetDevice(ctx->device));
    CK(ctx->body_activities.reserve((size_t)n * sizeof(BodyActivityRecord)));
    CK(ctx->body_bounds.reserve((size_t)n * 32));
    CK(cudaMemcpyAsync(ctx->body_activities.ptr, activities, (size_t)n * sizeof(BodyActivityRecord), cudaMemcpyHostToDevice, ctx->stream));
    // PoseIntegrator.PredictBoundingBoxes calls Callbacks.PrepareForIntegration(dt) with the frame dt (PoseIntegrator.cs:L428)
    const IntegrationTerms t = prepare_for_integration(ctx, dt);
    PredictParams p{};
    p.dt = dt;
    for (int i = 0; i < 3; ++i) p.gravity_dt[i] = t.gravity_dt[i];
    p.linear_damping_dt = t.linear_damping_dt;
    p.angular_damping_dt = t.angular_damping_dt;
    p.integrate_velocity_for_kinematics = ctx->integ.integrate_velocity_for_kinematics;
    p.integrate_extensions = integrate_extensions(ctx);
    p.accelerations = (p.integrate_extensions & kIntegrateAccelerations) ? ctx->accelerations.as<float4>() : nullptr;
    for (int i = 0; i < 3; ++i) p.attractor_center[i] = ctx->attractor_center[i];
    p.attractor_dt = t.attractor_dt;
    launch_predict_bounding_boxes(ctx->B, ctx->body_shapes.as<BodyShape>(), ctx->body_activities.as<BodyActivityRecord>(), ctx->body_bounds.as<float4>(), p, ctx->stream);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(activities, ctx->body_activities.ptr, (size_t)n * sizeof(BodyActivityRecord), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(bounds_out, ctx->body_bounds.ptr, (size_t)n * 32, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return BEPUCUDA_OK;
}

uint32_t bepucuda_color_hash(uint32_t constraint_index) { return color_hash(constraint_index); }

int32_t bepucuda_color_constraints(bepucuda_ctx* ctx, int32_t constraint_count, int32_t bodies_per_constraint, const int32_t* encoded_body_references, int32_t body_count,
                                   int32_t fallback_batch_threshold, int32_t order, const uint32_t* priorities, int32_t* batch_indices_out, int32_t* batch_count_out,
                                   int32_t* rounds_out) {
    if (!ctx) return BEPUCUDA_ERR_INVALID_ARGUMENT;
    if (constraint_count < 0 || bodies_per_constraint < 1 || bodies_per_constraint > 4 || body_count < 0 || fallback_batch_threshold < 1 || fallback_batch_threshold > 64)
        return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "color_constraints: counts out of range (1..4 body slots, fallback threshold 1..64)");
    if (order < BEPUCUDA_COLOR_INSERTION_ORDER || order > BEPUCUDA_COLOR_BY_PRIORITY || (order == BEPUCUDA_COLOR_BY_PRIORITY && !priorities))
        return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "color_constraints: unknown order, or BEPUCUDA_COLOR_BY_PRIORITY without priorities");
    if (constraint_count > 0 && (!encoded_body_references || !batch_indices_out)) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "color_constraints: null buffer");
    if (batch_count_out) *batch_count_out = 0;
    if (rounds_out) *rounds_out = 0;
    if (constraint_count == 0) return BEPUCUDA_OK;
    CK(cudaSetDevice(ctx->device));
    // body references are validated on the host while they are being staged (one pass over memory the copy touches anyway)
    const size_t words = (size_t)constraint_count * bodies_per_constraint;
    for (size_t i = 0; i < words; ++i) {
        const int32_t enc = encoded_body_references[i];
        if (enc >= 0 && (int32_t)((uint32_t)enc & ((1u << 30) - 1u)) >= body_count) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "color_constraints: body reference out of range");
    }
    int64_t rounds = 0;
    const char* failed = nullptr;
    if (const cudaError_t e = color_constraints(ctx->coloring, constraint_count, bodies_per_constraint, encoded_body_references, body_count, fallback_batch_threshold, order,
                                                order == BEPUCUDA_COLOR_BY_PRIORITY ? priorities : nullptr, batch_indices_out, &rounds, &failed, ctx->stream))
        return cuda_fail(ctx, e, failed);
    if (rounds < 0) return fail(ctx, BEPUCUDA_ERR_CUDA, "color_constraints: no progress (internal error)");
    int32_t highest = -1;
    for (int32_t i = 0; i < constraint_count; ++i) highest = std::max(highest, batch_indices_out[i]);
    if (batch_count_out) *batch_count_out = highest + 1;
    if (rounds_out) *rounds_out = (int32_t)std::min<int64_t>(rounds, 0x7fffffff);
    return BEPUCUDA_OK;
}

int32_t bepucuda_find_sleepable_islands(bepucuda_ctx* ctx, const bepucuda_body_activity* activities, int32_t body_count, int32_t* island_of_body_out,
                                        int32_t* sleepable_roots_out, int32_t* sleepable_body_counts_out, int32_t* sleepable_count_out, int32_t* rounds_out) {
    if (!ctx) return BEPUCUDA_ERR_INVALID_ARGUMENT;
    if (ctx->peer_mode) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "find_sleepable_islands in peer mode: a rank holds only its own constraints and cannot see whole islands");
    if (!ctx->constraints_ready) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "find_sleepable_islands before end_constraints");
    if (body_count != ctx->body_count) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "find_sleepable_islands: the body count must match the last upload_bodies");
    if (!sleepable_count_out || (body_count > 0 && (!activities || !sleepable_roots_out || !sleepable_body_counts_out)))
        return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "find_sleepable_islands: null buffer");
    *sleepable_count_out = 0;
    if (rounds_out) *rounds_out = 0;
    if (body_count == 0) return BEPUCUDA_OK;
    CK(cudaSetDevice(ctx->device));
    int64_t rounds = 0;
    const char* failed = nullptr;
    if (const cudaError_t e = find_sleepable_islands(ctx->islands, ctx->tb_table.as<DeviceTypeBatch>(), ctx->work_table.as<WorkItem>(), ctx->topo.all_work_count, activities, body_count,
                                                     island_of_body_out, sleepable_roots_out, sleepable_body_counts_out, sleepable_count_out, &rounds, &failed, ctx->stream))
        return cuda_fail(ctx, e, failed);
    if (rounds < 0) return fail(ctx, BEPUCUDA_ERR_CUDA, "find_sleepable_islands: no convergence (internal error)");
    if (rounds_out) *rounds_out = (int32_t)std::min<int64_t>(rounds, 0x7fffffff);
    return BEPUCUDA_OK;
}

int32_t bepucuda_shard_export(bepucuda_ctx* ctx, bepucuda_ipc_handles* out) {
    if (!ctx || !out) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "shard_export: bad arguments");
    if (ctx->body_count <= 0) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "shard_export before upload_bodies");
    CK(cudaSetDevice(ctx->device));
    CK(ctx->shard_flags.reserve(kShardFlagBlockWords * sizeof(unsigned long long)));  // barrier flags, arrival counters and targets (ShardStage)
    CK(cudaMemset(ctx->shard_flags.ptr, 0, kShardFlagBlockWords * sizeof(unsigned long long)));
    void* ptrs[4] = {ctx->bodies.pose.ptr, ctx->bodies.velocity.ptr, ctx->bodies.inertia_world.ptr, ctx->shard_flags.ptr};
    for (int i = 0; i < 4; ++i) {
        cudaIpcMemHandle_t h;
        CK(cudaIpcGetMemHandle(&h, ptrs[i]));
        static_assert(sizeof(h) == 64, "cudaIpcMemHandle_t is 64 bytes");
        std::memcpy(out->bytes[i], &h, 64);
    }
    return BEPUCUDA_OK;
}

// The end of both shard imports: the context runs as rank p.rank of p.rank_count from its next describe on.
static int enter_peer_mode(bepucuda_ctx* ctx, const ShardPeers& p) {
    ctx->peers = p;
    ctx->peer_mode = true;
    ctx->exchange_counter = 0;
    ctx->constraints_ready = false;
    return BEPUCUDA_OK;
}

int32_t bepucuda_shard_import(bepucuda_ctx* ctx, int32_t rank, int32_t rank_count, const bepucuda_ipc_handles* all) {
    if (!ctx || !all || rank_count < 1 || rank_count > kMaxShardRanks || rank < 0 || rank >= rank_count) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "shard_import: bad arguments");
    if (!ctx->shard_flags.ptr) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "shard_import before shard_export");
    CK(cudaSetDevice(ctx->device));
    ShardPeers p{};
    p.rank = rank;
    p.rank_count = rank_count;
    for (int r = 0; r < rank_count; ++r) {
        void* ptrs[4] = {ctx->bodies.pose.ptr, ctx->bodies.velocity.ptr, ctx->bodies.inertia_world.ptr, ctx->shard_flags.ptr};
        if (r != rank)
            for (int i = 0; i < 4; ++i) {
                cudaIpcMemHandle_t h;
                std::memcpy(&h, all[r].bytes[i], 64);
                CK(cudaIpcOpenMemHandle(ctx->opened_ipc.emplace_back().put(), h, cudaIpcMemLazyEnablePeerAccess));
                ptrs[i] = ctx->opened_ipc.back();
            }
        p.pose[r] = (float4*)ptrs[0];
        p.velocity[r] = (float4*)ptrs[1];
        p.inertia_world[r] = (float4*)ptrs[2];
        p.flags[r] = (unsigned long long*)ptrs[3];
    }
    return enter_peer_mode(ctx, p);
}

int32_t bepucuda_shard_import_contexts(bepucuda_ctx* ctx, int32_t rank, int32_t rank_count, bepucuda_ctx* const* all) {
    if (!ctx || !all || rank_count < 1 || rank_count > kMaxShardRanks || rank < 0 || rank >= rank_count || all[rank] != ctx)
        return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "shard_import_contexts: bad arguments");
    CK(cudaSetDevice(ctx->device));
    ShardPeers p{};
    p.rank = rank;
    p.rank_count = rank_count;
    for (int r = 0; r < rank_count; ++r) {
        bepucuda_ctx* o = all[r];
        if (!o || !o->shard_flags.ptr || o->body_count != ctx->body_count) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "shard_import_contexts: every context needs the same bodies and a shard_export");
        if (o->device != ctx->device) {
            int can = 0;
            CK(cudaDeviceCanAccessPeer(&can, ctx->device, o->device));
            if (!can) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "shard_import_contexts: no peer access between the devices");
            cudaError_t e = cudaDeviceEnablePeerAccess(o->device, 0);
            if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) CK(e);
            (void)cudaGetLastError();
        }
        p.pose[r] = o->bodies.pose.as<float4>();
        p.velocity[r] = o->bodies.velocity.as<float4>();
        p.inertia_world[r] = o->bodies.inertia_world.as<float4>();
        p.flags[r] = (unsigned long long*)o->shard_flags.ptr;
    }
    return enter_peer_mode(ctx, p);
}

int32_t bepucuda_shard_set_global(bepucuda_ctx* ctx, const int32_t* first_batch, const uint8_t* constrained) {
    if (!ctx || !first_batch || !constrained) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "shard_set_global: bad arguments");
    ctx->global_first_batch.assign(first_batch, first_batch + ctx->body_count);
    ctx->global_constrained.assign(constrained, constrained + ctx->body_count);
    ctx->constraints_ready = false;
    return BEPUCUDA_OK;
}

int32_t bepucuda_shard_set_body_masks(bepucuda_ctx* ctx, const uint8_t* rank_masks) {
    if (!ctx || !rank_masks) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "shard_set_body_masks: bad arguments");
    ctx->body_masks.assign(rank_masks, rank_masks + ctx->body_count);
    ctx->constraints_ready = false;
    return BEPUCUDA_OK;
}

int32_t bepucuda_shard_set_fallback_rank(bepucuda_ctx* ctx, int32_t rank) {
    if (!ctx) return BEPUCUDA_ERR_INVALID_ARGUMENT;
    if (!ctx->peer_mode) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "shard_set_fallback_rank: the context is not in peer mode (bepucuda_shard_import*)");
    if (rank < -1 || rank >= ctx->peers.rank_count) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "shard_set_fallback_rank: rank out of range");
    ctx->fallback_rank = rank;
    ctx->constraints_ready = false;
    return BEPUCUDA_OK;
}

}  // extern "C"
