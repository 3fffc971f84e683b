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
#include "bepu_topology.h"

using namespace bepucuda;

namespace bepucuda {

// ---- small RAII helpers ------------------------------------------------------------------------------------------------------
// Memory that grows on demand (contents are not kept) and is freed with its owner: device memory, or page-locked host memory.
template <bool kPinnedHost> struct GrowBuffer {
    void* ptr = nullptr;
    size_t capacity = 0;
    GrowBuffer() = default;
    GrowBuffer(const GrowBuffer&) = delete;
    GrowBuffer& operator=(const GrowBuffer&) = delete;
    ~GrowBuffer() { release(); }
    cudaError_t reserve(size_t bytes) {
        if (bytes <= capacity) return cudaSuccess;
        release();
        size_t want = bytes + bytes / 4 + 256;
        cudaError_t e = kPinnedHost ? cudaMallocHost(&ptr, want) : cudaMalloc(&ptr, want);
        if (e == cudaSuccess) capacity = want;
        else ptr = nullptr;
        return e;
    }
    void release() {
        if (ptr) kPinnedHost ? cudaFreeHost(ptr) : cudaFree(ptr);
        ptr = nullptr;
        capacity = 0;
    }
    template <class T> T* as() const { return (T*)ptr; }
};
using DeviceBuffer = GrowBuffer<false>;
using PinnedBuffer = GrowBuffer<true>;

// Bump allocator over chunks that are never reallocated (uploads are enqueued against their addresses).
struct ChunkArena {
    struct Chunk { char* base; size_t size, used; };
    std::vector<Chunk> chunks;
    bool pinned_host = false;
    size_t min_chunk = (size_t)64 << 20;
    ChunkArena() = default;
    ChunkArena(const ChunkArena&) = delete;
    ChunkArena& operator=(const ChunkArena&) = delete;
    ~ChunkArena() {
        for (auto& c : chunks) { if (pinned_host) cudaFreeHost(c.base); else cudaFree(c.base); }
    }
    void reset() { for (auto& c : chunks) c.used = 0; }
    void* alloc(size_t bytes, cudaError_t* err) {
        bytes = (bytes + 255) & ~(size_t)255;
        for (auto& c : chunks)
            if (c.size - c.used >= bytes) {
                void* p = c.base + c.used;
                c.used += bytes;
                return p;
            }
        Chunk c{};
        c.size = std::max(bytes, min_chunk);
        cudaError_t e = pinned_host ? cudaMallocHost((void**)&c.base, c.size) : cudaMalloc((void**)&c.base, c.size);
        if (e != cudaSuccess) { if (err) *err = e; return nullptr; }
        c.used = bytes;
        chunks.push_back(c);
        return chunks.back().base;
    }
};

// Pinned copy of a host buffer that the caller may reuse as soon as the upload is enqueued, and the event after which the copy has read it.
struct StagedUpload {
    PinnedBuffer host;
    cudaEvent_t done = nullptr;
};

struct SourceTypeBatch {
    int batch_index, type_batch_index, type_id, count;
    float* host_impulses;
    int32_t* raw_refs;     // device, reference AOSOA-W layout
    float* raw_prestep;
    float* raw_impulses;
    size_t refs_bytes, prestep_bytes, impulse_bytes;
    std::vector<int32_t> host_refs;  // retained only for fallback batches (levelisation)
    // device-side contact update (bepucuda_update_contacts): feature ids of the resident impulses / of the frame being uploaded
    int32_t* raw_features_old = nullptr;
    int32_t* raw_features_new = nullptr;
    size_t feature_bytes = 0;
    // rows uploaded since the last transposition (kTransposePrestep / kTransposeImpulses): refresh_device_rows transposes only these, so the rows
    // of every other type batch, the accumulated impulses in particular, stay as the last solve left them on the device
    int32_t pending = 0;
    bool redistribute = false;
};

}  // namespace bepucuda

struct bepucuda_ctx {
    bepucuda_config cfg{};
    int device = 0;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev_solve_begin = nullptr, ev_solve_end = nullptr, ev_up_begin = nullptr, ev_up_end = nullptr, ev_down_begin = nullptr, ev_down_end = nullptr;
    bool up_open = false, have_solve = false, have_down = false, have_up = false;
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
    DeviceBuffer raw_bodies, pose, velocity, inertia_local, inertia_world, constrained, first_batch, sync_refcount, sync_mask;
    BodyBuffers B{};

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
    std::vector<void*> opened_ipc;
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

    // the captured stage sequence of the program (dropped when the program is replaced), and what its launches bake in besides the program
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t graph_exec = nullptr;
    BodyBuffers graph_bodies{};
    LaunchContext graph_launch{};

    bepucuda_timings timings{};
    int64_t h2d_accum = 0;
    struct HostRange { char* host; size_t bytes; char* dev; };
    std::vector<HostRange> host_ranges;    // page-locked + device-mapped host memory registered through bepucuda_host_register
    std::vector<CopyChunk> pending_h2d;    // batched copies waiting for the next flush
    DeviceBuffer chunk_table;
    StagedUpload chunk_stage[4];           // pinned ring for chunk tables
    int chunk_stage_next = 0;
    cudaEvent_t user_events[16] = {};
    DeviceBuffer body_shapes, body_activities, body_bounds;  // bepucuda_set_body_shapes / bepucuda_predict_bounding_boxes
    int shape_count = -1;
    DeviceBuffer color_refs, color_priorities, color_body_min, color_body_mask, color_out, color_lists, color_counts;  // bepucuda_color_constraints
    DeviceBuffer island_activities, island_label, island_blocked, island_count, island_flags, island_roots, island_counts, island_scalars, island_temp;  // bepucuda_find_sleepable_islands
    DeviceBuffer inverse_table, read_requests, read_records;  // bepucuda_read_constraints: the plan's inverse slot map, one call's requests and records
    PrestepWriteQueue prestep_writes;  // bepucuda_write_constraints since the last solve, applied by refresh_device_rows
    DeviceBuffer write_table, write_rows;
    StagedUpload write_stage, write_rows_stage;
    std::vector<cudaEvent_t> profile_events;
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

void open_upload_window(bepucuda_ctx* ctx) {
    if (!ctx->up_open) {
        cudaEventRecord(ctx->ev_up_begin, ctx->stream);
        ctx->up_open = true;
    }
}

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
// H2D copy of `bytes` at `src` through the pinned staging buffer of `st`.
int upload_staged(bepucuda_ctx* ctx, StagedUpload& st, void* dst, const void* src, size_t bytes) {
    if (!st.done) CK(cudaEventCreateWithFlags(&st.done, cudaEventDisableTiming));
    CK(cudaEventSynchronize(st.done));  // the previous upload has left the staging buffer
    CK(st.host.reserve(bytes));
    std::memcpy(st.host.ptr, src, bytes);
    CK(cudaMemcpyAsync(dst, st.host.ptr, bytes, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaEventRecord(st.done, ctx->stream));
    return BEPUCUDA_OK;
}

// Runs the queued chunks as one kernel. The chunk table travels through a ring of pinned staging buffers.
int flush_chunks(bepucuda_ctx* ctx, std::vector<CopyChunk>& list) {
    if (list.empty()) return BEPUCUDA_OK;
    const size_t bytes = list.size() * sizeof(CopyChunk);
    CK(ctx->chunk_table.reserve(bytes));
    StagedUpload& st = ctx->chunk_stage[ctx->chunk_stage_next];
    ctx->chunk_stage_next = (ctx->chunk_stage_next + 1) & 3;
    // The device-side table is reused by every flush: stream order keeps the previous batched copy ahead of this overwrite.
    { int rc = upload_staged(ctx, st, ctx->chunk_table.ptr, list.data(), bytes); if (rc != BEPUCUDA_OK) return rc; }
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

SourceTypeBatch* find_source(bepucuda_ctx* ctx, int32_t batch_index, int32_t type_batch_index) {
    for (auto& s : ctx->sources)
        if (s.batch_index == batch_index && s.type_batch_index == type_batch_index) return &s;
    return nullptr;
}

void invalidate_graph(bepucuda_ctx* ctx) {
    if (ctx->graph_exec) cudaGraphExecDestroy(ctx->graph_exec);
    if (ctx->graph) cudaGraphDestroy(ctx->graph);
    ctx->graph_exec = nullptr;
    ctx->graph = nullptr;
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
bool same_bodies(const BodyBuffers& a, const BodyBuffers& b) {
    return a.pose == b.pose && a.velocity == b.velocity && a.inertia_local == b.inertia_local && a.inertia_world == b.inertia_world && a.constrained == b.constrained &&
           a.first_batch == b.first_batch && a.count == b.count;
}

// Profiling sink of issue_stage_sequence: the launch of program op i sets launched[i] and is bracketed by events[2i] and events[2i + 1].
struct StageEvents {
    const std::vector<cudaEvent_t>& events;
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
    invalidate_graph(ctx);
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
    { int rc = flush_chunks(ctx, ctx->pending_h2d); if (rc != BEPUCUDA_OK) return rc; }
    bool any_pending = false, any_redistribute = false, descs_changed = false;
    for (size_t tb = 0; tb < ctx->topo.tbs.size(); ++tb) {
        const SourceTypeBatch& s = ctx->sources[(size_t)ctx->topo.tbs[tb].source];
        TransposeDesc& d = ctx->tdescs[tb];
        const int32_t flags = s.pending | (s.redistribute ? kDescRedistribute : 0);
        if (d.flags != flags || d.features_old != s.raw_features_old || d.features_new != s.raw_features_new) {
            d.flags = flags;
            d.features_old = s.raw_features_old;
            d.features_new = s.raw_features_new;
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
        { int rc = upload_staged(ctx, ctx->write_stage, ctx->write_table.ptr, q.writes.data(), bytes); if (rc != BEPUCUDA_OK) return rc; }
        { int rc = upload_staged(ctx, ctx->write_rows_stage, ctx->write_rows.ptr, q.rows.data(), row_bytes); if (rc != BEPUCUDA_OK) return rc; }
        ctx->h2d_accum += (int64_t)(bytes + row_bytes);
        launch_write_constraints(ctx->tb_table.as<DeviceTypeBatch>(), ctx->tdesc_table.as<TransposeDesc>(), ctx->write_table.as<PrestepWrite>(), ctx->write_rows.as<float>(),
                                 (int)q.writes.size(), ctx->stream);
        q.clear();
    }
    for (SourceTypeBatch& s : ctx->sources) {
        if (s.redistribute) std::swap(s.raw_features_old, s.raw_features_new);  // the resident impulses now belong to the new ids
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
    { int rc = refresh_device_rows(ctx); if (rc != BEPUCUDA_OK) return rc; }
    if (ctx->up_open) {
        cudaEventRecord(ctx->ev_up_end, ctx->stream);
        ctx->up_open = false;
        ctx->have_up = true;
    }
    ctx->timings.h2d_bytes = ctx->h2d_accum;
    ctx->h2d_accum = 0;
    // frame parameters (previous solve's copy has completed by stream order only after its graph, a stage profile's before it returned; wait for
    // it before reusing the pinned struct)
    CK(cudaEventSynchronize(ctx->ev_solve_end));
    FrameParams* fp = ctx->frame_params_host.as<FrameParams>();
    compute_frame_params(ctx, dt, fp);
    fp->exchange_base = ctx->exchange_counter;
    fp->shard_solve_index = ctx->shard_solve_index;
    CK(cudaMemcpyAsync(ctx->frame_params_dev.ptr, fp, sizeof(FrameParams), cudaMemcpyHostToDevice, ctx->stream));
    return BEPUCUDA_OK;
}

}  // namespace

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
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking);
    cudaEvent_t* evs[] = {&ctx->ev_solve_begin, &ctx->ev_solve_end, &ctx->ev_up_begin, &ctx->ev_up_end, &ctx->ev_down_begin, &ctx->ev_down_end};
    for (auto ev : evs)
        if (e == cudaSuccess) e = cudaEventCreate(ev);
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
    invalidate_graph(ctx);
    for (void* p : ctx->opened_ipc) cudaIpcCloseMemHandle(p);
    cudaEvent_t evs[] = {ctx->ev_solve_begin, ctx->ev_solve_end, ctx->ev_up_begin, ctx->ev_up_end, ctx->ev_down_begin, ctx->ev_down_end, ctx->accelerations_stage.done};
    for (auto ev : evs)
        if (ev) cudaEventDestroy(ev);
    for (auto ev : ctx->user_events)
        if (ev) cudaEventDestroy(ev);
    for (auto& st : ctx->chunk_stage)
        if (st.done) cudaEventDestroy(st.done);
    for (auto ev : ctx->profile_events) cudaEventDestroy(ev);
    if (ctx->stream) cudaStreamDestroy(ctx->stream);
    delete ctx;  // the device and pinned buffers free themselves, on the device set above
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
    if (threshold_changed && ctx->constraints_ready) ctx->constraints_ready = false;  // fallback split must be redone
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
    open_upload_window(ctx);
    const size_t bytes = (size_t)body_count * 32;
    CK(ctx->accelerations.reserve(std::max(bytes, (size_t)32)));
    if (bytes > 0) {
        // through a pinned staging copy, so that the caller's buffer is free when the call returns without waiting for the device
        int rc = upload_staged(ctx, ctx->accelerations_stage, ctx->accelerations.ptr, accelerations, bytes);
        if (rc != BEPUCUDA_OK) return rc;
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
    open_upload_window(ctx);
    const size_t n = (size_t)body_count;
    // constrained flags / ownership depend on the body count; force a rebuild of topology products.
    if (body_count != ctx->body_count) ctx->constraints_ready = false;
    CK(ctx->raw_bodies.reserve(n * 128));
    CK(ctx->pose.reserve(n * 32));
    CK(ctx->velocity.reserve(n * 32));
    CK(ctx->inertia_local.reserve(n * 32));
    CK(ctx->inertia_world.reserve(n * 32));
    const size_t old_constrained_cap = ctx->constrained.capacity;
    CK(ctx->constrained.reserve(n + 1));
    if (ctx->constrained.capacity != old_constrained_cap) CK(cudaMemsetAsync(ctx->constrained.ptr, 0, ctx->constrained.capacity, ctx->stream));
    ctx->body_count = body_count;
    BodyBuffers B{};
    B.pose = ctx->pose.as<float4>();
    B.velocity = ctx->velocity.as<float4>();
    B.inertia_local = ctx->inertia_local.as<float4>();
    B.inertia_world = ctx->inertia_world.as<float4>();
    B.constrained = ctx->constrained.as<uint8_t>();
    B.first_batch = ctx->first_batch.as<int32_t>();
    B.count = body_count;
    ctx->B = B;
    if (body_count > 0) {
        CK(cudaMemcpyAsync(ctx->raw_bodies.ptr, body_dynamics, n * 128, cudaMemcpyHostToDevice, ctx->stream));
        ctx->h2d_accum += (int64_t)n * 128;
        launch_split_bodies(ctx->raw_bodies.ptr, body_count, ctx->B, ctx->stream);
        CK(cudaGetLastError());
    }
    return BEPUCUDA_OK;
}

int32_t bepucuda_begin_constraints(bepucuda_ctx* ctx, int32_t source_bundle_width, int32_t batch_count) {
    if (!ctx || source_bundle_width < 1 || source_bundle_width > 64 || batch_count < 0) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "begin_constraints: bad arguments");
    CK(cudaSetDevice(ctx->device));
    CK(cudaStreamSynchronize(ctx->stream));  // staging arenas are recycled below
    open_upload_window(ctx);
    ctx->W = source_bundle_width;
    ctx->batch_count = batch_count;
    ctx->sources.clear();
    ctx->pending_h2d.clear();  // queued refreshes target raw-arena addresses that are recycled below; a re-describe uploads everything anyway
    ctx->prestep_writes.clear();  // slots of the old plan; the describe uploads the host's prestep, which ApplyDescription already wrote
    ctx->raw_arena.reset();
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
    const size_t bundles = ((size_t)constraint_count + W - 1) / W;
    SourceTypeBatch s{};
    s.batch_index = batch_index; s.type_batch_index = type_batch_index; s.type_id = type_id; s.count = constraint_count;
    s.host_impulses = accumulated_impulses;
    s.refs_bytes = bundles * t->bodies * W * 4;
    s.prestep_bytes = bundles * t->prestep_rows * W * 4;
    s.impulse_bytes = bundles * t->impulse_rows * W * 4;
    cudaError_t e = cudaSuccess;
    s.raw_refs = (int32_t*)ctx->raw_arena.alloc(s.refs_bytes, &e);
    s.raw_prestep = (float*)ctx->raw_arena.alloc(s.prestep_bytes, &e);
    s.raw_impulses = (float*)ctx->raw_arena.alloc(s.impulse_bytes, &e);
    if (!s.raw_refs || !s.raw_prestep || !s.raw_impulses) return cuda_fail(ctx, e, "raw arena");
    int rc;
    if ((rc = copy_in(ctx, s.raw_refs, body_references, s.refs_bytes)) != BEPUCUDA_OK) return rc;
    if ((rc = copy_in(ctx, s.raw_prestep, prestep, s.prestep_bytes)) != BEPUCUDA_OK) return rc;
    if ((rc = copy_in(ctx, s.raw_impulses, accumulated_impulses, s.impulse_bytes)) != BEPUCUDA_OK) return rc;
    if (batch_index >= ctx->fallback_threshold) s.host_refs.assign(body_references, body_references + s.refs_bytes / 4);
    ctx->sources.push_back(std::move(s));
    return BEPUCUDA_OK;
}

int32_t bepucuda_set_constrained_kinematics(bepucuda_ctx* ctx, const int32_t* body_indices, int32_t count) {
    if (!ctx || count < 0 || (count > 0 && !body_indices)) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "set_constrained_kinematics: bad arguments");
    ctx->kinematics.assign(body_indices, body_indices + count);
    if (ctx->constraints_ready) ctx->constraints_ready = false;
    return BEPUCUDA_OK;
}

int32_t bepucuda_end_constraints(bepucuda_ctx* ctx) {
    if (!ctx) return BEPUCUDA_ERR_INVALID_ARGUMENT;
    if (!ctx->constraints_open) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "end_constraints without begin_constraints");
    if (ctx->peer_mode && (int)ctx->body_masks.size() != ctx->body_count)
        return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "end_constraints: peer sharding needs bepucuda_shard_set_body_masks for the current body count");
    CK(cudaSetDevice(ctx->device));
    const int W = ctx->W;
    {
        std::vector<SourceView> views;
        for (const SourceTypeBatch& s : ctx->sources) views.push_back({s.batch_index, s.type_batch_index, s.type_id, s.count, s.host_refs.data()});
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
    CK(ctx->map_table.reserve(topo.maps.size() * 4 + 4));
    CK(ctx->inverse_table.reserve(topo.inverse.size() * sizeof(DeviceSlot) + 8));
    std::vector<DeviceTypeBatch> tbs(topo.tbs.size());
    ctx->tdescs.resize(topo.tbs.size());
    for (size_t i = 0; i < topo.tbs.size(); ++i) {
        const PlannedTypeBatch& p = topo.tbs[i];
        const SourceTypeBatch& s = ctx->sources[(size_t)p.source];
        const TypeInfo* t = get_type_info(p.type_id);
        tbs[i] = {p.type_id, p.bundle_count, p.device_batch, t->bodies, ctx->refs32.as<int32_t>() + p.refs_offset, ctx->prestep32.as<float>() + p.prestep_offset,
                  ctx->impulses32.as<float>() + p.impulse_offset};
        ctx->tdescs[i] = {s.raw_refs, s.raw_prestep, s.raw_impulses, p.map_offset < 0 ? nullptr : ctx->map_table.as<int32_t>() + p.map_offset, s.count, t->bodies, t->prestep_rows,
                          t->impulse_rows, topo.source_bundle_base[(size_t)p.source], kTransposePrestep | kTransposeImpulses, t->contacts, nullptr, nullptr};
    }
    ctx->records = work_records(topo, ctx->refs32.as<int32_t>(), ctx->prestep32.as<float>(), ctx->impulses32.as<float>());

    // ---- upload tables ----
    CK(ctx->tb_table.reserve(tbs.size() * sizeof(DeviceTypeBatch) + 16));
    CK(ctx->tdesc_table.reserve(ctx->tdescs.size() * sizeof(TransposeDesc) + 16));
    CK(ctx->work_table.reserve(topo.work.size() * sizeof(WorkItem) + 16));
    CK(ctx->record_table.reserve(ctx->records.size() * sizeof(WorkRecord) + 64));
    CK(ctx->kinematics_dev.reserve(ctx->kinematics.size() * 4 + 4));
    if (!tbs.empty()) CK(cudaMemcpyAsync(ctx->tb_table.ptr, tbs.data(), tbs.size() * sizeof(DeviceTypeBatch), cudaMemcpyHostToDevice, ctx->stream));
    if (!ctx->tdescs.empty()) CK(cudaMemcpyAsync(ctx->tdesc_table.ptr, ctx->tdescs.data(), ctx->tdescs.size() * sizeof(TransposeDesc), cudaMemcpyHostToDevice, ctx->stream));
    if (!topo.work.empty()) CK(cudaMemcpyAsync(ctx->work_table.ptr, topo.work.data(), topo.work.size() * sizeof(WorkItem), cudaMemcpyHostToDevice, ctx->stream));
    if (!ctx->records.empty()) CK(cudaMemcpyAsync(ctx->record_table.ptr, ctx->records.data(), ctx->records.size() * sizeof(WorkRecord), cudaMemcpyHostToDevice, ctx->stream));
    if (!topo.maps.empty()) CK(cudaMemcpyAsync(ctx->map_table.ptr, topo.maps.data(), topo.maps.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
    if (!topo.inverse.empty())
        CK(cudaMemcpyAsync(ctx->inverse_table.ptr, topo.inverse.data(), topo.inverse.size() * sizeof(DeviceSlot), cudaMemcpyHostToDevice, ctx->stream));
    if (!ctx->kinematics.empty()) CK(cudaMemcpyAsync(ctx->kinematics_dev.ptr, ctx->kinematics.data(), ctx->kinematics.size() * 4, cudaMemcpyHostToDevice, ctx->stream));

    // ---- transposition into AOSOA-32 + ownership analysis ----
    { int rc = flush_chunks(ctx, ctx->pending_h2d); if (rc != BEPUCUDA_OK) return rc; }
    launch_transpose_in_all(ctx->tb_table.as<DeviceTypeBatch>(), ctx->tdesc_table.as<TransposeDesc>(), ctx->work_table.as<WorkItem>(), topo.all_work_count, W,
                            kTransposeRefs | kTransposePrestep | kTransposeImpulses, ctx->stream);
    const size_t nb = (size_t)std::max(ctx->body_count, 1);
    CK(ctx->first_batch.reserve(nb * 4));
    CK(ctx->sync_refcount.reserve(nb * 4));
    CK(ctx->sync_mask.reserve(nb * 8));
    ctx->B.first_batch = ctx->first_batch.as<int32_t>();
    launch_fill_i32(ctx->first_batch.as<int32_t>(), nb, 0x7fffffff, ctx->stream);
    CK(cudaMemsetAsync(ctx->sync_refcount.ptr, 0, nb * 4, ctx->stream));
    CK(cudaMemsetAsync(ctx->sync_mask.ptr, 0, nb * 8, ctx->stream));
    CK(cudaMemsetAsync(ctx->constrained.ptr, 0, nb, ctx->stream));
    CK(cudaMemsetAsync(ctx->error_dev.ptr, 0, 32, ctx->stream));
    CK(ctx->source_bundle_flags.reserve((size_t)std::max(topo.source_bundles, 1) * 16));
    CK(cudaMemsetAsync(ctx->source_bundle_flags.ptr, 0, (size_t)std::max(topo.source_bundles, 1) * 16, ctx->stream));
    launch_ownership_pass1(ctx->tb_table.as<DeviceTypeBatch>(), ctx->work_table.as<WorkItem>(), topo.all_work_count, topo.sync_batch_count,
                           ctx->body_count, ctx->first_batch.as<int32_t>(), ctx->sync_refcount.as<int32_t>(), (unsigned long long*)ctx->sync_mask.ptr, ctx->error_dev.as<int32_t>(),
                           ctx->stream);
    if (ctx->peer_mode && nb > 0) {
        // peer sharding: the integration owner of a body is the lowest batch referencing it on ANY rank (computed by the host over the whole graph);
        // a body the graph first references in the fallback batch keeps the level this rank, the fallback rank, found for it
        if ((int)ctx->global_first_batch.size() != ctx->body_count) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "end_constraints: bepucuda_shard_set_global was not called for this body count");
        CK(ctx->global_first_batch_dev.reserve(nb * 4));
        CK(cudaMemcpyAsync(ctx->global_first_batch_dev.ptr, ctx->global_first_batch.data(), (size_t)ctx->body_count * 4, cudaMemcpyHostToDevice, ctx->stream));
        launch_merge_first_batch(ctx->first_batch.as<int32_t>(), ctx->global_first_batch_dev.as<int32_t>(), ctx->body_count, ctx->fallback_threshold, ctx->stream);
    }
    launch_ownership_rest(ctx->tb_table.as<DeviceTypeBatch>(), ctx->work_table.as<WorkItem>(), topo.all_work_count, ctx->body_count,
                          ctx->first_batch.as<int32_t>(), ctx->sync_refcount.as<int32_t>(), (const unsigned long long*)ctx->sync_mask.ptr, ctx->constrained.as<uint8_t>(),
                          ctx->kinematics_dev.as<int32_t>(), (int)ctx->kinematics.size(), ctx->error_dev.as<int32_t>(), ctx->tdesc_table.as<TransposeDesc>(), W,
                          ctx->source_bundle_flags.as<int32_t>(), ctx->stream);
    if (ctx->peer_mode) {
        // ... and a body is "constrained" (final pose pass) if any rank constrains it
        CK(cudaMemcpyAsync(ctx->constrained.ptr, ctx->global_constrained.data(), (size_t)ctx->body_count, cudaMemcpyHostToDevice, ctx->stream));
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

int32_t bepucuda_update_type_batch(bepucuda_ctx* ctx, int32_t batch_index, int32_t type_batch_index, const float* prestep, float* accumulated_impulses) {
    if (!ctx || !prestep || !accumulated_impulses) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "update_type_batch: bad arguments");
    if (!ctx->constraints_ready) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "update_type_batch before end_constraints");
    SourceTypeBatch* s = find_source(ctx, batch_index, type_batch_index);
    if (!s) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "update_type_batch: unknown type batch");
    CK(cudaSetDevice(ctx->device));
    open_upload_window(ctx);
    int rc;
    if ((rc = copy_in(ctx, s->raw_prestep, prestep, s->prestep_bytes)) != BEPUCUDA_OK) return rc;
    if ((rc = copy_in(ctx, s->raw_impulses, accumulated_impulses, s->impulse_bytes)) != BEPUCUDA_OK) return rc;
    s->host_impulses = accumulated_impulses;
    s->pending = kTransposePrestep | kTransposeImpulses;
    s->redistribute = false;  // the host took the impulses back
    ctx->data_dirty = true;
    return BEPUCUDA_OK;
}

static int ensure_feature_arrays(bepucuda_ctx* ctx, SourceTypeBatch& s) {
    if (s.raw_features_old) return BEPUCUDA_OK;
    s.feature_bytes = (size_t)s.count * get_type_info(s.type_id)->contacts * sizeof(int32_t);
    cudaError_t e = cudaSuccess;
    s.raw_features_old = (int32_t*)ctx->raw_arena.alloc(s.feature_bytes, &e);
    s.raw_features_new = (int32_t*)ctx->raw_arena.alloc(s.feature_bytes, &e);
    if (!s.raw_features_old || !s.raw_features_new) return cuda_fail(ctx, e, "raw arena (contact feature ids)");
    return BEPUCUDA_OK;
}

int32_t bepucuda_set_contact_features(bepucuda_ctx* ctx, int32_t batch_index, int32_t type_batch_index, const int32_t* feature_ids) {
    if (!ctx || !feature_ids) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "set_contact_features: bad arguments");
    if (!ctx->constraints_open && !ctx->constraints_ready) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "set_contact_features before the type batch was uploaded");
    SourceTypeBatch* s = find_source(ctx, batch_index, type_batch_index);
    if (!s) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "set_contact_features: unknown type batch");
    if (get_type_info(s->type_id)->contacts == 0) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "set_contact_features: not a contact constraint type");
    CK(cudaSetDevice(ctx->device));
    { int rc = ensure_feature_arrays(ctx, *s); if (rc != BEPUCUDA_OK) return rc; }
    // from a mapped buffer the ids are only queued: the next solve copies them, before the host writes the next frame's ids into the same buffer
    if (ctx->constraints_ready) ctx->data_dirty = true;
    return copy_in(ctx, s->raw_features_old, feature_ids, s->feature_bytes);
}

int32_t bepucuda_update_contacts(bepucuda_ctx* ctx, int32_t batch_index, int32_t type_batch_index, const float* prestep, const int32_t* new_feature_ids) {
    if (!ctx || !prestep || !new_feature_ids) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "update_contacts: bad arguments");
    if (!ctx->constraints_ready) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "update_contacts before end_constraints");
    SourceTypeBatch* s = find_source(ctx, batch_index, type_batch_index);
    if (!s) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "update_contacts: unknown type batch");
    if (get_type_info(s->type_id)->contacts == 0) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "update_contacts: not a contact constraint type");
    if (!s->raw_features_old) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "update_contacts: bepucuda_set_contact_features was never called for this type batch");
    if (s->redistribute) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "update_contacts: called twice for the same type batch without a solve in between");
    CK(cudaSetDevice(ctx->device));
    open_upload_window(ctx);
    int rc;
    if ((rc = copy_in(ctx, s->raw_prestep, prestep, s->prestep_bytes)) != BEPUCUDA_OK) return rc;
    if ((rc = copy_in(ctx, s->raw_features_new, new_feature_ids, s->feature_bytes)) != BEPUCUDA_OK) return rc;
    s->pending |= kTransposePrestep;  // the accumulated impulses stay resident
    s->redistribute = true;
    ctx->data_dirty = true;
    return BEPUCUDA_OK;
}

int32_t bepucuda_upload_body_motion(bepucuda_ctx* ctx, const void* body_dynamics, int32_t body_count) {
    if (!ctx || !body_dynamics || body_count != ctx->body_count) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "upload_body_motion: bad arguments (the body count must match the last upload_bodies)");
    if (body_count == 0) return BEPUCUDA_OK;
    CK(cudaSetDevice(ctx->device));
    open_upload_window(ctx);
    const size_t n = (size_t)body_count;
    if (char* alias = map_host(ctx, body_dynamics, n * 128)) {
        launch_scatter_body_motion(alias, body_count, ctx->B, ctx->stream);  // 64 of every 128 bytes read straight from the mapped host buffer
    } else {
        CK(cudaMemcpy2DAsync(ctx->raw_bodies.ptr, 128, body_dynamics, 128, 64, n, cudaMemcpyHostToDevice, ctx->stream));
        launch_scatter_body_motion(ctx->raw_bodies.ptr, body_count, ctx->B, ctx->stream);
    }
    CK(cudaGetLastError());
    ctx->h2d_accum += (int64_t)n * 64;
    return BEPUCUDA_OK;
}

int32_t bepucuda_download_body_motion(bepucuda_ctx* ctx, void* out, int32_t body_count) {
    if (!ctx || !out || body_count < 0 || body_count > ctx->body_count) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "download_body_motion: bad arguments");
    CK(cudaSetDevice(ctx->device));
    CK(cudaEventRecord(ctx->ev_down_begin, ctx->stream));
    const size_t n = (size_t)body_count;
    if (char* alias = map_host(ctx, out, n * 128)) {
        launch_gather_body_motion(alias, body_count, ctx->B, ctx->stream);
    } else {
        launch_gather_body_motion(ctx->raw_bodies.ptr, body_count, ctx->B, ctx->stream);
        CK(cudaMemcpy2DAsync(out, 128, ctx->raw_bodies.ptr, 128, 64, n, cudaMemcpyDeviceToHost, ctx->stream));
    }
    CK(cudaGetLastError());
    CK(cudaEventRecord(ctx->ev_down_end, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    ctx->have_down = true;
    ctx->timings.d2h_bytes = (int64_t)n * 64;
    return BEPUCUDA_OK;
}

int32_t bepucuda_solve(bepucuda_ctx* ctx, float dt) {
    if (!ctx || !(dt > 0)) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "solve: bad arguments");
    { int rc = check_accelerations(ctx, "solve"); if (rc != BEPUCUDA_OK) return rc; }
    CK(cudaSetDevice(ctx->device));
    if (!ctx->constraints_ready) {
        // No constraints were ever described (or the description was invalidated): only legal when nothing was uploaded.
        if (ctx->constraints_open) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "solve inside begin/end_constraints");
        if (!ctx->sources.empty()) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "solve: constraint description is stale; re-run begin/upload/end_constraints");
        int rc = bepucuda_begin_constraints(ctx, ctx->W, 0);
        if (rc == BEPUCUDA_OK) rc = bepucuda_end_constraints(ctx);
        if (rc != BEPUCUDA_OK) return rc;
    }
    { int rc = prepare_frame(ctx, dt); if (rc != BEPUCUDA_OK) return rc; }
    CK(cudaEventRecord(ctx->ev_solve_begin, ctx->stream));
    int64_t launches = 0;
    if (ctx->cfg.execution_mode == BEPUCUDA_EXEC_GRAPH) {
        const LaunchContext lc = launch_context(ctx, false);
        if (!ctx->graph_exec || !same_bodies(ctx->graph_bodies, ctx->B) || !same_launches(ctx->graph_launch, lc)) {
            invalidate_graph(ctx);
            CK(cudaStreamBeginCapture(ctx->stream, cudaStreamCaptureModeThreadLocal));
            int64_t n = 0;
            issue_stage_sequence(ctx, ctx->stream, &n);
            cudaError_t e = cudaStreamEndCapture(ctx->stream, &ctx->graph);
            if (e == cudaSuccess) e = cudaGraphInstantiate(&ctx->graph_exec, ctx->graph, 0);
            if (e != cudaSuccess) return cuda_fail(ctx, e, "graph capture");
            ctx->graph_bodies = ctx->B;
            ctx->graph_launch = lc;
            ctx->timings.kernel_launches = n;
            ++ctx->timings.graph_captures;
        }
        CK(cudaGraphLaunch(ctx->graph_exec, ctx->stream));
        launches = ctx->timings.kernel_launches;
    }
    if (ctx->cfg.execution_mode == BEPUCUDA_EXEC_STREAM) {
        issue_stage_sequence(ctx, ctx->stream, &launches);
        CK(cudaGetLastError());
    }
    CK(cudaEventRecord(ctx->ev_solve_end, ctx->stream));
    if (ctx->peer_mode) { ctx->exchange_counter += ctx->program.exchange_count; ++ctx->shard_solve_index; }  // the flag barrier and the arrival counters keep counting across solves
    ctx->have_solve = true;
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
    CK(cudaEventRecord(ctx->ev_down_begin, ctx->stream));
    launch_merge_bodies(ctx->raw_bodies.ptr, body_count, ctx->B, ctx->stream);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(out, ctx->raw_bodies.ptr, (size_t)body_count * 128, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaEventRecord(ctx->ev_down_end, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    ctx->have_down = true;
    ctx->timings.d2h_bytes = (int64_t)body_count * 128;
    return BEPUCUDA_OK;
}

int32_t bepucuda_download_impulses(bepucuda_ctx* ctx) {
    if (!ctx) return BEPUCUDA_ERR_INVALID_ARGUMENT;
    if (!ctx->constraints_ready) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "download_impulses before end_constraints");
    CK(cudaSetDevice(ctx->device));
    launch_transpose_out_all(ctx->tb_table.as<DeviceTypeBatch>(), ctx->tdesc_table.as<TransposeDesc>(), ctx->work_table.as<WorkItem>(), ctx->topo.all_work_count, ctx->W,
                             kTransposeImpulses, ctx->stream);
    CK(cudaGetLastError());
    int64_t bytes = 0;
    std::vector<CopyChunk> d2h;
    for (auto& s : ctx->sources) {
        if (char* alias = map_host(ctx, s.host_impulses, s.impulse_bytes)) queue_chunks(d2h, alias, s.raw_impulses, s.impulse_bytes);
        else CK(cudaMemcpyAsync(s.host_impulses, s.raw_impulses, s.impulse_bytes, cudaMemcpyDeviceToHost, ctx->stream));
        bytes += (int64_t)s.impulse_bytes;
    }
    { int rc = flush_chunks(ctx, d2h); if (rc != BEPUCUDA_OK) return rc; }
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
    launch_transpose_out_all(ctx->tb_table.as<DeviceTypeBatch>(), ctx->tdesc_table.as<TransposeDesc>(), ctx->work_table.as<WorkItem>(), ctx->topo.all_work_count, ctx->W,
                             kTransposePrestep, ctx->stream);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(prestep_out, s->raw_prestep, s->prestep_bytes, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return BEPUCUDA_OK;
}

static_assert(sizeof(bepucuda_constraint_location) == 16, "bepucuda_constraint_location is four int32");

int32_t bepucuda_read_constraints(bepucuda_ctx* ctx, int32_t count, const bepucuda_constraint_location* locations, int32_t* records_out) {
    if (!ctx) return BEPUCUDA_ERR_INVALID_ARGUMENT;
    if (ctx->peer_mode) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "read_constraints in peer mode: a rank holds its constraints compacted, so host locations do not address them");
    if (!ctx->constraints_ready) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "read_constraints before end_constraints");
    if (count < 0 || (count > 0 && (!locations || !records_out))) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "read_constraints: bad arguments");
    if (count == 0) return BEPUCUDA_OK;
    // every location is checked before any device work, so a bad one leaves records_out untouched
    std::vector<ReadRequest> requests((size_t)count);
    for (int32_t i = 0; i < count; ++i) {
        const bepucuda_constraint_location& l = locations[i];
        ResolvedLocation r;
        if (resolve_location(ctx->topo, l, &r) != BEPUCUDA_OK) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "read_constraints: " + no_constraint_at(i, l));
        ReadRequest& q = requests[(size_t)i];
        q.type_id = l.type_id;
        // a fallback constraint, a hole included, is looked up on the device through its inverse entry
        q.at = r.inverse_entry < 0 ? r.at : DeviceSlot{-1, (int32_t)r.inverse_entry};
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
    if (ctx->peer_mode) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "write_constraints in peer mode: a rank holds its constraints compacted, so host locations do not address them");
    if (!ctx->constraints_ready) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "write_constraints before end_constraints");
    if (count < 0 || (count > 0 && (!locations || !records))) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "write_constraints: bad arguments");
    if (count == 0) return BEPUCUDA_OK;
    // every location and record is checked before anything is queued, so a failing call changes nothing
    std::vector<DeviceSlot> slots((size_t)count);
    for (int32_t i = 0; i < count; ++i) {
        const bepucuda_constraint_location& l = locations[i];
        ResolvedLocation r;
        if (resolve_location(ctx->topo, l, &r) != BEPUCUDA_OK) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "write_constraints: " + no_constraint_at(i, l));
        if (r.at.type_batch < 0) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "write_constraints: " + no_constraint_at(i, l) + " (a hole of the fallback batch)");
        if (records[(size_t)i * 64] != l.type_id)
            return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "write_constraints: record " + std::to_string(i) + " has type id " + std::to_string(records[(size_t)i * 64]) +
                                                                ", its location type id " + std::to_string(l.type_id));
        slots[(size_t)i] = r.at;
    }
    CK(cudaSetDevice(ctx->device));
    open_upload_window(ctx);
    for (int32_t i = 0; i < count; ++i)
        ctx->prestep_writes.put(slots[(size_t)i], (const float*)(records + (size_t)i * 64 + kRecordPrestep), get_type_info(locations[i].type_id)->prestep_rows);
    ctx->data_dirty = true;
    return BEPUCUDA_OK;
}

int32_t bepucuda_get_timings(bepucuda_ctx* ctx, bepucuda_timings* out) {
    if (!ctx || !out) return BEPUCUDA_ERR_INVALID_ARGUMENT;
    CK(cudaSetDevice(ctx->device));
    CK(cudaStreamSynchronize(ctx->stream));
    { int rc = check_device_error_flag(ctx); if (rc != BEPUCUDA_OK) return rc; }
    if (ctx->have_solve) cudaEventElapsedTime(&ctx->timings.solve_ms, ctx->ev_solve_begin, ctx->ev_solve_end);
    if (ctx->have_up && !ctx->up_open) cudaEventElapsedTime(&ctx->timings.upload_ms, ctx->ev_up_begin, ctx->ev_up_end);
    if (ctx->have_down) cudaEventElapsedTime(&ctx->timings.download_ms, ctx->ev_down_begin, ctx->ev_down_end);
    *out = ctx->timings;
    return BEPUCUDA_OK;
}

int32_t bepucuda_event_record(bepucuda_ctx* ctx, int32_t slot) {
    if (!ctx || slot < 0 || slot >= 16) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "event_record: bad slot");
    CK(cudaSetDevice(ctx->device));
    if (!ctx->user_events[slot]) CK(cudaEventCreate(&ctx->user_events[slot]));
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
    { int rc = check_accelerations(ctx, "profile_stages"); if (rc != BEPUCUDA_OK) return rc; }
    CK(cudaSetDevice(ctx->device));
    std::memset(out, 0, sizeof(*out));
    const size_t need = ctx->program.ops.size() * 2;
    while (ctx->profile_events.size() < need) {
        cudaEvent_t ev;
        CK(cudaEventCreate(&ev));
        ctx->profile_events.push_back(ev);
    }
    { int rc = prepare_frame(ctx, dt); if (rc != BEPUCUDA_OK) return rc; }
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

static_assert(sizeof(bepucuda_body_shape) == sizeof(BodyShape) && sizeof(bepucuda_body_activity) == sizeof(BodyActivityRecord), "ABI structs mirror the device records");

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
    { int rc = check_accelerations(ctx, "predict_bounding_boxes"); if (rc != BEPUCUDA_OK) return rc; }
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
    constexpr int kRoundsPerChunk = 32;  // even: the ping-pong lists return to their starting roles after every chunk
    const size_t nb = (size_t)std::max(body_count, 1), nc = (size_t)constraint_count;
    CK(ctx->color_refs.reserve(words * 4));
    CK(ctx->color_priorities.reserve(nc * 4));
    CK(ctx->color_body_min.reserve(nb * 8));
    CK(ctx->color_body_mask.reserve(nb * 8));
    CK(ctx->color_out.reserve(nc * 4));
    CK(ctx->color_lists.reserve(nc * 8));
    CK(ctx->color_counts.reserve((kRoundsPerChunk + 1) * 4));
    CK(cudaMemcpyAsync(ctx->color_refs.ptr, encoded_body_references, words * 4, cudaMemcpyHostToDevice, ctx->stream));
    if (order == BEPUCUDA_COLOR_BY_PRIORITY) CK(cudaMemcpyAsync(ctx->color_priorities.ptr, priorities, nc * 4, cudaMemcpyHostToDevice, ctx->stream));
    ColoringBuffers cb{};
    cb.refs = ctx->color_refs.as<int32_t>();
    cb.priorities = ctx->color_priorities.as<uint32_t>();
    cb.body_min = ctx->color_body_min.as<unsigned long long>();
    cb.body_mask = ctx->color_body_mask.as<unsigned long long>();
    cb.batch_out = ctx->color_out.as<int32_t>();
    cb.list[0] = ctx->color_lists.as<int32_t>();
    cb.list[1] = ctx->color_lists.as<int32_t>() + nc;
    cb.counts = ctx->color_counts.as<unsigned int>();
    cb.constraint_count = constraint_count;
    cb.bodies_per_constraint = bodies_per_constraint;
    cb.body_count = body_count;
    cb.fallback_threshold = fallback_batch_threshold;
    cb.order = order;
    CK(cudaMemsetAsync(ctx->color_counts.ptr, 0, (kRoundsPerChunk + 1) * 4, ctx->stream));
    launch_color_init(cb, ctx->stream);
    unsigned int counts[kRoundsPerChunk + 1];
    int64_t rounds = 0;
    for (;;) {
        for (int r = 0; r < kRoundsPerChunk; ++r) launch_color_round(cb, r, ctx->stream);
        CK(cudaMemcpyAsync(counts, ctx->color_counts.ptr, sizeof(counts), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        CK(cudaGetLastError());
        int used = kRoundsPerChunk;
        for (int r = 0; r < kRoundsPerChunk; ++r)
            if (counts[r + 1] == 0) { used = r + 1; break; }
        rounds += used;
        if (counts[used] == 0) break;
        // every round assigns at least the constraint with the globally lowest key, so the list shrinks: the loop ends after at most constraint_count rounds
        if (counts[kRoundsPerChunk] >= counts[0]) return fail(ctx, BEPUCUDA_ERR_CUDA, "color_constraints: no progress (internal error)");
        counts[0] = counts[kRoundsPerChunk];
        for (int r = 1; r <= kRoundsPerChunk; ++r) counts[r] = 0;
        CK(cudaMemcpyAsync(ctx->color_counts.ptr, counts, sizeof(counts), cudaMemcpyHostToDevice, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));  // `counts` is a stack array: the copy must have read it before the next chunk's download overwrites it
    }
    CK(cudaMemcpyAsync(batch_indices_out, ctx->color_out.ptr, nc * 4, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    int32_t highest = -1;
    for (size_t i = 0; i < nc; ++i) highest = std::max(highest, batch_indices_out[i]);
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
    const size_t n = (size_t)body_count;
    CK(ctx->island_activities.reserve(n * sizeof(bepucuda_body_activity)));
    CK(ctx->island_label.reserve(n * 4));
    CK(ctx->island_blocked.reserve(n * 4));
    CK(ctx->island_count.reserve(n * 4));
    CK(ctx->island_flags.reserve(n));
    CK(ctx->island_roots.reserve(n * 4));
    CK(ctx->island_counts.reserve(n * 4));
    CK(ctx->island_scalars.reserve(8));  // [0]: hook pass changed something, [1]: number of sleepable roots
    IslandBuffers ib{};
    ib.tbs = ctx->tb_table.as<DeviceTypeBatch>();
    ib.work = ctx->work_table.as<WorkItem>();
    ib.work_count = ctx->topo.all_work_count;
    ib.activities = ctx->island_activities.as<uint8_t>();
    ib.label = ctx->island_label.as<int32_t>();
    ib.blocked = ctx->island_blocked.as<int32_t>();
    ib.count = ctx->island_count.as<int32_t>();
    ib.changed = ctx->island_scalars.as<unsigned int>();
    ib.body_count = body_count;
    int32_t* selected = ctx->island_scalars.as<int32_t>() + 1;
    size_t temp_bytes = 0;
    CK(launch_island_select(ib, nullptr, nullptr, nullptr, selected, nullptr, &temp_bytes, ctx->stream));
    CK(ctx->island_temp.reserve(std::max(temp_bytes, (size_t)16)));
    temp_bytes = ctx->island_temp.capacity;
    CK(cudaMemcpyAsync(ctx->island_activities.ptr, activities, n * sizeof(bepucuda_body_activity), cudaMemcpyHostToDevice, ctx->stream));
    launch_island_init(ib, ctx->stream);
    CK(cudaGetLastError());
    // every round that changes something joins at least two trees, so there are at most body_count of them; in practice O(log n)
    int64_t rounds = 0;
    if (ib.work_count > 0) {
        for (;;) {
            CK(cudaMemsetAsync(ib.changed, 0, 4, ctx->stream));
            launch_island_round(ib, ctx->stream);
            unsigned int changed = 0;
            CK(cudaMemcpyAsync(&changed, ib.changed, 4, cudaMemcpyDeviceToHost, ctx->stream));
            CK(cudaStreamSynchronize(ctx->stream));
            CK(cudaGetLastError());
            ++rounds;
            if (!changed) break;
            if (rounds > (int64_t)body_count) return fail(ctx, BEPUCUDA_ERR_CUDA, "find_sleepable_islands: no convergence (internal error)");
        }
    }
    launch_island_verdict(ib, ctx->stream);
    CK(launch_island_select(ib, ctx->island_flags.as<uint8_t>(), ctx->island_roots.as<int32_t>(), ctx->island_counts.as<int32_t>(), selected, ctx->island_temp.ptr, &temp_bytes,
                            ctx->stream));
    int32_t count = 0;
    CK(cudaMemcpyAsync(&count, selected, 4, cudaMemcpyDeviceToHost, ctx->stream));
    if (island_of_body_out) CK(cudaMemcpyAsync(island_of_body_out, ib.label, n * 4, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    if (count > 0) {
        CK(cudaMemcpyAsync(sleepable_roots_out, ctx->island_roots.ptr, (size_t)count * 4, cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaMemcpyAsync(sleepable_body_counts_out, ctx->island_counts.ptr, (size_t)count * 4, cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
    }
    *sleepable_count_out = count;
    if (rounds_out) *rounds_out = (int32_t)std::min<int64_t>(rounds, 0x7fffffff);
    return BEPUCUDA_OK;
}

int32_t bepucuda_shard_export(bepucuda_ctx* ctx, bepucuda_ipc_handles* out) {
    if (!ctx || !out) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "shard_export: bad arguments");
    if (ctx->body_count <= 0) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "shard_export before upload_bodies");
    CK(cudaSetDevice(ctx->device));
    CK(ctx->shard_flags.reserve(kShardFlagBlockWords * sizeof(unsigned long long)));  // barrier flags, arrival counters and targets (ShardStage)
    CK(cudaMemset(ctx->shard_flags.ptr, 0, kShardFlagBlockWords * sizeof(unsigned long long)));
    void* ptrs[4] = {ctx->pose.ptr, ctx->velocity.ptr, ctx->inertia_world.ptr, ctx->shard_flags.ptr};
    for (int i = 0; i < 4; ++i) {
        cudaIpcMemHandle_t h;
        CK(cudaIpcGetMemHandle(&h, ptrs[i]));
        static_assert(sizeof(h) == 64, "cudaIpcMemHandle_t is 64 bytes");
        std::memcpy(out->bytes[i], &h, 64);
    }
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
        void* ptrs[4] = {ctx->pose.ptr, ctx->velocity.ptr, ctx->inertia_world.ptr, ctx->shard_flags.ptr};
        if (r != rank)
            for (int i = 0; i < 4; ++i) {
                cudaIpcMemHandle_t h;
                std::memcpy(&h, all[r].bytes[i], 64);
                CK(cudaIpcOpenMemHandle(&ptrs[i], h, cudaIpcMemLazyEnablePeerAccess));
                ctx->opened_ipc.push_back(ptrs[i]);
            }
        p.pose[r] = (float4*)ptrs[0];
        p.velocity[r] = (float4*)ptrs[1];
        p.inertia_world[r] = (float4*)ptrs[2];
        p.flags[r] = (unsigned long long*)ptrs[3];
    }
    ctx->peers = p;
    ctx->peer_mode = true;
    ctx->exchange_counter = 0;
    if (ctx->constraints_ready) ctx->constraints_ready = false;
    return BEPUCUDA_OK;
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
        p.pose[r] = o->pose.as<float4>();
        p.velocity[r] = o->velocity.as<float4>();
        p.inertia_world[r] = o->inertia_world.as<float4>();
        p.flags[r] = (unsigned long long*)o->shard_flags.ptr;
    }
    ctx->peers = p;
    ctx->peer_mode = true;
    ctx->exchange_counter = 0;
    if (ctx->constraints_ready) ctx->constraints_ready = false;
    return BEPUCUDA_OK;
}

int32_t bepucuda_shard_set_global(bepucuda_ctx* ctx, const int32_t* first_batch, const uint8_t* constrained) {
    if (!ctx || !first_batch || !constrained) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "shard_set_global: bad arguments");
    ctx->global_first_batch.assign(first_batch, first_batch + ctx->body_count);
    ctx->global_constrained.assign(constrained, constrained + ctx->body_count);
    if (ctx->constraints_ready) ctx->constraints_ready = false;
    return BEPUCUDA_OK;
}

int32_t bepucuda_shard_set_body_masks(bepucuda_ctx* ctx, const uint8_t* rank_masks) {
    if (!ctx || !rank_masks) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "shard_set_body_masks: bad arguments");
    ctx->body_masks.assign(rank_masks, rank_masks + ctx->body_count);
    if (ctx->constraints_ready) ctx->constraints_ready = false;
    return BEPUCUDA_OK;
}

int32_t bepucuda_shard_set_fallback_rank(bepucuda_ctx* ctx, int32_t rank) {
    if (!ctx) return BEPUCUDA_ERR_INVALID_ARGUMENT;
    if (!ctx->peer_mode) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "shard_set_fallback_rank: the context is not in peer mode (bepucuda_shard_import*)");
    if (rank < -1 || rank >= ctx->peers.rank_count) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "shard_set_fallback_rank: rank out of range");
    ctx->fallback_rank = rank;
    if (ctx->constraints_ready) ctx->constraints_ready = false;
    return BEPUCUDA_OK;
}

}  // extern "C"
