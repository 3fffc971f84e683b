// libbepucuda host side: context, device memory, uploads/downloads, device tables of the topology plan (bepu_topology.h), stage launches, CUDA graph.
// C ABI declared in include/bepucuda.h. No CPU fallback lives here: without a usable CUDA device bepucuda_create fails.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/bepucuda.h"
#include "bepu_layout_kernels.h"
#include "bepu_coloring.h"
#include "bepu_bounds.h"
#include "bepu_topology.h"

using namespace bepucuda;

namespace bepucuda {

// ---- small RAII helpers ------------------------------------------------------------------------------------------------------
struct DeviceBuffer {
    void* ptr = nullptr;
    size_t capacity = 0;
    cudaError_t reserve(size_t bytes) {
        if (bytes <= capacity) return cudaSuccess;
        if (ptr) cudaFree(ptr);
        ptr = nullptr;
        capacity = 0;
        size_t want = bytes + bytes / 4 + 256;
        cudaError_t e = cudaMalloc(&ptr, want);
        if (e == cudaSuccess) capacity = want;
        return e;
    }
    void release() {
        if (ptr) cudaFree(ptr);
        ptr = nullptr;
        capacity = 0;
    }
    template <class T> T* as() const { return (T*)ptr; }
};

// Bump allocator over chunks that are never reallocated (uploads are enqueued against their addresses).
struct ChunkArena {
    struct Chunk { char* base; size_t size, used; };
    std::vector<Chunk> chunks;
    bool pinned_host = false;
    size_t min_chunk = (size_t)64 << 20;
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
    void release() {
        for (auto& c : chunks) { if (pinned_host) cudaFreeHost(c.base); else cudaFree(c.base); }
        chunks.clear();
    }
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
    bool resident_impulses = false, redistribute = false;
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
    void* accelerations_stage = nullptr;
    size_t accelerations_stage_bytes = 0;
    cudaEvent_t accelerations_staged = nullptr;
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
    bool constraints_open = false, constraints_ready = false, data_dirty = false, descs_dirty = false;
    std::vector<SourceTypeBatch> sources;
    ChunkArena raw_arena, pinned_arena;
    DeviceBuffer record_table, ref_rows, source_bundle_flags, refs32, prestep32, impulses32, tb_table, tdesc_table, work_table, map_table, bodies_per_type, kinematics_dev, frame_params_dev, error_dev;
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
    std::vector<uint8_t> global_constrained;
    uint32_t exchange_counter = 0;                                  // exchange points executed so far (flag barrier sequence)
    std::vector<int32_t> kinematics;
    StageProgram program;
    FrameParams* frame_params_host = nullptr;   // pinned

    cudaGraph_t graph = nullptr;
    cudaGraphExec_t graph_exec = nullptr;
    bool graph_valid = false;

    bepucuda_timings timings{};
    int64_t h2d_accum = 0;
    struct HostRange { char* host; size_t bytes; char* dev; };
    std::vector<HostRange> host_ranges;    // page-locked + device-mapped host memory registered through bepucuda_host_register
    std::vector<CopyChunk> pending_h2d;    // batched copies waiting for the next flush
    DeviceBuffer chunk_table;
    struct ChunkStage { void* host = nullptr; size_t capacity = 0; cudaEvent_t done = nullptr; };
    ChunkStage chunk_stage[4];             // pinned ring for chunk tables (a table must outlive its H2D copy)
    int chunk_stage_next = 0;
    cudaEvent_t user_events[16] = {};
    DeviceBuffer body_shapes, body_activities, body_bounds;  // bepucuda_set_body_shapes / bepucuda_predict_bounding_boxes
    int shape_count = -1;
    DeviceBuffer color_refs, color_priorities, color_body_min, color_body_mask, color_out, color_lists, color_counts;  // bepucuda_color_constraints
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
// Runs the queued chunks as one kernel. The chunk table travels through the pinned staging arena (recycled at begin_constraints / per flush).
int flush_chunks(bepucuda_ctx* ctx, std::vector<CopyChunk>& list) {
    if (list.empty()) return BEPUCUDA_OK;
    const size_t bytes = list.size() * sizeof(CopyChunk);
    CK(ctx->chunk_table.reserve(bytes));
    auto& st = ctx->chunk_stage[ctx->chunk_stage_next];
    ctx->chunk_stage_next = (ctx->chunk_stage_next + 1) & 3;
    if (!st.done) CK(cudaEventCreateWithFlags(&st.done, cudaEventDisableTiming));
    CK(cudaEventSynchronize(st.done));  // its previous use (4 flushes ago) is long finished
    if (st.capacity < bytes) {
        if (st.host) cudaFreeHost(st.host);
        st.host = nullptr;
        st.capacity = 0;
        CK(cudaMallocHost(&st.host, bytes * 2));
        st.capacity = bytes * 2;
    }
    std::memcpy(st.host, list.data(), bytes);
    // The device-side table is reused by every flush: stream order keeps the previous batched copy ahead of this overwrite.
    CK(cudaMemcpyAsync(ctx->chunk_table.ptr, st.host, bytes, cudaMemcpyHostToDevice, ctx->stream));
    launch_batched_copy(ctx->chunk_table.as<CopyChunk>(), (int)list.size(), ctx->stream);
    CK(cudaGetLastError());
    CK(cudaEventRecord(st.done, ctx->stream));
    list.clear();
    return BEPUCUDA_OK;
}

// H2D copy of one host buffer into the raw arena. Small buffers are packed through pinned staging so that hundreds of
// tiny type batches do not each pay a pageable-memory DMA setup; large ones go directly (fast when the host registered them).
int copy_in(bepucuda_ctx* ctx, void* dst, const void* src, size_t bytes) {
    if (bytes == 0) return BEPUCUDA_OK;
    if (char* alias = map_host(ctx, src, bytes)) {
        queue_chunks(ctx->pending_h2d, dst, alias, bytes);  // read straight from the mapped host buffer by the batched copy kernel at the next flush
        ctx->h2d_accum += (int64_t)bytes;
        return BEPUCUDA_OK;
    }
    if (bytes < ((size_t)256 << 10)) {
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

void invalidate_graph(bepucuda_ctx* ctx) {
    if (ctx->graph_exec) cudaGraphExecDestroy(ctx->graph_exec);
    if (ctx->graph) cudaGraphDestroy(ctx->graph);
    ctx->graph_exec = nullptr;
    ctx->graph = nullptr;
    ctx->graph_valid = false;
}

// Per-body accelerations or point gravity set: the WarmStart stages and the per-body passes launch the instantiations that apply them, so switching either on or
// off changes the launch sequence (a captured graph is rebuilt); their values are frame parameters.
bool integrator_extensions(const bepucuda_ctx* ctx) { return ctx->accelerations_count >= 0 || ctx->point_gravity; }

// Profiling sink of issue_stage_sequence: the launch of program op i sets launched[i] and is bracketed by events[2i] and events[2i + 1].
struct StageEvents {
    const std::vector<cudaEvent_t>& events;
    std::vector<int>& launched;
};

// Issues the whole stage sequence of one frame as individual launches on `s` (used directly in STREAM mode and under capture in GRAPH mode).
// With `profile`, stages are launched without programmatic dependent launch and without prologue prefetch, so that each event pair times one
// kernel alone.
void issue_stage_sequence(bepucuda_ctx* ctx, cudaStream_t s, int64_t* launches, const StageEvents* profile = nullptr) {
    const WorkRecord* records = ctx->record_table.as<WorkRecord>();
    const int32_t* ref_rows = ctx->ref_rows.as<int32_t>();
    const FrameParams* fp = ctx->frame_params_dev.as<FrameParams>();
    const int32_t* kin = ctx->kinematics_dev.as<int32_t>();
    ShardLaunch shard{ctx->peers, (long long)(ctx->peer32.as<int32_t>() - ctx->refs32.as<int32_t>()), {0, ctx->error_dev.as<int32_t>()}};
    int64_t n = 0;
    const int extensions = integrator_extensions(ctx) ? kLaunchIntegratorExtensions : 0;
    for (size_t i = 0; i < ctx->program.ops.size(); ++i) {
        const StageOp& op = ctx->program.ops[i];
        const bool barrier = op.exchange == kRankBarrier;
        // A sharded stage without constraints on this rank launches nothing but still counts as an exchange point: nothing arrives from this
        // rank there, and its arrival targets say so.
        if (barrier || (op.stage == kStageFinalPose ? ctx->B.count > 0 : op.work_count > 0)) {
            if (profile) cudaEventRecord(profile->events[2 * i], s);
            if (barrier) {
                // all ranks meet: before the first stage of a solve; around the incremental contact update, which reads the velocities of shared
                // bodies; and before the final pose pass
                launch_shard_barrier(ctx->peers, fp, op.exchange_index, ctx->error_dev.as<int32_t>(), s);
            } else if (op.stage <= kStageIncremental) {
                // a sharded stage stores the records it writes for shared bodies into the ranks that reference them, and its boundary bundles wait
                // for and announce arrivals themselves (ShardStage)
                shard.stage.exchange_index = op.exchange_index;
                // with per-body accelerations or point gravity the WarmStart stages keep the pose integration (warm_start_body)
                const int op_flags = extensions ? op.launch_flags & ~kLaunchBodiesIntegrated : op.launch_flags;
                const int flags = (profile ? op_flags & (kLaunchContactsOnly | kLaunchBodiesIntegrated) : kLaunchPdl | op_flags) | extensions;
                ctx->launchers->constraint_stage(op.stage, records + op.work_begin, ref_rows + (size_t)op.work_begin * 64, op.work_count, ctx->B, fp, flags,
                                                 op.exchange == kNoExchange ? nullptr : &shard, s);
            } else if (op.stage <= kStageKinematic) {
                ctx->launchers->kinematic_stage(op.stage, kin, op.work_count, ctx->B, fp, extensions, s);
            } else {
                ctx->launchers->final_pose(ctx->B, fp, extensions, s);
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

int upload_program(bepucuda_ctx* ctx) {
    ctx->program = build_stage_program(ctx->topo, ctx->iterations, (int)ctx->kinematics.size(), ctx->integ.integrate_velocity_for_kinematics != 0, ctx->peer_mode,
                                       ctx->body_count);
    if (ctx->peer_mode) {
        // publish, to every peer, how many boundary bundles of this rank arrive through each exchange point of one solve (ShardStage), and restart
        // the arrival counters other ranks increment here. Every rank does this for the same program, between solves.
        std::vector<unsigned long long> targets;
        std::string error;
        const int rc = exchange_targets(ctx->program, ctx->boundary_count, &targets, &error);
        if (rc != BEPUCUDA_OK) return fail(ctx, rc, error);
        CK(cudaStreamSynchronize(ctx->stream));
        for (int q = 0; q < ctx->peers.rank_count; ++q)
            if (q != ctx->peers.rank)
                CK(cudaMemcpy(ctx->peers.flags[q] + kShardTargetSlot + (size_t)ctx->peers.rank * kShardMaxExchanges, targets.data(), targets.size() * 8, cudaMemcpyDefault));
        CK(cudaMemset((unsigned long long*)ctx->shard_flags.ptr + kShardCounterSlot, 0, kMaxShardRanks * 8));
        ctx->shard_solve_index = 0;
    }
    // work issued under the previous program completes before that program and its graph are replaced
    CK(cudaStreamSynchronize(ctx->stream));
    invalidate_graph(ctx);
    ctx->timings.stage_count = ctx->program.stage_count;
    return BEPUCUDA_OK;
}

void compute_frame_params(bepucuda_ctx* ctx, float dt, FrameParams* fp) {
    const int substeps = (int)ctx->iterations.size();
    const float substepDt = dt / substeps;  // Solver_Solve.cs:L1417
    auto clamp01 = [](float v) { return v < 0.f ? 0.f : (v > 1.f ? 1.f : v); };
    const bepucuda_integrator_desc& d = ctx->integ;
    fp->dt = substepDt;
    fp->inverse_dt = 1.0f / substepDt;
    // PrepareForIntegration(substepDt): Demos/DemoCallbacks.cs:L79-86
    fp->linear_damping_dt = powf(clamp01(1 - d.linear_damping), substepDt);
    fp->angular_damping_dt = powf(clamp01(1 - d.angular_damping), substepDt);
    for (int i = 0; i < 3; ++i) fp->gravity_dt[i] = d.gravity[i] * substepDt;
    // IntegrateAfterSubstepping: PoseIntegrator.cs:L707-712
    const float finalDt = d.allow_substeps_for_unconstrained ? substepDt : dt;
    fp->final_dt = finalDt;
    fp->final_linear_damping_dt = powf(clamp01(1 - d.linear_damping), finalDt);
    fp->final_angular_damping_dt = powf(clamp01(1 - d.angular_damping), finalDt);
    for (int i = 0; i < 3; ++i) fp->final_gravity_dt[i] = d.gravity[i] * finalDt;
    fp->final_steps = d.allow_substeps_for_unconstrained ? substeps : 1;
    fp->angular_mode = d.angular_integration_mode;
    fp->integrate_velocity_for_kinematics = d.integrate_velocity_for_kinematics;
    // optional velocity terms (bepucuda_set_body_accelerations / bepucuda_set_point_gravity); PrepareForIntegration: gravityDt = dt * Gravity
    // (PlanetDemo.cs:L36-40)
    const unsigned long long accelerations = ctx->accelerations_count >= 0 ? (unsigned long long)ctx->accelerations.ptr : 0ull;
    fp->accelerations[0] = (uint32_t)accelerations;
    fp->accelerations[1] = (uint32_t)(accelerations >> 32);
    fp->integrate_extensions = (ctx->accelerations_count >= 0 ? kIntegrateAccelerations : 0u) | (ctx->point_gravity ? kIntegratePointGravity : 0u);
    for (int i = 0; i < 3; ++i) fp->attractor_center[i] = ctx->attractor_center[i];
    fp->attractor_dt = substepDt * ctx->attractor_strength;
    fp->final_attractor_dt = finalDt * ctx->attractor_strength;
}

// Accelerations set for another body count than the current one index the wrong bodies: solve, profile_stages and predict_bounding_boxes refuse
// to run before any device work.
int check_accelerations(bepucuda_ctx* ctx, const char* what) {
    if (ctx->accelerations_count >= 0 && ctx->accelerations_count != ctx->body_count)
        return fail(ctx, BEPUCUDA_ERR_BAD_STATE, std::string(what) + ": the body count changed after bepucuda_set_body_accelerations; set them again (or clear them with NULL)");
    return BEPUCUDA_OK;
}

// Brings the device AOSOA-32 rows up to date with what the host queued since the last solve (bepucuda_update_type_batch / bepucuda_update_contacts):
// flushes the batched copies, re-uploads the transposition descriptors when a type batch switched to resident impulses, transposes, and
// redistributes the resident penetration impulses of updated contact type batches from the old to the new feature ids.
int refresh_device_rows(bepucuda_ctx* ctx) {
    if (!ctx->data_dirty) return BEPUCUDA_OK;
    { int rc = flush_chunks(ctx, ctx->pending_h2d); if (rc != BEPUCUDA_OK) return rc; }
    bool any_redistribute = false;
    if (ctx->descs_dirty) {
        for (size_t tb = 0; tb < ctx->topo.tbs.size(); ++tb) {
            const SourceTypeBatch& s = ctx->sources[(size_t)ctx->topo.tbs[tb].source];
            TransposeDesc& d = ctx->tdescs[tb];
            d.flags = (s.resident_impulses ? kDescResidentImpulses : 0) | (s.redistribute ? kDescRedistribute : 0);
            d.features_old = s.raw_features_old;
            d.features_new = s.raw_features_new;
            any_redistribute |= s.redistribute;
        }
        CK(cudaMemcpyAsync(ctx->tdesc_table.ptr, ctx->tdescs.data(), ctx->tdescs.size() * sizeof(TransposeDesc), cudaMemcpyHostToDevice, ctx->stream));
    }
    launch_transpose_in_all(ctx->tb_table.as<DeviceTypeBatch>(), ctx->tdesc_table.as<TransposeDesc>(), ctx->work_table.as<WorkItem>(), ctx->topo.all_work_count, ctx->W,
                            kTransposePrestep | kTransposeImpulses, ctx->stream);
    if (any_redistribute) {
        launch_redistribute_impulses(ctx->tb_table.as<DeviceTypeBatch>(), ctx->tdesc_table.as<TransposeDesc>(), ctx->work_table.as<WorkItem>(), ctx->topo.all_work_count, ctx->stream);
        for (SourceTypeBatch& s : ctx->sources)
            if (s.redistribute) {
                std::swap(s.raw_features_old, s.raw_features_new);  // the resident impulses now belong to the new ids
                s.redistribute = false;
            }
        // descriptors still carry kDescRedistribute and the pre-swap pointers: they are rewritten by the next update (descs_dirty stays set)
    } else {
        ctx->descs_dirty = false;
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
    compute_frame_params(ctx, dt, ctx->frame_params_host);
    ctx->frame_params_host->exchange_base = ctx->exchange_counter;
    ctx->frame_params_host->shard_solve_index = ctx->shard_solve_index;
    CK(cudaMemcpyAsync(ctx->frame_params_dev.ptr, ctx->frame_params_host, sizeof(FrameParams), cudaMemcpyHostToDevice, ctx->stream));
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
    cudaError_t e = cudaSetDevice(ctx->device);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking);
    cudaEvent_t* evs[] = {&ctx->ev_solve_begin, &ctx->ev_solve_end, &ctx->ev_up_begin, &ctx->ev_up_end, &ctx->ev_down_begin, &ctx->ev_down_end};
    for (auto ev : evs)
        if (e == cudaSuccess) e = cudaEventCreate(ev);
    if (e == cudaSuccess) e = cudaMallocHost((void**)&ctx->frame_params_host, sizeof(FrameParams));
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
    DeviceBuffer* bufs[] = {&ctx->shard_flags, &ctx->peer32, &ctx->body_masks_dev, &ctx->boundary_flags_dev, &ctx->raw_bodies, &ctx->pose, &ctx->velocity, &ctx->inertia_local, &ctx->inertia_world, &ctx->constrained, &ctx->first_batch, &ctx->sync_refcount,
                            &ctx->sync_mask, &ctx->chunk_table, &ctx->record_table, &ctx->ref_rows, &ctx->body_shapes, &ctx->body_activities, &ctx->body_bounds, &ctx->color_refs, &ctx->color_priorities, &ctx->color_body_min, &ctx->color_body_mask, &ctx->color_out, &ctx->color_lists, &ctx->color_counts, &ctx->source_bundle_flags, &ctx->refs32, &ctx->prestep32, &ctx->impulses32, &ctx->tb_table, &ctx->tdesc_table, &ctx->work_table, &ctx->map_table,
                            &ctx->bodies_per_type, &ctx->kinematics_dev, &ctx->frame_params_dev, &ctx->error_dev, &ctx->accelerations};
    for (auto b : bufs) b->release();
    if (ctx->accelerations_stage) cudaFreeHost(ctx->accelerations_stage);
    if (ctx->accelerations_staged) cudaEventDestroy(ctx->accelerations_staged);
    ctx->raw_arena.release();
    ctx->pinned_arena.release();
    if (ctx->frame_params_host) cudaFreeHost(ctx->frame_params_host);
    for (auto ev : ctx->user_events)
        if (ev) cudaEventDestroy(ev);
    for (auto& st : ctx->chunk_stage) {
        if (st.host) cudaFreeHost(st.host);
        if (st.done) cudaEventDestroy(st.done);
    }
    for (auto ev : ctx->profile_events) cudaEventDestroy(ev);
    cudaEvent_t evs[] = {ctx->ev_solve_begin, ctx->ev_solve_end, ctx->ev_up_begin, ctx->ev_up_end, ctx->ev_down_begin, ctx->ev_down_end};
    for (auto ev : evs)
        if (ev) cudaEventDestroy(ev);
    if (ctx->stream) cudaStreamDestroy(ctx->stream);
    delete ctx;
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
        const bool was = integrator_extensions(ctx);
        ctx->accelerations_count = -1;
        if (was != integrator_extensions(ctx)) invalidate_graph(ctx);
        return BEPUCUDA_OK;
    }
    if (body_count != ctx->body_count) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "set_body_accelerations: the body count must match the last upload_bodies");
    CK(cudaSetDevice(ctx->device));
    open_upload_window(ctx);
    const size_t bytes = (size_t)body_count * 32;
    CK(ctx->accelerations.reserve(std::max(bytes, (size_t)32)));
    if (bytes > 0) {
        // through a pinned staging copy, so that the caller's buffer is free when the call returns without waiting for the device
        if (!ctx->accelerations_staged) CK(cudaEventCreateWithFlags(&ctx->accelerations_staged, cudaEventDisableTiming));
        CK(cudaEventSynchronize(ctx->accelerations_staged));  // the previous upload has left the staging buffer
        if (ctx->accelerations_stage_bytes < bytes) {
            if (ctx->accelerations_stage) cudaFreeHost(ctx->accelerations_stage);
            ctx->accelerations_stage = nullptr;
            ctx->accelerations_stage_bytes = 0;
            CK(cudaMallocHost(&ctx->accelerations_stage, bytes));
            ctx->accelerations_stage_bytes = bytes;
        }
        std::memcpy(ctx->accelerations_stage, accelerations, bytes);
        CK(cudaMemcpyAsync(ctx->accelerations.ptr, ctx->accelerations_stage, bytes, cudaMemcpyHostToDevice, ctx->stream));
        CK(cudaEventRecord(ctx->accelerations_staged, ctx->stream));
        ctx->h2d_accum += (int64_t)bytes;
    }
    if (!integrator_extensions(ctx)) invalidate_graph(ctx);
    ctx->accelerations_count = body_count;
    return BEPUCUDA_OK;
}

int32_t bepucuda_set_point_gravity(bepucuda_ctx* ctx, int32_t enabled, const float* center, float strength) {
    if (!ctx || (enabled && !center)) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "set_point_gravity: bad arguments");
    if (ctx->point_gravity != (enabled != 0) && ctx->accelerations_count < 0) invalidate_graph(ctx);
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
    if (body_count != ctx->body_count) {
        // constrained flags / ownership depend on the body count; force a rebuild of topology products.
        if (ctx->constraints_ready) ctx->constraints_ready = false;
        invalidate_graph(ctx);
    }
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
    if (B.pose != ctx->B.pose || B.velocity != ctx->B.velocity || B.inertia_local != ctx->B.inertia_local || B.inertia_world != ctx->B.inertia_world ||
        B.constrained != ctx->B.constrained || B.first_batch != ctx->B.first_batch || B.count != ctx->B.count)
        invalidate_graph(ctx);  // kernel arguments are baked into graph nodes
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
    ctx->raw_arena.reset();
    ctx->pinned_arena.reset();
    ctx->constraints_open = true;
    ctx->constraints_ready = false;
    invalidate_graph(ctx);
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
        const int rc = plan_topology(views, W, ctx->fallback_threshold, ctx->batch_count, ctx->body_count, ctx->peer_mode, &plan, &error);
        if (rc != BEPUCUDA_OK) return fail(ctx, rc, error);
        ctx->topo = std::move(plan);
    }
    const TopologyPlan& topo = ctx->topo;

    // ---- device arenas for the AOSOA-32 image, type batches, transposition descriptors, work records ----
    CK(ctx->refs32.reserve(topo.refs_words * 4 + 1024));  // slack: solver warps always read two body-reference rows
    CK(ctx->prestep32.reserve(topo.prestep_words * 4 + 4));
    CK(ctx->impulses32.reserve(topo.impulse_words * 4 + 4));
    CK(ctx->map_table.reserve(topo.maps.size() * 4 + 4));
    std::vector<DeviceTypeBatch> tbs(topo.tbs.size());
    ctx->tdescs.resize(topo.tbs.size());
    for (size_t i = 0; i < topo.tbs.size(); ++i) {
        const PlannedTypeBatch& p = topo.tbs[i];
        const SourceTypeBatch& s = ctx->sources[(size_t)p.source];
        const TypeInfo* t = get_type_info(p.type_id);
        tbs[i] = {p.type_id, p.bundle_count, p.device_batch, 0, ctx->refs32.as<int32_t>() + p.refs_offset, ctx->prestep32.as<float>() + p.prestep_offset,
                  ctx->impulses32.as<float>() + p.impulse_offset};
        ctx->tdescs[i] = {s.raw_refs, s.raw_prestep, s.raw_impulses, p.map_offset < 0 ? nullptr : ctx->map_table.as<int32_t>() + p.map_offset, s.count, t->bodies, t->prestep_rows,
                          t->impulse_rows, topo.source_bundle_base[(size_t)p.source], 0, nullptr, nullptr};
    }
    ctx->records = work_records(topo, ctx->refs32.as<int32_t>(), ctx->prestep32.as<float>(), ctx->impulses32.as<float>());

    // ---- upload tables ----
    int32_t bodies_per_type[64];
    for (int i = 0; i < 64; ++i) bodies_per_type[i] = get_type_info(i) ? get_type_info(i)->bodies : 0;
    CK(ctx->tb_table.reserve(tbs.size() * sizeof(DeviceTypeBatch) + 16));
    CK(ctx->tdesc_table.reserve(ctx->tdescs.size() * sizeof(TransposeDesc) + 16));
    CK(ctx->work_table.reserve(topo.work.size() * sizeof(WorkItem) + 16));
    CK(ctx->record_table.reserve(ctx->records.size() * sizeof(WorkRecord) + 64));
    CK(ctx->bodies_per_type.reserve(sizeof(bodies_per_type)));
    CK(ctx->kinematics_dev.reserve(ctx->kinematics.size() * 4 + 4));
    if (!tbs.empty()) CK(cudaMemcpyAsync(ctx->tb_table.ptr, tbs.data(), tbs.size() * sizeof(DeviceTypeBatch), cudaMemcpyHostToDevice, ctx->stream));
    if (!ctx->tdescs.empty()) CK(cudaMemcpyAsync(ctx->tdesc_table.ptr, ctx->tdescs.data(), ctx->tdescs.size() * sizeof(TransposeDesc), cudaMemcpyHostToDevice, ctx->stream));
    if (!topo.work.empty()) CK(cudaMemcpyAsync(ctx->work_table.ptr, topo.work.data(), topo.work.size() * sizeof(WorkItem), cudaMemcpyHostToDevice, ctx->stream));
    if (!ctx->records.empty()) CK(cudaMemcpyAsync(ctx->record_table.ptr, ctx->records.data(), ctx->records.size() * sizeof(WorkRecord), cudaMemcpyHostToDevice, ctx->stream));
    if (!topo.maps.empty()) CK(cudaMemcpyAsync(ctx->map_table.ptr, topo.maps.data(), topo.maps.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(ctx->bodies_per_type.ptr, bodies_per_type, sizeof(bodies_per_type), cudaMemcpyHostToDevice, ctx->stream));
    if (!ctx->kinematics.empty()) CK(cudaMemcpyAsync(ctx->kinematics_dev.ptr, ctx->kinematics.data(), ctx->kinematics.size() * 4, cudaMemcpyHostToDevice, ctx->stream));

    // ---- transposition into AOSOA-32 + ownership analysis ----
    { int rc = flush_chunks(ctx, ctx->pending_h2d); if (rc != BEPUCUDA_OK) return rc; }
    launch_transpose_in_all(ctx->tb_table.as<DeviceTypeBatch>(), ctx->tdesc_table.as<TransposeDesc>(), ctx->work_table.as<WorkItem>(), topo.all_work_count, W,
                            kTransposeRefs | kTransposePrestep | kTransposeImpulses, ctx->stream);
    const size_t nb = (size_t)std::max(ctx->body_count, 1);
    CK(ctx->first_batch.reserve(nb * 4));
    CK(ctx->sync_refcount.reserve(nb * 4));
    CK(ctx->sync_mask.reserve(nb * 8));
    ctx->B.first_batch = ctx->first_batch.as<int32_t>();  // the graph is re-captured below (upload_program)
    launch_fill_i32(ctx->first_batch.as<int32_t>(), nb, 0x7fffffff, ctx->stream);
    CK(cudaMemsetAsync(ctx->sync_refcount.ptr, 0, nb * 4, ctx->stream));
    CK(cudaMemsetAsync(ctx->sync_mask.ptr, 0, nb * 8, ctx->stream));
    CK(cudaMemsetAsync(ctx->constrained.ptr, 0, nb, ctx->stream));
    CK(cudaMemsetAsync(ctx->error_dev.ptr, 0, 32, ctx->stream));
    CK(ctx->source_bundle_flags.reserve((size_t)std::max(topo.source_bundles, 1) * 16));
    CK(cudaMemsetAsync(ctx->source_bundle_flags.ptr, 0, (size_t)std::max(topo.source_bundles, 1) * 16, ctx->stream));
    launch_ownership_pass1(ctx->tb_table.as<DeviceTypeBatch>(), ctx->work_table.as<WorkItem>(), topo.all_work_count, ctx->bodies_per_type.as<int32_t>(), topo.sync_batch_count,
                           ctx->body_count, ctx->first_batch.as<int32_t>(), ctx->sync_refcount.as<int32_t>(), (unsigned long long*)ctx->sync_mask.ptr, ctx->error_dev.as<int32_t>(),
                           ctx->stream);
    if (ctx->peer_mode && nb > 0) {
        // peer sharding: the integration owner of a body is the lowest batch referencing it on ANY rank (computed by the host over the whole graph)
        if ((int)ctx->global_first_batch.size() != ctx->body_count) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "end_constraints: bepucuda_shard_set_global was not called for this body count");
        CK(cudaMemcpyAsync(ctx->first_batch.ptr, ctx->global_first_batch.data(), (size_t)ctx->body_count * 4, cudaMemcpyHostToDevice, ctx->stream));
    }
    launch_ownership_rest(ctx->tb_table.as<DeviceTypeBatch>(), ctx->work_table.as<WorkItem>(), topo.all_work_count, ctx->bodies_per_type.as<int32_t>(), ctx->body_count,
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
        launch_boundary_flags(ctx->record_table.as<WorkRecord>(), n_rec, ctx->bodies_per_type.as<int32_t>(), (long long)(ctx->peer32.as<int32_t>() - ctx->refs32.as<int32_t>()),
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
    ctx->constraints_ready = true;
    ctx->data_dirty = false;
    return upload_program(ctx);
}

int32_t bepucuda_update_type_batch(bepucuda_ctx* ctx, int32_t batch_index, int32_t type_batch_index, const float* prestep, float* accumulated_impulses) {
    if (!ctx || !prestep || !accumulated_impulses) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "update_type_batch: bad arguments");
    if (!ctx->constraints_ready) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "update_type_batch before end_constraints");
    CK(cudaSetDevice(ctx->device));
    open_upload_window(ctx);
    for (auto& s : ctx->sources)
        if (s.batch_index == batch_index && s.type_batch_index == type_batch_index) {
            char* alias_p = map_host(ctx, prestep, s.prestep_bytes);
            char* alias_i = map_host(ctx, accumulated_impulses, s.impulse_bytes);
            if (alias_p && alias_i) {
                queue_chunks(ctx->pending_h2d, s.raw_prestep, alias_p, s.prestep_bytes);
                queue_chunks(ctx->pending_h2d, s.raw_impulses, alias_i, s.impulse_bytes);
            } else {
                // Direct copies only: the pinned staging arena is recycled per begin_constraints, not per frame.
                CK(cudaMemcpyAsync(s.raw_prestep, prestep, s.prestep_bytes, cudaMemcpyHostToDevice, ctx->stream));
                CK(cudaMemcpyAsync(s.raw_impulses, accumulated_impulses, s.impulse_bytes, cudaMemcpyHostToDevice, ctx->stream));
            }
            ctx->h2d_accum += (int64_t)(s.prestep_bytes + s.impulse_bytes);
            s.host_impulses = accumulated_impulses;
            if (s.resident_impulses) { s.resident_impulses = false; s.redistribute = false; ctx->descs_dirty = true; }  // the host took the impulses back
            ctx->data_dirty = true;
            return BEPUCUDA_OK;
        }
    return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "update_type_batch: unknown type batch");
}

static SourceTypeBatch* find_source(bepucuda_ctx* ctx, int32_t batch_index, int32_t type_batch_index) {
    for (auto& s : ctx->sources)
        if (s.batch_index == batch_index && s.type_batch_index == type_batch_index) return &s;
    return nullptr;
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
    return copy_in(ctx, s->raw_features_old, feature_ids, s->feature_bytes);
}

int32_t bepucuda_update_contacts(bepucuda_ctx* ctx, int32_t batch_index, int32_t type_batch_index, const float* prestep, const int32_t* new_feature_ids) {
    if (!ctx || !prestep || !new_feature_ids) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "update_contacts: bad arguments");
    if (!ctx->constraints_ready) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "update_contacts before end_constraints");
    SourceTypeBatch* s = find_source(ctx, batch_index, type_batch_index);
    if (!s) return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "update_contacts: unknown type batch");
    if (!s->raw_features_old) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "update_contacts: bepucuda_set_contact_features was never called for this type batch");
    if (s->redistribute) return fail(ctx, BEPUCUDA_ERR_BAD_STATE, "update_contacts: called twice for the same type batch without a solve in between");
    CK(cudaSetDevice(ctx->device));
    open_upload_window(ctx);
    // per-frame path: mapped (registered) host buffers go through the batched zero-copy kernel, anything else is copied directly -- never through the
    // pinned staging arena, which is only recycled by bepucuda_begin_constraints
    const void* srcs[2] = {prestep, new_feature_ids};
    void* dsts[2] = {s->raw_prestep, s->raw_features_new};
    const size_t sizes[2] = {s->prestep_bytes, s->feature_bytes};
    for (int i = 0; i < 2; ++i) {
        if (char* alias = map_host(ctx, srcs[i], sizes[i])) queue_chunks(ctx->pending_h2d, dsts[i], alias, sizes[i]);
        else CK(cudaMemcpyAsync(dsts[i], srcs[i], sizes[i], cudaMemcpyHostToDevice, ctx->stream));
        ctx->h2d_accum += (int64_t)sizes[i];
    }
    s->resident_impulses = true;
    s->redistribute = true;
    ctx->descs_dirty = true;
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
        if (!ctx->graph_valid) {
            CK(cudaStreamBeginCapture(ctx->stream, cudaStreamCaptureModeThreadLocal));
            int64_t n = 0;
            issue_stage_sequence(ctx, ctx->stream, &n);
            cudaError_t e = cudaStreamEndCapture(ctx->stream, &ctx->graph);
            if (e == cudaSuccess) e = cudaGraphInstantiate(&ctx->graph_exec, ctx->graph, 0);
            if (e != cudaSuccess) return cuda_fail(ctx, e, "graph capture");
            ctx->graph_valid = true;
            ctx->timings.kernel_launches = n;
        }
        if (ctx->graph_valid) {
            CK(cudaGraphLaunch(ctx->graph_exec, ctx->stream));
            launches = ctx->timings.kernel_launches;
        }
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
    CK(cudaSetDevice(ctx->device));
    for (auto& s : ctx->sources)
        if (s.batch_index == batch_index && s.type_batch_index == type_batch_index) {
            launch_transpose_out_all(ctx->tb_table.as<DeviceTypeBatch>(), ctx->tdesc_table.as<TransposeDesc>(), ctx->work_table.as<WorkItem>(), ctx->topo.all_work_count, ctx->W,
                                     kTransposePrestep, ctx->stream);
            CK(cudaGetLastError());
            CK(cudaMemcpyAsync(prestep_out, s.raw_prestep, s.prestep_bytes, cudaMemcpyDeviceToHost, ctx->stream));
            CK(cudaStreamSynchronize(ctx->stream));
            return BEPUCUDA_OK;
        }
    return fail(ctx, BEPUCUDA_ERR_INVALID_ARGUMENT, "download_prestep: unknown type batch");
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
    auto clamp01 = [](float v) { return v < 0.f ? 0.f : (v > 1.f ? 1.f : v); };
    PredictParams p{};
    p.dt = dt;
    for (int i = 0; i < 3; ++i) p.gravity_dt[i] = ctx->integ.gravity[i] * dt;
    p.linear_damping_dt = powf(clamp01(1 - ctx->integ.linear_damping), dt);
    p.angular_damping_dt = powf(clamp01(1 - ctx->integ.angular_damping), dt);
    p.integrate_velocity_for_kinematics = ctx->integ.integrate_velocity_for_kinematics;
    p.accelerations = ctx->accelerations_count >= 0 ? ctx->accelerations.as<float4>() : nullptr;
    p.integrate_extensions = (ctx->accelerations_count >= 0 ? kIntegrateAccelerations : 0u) | (ctx->point_gravity ? kIntegratePointGravity : 0u);
    for (int i = 0; i < 3; ++i) p.attractor_center[i] = ctx->attractor_center[i];
    p.attractor_dt = dt * ctx->attractor_strength;
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
    invalidate_graph(ctx);
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
    invalidate_graph(ctx);
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

}  // extern "C"
