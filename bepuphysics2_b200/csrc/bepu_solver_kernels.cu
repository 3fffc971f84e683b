// Compiled per numerics flavour (-DBEPU_NS=bepu_fast with FMA contraction / -DBEPU_NS=bepu_strict -fmad=false) and per unit (-DBEPU_UNIT=n),
// so that the big per-type switch of each kernel gets its own translation unit and the build parallelises:
//   0 WarmStartFirst stage   1 WarmStart stage   2 Solve stage   3 Incremental stage + kinematic + final pose + launcher table
#include <atomic>
#include "bepu_solver_kernels.cuh"
#include "bepu_layout_kernels.h"

namespace BEPU_NS {

void launch_stage_warm_start_first(const WorkRecord* records, const int32_t* ref_rows, int work_count, const BodyBuffers& B, const FrameParams* fp, int launch_flags, cudaStream_t s);
void launch_stage_warm_start(const WorkRecord* records, const int32_t* ref_rows, int work_count, const BodyBuffers& B, const FrameParams* fp, int launch_flags, cudaStream_t s);
void launch_stage_solve(const WorkRecord* records, const int32_t* ref_rows, int work_count, const BodyBuffers& B, const FrameParams* fp, int launch_flags, cudaStream_t s);
void launch_stage_warm_start_first_sharded(const WorkRecord* records, const int32_t* ref_rows, int work_count, const BodyBuffers& B, const FrameParams* fp, int launch_flags, const ShardPeers& peers, long long peer_delta, const ShardStage& shard, cudaStream_t s);
void launch_stage_warm_start_sharded(const WorkRecord* records, const int32_t* ref_rows, int work_count, const BodyBuffers& B, const FrameParams* fp, int launch_flags, const ShardPeers& peers, long long peer_delta, const ShardStage& shard, cudaStream_t s);
void launch_stage_solve_sharded(const WorkRecord* records, const int32_t* ref_rows, int work_count, const BodyBuffers& B, const FrameParams* fp, int launch_flags, const ShardPeers& peers, long long peer_delta, const ShardStage& shard, cudaStream_t s);

#ifndef BEPU_DEEP_MINB
#define BEPU_DEEP_MINB 12
#endif
constexpr int kDeepBatchBundles = 2150;  // more bundles than the uncapped build keeps resident at once (132 SMs x 16 warps on an H100 SXM)
template <int STAGE, int MINB>
static void launch_stage_variant(const WorkRecord* records, const int32_t* ref_rows, int work_count, const BodyBuffers& B, const FrameParams* fp, int launch_flags, cudaStream_t s) {
    static std::atomic<bool> carveout_set[64] = {};  // function attributes are per device: a process may hold contexts on several
    int device = 0;
    cudaGetDevice(&device);
    if (!carveout_set[device & 63]) {  // the staged stages keep one 6 KB slab per resident warp in shared memory
        cudaFuncSetAttribute(constraint_stage_kernel<STAGE, MINB>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        carveout_set[device & 63] = true;
    }
    const unsigned blocks = (unsigned)(((size_t)work_count * 32 + kStageBlockThreads - 1) / kStageBlockThreads);
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(blocks);
    cfg.blockDim = dim3(kStageBlockThreads);
    cfg.dynamicSmemBytes = 0;
    cfg.stream = s;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = (launch_flags & bepucuda::kLaunchPdl) ? 1 : 0;
    cudaLaunchKernelEx(&cfg, constraint_stage_kernel<STAGE, MINB>, records, ref_rows, work_count, B, fp, (launch_flags & bepucuda::kLaunchPrefetchRows) ? kStagePrefetchRows : 0);
}
template <int STAGE, int MINB>
static void launch_stage_variant_sharded(const WorkRecord* records, const int32_t* ref_rows, int work_count, const BodyBuffers& B, const FrameParams* fp, int launch_flags, const ShardPeers& peers, long long peer_delta,
                                         const ShardStage& shard, cudaStream_t s) {
    static std::atomic<bool> carveout_set[64] = {};
    int device = 0;
    cudaGetDevice(&device);
    if (!carveout_set[device & 63]) {
        cudaFuncSetAttribute(constraint_stage_kernel_sharded<STAGE, MINB>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        carveout_set[device & 63] = true;
    }
    const unsigned blocks = (unsigned)(((size_t)work_count * 32 + kStageBlockThreads - 1) / kStageBlockThreads);
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(blocks);
    cfg.blockDim = dim3(kStageBlockThreads);
    cfg.stream = s;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = (launch_flags & bepucuda::kLaunchPdl) ? 1 : 0;
    cudaLaunchKernelEx(&cfg, constraint_stage_kernel_sharded<STAGE, MINB>, records, ref_rows, work_count, B, fp, (launch_flags & bepucuda::kLaunchPrefetchRows) ? kStagePrefetchRows : 0, peers,
                       peer_delta, shard);
}
template <int STAGE>
static void launch_stage_sharded_t(const WorkRecord* records, const int32_t* ref_rows, int work_count, const BodyBuffers& B, const FrameParams* fp, int launch_flags, const ShardPeers& peers, long long peer_delta,
                                   const ShardStage& shard, cudaStream_t s) {
    if (work_count >= kDeepBatchBundles) launch_stage_variant_sharded<STAGE, BEPU_DEEP_MINB>(records, ref_rows, work_count, B, fp, launch_flags, peers, peer_delta, shard, s);
    else launch_stage_variant_sharded<STAGE, 1>(records, ref_rows, work_count, B, fp, launch_flags, peers, peer_delta, shard, s);
}
template <int STAGE>
static void launch_stage_t(const WorkRecord* records, const int32_t* ref_rows, int work_count, const BodyBuffers& B, const FrameParams* fp, int launch_flags, cudaStream_t s) {
    if (STAGE != kStageIncremental && work_count >= kDeepBatchBundles) launch_stage_variant<STAGE, BEPU_DEEP_MINB>(records, ref_rows, work_count, B, fp, launch_flags, s);
    else launch_stage_variant<STAGE, 1>(records, ref_rows, work_count, B, fp, launch_flags, s);
}

#if BEPU_UNIT == 0
void launch_stage_warm_start_first(const WorkRecord* records, const int32_t* ref_rows, int work_count, const BodyBuffers& B, const FrameParams* fp, int launch_flags, cudaStream_t s) {
    launch_stage_t<kStageWarmStartFirst>(records, ref_rows, work_count, B, fp, launch_flags, s);
}
void launch_stage_warm_start_first_sharded(const WorkRecord* records, const int32_t* ref_rows, int work_count, const BodyBuffers& B, const FrameParams* fp, int launch_flags, const ShardPeers& peers, long long peer_delta, const ShardStage& shard, cudaStream_t s) {
    launch_stage_sharded_t<kStageWarmStartFirst>(records, ref_rows, work_count, B, fp, launch_flags, peers, peer_delta, shard, s);
}
#elif BEPU_UNIT == 1
void launch_stage_warm_start(const WorkRecord* records, const int32_t* ref_rows, int work_count, const BodyBuffers& B, const FrameParams* fp, int launch_flags, cudaStream_t s) {
    launch_stage_t<kStageWarmStart>(records, ref_rows, work_count, B, fp, launch_flags, s);
}
void launch_stage_warm_start_sharded(const WorkRecord* records, const int32_t* ref_rows, int work_count, const BodyBuffers& B, const FrameParams* fp, int launch_flags, const ShardPeers& peers, long long peer_delta, const ShardStage& shard, cudaStream_t s) {
    launch_stage_sharded_t<kStageWarmStart>(records, ref_rows, work_count, B, fp, launch_flags, peers, peer_delta, shard, s);
}
#elif BEPU_UNIT == 2
void launch_stage_solve(const WorkRecord* records, const int32_t* ref_rows, int work_count, const BodyBuffers& B, const FrameParams* fp, int launch_flags, cudaStream_t s) {
    launch_stage_t<kStageSolve>(records, ref_rows, work_count, B, fp, launch_flags, s);
}
void launch_stage_solve_sharded(const WorkRecord* records, const int32_t* ref_rows, int work_count, const BodyBuffers& B, const FrameParams* fp, int launch_flags, const ShardPeers& peers, long long peer_delta, const ShardStage& shard, cudaStream_t s) {
    launch_stage_sharded_t<kStageSolve>(records, ref_rows, work_count, B, fp, launch_flags, peers, peer_delta, shard, s);
}
#elif BEPU_UNIT == 3
static void launch_constraint_stage(int stage, const WorkRecord* records, const int32_t* ref_rows, int work_count, const BodyBuffers& B, const FrameParams* fp, int launch_flags, cudaStream_t s) {
    if (work_count <= 0) return;
    switch (stage) {
        case kStageWarmStartFirst: launch_stage_warm_start_first(records, ref_rows, work_count, B, fp, launch_flags, s); break;
        case kStageWarmStart: launch_stage_warm_start(records, ref_rows, work_count, B, fp, launch_flags, s); break;
        case kStageSolve: launch_stage_solve(records, ref_rows, work_count, B, fp, launch_flags, s); break;
        case kStageIncremental: launch_stage_t<kStageIncremental>(records, ref_rows, work_count, B, fp, launch_flags, s); break;
        default: break;
    }
}
static void launch_constraint_stage_sharded(int stage, const WorkRecord* records, const int32_t* ref_rows, int work_count, const BodyBuffers& B, const FrameParams* fp, int launch_flags, const ShardPeers& peers,
                                            long long peer_delta, const ShardStage& shard, cudaStream_t s) {
    if (work_count <= 0) return;
    switch (stage) {
        case kStageWarmStartFirst: launch_stage_warm_start_first_sharded(records, ref_rows, work_count, B, fp, launch_flags, peers, peer_delta, shard, s); break;
        case kStageWarmStart: launch_stage_warm_start_sharded(records, ref_rows, work_count, B, fp, launch_flags, peers, peer_delta, shard, s); break;
        case kStageSolve: launch_stage_solve_sharded(records, ref_rows, work_count, B, fp, launch_flags, peers, peer_delta, shard, s); break;
        default: break;
    }
}
static void launch_kinematic_stage(int stage, const int32_t* kinematics, int count, const BodyBuffers& B, const FrameParams* fp, cudaStream_t s) {
    if (count <= 0) return;
    const unsigned blocks = (unsigned)((count + 127) / 128);
    if (stage == kStageKinematicFirst) kinematic_stage_kernel<kStageKinematicFirst><<<blocks, 128, 0, s>>>(kinematics, count, B, fp);
    else kinematic_stage_kernel<kStageKinematic><<<blocks, 128, 0, s>>>(kinematics, count, B, fp);
}
static void launch_final_pose(const BodyBuffers& B, const FrameParams* fp, cudaStream_t s) {
    if (B.count <= 0) return;
    final_pose_kernel<<<(unsigned)((B.count + 255) / 256), 256, 0, s>>>(B, fp);
}
static const bepucuda::SolverLaunchers kLaunchers = {&launch_constraint_stage, &launch_kinematic_stage, &launch_final_pose, &launch_constraint_stage_sharded};
#else
#error "BEPU_UNIT must be 0..3"
#endif

}  // namespace BEPU_NS

#if BEPU_UNIT == 3
namespace bepucuda {
#define BEPU_CAT2(a, b) a##b
#define BEPU_CAT(a, b) BEPU_CAT2(a, b)
const SolverLaunchers* BEPU_CAT(get_launchers_, BEPU_NS)() { return &BEPU_NS::kLaunchers; }
}  // namespace bepucuda
#endif
