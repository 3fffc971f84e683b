// Compiled per numerics flavour (-DBEPU_NS=bepu_fast with FMA contraction / -DBEPU_NS=bepu_strict -fmad=false) and per unit (-DBEPU_UNIT=n),
// so that the big per-type switch of each kernel gets its own translation unit and the build parallelises:
//   0 WarmStartFirst stage   1 WarmStart stage   2 Solve stage   3 Incremental stage + kinematic + final pose + launcher table
#include <atomic>
#include "bepu_solver_kernels.cuh"
#include "bepu_layout_kernels.h"

namespace BEPU_NS {

using StageLauncher = void(const WorkRecord* records, const int32_t* ref_rows, int work_count, const BodyBuffers& B, const FrameParams* fp, int launch_flags,
                           const ShardLaunch* shard, cudaStream_t s);
StageLauncher launch_stage_warm_start_first, launch_stage_warm_start, launch_stage_solve;  // units 0, 1, 2

#ifndef BEPU_DEEP_MINB
#define BEPU_DEEP_MINB 12
#endif
constexpr int kDeepBatchBundles = 2150;  // more bundles than the uncapped build keeps resident at once (132 SMs x 16 warps on an H100 SXM)
// Register budgets of the contact-only stage kernels (kLaunchContactsOnly, below kDeepBatchBundles). The next stage's CTAs can become resident (and
// run their prologue) only in the slots this one leaves free, so the head batches of a 100 k-body pile (1100-1500 bundles, 8-11 warps per SM)
// overlap where 16 warps did not. WarmStart: 10 two-warp CTAs = 20 warps per SM, at most 96 registers, no spills. Solve: 12 CTAs = 24 warps per
// SM at 80 registers (no spills in the fast build); on an H100 it took the Solve stages of the pile 5 % below the 96-register budget, while the
// WarmStart stages at 80 registers spill and were no faster.
#ifndef BEPU_CONTACT_MINB
#define BEPU_CONTACT_MINB 10
#endif
#ifndef BEPU_CONTACT_SOLVE_MINB
#define BEPU_CONTACT_SOLVE_MINB 12
#endif
// Launches one stage kernel instantiation (plain or sharded), one warp per bundle, and `extra_blocks` CTAs after the bundles'.
template <auto Kernel, class... Args>
static void launch_stage_kernel(int work_count, unsigned extra_blocks, int launch_flags, cudaStream_t s, Args... args) {
    static std::atomic<bool> carveout_set[64] = {};  // function attributes are per device: a process may hold contexts on several
    int device = 0;
    cudaGetDevice(&device);
    if (!carveout_set[device & 63]) {  // the staged stages keep one 6 KB slab per resident warp in shared memory
        cudaFuncSetAttribute(Kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        carveout_set[device & 63] = true;
    }
    const unsigned blocks = (unsigned)(((size_t)work_count * 32 + kStageBlockThreads - 1) / kStageBlockThreads) + extra_blocks;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(blocks);
    cfg.blockDim = dim3(kStageBlockThreads);
    cfg.stream = s;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = (launch_flags & bepucuda::kLaunchPdl) ? 1 : 0;
    cudaLaunchKernelEx(&cfg, Kernel, args...);
}
template <int STAGE, int MINB, bool kExt, bool kContacts>
static void launch_stage_instance(const WorkRecord* records, const int32_t* ref_rows, int work_count, const BodyBuffers& B, const FrameParams* fp, int launch_flags, const ShardLaunch* shard,
                                  cudaStream_t s) {
    const bool bodies_integrated = (launch_flags & bepucuda::kLaunchBodiesIntegrated) != 0;
    const int flags = ((launch_flags & bepucuda::kLaunchPrefetchRows) ? kStagePrefetchRows : 0) | ((launch_flags & bepucuda::kLaunchPrefetchBodies) ? kStagePrefetchBodies : 0) |
                      (bodies_integrated ? kStageBodiesIntegrated : 0);
    // the incremental contact update that integrates poses has one thread per body after its bundles (integrate_body_pose)
    const unsigned body_blocks = STAGE == kStageIncremental && bodies_integrated ? (unsigned)((B.count + kStageBlockThreads - 1) / kStageBlockThreads) : 0u;
    if (!shard) launch_stage_kernel<constraint_stage_kernel<STAGE, MINB, kExt, kContacts>>(work_count, body_blocks, launch_flags, s, records, ref_rows, work_count, B, fp, flags);
    else if constexpr (STAGE != kStageIncremental && !kContacts)  // the incremental contact update is never sharded; sharded stages run the full switch
        launch_stage_kernel<constraint_stage_kernel_sharded<STAGE, MINB, kExt>>(work_count, 0u, launch_flags, s, records, ref_rows, work_count, B, fp, flags, shard->peers,
                                                                               shard->peer_delta, shard->stage);
}
// The WarmStart stages integrate: contexts with per-body accelerations or point gravity run their own instantiation (kLaunchIntegratorExtensions).
template <int STAGE, int MINB, bool kContacts>
static void launch_stage_variant(const WorkRecord* records, const int32_t* ref_rows, int work_count, const BodyBuffers& B, const FrameParams* fp, int launch_flags, const ShardLaunch* shard,
                                 cudaStream_t s) {
    if constexpr (STAGE == kStageWarmStartFirst || STAGE == kStageWarmStart) {
        if (launch_flags & bepucuda::kLaunchIntegratorExtensions) return launch_stage_instance<STAGE, MINB, true, kContacts>(records, ref_rows, work_count, B, fp, launch_flags, shard, s);
    }
    launch_stage_instance<STAGE, MINB, false, kContacts>(records, ref_rows, work_count, B, fp, launch_flags, shard, s);
}
template <int STAGE>
static void launch_stage_t(const WorkRecord* records, const int32_t* ref_rows, int work_count, const BodyBuffers& B, const FrameParams* fp, int launch_flags, const ShardLaunch* shard, cudaStream_t s) {
    if constexpr (STAGE != kStageIncremental) {
        if (work_count >= kDeepBatchBundles) return launch_stage_variant<STAGE, BEPU_DEEP_MINB, false>(records, ref_rows, work_count, B, fp, launch_flags, shard, s);
        if (!shard && (launch_flags & bepucuda::kLaunchContactsOnly))
            return launch_stage_variant<STAGE, STAGE == kStageSolve ? BEPU_CONTACT_SOLVE_MINB : BEPU_CONTACT_MINB, true>(records, ref_rows, work_count, B, fp, launch_flags, shard, s);
    }
    launch_stage_variant<STAGE, 1, false>(records, ref_rows, work_count, B, fp, launch_flags, shard, s);
}

#if BEPU_UNIT == 0
void launch_stage_warm_start_first(const WorkRecord* records, const int32_t* ref_rows, int work_count, const BodyBuffers& B, const FrameParams* fp, int launch_flags, const ShardLaunch* shard, cudaStream_t s) {
    launch_stage_t<kStageWarmStartFirst>(records, ref_rows, work_count, B, fp, launch_flags, shard, s);
}
#elif BEPU_UNIT == 1
void launch_stage_warm_start(const WorkRecord* records, const int32_t* ref_rows, int work_count, const BodyBuffers& B, const FrameParams* fp, int launch_flags, const ShardLaunch* shard, cudaStream_t s) {
    launch_stage_t<kStageWarmStart>(records, ref_rows, work_count, B, fp, launch_flags, shard, s);
}
#elif BEPU_UNIT == 2
void launch_stage_solve(const WorkRecord* records, const int32_t* ref_rows, int work_count, const BodyBuffers& B, const FrameParams* fp, int launch_flags, const ShardLaunch* shard, cudaStream_t s) {
    launch_stage_t<kStageSolve>(records, ref_rows, work_count, B, fp, launch_flags, shard, s);
}
#elif BEPU_UNIT == 3
static void launch_constraint_stage(int stage, const WorkRecord* records, const int32_t* ref_rows, int work_count, const BodyBuffers& B, const FrameParams* fp, int launch_flags,
                                    const ShardLaunch* shard, cudaStream_t s) {
    static StageLauncher* const kStages[] = {&launch_stage_warm_start_first, &launch_stage_warm_start, &launch_stage_solve, &launch_stage_t<kStageIncremental>};
    if (work_count > 0 && stage >= kStageWarmStartFirst && stage <= kStageIncremental) kStages[stage](records, ref_rows, work_count, B, fp, launch_flags, shard, s);
}
// The per-body passes, like the WarmStart stages, have an instantiation of their own for per-body accelerations or point gravity.
template <bool kExt> static void launch_kinematic_instance(int stage, const int32_t* kinematics, int count, const BodyBuffers& B, const FrameParams* fp, cudaStream_t s) {
    const unsigned blocks = (unsigned)((count + 127) / 128);
    if (stage == kStageKinematicFirst) kinematic_stage_kernel<kStageKinematicFirst, kExt><<<blocks, 128, 0, s>>>(kinematics, count, B, fp);
    else kinematic_stage_kernel<kStageKinematic, kExt><<<blocks, 128, 0, s>>>(kinematics, count, B, fp);
}
static void launch_kinematic_stage(int stage, const int32_t* kinematics, int count, const BodyBuffers& B, const FrameParams* fp, int launch_flags, cudaStream_t s) {
    if (count <= 0) return;
    if (launch_flags & bepucuda::kLaunchIntegratorExtensions) launch_kinematic_instance<true>(stage, kinematics, count, B, fp, s);
    else launch_kinematic_instance<false>(stage, kinematics, count, B, fp, s);
}
static void launch_final_pose(const BodyBuffers& B, const FrameParams* fp, int launch_flags, cudaStream_t s) {
    if (B.count <= 0) return;
    const unsigned blocks = (unsigned)((B.count + 255) / 256);
    if (launch_flags & bepucuda::kLaunchIntegratorExtensions) final_pose_kernel<true><<<blocks, 256, 0, s>>>(B, fp);
    else final_pose_kernel<false><<<blocks, 256, 0, s>>>(B, fp);
}
static const bepucuda::SolverLaunchers kLaunchers = {&launch_constraint_stage, &launch_kinematic_stage, &launch_final_pose};
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
