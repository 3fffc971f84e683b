// Solver stage kernels (sm_90a): WarmStart (with embedded pose/velocity integration), Solve, IncrementallyUpdateForSubstep,
// the kinematic prepasses and the final pose pass. Included once per numerics flavour (BEPU_NS = bepu_fast with FMA
// contraction, bepu_strict with -fmad=false).
//
// Mapping: one warp = one 32-lane bundle, lane = constraint (TwoBodyTypeProcessor.cs:L176-224 processes one
// Vector<float>.Count-wide bundle per loop trip; here the trip is a warp). Constraint rows are 128-B coalesced lines;
// body state is gathered as 32-B records (two LDG.128 each) straight from L2 (ld.global.cg) — body data is the random
// part of the access pattern and is written by other warps of the same launch sequence, so it never goes through L1.
#pragma once
#include "bepu_contacts.cuh"
#include "bepu_joints_more.cuh"
#include "bepu_integration.cuh"
#include "bepu_device_types.h"

namespace BEPU_NS {

using namespace bepucuda;

// ---- body records: one 32-byte record = one DRAM sector = two back-to-back 128-bit loads/stores (LDG.E.128 / STG.E.128; sm_90 has no wider access)
struct F8 { float a, b, c, d, e, f, g, h; };
// Body records: both halves of a 32-B record are marked evict-last in L2 (and never allocated in L1: other warps of the launch sequence write
// them) so that the body arrays stay L2-resident while the constraint rows stream past them (those are fetched evict-first, see the bulk copies).
// Both halves are issued from one asm statement so that they leave as one pair and fill the same sector. sm_90 takes the evict-last priority
// as an L2 cache policy operand (the bare .L2::evict_last qualifier exists only on the 256-bit accesses of later architectures); the policy asm
// is not volatile so that the compiler can hoist it and share it between accesses.
#define BEPU_BODY_LD "ld.global.L1::no_allocate.L2::cache_hint.v4.f32"
#define BEPU_BODY_ST "st.global.L1::no_allocate.L2::cache_hint.v4.f32"
BEPU_DI uint64_t l2_evict_last_policy() {
    uint64_t policy;
    asm("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(policy));
    return policy;
}
BEPU_DI F8 ld256(const float4* p) {
    F8 r;
    asm volatile(BEPU_BODY_LD " {%0,%1,%2,%3}, [%8], %9;\n\t" BEPU_BODY_LD " {%4,%5,%6,%7}, [%8+16], %9;"
                 : "=f"(r.a), "=f"(r.b), "=f"(r.c), "=f"(r.d), "=f"(r.e), "=f"(r.f), "=f"(r.g), "=f"(r.h)
                 : "l"(p), "l"(l2_evict_last_policy())
                 : "memory");
    return r;
}
BEPU_DI void st256(float4* p, float a, float b, float c, float d, float e, float f, float g, float h) {
    asm volatile(BEPU_BODY_ST " [%0], {%1,%2,%3,%4}, %9;\n\t" BEPU_BODY_ST " [%0+16], {%5,%6,%7,%8}, %9;" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d), "f"(e), "f"(f), "f"(g), "f"(h),
                 "l"(l2_evict_last_policy())
                 : "memory");
}
BEPU_DI void load_velocity(const float4* vel, uint32_t i, Velocity& v) {
    const F8 r = ld256(vel + 2 * (size_t)i);
    v.lin = {r.a, r.b, r.c};
    v.ang = {r.e, r.f, r.g};
}
BEPU_DI void store_velocity(float4* vel, uint32_t i, const Velocity& v) { st256(vel + 2 * (size_t)i, v.lin.x, v.lin.y, v.lin.z, 0.0f, v.ang.x, v.ang.y, v.ang.z, 0.0f); }
BEPU_DI void load_inertia(const float4* in, uint32_t i, Inertia& r) {
    const F8 x = ld256(in + 2 * (size_t)i);
    r.t = {x.a, x.b, x.c, x.d, x.e, x.f};
    r.inv_mass = x.g;
}
BEPU_DI void store_inertia(float4* in, uint32_t i, const Inertia& r) { st256(in + 2 * (size_t)i, r.t.xx, r.t.yx, r.t.yy, r.t.zx, r.t.zy, r.t.zz, r.inv_mass, 0.0f); }
BEPU_DI void load_pose(const float4* pose, uint32_t i, V3& pos, Q4& q) {
    const F8 x = ld256(pose + 2 * (size_t)i);
    q = {x.a, x.b, x.c, x.d};
    pos = {x.e, x.f, x.g};
}
BEPU_DI void store_pose(float4* pose, uint32_t i, V3 pos, Q4 q) { st256(pose + 2 * (size_t)i, q.x, q.y, q.z, q.w, pos.x, pos.y, pos.z, 0.0f); }

// Per-body accelerations and point gravity (FrameParams::integrate_extensions != 0) at one integrating lane, after the declarative callback. Out of
// line, like the momentum-conserving angular modes, and reached only from the kExt instantiations of the WarmStart stages and the per-body
// passes. dt / attractorDt are those of the site's PrepareForIntegration; position is the pose the reference hands the callback there.
static __device__ __noinline__ Velocity integrate_velocity_extensions_at(uint32_t flags, const float4* accelerations, uint32_t idx, V3 lin, V3 ang, float dt, V3 position, V3 center,
                                                                         float attractorDt) {
    Velocity v{lin, ang};
    V3 linearAcceleration{0.0f, 0.0f, 0.0f}, angularAcceleration{0.0f, 0.0f, 0.0f};
    if (flags & kIntegrateAccelerations) {
        const F8 a = ld256(accelerations + 2 * (size_t)idx);
        linearAcceleration = {a.a, a.b, a.c};
        angularAcceleration = {a.e, a.f, a.g};
    }
    integrate_velocity_extensions(v, (flags & kIntegrateAccelerations) != 0, linearAcceleration, angularAcceleration, dt, (flags & kIntegratePointGravity) != 0, position, center,
                                  attractorDt);
    return v;
}
BEPU_DI void apply_velocity_extensions(const FrameParams& fp, uint32_t idx, V3 position, float dt, float attractorDt, Velocity& v) {
    const float4* accelerations = reinterpret_cast<const float4*>((unsigned long long)fp.accelerations[0] | ((unsigned long long)fp.accelerations[1] << 32));
    v = integrate_velocity_extensions_at(fp.integrate_extensions, accelerations, idx, v.lin, v.ang, dt, position, V3{fp.attractor_center[0], fp.attractor_center[1], fp.attractor_center[2]},
                                         attractorDt);
}

// Body records of body slots 0 and 1 that a plain stage kernel loaded before its grid-dependency wait (see constraint_stage_body); bit s of
// `slots` is set when slot s was loaded. kLaunchEarlyWorld: world inertia, and pose for kNeedsPose types. kLaunchEarlyOwned: local inertia and
// pose of an integrating slot.
struct EarlyBodies {
    uint32_t slots;
    Inertia inertia[2];
    V3 pos[2];
    Q4 q[2];
#ifdef BEPU_HAZARD
    Velocity velocity0;  // kCanarySolveVelocity: the velocity of slot 0, gathered before the wait (bit 2 of `slots`)
#endif
};

// GatherAndIntegrate for one body slot of one lane (TypeProcessor.cs:L1298-1397), after the velocity has been loaded. The lane integrates iff the
// device body reference carries kRefIntegrateBit; all other lanes read the world inertia their owner constraint stored earlier in this substep,
// which is bit-identical to what the reference's bundle-wide recompute would give them. kExt: the stage kernel instantiation for contexts with
// per-body accelerations or point gravity (the launcher picks it), so that the default path carries none of it.
// integrated: a WarmStart stage whose pose half the incremental contact update of this substep has done (kLaunchBodiesIntegrated,
// integrate_body_pose): the integrating lane reads the pose and world inertia that update stored and integrates the velocity only. Never in the
// kExt instantiations (resolve_stage_launch).
template <int STAGE, bool NeedsPose, bool kExt>
BEPU_DI void warm_start_body(uint32_t enc, const BodyBuffers& B, const FrameParams& fp, bool integrated, bool early_slot, const EarlyBodies& early, int s, BodyState& b,
                             Velocity& v) {
    const uint32_t idx = enc & kRefIndexMask;
    if (enc & kRefIntegrateBit) {
        if (STAGE == kStageWarmStart && !kExt && integrated) {
            if (early_slot) b.inertia = early.inertia[s];
            else load_inertia(B.inertia_world, idx, b.inertia);
            if (NeedsPose) load_pose(B.pose, idx, b.pos, b.q);
        } else {
            Inertia local;
            if (early_slot) {
                local = early.inertia[s];
                b.pos = early.pos[s];
                b.q = early.q[s];
            } else {
                load_inertia(B.inertia_local, idx, local);
                load_pose(B.pose, idx, b.pos, b.q);
            }
            b.inertia.inv_mass = local.inv_mass;
            if (STAGE == kStageWarmStart) {
                // IntegratePoseAndVelocity, TypeProcessor.cs:L1204-1248
                Q4 previousOrientation = b.q;
                integrate_pose_and_inertia(v.lin, v.ang, fp.dt, local.t, b.pos, b.q, b.inertia.t);
                if (fp.angular_mode == 1) integrate_angular_conserve_momentum(previousOrientation, local.t, b.inertia.t, v.ang);
                else if (fp.angular_mode == 2) integrate_angular_gyroscopic(b.q, local.t, v.ang, fp.dt);
                store_pose(B.pose, idx, b.pos, b.q);
            } else {
                // IntegrateVelocity, TypeProcessor.cs:L1251-1283
                b.inertia.t = rotate_inverse_inertia(local.t, b.q);
                if (fp.angular_mode == 1) {
                    Q4 previousOrientation = integrate_orientation(b.q, v.ang, fp.dt * -0.5f);
                    integrate_angular_conserve_momentum(previousOrientation, local.t, b.inertia.t, v.ang);
                } else if (fp.angular_mode == 2) {
                    integrate_angular_gyroscopic(b.q, local.t, v.ang, fp.dt);
                }
            }
            store_inertia(B.inertia_world, idx, b.inertia);
        }
        callback_integrate_velocity(v, fp.gravity_dt[0], fp.gravity_dt[1], fp.gravity_dt[2], fp.linear_damping_dt, fp.angular_damping_dt);
        // the callback sees the current pose in the first substep and the freshly integrated one after (TypeProcessor.cs:L1244, L1276)
        if constexpr (kExt) apply_velocity_extensions(fp, idx, b.pos, fp.dt, fp.attractor_dt, v);
    } else {
        if (STAGE == kStageWarmStart && !kExt && early_slot) b.inertia = early.inertia[s];  // only ever set for a non-integrating lane when integrated
        else load_inertia(B.inertia_world, idx, b.inertia);
        if (NeedsPose) load_pose(B.pose, idx, b.pos, b.q);
        if (STAGE == kStageWarmStartFirst && fp.angular_mode != 0 && (enc & kRefBundleIntegratesBit) && !(enc & kRefKinematicBit)) {
            // Reference quirk, reproduced for identical results: in the first substep IntegrateVelocity runs the momentum-conserving angular
            // update on EVERY lane of a bundle that contains an integrating lane and only masks the callback afterwards
            // (TypeProcessor.cs:L1259-1281), so non-owning dynamic lanes of such a (host-width) bundle get the update too.
            Inertia local;
            load_inertia(B.inertia_local, idx, local);
            V3 pos;
            Q4 q;
            load_pose(B.pose, idx, pos, q);
            if (fp.angular_mode == 1) integrate_angular_conserve_momentum(integrate_orientation(q, v.ang, fp.dt * -0.5f), local.t, b.inertia.t, v.ang);
            else integrate_angular_gyroscopic(q, local.t, v.ang, fp.dt);
        }
    }
}
template <int STAGE, bool NeedsPose, bool kExt>
BEPU_DI void gather_for_warm_start(uint32_t enc, const BodyBuffers& B, const FrameParams& fp, bool integrated, bool early_slot, const EarlyBodies& early, int s, BodyState& b,
                                   Velocity& v) {
    load_velocity(B.velocity, enc & kRefIndexMask, v);
    warm_start_body<STAGE, NeedsPose, kExt>(enc, B, fp, integrated, early_slot, early, s, b, v);
}

// ---- uniform call shapes over contact and joint types ------------------------------------------------------------------
template <class T, class PR, class AR> BEPU_DI void call_warm_start(const BodyState* b, PR p, AR a, Velocity* v) {
    if constexpr (T::kNeedsPose) T::warm_start(b, p, a, v);
    else if constexpr (T::kBodies == 2) T::warm_start(b[0].inertia, b[1].inertia, p, a, v[0], v[1]);
    else T::warm_start(b[0].inertia, p, a, v[0]);
}
template <class T, class PR, class AR> BEPU_DI void call_solve(const BodyState* b, float dt, float inverseDt, PR p, AR a, Velocity* v) {
    if constexpr (T::kNeedsPose) T::solve(b, dt, inverseDt, p, a, v);
    else if constexpr (T::kBodies == 2) T::solve(b[0].inertia, b[1].inertia, dt, inverseDt, p, a, v[0], v[1]);
    else T::solve(b[0].inertia, dt, inverseDt, p, a, v[0]);
}
template <class T> BEPU_DI void call_incremental(float dt, const Velocity* v, float* p) {
    if constexpr (T::kIncremental) {
        if constexpr (T::kBodies == 2) T::incremental_update(dt, v[0], v[1], p);
        else T::incremental_update(dt, v[0], p);
    }
}

// One constraint lane of one stage. refs addresses this lane in row 0 of the bundle's body references; enc0/enc1 are the (possibly prefetched)
// first two body references; p / a are the row accessors (global or staged); p_rw is the lane's raw prestep pointer for the in-place
// IncrementallyUpdateForSubstep.
BEPU_DI uint32_t ldg_nc_u32(const void* p) {
    uint32_t v;
    asm volatile("ld.global.nc.u32 %0, [%1];" : "=r"(v) : "l"(p));
    return v;
}
// Peer sharding (bepucuda_shard_*): a body another rank references too is also written into that rank's arrays, straight from the registers of
// the lane that computed it (NVLink peer stores; the per-(lane, slot) destination masks sit next to the body references at refs + peer_delta).
BEPU_DI void push_record(float4* const* arrays, uint32_t mask, uint32_t idx, float a, float b, float c, float d, float e, float f, float g, float h) {
    while (mask) {
        const int q = __ffs((int)mask) - 1;
        mask &= mask - 1u;
        float4* dst = arrays[q] + 2 * (size_t)idx;
        dst[0] = make_float4(a, b, c, d);
        dst[1] = make_float4(e, f, g, h);
    }
}
template <class T, int STAGE, bool kSharded, bool kExt, class PR, class AR>
BEPU_DI void run_lane(const int32_t* refs, PR p, AR a, float* p_rw, uint32_t enc0, uint32_t enc1, const BodyBuffers& B, const FrameParams& fp, bool integrated,
                      const EarlyBodies& early, const ShardPeers* peers = nullptr, long long peer_delta = 0) {
    constexpr int NB = T::kBodies;
    uint32_t enc[NB];
    enc[0] = enc0;
    if constexpr (NB > 1) enc[1] = enc1;
#pragma unroll
    for (int s = 2; s < NB; ++s) enc[s] = (uint32_t)__ldg(refs + s * kLanes);
    uint32_t push_to[kSharded ? NB : 1];  // ranks that need what this lane writes to body slot s; interior bundles (peer_delta == 0) have none
    if constexpr (kSharded) {
#pragma unroll
        for (int s = 0; s < NB; ++s) push_to[s] = peer_delta != 0 ? ldg_nc_u32(refs + peer_delta + s * kLanes) : 0u;
    }
    if ((int32_t)enc[0] == kRefEmpty) return;  // trailing lane of the last bundle, or a hole in a fallback bundle
    BodyState b[NB];
    Velocity v[NB];
    if constexpr (STAGE == kStageIncremental) {
#pragma unroll
        for (int s = 0; s < NB; ++s) load_velocity(B.velocity, enc[s] & kRefIndexMask, v[s]);
        call_incremental<T>(fp.dt, v, p_rw);
    } else if constexpr (STAGE == kStageSolve) {
#pragma unroll
        for (int s = 0; s < NB; ++s) {
            const uint32_t idx = enc[s] & kRefIndexMask;
#ifdef BEPU_HAZARD
            if (s == 0 && (early.slots & 4u)) v[s] = early.velocity0;
            else
#endif
                load_velocity(B.velocity, idx, v[s]);
            if (s < 2 && (early.slots >> s & 1u)) {
                b[s].inertia = early.inertia[s & 1];
                if (T::kNeedsPose) b[s].pos = early.pos[s & 1], b[s].q = early.q[s & 1];
            } else {
                load_inertia(B.inertia_world, idx, b[s].inertia);
                if (T::kNeedsPose) load_pose(B.pose, idx, b[s].pos, b[s].q);
            }
        }
        rows_ready(p);
        call_solve<T>(b, fp.dt, fp.inverse_dt, p, a, v);
#pragma unroll
        for (int s = 0; s < NB; ++s)
            if (!(enc[s] & kRefKinematicBit)) {
                store_velocity(B.velocity, enc[s] & kRefIndexMask, v[s]);
                if constexpr (kSharded) {
                    const uint32_t mask = push_to[s];
                    if (mask) push_record(peers->velocity, mask, enc[s] & kRefIndexMask, v[s].lin.x, v[s].lin.y, v[s].lin.z, 0.0f, v[s].ang.x, v[s].ang.y, v[s].ang.z, 0.0f);
                }
            }
    } else {
#pragma unroll
        for (int s = 0; s < NB; ++s) gather_for_warm_start<STAGE, T::kNeedsPose, kExt>(enc[s], B, fp, integrated, s < 2 && (early.slots >> s & 1u), early, s & 1, b[s], v[s]);
        rows_ready(p);
        call_warm_start<T>(b, p, a, v);
#pragma unroll
        for (int s = 0; s < NB; ++s)
            if (!(enc[s] & kRefKinematicBit)) {
                const uint32_t idx = enc[s] & kRefIndexMask;
                store_velocity(B.velocity, idx, v[s]);
                if constexpr (kSharded) {
                    const uint32_t mask = push_to[s];
                    if (mask) {
                        push_record(peers->velocity, mask, idx, v[s].lin.x, v[s].lin.y, v[s].lin.z, 0.0f, v[s].ang.x, v[s].ang.y, v[s].ang.z, 0.0f);
                        if (enc[s] & kRefIntegrateBit) {  // this lane integrated the body: its new world inertia (and pose) travel too
                            const Inertia& in = b[s].inertia;
                            push_record(peers->inertia_world, mask, idx, in.t.xx, in.t.yx, in.t.yy, in.t.zx, in.t.zy, in.t.zz, in.inv_mass, 0.0f);
                            if (STAGE == kStageWarmStart) push_record(peers->pose, mask, idx, b[s].q.x, b[s].q.y, b[s].q.z, b[s].q.w, b[s].pos.x, b[s].pos.y, b[s].pos.z, 0.0f);
                        }
                    }
                }
            }
    }
}

// Work records and body references are loaded with `asm volatile` so that the loads are ISSUED where the source places them (a whole pipeline
// stage before their first use); plain __ldg loads get sunk next to the first use by the compiler and the warp then eats the full latency there.
BEPU_DI int4 ldg_nc_v4(const void* p) {
    int4 v;
    asm volatile("ld.global.nc.v4.s32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}
BEPU_DI WorkRecord load_record(const WorkRecord* r) {
    const int4 lo = ldg_nc_v4(r), hi = ldg_nc_v4(reinterpret_cast<const int4*>(r) + 1);
    WorkRecord w;
    w.refs = reinterpret_cast<int32_t*>((unsigned long long)(unsigned int)lo.x | ((unsigned long long)(unsigned int)lo.y << 32));
    w.prestep = reinterpret_cast<float*>((unsigned long long)(unsigned int)lo.z | ((unsigned long long)(unsigned int)lo.w << 32));
    w.impulses = reinterpret_cast<float*>((unsigned long long)(unsigned int)hi.x | ((unsigned long long)(unsigned int)hi.y << 32));
    w.type_id = hi.z;
    w.live_lanes = hi.w;
    return w;
}

// Type registry: BatchTypeId constants of the reference (Contact/ContactConvexTypes.cs, ContactNonconvexTypes.cs, joint files).
#define BEPU_CONTACT_TYPES(X)                                                                                                     \
    X(0, ConvexOneBody<1>) X(1, ConvexOneBody<2>) X(2, ConvexOneBody<3>) X(3, ConvexOneBody<4>)                                   \
    X(4, ConvexTwoBody<1>) X(5, ConvexTwoBody<2>) X(6, ConvexTwoBody<3>) X(7, ConvexTwoBody<4>)                                   \
    X(8, NonconvexOneBody<2>) X(9, NonconvexOneBody<3>) X(10, NonconvexOneBody<4>)                                                \
    X(15, NonconvexTwoBody<2>) X(16, NonconvexTwoBody<3>) X(17, NonconvexTwoBody<4>)

// kContacts: the switch covers the contact types only (kKernelContacts, for device batches whose every bundle is a contact); it is about half the code of the full switch and fits a smaller register budget (bepu_solver_kernels.cu).
template <int STAGE, bool kSharded, bool kExt, bool kContacts, class PR, class AR>
BEPU_DI void run_bundle_rows(const WorkRecord& rec, int lane, PR p, AR a, uint32_t enc0, uint32_t enc1, const BodyBuffers& B, const FrameParams& fp, bool integrated,
                             const EarlyBodies& early, const ShardPeers* peers = nullptr, long long peer_delta = 0) {
    const int32_t* refs = rec.refs + lane;
    float* p_rw = rec.prestep + lane;
#define BEPU_CASE(ID, T) \
    case ID: run_lane<T, STAGE, kSharded, kExt>(refs, p, a, p_rw, enc0, enc1, B, fp, integrated, early, peers, peer_delta); break;
    if constexpr (kContacts) {
        switch (rec.type_id) {
            BEPU_CONTACT_TYPES(BEPU_CASE)
            default: break;
        }
    } else {
        switch (rec.type_id) {
            BEPU_CONTACT_TYPES(BEPU_CASE)
            BEPU_JOINT_TYPES(BEPU_CASE)
            BEPU_JOINT_TYPES_MORE(BEPU_CASE)
            default: break;
        }
    }
#undef BEPU_CASE
}
// Rows straight from HBM (the incremental stage).
template <int STAGE>
BEPU_DI void run_bundle(const WorkRecord& rec, int lane, uint32_t enc0, uint32_t enc1, const BodyBuffers& B, const FrameParams& fp) {
    run_bundle_rows<STAGE, false, false, false>(rec, lane, GlobalRows{rec.prestep + lane}, GlobalAcc{rec.impulses + lane}, enc0, enc1, B, fp, false, EarlyBodies{});
}
// The reference arena is padded, so reading a second body-reference row is always in bounds (one-body types ignore it).
template <int STAGE> BEPU_DI void run_bundle(const WorkRecord& rec, int lane, const BodyBuffers& B, const FrameParams& fp) {
    const uint32_t enc0 = ldg_nc_u32(rec.refs + lane), enc1 = ldg_nc_u32(rec.refs + kLanes + lane);
    run_bundle<STAGE>(rec, lane, enc0, enc1, B, fp);
}

// ---- bulk staging of one bundle's prestep + accumulated impulse block into shared memory (cp.async.bulk + mbarrier) ----------------
// Block sizes per type id (rows of 128 B), and the body slots and pose use the pre-wait body loads need; 0 for ids without a type.
struct StageRowCounts { uint8_t prestep[64], impulses[64], bodies[64], needs_pose[64]; };
__host__ __device__ constexpr StageRowCounts make_stage_row_counts() {
    StageRowCounts c{};
#define BEPU_ROWS(ID, T) \
    c.prestep[ID] = (uint8_t)T::kPrestepRows; c.impulses[ID] = (uint8_t)T::kImpulseRows; c.bodies[ID] = (uint8_t)T::kBodies; c.needs_pose[ID] = T::kNeedsPose ? 1 : 0;
    BEPU_CONTACT_TYPES(BEPU_ROWS)
    BEPU_JOINT_TYPES(BEPU_ROWS)
    BEPU_JOINT_TYPES_MORE(BEPU_ROWS)
#undef BEPU_ROWS
    return c;
}
__constant__ StageRowCounts kStageRowCounts = make_stage_row_counts();
constexpr int kStageSlabRows = 48;  // >= max(prestep rows + impulse rows) over all types (Contact4Nonconvex: 35 + 12)
constexpr int kStageSlabBytes = kStageSlabRows * kLanes * 4;

BEPU_DI uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
BEPU_DI void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
BEPU_DI void mbar_expect_tx(uint32_t bar, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory"); }
// Constraint rows are touched once per stage and the whole set is far larger than what is reused before the next stage: fetch them evict-first.
BEPU_DI uint64_t l2_evict_first_policy() {
    uint64_t policy;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(policy));
    return policy;
}
BEPU_DI void bulk_copy_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar, uint64_t policy) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(dst), "l"(src), "r"(bytes), "r"(bar),
                 "l"(policy)
                 : "memory");
}

// ---- kernels ------------------------------------------------------------------------------------------------------------
#ifndef BEPU_STAGE_BLOCK_THREADS
#define BEPU_STAGE_BLOCK_THREADS 64
#endif
constexpr int kStageBlockThreads = BEPU_STAGE_BLOCK_THREADS;

// One (batch, stage): one warp per bundle. In the WarmStart / Solve stages the bundle's whole prestep + accumulated-impulse block (contiguous in
// the AOSOA-32 layout) is fetched with ONE cp.async.bulk transaction pair into the warp's shared-memory slab, instead of ~30 dependent row loads
// spread through the constraint math.
//
// Programmatic dependent launch, with the trigger placed AFTER this kernel's own wait: the next stage's grid can start once every CTA here has
// passed `griddepcontrol.wait`, i.e. once the PREVIOUS stage has completed and flushed. So while a kernel runs its pre-wait prologue, everything
// older than its immediate predecessor is final, and the prologue may read whatever that one predecessor does not write: the work record and
// body references (immutable during a solve) always, and what the launch flags say (resolve_stage_launch, DESIGN §3): the whole row block
// (kLaunchPrefetchRows), which takes the bulk copy's latency off the critical path, and the body records of slots 0 and 1 (kLaunchEarlyWorld /
// kLaunchEarlyOwned), so that the post-wait gather is the velocities alone.
template <int STAGE, bool kContacts>
BEPU_DI void load_early_bodies(int type_id, uint32_t enc0, uint32_t enc1, const BodyBuffers& B, EarlyBodies& e) {
    if ((int32_t)enc0 == kRefEmpty) return;
    const int bodies = kStageRowCounts.bodies[type_id];
    const bool pose = !kContacts && kStageRowCounts.needs_pose[type_id];
#pragma unroll
    for (int s = 0; s < 2; ++s) {
        const uint32_t enc = s == 0 ? enc0 : enc1;
        const uint32_t idx = enc & kRefIndexMask;
        if (s >= bodies) break;
        if (STAGE == kStageSolve) {
            load_inertia(B.inertia_world, idx, e.inertia[s]);
            if (pose) load_pose(B.pose, idx, e.pos[s], e.q[s]);
            e.slots |= 1u << s;
        } else if (enc & kRefIntegrateBit) {
            load_inertia(B.inertia_local, idx, e.inertia[s]);
            load_pose(B.pose, idx, e.pos[s], e.q[s]);
            e.slots |= 1u << s;
        }
    }
}
// Arrival counting of the sharded stages (ShardStage). Lanes 0..rank_count-1 of a boundary warp each talk to one peer.
BEPU_DI void shard_announce(const ShardPeers& peers, int lane) {
    if (lane < peers.rank_count && lane != peers.rank)
        asm volatile("red.release.sys.global.add.u64 [%0], 1;" ::"l"(peers.flags[lane] + kShardCounterSlot + peers.rank) : "memory");
}
BEPU_DI void shard_wait(const ShardPeers& peers, int lane, uint32_t solve_index, uint32_t exchange_point, int32_t* error_flag) {
    if (lane < peers.rank_count && lane != peers.rank) {
        const unsigned long long* mine = peers.flags[peers.rank];
        const unsigned long long* targets = mine + kShardTargetSlot + (size_t)lane * kShardMaxExchanges;
        const unsigned long long want = (unsigned long long)solve_index * targets[kShardMaxExchanges - 1] + targets[exchange_point];
        unsigned long long seen;
        unsigned int spins = 0;
        do {
            asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(seen) : "l"(mine + kShardCounterSlot + lane) : "memory");
        } while (seen < want && ++spins < 100000000u);
        if (seen < want) atomicExch(error_flag, 5);  // a peer never arrived: results are void
    }
    __syncwarp();
}
// Body part of the incremental contact update (kLaunchBodiesIntegrated): thread i does the pose half of IntegratePoseAndVelocity
// for body i if a constraint lane integrates it (first_batch set; kinematic bodies have none), so that the WarmStart stage of the body's first
// batch only integrates its velocity. The velocity is loaded after the wait: the predecessor, the last stage of the previous substep, writes it.
// Pose and local inertia are loaded before it: no stage that can precede an incremental update writes them (Solve writes velocities and
// impulses, WarmStartFirst and, with this flag, WarmStart velocities and world inertia only; the kinematic pass of the previous substep, which
// writes kinematic poses, is older than that predecessor).
BEPU_DI void integrate_body_pose(int i, const BodyBuffers& B, const FrameParams* __restrict__ fpp, int flags) {
    const FrameParams fp = *fpp;
    const bool owned = i < B.count && (int32_t)ldg_nc_u32(B.first_batch + i) != 0x7fffffff;
    Inertia local;
    V3 pos;
    Q4 q;
    Velocity v;
    const bool early_velocity = owned && BEPU_CANARY(flags, kCanaryIncrementalVelocity);
    if (owned) {
        load_inertia(B.inertia_local, (uint32_t)i, local);
        load_pose(B.pose, (uint32_t)i, pos, q);
        if (early_velocity) load_velocity(B.velocity, (uint32_t)i, v);
    }
    pdl_wait_then_trigger(flags);
    if (!owned) return;
    if (!early_velocity) load_velocity(B.velocity, (uint32_t)i, v);
    Inertia world;
    world.inv_mass = local.inv_mass;
    integrate_pose_and_inertia(v.lin, v.ang, fp.dt, local.t, pos, q, world.t);
    store_pose(B.pose, (uint32_t)i, pos, q);
    store_inertia(B.inertia_world, (uint32_t)i, world);
}
// kIntegrated: the contact-only WarmStart of the launches with kLaunchBodiesIntegrated (integrated_constraint_stage_kernel). The other contact-only
// WarmStart instantiation is launched only without that flag, so it compiles no integrated path; the full-switch kernels read the flag.
template <int STAGE, bool kSharded, bool kExt, bool kContacts, bool kEarlyBodies, bool kIntegrated = false>
BEPU_DI void constraint_stage_body(const WorkRecord* __restrict__ records, const int32_t* __restrict__ ref_rows, int work_count, const BodyBuffers& B, const FrameParams* __restrict__ fpp, int flags, const ShardPeers* peers,
                                   long long peer_delta, const ShardStage* shard = nullptr) {
    constexpr bool kStaged = STAGE != kStageIncremental;
    constexpr int kWarps = kStageBlockThreads / 32;
    if constexpr (STAGE == kStageIncremental) {
        // the CTAs past the bundles' (launch_stage adds them with kLaunchBodiesIntegrated) hold one thread per body
        const int bundle_blocks = (work_count + kWarps - 1) / kWarps;
        if ((int)blockIdx.x >= bundle_blocks) return integrate_body_pose(((int)blockIdx.x - bundle_blocks) * kStageBlockThreads + (int)threadIdx.x, B, fpp, flags);
    }
    __shared__ __align__(128) float slab[kStaged ? kWarps * kStageSlabRows * kLanes : 1];
    __shared__ __align__(8) unsigned long long bars[kWarps];
    const int warp_in_block = threadIdx.x >> 5;
    const int global_warp = (blockIdx.x * kStageBlockThreads + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    WorkRecord rec{};
    uint32_t enc0 = (uint32_t)kRefEmpty, enc1 = 0;
    const int warp = global_warp;
    const bool active = warp < work_count;
    const uint32_t slab_addr = kStaged ? smem_u32(slab) + warp_in_block * kStageSlabBytes : 0;
    const uint32_t bar = smem_u32(&bars[warp_in_block]);
    const bool early_rows = kStaged && ((flags & kLaunchPrefetchRows) || BEPU_CANARY(flags, kCanaryRowPrefetch));
    uint32_t prestep_bytes = 0, impulse_bytes = 0;
    EarlyBodies early{};
    if (active) {
        rec = load_record(records + warp);
        if constexpr (kStaged) {
            prestep_bytes = kStageRowCounts.prestep[rec.type_id] * (kLanes * 4);
            impulse_bytes = kStageRowCounts.impulses[rec.type_id] * (kLanes * 4);
            if (lane == 0) {
                mbar_init(bar, 1);
                if (early_rows) {
                    const uint64_t policy = l2_evict_first_policy();
                    mbar_expect_tx(bar, prestep_bytes + impulse_bytes);
                    bulk_copy_g2s(slab_addr, rec.prestep, prestep_bytes, bar, policy);
                    bulk_copy_g2s(slab_addr + prestep_bytes, rec.impulses, impulse_bytes, bar, policy);
                }
            }
        }
        // the first two reference rows come from the packed copy next to the work list: their address does not depend on the record (no second round trip)
        enc0 = ldg_nc_u32(ref_rows + (size_t)warp * (2 * kLanes) + lane);
        enc1 = ldg_nc_u32(ref_rows + (size_t)warp * (2 * kLanes) + kLanes + lane);
        if constexpr (kStaged && kEarlyBodies) {
            // world mode on a WarmStart only in the instantiation the host launches it in (the integrated one), owned mode never there
            constexpr bool kWorld = STAGE == kStageSolve || kIntegrated, kOwned = STAGE != kStageSolve && !kIntegrated;
            if (kOwned && (flags & kLaunchEarlyOwned)) load_early_bodies<STAGE, kContacts>(rec.type_id, enc0, enc1, B, early);
            else if (kWorld && ((flags & kLaunchEarlyWorld) || (kIntegrated && BEPU_CANARY(flags, kCanaryEarlyWorldBehindIncremental))))
                load_early_bodies<kStageSolve, kContacts>(rec.type_id, enc0, enc1, B, early);
        }
#ifdef BEPU_HAZARD
        if (STAGE == kStageSolve && BEPU_CANARY(flags, kCanarySolveVelocity) && (int32_t)enc0 != kRefEmpty) {
            load_velocity(B.velocity, enc0 & kRefIndexMask, early.velocity0);
            early.slots |= 4u;
        }
#endif
    }
    const FrameParams fp = *fpp;
    pdl_wait_then_trigger(flags);
    const bool integrated = kIntegrated || (STAGE == kStageWarmStart && !kExt && !kContacts && (flags & kLaunchBodiesIntegrated));
    bool boundary = false;
    if constexpr (kSharded) {
        boundary = active && (rec.live_lanes & kRecordBoundaryBit) != 0;
        // records other ranks pushed in the previous exchange point are read below: all of them must have arrived
        if (boundary && shard->exchange_index > 0 && !BEPU_CANARY(flags, kCanarySkipShardWait)) shard_wait(*peers, lane, fp.shard_solve_index, shard->exchange_index - 1u, shard->error_flag);
    }
    if (!active) return;
    if constexpr (kStaged) {
        if (!early_rows && lane == 0) {
            const uint64_t policy = l2_evict_first_policy();
            mbar_expect_tx(bar, prestep_bytes + impulse_bytes);
            bulk_copy_g2s(slab_addr, rec.prestep, prestep_bytes, bar, policy);
            bulk_copy_g2s(slab_addr + prestep_bytes, rec.impulses, impulse_bytes, bar, policy);
        }
        __syncwarp();
        run_bundle_rows<STAGE, kSharded, kExt, kContacts>(rec, lane, StagedRows{slab_addr + lane * 4, bar, 0u}, StagedAcc{slab_addr + prestep_bytes + lane * 4, rec.impulses + lane}, enc0,
                                                          enc1, B, fp, integrated, early, peers, boundary ? peer_delta : 0);
        if constexpr (kSharded) {
            if (boundary) {
                __syncwarp();                  // every lane's peer stores are ordered before ...
                shard_announce(*peers, lane);  // ... the release that counts the warp as arrived
            }
        }
    } else {
        run_bundle<STAGE>(rec, lane, enc0, enc1, B, fp);
    }
}

// The pre-wait body loads are compiled into the uncapped and the contact-only budgets. The deep budget (full switch at 80 registers) would spill
// with them, and a batch several waves deep has only its first wave's CTAs in a prologue while the predecessor runs; the host never asks for them there.
template <int STAGE, int MINB, bool kExt, bool kContacts>
__global__ void __launch_bounds__(kStageBlockThreads, MINB) constraint_stage_kernel(const WorkRecord* __restrict__ records, const int32_t* __restrict__ ref_rows, int work_count, BodyBuffers B, const FrameParams* __restrict__ fpp, int flags) {
    constraint_stage_body<STAGE, false, kExt, kContacts, MINB == 1 || kContacts>(records, ref_rows, work_count, B, fpp, flags, nullptr, 0);
}
// The contact-only WarmStart of the launches whose poses and world inertias the incremental update of the substep integrated
// (integrated_warm_start_launch, bepu_topology.h): its integrating lanes integrate velocity only, so it carries no pose integration, no angular-mode
// branch and no local-inertia or pose load, about 40 % of the code of the integrating instantiation. It takes the template arguments of
// constraint_stage_kernel, so that tools which read kernel names (tests/tools/stage_timeline.py) see one more contact-only WarmStart.
template <int STAGE, int MINB, bool kExt, bool kContacts>
__global__ void __launch_bounds__(kStageBlockThreads, MINB) integrated_constraint_stage_kernel(const WorkRecord* __restrict__ records, const int32_t* __restrict__ ref_rows, int work_count, BodyBuffers B, const FrameParams* __restrict__ fpp, int flags) {
    static_assert(STAGE == kStageWarmStart && !kExt && kContacts, "integrated WarmStart launches are contact-only and never carry kExt");
    constraint_stage_body<STAGE, false, false, true, true, true>(records, ref_rows, work_count, B, fpp, flags, nullptr, 0);
}
// Peer-sharded variant (bepucuda_shard_*): the lane that writes a body another rank references stores the record into that rank's arrays too.
template <int STAGE, int MINB, bool kExt>
__global__ void __launch_bounds__(kStageBlockThreads, MINB)
constraint_stage_kernel_sharded(const WorkRecord* __restrict__ records, const int32_t* __restrict__ ref_rows, int work_count, BodyBuffers B, const FrameParams* __restrict__ fpp, int flags, const __grid_constant__ ShardPeers peers,
                                long long peer_delta, const __grid_constant__ ShardStage shard) {
    constraint_stage_body<STAGE, true, kExt, false, false>(records, ref_rows, work_count, B, fpp, flags, &peers, peer_delta, &shard);
}

#if BEPU_UNIT == 3  // the per-body passes are launched from unit 3 only
// IntegrateKinematicVelocities / IntegrateKinematicPosesAndVelocities (PoseIntegrator.cs:L451-487, L493-535)
template <int STAGE, bool kExt> BEPU_DI void run_kinematic(int i, const int32_t* kinematics, const BodyBuffers& B, const FrameParams& fp) {
    const uint32_t idx = (uint32_t)kinematics[i];
    Velocity v;
    load_velocity(B.velocity, idx, v);
    V3 pos{0.0f, 0.0f, 0.0f};
    Q4 q;
    if (STAGE == kStageKinematic) {
        load_pose(B.pose, idx, pos, q);
        pos = pos + v.lin * fp.dt;
        q = integrate_orientation(q, v.ang, fp.dt * 0.5f);
        store_pose(B.pose, idx, pos, q);
    }
    if (fp.integrate_velocity_for_kinematics) {
        callback_integrate_velocity(v, fp.gravity_dt[0], fp.gravity_dt[1], fp.gravity_dt[2], fp.linear_damping_dt, fp.angular_damping_dt);
        if constexpr (kExt) {
            // the callback sees the gathered pose in the first substep (PoseIntegrator.cs:L480) and the integrated one after (L529)
            if (STAGE == kStageKinematicFirst && (fp.integrate_extensions & kIntegratePointGravity)) load_pose(B.pose, idx, pos, q);
            apply_velocity_extensions(fp, idx, pos, fp.dt, fp.attractor_dt, v);
        }
        store_velocity(B.velocity, idx, v);
    }
}
template <int STAGE, bool kExt>
__global__ void kinematic_stage_kernel(const int32_t* __restrict__ kinematics, int count, BodyBuffers B, const FrameParams* __restrict__ fpp) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const FrameParams fp = *fpp;
    run_kinematic<STAGE, kExt>(i, kinematics, B, fp);
}

// IntegrateBundlesAfterSubstepping (PoseIntegrator.cs:L537-693), per body.
template <bool kExt> BEPU_DI void run_final_pose(int i, const BodyBuffers& B, const FrameParams& fp) {
    V3 pos;
    Q4 q;
    Velocity v;
    load_pose(B.pose, i, pos, q);
    load_velocity(B.velocity, i, v);
    if (B.constrained[i]) {
        // constrained bodies: the one trailing pose integration of (velocity -> solve) -> (pose -> velocity -> solve) ... -> pose
        q = integrate_orientation(q, v.ang, fp.dt * 0.5f);
        pos = pos + v.lin * fp.dt;
        store_pose(B.pose, i, pos, q);
        return;
    }
    Inertia local;
    load_inertia(B.inertia_local, i, local);
    const bool kinematic = local.inv_mass == 0.0f && local.t.xx == 0.0f && local.t.yx == 0.0f && local.t.yy == 0.0f && local.t.zx == 0.0f && local.t.zy == 0.0f && local.t.zz == 0.0f;
    const bool integrateVelocity = fp.integrate_velocity_for_kinematics || !kinematic;
    const float dt = fp.final_dt, halfDt = fp.final_dt * 0.5f;
    for (int step = 0; step < fp.final_steps; ++step) {
        if (integrateVelocity) {
            callback_integrate_velocity(v, fp.final_gravity_dt[0], fp.final_gravity_dt[1], fp.final_gravity_dt[2], fp.final_linear_damping_dt, fp.final_angular_damping_dt);
            if constexpr (kExt) apply_velocity_extensions(fp, i, pos, dt, fp.final_attractor_dt, v);  // the position before this step's update
        }
        pos = pos + v.lin * dt;
        if (fp.angular_mode == 1) {
            Q4 previousOrientation = q;
            q = integrate_orientation(q, v.ang, halfDt);
            integrate_angular_conserve_momentum(previousOrientation, local.t, rotate_inverse_inertia(local.t, q), v.ang);
        } else if (fp.angular_mode == 2) {
            q = integrate_orientation(q, v.ang, halfDt);
            integrate_angular_gyroscopic(q, local.t, v.ang, dt);
        } else {
            q = integrate_orientation(q, v.ang, halfDt);
        }
    }
    store_pose(B.pose, i, pos, q);
    if (integrateVelocity) store_velocity(B.velocity, i, v);
}
template <bool kExt> static __global__ void final_pose_kernel(BodyBuffers B, const FrameParams* __restrict__ fpp) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B.count) return;
    const FrameParams fp = *fpp;
    run_final_pose<kExt>(i, B, fp);
}
#endif

}  // namespace BEPU_NS
