// Host-side mirror of the slice of bepuphysics2 that sits directly above the solver hot path, written in C++ because the
// reference's own host language (C#/.NET 8) has no toolchain in this image. It owns the same raw buffers the reference
// owns (Bodies.ActiveSet.DynamicsState as 128-B AOS, Solver.ActiveSet.Batches[b].TypeBatches[t] as AOSOA-W) and feeds them
// to libbepucuda through exactly the C ABI a C# CudaTimestepper would P/Invoke (include/bepucuda.h, INTEGRATION.md).
//
// Mirrored (names kept): Bodies.Add and Bodies.RemoveAt with the handle pool and HandleToLocation (Bodies.cs:L183-260, BodySet.cs:L68-111),
// Solver.UpdateForBodyMemoryMove (Solver.cs:L1444-1482), Solver.Add -> TryAllocateInBatch -> AllocateInTypeBatch[ForFallback]
// (Solver.cs:L1093-1199, Constraints/TypeProcessor.cs:L314-334,L451-540), ConstrainedKinematicHandles (Solver.cs:L68),
// SolveDescription (SolveDescription.cs:L16-137), ITimestepper.Timestep's Solve slot (DefaultTimestepper.cs:L28-43), Solver.Remove ->
// RemoveFromBatch -> TypeProcessor.Remove, RemoveTypeBatchIfEmpty, RemoveBatchIfEmpty (Solver.cs:L1294-1405, TypeProcessor.cs:L634-720,
// ConstraintBatch.cs:L170-185).
// Not mirrored: sleeping, batch compression, collision detection (out of scope, SURVEY.md §2).
#include <algorithm>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <new>
#include <string>
#include <vector>

#include "../../../include/bepucuda.h"
#include "../bepu_type_table.h"

namespace {

constexpr uint32_t kKinematicMask = 1u << 30;  // Bodies_GatherScatter.cs:L109-110

template <class T> struct AlignedBuffer {  // BufferPool hands out 128-B aligned blocks carved from large pages (BufferPool.cs:L42); page-granular here so
                                          // that every buffer can be page-locked on its own (cudaHostRegister pins whole pages)
    T* data = nullptr;
    size_t capacity = 0;
    ~AlignedBuffer() { std::free(data); }
    void ensure(size_t count, size_t used) {
        if (count <= capacity) return;
        size_t cap = std::max<size_t>(count, capacity * 2);
        cap = std::max<size_t>(cap, 64);
        size_t bytes = ((cap * sizeof(T) + 4095) / 4096) * 4096;
        T* n = (T*)std::aligned_alloc(4096, bytes);
        if (!n) throw std::bad_alloc();
        std::memset(n, 0, bytes);
        if (data) std::memcpy(n, data, used * sizeof(T));
        std::free(data);
        data = n;
        capacity = bytes / sizeof(T);
    }
};

struct TypeBatch {  // Constraints/TypeBatch.cs:L10-27
    int type_id = -1;
    int bodies = 0, prestep_rows = 0, impulse_rows = 0;
    int constraint_count = 0;  // ConstraintCount (includes holes in the fallback batch)
    AlignedBuffer<int32_t> body_references;
    AlignedBuffer<float> prestep;
    AlignedBuffer<float> impulses;
    std::vector<int32_t> index_to_handle;
    int bundle_count(int W) const { return (constraint_count + W - 1) / W; }
    void ensure_bundles(int bundles, int W) {
        int used = bundle_count(W);
        body_references.ensure((size_t)bundles * bodies * W, (size_t)used * bodies * W);
        prestep.ensure((size_t)bundles * prestep_rows * W, (size_t)used * prestep_rows * W);
        impulses.ensure((size_t)bundles * impulse_rows * W, (size_t)used * impulse_rows * W);
    }
};

struct ConstraintBatch {  // ConstraintBatch.cs:L14-49
    std::vector<TypeBatch*> type_batches;
    int type_index_to_type_batch_index[64];
    ConstraintBatch() { std::fill(type_index_to_type_batch_index, type_index_to_type_batch_index + 64, -1); }
    ~ConstraintBatch() { for (auto t : type_batches) delete t; }
};

struct IndexSet {  // BepuUtilities/Collections/IndexSet.cs
    std::vector<uint64_t> flags;
    bool contains(int i) const { size_t w = (size_t)i >> 6; return w < flags.size() && ((flags[w] >> (i & 63)) & 1); }
    void set(int i) { size_t w = (size_t)i >> 6; if (w >= flags.size()) flags.resize(w + 1, 0); flags[w] |= (uint64_t)1 << (i & 63); }
    void unset(int i) { size_t w = (size_t)i >> 6; if (w < flags.size()) flags[w] &= ~((uint64_t)1 << (i & 63)); }
};

struct ConstraintLocation { int batch, type_id, index_in_type_batch; };  // batch -1: a removed handle

// One Solver.Add / Solver.Remove / Bodies.Add / Bodies.RemoveAt since the last describe or bepuhost_cuda_change, for bepuhost_cuda_change. A
// constraint entry: the location the call produced or consumed, and for an add its handle and encoded body references. A body add: its handle, and
// once that body is removed again its record as it was then. A body remove: the active-set index it removed. The last entry of a constraint run
// that another kind of entry follows keeps the constrained kinematics (active-set indices) as they were right after the run (`kinematics`).
enum ChangeKind { kConstraintAdd, kConstraintRemove, kBodyAdd, kBodyRemove };
struct ChangeEntry {
    ChangeKind kind;
    ConstraintLocation at;
    int handle;
    int32_t refs[4];
    std::vector<float> record;
    std::vector<int32_t> kinematics;
    bool kinematics_kept = false;
};

struct Simulation {
    int W;                       // Vector<float>.Count of the emulated host
    int fallback_batch_threshold;
    std::vector<int32_t> velocity_iterations;  // per substep
    bepucuda_integrator_desc integrator{};
    AlignedBuffer<float> dynamics;             // Bodies.ActiveSet.DynamicsState: 32 floats per body
    int body_count = 0;
    std::vector<int32_t> index_to_handle;      // Bodies.ActiveSet.IndexToHandle
    std::vector<int32_t> handle_to_index;      // Bodies.HandleToLocation (active set only; -1: no body)
    std::vector<int32_t> free_handles;         // Bodies.HandlePool's returned ids, taken last-in first-out (IdPool.Take)
    std::vector<ConstraintBatch*> batches;     // Solver.ActiveSet.Batches
    std::vector<IndexSet> batch_referenced_handles;  // by body handle
    std::vector<int32_t> constrained_kinematic_handles;
    IndexSet constrained_kinematic_set;
    std::vector<ConstraintLocation> handle_to_constraint;
    std::vector<int32_t> kinematic_constraint_count;  // per body handle: constraints referencing it as a kinematic (Bodies' constraint lists, kinematics only)
    std::vector<ChangeEntry> changes;
    std::vector<int32_t> kinematic_indices;   // constrained_kinematic_handles as active-set indices (kinematic_indices())
    std::string error;
    ~Simulation() { for (auto b : batches) delete b; }
};

bool is_kinematic(const float* body) {  // Bodies.cs:L339-353: all of local inverse inertia + inverse mass are zero
    for (int i = 16; i < 23; ++i)
        if (body[i] != 0.0f) return false;
    return true;
}

// The constrained kinematics as active-set indices: what the device takes.
const std::vector<int32_t>& kinematic_indices(Simulation& sim) {
    sim.kinematic_indices.clear();
    for (const int32_t h : sim.constrained_kinematic_handles) sim.kinematic_indices.push_back(sim.handle_to_index[(size_t)h]);
    return sim.kinematic_indices;
}

// Appends an entry of `kind` to the change log; a constraint run that this entry ends keeps the constrained kinematics it left.
ChangeEntry& log_change(Simulation& sim, ChangeKind kind) {
    if (!sim.changes.empty()) {
        ChangeEntry& last = sim.changes.back();
        if (last.kind != kind && (last.kind == kConstraintAdd || last.kind == kConstraintRemove)) {
            last.kinematics = kinematic_indices(sim);
            last.kinematics_kept = true;
        }
    }
    sim.changes.push_back({});
    sim.changes.back().kind = kind;
    return sim.changes.back();
}

TypeBatch* get_or_create_type_batch(Simulation& sim, ConstraintBatch& batch, int type_id) {
    int& idx = batch.type_index_to_type_batch_index[type_id];
    if (idx >= 0) return batch.type_batches[idx];
    int32_t nb = 0, p = 0, d = 0;
    if (bepucuda_type_info(type_id, &nb, &p, &d) != BEPUCUDA_OK) return nullptr;
    TypeBatch* t = new TypeBatch();
    t->type_id = type_id; t->bodies = nb; t->prestep_rows = p; t->impulse_rows = d;
    idx = (int)batch.type_batches.size();
    batch.type_batches.push_back(t);
    return t;
}

void write_lane(Simulation& sim, TypeBatch& t, int index, const int32_t* encoded, const float* prestep) {
    const int W = sim.W;
    const int bundle = index / W, inner = index % W;
    if (inner == 0 || index >= t.constraint_count) {
        // first lane of a (possibly new) bundle: all body references of the bundle start at -1 (TypeProcessor.cs:L287-296)
    }
    int32_t* refs = t.body_references.data + (size_t)bundle * t.bodies * W;
    for (int b = 0; b < t.bodies; ++b) refs[b * W + inner] = encoded[b];
    float* p = t.prestep.data + (size_t)bundle * t.prestep_rows * W;
    for (int r = 0; r < t.prestep_rows; ++r) p[r * W + inner] = prestep[r];
    float* a = t.impulses.data + (size_t)bundle * t.impulse_rows * W;
    for (int r = 0; r < t.impulse_rows; ++r) a[r * W + inner] = 0.0f;  // ClearLane (TypeProcessor.cs:L327)
}

void init_new_bundle(Simulation& sim, TypeBatch& t, int bundle) {
    const int W = sim.W;
    int32_t* refs = t.body_references.data + (size_t)bundle * t.bodies * W;
    for (int i = 0; i < t.bodies * W; ++i) refs[i] = -1;
    std::memset(t.prestep.data + (size_t)bundle * t.prestep_rows * W, 0, sizeof(float) * t.prestep_rows * W);
    std::memset(t.impulses.data + (size_t)bundle * t.impulse_rows * W, 0, sizeof(float) * t.impulse_rows * W);
}

// AllocateInTypeBatch (TypeProcessor.cs:L314-334)
int allocate_in_type_batch(Simulation& sim, TypeBatch& t, int handle) {
    const int W = sim.W;
    const int index = t.constraint_count;
    if (index % W == 0) {
        t.ensure_bundles(index / W + 1, W);
        init_new_bundle(sim, t, index / W);
    }
    t.constraint_count = index + 1;
    t.index_to_handle.resize(t.constraint_count, -1);
    t.index_to_handle[index] = handle;
    return index;
}

// AllocateInTypeBatchForFallback (TypeProcessor.cs:L451-540): a constraint may not share a bundle with any of its dynamic
// bodies; probe the last bundle, then up to 16 strided bundles, then open a new bundle.
int allocate_in_type_batch_for_fallback(Simulation& sim, TypeBatch& t, int handle, const int32_t* encoded) {
    const int W = sim.W;
    const int bundles = t.bundle_count(W);
    auto probe = [&](int bundle) -> int {
        const int32_t* refs = t.body_references.data + (size_t)bundle * t.bodies * W;
        for (int b = 0; b < t.bodies; ++b) {
            const int32_t mine = encoded[b] & ~(int32_t)kKinematicMask;
            if ((uint32_t)encoded[b] & kKinematicMask) continue;  // kinematics never block
            for (int i = 0; i < t.bodies * W; ++i)
                if (refs[i] == mine) return -1;
        }
        for (int l = 0; l < W; ++l)
            if (refs[l] < 0) return l;  // a free lane (first body slot is -1)
        return -1;
    };
    int target_bundle = -1, target_inner = -1;
    if (bundles > 0) {
        const int probe_count = 16;
        if (bundles <= probe_count + 1) {
            for (int k = 0; k < bundles && target_bundle < 0; ++k) {
                int l = probe(k);
                if (l >= 0) { target_bundle = k; target_inner = l; }
            }
        } else {
            int l = probe(bundles - 1);
            if (l >= 0) { target_bundle = bundles - 1; target_inner = l; }
            else {
                const int last = bundles - 1;
                int next = (int)(((uint32_t)handle * 2654435761u) & 0x7fffffffu) % last;
                const int jump = bundles / probe_count;
                const int remainder = last - jump * probe_count;
                for (int pi = 0; pi < probe_count; ++pi) {
                    l = probe(next);
                    if (l >= 0) { target_bundle = next; target_inner = l; break; }
                    next += jump;
                    if (pi < remainder) ++next;
                    if (next >= bundles) next -= bundles;
                }
            }
        }
    }
    if (target_bundle < 0) {
        t.ensure_bundles(bundles + 1, W);
        init_new_bundle(sim, t, bundles);
        const int index = bundles * W;
        t.constraint_count = index + 1;
        t.index_to_handle.resize(t.constraint_count, -1);
        t.index_to_handle[index] = handle;
        return index;
    }
    const int index = target_bundle * W + target_inner;
    if (index >= t.constraint_count) t.constraint_count = index + 1;
    t.index_to_handle.resize(std::max<size_t>(t.index_to_handle.size(), (size_t)t.constraint_count), -1);
    t.index_to_handle[index] = handle;
    return index;
}

// GetBlockingBodyHandles (Solver.cs:L1058-1078): encodes the body references (active-set index, kinematic flag in bit 30) and lists the dynamic
// handles, the only ones that take part in batch membership.
int encode_references(Simulation& sim, int type_id, const int32_t* body_handles, int32_t* encoded, int32_t* blocking, int* blocking_count, int* body_count_out) {
    int32_t nb = 0;
    if (bepucuda_type_info(type_id, &nb, nullptr, nullptr) != BEPUCUDA_OK) { sim.error = "unsupported constraint type"; return -1; }
    *blocking_count = 0;
    for (int i = 0; i < nb; ++i) {
        const int h = body_handles[i];
        if (h < 0 || h >= (int)sim.handle_to_index.size() || sim.handle_to_index[(size_t)h] < 0) { sim.error = "body handle out of range"; return -1; }
        const int index = sim.handle_to_index[(size_t)h];
        if (is_kinematic(sim.dynamics.data + (size_t)index * 32)) encoded[i] = index | (int32_t)kKinematicMask;
        else { encoded[i] = index; blocking[(*blocking_count)++] = h; }
    }
    *body_count_out = nb;
    return 0;
}

// AllocateInBatch (Solver.cs:L1016-1056) into a batch that is known to fit.
int allocate_in_batch(Simulation& sim, int target, int type_id, int nb, const int32_t* encoded, const int32_t* blocking, int blocking_count, const float* prestep) {
    const int handle = (int)sim.handle_to_constraint.size();
    for (int i = 0; i < nb; ++i)
        if ((uint32_t)encoded[i] & kKinematicMask) {
            const int h = sim.index_to_handle[(size_t)(encoded[i] & ~(int32_t)kKinematicMask)];
            if (!sim.constrained_kinematic_set.contains(h)) { sim.constrained_kinematic_set.set(h); sim.constrained_kinematic_handles.push_back(h); }
            if ((int)sim.kinematic_constraint_count.size() <= h) sim.kinematic_constraint_count.resize((size_t)h + 1, 0);
            ++sim.kinematic_constraint_count[(size_t)h];
        }
    TypeBatch* tb = get_or_create_type_batch(sim, *sim.batches[target], type_id);
    if (!tb) { sim.error = "unsupported constraint type"; return -1; }
    int index = target == sim.fallback_batch_threshold ? allocate_in_type_batch_for_fallback(sim, *tb, handle, encoded) : allocate_in_type_batch(sim, *tb, handle);
    write_lane(sim, *tb, index, encoded, prestep);
    for (int i = 0; i < blocking_count; ++i) sim.batch_referenced_handles[target].set(blocking[i]);
    sim.handle_to_constraint.push_back({target, type_id, index});
    ChangeEntry& e = log_change(sim, kConstraintAdd);
    e.at = {target, type_id, index};
    e.handle = handle;
    for (int i = 0; i < 4; ++i) e.refs[i] = i < nb ? encoded[i] : -1;
    return handle;
}

// Moves lane `from` of `t` into lane `to` (TypeProcessor.Move / whole-bundle pulls): body references, prestep, impulses, and the handle's location.
void move_lane(Simulation& sim, TypeBatch& t, int from, int to) {
    const int W = sim.W;
    auto lane = [&](auto* data, int rows, int index, int r) -> auto& { return data[((size_t)(index / W) * rows + r) * W + index % W]; };
    for (int r = 0; r < t.bodies; ++r) lane(t.body_references.data, t.bodies, to, r) = lane(t.body_references.data, t.bodies, from, r);
    for (int r = 0; r < t.prestep_rows; ++r) lane(t.prestep.data, t.prestep_rows, to, r) = lane(t.prestep.data, t.prestep_rows, from, r);
    for (int r = 0; r < t.impulse_rows; ++r) lane(t.impulses.data, t.impulse_rows, to, r) = lane(t.impulses.data, t.impulse_rows, from, r);
    const int handle = t.index_to_handle[(size_t)from];
    t.index_to_handle[(size_t)to] = handle;
    t.index_to_handle[(size_t)from] = -1;
    if (handle >= 0) sim.handle_to_constraint[(size_t)handle].index_in_type_batch = to;
}
void clear_lane_references(Simulation& sim, TypeBatch& t, int index) {  // RemoveBodyReferencesLane
    for (int r = 0; r < t.bodies; ++r) t.body_references.data[((size_t)(index / sim.W) * t.bodies + r) * sim.W + index % sim.W] = -1;
}

// Solver.Remove (Solver.cs:L1385-1405): the bodies' kinematic bookkeeping, RemoveFromBatch (L1344-1358) with TypeProcessor.Remove (TypeProcessor.cs:
// L634-720), RemoveTypeBatchIfEmpty (ConstraintBatch.cs:L170-185) and RemoveBatchIfEmpty (Solver.cs:L1294-1336).
int solver_remove(Simulation& sim, int handle) {
    if (handle < 0 || handle >= (int)sim.handle_to_constraint.size() || sim.handle_to_constraint[(size_t)handle].batch < 0) { sim.error = "no such constraint handle"; return -1; }
    const ConstraintLocation at = sim.handle_to_constraint[(size_t)handle];
    ChangeEntry& logged = log_change(sim, kConstraintRemove);
    logged.at = at;
    logged.handle = handle;
    ConstraintBatch& batch = *sim.batches[(size_t)at.batch];
    const int tb_index = batch.type_index_to_type_batch_index[at.type_id];
    TypeBatch& t = *batch.type_batches[(size_t)tb_index];
    const int W = sim.W, index = at.index_in_type_batch;
    const int32_t* refs = t.body_references.data + (size_t)(index / W) * t.bodies * W + index % W;
    for (int b = 0; b < t.bodies; ++b) {
        const int32_t enc = refs[(size_t)b * W];
        const int body = sim.index_to_handle[(size_t)(enc & ~(int32_t)kKinematicMask)];
        if ((uint32_t)enc & kKinematicMask) {
            // RemoveConstraintReferencesFromBodiesEnumerator: the last constraint of a kinematic takes it out of ConstrainedKinematicHandles (FastRemove)
            if (--sim.kinematic_constraint_count[(size_t)body] == 0) {
                auto& list = sim.constrained_kinematic_handles;
                const auto it = std::find(list.begin(), list.end(), body);
                *it = list.back();
                list.pop_back();
                sim.constrained_kinematic_set.unset(body);
            }
        } else if (at.batch < sim.fallback_batch_threshold) {
            sim.batch_referenced_handles[(size_t)at.batch].unset(body);  // RemoveBodyHandlesFromBatchForConstraint
        }
    }
    if (at.batch == sim.fallback_batch_threshold) {
        // The fallback batch's body set decides nothing here (it accepts every constraint), so it is not kept up to date.
        t.index_to_handle[(size_t)index] = -1;
        clear_lane_references(sim, t, index);
        const int removed_bundle = index / W;
        bool empty = true;
        for (int l = 0; l < W; ++l) empty = empty && t.body_references.data[(size_t)removed_bundle * t.bodies * W + l] < 0;
        if (empty) {
            int last = t.bundle_count(W) - 1;
            if (removed_bundle != last) {
                for (int l = 0; l < W; ++l) {
                    const int from = last * W + l;
                    if (from < t.constraint_count && t.body_references.data[(size_t)last * t.bodies * W + l] >= 0) move_lane(sim, t, from, removed_bundle * W + l);
                    else {  // a hole moves as it is: its body references
                        for (int r = 0; r < t.bodies; ++r) t.body_references.data[((size_t)removed_bundle * t.bodies + r) * W + l] = t.body_references.data[((size_t)last * t.bodies + r) * W + l];
                    }
                }
                --last;
            }
            int lanes = 0;
            for (int l = 0; l < W; ++l)
                if (last >= 0 && t.body_references.data[(size_t)last * t.bodies * W + l] >= 0) lanes = l + 1;
            t.constraint_count = std::max(last, 0) * W + lanes;
            t.index_to_handle.resize((size_t)t.constraint_count);
        }
    } else {
        const int last = t.constraint_count - 1;
        if (index < last) move_lane(sim, t, last, index);
        else t.index_to_handle[(size_t)index] = -1;
        clear_lane_references(sim, t, last);
        t.constraint_count = last;
        t.index_to_handle.resize((size_t)last);
    }
    sim.handle_to_constraint[(size_t)handle] = {-1, -1, -1};
    if (t.constraint_count == 0) {
        batch.type_index_to_type_batch_index[at.type_id] = -1;
        delete batch.type_batches[(size_t)tb_index];
        batch.type_batches[(size_t)tb_index] = batch.type_batches.back();
        batch.type_batches.pop_back();
        if (tb_index < (int)batch.type_batches.size()) batch.type_index_to_type_batch_index[batch.type_batches[(size_t)tb_index]->type_id] = tb_index;
        if (at.batch == (int)sim.batches.size() - 1)
            while (!sim.batches.empty() && sim.batches.back()->type_batches.empty()) {
                delete sim.batches.back();
                sim.batches.pop_back();
                sim.batch_referenced_handles.pop_back();
            }
    }
    return 0;
}

// Solver.Add (Solver.cs:L1182-1199): greedy first fit over batches; kinematics never block (GetBlockingBodyHandles L1058-1078);
// batch index == FallbackBatchThreshold is the fallback batch and accepts everything (TryAllocateInBatch L1093-1140).
int solver_add(Simulation& sim, int type_id, const int32_t* body_handles, const float* prestep) {
    int32_t encoded[4], blocking[4];
    int blocking_count = 0, nb = 0;
    if (encode_references(sim, type_id, body_handles, encoded, blocking, &blocking_count, &nb) != 0) return -1;
    for (int target = 0; target <= (int)sim.batches.size(); ++target) {
        if (target == (int)sim.batches.size()) {
            sim.batches.push_back(new ConstraintBatch());
            sim.batch_referenced_handles.emplace_back();
        } else if (target < sim.fallback_batch_threshold) {
            bool fits = true;
            for (int i = 0; i < blocking_count; ++i) fits = fits && !sim.batch_referenced_handles[target].contains(blocking[i]);
            if (!fits) continue;
        }
        return allocate_in_batch(sim, target, type_id, nb, encoded, blocking, blocking_count, prestep);
    }
    sim.error = "constraint add failed";
    return -1;
}

// The add path of callers that already know the batch (the narrow phase: FindCandidateBatch, then TryAllocateInBatch at that index,
// Solver.cs:L984-1014, L1093-1140; here: a batch index computed by bepucuda_color_constraints). Fails if the batch cannot hold the constraint.
int solver_add_in_batch(Simulation& sim, int target, int type_id, const int32_t* body_handles, const float* prestep) {
    int32_t encoded[4], blocking[4];
    int blocking_count = 0, nb = 0;
    if (encode_references(sim, type_id, body_handles, encoded, blocking, &blocking_count, &nb) != 0) return -1;
    if (target < 0 || target > sim.fallback_batch_threshold) { sim.error = "batch index out of range"; return -1; }
    while ((int)sim.batches.size() <= target) {  // empty batches may sit between occupied ones (the reference tolerates them too, Solver_Solve.cs:L794-796)
        sim.batches.push_back(new ConstraintBatch());
        sim.batch_referenced_handles.emplace_back();
    }
    if (target < sim.fallback_batch_threshold)
        for (int i = 0; i < blocking_count; ++i)
            if (sim.batch_referenced_handles[target].contains(blocking[i])) { sim.error = "the batch already references one of the constraint's dynamic bodies"; return -1; }
    return allocate_in_batch(sim, target, type_id, nb, encoded, blocking, blocking_count, prestep);
}

// Per active-set index: the handles of the live constraints that reference it.
std::vector<std::vector<int>> constraints_by_body(const Simulation& sim) {
    std::vector<std::vector<int>> out((size_t)sim.body_count);
    for (size_t h = 0; h < sim.handle_to_constraint.size(); ++h) {
        const ConstraintLocation& loc = sim.handle_to_constraint[h];
        if (loc.batch < 0) continue;
        const ConstraintBatch& batch = *sim.batches[(size_t)loc.batch];
        const TypeBatch& t = *batch.type_batches[(size_t)batch.type_index_to_type_batch_index[loc.type_id]];
        const int32_t* refs = t.body_references.data + (size_t)(loc.index_in_type_batch / sim.W) * t.bodies * sim.W + loc.index_in_type_batch % sim.W;
        for (int b = 0; b < t.bodies; ++b) {
            auto& list = out[(size_t)(refs[(size_t)b * sim.W] & ~(int32_t)kKinematicMask)];
            if (list.empty() || list.back() != (int)h) list.push_back((int)h);
        }
    }
    return out;
}

// Bodies.Remove (Bodies.cs:L244-260) of every listed body, in list order: first Solver.Remove of every constraint that references each body, the
// last added first (the reference walks the body's constraint list from its end), then RemoveFromActiveSet (L214-239) of each body: BodySet.RemoveAt
// moves the last body into the slot (BodySet.cs:L83-111) and Solver.UpdateForBodyMemoryMove points the moved body's constraint references at it,
// the kinematic bit kept (TypeProcessor.UpdateForBodyMemoryMove, TypeProcessor.cs:L807-817); the handle goes back to the pool. This leaves the state
// the reference's one Bodies.Remove per body leaves: a constraint remove moves lanes and a body move rewrites reference values, so the two commute.
// Grouped, the change log holds one run of constraint removes and one of body removes.
void bodies_remove(Simulation& sim, const std::vector<int32_t>& handles) {
    const int W = sim.W;
    std::vector<std::vector<int>> by_body = constraints_by_body(sim);
    for (const int32_t handle : handles) {
        const auto& attached = by_body[(size_t)sim.handle_to_index[(size_t)handle]];
        for (auto it = attached.rbegin(); it != attached.rend(); ++it)
            if (sim.handle_to_constraint[(size_t)*it].batch >= 0) solver_remove(sim, *it);
    }
    for (const int32_t handle : handles) {
        const int index = sim.handle_to_index[(size_t)handle], last = sim.body_count - 1;
        ChangeEntry& logged = log_change(sim, kBodyRemove);
        logged.at = {-1, -1, index};
        logged.handle = handle;
        // a body added since the last forward and removed again: its add entry sends the record it had
        for (auto it = sim.changes.rbegin(); it != sim.changes.rend(); ++it)
            if (it->kind == kBodyAdd && it->handle == handle && it->record.empty()) {
                it->record.assign(sim.dynamics.data + (size_t)index * 32, sim.dynamics.data + (size_t)index * 32 + 32);
                break;
            }
        if (index < last) {
            std::memcpy(sim.dynamics.data + (size_t)index * 32, sim.dynamics.data + (size_t)last * 32, 32 * sizeof(float));
            const int moved_handle = sim.index_to_handle[(size_t)last];
            sim.index_to_handle[(size_t)index] = moved_handle;
            sim.handle_to_index[(size_t)moved_handle] = index;
            for (const int h : by_body[(size_t)last]) {
                const ConstraintLocation& loc = sim.handle_to_constraint[(size_t)h];
                if (loc.batch < 0) continue;
                ConstraintBatch& batch = *sim.batches[(size_t)loc.batch];
                TypeBatch& t = *batch.type_batches[(size_t)batch.type_index_to_type_batch_index[loc.type_id]];
                int32_t* refs = t.body_references.data + (size_t)(loc.index_in_type_batch / W) * t.bodies * W + loc.index_in_type_batch % W;
                for (int b = 0; b < t.bodies; ++b)
                    if ((refs[(size_t)b * W] & ~(int32_t)kKinematicMask) == last) refs[(size_t)b * W] = index | (refs[(size_t)b * W] & (int32_t)kKinematicMask);
            }
            by_body[(size_t)index] = std::move(by_body[(size_t)last]);
        }
        by_body.pop_back();
        sim.index_to_handle.pop_back();
        sim.handle_to_index[(size_t)handle] = -1;
        sim.free_handles.push_back(handle);
        --sim.body_count;
    }
}

}  // namespace

extern "C" {

struct bepuhost_type_batch_view {
    int32_t type_id, constraint_count, bodies, prestep_rows, impulse_rows, bundle_count;
    int32_t* body_references;
    float* prestep;
    float* accumulated_impulses;
};

void* bepuhost_create(int32_t bundle_width, int32_t fallback_batch_threshold) {
    if (bundle_width < 1 || bundle_width > 32 || fallback_batch_threshold < 1) return nullptr;
    Simulation* s = new Simulation();
    s->W = bundle_width;
    s->fallback_batch_threshold = fallback_batch_threshold;
    s->velocity_iterations = {1};
    s->integrator.gravity[0] = 0; s->integrator.gravity[1] = -10; s->integrator.gravity[2] = 0;
    s->integrator.linear_damping = 0.03f;
    s->integrator.angular_damping = 0.03f;
    return s;
}
void bepuhost_destroy(void* sim) { delete (Simulation*)sim; }
// Contacts per constraint of a type id (bepu_type_table.h); 0 for joints and ids without a type.
int32_t bepuhost_contact_count(int32_t type_id) { return bepucuda::contact_count_of_type(type_id); }
const char* bepuhost_last_error(void* sim) { return ((Simulation*)sim)->error.c_str(); }

// SolveDescription(velocityIterationCount, substepCount) with an optional per-substep schedule (SolveDescription.cs:L21-38).
int32_t bepuhost_set_solve_description(void* simp, int32_t substep_count, const int32_t* velocity_iterations_per_substep) {
    Simulation& sim = *(Simulation*)simp;
    if (substep_count < 1 || !velocity_iterations_per_substep) return -1;
    sim.velocity_iterations.assign(velocity_iterations_per_substep, velocity_iterations_per_substep + substep_count);
    return 0;
}
int32_t bepuhost_set_integrator(void* simp, const bepucuda_integrator_desc* d) {
    ((Simulation*)simp)->integrator = *d;
    return 0;
}

// Bodies.Add: appends `count` BodyDynamics records (32 floats each) at the end of the active set; returns the handle of the first. Handles come
// from the handle pool (IdPool.Take: the last returned handle first, else the next new one), so they equal active-set indices until a body is removed.
int32_t bepuhost_add_bodies(void* simp, const float* dynamics, int32_t count) {
    Simulation& sim = *(Simulation*)simp;
    const int first = sim.body_count;
    sim.dynamics.ensure((size_t)(first + count) * 32, (size_t)first * 32);
    std::memcpy(sim.dynamics.data + (size_t)first * 32, dynamics, (size_t)count * 32 * sizeof(float));
    int32_t first_handle = -1;
    for (int i = 0; i < count; ++i) {
        int handle = (int)sim.handle_to_index.size();
        if (!sim.free_handles.empty()) {
            handle = sim.free_handles.back();
            sim.free_handles.pop_back();
        } else {
            sim.handle_to_index.push_back(-1);
        }
        sim.handle_to_index[(size_t)handle] = first + i;
        sim.index_to_handle.push_back(handle);
        log_change(sim, kBodyAdd).handle = handle;
        if (i == 0) first_handle = handle;
    }
    sim.body_count += count;
    return first_handle;
}
// Bodies.Remove for `count` distinct body handles in order (bodies_remove). Returns 0, or -1 with nothing removed when a handle names no body or
// is listed twice.
int32_t bepuhost_remove_bodies(void* simp, int32_t count, const int32_t* handles) {
    Simulation& sim = *(Simulation*)simp;
    std::vector<int32_t> list(handles, handles + count);
    IndexSet seen;
    for (const int32_t h : list) {
        if (h < 0 || h >= (int32_t)sim.handle_to_index.size() || sim.handle_to_index[(size_t)h] < 0 || seen.contains(h)) { sim.error = "no such body handle, or one listed twice"; return -1; }
        seen.set(h);
    }
    bodies_remove(sim, list);
    return 0;
}
float* bepuhost_body_dynamics(void* simp) { return ((Simulation*)simp)->dynamics.data; }
int32_t bepuhost_body_count(void* simp) { return ((Simulation*)simp)->body_count; }
// Bodies.ActiveSet.IndexToHandle (body_count entries) and HandleToLocation's active-set index of a handle (-1: no body).
const int32_t* bepuhost_body_handles(void* simp) { return ((Simulation*)simp)->index_to_handle.data(); }
int32_t bepuhost_body_index(void* simp, int32_t handle) {
    const Simulation& sim = *(Simulation*)simp;
    return handle >= 0 && handle < (int32_t)sim.handle_to_index.size() ? sim.handle_to_index[(size_t)handle] : -1;
}

// Solver.Add for `count` constraints of one type in order. body_handles: count x bodies; prestep: count x prestep floats in the type's
// prestep row order (what IConstraintDescription.ApplyDescription writes). Returns the first constraint handle or -1.
int32_t bepuhost_add_constraints(void* simp, int32_t type_id, int32_t count, const int32_t* body_handles, const float* prestep) {
    Simulation& sim = *(Simulation*)simp;
    int32_t nb = 0, p = 0;
    if (bepucuda_type_info(type_id, &nb, &p, nullptr) != BEPUCUDA_OK) { sim.error = "unsupported constraint type"; return -1; }
    int first = -1;
    for (int i = 0; i < count; ++i) {
        int h = solver_add(sim, type_id, body_handles + (size_t)i * nb, prestep + (size_t)i * p);
        if (h < 0) return -1;
        if (i == 0) first = h;
    }
    return first;
}
// Like bepuhost_add_constraints with the batch of every constraint given (computed by bepucuda_color_constraints).
int32_t bepuhost_add_constraints_in_batches(void* simp, int32_t type_id, int32_t count, const int32_t* body_handles, const float* prestep, const int32_t* batch_indices) {
    Simulation& sim = *(Simulation*)simp;
    int32_t nb = 0, p = 0;
    if (bepucuda_type_info(type_id, &nb, &p, nullptr) != BEPUCUDA_OK) { sim.error = "unsupported constraint type"; return -1; }
    int32_t first = -1;
    for (int i = 0; i < count; ++i) {
        const int h = solver_add_in_batch(sim, batch_indices[i], type_id, body_handles + (size_t)i * nb, prestep + (size_t)i * p);
        if (h < 0) return -1;
        if (i == 0) first = h;
    }
    return first;
}
// Solver.Remove for `count` handles in order. Returns 0, or -1 at the first handle that names no constraint (the ones before it are removed).
int32_t bepuhost_remove_constraints(void* simp, int32_t count, const int32_t* handles) {
    Simulation& sim = *(Simulation*)simp;
    for (int32_t i = 0; i < count; ++i)
        if (solver_remove(sim, handles[i]) != 0) return -1;
    return 0;
}
// In handle (= add) order (-1 for a removed handle): the encoded body references of every constraint, 4 slots each (-1 = unused), and its batch index.
int32_t bepuhost_export_constraint_references(void* simp, int32_t* references_out, int32_t* batch_indices_out) {
    Simulation& sim = *(Simulation*)simp;
    const int W = sim.W;
    for (size_t h = 0; h < sim.handle_to_constraint.size(); ++h) {
        const ConstraintLocation& loc = sim.handle_to_constraint[h];
        if (loc.batch < 0) {  // removed
            for (int b = 0; b < 4; ++b) references_out[h * 4 + b] = -1;
            if (batch_indices_out) batch_indices_out[h] = -1;
            continue;
        }
        ConstraintBatch& batch = *sim.batches[loc.batch];
        TypeBatch& t = *batch.type_batches[batch.type_index_to_type_batch_index[loc.type_id]];
        const int bundle = loc.index_in_type_batch / W, inner = loc.index_in_type_batch % W;
        const int32_t* refs = t.body_references.data + (size_t)bundle * t.bodies * W;
        for (int b = 0; b < 4; ++b) references_out[h * 4 + b] = b < t.bodies ? refs[b * W + inner] : -1;
        if (batch_indices_out) batch_indices_out[h] = loc.batch;
    }
    return (int32_t)sim.handle_to_constraint.size();
}
int32_t bepuhost_constraint_location(void* simp, int32_t handle, int32_t* batch, int32_t* type_id, int32_t* index_in_type_batch) {
    Simulation& sim = *(Simulation*)simp;
    if (handle < 0 || handle >= (int)sim.handle_to_constraint.size() || sim.handle_to_constraint[handle].batch < 0) return -1;
    *batch = sim.handle_to_constraint[handle].batch;
    *type_id = sim.handle_to_constraint[handle].type_id;
    *index_in_type_batch = sim.handle_to_constraint[handle].index_in_type_batch;
    return 0;
}
int32_t bepuhost_constraint_count(void* simp) { return (int32_t)((Simulation*)simp)->handle_to_constraint.size(); }
int32_t bepuhost_batch_count(void* simp) { return (int32_t)((Simulation*)simp)->batches.size(); }
int32_t bepuhost_type_batch_count(void* simp, int32_t batch) { return (int32_t)((Simulation*)simp)->batches[batch]->type_batches.size(); }
int32_t bepuhost_get_type_batch(void* simp, int32_t batch, int32_t type_batch, bepuhost_type_batch_view* out) {
    Simulation& sim = *(Simulation*)simp;
    if (batch < 0 || batch >= (int)sim.batches.size()) return -1;
    auto& tbs = sim.batches[batch]->type_batches;
    if (type_batch < 0 || type_batch >= (int)tbs.size()) return -1;
    TypeBatch& t = *tbs[type_batch];
    out->type_id = t.type_id; out->constraint_count = t.constraint_count; out->bodies = t.bodies;
    out->prestep_rows = t.prestep_rows; out->impulse_rows = t.impulse_rows; out->bundle_count = t.bundle_count(sim.W);
    out->body_references = t.body_references.data; out->prestep = t.prestep.data; out->accumulated_impulses = t.impulses.data;
    return 0;
}
int32_t bepuhost_constrained_kinematic_count(void* simp) { return (int32_t)((Simulation*)simp)->constrained_kinematic_handles.size(); }
// Solver.ConstrainedKinematicHandles as active-set indices (valid until the next call).
const int32_t* bepuhost_constrained_kinematics(void* simp) { return kinematic_indices(*(Simulation*)simp).data(); }
int32_t bepuhost_bundle_width(void* simp) { return ((Simulation*)simp)->W; }
int32_t bepuhost_fallback_batch_threshold(void* simp) { return ((Simulation*)simp)->fallback_batch_threshold; }
int32_t bepuhost_substep_count(void* simp) { return (int32_t)((Simulation*)simp)->velocity_iterations.size(); }
const int32_t* bepuhost_velocity_iterations(void* simp) { return ((Simulation*)simp)->velocity_iterations.data(); }
const bepucuda_integrator_desc* bepuhost_integrator(void* simp) { return &((Simulation*)simp)->integrator; }

// ---- CudaTimestepper: what replaces `simulation.Solve(dt, threadDispatcher)` in DefaultTimestepper.Timestep -----------------
// (DefaultTimestepper.cs:L28-43). Exactly the P/Invoke sequence shown in INTEGRATION.md.

// Full description of the active set: bodies + every type batch + constrained kinematics. Call when topology changed.
int32_t bepuhost_cuda_describe(void* simp, bepucuda_ctx* ctx) {
    Simulation& sim = *(Simulation*)simp;
    int32_t rc;
    if ((rc = bepucuda_set_solve_description(ctx, (int32_t)sim.velocity_iterations.size(), sim.velocity_iterations.data(), sim.fallback_batch_threshold)) != 0) return rc;
    if ((rc = bepucuda_set_integrator(ctx, &sim.integrator)) != 0) return rc;
    if ((rc = bepucuda_upload_bodies(ctx, sim.dynamics.data, sim.body_count)) != 0) return rc;
    if ((rc = bepucuda_begin_constraints(ctx, sim.W, (int32_t)sim.batches.size())) != 0) return rc;
    for (int b = 0; b < (int)sim.batches.size(); ++b) {
        auto& tbs = sim.batches[b]->type_batches;
        for (int t = 0; t < (int)tbs.size(); ++t) {
            TypeBatch& tb = *tbs[t];
            if ((rc = bepucuda_upload_type_batch(ctx, b, t, tb.type_id, tb.constraint_count, tb.body_references.data, tb.prestep.data, tb.impulses.data)) != 0) return rc;
        }
    }
    const std::vector<int32_t>& kinematics = kinematic_indices(sim);
    if ((rc = bepucuda_set_constrained_kinematics(ctx, kinematics.data(), (int32_t)kinematics.size())) != 0) return rc;
    sim.changes.clear();
    return bepucuda_end_constraints(ctx);
}

// The body and constraint adds and removes since the last describe or change on the resident state: one bepucuda_add_bodies /
// bepucuda_remove_bodies / bepucuda_add_constraints / bepucuda_remove_constraints per run of entries of one kind, in the order they were made. A
// constraint run carries the constrained kinematics (active-set indices) as they were right after it. An add's record is its lane as the host holds
// it now (body references as encoded when it was added, impulses the host may have written since, prestep); a constraint added and removed again
// since sends its body references and zero rows. A body add sends the body's record as the host holds it now, or, for a body removed again since,
// the record it had then; a body remove sends the active-set index it removed. add_feature_ids: 4 int32 per constraint add in order, or NULL when
// no add is a contact. At a failing call the runs before it leave the log and its code is returned; the failing run and those after it stay
// (add_feature_ids then starts at the first add still logged).
int32_t bepuhost_cuda_change(void* simp, bepucuda_ctx* ctx, const int32_t* add_feature_ids) {
    Simulation& sim = *(Simulation*)simp;
    const int W = sim.W;
    size_t adds = 0;
    for (size_t i = 0; i < sim.changes.size();) {
        const ChangeKind kind = sim.changes[i].kind;
        size_t j = i;
        while (j < sim.changes.size() && sim.changes[j].kind == kind) ++j;
        const int32_t n = (int32_t)(j - i);
        const std::vector<int32_t>& kin = sim.changes[j - 1].kinematics_kept ? sim.changes[j - 1].kinematics : kinematic_indices(sim);
        std::vector<bepucuda_constraint_location> locations;
        std::vector<int32_t> records, indices;
        std::vector<float> bodies;
        for (size_t k = i; k < j; ++k) {
            const ChangeEntry& e = sim.changes[k];
            if (kind == kBodyAdd) {
                const float* r = e.record.empty() ? sim.dynamics.data + (size_t)sim.handle_to_index[(size_t)e.handle] * 32 : e.record.data();
                bodies.insert(bodies.end(), r, r + 32);
                continue;
            }
            if (kind == kBodyRemove) {
                indices.push_back(e.at.index_in_type_batch);
                continue;
            }
            locations.push_back({0, e.at.batch, e.at.type_id, e.at.index_in_type_batch});
            if (kind == kConstraintRemove) continue;
            records.resize(records.size() + 64, 0);
            int32_t* r = records.data() + records.size() - 64;
            r[0] = e.at.type_id;
            r[1] = 1;
            const bepucuda::TypeRow* t = bepucuda::type_row(e.at.type_id);
            for (int b = 0; b < t->bodies; ++b) r[2 + b] = e.refs[b];
            const ConstraintLocation now = sim.handle_to_constraint[(size_t)e.handle];
            if (now.batch < 0) continue;
            ConstraintBatch& batch = *sim.batches[(size_t)now.batch];
            const TypeBatch& tb = *batch.type_batches[(size_t)batch.type_index_to_type_batch_index[now.type_id]];
            const size_t bundle = (size_t)(now.index_in_type_batch / W), lane = (size_t)(now.index_in_type_batch % W);
            for (int q = 0; q < tb.impulse_rows; ++q) std::memcpy(r + 6 + q, tb.impulses.data + (bundle * tb.impulse_rows + q) * W + lane, 4);
            for (int q = 0; q < tb.prestep_rows; ++q) std::memcpy(r + 18 + q, tb.prestep.data + (bundle * tb.prestep_rows + q) * W + lane, 4);
        }
        int32_t rc = 0;
        switch (kind) {
            case kBodyAdd: rc = bepucuda_add_bodies(ctx, bodies.data(), n, nullptr, nullptr); break;
            case kBodyRemove: rc = bepucuda_remove_bodies(ctx, n, indices.data()); break;
            case kConstraintRemove: rc = bepucuda_remove_constraints(ctx, n, locations.data(), kin.data(), (int32_t)kin.size()); break;
            case kConstraintAdd:
                rc = bepucuda_add_constraints(ctx, n, locations.data(), records.data(), add_feature_ids ? add_feature_ids + adds * 4 : nullptr, kin.data(), (int32_t)kin.size());
                break;
        }
        if (rc != 0) {
            sim.changes.erase(sim.changes.begin(), sim.changes.begin() + (std::ptrdiff_t)i);  // the runs before it went through: not forwarded again
            return rc;
        }
        if (kind == kConstraintAdd) adds += (size_t)n;
        i = j;
    }
    sim.changes.clear();
    return 0;
}

// Per-frame refresh with unchanged topology: body state + the prestep/impulse data the narrow phase rewrote.
int32_t bepuhost_cuda_refresh(void* simp, bepucuda_ctx* ctx) {
    Simulation& sim = *(Simulation*)simp;
    int32_t rc;
    if ((rc = bepucuda_upload_bodies(ctx, sim.dynamics.data, sim.body_count)) != 0) return rc;
    for (int b = 0; b < (int)sim.batches.size(); ++b) {
        auto& tbs = sim.batches[b]->type_batches;
        for (int t = 0; t < (int)tbs.size(); ++t)
            if ((rc = bepucuda_update_type_batch(ctx, b, t, tbs[t]->prestep.data, tbs[t]->impulses.data)) != 0) return rc;
    }
    return 0;
}

// Per-frame refresh through the device-side contact update (bepucuda_update_contacts): body motion + new prestep + new contact feature ids; the
// accumulated impulses stay on the device. `feature_pool` holds the ids of every CONTACT type batch back to back in (batch, type batch) order,
// [constraint][contact] each (what a PairCache walk produces). set_only != 0: bepucuda_set_contact_features (the ids of the uploaded impulses).
int32_t bepuhost_cuda_update_contacts(void* simp, bepucuda_ctx* ctx, const int32_t* feature_pool, int32_t set_only) {
    Simulation& sim = *(Simulation*)simp;
    int32_t rc;
    if (!set_only && (rc = bepucuda_upload_body_motion(ctx, sim.dynamics.data, sim.body_count)) != 0) return rc;
    size_t at = 0;
    for (int b = 0; b < (int)sim.batches.size(); ++b) {
        auto& tbs = sim.batches[b]->type_batches;
        for (int t = 0; t < (int)tbs.size(); ++t) {
            const int n = bepucuda::type_row(tbs[t]->type_id)->contacts;
            if (n == 0) continue;
            rc = set_only ? bepucuda_set_contact_features(ctx, b, t, feature_pool + at) : bepucuda_update_contacts(ctx, b, t, tbs[t]->prestep.data, feature_pool + at);
            if (rc != 0) return rc;
            at += (size_t)tbs[t]->constraint_count * n;
        }
    }
    return 0;
}

// Solve slot of the timestep: device solve, then results back into the host's own buffers.
int32_t bepuhost_cuda_solve(void* simp, bepucuda_ctx* ctx, float dt, int32_t download) {
    Simulation& sim = *(Simulation*)simp;
    int32_t rc;
    if ((rc = bepucuda_solve(ctx, dt)) != 0) return rc;
    if (download) {
        if ((rc = bepucuda_download_bodies(ctx, sim.dynamics.data, sim.body_count)) != 0) return rc;
        if ((rc = bepucuda_download_impulses(ctx)) != 0) return rc;
    }
    return 0;
}

// Mirrors the contact-depth mutation of IncrementallyUpdateForSubstep back into the host prestep buffers (test use).
int32_t bepuhost_cuda_download_prestep(void* simp, bepucuda_ctx* ctx) {
    Simulation& sim = *(Simulation*)simp;
    for (int b = 0; b < (int)sim.batches.size(); ++b) {
        auto& tbs = sim.batches[b]->type_batches;
        for (int t = 0; t < (int)tbs.size(); ++t) {
            int32_t rc = bepucuda_download_prestep(ctx, b, t, tbs[t]->prestep.data);
            if (rc != 0) return rc;
        }
    }
    return 0;
}

// Page-locks the simulation's buffers (the C# side would register its BufferPool blocks once).
int32_t bepuhost_cuda_register_buffers(void* simp, bepucuda_ctx* ctx) {
    Simulation& sim = *(Simulation*)simp;
    const int W = sim.W;
    int32_t rc;
    if (sim.body_count > 0 && (rc = bepucuda_host_register(ctx, sim.dynamics.data, (int64_t)sim.dynamics.capacity * 4)) != 0) return rc;
    for (auto b : sim.batches)
        for (auto t : b->type_batches) {
            if ((rc = bepucuda_host_register(ctx, t->body_references.data, (int64_t)t->body_references.capacity * 4)) != 0) return rc;
            if ((rc = bepucuda_host_register(ctx, t->prestep.data, (int64_t)t->prestep.capacity * 4)) != 0) return rc;
            if ((rc = bepucuda_host_register(ctx, t->impulses.data, (int64_t)t->impulses.capacity * 4)) != 0) return rc;
        }
    (void)W;
    return 0;
}
int32_t bepuhost_cuda_unregister_buffers(void* simp, bepucuda_ctx* ctx) {
    Simulation& sim = *(Simulation*)simp;
    if (sim.body_count > 0) bepucuda_host_unregister(ctx, sim.dynamics.data);
    for (auto b : sim.batches)
        for (auto t : b->type_batches) {
            bepucuda_host_unregister(ctx, t->body_references.data);
            bepucuda_host_unregister(ctx, t->prestep.data);
            bepucuda_host_unregister(ctx, t->impulses.data);
        }
    return 0;
}

}  // extern "C"
