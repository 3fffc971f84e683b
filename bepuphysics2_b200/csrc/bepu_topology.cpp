// Constraint topology: type registry, device batches and work list (plan_topology), stage program (build_stage_program). Plain C++: no CUDA
// runtime call, so that the CPU suite can check what the device is told to run.
#include "bepu_topology.h"

#include <algorithm>
#include <array>
#include <cstring>
#include <numeric>
#include <unordered_map>

#include "../../include/bepucuda.h"
#include "bepu_type_table.h"

namespace bepucuda {

// ---- type registry -------------------------------------------------------------------------------------------------------
// SURVEY.md §8d algorithmic bytes, from the rows of bepu_type_table.h (R / W: floats the access filters read / write, summed over the bodies):
//   solve       = 4 * (P + 2D + n + R + W)
//   warm start  = 4 * (P + D + n + R' + W')              (non-integrating lane, WarmStart filters)
//   incremental = 4 * (P_read + contacts_written + n + 6n)  contacts only; joints have no incremental update
const TypeInfo* get_type_info(int type_id) {
    static const std::array<TypeInfo, 64> types = [] {
        std::array<TypeInfo, 64> t{};
        for (const TypeRow& r : kTypeTable) {
            const int32_t P = r.prestep_rows, D = r.impulse_rows, n = r.bodies;
            t[(size_t)r.id] = {n, P, D, r.contacts, 4 * (P + 2 * D + n + r.solve_read + r.solve_written), 4 * (P + D + n + r.warm_start_read + r.warm_start_written),
                               r.contacts > 0 ? 4 * (P + r.contacts + n + 6 * n) : 0, r.name};
        }
        return t;
    }();
    if (type_id < 0 || type_id >= 64 || !types[(size_t)type_id].name) return nullptr;
    return &types[(size_t)type_id];
}

// ---- device batches and work list ----------------------------------------------------------------------------------------
static bool dynamic_ref(int32_t enc) { return enc >= 0 && !((uint32_t)enc & kRefKinematicBit); }

int plan_topology(const std::vector<SourceView>& sources, int W, int fallback_threshold, int batch_count, int body_count, bool peer_mode, TopologyPlan* plan,
                  std::string* error, int rank, int fallback_rank) {
    TopologyPlan& p = *plan;
    p = TopologyPlan{};
    p.fallback_rank = peer_mode ? fallback_rank : -1;
    // sources in (batch, type batch) order
    std::vector<int> order(sources.size());
    std::iota(order.begin(), order.end(), 0);
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) {
        const SourceView &x = sources[(size_t)a], &y = sources[(size_t)b];
        return x.batch_index != y.batch_index ? x.batch_index < y.batch_index : x.type_batch_index < y.type_batch_index;
    });
    p.source_live.assign(sources.size(), 0);
    p.source_bundle_base.assign(sources.size(), 0);
    p.source_type_batch.assign(sources.size(), -1);
    p.source_inverse_offset.assign(sources.size(), -1);
    p.source_count.assign(sources.size(), 0);
    p.location_source.assign((size_t)std::max(batch_count, 0) * 64, -1);
    for (size_t i = sources.size(); i-- > 0;) {  // the first type batch of a (batch, type id) answers for it
        const SourceView& s = sources[i];
        p.source_count[i] = s.count;
        if (s.batch_index >= 0 && s.batch_index < batch_count && s.type_id >= 0 && s.type_id < 64) p.location_source[(size_t)s.batch_index * 64 + (size_t)s.type_id] = (int32_t)i;
    }
    for (int si : order) {
        p.source_bundle_base[(size_t)si] = p.source_bundles;
        p.source_bundles += (sources[(size_t)si].count + W - 1) / W;
    }
    std::vector<std::vector<int>> batch_tbs;  // device batch -> device type batches
    auto add_tb = [&](int source, int device_batch, int constraints, int64_t map_offset) {
        batch_tbs[(size_t)device_batch].push_back((int)p.tbs.size());
        p.tbs.push_back({sources[(size_t)source].type_id, (constraints + 31) / 32, device_batch, source, map_offset, 0, 0, 0});
    };

    // synchronized batches: device batch index == host batch index (empty batches stay as empty slots), so ranks of a sharded graph agree on
    // batch numbers
    for (int si : order) {
        const SourceView& s = sources[(size_t)si];
        if (s.batch_index >= fallback_threshold) continue;
        while ((int)batch_tbs.size() <= s.batch_index) batch_tbs.emplace_back();
        p.source_type_batch[(size_t)si] = (int32_t)p.tbs.size();
        add_tb(si, s.batch_index, s.count, -1);
        p.source_live[(size_t)si] = s.count;
        p.constraint_count += s.count;
    }
    if (peer_mode) {
        // every rank runs the exchange point of every batch, also of batches it has no constraint in
        while ((int)batch_tbs.size() < std::min(batch_count, fallback_threshold)) batch_tbs.emplace_back();
        // the sequential fallback batch runs whole on one rank, the fallback rank, in the levels below
        for (const SourceView& s : sources)
            if (s.batch_index >= fallback_threshold && rank != p.fallback_rank) {
                *error = p.fallback_rank < 0 ? "end_constraints: the sequential fallback batch is not supported across ranks"
                                             : "end_constraints: a type batch of the sequential fallback batch was uploaded on rank " + std::to_string(rank) +
                                                   ", but only the fallback rank " + std::to_string(p.fallback_rank) + " may run it";
                return BEPUCUDA_ERR_BAD_STATE;
            }
    }
    p.sync_batch_count = (int)batch_tbs.size();

    // Fallback levelisation. The reference executes fallback bundles one after another on a single thread (Solver_Solve.cs:L546-583); within a
    // bundle no dynamic body repeats (TypeProcessor.cs:L338-359). A constraint's level is 1 + the highest level of any earlier-bundle constraint
    // sharing a dynamic body with it: executing levels in order with a barrier in between preserves every read-after-write of the sequential
    // loop, so results are identical.
    std::vector<int32_t> last_level;  // per body: highest level assigned so far (0 = none)
    struct Slot { int level; int rank; int constraint; };  // rank: position of the source in `order`
    std::vector<Slot> slots;
    std::vector<int> lane_level((size_t)W);
    for (size_t rank = 0; rank < order.size(); ++rank) {
        const SourceView& s = sources[(size_t)order[rank]];
        if (s.batch_index < fallback_threshold) continue;
        if (last_level.empty()) last_level.assign((size_t)body_count, 0);
        p.source_inverse_offset[(size_t)order[rank]] = (int64_t)p.inverse.size();
        p.inverse.resize(p.inverse.size() + (size_t)s.count, DeviceSlot{-1, -1});  // holes keep {-1, -1}
        const int nb = get_type_info(s.type_id)->bodies;
        const int bundles = (s.count + W - 1) / W;
        auto ref = [&](int k, int b, int l) { return s.refs[((size_t)k * nb + b) * W + l]; };
        for (int k = 0; k < bundles; ++k) {
            // all lanes of a bundle read the state left by earlier bundles
            for (int l = 0; l < W; ++l) {
                lane_level[(size_t)l] = 0;
                if (k * W + l >= s.count || ref(k, 0, l) < 0) continue;  // padding, hole
                int lvl = 0;
                for (int b = 0; b < nb; ++b) {
                    const int32_t enc = ref(k, b, l);
                    if (!dynamic_ref(enc)) continue;
                    const uint32_t idx = (uint32_t)enc & kRefIndexMask;
                    if ((int)idx >= body_count) {
                        *error = "end_constraints: body reference out of range";
                        return BEPUCUDA_ERR_INVALID_ARGUMENT;
                    }
                    lvl = std::max(lvl, last_level[idx]);
                }
                lane_level[(size_t)l] = lvl + 1;
            }
            for (int l = 0; l < W; ++l) {
                if (lane_level[(size_t)l] == 0) continue;
                for (int b = 0; b < nb; ++b)
                    if (dynamic_ref(ref(k, b, l))) last_level[(uint32_t)ref(k, b, l) & kRefIndexMask] = lane_level[(size_t)l];
                // TypeProcessor.cs:L338-359: a fallback bundle never holds a dynamic body twice (two lanes of one level would race on its record)
                for (int l2 = 0; l2 < l; ++l2) {
                    if (lane_level[(size_t)l2] == 0) continue;
                    for (int b = 0; b < nb; ++b) {
                        const int32_t e1 = ref(k, b, l);
                        if (!dynamic_ref(e1)) continue;
                        for (int b2 = 0; b2 < nb; ++b2) {
                            const int32_t e2 = ref(k, b2, l2);
                            if (dynamic_ref(e2) && (((uint32_t)e1 ^ (uint32_t)e2) & kRefIndexMask) == 0) {
                                *error = "end_constraints: a fallback bundle references the same dynamic body more than once";
                                return BEPUCUDA_ERR_BATCH_INVARIANT;
                            }
                        }
                    }
                }
                slots.push_back({lane_level[(size_t)l], (int)rank, k * W + l});
                ++p.source_live[(size_t)order[rank]];
                ++p.constraint_count;
            }
        }
    }
    // one device batch per level; within it one device type batch per source, its slots mapped to the source constraints
    std::stable_sort(slots.begin(), slots.end(), [](const Slot& a, const Slot& b) { return a.level != b.level ? a.level < b.level : a.rank < b.rank; });
    for (size_t i = 0; i < slots.size();) {
        const int level = slots[i].level;
        batch_tbs.emplace_back();
        ++p.fallback_levels;
        while (i < slots.size() && slots[i].level == level) {
            const int rank = slots[i].rank;
            size_t j = i;
            while (j < slots.size() && slots[j].level == level && slots[j].rank == rank) ++j;
            const int source = order[(size_t)rank];
            add_tb(source, (int)batch_tbs.size() - 1, (int)(j - i), (int64_t)p.maps.size());
            for (size_t q = i; q < j; ++q) {
                p.maps.push_back(slots[q].constraint);
                p.inverse[(size_t)p.source_inverse_offset[(size_t)source] + (size_t)slots[q].constraint] = {(int32_t)p.tbs.size() - 1, (int32_t)(q - i)};
            }
            p.maps.resize((size_t)p.tbs.back().map_offset + (size_t)p.tbs.back().bundle_count * 32, -1);
            i = j;
        }
    }

    // arenas of the AOSOA-32 image
    for (PlannedTypeBatch& tb : p.tbs) {
        const TypeInfo* t = get_type_info(tb.type_id);
        tb.refs_offset = p.refs_words;
        tb.prestep_offset = p.prestep_words;
        tb.impulse_offset = p.impulse_words;
        p.refs_words += (size_t)tb.bundle_count * t->bodies * 32;
        p.prestep_words += (size_t)tb.bundle_count * t->prestep_rows * 32;
        p.impulse_words += (size_t)tb.bundle_count * t->impulse_rows * 32;
    }

    // work lists: per device batch (one warp per bundle), then the incremental-update list over all contact bundles
    auto add_bundles = [&](int tb) {
        const PlannedTypeBatch& d = p.tbs[(size_t)tb];
        for (int k = 0; k < d.bundle_count; ++k) {
            p.work.push_back({tb, k});
            // identity-mapped type batches: lanes beyond the source count are padding; mapped (fallback level) ones: -1 entries are padding
            int live = 0;
            if (d.map_offset < 0) live = std::max(0, std::min(32, sources[(size_t)d.source].count - k * 32));
            else for (int l = 0; l < 32; ++l) live += p.maps[(size_t)d.map_offset + (size_t)k * 32 + l] >= 0;
            p.bundle_live.push_back(live);
        }
    };
    for (const auto& list : batch_tbs) {
        const int begin = (int)p.work.size();
        bool contacts_only = true;
        for (int tb : list) {
            contacts_only = contacts_only && get_type_info(p.tbs[(size_t)tb].type_id)->contacts > 0;
            add_bundles(tb);
        }
        p.batches.push_back({begin, (int)p.work.size() - begin, contacts_only ? 1 : 0});
    }
    p.all_work_count = (int)p.work.size();
    p.inc_begin = p.all_work_count;
    for (size_t tb = 0; tb < p.tbs.size(); ++tb)
        if (get_type_info(p.tbs[tb].type_id)->contacts > 0) add_bundles((int)tb);
    p.inc_count = (int)p.work.size() - p.inc_begin;
    return BEPUCUDA_OK;
}

int resolve_location(const TopologyPlan& plan, const bepucuda_constraint_location& l, ResolvedLocation* out) {
    const size_t key = (size_t)l.batch_index * 64 + (size_t)l.type_id;
    const int32_t s = l.set_index == 0 && l.batch_index >= 0 && l.type_id >= 0 && l.type_id < 64 && key < plan.location_source.size() ? plan.location_source[key] : -1;
    if (s < 0 || l.index_in_type_batch < 0 || l.index_in_type_batch >= plan.source_count[(size_t)s]) return BEPUCUDA_ERR_INVALID_ARGUMENT;
    out->source = s;
    const int32_t tb = plan.source_type_batch[(size_t)s];
    if (tb >= 0) {
        out->at = {tb, l.index_in_type_batch};
        out->inverse_entry = -1;
    } else {
        out->inverse_entry = plan.source_inverse_offset[(size_t)s] + l.index_in_type_batch;
        out->at = plan.inverse[(size_t)out->inverse_entry];
    }
    return BEPUCUDA_OK;
}

void PrestepWriteQueue::plan(const TopologyPlan& p) {
    writes.clear();
    rows.clear();
    entry_of_slot_.clear();
    slot_base_.resize(p.tbs.size());
    slots_ = 0;
    for (size_t i = 0; i < p.tbs.size(); ++i) {
        slot_base_[i] = slots_;
        slots_ += (int64_t)p.tbs[i].bundle_count * 32;
    }
}

void PrestepWriteQueue::put(DeviceSlot at, const float* r, int count) {
    if (entry_of_slot_.empty()) entry_of_slot_.assign((size_t)slots_, -1);
    int32_t& entry = entry_of_slot_[(size_t)(slot_base_[(size_t)at.type_batch] + at.slot)];
    if (entry < 0) {
        entry = (int32_t)writes.size();
        writes.push_back({at, (int32_t)rows.size()});
        rows.resize(rows.size() + (size_t)count);
    }
    std::memcpy(rows.data() + writes[(size_t)entry].row0, r, (size_t)count * sizeof(float));
}

void PrestepWriteQueue::clear() {
    for (const PrestepWrite& w : writes) entry_of_slot_[(size_t)(slot_base_[(size_t)w.at.type_batch] + w.at.slot)] = -1;
    writes.clear();
    rows.clear();
}

int check_body_write(bool bodies_uploaded, int32_t body_count, const void* body_dynamics, int32_t count, const int32_t* body_indices, const char** why) {
    if (count < 0 || (count > 0 && (!body_dynamics || !body_indices))) {
        *why = "bad arguments";
        return BEPUCUDA_ERR_INVALID_ARGUMENT;
    }
    if (!bodies_uploaded) {
        *why = "before upload_bodies";
        return BEPUCUDA_ERR_BAD_STATE;
    }
    for (int32_t i = 0; i < count; ++i)
        if (body_indices[i] < 0 || body_indices[i] >= body_count) {
            *why = "a body index outside the bodies of the last upload_bodies";
            return BEPUCUDA_ERR_INVALID_ARGUMENT;
        }
    return BEPUCUDA_OK;
}

void gather_motion_halves(const void* body_dynamics, const int32_t* body_indices, int32_t count, float* out) {
    const char* records = (const char*)body_dynamics;
    for (int32_t i = 0; i < count; ++i) std::memcpy(out + (size_t)i * 16, records + (size_t)body_indices[i] * 128, 64);
}

// ---- constraint adds and removes ---------------------------------------------------------------------------------------------------------
namespace {
struct Replay {
    ChangeState& st;
    int W, threshold, body_count;
    std::vector<LaneCopy>& ops;
    std::string& error;
    std::vector<int32_t> tb_count;  // per batch: its type batches

    int fail(int32_t i, const std::string& why) {
        error = "entry " + std::to_string(i) + ": " + why;
        return BEPUCUDA_ERR_INVALID_ARGUMENT;
    }
    int find(int32_t batch, int32_t type_id) const {
        for (size_t s = 0; s < st.sources.size(); ++s)
            if (st.sources[s].type_batch_index >= 0 && st.sources[s].batch_index == batch && st.sources[s].type_id == type_id) return (int)s;
        return -1;
    }
    // the first body reference of lane `index` (fallback sources), -1 beyond the bundles
    int32_t first_ref(const ChangeSource& s, int nb, int32_t index) const {
        const size_t at = (size_t)(index / W) * nb * W + (size_t)(index % W);
        return at < s.refs.size() ? s.refs[at] : -1;
    }
    void set_lane_refs(ChangeSource& s, int nb, int32_t index, const int32_t* v) {
        for (int b = 0; b < nb; ++b) s.refs[((size_t)(index / W) * nb + b) * W + (size_t)(index % W)] = v ? v[b] : -1;
    }
    int add(int32_t i, const bepucuda_constraint_location& l, const int32_t* record) {
        const TypeInfo* t = get_type_info(l.type_id);
        if (l.set_index != 0 || !t) return fail(i, "not a location of the active set with a supported type id");
        if (record[0] != l.type_id) return fail(i, "record type id " + std::to_string(record[0]) + ", location type id " + std::to_string(l.type_id));
        for (int b = 0; b < t->bodies; ++b) {
            const int32_t v = record[kRecordRefs + b];
            if (v < 0 || (int64_t)((uint32_t)v & ~kRefKinematicBit) >= (int64_t)body_count) return fail(i, "body reference out of range");
        }
        if (l.batch_index < 0 || l.batch_index > st.batch_count) return fail(i, "batch index out of range");
        if (l.batch_index == st.batch_count) {
            ++st.batch_count;
            tb_count.push_back(0);
        }
        const bool fallback = l.batch_index >= threshold;
        int s = find(l.batch_index, l.type_id);
        if (s < 0) {
            if (l.index_in_type_batch != 0) return fail(i, "a new type batch starts at index 0");
            st.sources.push_back({l.batch_index, tb_count[(size_t)l.batch_index]++, l.type_id, 0, {}});
            s = (int)st.sources.size() - 1;
        }
        ChangeSource& src = st.sources[(size_t)s];
        const int32_t index = l.index_in_type_batch, bundles = (src.count + W - 1) / W;
        if (!fallback) {
            if (index != src.count) return fail(i, "a synchronized add goes to index ConstraintCount = " + std::to_string(src.count));
        } else if (index == bundles * W) {
            src.refs.resize((size_t)(bundles + 1) * t->bodies * W, -1);  // a new bundle: every lane empty
        } else if (index < 0 || index > bundles * W || first_ref(src, t->bodies, index) >= 0) {
            return fail(i, "a fallback add goes to an empty lane or to the first lane of a new bundle");
        }
        if (fallback) set_lane_refs(src, t->bodies, index, record + kRecordRefs);
        src.count = std::max(src.count, index + 1);
        ops.push_back({s, index, kLaneNew, i});
        return BEPUCUDA_OK;
    }
    int remove(int32_t i, const bepucuda_constraint_location& l) {
        const int s = l.set_index == 0 && l.type_id >= 0 && l.type_id < 64 ? find(l.batch_index, l.type_id) : -1;
        if (s < 0 || l.index_in_type_batch < 0 || l.index_in_type_batch >= st.sources[(size_t)s].count) return fail(i, "names no constraint of the active set");
        ChangeSource& src = st.sources[(size_t)s];
        const int nb = get_type_info(src.type_id)->bodies;
        const int32_t index = l.index_in_type_batch;
        if (src.batch_index >= threshold) {
            if (first_ref(src, nb, index) < 0) return fail(i, "a hole of the fallback batch");
            ops.push_back({s, index, kLaneClear, 0});
            set_lane_refs(src, nb, index, nullptr);
            const int32_t removed_bundle = index / W;
            bool empty = true;
            for (int l2 = 0; l2 < W; ++l2) empty = empty && first_ref(src, nb, removed_bundle * W + l2) < 0;
            if (empty) {
                int32_t last = (src.count + W - 1) / W - 1;
                if (removed_bundle != last) {
                    for (int l2 = 0; l2 < W; ++l2) {
                        ops.push_back({s, removed_bundle * W + l2, s, last * W + l2});
                        for (int b = 0; b < nb; ++b) src.refs[((size_t)removed_bundle * nb + b) * W + l2] = src.refs[((size_t)last * nb + b) * W + l2];
                    }
                    --last;
                }
                int32_t lanes = 0;
                for (int l2 = 0; l2 < W; ++l2)
                    if (first_ref(src, nb, last * W + l2) >= 0) lanes = l2 + 1;
                src.count = last * W + lanes;
                src.refs.resize((size_t)((src.count + W - 1) / W) * nb * W);
            }
        } else {
            const int32_t last = src.count - 1;
            if (index < last) ops.push_back({s, index, s, last});
            src.count = last;
        }
        if (src.count == 0) {
            // ConstraintBatch.RemoveTypeBatchIfEmpty: the batch's last type batch takes the removed one's index
            const int32_t batch = src.batch_index, removed = src.type_batch_index;
            src.type_batch_index = -1;
            for (ChangeSource& o : st.sources)
                if (o.type_batch_index == tb_count[(size_t)batch] - 1 && o.batch_index == batch) o.type_batch_index = removed;
            --tb_count[(size_t)batch];
            // Solver.RemoveBatchIfEmpty: only the last batch goes, and with it the empty batches it reveals
            if (batch == st.batch_count - 1)
                while (st.batch_count > 0 && tb_count[(size_t)st.batch_count - 1] == 0) {
                    --st.batch_count;
                    tb_count.pop_back();
                }
        }
        return BEPUCUDA_OK;
    }
};
}  // namespace

int replay_changes(ChangeState* state, bool remove, int W, int fallback_threshold, int body_count, int32_t count, const bepucuda_constraint_location* locations,
                   const int32_t* records, std::vector<LaneCopy>* ops, std::string* error) {
    Replay r{*state, W, fallback_threshold, body_count, *ops, *error, std::vector<int32_t>((size_t)std::max(state->batch_count, 0), 0)};
    for (const ChangeSource& s : state->sources)
        if (s.type_batch_index >= 0 && s.batch_index >= 0 && s.batch_index < state->batch_count) ++r.tb_count[(size_t)s.batch_index];
    for (int32_t i = 0; i < count; ++i) {
        const int rc = remove ? r.remove(i, locations[i]) : r.add(i, locations[i], records + (size_t)i * 64);
        if (rc != BEPUCUDA_OK) return rc;
    }
    return BEPUCUDA_OK;
}

std::vector<LaneCopy> compose_lane_ops(const std::vector<LaneCopy>& ops) {
    std::vector<LaneCopy> out;
    std::unordered_map<int64_t, size_t> written;  // lane -> its entry of `out`
    written.reserve(ops.size() * 2);
    auto key = [](int32_t source, int32_t index) { return ((int64_t)source << 32) | (uint32_t)index; };
    for (const LaneCopy& op : ops) {
        LaneCopy origin = op;
        if (op.src_source >= 0) {
            const auto from = written.find(key(op.src_source, op.src_index));
            if (from != written.end()) origin = {op.dst_source, op.dst_index, out[from->second].src_source, out[from->second].src_index};
        }
        const auto [at, inserted] = written.try_emplace(key(op.dst_source, op.dst_index), out.size());
        if (inserted) out.push_back(origin);
        else out[at->second] = origin;
    }
    // a lane that ends with its own rows needs no copy
    out.erase(std::remove_if(out.begin(), out.end(), [](const LaneCopy& o) { return o.src_source == o.dst_source && o.src_index == o.dst_index; }), out.end());
    return out;
}

int replay_body_removes(int32_t body_count, int32_t count, const int32_t* body_indices, int32_t* final_count, std::vector<int32_t>* moved_to, std::string* error) {
    if (count < 0 || body_count < 0 || (count > 0 && !body_indices)) {
        *error = "bad arguments";
        return BEPUCUDA_ERR_INVALID_ARGUMENT;
    }
    // slot -> the original index of the body it holds, for the slots whose body moved (every other slot holds its own)
    std::unordered_map<int32_t, int32_t> at;
    at.reserve((size_t)count * 2);
    auto body_at = [&](int32_t slot) {
        const auto it = at.find(slot);
        return it == at.end() ? slot : it->second;
    };
    int32_t n = body_count;
    for (int32_t i = 0; i < count; ++i) {
        const int32_t index = body_indices[i];
        if (index < 0 || index >= n) {
            *error = "entry " + std::to_string(i) + ": body index " + std::to_string(index) + " outside the " + std::to_string(n) + " bodies at that entry";
            return BEPUCUDA_ERR_INVALID_ARGUMENT;
        }
        --n;
        if (index < n) at[index] = body_at(n);
        at.erase(n);
    }
    *final_count = n;
    moved_to->assign((size_t)count, -1);
    for (const auto& [slot, original] : at) (*moved_to)[(size_t)(original - n)] = slot;
    return BEPUCUDA_OK;
}

std::vector<WorkRecord> work_records(const TopologyPlan& plan, int32_t* refs, float* prestep, float* impulses) {
    std::vector<WorkRecord> records(plan.work.size());
    for (size_t i = 0; i < plan.work.size(); ++i) {
        const WorkItem& w = plan.work[i];
        const PlannedTypeBatch& tb = plan.tbs[(size_t)w.type_batch];
        const TypeInfo* t = get_type_info(tb.type_id);
        WorkRecord& r = records[i];
        r.refs = refs + tb.refs_offset + (size_t)w.bundle * t->bodies * 32;
        r.prestep = prestep + tb.prestep_offset + (size_t)w.bundle * t->prestep_rows * 32;
        r.impulses = impulses + tb.impulse_offset + (size_t)w.bundle * t->impulse_rows * 32;
        r.type_id = tb.type_id;
        r.live_lanes = plan.bundle_live[i];
    }
    return records;
}

// ---- stage program ---------------------------------------------------------------------------------------------------------
StageProgram build_stage_program(const TopologyPlan& plan, const std::vector<int32_t>& iterations, int kinematic_count, bool integrate_velocity_for_kinematics,
                                 bool peer_mode, int body_count) {
    StageProgram prog;
    std::vector<StageOp>& ops = prog.ops;
    std::vector<char> joins;  // per op: it belongs to the exchange point of the op before it (a later level of a fallback section)
    auto push = [&](int32_t stage, int32_t begin, int32_t count, int32_t exchange, int32_t flags, int64_t bytes, bool join = false) {
        ops.push_back({stage, begin, count, exchange, 0u, flags, bytes});
        joins.push_back(join);
    };
    // algorithmic bytes of one pass over a slice of the work list, summed once per device batch (a program repeats every batch many times)
    auto work_bytes = [&](int32_t begin, int32_t count, int32_t TypeInfo::*per) {
        int64_t bytes = 0;
        for (int32_t w = begin; w < begin + count; ++w)
            bytes += (int64_t)(get_type_info(plan.tbs[(size_t)plan.work[(size_t)w].type_batch].type_id)->*per) * plan.bundle_live[(size_t)w];
        return bytes;
    };
    std::vector<int64_t> warm_start_bytes, solve_bytes;
    for (const TopologyPlan::Batch& bw : plan.batches) {
        warm_start_bytes.push_back(work_bytes(bw.begin, bw.count, &TypeInfo::warm_start_bytes));
        solve_bytes.push_back(work_bytes(bw.begin, bw.count, &TypeInfo::solve_bytes));
    }
    // Peer mode with a fallback rank: the fallback section of a pass (its levels, in order, on the fallback rank alone) is one exchange point.
    // Boundary warps of every level wait for what peers pushed before the section, and the peers' next stage waits for every level's arrivals.
    const bool fallback_section = peer_mode && plan.fallback_rank >= 0;
    auto batch_stages = [&](int32_t stage, int32_t flags) {
        // in peer mode every rank runs the exchange point of every batch, also of one it has no constraint in
        for (size_t b = 0; b < plan.batches.size(); ++b) {
            const TopologyPlan::Batch& bw = plan.batches[b];
            if (bw.count > 0 || (peer_mode && (int)b < plan.sync_batch_count))
                push(stage, bw.begin, bw.count, peer_mode ? (int32_t)b : kNoExchange, flags | (bw.contacts_only ? kOpContactsOnly : 0),
                     stage == kStageSolve ? solve_bytes[b] : warm_start_bytes[b], fallback_section && (int)b > plan.sync_batch_count);
        }
        // a rank without fallback levels holds the section's place, as empty synchronized batches do
        if (fallback_section && plan.fallback_levels == 0) push(stage, plan.all_work_count, 0, plan.sync_batch_count, flags, 0);
    };
    // peer-sharded solves keep the integration in the owning lane, which also pushes the new records to the peers
    const int32_t integrable = plan.inc_count > 0 && !peer_mode ? kOpIntegrable : 0;
    const int64_t incremental_bytes = work_bytes(plan.inc_begin, plan.inc_count, &TypeInfo::incremental_bytes);
    const int64_t kinematic_bytes = (int64_t)kinematic_count * 108;  // per-body passes: 108 bytes per body
    const int substeps = (int)iterations.size();
    for (int s = 0; s < substeps; ++s) {
        if (s > 0) {
            // peer sharding: what peers pushed in the last Solve stages must have arrived before the contact update reads velocities
            if (peer_mode) push(kStageKinematic, 0, 0, kRankBarrier, 0, 0);
            if (plan.inc_count > 0) push(kStageIncremental, plan.inc_begin, plan.inc_count, kNoExchange, integrable, incremental_bytes);
            if (kinematic_count > 0) push(kStageKinematic, 0, kinematic_count, kNoExchange, 0, kinematic_bytes);
        } else if (integrate_velocity_for_kinematics && kinematic_count > 0) {
            push(kStageKinematicFirst, 0, kinematic_count, kNoExchange, 0, kinematic_bytes);
        }
        // all ranks meet before the first stage of a substep's WarmStart: after every peer's last Solve stage has completed, before any peer's
        // WarmStart stage stores into this rank's arrays
        if (peer_mode) push(kStageKinematic, 0, 0, kRankBarrier, 0, 0);
        if (s == 0) batch_stages(kStageWarmStartFirst, 0);
        else batch_stages(kStageWarmStart, integrable);
        for (int it = 0; it < iterations[(size_t)s]; ++it) batch_stages(kStageSolve, 0);
    }
    if (peer_mode) push(kStageKinematic, 0, 0, kRankBarrier, 0, 0);  // ... and before the final pose pass reads them
    push(kStageFinalPose, 0, body_count, kNoExchange, 0, (int64_t)body_count * 108);

    const StageOp* previous = nullptr;  // last launched stage (rank barriers write nothing)
    for (size_t i = 0; i < ops.size(); ++i) {
        StageOp& op = ops[i];
        op.exchange_index = joins[i] ? prog.exchange_count - 1 : prog.exchange_count;
        if (op.exchange != kNoExchange && !joins[i]) ++prog.exchange_count;
        if (op.exchange == kRankBarrier) continue;
        if (op.stage <= kStageIncremental) {
            // what the PDL prologue may read (DESIGN §3): not what the op launched just before writes
            if (op.stage != kStageIncremental && previous && previous->stage != kStageIncremental && !(previous->stage <= kStageSolve && previous->work_begin == op.work_begin))
                op.launch_flags |= kOpRowsFree;
            if (op.stage <= kStageSolve && previous && !(previous->stage <= kStageWarmStart && previous->work_begin == op.work_begin))
                op.launch_flags |= kOpBodiesFree;
        }
        if (op.stage == kStageFinalPose ? body_count > 0 : op.work_count > 0) previous = &op;
        if (op.work_count > 0 || op.stage == kStageFinalPose) ++prog.stage_count;
        if (op.stage != kStageKinematicFirst && op.stage != kStageKinematic) prog.algorithmic_bytes += op.algorithmic_bytes;
    }
    int64_t iterations_per_constraint = 0;
    for (int32_t n : iterations) iterations_per_constraint += n;
    prog.constraint_iterations = plan.constraint_count * iterations_per_constraint;
    return prog;
}

StageLaunch resolve_stage_launch(const StageOp& op, const LaunchContext& lc) {
    const int32_t ext = lc.integrator_extensions ? kLaunchIntegratorExtensions : 0;
    if (op.stage > kStageIncremental) return {kKernelFull, ext};  // the per-body passes
    const bool sharded = op.exchange != kNoExchange;
    StageLaunch l{kKernelFull, 0};
    if (op.stage != kStageIncremental && op.work_count >= kDeepBatchBundles) l.kernel = kKernelDeep;
    else if ((op.launch_flags & kOpContactsOnly) && !sharded) l.kernel = kKernelContacts;
    if (op.stage == kStageWarmStartFirst || op.stage == kStageWarmStart) l.flags |= ext;
    // The momentum-conserving angular modes need the orientation before the update in the owning lane; the point-gravity term reads the pose, and
    // loading it took the contact-only kExt WarmStart kernel past its register budget.
    if ((op.launch_flags & kOpIntegrable) && lc.angular_mode == 0 && !ext) l.flags |= kLaunchBodiesIntegrated;
    if (lc.profile) return l;
    l.flags |= kLaunchPdl | ((op.launch_flags & kOpRowsFree) ? kLaunchPrefetchRows : 0);
    // No body record before the wait on sharded kernels (a peer's stores are known to have arrived only after shard_wait) nor on deep ones (the
    // loads would spill there). A flagged WarmStart writes no pose and no world inertia, so the contact-only one loads world inertia like a Solve
    // stage unless its predecessor is the incremental update (which row prefetch excludes); no contact type reads a pose.
    if (!(op.launch_flags & kOpBodiesFree) || sharded || l.kernel == kKernelDeep) return l;
    if (!(l.flags & kLaunchBodiesIntegrated)) l.flags |= op.stage == kStageSolve ? kLaunchEarlyWorld : kLaunchEarlyOwned;
    else if (l.kernel == kKernelContacts && (l.flags & kLaunchPrefetchRows)) l.flags |= kLaunchEarlyWorld;
    return l;
}

bool same_launches(const LaunchContext& a, const LaunchContext& b) {
    // resolve_stage_launch reads the angular mode only as zero / non-zero, and only without integrator extensions
    return a.integrator_extensions == b.integrator_extensions && a.profile == b.profile &&
           (a.integrator_extensions || (a.angular_mode == 0) == (b.angular_mode == 0));
}

int exchange_targets(const StageProgram& program, const std::vector<int32_t>& boundary_count, std::vector<unsigned long long>* targets, std::string* error) {
    if (program.exchange_count + 1 > (uint32_t)kShardMaxExchanges) {
        *error = "peer sharding: more than 4095 exchange points per solve";
        return BEPUCUDA_ERR_BAD_STATE;
    }
    targets->assign((size_t)kShardMaxExchanges, 0ull);
    unsigned long long arrived = 0;
    for (const StageOp& op : program.ops) {
        if (op.exchange == kNoExchange) continue;
        if (op.exchange >= 0 && op.work_count > 0) arrived += (unsigned long long)boundary_count[(size_t)op.exchange];
        (*targets)[op.exchange_index] = arrived;
    }
    targets->back() = arrived;
    return BEPUCUDA_OK;
}

std::vector<int32_t> sort_boundary_first(const TopologyPlan& plan, const uint8_t* is_boundary, std::vector<WorkRecord>& records) {
    std::vector<int32_t> boundary_count(plan.batches.size(), 0);
    std::vector<WorkRecord> sorted;
    for (size_t b = 0; b < plan.batches.size(); ++b) {
        const int begin = plan.batches[b].begin, count = plan.batches[b].count;
        sorted.clear();
        for (int pass = 0; pass < 2; ++pass)
            for (int i = begin; i < begin + count; ++i)
                if ((is_boundary[(size_t)i] != 0) == (pass == 0)) {
                    WorkRecord r = records[(size_t)i];
                    r.live_lanes = (r.live_lanes & ~kRecordBoundaryBit) | (pass == 0 ? kRecordBoundaryBit : 0);
                    sorted.push_back(r);
                    boundary_count[b] += pass == 0;
                }
        std::copy(sorted.begin(), sorted.end(), records.begin() + begin);
    }
    return boundary_count;
}

}  // namespace bepucuda
