// CPU restatement of IslandSleeper.CollectIsland (BepuPhysics/IslandSleeper.cs:L113-223) over the active constraint graph of a set of
// reference-layout (AOSOA-W) type batches: the checker tests/test_islands.py holds bepucuda_find_sleepable_islands to. Test infrastructure only,
// compiled for the host by tests/island_checker.py.
#include <algorithm>
#include <cstdint>
#include <vector>

namespace {

// Bodies_GatherScatter.cs:L107-139: bit 30 marks a kinematic body, bit 31 an empty lane; the rest is the active-set index
constexpr int32_t kBodyReferenceMask = (int32_t)~((1u << 31) | (1u << 30));

struct IslandGraph {
    // Bodies.ActiveSet.Constraints[bodyIndex] (the constraint list of every body) and, per constraint, the decoded references
    // Solver.EnumerateConnectedBodyReferences reports (Solver.cs:L1765-1784: the kinematic flag is stripped). Empty lanes (-1) are no constraint.
    std::vector<int32_t> body_begin, body_constraints, constraint_begin, constraint_bodies;
};
struct ForcedSleepPredicate {  // IslandSleeper.cs:L76-84
    bool matches(int) const { return true; }
};
struct SleepPredicate {  // IslandSleeper.cs:L85-93: Bodies.ActiveSet.Activity[bodyIndex].SleepCandidate
    const uint8_t* candidates;
    bool matches(int bodyIndex) const { return candidates[bodyIndex] != 0; }
};
// consideredBodies / consideredConstraints are the IndexSets CollectIsland creates empty per call (L191-192); the caller passes them cleared and
// gets them back cleared, which saves allocating one bit per active body for every traversal.
struct IslandScratch {
    std::vector<uint8_t> considered_bodies, considered_constraints;
    std::vector<int32_t> touched_constraints, visitation_stack;
};

// PushBody, L113-128
template <class TPredicate>
bool push_body(int bodyIndex, IslandScratch& s, std::vector<int32_t>& bodyIndices, const TPredicate& predicate) {
    if (!s.considered_bodies[bodyIndex]) {
        if (!predicate.matches(bodyIndex)) return false;
        bodyIndices.push_back(bodyIndex);
        s.considered_bodies[bodyIndex] = 1;
        s.visitation_stack.push_back(bodyIndex);
    }
    return true;
}

// EnqueueUnvisitedNeighbors, L131-161: every not yet considered constraint of the body, followed to each of its OTHER bodies (ConstraintBodyEnumerator,
// L60-73, skips the source body)
template <class TPredicate>
bool enqueue_unvisited_neighbors(const IslandGraph& g, int bodyIndex, IslandScratch& s, std::vector<int32_t>& bodyIndices, const TPredicate& predicate) {
    for (int i = g.body_begin[bodyIndex]; i < g.body_begin[bodyIndex + 1]; ++i) {
        const int c = g.body_constraints[i];
        if (s.considered_constraints[c]) continue;
        s.considered_constraints[c] = 1;
        s.touched_constraints.push_back(c);
        for (int j = g.constraint_begin[c]; j < g.constraint_begin[c + 1]; ++j) {
            const int connected = g.constraint_bodies[j];
            if (connected == bodyIndex) continue;
            if (!push_body(connected, s, bodyIndices, predicate)) return false;
        }
    }
    return true;
}

// CollectIsland, L174-223. bodyIndices receives the traversed bodies that pass the predicate.
template <class TPredicate>
bool collect_island(const IslandGraph& g, int startingActiveBodyIndex, IslandScratch& s, std::vector<int32_t>& bodyIndices, const TPredicate& predicate) {
    bool disqualified = !push_body(startingActiveBodyIndex, s, bodyIndices, predicate);
    while (!disqualified && !s.visitation_stack.empty()) {
        const int next = s.visitation_stack.back();  // TryPop: depth first
        s.visitation_stack.pop_back();
        disqualified = !enqueue_unvisited_neighbors(g, next, s, bodyIndices, predicate);
    }
    // what the Dispose calls of L218-221 amount to: the next traversal starts with empty sets
    for (int b : bodyIndices) s.considered_bodies[b] = 0;
    for (int c : s.touched_constraints) s.considered_constraints[c] = 0;
    s.touched_constraints.clear();
    s.visitation_stack.clear();
    return !disqualified;
}

}  // namespace

// One reference-layout type batch: body_references[bundle][slot][bundle_width], `bodies` slots per constraint.
struct island_type_batch {
    int32_t bodies;
    int32_t constraint_count;
    const int32_t* body_references;
};

// Runs CollectIsland from every body that no earlier traversal reached, in ascending index order, so the start is the island's smallest index: once
// with ForcedSleepPredicate to collect the whole island (labels, body count) and once with SleepPredicate for the verdict. The outputs are those of
// bepucuda_find_sleepable_islands. Returns the number of sleepable islands, negative on bad arguments.
extern "C" int32_t collect_sleepable_islands(const island_type_batch* type_batches, int32_t type_batch_count, int32_t bundle_width, int32_t body_count,
                                             const uint8_t* sleep_candidates, int32_t* island_of_body_out, int32_t* sleepable_roots_out,
                                             int32_t* sleepable_body_counts_out) {
    if (body_count < 0 || type_batch_count < 0 || bundle_width < 1) return -1;
    IslandGraph g;
    std::vector<int32_t> degree((size_t)body_count + 1, 0);
    g.constraint_begin.push_back(0);
    for (int t = 0; t < type_batch_count; ++t) {
        const island_type_batch& tb = type_batches[t];
        if (tb.bodies < 1 || tb.bodies > 4) return -3;
        for (int i = 0; i < tb.constraint_count; ++i) {
            const size_t bundle = (size_t)(i / bundle_width), inner = (size_t)(i % bundle_width);
            const size_t first = g.constraint_bodies.size();
            for (int slot = 0; slot < tb.bodies; ++slot) {
                const int32_t raw = tb.body_references[(bundle * tb.bodies + slot) * bundle_width + inner];
                if (raw < 0) continue;
                const int32_t index = raw & kBodyReferenceMask;
                if (index >= body_count) return -2;
                // a body one constraint references twice (a kinematic one) gets the constraint once in its list
                if (std::find(g.constraint_bodies.begin() + first, g.constraint_bodies.end(), index) != g.constraint_bodies.end()) continue;
                g.constraint_bodies.push_back(index);
                ++degree[index];
            }
            if (g.constraint_bodies.size() > first) g.constraint_begin.push_back((int32_t)g.constraint_bodies.size());
        }
    }
    const int constraint_count = (int)g.constraint_begin.size() - 1;
    g.body_begin.assign((size_t)body_count + 1, 0);
    for (int i = 0; i < body_count; ++i) g.body_begin[i + 1] = g.body_begin[i] + degree[i];
    g.body_constraints.resize(g.constraint_bodies.size());
    std::vector<int32_t> fill(g.body_begin.begin(), g.body_begin.end() - 1);
    for (int c = 0; c < constraint_count; ++c)
        for (int j = g.constraint_begin[c]; j < g.constraint_begin[c + 1]; ++j) g.body_constraints[fill[g.constraint_bodies[j]]++] = c;
    IslandScratch s;
    s.considered_bodies.assign((size_t)body_count, 0);
    s.considered_constraints.assign((size_t)constraint_count, 0);
    std::vector<uint8_t> assigned((size_t)body_count, 0);
    std::vector<int32_t> island, passing;
    const ForcedSleepPredicate everything{};
    const SleepPredicate sleepable{sleep_candidates};
    int32_t count = 0;
    for (int start = 0; start < body_count; ++start) {
        if (assigned[start]) continue;
        island.clear();
        collect_island(g, start, s, island, everything);
        for (int b : island) {
            assigned[b] = 1;
            if (island_of_body_out) island_of_body_out[b] = start;
        }
        passing.clear();
        if (collect_island(g, start, s, passing, sleepable)) {
            sleepable_roots_out[count] = start;
            sleepable_body_counts_out[count] = (int32_t)island.size();
            ++count;
        }
    }
    return count;
}
