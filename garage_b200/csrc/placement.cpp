// Placement and quorums for erasure-coded blocks (SURVEY.md section 8 row f4): see
// include/garage_placement.h for what each entry point mirrors in the reference.  Pure host code.
#include "../../include/garage_placement.h"

#include <algorithm>
#include <cstring>
#include <limits>
#include <map>
#include <memory>
#include <new>
#include <queue>
#include <tuple>
#include <vector>

struct garage_layout {
    uint64_t version = 0;
    int n_nodes = 0, rf = 0;
    std::vector<int32_t> zone;
    std::vector<uint64_t> capacity;
    std::vector<uint8_t> ring;  // NB_PARTITIONS * rf node indices: shard i of partition p at ring[p*rf + i]
    uint64_t partition_size = 0;
};

namespace {

constexpr int NP = GARAGE_NB_PARTITIONS;

// ---------------------------------------------------------------- max flow (Dinic)
struct Flow {
    struct Edge {
        int to;
        int64_t cap;  // residual capacity
    };
    std::vector<Edge> e;               // edge 2i and its reverse 2i+1
    std::vector<std::vector<int>> adj; // vertex -> edge ids
    std::vector<int> level, it;
    explicit Flow(int n) : adj(n), level(n), it(n) {}
    int add(int u, int v, int64_t cap)
    {
        e.push_back({v, cap});
        e.push_back({u, 0});
        adj[u].push_back((int)e.size() - 2);
        adj[v].push_back((int)e.size() - 1);
        return (int)e.size() - 2;
    }
    bool bfs(int s, int t)
    {
        std::fill(level.begin(), level.end(), -1);
        std::queue<int> q;
        level[s] = 0;
        q.push(s);
        while (!q.empty()) {
            const int u = q.front();
            q.pop();
            for (int id : adj[u])
                if (e[id].cap > 0 && level[e[id].to] < 0) {
                    level[e[id].to] = level[u] + 1;
                    q.push(e[id].to);
                }
        }
        return level[t] >= 0;
    }
    int64_t dfs(int u, int t, int64_t f)
    {
        if (u == t) return f;
        for (int &i = it[u]; i < (int)adj[u].size(); i++) {
            const int id = adj[u][i];
            if (e[id].cap > 0 && level[e[id].to] == level[u] + 1) {
                const int64_t d = dfs(e[id].to, t, std::min(f, e[id].cap));
                if (d > 0) {
                    e[id].cap -= d;
                    e[id ^ 1].cap += d;
                    return d;
                }
            }
        }
        return 0;
    }
    int64_t run(int s, int t)  // augments whatever flow is already there
    {
        int64_t total = 0;
        while (bfs(s, t)) {
            std::fill(it.begin(), it.end(), 0);
            while (int64_t f = dfs(s, t, std::numeric_limits<int64_t>::max())) total += f;
        }
        return total;
    }
    int64_t flow_on(int id) const { return e[id ^ 1].cap; }
};

struct Problem {
    int n_nodes, rf, zr, max_per_zone;
    const int32_t *zone;
    const uint64_t *capacity;
    std::vector<int> storage;              // node ids with capacity
    std::vector<int> zone_id;              // per node: dense zone index (or -1 for gateways)
    int nz = 0;
};

// Vertices: S, T, per partition {up, down}, per (partition, zone) {in, out}, per storage node one.
// up carries zr units, at most one per zone (so >= zr zones are used); down carries the other rf - zr; a zone's
// total for one partition is capped between `in` and `out`; out -> node edges carry one shard; a node takes
// capacity / partition_size partitions.  (Same constraints as the reference's optimiser, version.rs:558-596.)
struct Graph {
    Flow f;
    int S, T;
    std::vector<int> assoc;  // edge id of (p, storage index) association
    std::vector<int> sink;   // edge id of node -> T
    std::vector<int64_t> held_back;  // capacity of node -> T not yet released (see `even`)
    // only_prev: associations that are not in that layout start closed (open_all() opens them).
    // even: a node's capacity starts at its proportional share of the NP * rf shards, the rest is released by
    // release_capacity() -- a maximum flow is otherwise free to fill 19 nodes to the brim and leave the 20th short.
    Graph(const Problem &P, uint64_t size, const garage_layout *only_prev, bool even = false)
        : f(2 + NP * 2 + NP * P.nz * 2 + (int)P.storage.size()), S(0), T(1)
    {
        const int ns = (int)P.storage.size();
        auto up = [&](int p) { return 2 + p * 2; };
        auto down = [&](int p) { return 2 + p * 2 + 1; };
        auto zin = [&](int p, int z) { return 2 + NP * 2 + (p * P.nz + z) * 2; };
        auto zout = [&](int p, int z) { return 2 + NP * 2 + (p * P.nz + z) * 2 + 1; };
        auto node = [&](int si) { return 2 + NP * 2 + NP * P.nz * 2 + si; };
        assoc.assign((size_t)NP * ns, -1);
        for (int p = 0; p < NP; p++) {
            f.add(S, up(p), P.zr);
            f.add(S, down(p), P.rf - P.zr);
            for (int z = 0; z < P.nz; z++) {
                f.add(up(p), zin(p, z), 1);
                f.add(down(p), zin(p, z), P.rf);
                f.add(zin(p, z), zout(p, z), P.max_per_zone > 0 ? P.max_per_zone : P.rf);
            }
        }
        long double total_cap = 0;
        for (int n : P.storage) total_cap += (long double)P.capacity[n];
        for (int si = 0; si < ns; si++) {
            const int n = P.storage[si];
            const int64_t full = (int64_t)std::min<uint64_t>(P.capacity[n] / size, NP);
            int64_t first = full;
            if (even) first = std::min<int64_t>(full, (int64_t)((long double)NP * P.rf * (long double)P.capacity[n] / total_cap));
            sink.push_back(f.add(node(si), T, first));
            held_back.push_back(full - first);
            for (int p = 0; p < NP; p++) {
                int64_t cap = 1;
                if (only_prev) {
                    cap = 0;
                    for (int i = 0; i < only_prev->rf; i++)
                        if (only_prev->ring[(size_t)p * only_prev->rf + i] == n) cap = 1;
                }
                assoc[(size_t)p * ns + si] = f.add(zout(p, P.zone_id[n]), node(si), cap);
            }
        }
    }
};

void open_all(Graph &g)
{
    for (int id : g.assoc)
        if (g.f.e[id].cap == 0 && g.f.flow_on(id) == 0) g.f.e[id].cap = 1;
}

void release_capacity(Graph &g)
{
    for (size_t i = 0; i < g.sink.size(); i++) {
        g.f.e[g.sink[i]].cap += g.held_back[i];
        g.held_back[i] = 0;
    }
}

bool feasible(const Problem &P, uint64_t size)
{
    if (size == 0) return false;
    Graph g(P, size, nullptr);
    return g.f.run(g.S, g.T) == (int64_t)NP * P.rf;
}

int setup(Problem &P, int n_nodes, const int32_t *zone, const uint64_t *capacity, int rf, int zone_redundancy,
          int max_per_zone)
{
    P.n_nodes = n_nodes;
    P.rf = rf;
    P.zone = zone;
    P.capacity = capacity;
    P.max_per_zone = max_per_zone;
    P.zone_id.assign(n_nodes, -1);
    std::map<int32_t, int> ids;
    for (int n = 0; n < n_nodes; n++)
        if (capacity[n] > 0) {
            P.storage.push_back(n);
            auto it = ids.find(zone[n]);
            if (it == ids.end()) it = ids.emplace(zone[n], (int)ids.size()).first;
            P.zone_id[n] = it->second;
        }
    P.nz = (int)ids.size();
    P.zr = zone_redundancy == 0 ? std::min(P.nz, rf) : zone_redundancy;
    if ((int)P.storage.size() < rf || P.nz < P.zr || P.zr > rf) return GARAGE_LAYOUT_E_INFEASIBLE;
    if (max_per_zone > 0 && (int64_t)max_per_zone * P.nz < rf) return GARAGE_LAYOUT_E_INFEASIBLE;
    return GARAGE_LAYOUT_OK;
}

bool valid_common(int n_nodes, const int32_t *zone, const uint64_t *capacity, int rf)
{
    return n_nodes >= 1 && n_nodes <= GARAGE_LAYOUT_MAX_NODES && zone && capacity && rf >= 1 && rf <= n_nodes;
}

}  // namespace

extern "C" {

int garage_layout_partition_of(const uint8_t hash[32])
{
    if (!hash) return GARAGE_LAYOUT_E_INVALID;
    const unsigned top = ((unsigned)hash[0] << 8) | hash[1];  // u16::from_be_bytes(hash[0..2])
    return (int)(top >> (16 - GARAGE_PARTITION_BITS));
}

int garage_layout_compute(garage_layout **out, uint64_t version, int n_nodes, const int32_t *zone,
                          const uint64_t *capacity, int replication_factor, int zone_redundancy, int max_per_zone,
                          const garage_layout *previous)
{
    if (!out) return GARAGE_LAYOUT_E_INVALID;
    *out = nullptr;
    if (!valid_common(n_nodes, zone, capacity, replication_factor) || zone_redundancy < 0 || max_per_zone < 0)
        return GARAGE_LAYOUT_E_INVALID;
    if (previous && (previous->n_nodes != n_nodes || previous->rf != replication_factor)) return GARAGE_LAYOUT_E_INVALID;
    try {
        Problem P;
        int rc = setup(P, n_nodes, zone, capacity, replication_factor, zone_redundancy, max_per_zone);
        if (rc) return rc;
        const int rf = replication_factor, ns = (int)P.storage.size();
        // largest partition size for which an assignment exists (feasibility is monotone in the size)
        uint64_t hi = 0, total = 0;
        for (int n : P.storage) {
            hi = std::max(hi, capacity[n]);
            total += capacity[n] / 4;  // (no overflow for 256 nodes of 2^56 bytes)
        }
        hi = std::min(hi, std::max<uint64_t>(1, total / ((uint64_t)NP * rf / 4)));  // the average load bounds the size
        if (!feasible(P, 1)) return GARAGE_LAYOUT_E_INFEASIBLE;
        uint64_t lo = 1;  // feasible
        while (lo < hi) {
            const uint64_t mid = lo + (hi - lo + 1) / 2;
            if (feasible(P, mid)) lo = mid;
            else hi = mid - 1;
        }
        // the assignment itself: first with the associations of the previous version only, then everything
        // (flow into the sink never shrinks while augmenting, so what a stage gave a node stays with it)
        Graph g(P, lo, previous, /*even=*/true);
        int64_t got = g.f.run(g.S, g.T);
        if (previous) {
            open_all(g);
            got += g.f.run(g.S, g.T);
        }
        release_capacity(g);
        got += g.f.run(g.S, g.T);
        if (got != (int64_t)NP * rf) return GARAGE_LAYOUT_E_INFEASIBLE;

        std::unique_ptr<garage_layout> L(new garage_layout());
        L->version = version;
        L->n_nodes = n_nodes;
        L->rf = rf;
        L->zone.assign(zone, zone + n_nodes);
        L->capacity.assign(capacity, capacity + n_nodes);
        L->partition_size = lo;
        L->ring.assign((size_t)NP * rf, 0);
        for (int p = 0; p < NP; p++) {
            std::vector<int> chosen;
            for (int si = 0; si < ns; si++)
                if (g.f.flow_on(g.assoc[(size_t)p * ns + si]) > 0) chosen.push_back(P.storage[si]);
            if ((int)chosen.size() != rf) return GARAGE_LAYOUT_E_INFEASIBLE;
            std::vector<int> slot(rf, -1);
            std::vector<char> placed(n_nodes, 0);
            if (previous)  // a node that stays keeps its shard index: its shard does not move
                for (int i = 0; i < rf; i++) {
                    const int n = previous->ring[(size_t)p * rf + i];
                    if (std::find(chosen.begin(), chosen.end(), n) != chosen.end()) {
                        slot[i] = n;
                        placed[n] = 1;
                    }
                }
            // the others: round-robin over zones (consecutive indices in different zones, so data shards are spread),
            // rotated by the partition number (which nodes hold parity varies from partition to partition)
            std::vector<std::vector<int>> by_zone(P.nz);
            for (int n : chosen)
                if (!placed[n]) by_zone[P.zone_id[n]].push_back(n);
            std::vector<int> rest;
            for (size_t r = 0;; r++) {
                bool any = false;
                for (int z = 0; z < P.nz; z++)
                    if (r < by_zone[z].size()) {
                        rest.push_back(by_zone[z][r]);
                        any = true;
                    }
                if (!any) break;
            }
            if (!rest.empty() && !previous) std::rotate(rest.begin(), rest.begin() + (p % (int)rest.size()), rest.end());
            size_t ri = 0;
            for (int i = 0; i < rf; i++)
                if (slot[i] < 0) slot[i] = rest[ri++];
            for (int i = 0; i < rf; i++) L->ring[(size_t)p * rf + i] = (uint8_t)slot[i];
        }
        *out = L.release();
        return GARAGE_LAYOUT_OK;
    } catch (const std::bad_alloc &) {
        return GARAGE_LAYOUT_E_NOMEM;
    }
}

int garage_layout_from_ring(garage_layout **out, uint64_t version, int n_nodes, const int32_t *zone,
                            const uint64_t *capacity, int replication_factor, const uint8_t *ring)
{
    if (!out) return GARAGE_LAYOUT_E_INVALID;
    *out = nullptr;
    if (!valid_common(n_nodes, zone, capacity, replication_factor) || !ring) return GARAGE_LAYOUT_E_INVALID;
    for (size_t i = 0; i < (size_t)NP * replication_factor; i++)
        if (ring[i] >= n_nodes) return GARAGE_LAYOUT_E_INVALID;
    try {
        std::unique_ptr<garage_layout> L(new garage_layout());
        L->version = version;
        L->n_nodes = n_nodes;
        L->rf = replication_factor;
        L->zone.assign(zone, zone + n_nodes);
        L->capacity.assign(capacity, capacity + n_nodes);
        L->ring.assign(ring, ring + (size_t)NP * replication_factor);
        *out = L.release();
        return GARAGE_LAYOUT_OK;
    } catch (const std::bad_alloc &) {
        return GARAGE_LAYOUT_E_NOMEM;
    }
}

void garage_layout_free(garage_layout *l) { delete l; }

int garage_layout_nodes_of(const garage_layout *l, const uint8_t hash[32], int32_t *out)
{
    if (!l || !hash || !out) return GARAGE_LAYOUT_E_INVALID;
    const int p = garage_layout_partition_of(hash);
    for (int i = 0; i < l->rf; i++) out[i] = l->ring[(size_t)p * l->rf + i];
    return GARAGE_LAYOUT_OK;
}

int garage_layout_ring(const garage_layout *l, uint8_t *out)
{
    if (!l || !out) return GARAGE_LAYOUT_E_INVALID;
    memcpy(out, l->ring.data(), l->ring.size());
    return GARAGE_LAYOUT_OK;
}

int garage_layout_replication_factor(const garage_layout *l) { return l ? l->rf : GARAGE_LAYOUT_E_INVALID; }
uint64_t garage_layout_version(const garage_layout *l) { return l ? l->version : 0; }
uint64_t garage_layout_partition_size(const garage_layout *l) { return l ? l->partition_size : 0; }

int garage_layout_check(const garage_layout *l, int zone_redundancy, int max_per_zone, garage_layout_stats *stats)
{
    if (!l || zone_redundancy < 0 || max_per_zone < 0) return GARAGE_LAYOUT_E_INVALID;
    try {
        std::map<int32_t, int> ids;
        int storage = 0;
        for (int n = 0; n < l->n_nodes; n++)
            if (l->capacity[n] > 0) {
                storage++;
                ids.emplace(l->zone[n], 0);
            }
        const int nz = (int)ids.size();
        const int zr = zone_redundancy == 0 ? std::min(nz, l->rf) : zone_redundancy;
        std::vector<int> load(l->n_nodes, 0);
        int min_zones = l->rf, max_zone_load = 0, rc = GARAGE_LAYOUT_OK;
        auto fail = [&](int code) {
            if (rc == GARAGE_LAYOUT_OK) rc = code;
        };
        for (int p = 0; p < NP; p++) {
            std::map<int32_t, int> zl;
            std::vector<char> seen(l->n_nodes, 0);
            for (int i = 0; i < l->rf; i++) {
                const int n = l->ring[(size_t)p * l->rf + i];
                if (seen[n]) fail(GARAGE_LAYOUT_E_DUPLICATE);
                seen[n] = 1;
                if (l->capacity[n] == 0) fail(GARAGE_LAYOUT_E_GATEWAY);
                load[n]++;
                zl[l->zone[n]]++;
            }
            min_zones = std::min(min_zones, (int)zl.size());
            for (auto &kv : zl) max_zone_load = std::max(max_zone_load, kv.second);
        }
        if (min_zones < zr) fail(GARAGE_LAYOUT_E_ZONES);
        if (max_per_zone > 0 && max_zone_load > max_per_zone) fail(GARAGE_LAYOUT_E_ZONE_LOAD);
        int lo = NP + 1, hi = 0;
        for (int n = 0; n < l->n_nodes; n++)
            if (l->capacity[n] > 0) {
                lo = std::min(lo, load[n]);
                hi = std::max(hi, load[n]);
                if (l->partition_size > 0 && (uint64_t)load[n] > l->capacity[n] / l->partition_size) fail(GARAGE_LAYOUT_E_CAPACITY);
            }
        if (stats) {
            stats->min_zones_per_partition = min_zones;
            stats->max_shards_per_zone = max_zone_load;
            stats->min_partitions_per_node = storage ? lo : 0;
            stats->max_partitions_per_node = hi;
            stats->storage_nodes = storage;
            stats->zones = nz;
        }
        return rc;
    } catch (const std::bad_alloc &) {
        return GARAGE_LAYOUT_E_NOMEM;
    }
}

int garage_layout_transition(const garage_layout *from, const garage_layout *to, int partition, int32_t *index,
                             int32_t *node_from, int32_t *node_to)
{
    if (!from || !to || from->rf != to->rf || partition >= NP) return GARAGE_LAYOUT_E_INVALID;
    const int rf = from->rf;
    int count = 0;
    for (int p = partition < 0 ? 0 : partition; p < (partition < 0 ? NP : partition + 1); p++)
        for (int i = 0; i < rf; i++) {
            const int a = from->ring[(size_t)p * rf + i], b = to->ring[(size_t)p * rf + i];
            if (a == b) continue;
            if (partition >= 0) {
                if (index) index[count] = i;
                if (node_from) node_from[count] = a;
                if (node_to) node_to[count] = b;
            }
            count++;
        }
    return count;
}

// ---------------------------------------------------------------- quorums
int garage_ec_write_quorum(int k, int m, int mode)
{
    if (k < 1 || m < 0 || mode < GARAGE_CONSISTENT || mode > GARAGE_DANGEROUS) return GARAGE_LAYOUT_E_INVALID;
    return mode == GARAGE_DANGEROUS ? k : std::min(k + m, k + 1);
}

int garage_ec_read_quorum(int k, int m, int mode)
{
    if (k < 1 || m < 0 || mode < GARAGE_CONSISTENT || mode > GARAGE_DANGEROUS) return GARAGE_LAYOUT_E_INVALID;
    return k;
}

// ---------------------------------------------------------------- write plan + quorum sets
int garage_layout_write_plan(const garage_layout *const *versions, int n_versions, const uint8_t hash[32],
                             garage_shard_request *out, int cap)
{
    if (!versions || n_versions < 1 || n_versions > 32 || !hash || !out) return GARAGE_LAYOUT_E_INVALID;
    for (int v = 0; v < n_versions; v++)
        if (!versions[v] || versions[v]->rf != versions[0]->rf) return GARAGE_LAYOUT_E_INVALID;
    const int rf = versions[0]->rf, p = garage_layout_partition_of(hash);
    int n = 0;
    for (int v = 0; v < n_versions; v++)
        for (int i = 0; i < rf; i++) {
            const int node = versions[v]->ring[(size_t)p * rf + i];
            int j = 0;
            while (j < n && !(out[j].node == node && out[j].index == i)) j++;
            if (j == n) {
                if (n == cap) return GARAGE_LAYOUT_E_INVALID;
                out[n].node = node;
                out[n].index = i;
                out[n].set_mask = 0;
                n++;
            }
            out[j].set_mask |= 1u << v;
        }
    return n;
}

}  // extern "C"

struct garage_quorum_tracker {
    std::vector<uint32_t> mask;  // per request
    std::vector<int8_t> result;  // 0 unknown, 1 ok, -1 failed
    std::vector<int> ok, err, len;
    int quorum = 0, state = GARAGE_QUORUM_PENDING;
};

extern "C" {

int garage_quorum_tracker_new(garage_quorum_tracker **out, const garage_shard_request *reqs, int n_reqs, int n_sets,
                              int quorum)
{
    if (!out) return GARAGE_LAYOUT_E_INVALID;
    *out = nullptr;
    if (!reqs || n_reqs < 1 || n_sets < 1 || n_sets > 32 || quorum < 1) return GARAGE_LAYOUT_E_INVALID;
    try {
        std::unique_ptr<garage_quorum_tracker> t(new garage_quorum_tracker());
        t->quorum = quorum;
        t->ok.assign(n_sets, 0);
        t->err.assign(n_sets, 0);
        t->len.assign(n_sets, 0);
        t->result.assign(n_reqs, 0);
        for (int i = 0; i < n_reqs; i++) {
            if (n_sets < 32 && (reqs[i].set_mask >> n_sets) != 0) return GARAGE_LAYOUT_E_INVALID;
            t->mask.push_back(reqs[i].set_mask);
            for (int s = 0; s < n_sets; s++)
                if (reqs[i].set_mask >> s & 1) t->len[s]++;
        }
        // a set smaller than the quorum can never succeed (rpc_helper.rs:737-742 reports that on the first failure;
        // here it is known up front)
        for (int s = 0; s < n_sets; s++)
            if (t->len[s] < quorum) t->state = GARAGE_QUORUM_FAILED;
        *out = t.release();
        return GARAGE_LAYOUT_OK;
    } catch (const std::bad_alloc &) {
        return GARAGE_LAYOUT_E_NOMEM;
    }
}

int garage_quorum_tracker_register(garage_quorum_tracker *t, int request, int ok)
{
    if (!t || request < 0 || request >= (int)t->result.size()) return GARAGE_LAYOUT_E_INVALID;
    if (t->result[request] != 0) return t->state;  // a request answers once
    t->result[request] = ok ? 1 : -1;
    for (size_t s = 0; s < t->ok.size(); s++)
        if (t->mask[request] >> s & 1) (ok ? t->ok[s] : t->err[s])++;
    if (t->state != GARAGE_QUORUM_PENDING) return t->state;  // decided earlier: later answers change nothing
    bool all = true, dead = false;
    for (size_t s = 0; s < t->ok.size(); s++) {
        all &= t->ok[s] >= t->quorum;
        dead |= t->err[s] + t->quorum > t->len[s];
    }
    if (all) t->state = GARAGE_QUORUM_OK;  // checked first, like try_write_many_sets_inner
    else if (dead) t->state = GARAGE_QUORUM_FAILED;
    return t->state;
}

int garage_quorum_tracker_state(const garage_quorum_tracker *t) { return t ? t->state : GARAGE_LAYOUT_E_INVALID; }
void garage_quorum_tracker_free(garage_quorum_tracker *t) { delete t; }

// ---------------------------------------------------------------- read plan
int garage_layout_read_plan(const garage_layout *const *active, int n_active, const garage_layout *const *old, int n_old,
                            const uint8_t hash[32], int k, int our_node, const uint32_t *ping_us, garage_shard_source *out,
                            int cap)
{
    if (!active || n_active < 1 || n_old < 0 || (n_old > 0 && !old) || !hash || !out || k < 1) return GARAGE_LAYOUT_E_INVALID;
    const garage_layout *cur = active[n_active - 1];
    if (!cur || k > cur->rf) return GARAGE_LAYOUT_E_INVALID;
    for (int v = 0; v < n_active; v++)
        if (!active[v] || active[v]->rf != cur->rf || active[v]->n_nodes != cur->n_nodes) return GARAGE_LAYOUT_E_INVALID;
    for (int v = 0; v < n_old; v++)
        if (!old[v] || old[v]->rf != cur->rf || old[v]->n_nodes != cur->n_nodes) return GARAGE_LAYOUT_E_INVALID;
    try {
        const int rf = cur->rf, p = garage_layout_partition_of(hash);
        const bool have_zone = our_node >= 0 && our_node < cur->n_nodes;
        const int32_t our_zone = have_zone ? cur->zone[our_node] : 0;
        // request_order (rpc_helper.rs:621-660) with "is a parity shard" in front: k data shards need no decode
        auto ordered = [&](const garage_layout *l) {
            std::vector<int> idx(rf);
            for (int i = 0; i < rf; i++) idx[i] = i;
            auto key = [&](int i) {
                const int n = l->ring[(size_t)p * rf + i];
                const uint32_t ping = ping_us ? ping_us[n] : 10000000u;
                return std::make_tuple(i >= k, n != our_node, !have_zone || cur->zone[n] != our_zone, ping, i);
            };
            std::stable_sort(idx.begin(), idx.end(), [&](int a, int b) { return key(a) < key(b); });
            return idx;
        };
        std::vector<garage_shard_source> plan;
        auto has = [&](int node, int index) {
            for (auto &s : plan)
                if (s.node == node && s.index == index) return true;
            return false;
        };
        if (n_active == 1) {
            for (int i : ordered(cur)) plan.push_back({(int32_t)cur->ring[(size_t)p * rf + i], i, 0});
        } else {
            std::vector<std::vector<int>> ord;
            for (int v = 0; v < n_active; v++) ord.push_back(ordered(active[v]));
            for (int r = 0; r < rf; r++)
                for (int v = 0; v < n_active; v++) {  // older versions first: most blocks predate the change
                    const int i = ord[v][r], n = active[v]->ring[(size_t)p * rf + i];
                    if (has(n, i)) continue;
                    const garage_shard_source s{n, i, v};
                    if (n == our_node) plan.insert(plan.begin(), s);  // asking ourselves is free
                    else plan.push_back(s);
                }
        }
        for (int v = 0; v < n_old; v++)  // blocks not yet moved to their new nodes
            for (int i : ordered(old[v])) {
                const int n = old[v]->ring[(size_t)p * rf + i];
                if (!has(n, i)) plan.push_back({n, i, n_active + v});
            }
        if ((int)plan.size() > cap) return GARAGE_LAYOUT_E_INVALID;
        std::copy(plan.begin(), plan.end(), out);
        return (int)plan.size();
    } catch (const std::bad_alloc &) {
        return GARAGE_LAYOUT_E_NOMEM;
    }
}

}  // extern "C"

// ================================================================= drive layout (DESIGN.md section 5.7)
struct garage_drive_layout {
    std::vector<uint64_t> capacity;            // per directory: 0 = read-only
    std::vector<uint8_t> prim;                 // GARAGE_DRIVE_NPART primaries
    std::vector<std::vector<uint8_t>> sec;     // per partition: secondaries in read order
};

namespace {

constexpr int DNP = GARAGE_DRIVE_NPART;

bool drive_dirs_ok(int n_dirs, const uint64_t *capacity)
{
    if (n_dirs < 1 || n_dirs > GARAGE_DRIVE_MAX_DIRS || !capacity) return false;
    for (int i = 0; i < n_dirs; i++)
        if (capacity[i] > 0) return true;
    return false;
}

// end of directory i's run of partitions: floor(cumulative capacity through i * NPART / total capacity).  The
// product fits in 128 bits for any u64 capacities.
std::vector<int> drive_run_ends(int n_dirs, const uint64_t *capacity)
{
    unsigned __int128 total = 0, cum = 0;
    for (int i = 0; i < n_dirs; i++) total += capacity[i];
    std::vector<int> end(n_dirs);
    for (int i = 0; i < n_dirs; i++) {
        cum += capacity[i];
        end[i] = (int)(cum * DNP / total);
    }
    return end;
}

// every non-empty directory with only[i] set becomes a secondary of each partition it is not primary of, unless it is one
// already
void drive_add_non_empty(garage_drive_layout &l, const uint8_t *non_empty, const std::vector<uint8_t> &only)
{
    if (!non_empty) return;
    for (int i = 0; i < (int)l.capacity.size(); i++) {
        if (!non_empty[i] || !only[i]) continue;
        for (int p = 0; p < DNP; p++)
            if (l.prim[p] != i && std::find(l.sec[p].begin(), l.sec[p].end(), (uint8_t)i) == l.sec[p].end())
                l.sec[p].push_back((uint8_t)i);
    }
}

}  // namespace

extern "C" {

int garage_drive_partition_of(const uint8_t hash[32])
{
    if (!hash) return GARAGE_LAYOUT_E_INVALID;
    return (int)((((unsigned)hash[2] << 8) | hash[3]) % DNP);
}

int garage_drive_layout_init(garage_drive_layout **out, int n_dirs, const uint64_t *capacity, const uint8_t *non_empty)
{
    if (!out) return GARAGE_LAYOUT_E_INVALID;
    *out = nullptr;
    if (!drive_dirs_ok(n_dirs, capacity)) return GARAGE_LAYOUT_E_INVALID;
    try {
        std::unique_ptr<garage_drive_layout> l(new garage_drive_layout());
        l->capacity.assign(capacity, capacity + n_dirs);
        l->prim.assign(DNP, 0);
        l->sec.assign(DNP, {});
        const std::vector<int> end = drive_run_ends(n_dirs, capacity);
        for (int i = 0, p = 0; i < n_dirs; i++)  // a read-only directory's run is empty
            for (; p < end[i]; p++) l->prim[p] = (uint8_t)i;
        drive_add_non_empty(*l, non_empty, std::vector<uint8_t>(n_dirs, 1));
        *out = l.release();
        return GARAGE_LAYOUT_OK;
    } catch (const std::bad_alloc &) {
        return GARAGE_LAYOUT_E_NOMEM;
    }
}

int garage_drive_layout_update(garage_drive_layout **out, const garage_drive_layout *prev, const int *prev_index,
                               int n_dirs, const uint64_t *capacity, const uint8_t *non_empty)
{
    if (!out) return GARAGE_LAYOUT_E_INVALID;
    *out = nullptr;
    if (!prev || !prev_index || !drive_dirs_ok(n_dirs, capacity)) return GARAGE_LAYOUT_E_INVALID;
    const int n_prev = (int)prev->capacity.size();
    try {
        std::vector<int> old2new(n_prev, -1);
        for (int i = 0; i < n_dirs; i++) {
            const int o = prev_index[i];
            if (o < -1 || o >= n_prev || (o >= 0 && old2new[o] >= 0)) return GARAGE_LAYOUT_E_INVALID;
            if (o >= 0) old2new[o] = i;
        }
        std::unique_ptr<garage_drive_layout> l(new garage_drive_layout());
        bool same = n_dirs == n_prev;
        for (int i = 0; same && i < n_dirs; i++) same = prev_index[i] == i && capacity[i] == prev->capacity[i];
        if (same) {  // the same list: the same layout
            *l = *prev;
            *out = l.release();
            return GARAGE_LAYOUT_OK;
        }
        l->capacity.assign(capacity, capacity + n_dirs);
        l->prim.assign(DNP, 0);
        l->sec.assign(DNP, {});
        // secondaries carry over, removed directories dropped
        for (int p = 0; p < DNP; p++)
            for (uint8_t o : prev->sec[p])
                if (old2new[o] >= 0) l->sec[p].push_back((uint8_t)old2new[o]);
        // each surviving directory keeps its primaries (in partition order)
        std::vector<std::vector<int>> dir_prim(n_dirs);
        for (int p = 0; p < DNP; p++)
            if (old2new[prev->prim[p]] >= 0) dir_prim[old2new[prev->prim[p]]].push_back(p);
        // targets: differences of the floors of cumulative capacity
        std::vector<int> target(n_dirs, 0);
        const std::vector<int> end = drive_run_ends(n_dirs, capacity);
        for (int i = 0; i < n_dirs; i++) target[i] = end[i] - (i ? end[i - 1] : 0);
        // over target: give up the highest-numbered partitions, keeping them as a secondary
        for (int i = 0; i < n_dirs; i++)
            while ((int)dir_prim[i].size() > target[i]) {
                const int p = dir_prim[i].back();
                dir_prim[i].pop_back();
                if (std::find(l->sec[p].begin(), l->sec[p].end(), (uint8_t)i) == l->sec[p].end())
                    l->sec[p].push_back((uint8_t)i);
            }
        std::vector<int> owner(DNP, -1);
        for (int i = 0; i < n_dirs; i++)
            for (int p : dir_prim[i]) owner[p] = i;
        std::vector<int> unassigned;
        for (int p = 0; p < DNP; p++)
            if (owner[p] < 0) unassigned.push_back(p);
        // below target, in list order: take unassigned partitions, highest-numbered first
        for (int i = 0; i < n_dirs; i++)
            for (int need = target[i] - (int)dir_prim[i].size(); need > 0; need--) {
                const int p = unassigned.back();
                unassigned.pop_back();
                owner[p] = i;
                auto &s = l->sec[p];
                s.erase(std::remove(s.begin(), s.end(), (uint8_t)i), s.end());
            }
        for (int p = 0; p < DNP; p++) l->prim[p] = (uint8_t)owner[p];
        // newly listed non-empty directories become secondaries everywhere they are not primary
        std::vector<uint8_t> fresh(n_dirs);
        for (int i = 0; i < n_dirs; i++) fresh[i] = prev_index[i] < 0;
        drive_add_non_empty(*l, non_empty, fresh);
        *out = l.release();
        return GARAGE_LAYOUT_OK;
    } catch (const std::bad_alloc &) {
        return GARAGE_LAYOUT_E_NOMEM;
    }
}

int garage_drive_layout_drop_secondaries(garage_drive_layout **out, const garage_drive_layout *l)
{
    if (!out) return GARAGE_LAYOUT_E_INVALID;
    *out = nullptr;
    if (!l) return GARAGE_LAYOUT_E_INVALID;
    try {
        std::unique_ptr<garage_drive_layout> r(new garage_drive_layout(*l));
        for (auto &s : r->sec) s.clear();
        *out = r.release();
        return GARAGE_LAYOUT_OK;
    } catch (const std::bad_alloc &) {
        return GARAGE_LAYOUT_E_NOMEM;
    }
}

int garage_drive_layout_n_dirs(const garage_drive_layout *l) { return l ? (int)l->capacity.size() : GARAGE_LAYOUT_E_INVALID; }

int garage_drive_layout_primary(const garage_drive_layout *l, int part)
{
    if (!l || part < 0 || part >= DNP) return GARAGE_LAYOUT_E_INVALID;
    return l->prim[part];
}

int garage_drive_layout_secondaries(const garage_drive_layout *l, int part, uint8_t *out, int cap)
{
    if (!l || part < 0 || part >= DNP || cap < 0 || (cap > 0 && !out)) return GARAGE_LAYOUT_E_INVALID;
    const auto &s = l->sec[part];
    for (int i = 0; i < (int)s.size() && i < cap; i++) out[i] = s[i];
    return (int)s.size();
}

// image: "GDL1", n_dirs, n_dirs little-endian u64 capacities, then per partition: primary, count, secondaries
size_t garage_drive_layout_serialize(const garage_drive_layout *l, uint8_t *out, size_t cap)
{
    if (!l) return 0;
    std::vector<uint8_t> b = {'G', 'D', 'L', '1', (uint8_t)l->capacity.size()};
    for (uint64_t c : l->capacity)
        for (int j = 0; j < 8; j++) b.push_back((uint8_t)(c >> (8 * j)));
    for (int p = 0; p < DNP; p++) {
        b.push_back(l->prim[p]);
        b.push_back((uint8_t)l->sec[p].size());
        b.insert(b.end(), l->sec[p].begin(), l->sec[p].end());
    }
    if (out && cap >= b.size()) memcpy(out, b.data(), b.size());
    return b.size();
}

int garage_drive_layout_deserialize(garage_drive_layout **out, const uint8_t *buf, size_t len)
{
    if (!out) return GARAGE_LAYOUT_E_INVALID;
    *out = nullptr;
    if (!buf || len < 5 || memcmp(buf, "GDL1", 4) != 0) return GARAGE_LAYOUT_E_INVALID;
    try {
        std::unique_ptr<garage_drive_layout> l(new garage_drive_layout());
        const int n = buf[4];
        size_t at = 5;
        if (len < at + (size_t)n * 8) return GARAGE_LAYOUT_E_INVALID;
        l->capacity.assign(n, 0);
        for (int i = 0; i < n; i++, at += 8)
            for (int j = 0; j < 8; j++) l->capacity[i] |= (uint64_t)buf[at + j] << (8 * j);
        if (!drive_dirs_ok(n, l->capacity.data())) return GARAGE_LAYOUT_E_INVALID;
        l->prim.assign(DNP, 0);
        l->sec.assign(DNP, {});
        for (int p = 0; p < DNP; p++) {
            if (at + 2 > len) return GARAGE_LAYOUT_E_INVALID;
            const int pr = buf[at], ns = buf[at + 1];
            at += 2;
            if (pr >= n || l->capacity[pr] == 0 || ns >= n || at + ns > len) return GARAGE_LAYOUT_E_INVALID;
            l->prim[p] = (uint8_t)pr;
            for (int j = 0; j < ns; j++) {
                const uint8_t d = buf[at + j];
                auto &s = l->sec[p];
                if (d >= n || d == pr || std::find(s.begin(), s.end(), d) != s.end()) return GARAGE_LAYOUT_E_INVALID;
                s.push_back(d);
            }
            at += ns;
        }
        if (at != len) return GARAGE_LAYOUT_E_INVALID;
        *out = l.release();
        return GARAGE_LAYOUT_OK;
    } catch (const std::bad_alloc &) {
        return GARAGE_LAYOUT_E_NOMEM;
    }
}

void garage_drive_layout_free(garage_drive_layout *l) { delete l; }

}  // extern "C"
