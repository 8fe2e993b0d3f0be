/*
 * garage_placement.h -- placement and quorums for erasure-coded blocks (SURVEY.md section 8 row f4),
 * part of libgarage_block.so.  Pure host code: no CUDA, no I/O.
 *
 * What the reference does for replicated blocks, and what changes with shards:
 *
 *  - `LayoutVersion::nodes_of(hash, n)` (src/rpc/layout/version.rs:117-137) maps the top
 *    PARTITION_BITS = 8 bits of the hash (`partition_of`, :101-104) to `replication_factor`
 *    nodes out of `ring_assignment_data`.  Replicas are interchangeable; SHARDS ARE NOT: with
 *    replication_factor = k+m the i-th node of the list stores shard i.  Everything below keeps
 *    that index next to the node.
 *  - The layout optimiser (version.rs:300-640) maximises the partition size subject to: distinct
 *    nodes per partition, every partition in >= zone_redundancy zones, node load <= capacity.  It
 *    works for any replication_factor, so a Garage cluster would keep using it; garage_layout_compute
 *    is a stand-in with the same constraints (max-flow feasibility + binary search on the partition
 *    size) so that the mirror and the tests have rings to work with, plus the two things shards add:
 *    `max_per_zone` (a zone failure loses at most that many shards of any block: <= m keeps every
 *    block decodable) and index stability (a node that stays in a partition keeps its shard index,
 *    so a layout change moves only the shards of nodes that actually changed).
 *    garage_layout_from_ring takes a ring computed elsewhere (the reference's own optimiser).
 *  - Writes go to every node of every active layout version and succeed once a quorum is reached in
 *    EACH version's node set (`try_write_many_sets`, src/rpc/rpc_helper.rs:432-538,
 *    `QuorumSetResultTracker` :664-760).  With shards a node that sits at different indices in two
 *    versions needs two different shards: the write plan is a list of (node, index) requests and the
 *    sets each one counts for.  Quorum: k+1 (`write_quorum`, src/rpc/replication_mode.rs:52-60,
 *    generalised: one more than the k any reader needs).
 *  - Reads: the reference asks nodes one after another for a full copy (src/block/manager.rs:292-334)
 *    in the order of `block_read_nodes_of` (rpc_helper.rs:570-619: active versions interleaved older to
 *    newer by preference rank, ourselves first, then historical versions) with `request_order`
 *    (:621-660: self, same zone, lowest ping).  A shard read is a k-of-(k+m) gather -- exactly
 *    `try_call_many` with quorum k (:290-411) -- so the read plan is that same order over (node, index)
 *    sources, data shards before parity (k data shards need no decode).
 */
#ifndef GARAGE_PLACEMENT_H
#define GARAGE_PLACEMENT_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GARAGE_PARTITION_BITS 8
#define GARAGE_NB_PARTITIONS 256
#define GARAGE_LAYOUT_MAX_NODES 256 /* ring_assignment_data holds compact u8 node indices */

#define GARAGE_LAYOUT_OK 0
#define GARAGE_LAYOUT_E_INVALID -1     /* bad arguments                                              */
#define GARAGE_LAYOUT_E_INFEASIBLE -2  /* no assignment satisfies the constraints                    */
#define GARAGE_LAYOUT_E_NOMEM -3
#define GARAGE_LAYOUT_E_DUPLICATE -4   /* check: a partition lists a node twice                      */
#define GARAGE_LAYOUT_E_GATEWAY -5     /* check: a node without capacity stores data                 */
#define GARAGE_LAYOUT_E_ZONES -6       /* check: a partition spans fewer zones than required         */
#define GARAGE_LAYOUT_E_ZONE_LOAD -7   /* check: a zone holds more shards of a partition than allowed */
#define GARAGE_LAYOUT_E_CAPACITY -8    /* check: a node holds more partitions than its capacity buys */

typedef struct garage_layout garage_layout; /* one layout VERSION */

/* zone[i] = zone id of node i (any integers), capacity[i] = 0 for a gateway node.
 * zone_redundancy: 0 = maximum (min(number of zones with storage nodes, replication_factor)).
 * max_per_zone: 0 = no limit; otherwise no zone gets more than that many shards of a partition.
 * previous: NULL, or the version this one replaces (same node numbering): associations are kept
 * where possible and surviving nodes keep their shard index.                                       */
int garage_layout_compute(garage_layout **out, uint64_t version, int n_nodes, const int32_t *zone,
                          const uint64_t *capacity, int replication_factor, int zone_redundancy,
                          int max_per_zone, const garage_layout *previous);
/* ring = GARAGE_NB_PARTITIONS * replication_factor node indices (ring_assignment_data)            */
int garage_layout_from_ring(garage_layout **out, uint64_t version, int n_nodes, const int32_t *zone,
                            const uint64_t *capacity, int replication_factor, const uint8_t *ring);
void garage_layout_free(garage_layout *l);

int garage_layout_partition_of(const uint8_t hash[32]); /* version.rs:101-104 */
/* out[i] = node that stores shard i of the block `hash`                                            */
int garage_layout_nodes_of(const garage_layout *l, const uint8_t hash[32], int32_t *out);
int garage_layout_ring(const garage_layout *l, uint8_t *out); /* NB_PARTITIONS * rf               */
int garage_layout_replication_factor(const garage_layout *l);
uint64_t garage_layout_version(const garage_layout *l);
uint64_t garage_layout_partition_size(const garage_layout *l); /* 0 for from_ring                  */

typedef struct {
    int32_t min_zones_per_partition;
    int32_t max_shards_per_zone;         /* over all partitions and zones                           */
    int32_t min_partitions_per_node;     /* over storage nodes                                      */
    int32_t max_partitions_per_node;
    int32_t storage_nodes;
    int32_t zones;
} garage_layout_stats;
/* GARAGE_LAYOUT_OK or the first violated constraint (GARAGE_LAYOUT_E_*); stats filled either way   */
int garage_layout_check(const garage_layout *l, int zone_redundancy, int max_per_zone, garage_layout_stats *stats);

/* shards of partition `partition` whose holder changes from `from` to `to`: index[j] moves from
 * node_from[j] to node_to[j].  Returns the count (<= rf).  partition < 0: only count, over all
 * partitions (the data movement of the layout change, in shards).                                  */
int garage_layout_transition(const garage_layout *from, const garage_layout *to, int partition,
                             int32_t *index, int32_t *node_from, int32_t *node_to);

/* ---- quorums ------------------------------------------------------------------------------------ */
#define GARAGE_CONSISTENT 0
#define GARAGE_DEGRADED 1
#define GARAGE_DANGEROUS 2
int garage_ec_write_quorum(int k, int m, int consistency_mode); /* k+1 capped at k+m; dangerous: k  */
int garage_ec_read_quorum(int k, int m, int consistency_mode);  /* k: any k shards decode            */

/* ---- write plan + quorum sets ------------------------------------------------------------------- */
typedef struct {
    int32_t node;
    int32_t index;     /* which shard this node gets                                                */
    uint32_t set_mask; /* bit v: counts towards the quorum of versions[v]                          */
} garage_shard_request;
/* versions: the active layout versions, oldest first (<= 32).  Returns the number of requests.     */
int garage_layout_write_plan(const garage_layout *const *versions, int n_versions, const uint8_t hash[32],
                             garage_shard_request *out, int cap);

typedef struct garage_quorum_tracker garage_quorum_tracker;
#define GARAGE_QUORUM_PENDING 0
#define GARAGE_QUORUM_OK 1      /* a quorum of successes in every set                               */
#define GARAGE_QUORUM_FAILED -1 /* some set can no longer reach its quorum                          */
int garage_quorum_tracker_new(garage_quorum_tracker **out, const garage_shard_request *reqs, int n_reqs,
                              int n_sets, int quorum);
int garage_quorum_tracker_register(garage_quorum_tracker *t, int request, int ok);
int garage_quorum_tracker_state(const garage_quorum_tracker *t);
void garage_quorum_tracker_free(garage_quorum_tracker *t);

/* ---- read plan ---------------------------------------------------------------------------------- */
typedef struct {
    int32_t node;
    int32_t index;
    int32_t version; /* position in `active` (0 = oldest), or n_active + position in `old`          */
} garage_shard_source;
/* active: oldest first; old: historical versions, most recent first; k: data shards come first.
 * our_node: -1 if the caller stores nothing.  ping_us: per node, NULL = unknown (10 s, like the
 * reference).  Zones are those of the newest active version.  The gatherer starts the first k sources
 * with distinct indices and, on each error, the next source whose index is not yet covered.        */
int garage_layout_read_plan(const garage_layout *const *active, int n_active, const garage_layout *const *old,
                            int n_old, const uint8_t hash[32], int k, int our_node, const uint32_t *ping_us,
                            garage_shard_source *out, int cap);

/* ---- drive layout: a node's shards over several data directories (DESIGN.md section 5.7) ---------
 * Garage's multi-drive data_dir: a hash's drive partition has one primary directory (writes go there)
 * and an ordered list of secondary directories (reads look there after the primary).  Directory i is
 * active with capacity[i] > 0, read-only with capacity[i] = 0; at least one is active.  non_empty[i]:
 * the directory holds a garage-marker file or a hex-named subdirectory (NULL = none is).  Errors:
 * GARAGE_LAYOUT_E_INVALID (= GARAGE_EC_E_INVALID) for no active directory, more than
 * GARAGE_DRIVE_MAX_DIRS directories or a prev_index naming a previous directory twice or none. */
#define GARAGE_DRIVE_NPART 1024
#define GARAGE_DRIVE_MAX_DIRS 16
typedef struct garage_drive_layout garage_drive_layout;
/* the big-endian u16 of hash bytes 2 and 3, mod GARAGE_DRIVE_NPART                                 */
int garage_drive_partition_of(const uint8_t hash[32]);
int garage_drive_layout_init(garage_drive_layout **out, int n_dirs, const uint64_t *capacity, const uint8_t *non_empty);
/* prev_index[i]: new directory i's index in prev (the same path), -1 for a directory prev did not list */
int garage_drive_layout_update(garage_drive_layout **out, const garage_drive_layout *prev, const int *prev_index,
                               int n_dirs, const uint64_t *capacity, const uint8_t *non_empty);
/* the same primaries, no secondaries (a finished rebalance)                                         */
int garage_drive_layout_drop_secondaries(garage_drive_layout **out, const garage_drive_layout *l);
int garage_drive_layout_n_dirs(const garage_drive_layout *l);
int garage_drive_layout_primary(const garage_drive_layout *l, int part);
/* partition part's secondaries, in read order, into out (at most cap); returns their number          */
int garage_drive_layout_secondaries(const garage_drive_layout *l, int part, uint8_t *out, int cap);
/* a byte image of the layout (directories' capacities, primaries, secondaries): the bytes needed are
 * returned and written if cap allows.  _deserialize checks an image and rebuilds the layout from it. */
size_t garage_drive_layout_serialize(const garage_drive_layout *l, uint8_t *out, size_t cap);
int garage_drive_layout_deserialize(garage_drive_layout **out, const uint8_t *buf, size_t len);
void garage_drive_layout_free(garage_drive_layout *l);

#ifdef __cplusplus
}
#endif
#endif
