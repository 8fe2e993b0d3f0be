/*
 * garage_block_manager.h -- C view of the C++ host-side mirror of Garage's
 * garage_block::manager::BlockManager for the erasure-coded block path
 * (garage_b200/csrc/block_manager.{h,cpp} -> libgarage_block.so).
 *
 * Garage is Rust and there is no Rust toolchain in this environment, so the host side above
 * the C ABI (include/garage_ec.h) is written in C++ with the reference's names, argument
 * meaning and error behaviour; it talks to the GPU ONLY through garage_ec_* (it is exactly the
 * code a Rust maintainer would write in src/block, see INTEGRATION.md).  A "cluster" is
 * n_nodes in-process node stores (the reference tests multi-node the same way: several
 * instances on localhost in one process, src/net/test.rs:15-60, script/test-smoke.sh).
 *
 * Mirrored reference surface (SURVEY.md section 8 a1-a8, f1-f3):
 *   rpc_put_block           src/block/manager.rs:366-408   (encode, shard i -> node who[i])
 *   rpc_get_block           src/block/manager.rs:344-363, 276-339 (any k of k+m, reconstruct)
 *   resync_block (fetch)    src/block/resync.rs:460-500    (rebuild this node's shard)
 *   read_block / verify     src/block/manager.rs:554-609, src/block/block.rs:69-83
 *                           (per-shard blake2sum; corrupt -> quarantine + resync queue)
 *   ScrubWorker             src/block/repair.rs:438-490    (sweep of one node's shards)
 *   write_block             src/block/manager.rs:517-530, 720-805 (local durable store)
 *   block_incref/decref     src/block/manager.rs:452-500, get_block_rc :421-449 (src/block/rc.rs)
 *   ResyncWorker / backoff  src/block/resync.rs:119-134, 241-336, 605-655 (scheduled queue, ErrorCounter,
 *                           clear_backoff), list_resync_errors manager.rs:429-449
 *   batching front-end      (row f1) concurrent PUT / resync calls coalesced into GPU batches,
 *                           back-pressure like buffer_kb_semaphore (manager.rs:156,380-385)
 */
#ifndef GARAGE_BLOCK_MANAGER_H
#define GARAGE_BLOCK_MANAGER_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* errors: mirror garage_util::error::Error variants on this path (src/util/error.rs:14-82) */
#define GARAGE_BM_OK 0
#define GARAGE_BM_E_CORRUPT_DATA (-10)  /* Error::CorruptData(hash)  */
#define GARAGE_BM_E_MISSING_BLOCK (-11) /* Error::MissingBlock(hash) */
#define GARAGE_BM_E_MESSAGE (-12)       /* Error::Message(..)        */
#define GARAGE_BM_E_QUORUM (-13)        /* Error::Quorum(..) from try_write_many_sets */
/* GARAGE_EC_E_* codes (-1..-6) pass through unchanged */

typedef struct garage_bm garage_bm;

/* a code the store may still hold shards of: RS(k, m), LRC(k, local_groups, m - local_groups), PB(k, m) or Clay(k, m) */
typedef struct {
    int k, m;
    int local_groups; /* 0: not LRC */
    int piggyback;    /* 0 or 1 */
    int clay;         /* 0 or 1: Clay(k, m), garage_ec_create_clay's rules; not with local_groups or piggyback */
} garage_bm_code;

#define GARAGE_BM_MAX_PREVIOUS_CODES 4

/* One layout version over the manager's n_nodes node stores (DESIGN.md section 5.2).  The fields mean what they mean
 * to garage_layout_compute: zone[i] = zone of node i, capacity[i] = 0 for a node that stores nothing in this version
 * (a gateway, or a node being removed), zone_redundancy 0 = maximum, max_per_zone 0 = no limit (at most m).       */
typedef struct {
    const int32_t *zone;      /* n_nodes entries */
    const uint64_t *capacity; /* n_nodes entries */
    int zone_redundancy;
    int max_per_zone;
} garage_bm_layout_spec;

#define GARAGE_BM_MAX_LAYOUT_VERSIONS 4 /* active layout versions at once */

/* One data directory of a node (Garage's data_dir = [{path, capacity}, {path, read_only}]; DESIGN.md section 5.7).
 * path is relative to the node directory <data_dir>/node<N>; "." is the node directory itself.                      */
typedef struct {
    const char *path;
    uint64_t capacity; /* > 0 unless read_only: the share of the node's partitions the drive is the primary of */
    int read_only;     /* 1: read and rebalanced off, never written                                            */
} garage_bm_data_dir;

#define GARAGE_BM_MAX_DATA_DIRS 16

typedef struct {
    int data_shards;                /* k  (config: erasure_coding.data_shards)   */
    int parity_shards;              /* m                                          */
    int cuda_device;
    int n_nodes;                    /* >= k+m storage nodes in the simulated cluster */
    uint32_t block_size;            /* util/config.rs:273-275, default 1 MiB          */
    uint64_t block_ram_buffer_max;  /* util/config.rs:276-278, default 256 MiB        */
    uint32_t batch_max_blocks;      /* f1: max blocks per GPU batch                   */
    uint32_t batch_linger_us;       /* f1: how long the first block of a batch waits  */
    const char *data_dir;           /* NULL/"": shards in memory; else <data_dir>/node<N>/<hh>/<hh>/<hash>.shard
                                       (64-byte header {GEC1,k,m,index,sum_kind,block_len,shard_len,tag,header check}
                                       + bytes; tmp-file -> rename, *.corrupted quarantine: manager.rs:720-819)  */
    int shard_sum_kind;             /* GARAGE_EC_SUM_ADLER8 (default) or GARAGE_EC_SUM_BLAKE2: the per-shard tag  */
    int verify_content_hash;        /* 1 (default): rpc_get_block checks blake2sum(block) == hash like
                                       DataBlock::verify (block.rs:69-83) and hunts the bad shard on mismatch     */
    int data_fsync;                 /* util/config.rs data_fsync: fsync file + directory before/after the rename  */
    uint32_t block_gc_delay_ms;     /* BLOCK_GC_DELAY (manager.rs:49-52, 10 min): a shard whose block dropped to
                                       rc 0 is deleted by resync only after this delay                            */
    int local_groups;               /* 0 (default): RS(k, m).  l > 0: LRC(k, l, m - l) (garage_ec_create_lrc): one
                                       lost shard is resynced from the k/l other shards of its group.  Recorded in
                                       every shard file header and wire message; a shard of another code is
                                       quarantined like a k / m mismatch                                          */
    int piggyback;                  /* 0 (default).  1: piggybacked RS PB(k, m) (garage_ec_create_piggyback, needs
                                       2 <= m <= 4, k <= 16): resync and a degraded GET fetch only the planned
                                       halves (ranged reads, each checked against its adler8 segment tags), k + |G_i|
                                       halves for one lost data shard.  GARAGE_EC_E_INVALID with local_groups > 0 or
                                       shard_sum_kind = GARAGE_EC_SUM_BLAKE2.  Recorded in the shard file header; a
                                       shard of another code is quarantined                                       */
    /* Changing a store's code (file store; DESIGN.md section 5.1).  Default: none, and a shard of any code but the
       configured one is quarantined.  GARAGE_EC_E_INVALID before any CUDA call for: more than
       GARAGE_BM_MAX_PREVIOUS_CODES entries, a NULL list with entries, an entry equal to the configured code or to
       another entry (k, m, local_groups, piggyback and clay all equal: Clay(6,3) may precede Clay(10,4), and RS(10,4)
       may), an entry garage_ec_create* would reject or with more than n_nodes shards, a PB entry with
       GARAGE_EC_SUM_BLAKE2 tags, legacy_replicas < 0 or > n_nodes.                                               */
    const garage_bm_code *previous_codes; /* codes whose shards are read and converted (old .shard / .legacy files) */
    int n_previous_codes;
    int legacy_replicas;            /* replication factor of a previous replicated layout (0 = none): whole-block
                                       files <node dir>/<hh>/<hh>/<64 hex> on the first legacy_replicas nodes of the
                                       block's ring row, read and converted like a previous code                   */
    /* Cluster layout (DESIGN.md section 5.2).  NULL: partition p on nodes (p mod n_nodes) + i, as before.  Otherwise
       version 1 is garage_layout_compute(1, ..., previous = NULL) of this spec.  GARAGE_EC_E_INVALID before any CUDA
       call for: a NULL array, a negative zone_redundancy or max_per_zone, max_per_zone > m, fewer than k+m nodes with
       capacity, or a layout garage_layout_compute finds infeasible.  A file store keeps its layout history in
       <data_dir>/layout; on restart that file wins over this field.                                              */
    const garage_bm_layout_spec *layout;
    int clay;                       /* 0 (default).  1: Clay(k, m) (garage_ec_create_clay: 2 <= m <= 4, k >= 2,
                                       alpha <= 256).  Resync of one lost shard hands the rebuild only the
                                       garage_ec_read_ranges runs of every other shard (1/m of each; holders check
                                       their whole shard's tag first, a bad one is quarantined and the rebuild falls
                                       back to k whole shards).  Recorded in the shard file header (pad[1] = 2); a
                                       shard of another code is quarantined.  GARAGE_EC_E_INVALID with
                                       local_groups > 0 or piggyback, and, unless clay_layout is set, with `layout`
                                       set or a layout file on disk; garage_bm_apply_layout then refuses the store
                                       too.  Conversion to and from Clay works through previous_codes             */
    int clay_layout;                /* 0 (default): a Clay store keeps the fixed ring, as above.  1: a Clay store
                                       takes `layout`, a layout file and garage_bm_apply_layout like any other code
                                       (DESIGN.md section 5.3): a shard no active version has a copy of is rebuilt
                                       from the garage_ec_read_ranges runs of the others, each one read whole from
                                       the first version that has it.  GARAGE_EC_E_INVALID without clay, or for any
                                       other value                                                                */
} garage_bm_config;

typedef struct {
    uint64_t bytes_written, bytes_read;      /* block.bytes_written / bytes_read  (metrics.rs) */
    uint64_t corruption_counter;             /* block.corruption_counter                        */
    uint64_t resync_counter, resync_error_counter, resync_recv_counter;
    uint64_t delete_counter;
    uint64_t put_calls, put_batches;         /* f1: how well PUTs were coalesced                */
    uint64_t reconstruct_calls, reconstruct_batches;
    uint64_t scrub_shards_checked, scrub_corruptions;
    uint64_t resync_queue_length;            /* block.resync_queue_length (all nodes)            */
    uint64_t encode_call_us, reconstruct_call_us; /* wall time spent inside garage_ec_* batch calls */
    uint64_t corrupt_data_errors;            /* GETs whose reassembled block failed the content hash */
    uint64_t write_errors;                   /* shard writes that failed (ENOSPC, EACCES, ...)      */
    uint64_t resync_shards_read;             /* shards read by resync_block's fetch branch (the read
                                                set of garage_ec_read_set: k for RS, k/l for an LRC
                                                local repair)                                       */
    uint64_t resync_bytes_read;              /* bytes read by that fetch branch (PB reads half shards) */
    uint64_t convert_blocks;                 /* blocks rewritten under the configured code (>= k+1 shards stored) */
    uint64_t convert_bytes_read;             /* legacy shard / replica bytes read by conversions               */
    uint64_t convert_bytes_written;          /* configured-code shard bytes durably written by conversions      */
    uint64_t convert_errors;                 /* conversions that failed (unrecoverable source, no write quorum) */
    uint64_t convert_call_us;                /* wall time inside garage_ec_transcode                            */
    uint64_t legacy_gets;                    /* GETs served from a previous code's stripe or a replica          */
    uint64_t legacy_deleted;                 /* legacy shard / replica files deleted                            */
    uint64_t layout_shards_copied;           /* shards a layout sync copied from an older version's holder      */
    uint64_t layout_shards_rebuilt;          /* shards a layout sync (or resync) rebuilt on the GPU             */
    uint64_t layout_bytes_read;              /* bytes read by those copies and rebuilds                         */
    uint64_t layout_bytes_written;           /* bytes they wrote                                                */
    uint64_t layout_deleted;                 /* shards deleted once the newest version no longer assigned them  */
    uint64_t layout_sync_errors;             /* shards a sync could neither copy nor rebuild (or not write)     */
    uint64_t layout_version;                 /* the newest active layout version                                */
    uint64_t resync_bytes_fetched;           /* bytes resync_block's fetch branch handed to the rebuild: what would
                                                cross the network in Garage.  Clay: the repair runs (1/m of each
                                                helper); RS, LRC and PB: resync_bytes_read                          */
    uint64_t deep_scrub_blocks;              /* blocks garage_bm_deep_scrub_step checked (content hash + parity) */
    uint64_t deep_scrub_skipped;             /* blocks it skipped because a shard was missing or bad            */
    uint64_t deep_scrub_parity_bad;          /* stale parity shards it quarantined                               */
    uint64_t deep_scrub_content_errors;      /* blocks whose content hash failed and whose hunt found no culprit */
    uint64_t deep_check_call_us;             /* wall time inside garage_ec_deep_check                            */
    uint64_t layout_bytes_fetched;           /* bytes handed to layout copies and rebuilds: what would cross the network
                                                in Garage.  A Clay repair counts its runs (1/m of each helper);
                                                everything else equals layout_bytes_read                            */
} garage_bm_metrics;
/* Counters of garage_bm_rpc_get_block_range, in a struct of their own so that garage_bm_metrics keeps the layout older
 * callers were built against. */
typedef struct garage_bm_range_metrics {
    uint64_t range_gets;          /* garage_bm_rpc_get_block_range calls                                   */
    uint64_t range_degraded;      /* ranged GETs whose range needed an absent data shard (went to the GPU)  */
    uint64_t range_bytes_read;    /* tag-span bytes those GETs read from shard files                      */
    uint64_t range_bytes_fetched; /* the planned run bytes: what would cross the network in Garage         */
} garage_bm_range_metrics;
/* Counters of garage_bm_stripe_repair_step, in a struct of their own for the same reason. */
typedef struct garage_bm_stripe_repair_metrics {
    uint64_t stripe_repairs;              /* stripes with at least one shard written                            */
    uint64_t stripe_repair_shards;        /* shards written                                                     */
    uint64_t stripe_repair_bytes_read;    /* bytes the holders read from their shard files                      */
    uint64_t stripe_repair_bytes_fetched; /* bytes handed to the rebuild: what would cross the network in Garage.
                                             Clay: the repair runs (1/m of each helper for one absent shard)    */
    uint64_t stripe_repair_bytes_written; /* bytes of the shards written                                        */
    uint64_t stripe_repair_errors;        /* unrecoverable stripes + shard writes that failed                   */
    uint64_t stripe_repair_call_us;       /* wall time inside garage_ec_reconstruct_stripes                     */
} garage_bm_stripe_repair_metrics;
/* Counters of salvage (DESIGN.md section 5.14): a GET, resync or stripe repair whose survivors could not rebuild the
 * configured stripe of an adler8 store (RS, LRC or PB) rebuilds it segment by segment from the live shards and their
 * quarantined copies (garage_ec_reconstruct_segments), proven by the block's content hash.  A struct of its own for
 * the same reason. */
typedef struct garage_bm_salvage_metrics {
    uint64_t salvage_attempts;             /* stripes salvage was tried on                                        */
    uint64_t salvage_blocks;               /* stripes salvaged: rebuilt and proven by the content hash            */
    uint64_t salvage_failures;             /* tries that ended in an unrecoverable unit or a content-hash mismatch */
    uint64_t salvage_units_rebuilt;        /* (shard, unit) pieces rebuilt: a segment, for PB a pair of segments  */
    uint64_t salvage_quarantined_segments; /* segments taken from quarantined copies                              */
    uint64_t salvage_bytes_read;           /* shard bytes read, live and quarantined copies                        */
    uint64_t salvage_call_us;              /* wall time inside garage_ec_reconstruct_segments_stripes              */
} garage_bm_salvage_metrics;
/* Counters of repair by segment (DESIGN.md section 5.15): a resync of a shard its node quarantined because its adler8
 * tag failed keeps the copy's units that pass their segment tags and rebuilds only the others, from the same columns
 * of the survivors (garage_ec_segment_read_ranges, garage_ec_reconstruct_segments_stripes).  RS, LRC and PB stores
 * with adler8 tags and one active layout version.  These bytes are counted in resync_bytes_read and
 * resync_bytes_fetched too.  A struct of its own for the same reason. */
typedef struct garage_bm_segment_repair_metrics {
    uint64_t repairs;       /* shards written by the partial path                                           */
    uint64_t units_rebuilt; /* (shard, unit) pieces rebuilt: a segment, for PB a pair of segments           */
    uint64_t bytes_read;    /* quarantined-copy + survivor span bytes read                                  */
    uint64_t bytes_fetched; /* survivor run bytes: what would cross the network in Garage                   */
    uint64_t fallbacks;     /* partial tries (the node held a quarantined copy) that ended in the whole-shard path */
    uint64_t call_us;       /* wall time inside garage_ec_reconstruct_segments_stripes                      */
} garage_bm_segment_repair_metrics;
/* Counters of the drives (DESIGN.md section 5.7), in a struct of their own for the same reason. */
typedef struct garage_bm_drive_metrics {
    uint64_t rebalance_files_moved; /* files garage_bm_rebalance_step wrote to their primary drive (old copy removed) */
    uint64_t rebalance_bytes_moved; /* their bytes, file headers included                                            */
    uint64_t rebalance_errors;      /* moves whose write or removal failed (the file stays readable where it was)   */
    uint64_t drive_marker_errors;   /* marker checks that failed (at create or garage_bm_set_data_dirs)             */
} garage_bm_drive_metrics;

/* Counters of the scheduled resync (DESIGN.md section 5.8), in a struct of their own for the same reason. */
typedef struct garage_bm_resync_metrics {
    uint64_t resync_error_entries;     /* (node, hash) entries of the error table, all nodes                        */
    uint64_t resync_deferred;          /* entries garage_bm_resync_step queued again without a try: backoff, GC delay */
    uint64_t resync_steps;             /* garage_bm_resync_step calls that ran                                      */
    uint64_t resync_retry_nows;        /* entries garage_bm_resync_retry_now made due                               */
    uint64_t resync_failed_bytes_read; /* bytes read by resyncs that failed (part of resync_bytes_read)             */
} garage_bm_resync_metrics;

/* Counters of the SSE-C calls (DESIGN.md section 5.9), in a struct of their own for the same reason. */
typedef struct garage_bm_sealed_metrics {
    uint64_t sealed_puts;          /* garage_bm_rpc_put_block_sealed calls that sealed their block               */
    uint64_t sealed_batches;       /* garage_ec_seal_blocks calls of the encode dispatchers                      */
    uint64_t opened_gets;          /* garage_bm_rpc_get_block_opened calls that returned a plaintext             */
    uint64_t opened_auth_failures; /* opened GETs that ended in GARAGE_EC_E_AUTH                                 */
    uint64_t opened_fallbacks;     /* opened GETs that went through rpc_get_block (stale shard, previous code,
                                      replica or missing stripe) before the block was opened                   */
    uint64_t seal_call_us;         /* wall time inside garage_ec_seal_blocks                                    */
    uint64_t open_call_us;         /* wall time inside garage_ec_open_stripes                                   */
} garage_bm_sealed_metrics;
/* Counters of garage_bm_rpc_get_block_range_opened (DESIGN.md section 5.10), in a struct of their own for the same
 * reason. */
typedef struct garage_bm_sealed_range_metrics {
    uint64_t gets;               /* garage_bm_rpc_get_block_range_opened calls                                      */
    uint64_t degraded_gets;      /* of those, ranges whose prefix or span needed an absent data shard rebuilt       */
    uint64_t bytes_read;         /* tag-span bytes those GETs read from shard files                                */
    uint64_t bytes_fetched;      /* the planned run bytes: what would cross the network in Garage                  */
    uint64_t auth_failures;      /* calls that ended in GARAGE_EC_E_AUTH                                            */
    uint64_t fallbacks;          /* ranges that failed a tag and went through one whole-block opened GET            */
    uint64_t call_us;            /* wall time inside garage_bm_rpc_get_block_range_opened                           */
    uint64_t open_range_call_us; /* wall time inside garage_ec_open_range_stripes                                   */
} garage_bm_sealed_range_metrics;
/* Counters of garage_bm_rpc_put_block_resealed (DESIGN.md section 5.11), in a struct of their own for the same
 * reason. */
typedef struct garage_bm_reseal_metrics {
    uint64_t calls;            /* garage_bm_rpc_put_block_resealed calls                                            */
    uint64_t batches;          /* garage_ec_reseal_stripes calls of the reconstruct dispatchers                    */
    uint64_t sources_gathered; /* source blocks gathered from their stripes                                        */
    uint64_t bytes_read;       /* shard bytes those gathers and the fallbacks read                                 */
    uint64_t auth_failures;    /* calls that ended in GARAGE_EC_E_AUTH                                              */
    uint64_t fallbacks;        /* sources read through garage_bm_rpc_get_block (stale shard, previous code, replica) */
    uint64_t call_us;          /* wall time inside garage_bm_rpc_put_block_resealed                                 */
    uint64_t reseal_call_us;   /* wall time inside garage_ec_reseal_stripes                                         */
} garage_bm_reseal_metrics;

/* One entry of a node's resync error table (Garage's BlockResyncErrorInfo, manager.rs:429-449).                    */
typedef struct garage_bm_resync_error {
    int32_t node;
    uint8_t hash[32];
    long long rc;          /* garage_bm_get_block_rc                                                            */
    uint64_t errors;       /* failed tries since the last success                                               */
    uint64_t last_try_ms;  /* time of the last failed try (or as set by retry-now)                              */
    uint64_t next_try_ms;  /* last_try_ms + 60 000 << min(errors - 1, 6): 1 minute up to 64 minutes             */
    int32_t last_status;   /* what the last failed try returned (GARAGE_BM_E_* / GARAGE_EC_E_*)                 */
} garage_bm_resync_error;

/* The state of one index of a block's stripe in garage_bm_block_info */
#define GARAGE_BM_SHARD_VALID 0       /* header checks out (and, with check_tags, the shard tag)                     */
#define GARAGE_BM_SHARD_ABSENT 1      /* no file of this index                                                        */
#define GARAGE_BM_SHARD_DOWN 2        /* the holder is down                                                           */
#define GARAGE_BM_SHARD_BAD_HEADER 3  /* damaged header, or one naming another code, index or block length           */
#define GARAGE_BM_SHARD_BAD_TAG 4     /* header fine, bytes fail the tag (only with check_tags)                       */
#define GARAGE_BM_SHARD_QUARANTINED 5 /* no shard, a quarantined .corrupted file                                      */
#define GARAGE_BM_SHARD_PREVIOUS 6    /* no shard of the configured code, a previous code's shard or a replica        */
#define GARAGE_BM_MAX_SHARDS 40       /* GARAGE_EC_MAX_K + GARAGE_EC_MAX_M                                            */

typedef struct garage_bm_block_status {
    long long rc;                                /* garage_bm_get_block_rc                                            */
    garage_bm_code code;                         /* the configured code                                               */
    uint32_t block_len;                          /* from a valid shard's header; 0 if there is none                   */
    int32_t n_shards;                            /* k + m: the entries below that are set                             */
    int32_t node[GARAGE_BM_MAX_SHARDS];          /* holder of index i in the newest layout version                    */
    int32_t state[GARAGE_BM_MAX_SHARDS];         /* GARAGE_BM_SHARD_*                                                 */
    uint64_t resync_errors[GARAGE_BM_MAX_SHARDS];/* that holder's resync error count for the block                    */
    int32_t recoverable;                         /* every index that is not valid can be rebuilt from the valid ones  */
    uint8_t read_set[GARAGE_BM_MAX_SHARDS];      /* recoverable with some index not valid: the indices that rebuild
                                                    reads (garage_ec_read_set); all 0 otherwise                        */
} garage_bm_block_status;

void garage_bm_default_config(garage_bm_config *cfg);
int garage_bm_create(garage_bm **out, const garage_bm_config *cfg);
/* garage_bm_create with several drives per node (file store; DESIGN.md section 5.7); garage_bm_config keeps the size
 * older callers allocate, so the drive list comes here.  data_dirs NULL / n_data_dirs 0: garage_bm_create exactly,
 * every file under the node directory.  Otherwise each node spreads its files over these directories by the drive
 * layout (include/garage_placement.h), recorded in <data_dir>/node<N>/data_layout with a garage-marker file in every
 * drive; on restart that file wins over this list, which only seeds nodes without one.  A node whose recorded marker
 * is missing or different starts down.  GARAGE_EC_E_INVALID before any CUDA call for: drives on the memory store, a
 * NULL list with entries, a negative count, more than GARAGE_BM_MAX_DATA_DIRS entries, a NULL, empty, absolute or
 * repeated path or one outside the node directory, capacity 0 without read_only, or no drive with capacity.        */
int garage_bm_create_with_drives(garage_bm **out, const garage_bm_config *cfg, const garage_bm_data_dir *data_dirs,
                                 int n_data_dirs);
/* garage_bm_create_with_drives on several GPUs of the host (DESIGN.md section 5.13); cfg->cuda_device is not read.  One
 * dispatcher group per listed device: its encode and reconstruct dispatchers, a context per code for the sweeps, and
 * its pinned slot pools on the device's NUMA node.  Every call that reaches the GPU is routed to one group by the
 * calling thread's NUMA node: among the groups whose GPU is on that node (all groups if none is) the one with the
 * fewest calls in flight, ties round robin.  A batch never spans groups.  The same device may be listed more than
 * once (two groups on one GPU).  data_dirs NULL / n_data_dirs 0: every file under the node directory, as
 * garage_bm_create.  GARAGE_EC_E_INVALID before any context is created or thread started for a NULL list, n_devices
 * outside 1..GARAGE_BM_MAX_DEVICES, a negative device, one at or past garage_ec_device_count, or anything
 * garage_bm_create_with_drives refuses; GARAGE_EC_E_NODEVICE on a host with no device.  A group that cannot be built
 * fails the whole call, and what was built is torn down.  garage_bm_create(_with_drives) are this call on
 * {cfg->cuda_device}.                                                                                            */
#define GARAGE_BM_MAX_DEVICES 16
int garage_bm_create_on_devices(garage_bm **out, const garage_bm_config *cfg, const garage_bm_data_dir *data_dirs,
                                int n_data_dirs, const int *cuda_devices, int n_devices);
void garage_bm_destroy(garage_bm *bm);

/* One dispatcher group (garage_bm_create_on_devices), in list order. */
typedef struct {
    int cuda_device;
    int numa_node;          /* the GPU's NUMA node (garage_ec_numa_info), -1 = unknown                             */
    uint64_t batches;       /* GPU calls of the group: dispatcher batches and the sweeps' own calls                */
    uint64_t blocks;        /* blocks (or shards, for the scrub) those calls carried                               */
    uint64_t bytes;         /* their stored bytes                                                                  */
    uint64_t routed_local;  /* calls routed here from a thread on the GPU's node                                   */
    uint64_t routed_remote; /* calls routed here from any other node (no group on the caller's node)               */
    int pool_numa_node;     /* the node the group's pinned pools landed on (garage_ec_numa_info), -1 = unknown     */
} garage_bm_device_metrics;
/* *n = the number of groups; at most cap entries are written to out.  GARAGE_EC_E_INVALID for NULL bm or n, cap < 0,
 * or out NULL with cap > 0.                                                                                      */
int garage_bm_get_device_metrics(garage_bm *bm, garage_bm_device_metrics *out, int cap, int *n);

/* util/data.rs:130-138 */
void garage_bm_blake2sum(const uint8_t *data, size_t len, uint8_t hash_out[32]);

/* manager.rs:366-408.  hash = blake2sum(data) (put.rs:448).  Thread-safe; concurrent calls are
 * batched.  Returns GARAGE_BM_E_QUORUM if fewer than k+1 (or k+m if smaller) shards were stored. */
int garage_bm_rpc_put_block(garage_bm *bm, const uint8_t hash[32], const uint8_t *data, size_t len);

/* manager.rs:344-363: the block's bytes (whole buffer instead of a ByteStream).
 * GARAGE_BM_E_MISSING_BLOCK if fewer than k valid shards can be gathered.                       */
int garage_bm_rpc_get_block(garage_bm *bm, const uint8_t hash[32], uint8_t *out, size_t cap,
                            size_t *out_len);
/* SSE-C PUT (src/api/s3/put.rs:441-466, DESIGN.md sections 2.6 and 5.9): the plaintext (len <= block_size) is sealed
 * with AES-256-GCM STREAM chunks under key32 and a fresh 8-byte nonce prefix from getrandom(2) -- key32 NULL: stored
 * as plaintext (len >= 1) -- by the encode batcher, then stored exactly as garage_bm_rpc_put_block stores a block of
 * sealed_len bytes.  hash_out = the block's content address, blake2sum of the sealed block.  No key is kept or logged. */
int garage_bm_rpc_put_block_sealed(garage_bm *bm, const uint8_t *key32, const uint8_t *data, size_t len,
                                   uint8_t hash_out[32]);
/* SSE-C GET (EncryptionParams::get_block, src/api/s3/encryption.rs:269-279): the plaintext of block `hash` sealed
 * under key32.  Gathered like garage_bm_rpc_get_block; the rebuild, the content-hash check and the decryption are one
 * garage_ec_open_stripes call of the reconstruct dispatchers.  A block that does not hash to its address, or that only
 * a previous code or a replica holds, is read by garage_bm_rpc_get_block (stale-shard hunt included) and then opened.
 * GARAGE_EC_E_AUTH if a tag or the framing fails (wrong key, tampered block); GARAGE_BM_E_MISSING_BLOCK as
 * garage_bm_rpc_get_block; GARAGE_EC_E_INVALID if the plaintext exceeds cap.                                        */
int garage_bm_rpc_get_block_opened(garage_bm *bm, const uint8_t hash[32], const uint8_t *key32, uint8_t *out, size_t cap,
                                   size_t *out_len);
void garage_bm_get_sealed_metrics(garage_bm *bm, garage_bm_sealed_metrics *out);

/* Ranged SSE-C GET (body_from_blocks_range, src/api/s3/get.rs:650-743, and UploadPartCopy with a source range,
 * src/api/s3/copy.rs:396-469, of an SSE-C object): plaintext bytes [offset, offset + len) of block `hash` sealed under
 * key32.  Gathered like garage_bm_rpc_get_block_range, with the runs of garage_ec_open_range_plan (the nonce prefix and
 * the touched chunks); one garage_ec_open_range_stripes call of the reconstruct dispatchers rebuilds, checks and
 * decrypts them.  *out_len = len.  The whole plaintext, and blocks held only under a previous code or as replicas, are
 * served by garage_bm_rpc_get_block_opened and sliced.  A touched chunk that fails its tag is retried once as a
 * whole-block garage_bm_rpc_get_block_opened, whose content-hash check finds and quarantines a stale shard: its bytes
 * are served if it succeeds, GARAGE_EC_E_AUTH is returned if it fails authentication (a wrong key).  Integrity: as
 * DESIGN.md section 2.7 -- the touched chunks are proven, untouched chunks and the content hash are not.
 * GARAGE_EC_E_INVALID if offset + len exceeds the plaintext or len > cap; GARAGE_BM_E_MISSING_BLOCK as
 * garage_bm_rpc_get_block.                                                                                         */
int garage_bm_rpc_get_block_range_opened(garage_bm *bm, const uint8_t hash[32], const uint8_t *key32, uint32_t offset,
                                         uint32_t len, uint8_t *out, size_t cap, size_t *out_len);
void garage_bm_get_sealed_range_metrics(garage_bm *bm, garage_bm_sealed_range_metrics *out);

/* Copy with re-encryption into an SSE-C block (handle_copy_reencrypt, src/api/s3/copy.rs:320-349, through save_stream's
 * block loop; UploadPartCopy, copy.rs:506-636, one call per Defragmenter output; DESIGN.md sections 2.8 and 5.11): the
 * destination block is the plaintext pieces[0..n_pieces) -- bytes [offset, offset + len) of the plaintext of stored
 * block `hash` -- concatenated and sealed under dst_key32 and a fresh nonce prefix from getrandom(2).  src_key32: the
 * key every source is sealed under, or NULL: the sources are plaintext blocks.  Each distinct source is gathered once,
 * as garage_bm_rpc_get_block_opened gathers it, and proven whole (content hash, every chunk tag); a batch of copies
 * is one garage_ec_reseal_stripes call of the reconstruct dispatchers.  No plaintext is in host memory on any path.  A
 * source that does not hash to its address or that only a previous code or a replica holds is read by
 * garage_bm_rpc_get_block (stale-shard hunt included) and the copy is retried once.  The result is stored exactly as
 * garage_bm_rpc_put_block stores a block of its sealed length; refcounts are not touched.  hash_out = its content
 * address, *stored_len_out (nullable) = its sealed length.  GARAGE_EC_E_INVALID for NULL dst_key32, n_pieces outside
 * 1..GARAGE_BM_MAX_PIECES, an empty piece, a total length over block_size or a piece past its source's plaintext;
 * GARAGE_EC_E_AUTH if a source fails a tag or its framing (nothing is stored); GARAGE_BM_E_MISSING_BLOCK as
 * garage_bm_rpc_get_block.                                                                                         */
#define GARAGE_BM_MAX_PIECES 64
typedef struct garage_bm_piece {
    uint8_t hash[32];
    uint32_t offset, len;
} garage_bm_piece;
int garage_bm_rpc_put_block_resealed(garage_bm *bm, const garage_bm_piece *pieces, int n_pieces, const uint8_t *src_key32,
                                     const uint8_t *dst_key32, uint8_t hash_out[32], uint32_t *stored_len_out);
/* The two SSE-C writes with the S3 checksum of the block's plaintext (DESIGN.md sections 2.9 and 5.12): crc_kind
 * GARAGE_EC_CRC_NONE / _CRC32 / _CRC32C, *crc_out = the CRC32 or CRC32C of the plaintext (0 for NONE), computed by the
 * same GPU call that seals the block -- for a copy that falls back to garage_bm_rpc_get_block, by the retry's -- so the
 * plaintext still never reaches host memory.  The caller folds the blocks' values into the object's checksum with
 * garage_ec_crc_combine.  Otherwise exactly garage_bm_rpc_put_block_sealed / _resealed; GARAGE_EC_E_INVALID also for
 * an unknown kind or a NULL crc_out.                                                                               */
int garage_bm_rpc_put_block_sealed_crc(garage_bm *bm, const uint8_t *key32, const uint8_t *data, size_t len,
                                       uint8_t crc_kind, uint8_t hash_out[32], uint32_t *crc_out);
int garage_bm_rpc_put_block_resealed_crc(garage_bm *bm, const garage_bm_piece *pieces, int n_pieces,
                                         const uint8_t *src_key32, const uint8_t *dst_key32, uint8_t crc_kind,
                                         uint8_t hash_out[32], uint32_t *stored_len_out, uint32_t *crc_out);
void garage_bm_get_reseal_metrics(garage_bm *bm, garage_bm_reseal_metrics *out);

/* Bytes [offset, offset + len) of a block (body_from_blocks_range, src/api/s3/get.rs:650-743; the source range of
 * UploadPartCopy, src/api/s3/copy.rs:396-469), reading only the shards and columns garage_ec_range_plan names, each as
 * the adler8 tag span that covers its runs (BLAKE2 stores: whole shards).  *out_len = len.  A range whose touched data
 * shards are all present never reaches the GPU; the others are rebuilt by the reconstruct dispatchers.
 * Integrity: a ranged read is proven by the shard tags only -- the block's blake2sum needs the whole block -- so a
 * stale shard that is consistent with its own tag is found by the deep scrub (garage_bm_deep_scrub_step), not here.
 * The whole block (offset 0, len = block length), and blocks held only under a previous code or as replicas, are
 * served by garage_bm_rpc_get_block (content hash checked) and sliced.  GARAGE_EC_E_INVALID if offset + len exceeds
 * the block or len > cap; GARAGE_BM_E_MISSING_BLOCK as garage_bm_rpc_get_block.                               */
int garage_bm_rpc_get_block_range(garage_bm *bm, const uint8_t hash[32], uint32_t offset, uint32_t len, uint8_t *out,
                                  size_t cap, size_t *out_len);

/* manager.rs:452-500 block_incref / block_decref (called by BlockRefTable::updated,
 * src/model/s3/block_ref_table.rs:69-85): 0 -> 1 and 1 -> 0 transitions queue a resync on every
 * storage node of the block; get_block_rc (manager.rs:421-449) returns -1 for a block that was
 * never counted (treated as referenced).                                                        */
int garage_bm_block_incref(garage_bm *bm, const uint8_t hash[32]);
int garage_bm_block_decref(garage_bm *bm, const uint8_t hash[32]);
long long garage_bm_get_block_rc(garage_bm *bm, const uint8_t hash[32]);

/* resync.rs:354-503 for storage node `node`: fetch branch (rc > 0, shard absent: rebuild it from the
 * survivors garage_ec_read_set names -- k for RS, the shard's local group for LRC) and the deletion half of the offload branch (rc == 0, shard present: delete it).   */
int garage_bm_resync_block(garage_bm *bm, int node, const uint8_t hash[32]);
/* drain node's resync queue with `workers` concurrent workers (resync.rs:43: up to 8);
 * returns the number of blocks that could not be resynced (they stay queued, with backoff
 * semantics left to the caller; garage_bm_resync_step below applies Garage's).                  */
int garage_bm_resync_all(garage_bm *bm, int node, int workers, uint64_t *resynced);
/* RepairWorker (repair.rs:35-155): enqueue every hash this node should hold but does not.        */
int garage_bm_repair_enqueue_missing(garage_bm *bm, int node, uint64_t *enqueued);

/* Scheduled resync (DESIGN.md section 5.8).  Each node's resync queue holds one entry per hash with the time it falls
 * due; everything queued by the calls above is due at once, and garage_bm_resync_all still drains the whole queue
 * (its successes also clear their error entries).  Times are ms since the epoch, or garage_bm_debug_set_clock_ms's.
 *
 * garage_bm_resync_step is one pass of Garage's ResyncWorker (resync.rs:258-336) over node's queue: the entries due
 * now, in (due time, hash) order, at most max_blocks of them (0 = all), run by `workers` threads (1..8):
 *   - an entry whose error entry's next_try_ms is later than now is queued again at next_try_ms, read nothing
 *     (*deferred);
 *   - a block still inside block_gc_delay_ms is queued again at the time it becomes deletable (*deferred);
 *   - a failed resync_block adds one to the entry's errors, sets last_try_ms = now and queues it at next_try_ms
 *     (*failed); a success removes the error entry (*resynced).
 * *wait_ms = ms until the queue's first entry falls due (0 if one is due), 10 000 for an empty queue (IdleFor).
 * File store: from the first step or retry-now on, the node's queue and error table are kept in <data_dir>/node<N>/resync
 * (written at the end of each step that took an entry, on retry-now and at destroy; tmp file, fsync and rename under
 * data_fsync) and
 * loaded at create; a node that never ran either writes no file.  GARAGE_EC_E_INVALID for a bad node or workers
 * outside 1..8; GARAGE_BM_E_MESSAGE if the node is down or the file cannot be written.  Output pointers may be NULL.
 * Steps of different nodes may run together and with PUTs and resync_all; a node's own steps run one at a time.
 * The workers are threads of the step's own; the calling thread's CPU affinity is left as it was.                  */
int garage_bm_resync_step(garage_bm *bm, int node, int workers, size_t max_blocks, uint64_t *resynced, uint64_t *failed,
                          uint64_t *deferred, int64_t *wait_ms);
/* garage block list-errors: the error entries of `node` (-1: every node) in node then hash order.  *n = their number
 * and at most cap of them are written to out, so *n > cap means the list was cut (out NULL, cap 0: a size query).
 * GARAGE_EC_E_INVALID only for a bad node, n NULL, or out NULL with cap > 0.                                       */
int garage_bm_list_resync_errors(garage_bm *bm, int node, garage_bm_resync_error *out, size_t cap, size_t *n);
/* garage block retry-now (clear_backoff, resync.rs:119-134): the entry of hash (NULL: every error entry of node) keeps
 * its error count, gets last_try_ms = now - its delay and is due now.  GARAGE_BM_E_MESSAGE for a hash without an
 * error entry on node.  *n (nullable) = entries made due.                                                         */
int garage_bm_resync_retry_now(garage_bm *bm, int node, const uint8_t *hash32, uint64_t *n);
/* garage block info under erasure coding: for each index of the block's row in the newest layout version, its holder
 * and GARAGE_BM_SHARD_* state, and that holder's resync error count; whether the stripe can be rebuilt, decided by
 * garage_ec_read_set over the valid indices, and the read set of that rebuild.  Read-only: nothing is quarantined,
 * queued or written.  check_tags = 0: "valid" means the header checks out; 1: every shard is read and its tag
 * checked, outside the holder's lock (only the header look holds it).  GARAGE_EC_E_INVALID for NULL hash or out.  */
int garage_bm_block_info(garage_bm *bm, const uint8_t hash[32], int check_tags, garage_bm_block_status *out);
/* Test clock of the scheduled queue and the error table (not of block_gc_delay_ms): now_ms > 0 is "now", 0 the real
 * clock.  Set it before anything is queued: entries queued earlier carry real-clock due times.                  */
int garage_bm_debug_set_clock_ms(garage_bm *bm, uint64_t now_ms);
void garage_bm_get_resync_metrics(garage_bm *bm, garage_bm_resync_metrics *out);

/* ScrubWorker sweep over all shards stored on `node` (repair.rs:438-490): GPU blake2sum of each
 * shard; a mismatch quarantines the shard (.corrupted, manager.rs:807-819) and queues a resync
 * (manager.rs:592-605).                                                                         */
int garage_bm_scrub(garage_bm *bm, int node, uint64_t *checked, uint64_t *corrupt);
/* the same sweep in resumable steps -- the scrub checkpoint of the reference (ScrubWorker persists its
 * BlockStoreIterator position every 60 s, repair.rs:186-193,460-464): shards are visited in hash order
 * starting after cursor32 (NULL = from the start), at most max_shards (0 = all); cursor_out32 is the
 * position to persist, *finished = 1 once the end of the node's store was reached.                */
int garage_bm_scrub_step(garage_bm *bm, int node, const uint8_t *cursor32, size_t max_shards,
                         uint8_t cursor_out32[32], int *finished, uint64_t *checked, uint64_t *corrupt);

/* Deep scrub (DESIGN.md section 5.4), resumable in hash order like garage_bm_scrub_step: the known blocks not at rc 0
 * whose deep-scrub owner is `node` -- the first up node of the block's row in the newest layout version -- after
 * cursor32 (NULL = from the start), at most max_blocks of them (0 = all).  In batches of batch_max_blocks, all k+m
 * shards of the configured stripe are read (tags checked on read) and garage_ec_deep_check proves the block's content
 * hash and every parity row on the GPU:
 *   - hash and parity right: clean;
 *   - hash right, parity rows wrong: every flagged parity shard is quarantined (and queued for resync);
 *   - hash wrong: the stale-shard hunt of GET quarantines the culprit, or, if no consistent set exists, the block
 *     counts in deep_scrub_content_errors and no file is touched.
 * A block with a configured shard missing or bad is skipped (its resync queued); a block held only under a previous
 * code or as replicas is skipped without one.  *checked = blocks deep-checked, *repaired = shards quarantined.
 * GARAGE_BM_E_MESSAGE if `node` is down.                                                                          */
int garage_bm_deep_scrub_step(garage_bm *bm, int node, const uint8_t *cursor32, size_t max_blocks,
                              uint8_t cursor_out32[32], int *finished, uint64_t *checked, uint64_t *repaired);

/* Stripe repair (DESIGN.md section 5.6), resumable in hash order like garage_bm_deep_scrub_step over the same blocks:
 * the known blocks not at rc 0 whose owner is `node` (the deep-scrub owner rule).  For each block:
 *   - probe: each of the k+m holders is asked whether it holds a shard of its index whose file header checks out (no
 *     shard bytes are read; Garage's NeedBlockQuery).  missing = k+m - present, a down holder counting as missing;
 *     the targets are the missing indices whose holder is up;
 *   - skip the block if it has no target or missing < min_missing (min_missing <= 1: every block with a target), or
 *     if no shard of the configured code is present and previous codes or replicas are configured;
 *   - gather once, want = the targets, through the code's own plan (RS: the first k; LRC: the union of the local
 *     groups; PB: the planned halves; Clay: the repair runs when exactly one shard is absent, k whole shards
 *     otherwise), tags checked on read.  A bad survivor is quarantined and the plan recomputed; if its holder is up
 *     it becomes one more target;
 *   - rebuild batch_max_blocks stripes per garage_ec_reconstruct_stripes, and write each rebuilt shard to its holder.
 * Nothing is fatal: an unrecoverable stripe and a failed shard write each count one stripe_repair_errors, and the
 * other targets of the stripe are still written.  *repaired_blocks = stripes with a shard written, *rebuilt_shards =
 * shards written.  GARAGE_BM_E_MESSAGE if `node` is down; GARAGE_EC_E_INVALID while more than one layout version is
 * active (layout sync rebuilds then).  Calls for different owners, and resync_all, may run concurrently.          */
int garage_bm_stripe_repair_step(garage_bm *bm, int node, const uint8_t *cursor32, size_t max_blocks, int min_missing,
                                 uint8_t cursor_out32[32], int *finished, uint64_t *repaired_blocks,
                                 uint64_t *rebuilt_shards);

/* Conversion sweep of `node` (DESIGN.md section 5.1), resumable in hash order like garage_bm_scrub_step: every block
 * with a legacy shard or replica on `node`, after cursor32 (NULL = from the start), at most max_blocks (0 = all):
 *   - the configured stripe holds its write quorum: this node deletes its legacy copies;
 *   - rc 0: the legacy copies are deleted once block_gc_delay_ms has passed, nothing is converted;
 *   - this node is the block's converter (the first up node holding a legacy copy, in code order, shard index
 *     order, then replica order): the old data shards (or the replica) go through garage_ec_transcode in batches
 *     of batch_max_blocks, the new data shards are checked against the content hash before anything is written,
 *     the k+m new shards are written, and once k+1 are durable the legacy copies on the up nodes are deleted.
 * *converted = blocks this call converted.  A block that could not be converted keeps every legacy copy.        */
int garage_bm_convert_step(garage_bm *bm, int node, const uint8_t *cursor32, size_t max_blocks, uint8_t cursor_out32[32],
                           int *finished, uint64_t *converted);

/* Changing the cluster layout (file store; DESIGN.md section 5.2).  garage_bm_apply_layout computes the next version
 * with previous = the newest one (nodes that stay keep their shard index) and makes it active; PUTs then write to
 * every active version and need k+1 shards in each.  GARAGE_EC_E_INVALID for the memory store, with previous_codes or
 * legacy_replicas configured, for a spec garage_bm_create would reject, or when more than
 * GARAGE_BM_MAX_LAYOUT_VERSIONS versions would be active.  *version_out = the new version.                       */
int garage_bm_apply_layout(garage_bm *bm, const garage_bm_layout_spec *spec, uint64_t *version_out);
/* Layout sync of `node`, resumable in hash order like garage_bm_scrub_step: every block the newest version assigns
 * to `node` and every shard `node` holds, after cursor32 (NULL = from the start), at most max_blocks (0 = all):
 *   - receive: the node lacks a valid shard of its newest index: copy it from that index's holder in an older active
 *     version (oldest first, tag checked), else rebuild it on the GPU from the survivors of every active version;
 *   - offload: the node holds an index the newest version does not give it: deleted once the newest stripe is seen
 *     with k+1 valid shards at their assigned (node, index); a block at rc 0 is deleted after block_gc_delay_ms.
 * A full pass (cursor NULL to *finished) that leaves nothing to receive records the node as synced; once every
 * storage node of the newest version is, the older versions are retired.  *moved = shards copied or rebuilt.
 * Its renames, writes and deletes count as file operations for garage_bm_debug_convert_stop_after.  Calls for
 * different nodes may run concurrently (their GPU rebuild batches then run one at a time); a node's own steps are
 * made one after another.                                                                                      */
int garage_bm_layout_sync_step(garage_bm *bm, int node, const uint8_t *cursor32, size_t max_blocks,
                               uint8_t cursor_out32[32], int *finished, uint64_t *moved);
/* the active layout versions, oldest first; returns their number (at most cap are written)                       */
int garage_bm_layout_versions(garage_bm *bm, uint64_t *out, int cap);

/* Drives (file store; DESIGN.md section 5.7).  garage_bm_set_data_dirs: node `node` restarts with this data_dir list
 * (the same rules as garage_bm_config.data_dirs): the drive layout is updated by path (initialised if the node has
 * none), the markers checked and <node dir>/data_layout written.  GARAGE_EC_E_INVALID for a list create would
 * reject; GARAGE_BM_E_MESSAGE if a drive fails its marker check, which leaves the node down and its layout as it was;
 * on success the node is up.                                                                                      */
int garage_bm_set_data_dirs(garage_bm *bm, int node, const garage_bm_data_dir *dirs, int n);
/* RebalanceWorker (repair.rs:531-626), resumable in hash order like garage_bm_scrub_step: the hashes with a file on a
 * drive other than their primary, after cursor32 (NULL = from the start), at most max_files of them (0 = all).  Each
 * such .shard, .legacy or replica file is read and checked (shards by header and tag; a replica is moved as it is),
 * written to the primary, then the old copy removed; a copy the primary already has is removed only.  A shard that
 * fails is quarantined next to itself and queued for resync.  A full pass (cursor NULL to *finished) that left no
 * misplaced file behind, with no drive change meanwhile, drops the secondaries and persists the layout.  Its writes
 * and removals count as file operations for garage_bm_debug_convert_stop_after.  *moved = files moved.
 * GARAGE_EC_E_INVALID for a node without drives, GARAGE_BM_E_MESSAGE if the node is down.                         */
int garage_bm_rebalance_step(garage_bm *bm, int node, const uint8_t *cursor32, size_t max_files, uint8_t cursor_out32[32],
                             int *finished, uint64_t *moved);
void garage_bm_get_drive_metrics(garage_bm *bm, garage_bm_drive_metrics *out);

/* native closed-loop load generator (row f1: the batching front-end decides real-world throughput):
 * `threads` client threads each PUT (mode 0) or GET (mode 1) `blocks_per_thread` blocks of `block_len`
 * bytes (splitmix64 stream of `seed`; a GET run must follow a PUT run with the same arguments).  The
 * content hashes are computed before the clock starts (put.rs:448 does that in the API layer).        */
int garage_bm_bench(garage_bm *bm, int threads, int blocks_per_thread, uint32_t block_len, int mode,
                    uint64_t seed, double *gib_per_s, uint64_t *errors);

/* fault injection / inspection for tests */
int garage_bm_set_node_up(garage_bm *bm, int node, int up);
int garage_bm_corrupt_shard(garage_bm *bm, int node, const uint8_t hash[32], size_t byte_off);
/* what = 1: stored block_len + 1; what = 2: stored shard index + 1 (header check left alone)          */
int garage_bm_corrupt_shard_header(garage_bm *bm, int node, const uint8_t hash[32], int what);
/* overwrite the shard with a self-consistent shard of OTHER content (valid tag, right index): only the
 * whole-block content hash can notice                                                                 */
int garage_bm_plant_stale_shard(garage_bm *bm, int node, const uint8_t hash[32]);
/* file store only: make every write to the node's directory fail (like ENOSPC / EACCES / a lost mount) */
int garage_bm_set_node_readonly(garage_bm *bm, int node, int readonly);
int garage_bm_drop_shard(garage_bm *bm, int node, const uint8_t hash[32]);
/* after n_ops more file operations of conversions and layout syncs (renames to .legacy, shard writes, deletes), make
 * every further one fail, as if the process had stopped there; n_ops < 0 turns it off                            */
int garage_bm_debug_convert_stop_after(garage_bm *bm, long n_ops);
int garage_bm_node_shard_index(garage_bm *bm, int node, const uint8_t hash[32]); /* -1 if none */
/* the newest active layout version's row: shard i of the block on nodes_out[i]                                  */
int garage_bm_storage_nodes_of(garage_bm *bm, const uint8_t hash[32], int *nodes_out /* k+m */);
void garage_bm_get_metrics(garage_bm *bm, garage_bm_metrics *out);
void garage_bm_get_range_metrics(garage_bm *bm, garage_bm_range_metrics *out);
void garage_bm_get_stripe_repair_metrics(garage_bm *bm, garage_bm_stripe_repair_metrics *out);
void garage_bm_get_salvage_metrics(garage_bm *bm, garage_bm_salvage_metrics *out);
void garage_bm_get_segment_repair_metrics(garage_bm *bm, garage_bm_segment_repair_metrics *out);

#ifdef __cplusplus
}
#endif
#endif
