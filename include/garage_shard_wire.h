/*
 * garage_shard_wire.h -- wire / metadata encoding of one erasure-coded shard (SURVEY.md section 8
 * rows a8 / f3), part of libgarage_block.so.
 *
 * Reference: the block RPC carries `BlockRpc::PutBlock { hash, header: DataBlockHeader }`
 * (src/block/manager.rs:54-69, src/block/block.rs:12-16) serialised by rmp-serde as a msgpack MAP
 * with field names (`Serializer::with_struct_map`, src/util/migrate.rs:32-38); format changes are
 * versioned by a marker prefix and a `Migrate::Previous` chain (src/util/migrate.rs:5-39, used e.g.
 * by ScrubWorkerPersisted, src/block/repair.rs:214-229).  With erasure coding a node receives one
 * SHARD, so the message needs the shard index, the code (k, m), the unpadded block length and the
 * shard's integrity tag.  This is that message, encoded the same way:
 *
 *   v1 (erasure coded)  marker "GEC1shdr" + msgpack map
 *        { "hash": bin32, "header": "Plain" | "Compressed", "k": uint, "m": uint, "index": uint,
 *          "block_len": uint, "shard_len": uint, "sum_kind": uint, "sum": bin32[, "l": uint][, "pb": 1][, "clay": 1] }
 *        "l" (LRC local groups, garage_ec_create_lrc) is present only for an LRC code (l > 0), "pb" only
 *        for a piggybacked RS code (garage_ec_create_piggyback) and "clay" only for a Clay code
 *        (garage_ec_create_clay), so RS messages are byte for byte what they
 *        were before either existed.
 *   v0 (Previous)       the reference's replicated PutBlock payload, no marker:
 *        { "hash": bin32, "header": "Plain" | "Compressed" }
 *        migrate(v0) = the whole block as the only shard of a (k = 1, m = 0) code, index 0,
 *        block_len / shard_len unknown (0: taken from the attached stream), no shard tag --
 *        so blocks written before the upgrade stay readable.
 *
 * decode() follows Migrate::decode: marker + current format first, else the previous format.
 */
#ifndef GARAGE_SHARD_WIRE_H
#define GARAGE_SHARD_WIRE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GARAGE_SHARD_WIRE_MARKER "GEC1shdr"
#define GARAGE_SHARD_HEADER_PLAIN 0      /* DataBlockHeader::Plain      */
#define GARAGE_SHARD_HEADER_COMPRESSED 1 /* DataBlockHeader::Compressed */

typedef struct {
    uint8_t hash[32];   /* content address of the BLOCK (blake2sum of its plain bytes)            */
    uint8_t header;     /* GARAGE_SHARD_HEADER_*: what the block bytes are (before splitting)     */
    uint8_t k, m;       /* the code; k = 1, m = 0 for a migrated replicated block                 */
    uint8_t index;      /* which of the k+m shards                                                */
    uint8_t sum_kind;   /* GARAGE_EC_SUM_* of `sum` (include/garage_ec.h)                         */
    uint8_t migrated;   /* set by decode when the bytes were the previous (replicated) format     */
    uint32_t block_len; /* unpadded length of the whole block                                     */
    uint32_t shard_len; /* ceil(block_len / k)                                                    */
    uint8_t sum[32];    /* integrity tag of this shard's bytes                                    */
    uint8_t l;          /* LRC local groups (0 < l < m, k % l == 0); 0 = RS                        */
    uint8_t pb;         /* 1: piggybacked RS PB(k, m) (l = 0, 2 <= m <= 4, k <= 16); 0 = not PB     */
    uint8_t clay;       /* 1: Clay(k, m) (l = 0, pb = 0, 2 <= m <= 4); 0 = not Clay                 */
} garage_shard_header;

/* returns the encoded length, or 0 if `cap` is too small / the header is invalid (<= 160 bytes)   */
size_t garage_shard_wire_encode(const garage_shard_header *h, uint8_t *out, size_t cap);
/* 0 on success, -1 if the bytes are neither format                                               */
int garage_shard_wire_decode(const uint8_t *bytes, size_t len, garage_shard_header *out);
/* the previous format, for tests and for talking to not-yet-upgraded nodes                        */
size_t garage_shard_wire_encode_v0(const uint8_t hash[32], int header, uint8_t *out, size_t cap);

#ifdef __cplusplus
}
#endif
#endif
