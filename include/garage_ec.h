/*
 * garage_ec.h -- C ABI of libgarage_ec.so: the H100 (sm_90a) erasure-coding block path
 * for Garage.
 *
 * The reference (deuxfleurs-org/garage v1.2.0) has no FFI and no erasure coding; its
 * drop-in boundary is the Rust surface of garage_block::manager::BlockManager
 * (SURVEY.md section 8(b)).  Each entry point below names the reference call site whose
 * CPU-side per-block work it replaces; the Rust `src/block/cuda` shim that binds these
 * symbols is shown in INTEGRATION.md.
 *
 * Conventions (mirroring the reference's, SURVEY.md section 8(b)):
 *   errors     every call returns 0 or a negative GARAGE_EC_E_* code; nothing aborts or
 *              throws across the boundary (reference: Result<_, garage_util::error::Error>,
 *              src/util/error.rs:14-82; Rust maps non-zero to Error::Message /
 *              Error::CorruptData so resync's backoff handles it, src/block/resync.rs:300-315).
 *   ownership  caller owns every buffer; the library keeps no pointer after a HOST call
 *              returns, or after the stream work of a DEVICE call completes
 *              (reference: bytes::Bytes, immutable + refcounted).
 *   threading  a context may be used from many OS threads at once (reference: tokio
 *              spawn_blocking, src/block/block.rs:86, src/api/s3/put.rs:419,446).
 *   no CPU fallback: if there is no usable CUDA device, garage_ec_create fails with
 *              GARAGE_EC_E_NODEVICE.
 *
 * Arithmetic (normative definition in DESIGN.md; CPU oracle under oracle/):
 *   GF(2^8), polynomial 0x11D, alpha = 2.  One stripe = one block (post-compression bytes
 *   of DataBlock::from_buffer, src/block/block.rs:85-96).  shard_len = ceil(block_len/k);
 *   data shard j = block bytes [j*shard_len,(j+1)*shard_len) zero-padded; parity row
 *   i = XOR_j P[i][j] * data[j].
 *
 * Batch geometry ("shard layout"), shared by encode / reconstruct / verify:
 *   stride      bytes between consecutive shards; multiple of 16; >= every shard_len[s];
 *               (k+m)*stride < 4 GiB
 *   shard_len   per-stripe valid bytes per shard (NULL = `stride` for every stripe).
 *               Bytes in [shard_len, roundup16(shard_len)) of every OUTPUT shard are
 *               written as zero; input bytes there are ignored.  Beyond roundup16 nothing
 *               is written; input bytes up to `stride` may be read (the tile loads of the
 *               k >= 13 kernels fetch whole 512-byte rows) but never influence a result,
 *               so the whole n * shards * stride array must be addressable.
 *   all base pointers 16-byte aligned.
 */
#ifndef GARAGE_EC_H
#define GARAGE_EC_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GARAGE_EC_ABI_VERSION 1

/* error codes */
#define GARAGE_EC_OK 0
#define GARAGE_EC_E_INVALID (-1)       /* bad argument / geometry */
#define GARAGE_EC_E_CUDA (-2)          /* CUDA runtime error, see garage_ec_last_error */
#define GARAGE_EC_E_NOMEM (-3)         /* host or device allocation failed */
#define GARAGE_EC_E_UNRECOVERABLE (-4) /* >= 1 stripe could not be rebuilt; see status[] */
#define GARAGE_EC_E_NODEVICE (-5)      /* no CUDA device / wrong architecture */
#define GARAGE_EC_E_ALIGN (-6)         /* pointer or stride alignment violated */
#define GARAGE_EC_E_AUTH (-7)          /* a block failed authentication (a GCM tag, or its framing); see status[] */

/* matrix kinds */
#define GARAGE_EC_VANDERMONDE 0 /* systematic Vandermonde (default), G = V * inv(V[0..k)) */
#define GARAGE_EC_CAUCHY 1      /* P[i][j] = 1/((k+i) xor j) */

/* where the caller's buffers live */
#define GARAGE_EC_MEM_HOST 0   /* all pointers host; call is synchronous */
#define GARAGE_EC_MEM_DEVICE 1 /* all pointers device (this ctx's GPU); call enqueues on `stream` */

/* limits of this build */
#define GARAGE_EC_MAX_K 32
#define GARAGE_EC_MAX_M 8

typedef struct garage_ec_ctx garage_ec_ctx;

/* ---- lifecycle -------------------------------------------------------------------------
 * One context per (GPU, k, m, matrix).  Replaces nothing in the reference: it is the state
 * a BlockManager built with `erasure_coding = {data_shards, parity_shards}` would hold
 * next to `data_layout` (src/block/manager.rs:122-192).                                    */
int garage_ec_create(garage_ec_ctx **out, int cuda_device, int k, int m, int matrix_kind);
/* same, with an explicit m x k parity matrix (row-major) -- used by non-zero ranks after
 * the NCCL broadcast of rank 0's matrix (SURVEY.md section 8(e)).                          */
int garage_ec_create_with_matrix(garage_ec_ctx **out, int cuda_device, int k, int m,
                                 const uint8_t *parity_rows);
/* Locally repairable code LRC(k, l, r): m = l + r parity shards.  The k data shards form l groups of k/l;
 * parity k+g (g < l) is the XOR of group g, parities k+l.. are the r Cauchy rows of RS(k, r)
 * (P[i][j] = 1/((k+i) xor j)).  One lost shard of a group is rebuilt from the other k/l shards of the
 * group instead of from k shards.  Needs l >= 1, r >= 1, k % l == 0, l + r <= GARAGE_EC_MAX_M,
 * k <= GARAGE_EC_MAX_K; GARAGE_EC_E_INVALID otherwise, before any CUDA call.  Encode / verify /
 * reconstruct / scrub_repair / *_blocks work unchanged; reconstruct decides recoverability by rank
 * (DESIGN.md section 2), so some patterns with fewer than k present shards decode.                   */
int garage_ec_create_lrc(garage_ec_ctx **out, int cuda_device, int k, int l, int r);
/* Piggybacked Reed-Solomon PB(k, m) (DESIGN.md section 2.2): RS(k, m) with parity rows of `matrix_kind`, every
 * shard cut in an a-half and a b-half; the b-half of parity i >= 1 also carries the XOR of the a-halves of data
 * group G_i (m-1 contiguous groups).  Same storage and the same any-m-loss tolerance as RS(k, m); one lost data
 * shard is rebuilt from k + |G_i| halves instead of 2k (PB(10,4): 0.65-0.70 of the bytes).  Every stripe's
 * shard_len must be a multiple of 32 (garage_ec_code_shard_len gives a multiple of 128).  For a stripe where it is
 * not, a DEVICE call rebuilds and encodes nothing (encode writes nothing for it, verify sets every mismatch bit,
 * reconstruct reports GARAGE_EC_E_INVALID in status[]); a HOST call returns GARAGE_EC_E_INVALID before any GPU work.  Needs
 * 1 <= k <= 16, 2 <= m <= 4; GARAGE_EC_E_INVALID otherwise, before any CUDA call.                                  */
int garage_ec_create_piggyback(garage_ec_ctx **out, int cuda_device, int k, int m, int matrix_kind);
/* Clay code Clay(k, m) (DESIGN.md section 2.4): MDS, any m losses decode, and one lost shard -- data or parity -- is
 * rebuilt from 1/m of each of the other k+m-1 shards (Clay(10,4): 0.33 of RS(10,4)'s repair bytes).  q = m,
 * t = ceil((k+m)/q), alpha = q^t layers per shard, s = q*t - k - m virtual nodes; every layer is coupled from a
 * codeword of RS(k+s, m) with parity rows of `matrix_kind`.  Every stripe's shard_len must be a multiple of 16*alpha
 * (garage_ec_code_shard_len gives one); for a stripe where it is not, a DEVICE call behaves as for PB (encode writes
 * nothing, verify sets every mismatch bit, reconstruct reports GARAGE_EC_E_INVALID in status[]) and a HOST call
 * returns GARAGE_EC_E_INVALID before any GPU work.  Needs m in {2, 3, 4}, k >= 2, alpha <= 256 (Clay(10,4): 256,
 * Clay(6,3): 27); GARAGE_EC_E_INVALID otherwise, before any CUDA call.  garage_ec_matrix and garage_ec_read_plan
 * return GARAGE_EC_E_INVALID on a Clay context; garage_ec_read_ranges names what to fetch.                        */
int garage_ec_create_clay(garage_ec_ctx **out, int cuda_device, int k, int m, int matrix_kind);
void garage_ec_destroy(garage_ec_ctx *ctx);

int garage_ec_matrix(const garage_ec_ctx *ctx, uint8_t *out_m_by_k); /* parity rows, row-major */
int garage_ec_params(const garage_ec_ctx *ctx, int *k, int *m, int *cuda_device);
/* LRC contexts: (l, r); RS contexts: (0, m).  garage_ec_matrix returns the l local rows, then the r global rows. */
int garage_ec_code_info(const garage_ec_ctx *ctx, int *local_groups, int *global_parity);
/* Which shards a gatherer should fetch to rebuild the wanted absent shards of ONE stripe (host only, no GPU
 * work): read_out[i] = 1 iff reconstruct reads shard i.  present / want / read_out: k+m bytes; want NULL =
 * every absent shard.  RS: the first k present shards.  LRC: the other members of each wanted shard's
 * local group when every wanted shard is the only absent member of its group, else a rank basis of the
 * present shards taken greedily in index order (DESIGN.md section 2).  GARAGE_EC_E_UNRECOVERABLE if a
 * wanted shard cannot be rebuilt.  Presenting only these shards to reconstruct rebuilds the same bytes. */
int garage_ec_read_set(const garage_ec_ctx *ctx, const uint8_t *present, const uint8_t *want, uint8_t *read_out);
/* PB contexts: *groups = m-1 and group_of[j] = i (1..m-1) for data shard j of G_i (k bytes, nullable); RS and LRC
 * contexts: 0 groups, group_of[] all 0.                                                                          */
int garage_ec_piggyback_info(const garage_ec_ctx *ctx, int *groups, uint8_t *group_of);
/* Clay contexts: q, t, alpha, the virtual node count s and (nullable) the m x (k+s) base-code parity rows, row-major.
 * Other contexts: alpha = 1, the rest 0, base_rows untouched.                                                       */
int garage_ec_clay_info(const garage_ec_ctx *ctx, int *q, int *t, int *alpha, int *virtual_nodes, uint8_t *base_rows);
/* Byte runs of the shards a gatherer fetches to rebuild the wanted absent shards of ONE stripe (host only):
 * {shard, offset, len} in shard then offset order, adjacent runs merged.  RS and LRC: whole shards of
 * garage_ec_read_set; PB: the planned halves; Clay: when exactly one shard is absent and wanted, its repair runs in
 * every other shard (q^y0 sub-chunks of shard_len/alpha bytes every q^(y0+1)), else the first k present shards
 * whole.  Presenting only these bytes to reconstruct rebuilds the same output.  *n_ranges = the number of runs;
 * GARAGE_EC_E_INVALID if it exceeds cap (nothing past cap is written) or shard_len breaks the code's framing
 * (PB: % 32, Clay: % (16*alpha)); GARAGE_EC_E_UNRECOVERABLE if a wanted shard cannot be rebuilt.                    */
typedef struct garage_ec_range {
    uint32_t shard, offset, len;
} garage_ec_range;
int garage_ec_read_ranges(const garage_ec_ctx *ctx, const uint8_t *present, const uint8_t *want, uint32_t shard_len,
                          garage_ec_range *ranges, size_t cap, size_t *n_ranges);
/* Shard length of a block_len-byte block under this context's code: ceil(block_len / k) for RS and LRC, that
 * rounded up to a multiple of 128 for PB, of 16*alpha for Clay.  The block-level calls frame blocks with it.  GARAGE_EC_E_INVALID if
 * that length does not fit in 32 bits (PB(1, m) with block_len > 2^32 - 128).                                   */
int garage_ec_code_shard_len(const garage_ec_ctx *ctx, uint32_t block_len, uint32_t *shard_len);
/* Half-shard form of garage_ec_read_set: halves_out[i] bit 0 = read the a-half [0, shard_len/2) of shard i,
 * bit 1 = read the b-half.  PB: rule 1 (k + |G_i| halves) or rule 2 (DESIGN.md section 2.2); RS and LRC: 3 for every
 * shard of garage_ec_read_set.  garage_ec_read_set on a PB context reports a shard iff any of its halves is read. */
int garage_ec_read_plan(const garage_ec_ctx *ctx, const uint8_t *present, const uint8_t *want, uint8_t *halves_out);
const char *garage_ec_strerror(int code);
/* detail of the last GARAGE_EC_E_CUDA on this context (thread-unsafe snapshot; "" if none) */
const char *garage_ec_last_error(const garage_ec_ctx *ctx);
int garage_ec_abi_version(void);

/* ---- geometry helpers ------------------------------------------------------------------ */
uint32_t garage_ec_shard_len(uint32_t block_len, int k); /* ceil(block_len / k)            */
size_t garage_ec_stride_for(uint32_t shard_len);         /* shard_len rounded up to 128 B   */

/* ---- ENCODE -- call site: BlockManager::rpc_put_block, src/block/manager.rs:366-408,
 * right after DataBlock::from_buffer (manager.rs:376): the k data shards of each block go in,
 * the m parity shards come out; shard i is then sent to node i of the (k+m)-node set.
 *   data   : n * k * stride bytes, shard j of stripe s at (s*k + j) * stride
 *   parity : n * m * stride bytes, row  i of stripe s at (s*m + i) * stride
 * A stripe whose shard_len exceeds `stride` is malformed, for every code: a HOST call returns
 * GARAGE_EC_E_INVALID before any GPU work; a DEVICE call writes nothing of that stripe's parity
 * and encodes the other stripes.                                                            */
int garage_ec_encode(garage_ec_ctx *ctx, const uint8_t *data, uint8_t *parity,
                     const uint32_t *shard_len, size_t stride, size_t n_stripes, int mem_kind,
                     void *cuda_stream);

/* ---- RECONSTRUCT -- call sites: BlockManager::rpc_get_raw_block_internal,
 * src/block/manager.rs:276-339 (GET: any k of k+m shards arrived, rebuild the missing data
 * shards) and BlockResyncManager::resync_block fetch branch, src/block/resync.rs:460-500
 * (repair: rebuild this node's own shard from k survivors).
 *   shards  : n * (k+m) * stride bytes, shard i of stripe s at (s*(k+m) + i) * stride
 *   present : n * (k+m) bytes in {0,1}
 *   want    : NULL = rebuild every absent shard; else n*(k+m) bytes, only absent shards
 *             with want != 0 are rebuilt (GET wants data shards only; resync wants one)
 *   status  : n int32: 0 ok, GARAGE_EC_E_UNRECOVERABLE if a wanted shard cannot be rebuilt (RS: < k
 *             present; stripe untouched)
 * Survivors used: those of garage_ec_read_set (RS: the first k present shards in index order); only
 * they are read, and HOST calls copy only them to the GPU.  HOST calls return
 * GARAGE_EC_E_UNRECOVERABLE if any stripe was; DEVICE calls only fill status[].  A stripe
 * whose shard_len exceeds `stride` is malformed, for every code: a HOST call returns
 * GARAGE_EC_E_INVALID before any GPU work; a DEVICE call reports GARAGE_EC_E_INVALID in its
 * status[], reads and writes nothing of it, and rebuilds the other stripes.                 */
int garage_ec_reconstruct(garage_ec_ctx *ctx, uint8_t *shards, const uint8_t *present,
                          const uint8_t *want, int32_t *status, const uint32_t *shard_len,
                          size_t stride, size_t n_stripes, int mem_kind, void *cuda_stream);

/* Gather form of the HOST-mode reconstruct for batching front-ends (SURVEY.md section 8 row f1): every
 * caller (a GET that lost shards, one of the 8 resync workers, src/block/resync.rs:43) owns its own
 * buffer -- stripes[s] points at the k+m shards of stripe s, `stride` apart -- and the batch is just the
 * list of those pointers: nobody copies shards into a contiguous staging array.  Pinned buffers from
 * garage_ec_host_alloc make the copies DMA-speed.  Same semantics as garage_ec_reconstruct(MEM_HOST). */
int garage_ec_reconstruct_stripes(garage_ec_ctx *ctx, uint8_t *const *stripes, const uint8_t *present,
                                  const uint8_t *want, int32_t *status, const uint32_t *shard_len,
                                  size_t stride, size_t n_stripes);

/* ---- RECONSTRUCT BY SEGMENT (normative: DESIGN.md section 2.10) -- a stripe with more than m damaged shards whose
 * damage falls in different adler8 segments: every segment of a stripe covers the same byte columns of all k+m shards,
 * and each is decoded on its own.  Shard layout, stride and alignment rules: those of garage_ec_reconstruct.
 *   seg_present : n * (k+m) bytes; bit g set = segment g of shard i holds valid bytes (0x00 a wholly absent shard, 0xFF
 *                 a whole one).  Segment g of a stripe = [g*S, min(L, (g+1)*S)), S = roundup16(ceil(L/8)): the adler8
 *                 segments, the runs garage_ec_tag_span names.  An empty segment counts as present.
 *   want        : NULL = every shard with a cleared bit; else n * (k+m) bytes, only wanted shards are completed.
 *   Units       : RS and LRC: one segment.  PB: segments g and g+4 (g < 4), with L % 128 == 0 so that S = L/8; a shard
 *                 is present in a PB unit only if both bits are set.  Each unit is decoded from the code's own read
 *                 set for the unit's presence map (RS: the first k present shards; LRC: the local group when it
 *                 suffices; PB: garage_ec_read_plan), and every missing unit of a wanted shard is rebuilt from it.  A
 *                 unit's verdict is garage_ec_reconstruct's for that presence map and want.
 *   Writes      : only the bytes of rebuilt units, and the zero tail [L, roundup16(L)) of a shard whose last unit is
 *                 rebuilt.  A unit whose bytes are present is never written.
 *   status      : n int32 (nullable in DEVICE mode): 0; GARAGE_EC_E_UNRECOVERABLE if a unit cannot be rebuilt (nothing
 *                 of the stripe is written); DEVICE only: GARAGE_EC_E_INVALID for an L past `stride` or, for PB, an L
 *                 that is not a multiple of 128 (nothing of the stripe is read or written).
 * With every seg_present byte 0x00 or 0xFF the output is byte-identical to garage_ec_reconstruct with
 * present = (byte == 0xFF).  Clay contexts return GARAGE_EC_E_INVALID before any CUDA call: a Clay shard's layers are
 * coupled across the whole shard, so its segments are not independent codewords.
 *   DEVICE: only kernels and stream-ordered scratch are enqueued (capturable in a CUDA graph); reads only the survivor
 *           bytes of each unit's read set, never past byte n*(k+m)*stride of `shards`.
 *   HOST:   synchronous; GARAGE_EC_E_INVALID before any GPU work for a malformed L; uploads only the survivor units of
 *           stripes that have work and downloads only the rebuilt units; returns GARAGE_EC_E_UNRECOVERABLE if any
 *           stripe was.  The _stripes form is the gather form, as garage_ec_reconstruct_stripes.                    */
int garage_ec_reconstruct_segments(garage_ec_ctx *ctx, uint8_t *shards, const uint8_t *seg_present,
                                   const uint8_t *want, int32_t *status, const uint32_t *shard_len,
                                   size_t stride, size_t n_stripes, int mem_kind, void *cuda_stream);
int garage_ec_reconstruct_segments_stripes(garage_ec_ctx *ctx, uint8_t *const *stripes,
                                           const uint8_t *seg_present, const uint8_t *want, int32_t *status,
                                           const uint32_t *shard_len, size_t stride, size_t n_stripes);
/* garage_ec_segment_read_ranges (host only, ONE stripe of shard length shard_len; seg_present / want: k+m bytes, as
 * for garage_ec_reconstruct_segments): the byte runs {shard, offset, len} garage_ec_reconstruct_segments reads to
 * complete the wanted shards -- for every unit in which a wanted shard is absent, the unit's columns of each shard of
 * that unit's read set (RS: the first k present; LRC: the local group when it suffices; PB: the garage_ec_read_plan
 * halves).  Runs are in garage_ec_read_ranges' order and merge rule: by shard, then offset, adjacent runs merged.
 * Bytes outside them are never read: a stripe holding only these runs (and its own present units) rebuilds to the
 * same bytes.  GARAGE_EC_E_INVALID on a Clay context, for PB with shard_len % 128 != 0, or when the runs pass `cap`
 * (*n_ranges = the runs needed); GARAGE_EC_E_UNRECOVERABLE when a unit cannot be rebuilt.                          */
int garage_ec_segment_read_ranges(const garage_ec_ctx *ctx, const uint8_t *seg_present, const uint8_t *want,
                                  uint32_t shard_len, garage_ec_range *ranges, size_t cap, size_t *n_ranges);

/* ---- VERIFY (scrub) -- call sites: DataBlock::verify via BlockManager::read_block,
 * src/block/manager.rs:554-609 / src/block/block.rs:69-83, driven by ScrubWorker::work,
 * src/block/repair.rs:438-490: recompute parity from the k data shards and compare with
 * the stored parity.  mismatch[s] bit i set iff parity row i differs.  A stripe whose
 * shard_len exceeds `stride` is malformed, for every code: a HOST call returns
 * GARAGE_EC_E_INVALID before any GPU work; a DEVICE call sets its m low mismatch bits and
 * reads nothing of it.                                                                      */
int garage_ec_verify(garage_ec_ctx *ctx, const uint8_t *shards, uint32_t *mismatch,
                     const uint32_t *shard_len, size_t stride, size_t n_stripes, int mem_kind,
                     void *cuda_stream);

/* ---- DEEP CHECK (deep scrub) -- what ScrubWorker::work proves for a plain block (src/block/repair.rs:438-490,
 * DataBlock::verify, src/block/block.rs:69-83: blake2sum(block) == hash), done on a stored stripe, together with
 * garage_ec_verify.  Per stripe s of the shard layout (k+m shards, `stride` apart):
 *   block_len : n values; L = garage_ec_code_shard_len(block_len[s]); the block is the first block_len bytes of data
 *               shards 0..k-1 concatenated (DESIGN.md section 2.3).  Shard bytes in [L, stride) are ignored
 *   hashes    : n * 32 bytes, the content addresses
 *   hash_bad  : n bytes out, 1 iff the block's blake2sum differs from hashes[s]
 *   mismatch  : n uint32 out, exactly garage_ec_verify's result for the stripe with shard_len = L (bit i = parity k+i)
 * A stripe whose L exceeds `stride`: a HOST call returns GARAGE_EC_E_INVALID before any GPU work; a DEVICE call
 * reports hash_bad = 1 and all m mismatch bits, and reads nothing of it.  DEVICE: all pointers device memory (hashes
 * 8-byte aligned), only kernels and stream-ordered scratch are enqueued (capturable in a CUDA graph).  HOST: uploads
 * roundup16(L) bytes of each shard.                                                                                 */
int garage_ec_deep_check(garage_ec_ctx *ctx, const uint8_t *shards, const uint32_t *block_len, const uint8_t *hashes,
                         uint8_t *hash_bad, uint32_t *mismatch, size_t stride, size_t n_stripes, int mem_kind,
                         void *cuda_stream);

/* ---- PER-SHARD INTEGRITY (SURVEY.md section 8 row f2) -- call sites: DataBlock::verify,
 * src/block/block.rs:69-83 (Plain => blake2sum(data) == hash) and read_block_from,
 * src/block/manager.rs:577-609.  A node stores 1/k of a block, so the whole-block hash cannot be
 * checked locally: every shard carries its own blake2sum (BLAKE2b-512 truncated to 32 bytes,
 * src/util/data.rs:130-138), computed here over [0, shard_len) of each shard.
 *   shards          : n_stripes * shards_per_stripe shards, `stride` apart (shard layout)
 *   shards_per_stripe: k (a data array), m (a parity array) or k+m
 *   sums_out        : 32 bytes per shard
 * garage_ec_check_sums compares with `expect` instead: bad_out[i] = 1 iff shard i differs.
 * shard_len may be any length up to `stride`.  A stripe whose shard_len exceeds `stride` is
 * malformed: a HOST call returns GARAGE_EC_E_INVALID before any GPU work; a DEVICE call reads
 * nothing of its shards, leaves their sums_out bytes untouched and sets their bad_out to 1.    */
int garage_ec_shard_sums(garage_ec_ctx *ctx, const uint8_t *shards, const uint32_t *shard_len,
                         size_t stride, size_t n_stripes, int shards_per_stripe, uint8_t *sums_out,
                         int mem_kind, void *cuda_stream);
int garage_ec_check_sums(garage_ec_ctx *ctx, const uint8_t *shards, const uint8_t *expect,
                         const uint32_t *shard_len, size_t stride, size_t n_stripes,
                         int shards_per_stripe, uint8_t *bad_out, int mem_kind, void *cuda_stream);
/* ---- SCRUB + REPAIR sweep (BASELINE config 5) -- ScrubWorker::work (src/block/repair.rs:438-490)
 * feeding resync (src/block/resync.rs:354-503) in one pass: blake2sum every shard, treat the ones
 * whose sum differs from `expect_sums` as erased, rebuild them in place from the first k intact
 * shards.  bad_out[s*(k+m)+i] = 1 iff shard i was corrupt; status[s] = 0 or
 * GARAGE_EC_E_UNRECOVERABLE (> m corrupt shards: reported, never fatal -- resync.rs:300-315).
 * A stripe whose shard_len exceeds `stride` is malformed, for every code: a HOST call returns
 * GARAGE_EC_E_INVALID before any GPU work; a DEVICE call reads and writes nothing of it, sets
 * bad_out of all its k+m shards to 1 and reports GARAGE_EC_E_INVALID in its status[].         */
int garage_ec_scrub_repair(garage_ec_ctx *ctx, uint8_t *shards, const uint8_t *expect_sums,
                           uint8_t *bad_out, int32_t *status, const uint32_t *shard_len,
                           size_t stride, size_t n_stripes, int mem_kind, void *cuda_stream);
/* host-side blake2sum of one buffer (the same function, for block hashes / small inputs)       */
void garage_ec_blake2sum(const uint8_t *data, size_t len, uint8_t out32[32]);
/* Which 32-byte tag the per-shard integrity calls of a context compute and compare
 * (garage_ec_shard_sums / _check_sums / _scrub_repair / _encode_blocks_with_sums):
 *   GARAGE_EC_SUM_BLAKE2 (default)  Garage's blake2sum of the shard (src/util/data.rs:130-138):
 *                     cryptographic, compute-bound on the GPU (~0.5 TB/s).
 *   GARAGE_EC_SUM_ADLER8  the shard cut in 8 segments of roundup16(ceil(len/8)) bytes, tag = the 8
 *                     little-endian zlib Adler-32 values of the segments (empty segment: 1).  Catches
 *                     bit rot, which is all scrub needs -- the block's content address stays its
 *                     blake2sum -- and streams at HBM speed (SURVEY.md section 8 row f2 allows a cheap
 *                     per-shard checksum).  The shard file header records which kind it carries.
 * garage_ec_shard_sum_host computes either tag on the CPU (nodes without a GPU, single shards).   */
#define GARAGE_EC_SUM_BLAKE2 0
#define GARAGE_EC_SUM_ADLER8 1
int garage_ec_set_sum_kind(garage_ec_ctx *ctx, int kind);
/* How HOST-mode calls of this context wait for the GPU: 0 (default) = cudaStreamSynchronize, the driver
 * spins on a CPU (lowest latency); 1 = block on an event, the waiting thread sleeps.  For callers that
 * keep several calls in flight from a small CPU budget -- the batching dispatchers in front of
 * rpc_put_block: three spinning waiters are three of the ~12 CPUs a host has per GPU.                   */
int garage_ec_set_wait_mode(garage_ec_ctx *ctx, int blocking);
int garage_ec_shard_sum_host(int kind, const uint8_t *data, size_t len, uint8_t out32[32]);
/* Check one half of a shard (a ranged read, half_bytes = shard_len/2 bytes, which = 0 for the a-half, 1 for the
 * b-half) against the shard's stored adler8 tag: with shard_len % 128 == 0 a half is exactly 4 of the 8 segments.
 * 0 if the 4 Adler-32 values match, 1 if not; GARAGE_EC_E_INVALID for GARAGE_EC_SUM_BLAKE2 (a whole-shard hash)
 * and for shard_len % 128 != 0.                                                                                   */
int garage_ec_check_shard_half_host(int kind, const uint8_t *half_bytes, uint32_t shard_len, int which,
                                    const uint8_t tag32[32]);
/* The part of a shard's tag that proves the run [off, off + len) of a shard_len-byte shard: *span_off / *span_len =
 * the smallest run of whole adler8 segments covering it (GARAGE_EC_SUM_ADLER8; segments of
 * roundup16(ceil(shard_len/8)) bytes, the last one cut at shard_len; len = 0: an empty span at off), or the whole
 * shard (GARAGE_EC_SUM_BLAKE2).  GARAGE_EC_E_INVALID for an unknown kind or off + len > shard_len.
 * garage_ec_check_shard_span_host checks such a span (`bytes` = its span_len bytes) against the shard's 32-byte
 * tag: 0 if every covered segment (BLAKE2: the shard's hash) matches, 1 if not; GARAGE_EC_E_INVALID for a span that
 * is not whole segments (BLAKE2: not the whole shard).                                                            */
int garage_ec_tag_span(int kind, uint32_t shard_len, uint32_t off, uint32_t len, uint32_t *span_off, uint32_t *span_len);
int garage_ec_check_shard_span_host(int kind, const uint8_t *bytes, uint32_t shard_len, uint32_t span_off,
                                    uint32_t span_len, const uint8_t tag32[32]);

/* ---- BLOCK-LEVEL convenience (host memory only) -----------------------------------------
 * What rpc_put_block hands over is a contiguous block (bytes::Bytes), not shards.  These do
 * the framing (split + zero pad, src/api/s3/put.rs:583-617 block sizes) on the way to the
 * GPU so the Rust side needs no extra copy.
 *   blocks[s]     : block_len[s] bytes (host)
 *   parity_out    : n * m * stride bytes (host), row i of block s at (s*m + i) * stride.
 *                   The k data shards are just the slices block[j*L .. (j+1)*L) with
 *                   L = garage_ec_shard_len(block_len, k) (zero padded), so they never
 *                   cross PCIe back: Rust sends those slices of the original Bytes.
 *   stride        : >= garage_ec_shard_len(max block_len, k), multiple of 16               */
int garage_ec_encode_blocks(garage_ec_ctx *ctx, const uint8_t *const *blocks,
                            const uint32_t *block_len, size_t n_blocks, uint8_t *parity_out,
                            size_t stride);
/* same, and also returns the blake2sum of every shard (k data then m parity per block,
 * sums_out = n * (k+m) * 32 bytes), computed while the shards are on the device (row f2).   */
int garage_ec_encode_blocks_with_sums(garage_ec_ctx *ctx, const uint8_t *const *blocks,
                                      const uint32_t *block_len, size_t n_blocks,
                                      uint8_t *parity_out, uint8_t *sums_out, size_t stride);
/* inverse for GET: shards (host, shard layout) + present -> blocks_out[s] (block_len[s]
 * bytes each).  Runs reconstruct only for stripes with an absent data shard.               */
int garage_ec_decode_blocks(garage_ec_ctx *ctx, const uint8_t *shards, const uint8_t *present,
                            const uint32_t *block_len, size_t n_blocks, size_t stride,
                            uint8_t *const *blocks_out, int32_t *status);

/* ---- RANGED READS -- call sites: body_from_blocks_range (S3 GetObject with a Range header, src/api/s3/get.rs:650-743)
 * and UploadPartCopy with x-amz-copy-source-range (src/api/s3/copy.rs:396-469, 511-540): bytes [offset, offset + len)
 * of a block, reading only the shards and columns they need (DESIGN.md section 2.5).  Block byte o is byte o % L of
 * data shard o / L, L = garage_ec_code_shard_len.  A range whose touched data shards are all present needs their
 * range bytes only, and no GPU.  Otherwise the absent touched data shards are rebuilt over one window [w0, w0 + w):
 * the smallest 16-byte aligned interval covering the window coordinates of the range's bytes in them -- c for RS and
 * LRC, c mod L/2 for PB, c mod L/alpha for Clay (a range that wraps round a half / layer, or spans two absent shards
 * across their boundary, may widen it to the whole half / layer / shard) -- of every half (PB) or layer (Clay).
 *
 * garage_ec_range_plan (host only, one request): the byte runs a gatherer fetches, in the format, order and merge
 * rule of garage_ec_read_ranges (overlapping runs are merged too): the range bytes of the present touched data
 * shards, and, if a touched data shard is absent, the runs the code's own plan names for want = the absent touched
 * data shards, cut to the window (RS / LRC: garage_ec_read_set shards; PB: garage_ec_read_plan halves; Clay: the
 * repair layers of garage_ec_read_ranges when that shard is the only absent one, else every layer of the first k
 * present shards).  *needs_gpu (nullable) = 1 iff a touched data shard is absent.  GARAGE_EC_E_INVALID for
 * offset + len > block_len or more than cap runs; GARAGE_EC_E_UNRECOVERABLE if the absent touched data shards cannot
 * be rebuilt.  A Clay range of a layer (L/alpha bytes) or more in an absent shard costs a whole-shard repair.
 *
 * garage_ec_decode_range: n requests on the shard layout (stride rules of reconstruct; only the planned runs need
 * hold valid bytes).  block_len / offset / len: n values each.  Request s writes its len[s] bytes at
 * out + s*out_stride; status (nullable, n int32): 0, GARAGE_EC_E_UNRECOVERABLE (nothing written) or -- DEVICE --
 * GARAGE_EC_E_INVALID for offset + len > block_len or a shard length past `stride`.
 *   DEVICE: all pointers device memory; out 16-byte aligned, out_stride a multiple of 16 >= roundup16(len[s]), bytes
 *           [len, roundup16(len)) of a request are written as zero.  Only kernels and stream-ordered scratch of about
 *           n*(k+m)*stride bytes are enqueued (capturable in a CUDA graph).  shards is never written.
 *   HOST:   synchronous; any output alignment.  Uploads only the planned window runs, packed into sub-stripes,
 *           downloads only the rebuilt range bytes; present range bytes are copied on the host.  GARAGE_EC_E_INVALID
 *           before any GPU work for an invalid request; GARAGE_EC_E_UNRECOVERABLE if any request was.
 * garage_ec_decode_range_stripes: the HOST gather form -- stripe s at stripes[s] (its k+m shards `stride` apart),
 * request s writes at outs[s] -- as garage_ec_reconstruct_stripes is to garage_ec_reconstruct.                     */
int garage_ec_range_plan(const garage_ec_ctx *ctx, const uint8_t *present, uint32_t block_len, uint32_t offset,
                         uint32_t len, garage_ec_range *ranges, size_t cap, size_t *n_ranges, int *needs_gpu);
int garage_ec_decode_range(garage_ec_ctx *ctx, const uint8_t *shards, const uint8_t *present, const uint32_t *block_len,
                           const uint32_t *offset, const uint32_t *len, size_t stride, uint8_t *out, size_t out_stride,
                           int32_t *status, size_t n, int mem_kind, void *cuda_stream);
int garage_ec_decode_range_stripes(garage_ec_ctx *ctx, const uint8_t *const *stripes, const uint8_t *present,
                                   const uint32_t *block_len, const uint32_t *offset, const uint32_t *len, size_t stride,
                                   uint8_t *const *outs, int32_t *status, size_t n);

/* ---- TRANSCODE -- changing a cluster's code (DESIGN.md section 2.3): resync after an `erasure_coding` config change
 * rewrites every block stored under an old code -- a whole-block replica (src = NULL), RS, LRC or PB -- under the
 * configured one.  A block under code S is the first block_len bytes of S's data shards concatenated; the output is
 * exactly dst's encode of that block: data shard j = block bytes [j*L_d, (j+1)*L_d) zero padded, L_d =
 * garage_ec_code_shard_len(dst, block_len), and dst's own parities.
 *   src_shards  : shard layout of `src` (stride src_stride); src = NULL: block s at s*src_stride
 *   src_present : n*(k_s+m_s) bytes, nullable (= all present); must be NULL when src = NULL.  A stripe with an absent
 *                 data shard first has it rebuilt by src's own plan (garage_ec_read_plan: only those pieces are read)
 *   block_len   : n values
 *   dst_shards  : shard layout of `dst` (stride dst_stride).  Nothing is written past roundup16(L_d) of a shard
 *   dst_sums    : nullable; (k_d+m_d)*32 bytes per stripe, dst's tag kind (garage_ec_set_sum_kind) of every shard
 *   status      : n int32, nullable: 0; GARAGE_EC_E_UNRECOVERABLE (the source stripe cannot be rebuilt: its destination
 *                 shards are not written); GARAGE_EC_E_INVALID (PB geometry, DESIGN.md section 2.2, or -- DEVICE mode --
 *                 a length that does not fit its stride: nothing written)
 * Strides follow the shard-layout rules of each code.  GARAGE_EC_E_INVALID before any CUDA call for dst = NULL,
 * contexts on different devices, a stride too small for a block (HOST mode) or a length past 32 bits.
 * DEVICE: all pointers device memory of dst's GPU; enqueues only kernels and stream-ordered allocations on `stream`
 * (capturable in a CUDA graph).  The absent source data shards of src_shards are OVERWRITTEN with their rebuilt bytes,
 * as garage_ec_reconstruct does.  dst_sums of a failed stripe is unspecified.
 * HOST: all pointers host; uploads only what the source plan reads, never writes src_shards, downloads the destination
 * shards and tags of the stripes that converted; returns GARAGE_EC_E_UNRECOVERABLE if any stripe failed.           */
int garage_ec_transcode(garage_ec_ctx *dst, garage_ec_ctx *src, uint8_t *src_shards, const uint8_t *src_present,
                        const uint32_t *block_len, size_t src_stride, uint8_t *dst_shards, size_t dst_stride,
                        uint8_t *dst_sums, int32_t *status, size_t n_stripes, int mem_kind, void *cuda_stream);

/* ---- SSE-C -- call sites: the "Encrypt and hash (blake2) block" stage of PutObject (src/api/s3/put.rs:441-466:
 * EncryptionParams::encrypt_block, then blake2sum) and EncryptionParams::get_block (src/api/s3/encryption.rs:269-279,
 * DecryptStream, encryption.rs:431-540).  DESIGN.md section 2.6 is normative.  A plain block P of len bytes sealed
 * under a 32-byte key K and an 8-byte nonce prefix N is B = N || C_0 || ... || C_{n-1}, n = max(1, ceil(len/4096)),
 * C_c = AES-256-GCM(K, nonce = N || LE32(c | (c == n-1) << 31), aad = empty, P[4096c, min(4096(c+1), len))) =
 * ciphertext || 16-byte tag: aead's StreamLE31 over Garage's 4096-byte chunks.  sealed_len = 8 + len + 16n.  The stored
 * block is B: its content address is blake2sum(B), and data shard j = B[jL, (j+1)L) zero padded, L =
 * garage_ec_code_shard_len(sealed_len), so every other call of this header works on it unchanged.
 * Keys are secrets: the library's device and pinned copies of keys and key schedules are zeroed before a HOST call
 * returns and before the stream work of a DEVICE call ends, and no key reaches garage_ec_last_error.
 *
 * garage_ec_sealed_len: 8 + plain_len + 16 * max(1, ceil(plain_len / 4096)); GARAGE_EC_E_INVALID past 32 bits.
 *
 * garage_ec_seal: block s is plain_len[s] bytes at plain + s*plain_stride (plain_stride a multiple of 16 >= every
 * plain_len; the whole row may be read).  keys / nonces: 32 / 8 bytes per block, or both NULL: B = P (Garage's
 * Plaintext).  shards (shard layout, k+m shards per block) gets exactly the context's encode of B -- nothing is written
 * past roundup16(L) of a shard --, hashes[32 s] = blake2sum(B), sums (nullable) the context's tag of every shard, as
 * garage_ec_encode_blocks_with_sums.  DEVICE: all pointers device memory (plain_len 4-byte, hashes and sums 8-byte
 * aligned); only kernels and stream-ordered scratch are enqueued (capturable in a CUDA graph); a block whose L exceeds
 * `stride` or whose plain_len exceeds plain_stride is malformed: nothing of its shards is written and its hash and tags
 * are unspecified.  HOST: synchronous, GARAGE_EC_E_INVALID before any GPU work for such a block; downloads
 * roundup16(L) bytes of all k+m shards.  garage_ec_seal_blocks is the HOST gather form: block s at blocks[s].
 *
 * garage_ec_open: the inverse for stored blocks (shard layout, present: n*(k+m) bytes, sealed_len / hashes / keys: n
 * values).  Absent data shards are rebuilt by the code's own plan, reading only what garage_ec_read_set names for the
 * data shards (HOST: only those and the present data shards are uploaded; DEVICE: the absent data shards of `shards`
 * are OVERWRITTEN with their rebuilt bytes).  hash_bad[s] = 1 iff blake2sum(B) != hashes[s].  Every chunk's tag is
 * checked.  status[s]: 0; GARAGE_EC_E_UNRECOVERABLE; GARAGE_EC_E_AUTH for a failed tag or a sealed_len the framing cannot
 * hold (< 24, or (sealed_len - 8) mod 4112 in 1..15); DEVICE only: GARAGE_EC_E_INVALID for an L past `stride` or a
 * plaintext past plain_stride.  Only a block with status 0 and hash_bad 0 has its plaintext written (at plain +
 * s*plain_stride; DEVICE writes zeros up to roundup16 of its length) and plain_len_out[s] set.  keys is required.
 * DEVICE: as for seal (sealed_len and plain_len_out 4-byte, status 4-byte, hashes 8-byte aligned).  HOST: synchronous;
 * GARAGE_EC_E_INVALID before any GPU work for an L past `stride` or a plaintext past plain_stride; returns
 * GARAGE_EC_E_UNRECOVERABLE if any block was, else GARAGE_EC_E_AUTH if any block failed authentication; hash_bad does not
 * fail the call.  garage_ec_open_stripes is the HOST gather form: stripe s at stripes[s] (its k+m shards `stride`
 * apart), plaintext s written to plains[s] (room for sealed_len[s] - 24 bytes suffices).                            */
int garage_ec_sealed_len(uint32_t plain_len, uint32_t *sealed_len);
int garage_ec_seal(garage_ec_ctx *ctx, const uint8_t *plain, size_t plain_stride, const uint32_t *plain_len,
                   const uint8_t *keys, const uint8_t *nonces, uint8_t *shards, size_t stride, uint8_t *hashes,
                   uint8_t *sums, size_t n, int mem_kind, void *cuda_stream);
int garage_ec_seal_blocks(garage_ec_ctx *ctx, const uint8_t *const *blocks, const uint32_t *plain_len, const uint8_t *keys,
                          const uint8_t *nonces, uint8_t *shards, size_t stride, uint8_t *hashes, uint8_t *sums, size_t n);
int garage_ec_open(garage_ec_ctx *ctx, uint8_t *shards, const uint8_t *present, const uint32_t *sealed_len,
                   const uint8_t *hashes, const uint8_t *keys, uint8_t *plain, size_t plain_stride,
                   uint32_t *plain_len_out, uint8_t *hash_bad, int32_t *status, size_t stride, size_t n, int mem_kind,
                   void *cuda_stream);
int garage_ec_open_stripes(garage_ec_ctx *ctx, uint8_t *const *stripes, const uint8_t *present, const uint32_t *sealed_len,
                           const uint8_t *hashes, const uint8_t *keys, uint8_t *const *plains, uint32_t *plain_len_out,
                           uint8_t *hash_bad, int32_t *status, size_t stride, size_t n);

/* ---- SSE-C RANGED OPEN -- call sites: body_from_blocks_range (src/api/s3/get.rs:650-743) and UploadPartCopy with a
 * source range (src/api/s3/copy.rs:396-469, 511-540) when the object is SSE-C, through EncryptionParams::get_block:
 * plaintext bytes [offset, offset + len) of a sealed block, proven from the chunks they touch and the nonce prefix
 * alone (DESIGN.md section 2.7 is normative).  A block sealed to S bytes has n = (S - 8 + 4111) / 4112 chunks and
 * P = S - 8 - 16n plaintext bytes; the range touches chunks c0 = offset / 4096 .. c1 = (offset + len - 1) / 4096 and needs
 * the prefix B[0, 8) and the span B[8 + 4112 c0, min(S, 8 + 4112 (c1 + 1))).  Chunk c is opened under nonce
 * N || LE32(c | (c == n-1) << 31).  What a ranged open proves: every touched chunk is the authentic chunk c of a block
 * sealed under this key with this N.  It does not prove that untouched chunks are intact or that the block still
 * hashes to its address (the deep scrub does).
 *
 * garage_ec_sealed_range (host only): *span_off / *span_len, *c0 and *n_chunks = c1 - c0 + 1 of one range; an empty
 * range touches nothing (n_chunks = span_len = 0, span_off = min(S, 8 + 4112 * (offset / 4096))).  GARAGE_EC_E_AUTH for
 * an S the framing cannot hold (as garage_ec_open), GARAGE_EC_E_INVALID for offset + len > P.
 *
 * garage_ec_open_range_plan (host only, one request): the byte runs a gatherer fetches, in garage_ec_range_plan's
 * format and merge rule: its runs for the prefix and for the span, merged.  Nothing for an empty range.  *needs_gpu
 * (nullable) = 1 iff a data shard the prefix or the span touches is absent.  Errors as garage_ec_sealed_range, then as
 * garage_ec_range_plan.
 *
 * garage_ec_open_range: n requests on the shard layout (stride rules of reconstruct; only the planned runs need hold
 * valid bytes; shards is never written).  sealed_len / offset / len: n values; keys: 32 bytes per request.  Request s
 * writes its len[s] plaintext bytes at out + s*out_stride only if every chunk it touches passed its tag.  status (n
 * int32, required): 0; GARAGE_EC_E_UNRECOVERABLE; GARAGE_EC_E_AUTH (a touched chunk's tag or the prefix fails, or S is
 * malformed); DEVICE only: GARAGE_EC_E_INVALID for a range past P, an L past `stride` or roundup16(len) past
 * out_stride.  An empty range of a well-framed block is status 0 and writes nothing.
 *   DEVICE: all pointers device memory; out 16-byte aligned, out_stride a multiple of 16, bytes [len, roundup16(len))
 *           written as zero; sealed_len / offset / len / status 4-byte aligned.  Only kernels and stream-ordered
 *           scratch of about 2n((k+m)*stride + out_stride) bytes are enqueued (capturable in a CUDA graph).
 *   HOST:   synchronous; any output alignment.  GARAGE_EC_E_INVALID before any GPU work for a range past P or an L past
 *           `stride`.  Uploads only the planned runs (present span and prefix bytes too: they are ciphertext),
 *           downloads only the len plaintext bytes; returns GARAGE_EC_E_UNRECOVERABLE if any request was, else
 *           GARAGE_EC_E_AUTH if any request failed authentication.
 * Key schedules and the library's copies of keys are zeroed as for garage_ec_open.  garage_ec_open_range_stripes is
 * the HOST gather form: stripe s at stripes[s] (its k+m shards `stride` apart), request s writes at outs[s].          */
int garage_ec_sealed_range(uint32_t sealed_len, uint32_t offset, uint32_t len, uint32_t *span_off, uint32_t *span_len,
                           uint32_t *c0, uint32_t *n_chunks);
int garage_ec_open_range_plan(const garage_ec_ctx *ctx, const uint8_t *present, uint32_t sealed_len, uint32_t offset,
                              uint32_t len, garage_ec_range *ranges, size_t cap, size_t *n_ranges, int *needs_gpu);
int garage_ec_open_range(garage_ec_ctx *ctx, const uint8_t *shards, const uint8_t *present, const uint32_t *sealed_len,
                         const uint8_t *keys, const uint32_t *offset, const uint32_t *len, size_t stride, uint8_t *out,
                         size_t out_stride, int32_t *status, size_t n, int mem_kind, void *cuda_stream);
int garage_ec_open_range_stripes(garage_ec_ctx *ctx, const uint8_t *const *stripes, const uint8_t *present,
                                 const uint32_t *sealed_len, const uint8_t *keys, const uint32_t *offset,
                                 const uint32_t *len, size_t stride, uint8_t *const *outs, int32_t *status, size_t n);

/* ---- SSE-C RESEAL -- call sites: CopyObject with re-encryption (handle_copy_reencrypt, src/api/s3/copy.rs:320-349,
 * through save_stream's block loop) and UploadPartCopy with an encrypted source or destination (copy.rs:506-636, one
 * call per Defragmenter output) when the destination is SSE-C: stored source blocks are opened and their plaintext,
 * cut into pieces, is sealed into new blocks under new keys, without the plaintext ever leaving the chunk kernel's
 * registers and shared memory (DESIGN.md section 2.8 is normative).
 *
 * Sources: n_src stored blocks (shard layout, present: n_src*(k+m) bytes, src_len = the stored length S_i, src_hashes
 * the content addresses).  src_keys: 32 bytes per source, or NULL: every source is Garage Plaintext (P_i = B_i).
 * Destinations: destination d is the pieces [piece_start[d], piece_start[d+1]) of `pieces` (piece_start has n_dst + 1
 * entries); piece {src, offset, len} is plaintext bytes P_src[offset, offset + len), and Q_d is the concatenation of
 * d's pieces.  B'_d = the seal (garage_ec_seal) of Q_d under dst_keys[32 d] and dst_nonces[8 d]; both are required.
 *
 * Every source is proven whole as garage_ec_open proves a block: absent data shards rebuilt by the code's own plan,
 * src_hash_bad[i] = blake2sum(B_i) != src_hashes[i], every chunk tag of a keyed source checked; src_status[i] = 0,
 * GARAGE_EC_E_UNRECOVERABLE, GARAGE_EC_E_AUTH (a tag or the framing), or (DEVICE) GARAGE_EC_E_INVALID (L past stride).
 * Destination d is written only if every source it names has status 0 and hash_bad 0: dst_shards gets exactly the
 * context's encode of B'_d (nothing past roundup16(L') of a shard), dst_hashes[32 d] = blake2sum(B'_d), dst_sums
 * (nullable) its shard tags and dst_len_out[d] = len(B'_d).  Otherwise no byte of its shards is written, its hash and
 * tags are unspecified, and status[d] = GARAGE_EC_E_UNRECOVERABLE if a named source is unrecoverable or does not hash
 * to its address, else GARAGE_EC_E_AUTH, else (DEVICE) GARAGE_EC_E_INVALID for an empty piece list, an empty piece, a
 * piece past its source's plaintext or an L' past `stride`.  n_dst == 0 does nothing.
 *   DEVICE: all pointers device memory; shards 16-byte aligned, src_len / pieces / piece_start / dst_len_out / the
 *           status arrays 4-byte, hashes and sums 8-byte aligned.  Absent source data shards are OVERWRITTEN with their
 *           rebuilt bytes.  Only kernels and stream-ordered scratch are enqueued (capturable in a CUDA graph).
 *   HOST:   synchronous.  GARAGE_EC_E_INVALID before any GPU work for a bad piece list, a source no piece names, a
 *           piece past its source's plaintext, or an L or L' past `stride`.  Destinations are staged in chunks; each uploads only the source
 *           bytes garage_ec_open would upload for the sources its pieces name (ciphertext: no plaintext crosses PCIe)
 *           and downloads roundup16(L') bytes of the k+m shards of its destinations that passed.  Returns
 *           GARAGE_EC_E_UNRECOVERABLE if any destination was, else GARAGE_EC_E_AUTH if any failed authentication.
 * Key schedules and the library's copies of keys are zeroed as for garage_ec_open.  garage_ec_reseal_stripes is the
 * HOST gather form: source stripe i at src_stripes[i] (its k+m shards `stride` apart).                              */
typedef struct garage_ec_piece {
    uint32_t src, offset, len;
} garage_ec_piece;
int garage_ec_reseal(garage_ec_ctx *ctx, uint8_t *src_shards, const uint8_t *src_present, const uint32_t *src_len,
                     const uint8_t *src_hashes, const uint8_t *src_keys, size_t n_src, const garage_ec_piece *pieces,
                     const uint32_t *piece_start, const uint8_t *dst_keys, const uint8_t *dst_nonces,
                     uint8_t *dst_shards, uint8_t *dst_hashes, uint8_t *dst_sums, uint32_t *dst_len_out,
                     uint8_t *src_hash_bad, int32_t *src_status, int32_t *status, size_t stride, size_t n_dst,
                     int mem_kind, void *cuda_stream);
int garage_ec_reseal_stripes(garage_ec_ctx *ctx, uint8_t *const *src_stripes, const uint8_t *src_present,
                             const uint32_t *src_len, const uint8_t *src_hashes, const uint8_t *src_keys, size_t n_src,
                             const garage_ec_piece *pieces, const uint32_t *piece_start, const uint8_t *dst_keys,
                             const uint8_t *dst_nonces, uint8_t *dst_shards, uint8_t *dst_hashes, uint8_t *dst_sums,
                             uint32_t *dst_len_out, uint8_t *src_hash_bad, int32_t *src_status, int32_t *status,
                             size_t stride, size_t n_dst);

/* ---- SSE-C CHECKSUMS -- call sites: the Checksummer of PutObject / UploadPart (src/api/s3/put.rs:413-437,
 * checksum.rs) for an SSE-C object whose checksum is CRC32 or CRC32C, and of CopyObject / UploadPartCopy into an SSE-C
 * destination (copy.rs:76-79, 143-147, 507-508, 656-658): the S3 checksum of each block's plaintext, computed in the
 * chunk kernel from the plaintext it already holds, so that it never reaches host memory (DESIGN.md section 2.9 is
 * normative).  Kinds, one byte per block: GARAGE_EC_CRC_NONE, GARAGE_EC_CRC_CRC32 (zlib's CRC-32, reflected 0xEDB88320)
 * or GARAGE_EC_CRC_CRC32C (Castagnoli, reflected 0x82F63B78); both init and final XOR 0xFFFFFFFF, the CRC of the empty
 * string 0.  A batch may mix kinds.  S3 stores the value as its 4 big-endian bytes.
 *
 * garage_ec_seal_crc / garage_ec_seal_blocks_crc: garage_ec_seal / garage_ec_seal_blocks plus crc_kind (n bytes, NULL:
 * no checksums) and crcs (n uint32, required when crc_kind is not NULL).  crcs[s] = the CRC of plaintext block s for
 * every block with a kind that is written, 0 for every other block; all other outputs are byte-identical to the call
 * without checksums.  A kind above GARAGE_EC_CRC_CRC32C is refused as the other per-block input errors are: HOST
 * returns GARAGE_EC_E_INVALID before any GPU work, DEVICE treats the block as malformed (nothing of its shards is
 * written).  DEVICE: crc_kind and crcs are device memory, crcs 4-byte aligned; still only kernels and stream-ordered
 * scratch (one 32-bit accumulator per block) are enqueued.  HOST: uploads n more bytes and downloads 4n more.
 *
 * garage_ec_reseal_crc / garage_ec_reseal_stripes_crc: the reseal calls with the same two arguments, indexed by
 * destination: crcs[d] = the CRC of Q_d for a destination with a kind that passes (dst_len_out[d] set); unspecified
 * otherwise.  An unknown kind: HOST GARAGE_EC_E_INVALID before any GPU work; DEVICE status[d] = GARAGE_EC_E_INVALID.
 *
 * garage_ec_crc_combine (host only, no device): *out = CRC(A || B) from crc_a = CRC(A), crc_b = CRC(B) and len_b =
 * |B| (zlib's crc32_combine; len_b = 0 gives crc_a) -- how a caller folds block checksums into a part's or an
 * object's.  GARAGE_EC_E_INVALID for a kind other than CRC32 / CRC32C or a NULL out.                                */
#define GARAGE_EC_CRC_NONE 0
#define GARAGE_EC_CRC_CRC32 1
#define GARAGE_EC_CRC_CRC32C 2
int garage_ec_seal_crc(garage_ec_ctx *ctx, const uint8_t *plain, size_t plain_stride, const uint32_t *plain_len,
                       const uint8_t *keys, const uint8_t *nonces, uint8_t *shards, size_t stride, uint8_t *hashes,
                       uint8_t *sums, const uint8_t *crc_kind, uint32_t *crcs, size_t n, int mem_kind, void *cuda_stream);
int garage_ec_seal_blocks_crc(garage_ec_ctx *ctx, const uint8_t *const *blocks, const uint32_t *plain_len,
                              const uint8_t *keys, const uint8_t *nonces, uint8_t *shards, size_t stride, uint8_t *hashes,
                              uint8_t *sums, const uint8_t *crc_kind, uint32_t *crcs, size_t n);
int garage_ec_reseal_crc(garage_ec_ctx *ctx, uint8_t *src_shards, const uint8_t *src_present, const uint32_t *src_len,
                         const uint8_t *src_hashes, const uint8_t *src_keys, size_t n_src, const garage_ec_piece *pieces,
                         const uint32_t *piece_start, const uint8_t *dst_keys, const uint8_t *dst_nonces,
                         uint8_t *dst_shards, uint8_t *dst_hashes, uint8_t *dst_sums, uint32_t *dst_len_out,
                         uint8_t *src_hash_bad, int32_t *src_status, int32_t *status, const uint8_t *crc_kind,
                         uint32_t *crcs, size_t stride, size_t n_dst, int mem_kind, void *cuda_stream);
int garage_ec_reseal_stripes_crc(garage_ec_ctx *ctx, uint8_t *const *src_stripes, const uint8_t *src_present,
                                 const uint32_t *src_len, const uint8_t *src_hashes, const uint8_t *src_keys, size_t n_src,
                                 const garage_ec_piece *pieces, const uint32_t *piece_start, const uint8_t *dst_keys,
                                 const uint8_t *dst_nonces, uint8_t *dst_shards, uint8_t *dst_hashes, uint8_t *dst_sums,
                                 uint32_t *dst_len_out, uint8_t *src_hash_bad, int32_t *src_status, int32_t *status,
                                 const uint8_t *crc_kind, uint32_t *crcs, size_t stride, size_t n_dst);
int garage_ec_crc_combine(int kind, uint32_t crc_a, uint32_t crc_b, uint64_t len_b, uint32_t *out);

/* ---- utilities used by the harness ------------------------------------------------------
 * device-side synthetic data (same splitmix64 counter stream as the oracle's
 * generator): fills dst[0..len) (device) with stream bytes at `offset`
 * (len, offset multiples of 8).                                                            */
int garage_ec_fill_random(garage_ec_ctx *ctx, uint8_t *dst_device, size_t len, uint64_t seed,
                          uint64_t offset, void *cuda_stream);
/* pinned host memory for block / shard buffers: the Rust side lands the HTTP body copy
 * (BytesBuf::take_exact, src/net/bytes_buf.rs:66-117) directly in such a buffer so the DMA
 * engines can read it.  Pageable memory is accepted everywhere, only slower.               */
int garage_ec_host_alloc(garage_ec_ctx *ctx, void **out, size_t bytes);
/* same, write-combined (cudaHostAllocWriteCombined): for buffers the CPU only WRITES sequentially and the
 * GPU reads (upload landing buffers) or the GPU writes and the CPU hands on without reading; CPU reads
 * from such memory are very slow.  The pages are not snooped during DMA.                              */
int garage_ec_host_alloc_wc(garage_ec_ctx *ctx, void **out, size_t bytes);
/* memcpy into a pinned buffer that the GPU reads next (the landing copy of a PUT body, BytesBuf::take_exact,
 * src/net/bytes_buf.rs:66-117; the survivors of a degraded GET).  Uses non-temporal stores so that the DMA
 * read finds the bytes in DRAM instead of snooping them out of the writing core's cache (7x faster upload
 * of freshly written data on the measured hosts).                                                          */
void garage_ec_copy_for_dma(void *dst_pinned, const void *src, size_t n);
void garage_ec_host_free(garage_ec_ctx *ctx, void *ptr);
/* NUMA placement.  On a multi-socket host each GPU hangs off one socket; garage_ec_host_alloc
 * places its pages on that socket's memory node (preferred-node policy + first touch from a CPU
 * of the node, both restored before returning), so DMA never crosses the inter-socket link.
 * garage_ec_numa_info reports the GPU's node and the node the last garage_ec_host_alloc of this
 * context landed on (-1 = unknown).  garage_ec_bind_thread pins the CALLING thread to the CPUs
 * of the GPU's node -- for the threads that fill those buffers (the batching workers in front of
 * rpc_put_block / the 8 resync workers, src/block/resync.rs:43; spawn_blocking threads,
 * src/block/block.rs:86): returns 0 if bound, 1 if nothing was changed (topology unknown or not
 * permitted).                                                                               */
int garage_ec_numa_info(const garage_ec_ctx *ctx, int *gpu_node, int *last_alloc_node);
int garage_ec_bind_thread(const garage_ec_ctx *ctx);
/* the number of CUDA devices this process sees (cudaGetDeviceCount); 0 if there is none or no driver.  Creates no
 * context: the block manager checks a device list with it before it creates any.                              */
int garage_ec_device_count(void);

/* number of kernel launches issued by this context so far (bench.py's gpu_launches)        */
uint64_t garage_ec_launch_count(const garage_ec_ctx *ctx);
/* per-kernel CUDA-event timing of the RS kernels (encode / reconstruct / verify main
 * kernel, recorded on the stream they were launched on).  garage_ec_timing_read waits for
 * the recorded kernels, adds their durations to *total_ms / *launches and resets.          */
int garage_ec_set_timing(garage_ec_ctx *ctx, int enabled);
int garage_ec_timing_read(garage_ec_ctx *ctx, double *total_ms, uint64_t *launches);

/* test hook: the n_calls-th checked CUDA runtime call issued by this context from now on fails
 * (n_calls = 0: the next one; < 0: off).  Used by the fault-injection tests of the HOST-mode
 * ownership contract: after a failed call returns, nothing may still write the caller's buffers. */
int garage_ec_debug_fail_after(garage_ec_ctx *ctx, long n_calls);

#ifdef __cplusplus
}
#endif
#endif /* GARAGE_EC_H */
