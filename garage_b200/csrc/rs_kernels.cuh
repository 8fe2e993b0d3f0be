// rs_kernels.cuh -- sm_90a kernels of the Garage erasure-coding block path.
//
// What they compute (normative definition: DESIGN.md "Arithmetic"):
//     out[i][t] = XOR_j C[i][j] * src[j][t]         over GF(2^8)/0x11D, byte-wise
// for rows i of a small coefficient matrix C (the parity rows P for encode/verify, a
// per-stripe composed decode matrix for reconstruct) and the k source shards of a stripe.
// Reference call sites this replaces work at: BlockManager::rpc_put_block
// (src/block/manager.rs:366-408), rpc_get_raw_block_internal (manager.rs:276-339),
// BlockResyncManager::resync_block (src/block/resync.rs:460-500), DataBlock::verify /
// ScrubWorker::work (src/block/block.rs:69-83, src/block/repair.rs:438-490).
//
// Design (DESIGN.md "Kernels"):
//  * HBM-bound byte work, no tensor cores.  The per-byte GF multiply-accumulate for up to 4
//    output rows is ONE shared-memory lookup: T_j[x] = {C0j*x, C1j*x, C2j*x, C3j*x} packed in
//    a 32-bit word, so a data byte costs one LDS + one XOR for all four rows.
//  * Conflict-free lookups with small tables ("sub-warp interleaving", mixed group sizes).
//    G tables share one 32 KB group: table `sub` of the group is replicated R = 32/G times in
//    banks [sub*R, sub*R + R) of every 128-byte row x.  The warp is cut in G sub-warps of R
//    lanes; at phase p of the group sub-warp q works on source base + (p xor q), so every
//    sub-warp is in a different table and every lane owns its bank:
//    word = group*8192 + x*32 + (lane xor p*R).  XOR accumulation commutes, so the per-lane
//    source order costs nothing.  k sources are decomposed greedily into groups of 32/16/8/4/2/1
//    tables (no padding lookups): RS(10,4) = one group of 8 + one group of 2 = 64 KB (round 1
//    used uniform G = 2: 160 KB), k = 16 -> 32 KB, k = 32 -> 32 KB.
//  * Two ways to bring a 16-byte column of every source to the lanes (StreamCfg::kTma):
//      LDG  : k x ld.global.nc.v4 per lane straight into registers, the next column's vectors
//             prefetched into a second register set (group size capped at 8 so that a warp
//             instruction still reads >= 64 contiguous bytes per shard);
//      TMA  : one elected lane issues k cp.async.bulk (1-D TMA) copies of 512 bytes -- the
//             warp's 32 columns of each shard -- into the warp's private shared-memory stage
//             and arms the stage's mbarrier with the byte count; the warp waits on the
//             mbarrier, pulls its vectors with conflict-free LDS.128, and immediately re-arms
//             the stage for its next work item, so the copy flies while the lookups run.  No
//             prefetch registers, any lane may read any source row, which is what allows the
//             16- and 32-table groups and k up to 32 at full speed.
//  * Reconstruct (per-stripe matrices) runs WITHOUT block-wide barriers: two table buffers, a
//    builder warp that stages the next stripe's plan and builds its tables while the consumer
//    warps stream the current stripe, mbarriers `full[b]` (tables of buffer b ready) and
//    `empty[b]` (every consumer warp has left the stripe that used buffer b).  Consumer warps
//    claim 32-column chunks from a per-stripe shared counter and flow from stripe to stripe on
//    their own.
//  * log/antilog tables sit in __constant__ memory and are staged to shared memory by the
//    decode-planning kernel; the product tables are built from xtime chains (no log lookups).
//  * Persistent grid: one CTA per SM.  Encode / verify warps with whole-item TMA staging claim their work items
//    from a per-launch counter (StreamCfg::kDynamic); the other uniform shapes keep a fixed stride.
#pragma once
#include <cuda.h>  // CUtensorMap (type only; the encoder is fetched through cudaGetDriverEntryPoint)
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "../../include/garage_ec.h"  // GARAGE_EC_E_* status codes
#include "blake2b.h"
#include "gf256.h"

namespace garage_ec {

// ---- tuning overrides (tools/build_variants.py); -1 = per-shape default -------------------
#ifndef GEC_TMA_ENC
#define GEC_TMA_ENC -1
#endif
#ifndef GEC_TMA_PLAN
#define GEC_TMA_PLAN -1
#endif
#ifndef GEC_TMA_VER
#define GEC_TMA_VER -1
#endif
#ifndef GEC_NW_ENC
#define GEC_NW_ENC 0  // consumer warps; 0 = default
#endif
#ifndef GEC_NW_PLAN
#define GEC_NW_PLAN 0
#endif
#ifndef GEC_NW_VER
#define GEC_NW_VER 0
#endif
#ifndef GEC_TMAP_FROM_K
// uniform modes, TMA path: ONE 2-D tensor copy (k rows x 512 B) per work item instead of k 1-D copies, from this k
// on.  The single copy saves ~7 issue slots per source row, which is what matters for k >= 13, while k <= 12 encode
// is faster with k independent 1-D copies in flight.  0 = never.
#define GEC_TMAP_FROM_K 13
#endif
#define GEC_TMAP (GEC_TMAP_FROM_K > 0)
#ifndef GEC_SPLIT_STAGE
#define GEC_SPLIT_STAGE 1
#endif
#ifndef GEC_LDG_MAXLG
#define GEC_LDG_MAXLG 3  // LDG path: largest table group = 2^3 tables (64 contiguous bytes per shard and instruction)
#endif
#ifndef GEC_TMA_FROM_K
#define GEC_TMA_FROM_K 5  // encode / reconstruct use the TMA staging from this k on (k <= 4 is as fast with LDG)
#endif
#ifndef GEC_CLAIM_RUN
#define GEC_CLAIM_RUN 2  // uniform modes, dynamic schedule: consecutive work items a warp claims at once
#endif
#ifndef GEC_TAIL_PARTS
// reconstruct: the last 2 x (CTAs) stripes of a launch are claimed in this many chunk ranges each, so that the end of
// the launch is shared by every SM instead of the few that claimed the last whole stripes
#define GEC_TAIL_PARTS 4
#endif
#ifndef GEC_NULL_MATH
// 1 = traffic-ceiling build: column_compute skips the table lookups and the transpose and stores XORs of the
// staged source vectors, with loads, stages, barriers, item order and stores unchanged.  Its outputs are WRONG;
// only tools/build_variants.py builds it, to measure what the memory traffic alone allows.
#define GEC_NULL_MATH 0
#endif

constexpr int kMaxK = 32;
constexpr int kMaxM = 8;
constexpr int kRowsPerPass = 4;          // output rows packed in one 32-bit table word
constexpr uint32_t kGroupBytes = 32768;  // one table group: 256 rows x 32 banks x 4 B
constexpr int kMaxGroups = 6;
constexpr uint32_t kStageRowBytes = 512;  // 32 columns x 16 B of one shard
constexpr uint32_t kSmemLimit = 227 * 1024;

enum ApplyMode { kModeEncode = 0, kModePlan = 1, kModeVerify = 2, kModeUnits = 3 };
// kModeUnits (garage_ec_reconstruct_segments, DESIGN.md 4.13) is kModePlan over a list of adler8 units instead of
// stripes: the same launch shape, tables and consumer warps, only the builder addresses a unit
__host__ __device__ constexpr int cfg_mode(int mode) { return mode == kModeUnits ? kModePlan : mode; }

// ---- table layout: k sources -> groups of 2^lg tables ---------------------------------------
struct TabLayout {
    int nslots;   // >= k; slots >= k are zero tables (only when the group budget forces padding)
    int ngroups;  // 32 KB each
    int lg[kMaxGroups];    // log2(tables in the group)
    int base[kMaxGroups];  // first slot of the group
};
// greedy decomposition of the smallest k' >= k that needs <= maxgroups groups of <= 2^maxlg tables
__host__ __device__ constexpr TabLayout make_layout(int k, int maxlg, int maxgroups)
{
    for (int kp = k; kp <= 2 * kMaxK; kp++) {
        TabLayout L{};
        int rem = kp, pos = 0, ng = 0;
        bool ok = true;
        while (rem > 0) {
            int lg = maxlg;
            while ((1 << lg) > rem) lg--;
            if (ng >= kMaxGroups || ng >= maxgroups) {
                ok = false;
                break;
            }
            L.lg[ng] = lg;
            L.base[ng] = pos;
            ng++;
            pos += 1 << lg;
            rem -= 1 << lg;
        }
        if (ok) {
            L.nslots = kp;
            L.ngroups = ng;
            return L;
        }
    }
    return TabLayout{};
}
__host__ __device__ constexpr int slot_group(const TabLayout &L, int u)
{
    int g = 0;
    for (int i = 0; i < L.ngroups; i++)
        if (u >= L.base[i]) g = i;
    return g;
}

// Per-stripe decode plan of one stripe as the streaming kernel needs it (two slots, one per
// table buffer).
struct PlanSlot {
    unsigned long long key_present, key_out;
    uint32_t sid;         // stripe index (>= n: no more work)
    int32_t rows;         // rows to produce in this pass (<= 0: nothing to do)
    uint32_t chunk_next;  // next unclaimed 32-column chunk of this stripe
    uint32_t chunk_end;   // end of the stripe's chunk range claimed in this work unit
    uint32_t len;         // shard_len of the stripe
    uint32_t nsurv;       // sources read; sources >= nsurv are neither fetched nor looked up (zero vectors)
    uint32_t src_off[kMaxK];             // byte offset of source j inside the stripe
    uint32_t dst_off[kRowsPerPass];      // byte offset of output row i inside the stripe
    uint8_t coef[kRowsPerPass * kMaxK];  // coef[i*kMaxK + j]
};
constexpr uint32_t kAuxBytes = 2 * sizeof(PlanSlot) + 8 * (4 + 32) + 64;  // plan slots + mbarriers

// Which way the columns reach the lanes, and how many warps stream, per (k, mode): picked from
// sweeps of both paths x 8..32 warps for k = 4, 6, 8, 10, 12.  What bounds them is per SM and the
// same on every sm_90 part: 227 KB of shared memory per block and 64 K registers.
__host__ __device__ constexpr bool cfg_default_tma(int k, int mode)
{
    if (mode == kModeVerify) return k == 4 || k > 6;  // verify: LDG with prefetch wins for k = 1..3, 5, 6
    // reconstruct of k = 7 (4+2+1: three table groups, 192 KB for two buffers): LDG is faster than TMA with one
    // padded group of 8 and 27 warps
    if (mode == kModePlan && k == 7) return false;
    return k >= GEC_TMA_FROM_K;
}
__host__ __device__ constexpr int cfg_nw_ldg(int k, int mode)
{
    if (mode == kModeVerify) return k <= 4 ? 24 : 16;
    return k <= 4 ? 32 : (k <= 6 ? 24 : (k <= 8 ? 20 : 16));
}
// TMA path, k <= 12: measured optimum (total warps; reconstruct includes the builder warp and is then
// clamped to what the stage memory allows); larger k: by register budget (cfg_nw_tma)
// RS(10,4) encode and reconstruct: 12 warps measured 0.5 % faster than 16 (encode, with the dynamic schedule) and 20
// (reconstruct); 8 warps were slower.  Other k were not re-swept.
__host__ __device__ constexpr int cfg_nw_tma_small(int k, int mode)
{
    if (mode == kModePlan) return k <= 6 ? 32 : (k <= 8 ? 28 : (k == 10 ? 12 : 24));
    if (mode == kModeVerify) return k <= 4 ? 28 : (k <= 8 ? 20 : 16);
    return k <= 8 ? 20 : (k == 10 ? 12 : 16);
}
// TMA: at most 3 table groups per buffer, fewer (= more zero-table padding) when the table buffers
// would not leave room for the stages of `want_nw` warps (reconstruct doubles the tables: k = 7 as
// 4+2+1 is 192 KB of tables and 8 warps, as one padded group of 8 it is 64 KB and 28 warps)
__host__ __device__ constexpr int cfg_tma_groups(int k, int bufs, int stage_rows, int want_nw)
{
    for (int g = 3; g > 1; g--) {
        const TabLayout L = make_layout(k, 5, g);
        if ((uint32_t)bufs * L.ngroups * kGroupBytes + kAuxBytes + (uint32_t)want_nw * stage_rows * kStageRowBytes <= kSmemLimit) return g;
    }
    return 1;
}
__host__ __device__ constexpr int cfg_nw_tma(int regs_est, uint32_t tab_bytes, int stage_rows)
{
    // the register file is split over the 4 sub-partitions of an SM (16384 registers each), so the
    // per-thread budget only changes with ceil(warps / 4): 8 warps 255, 12: 168, 16: 128, 20: 96, 24: 80
    int nw = 8;
    for (int cand = 24; cand > 8; cand -= 4) {
        const int cap = 16384 / (cand / 4 * 32) / 8 * 8;
        if (cap >= regs_est) {
            nw = cand;
            break;
        }
    }
    while (nw > 4 && tab_bytes + kAuxBytes + (uint32_t)nw * stage_rows * kStageRowBytes > kSmemLimit) nw -= 4;
    return nw;
}

__host__ __device__ constexpr int cfg_fit_nw(int nw, uint32_t tab_bytes, int stage_rows, bool builder)
{
    while (nw > 4 && tab_bytes + kAuxBytes + (uint32_t)(nw - (builder ? 1 : 0)) * stage_rows * kStageRowBytes > kSmemLimit) nw -= 4;
    return nw;
}

// ---- launch shape / shared-memory carve-up per (K, MODE), all compile time ------------------
template <int K, int MODE> struct StreamCfg {
    static constexpr int kTmaOverride = MODE == kModeEncode ? GEC_TMA_ENC : (MODE == kModePlan ? GEC_TMA_PLAN : GEC_TMA_VER);
    static constexpr bool kTma = K > 16 || (kTmaOverride >= 0 ? (kTmaOverride != 0) : cfg_default_tma(K, MODE));
    static constexpr int kBufs = MODE == kModePlan ? 2 : 1;  // table buffers
    // reconstruct of k > 16: the stage holds ONE table group's rows (<= 16) at a time and an item is streamed
    // in one phase per group -- with two table buffers a full k x 512 B stage per warp leaves room for only
    // 7 consumer warps (RS(20,4) reconstruct 0.69 of peak)
    // (the same for encode / verify of k > 16: reading all k vectors of a column into registers at once spills)
    static constexpr bool kSplit = kTma && K > 16 && GEC_SPLIT_STAGE;
    static constexpr int kSrcRows = kSplit ? 16 : K;  // source rows of a stage; stored parity rows (verify) follow
    static constexpr int kStageRows = kTma ? kSrcRows + (MODE == kModeVerify ? kRowsPerPass : 0) : 0;
    static constexpr int kNwOverride = MODE == kModeEncode ? GEC_NW_ENC : (MODE == kModePlan ? GEC_NW_PLAN : GEC_NW_VER);

    // LDG: groups of <= 8 tables (>= 64 contiguous bytes per shard and warp instruction), tables
    // <= 192 KB so that >= 32 KB stay L1 (round 1: 224 KB of tables starved the global loads).
    // TMA: groups of <= 32 tables, <= 3 groups per buffer; the loads bypass L1.
    static constexpr int kMaxLg = kSplit ? 4 : (kTma ? 5 : GEC_LDG_MAXLG);
    static constexpr int kMaxGrp = kTma ? cfg_tma_groups(K, kBufs, kStageRows, K <= 12 ? 16 : 8) : 6 / kBufs;
    static constexpr TabLayout kLay = make_layout(K, kMaxLg, kMaxGrp);
    static constexpr int S = kLay.nslots;
    static constexpr uint32_t kTabBytes = (uint32_t)kBufs * kLay.ngroups * kGroupBytes;

    // consumer warps: LDG shapes from the round-1 sweeps (2 x S x 4 registers of column data);
    // TMA: S x 4 registers of column data, capped by the stage memory
    static constexpr int kWarpsDefault =
        !kTma ? cfg_nw_ldg(K, MODE)
              : (K <= 12 ? cfg_fit_nw(cfg_nw_tma_small(K, MODE), kTabBytes, kStageRows, MODE == kModePlan)
                 : (MODE == kModePlan && (K <= 16 || kSplit))
                     ? cfg_fit_nw(16, kTabBytes, kStageRows, true)  // sweep: RS(14,4) 0.81 -> 0.92, RS(16,4) 0.89 -> 0.95
                     : cfg_nw_tma(4 * (kSplit ? 16 : S) + 76, kTabBytes, kStageRows));
    // an override (tuning builds) is clamped to what the stage memory allows
    static constexpr int kWarpsAll =
        kNwOverride > 0 ? (kTma ? cfg_fit_nw(kNwOverride, kTabBytes, kStageRows, MODE == kModePlan) : kNwOverride) : kWarpsDefault;
    // reconstruct: the last warp is the table builder
    static constexpr int kWarps = MODE == kModePlan ? kWarpsAll - 1 : kWarpsAll;  // consumer warps
    // uniform modes: warps claim work items from a counter instead of a fixed stride.  Measured on H100 for
    // k = 4..32: faster with whole-item TMA staging at <= 20 warps (RS(10,4) encode 2.09 -> 1.98 ms), slower with
    // LDG, with 28 warps (k = 4 verify) and with split staging (k > 16), which keep the fixed stride.
    static constexpr bool kDynamic = MODE != kModePlan && kTma && !kSplit && kWarps <= 20;
    static constexpr int kThreads = 32 * kWarpsAll;
    static constexpr uint32_t kStageBytes = (uint32_t)kWarps * kStageRows * kStageRowBytes;
    static constexpr uint32_t kSmem = kTabBytes + kStageBytes + kAuxBytes;
    static_assert(kLay.nslots >= K && kLay.ngroups >= 1, "no table layout for this k");
    static_assert(kSmem <= kSmemLimit, "shared memory budget exceeded");
    static_assert(kThreads <= 1024 && kWarps >= 1, "bad launch shape");
};

// GF(2^8) antilog / log tables, pinned in constant memory.  Kernels that need general products
// (decode planning) stage them into shared memory with warp-UNIFORM 16-byte constant loads:
// a per-lane byte index into __constant__ memory serialises 32-way in the constant cache (the
// first version of the RS plan kernel spent 30 of its 40 us there).
struct GfTables {
    uint8_t exp[512];
    uint8_t log[256];
};
__constant__ __align__(16) GfTables c_gf = {GARAGE_EC_GF_EXP_INIT, GARAGE_EC_GF_LOG_INIT};

__device__ __forceinline__ void stage_gf_tables(uint8_t *s_gf /* 768 B, 16-byte aligned */)
{
    const uint4 *src = reinterpret_cast<const uint4 *>(&c_gf);
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    for (uint32_t i = warp; i < sizeof(GfTables) / 16; i += nwarps) {
        const uint4 v = src[i];  // same address in every lane: one constant-cache broadcast
        if (lane < 4)
            reinterpret_cast<uint32_t *>(s_gf)[i * 4 + lane] = lane == 0 ? v.x : (lane == 1 ? v.y : (lane == 2 ? v.z : v.w));
    }
}

// Per-stripe decode plan, produced by plan_kernel, consumed by rs_apply_kernel<kModePlan>.  Indices are generator
// rows: shards, or PB half-rows q = 2*shard + half.
struct __align__(16) StripePlan {
    unsigned long long key_present;  // bit i: row i present (PB: candidate)
    unsigned long long key_out;      // bit i: row i is rebuilt
    uint8_t nrows;                   // number of rows rebuilt (0..kMaxM)
    uint8_t unrecoverable;           // 1 if a wanted shard cannot be rebuilt
    uint8_t nsurv;                   // sources read: surv[0..nsurv) (k for RS; <= k for LRC, <= 2k for PB)
    uint8_t pad[5];
    uint8_t surv[kMaxK];           // source row indices, ascending (RS: the first k present)
    uint8_t out_idx[kMaxM];        // rebuilt row indices
    uint8_t coef[kMaxM][kMaxK];  // out[r] = XOR_j coef[r][j] * row[surv[j]]
};

// adler8 tag segment length of a len-byte shard (the tag is described with adler8_shards_kernel below)
__host__ __device__ inline uint32_t adler8_seg_bytes(uint32_t len)
{
    return (((len + 7) / 8) + 15) / 16 * 16;
}
// Columns of unit g of a stripe of shard length L (DESIGN.md 2.10): RS and LRC, adler8 segment g,
// [g*S, min(L, (g+1)*S)) with S = adler8_seg_bytes(L); PB (L % 128 == 0), columns [g*L/8, (g+1)*L/8) of each half, which
// are segments g and g+4.  An empty unit has len 0.
__host__ __device__ inline void unit_columns(uint32_t L, uint32_t g, bool pb, uint32_t *base, uint32_t *len)
{
    const uint32_t S = pb ? L / 8 : adler8_seg_bytes(L), a = g * S;
    *base = a;
    *len = pb ? S : (a >= L ? 0u : (L - a < S ? L - a : S));
}
// Is shard i present in unit g, from its seg_present byte b (bit g: segment g holds valid bytes)?  A PB unit needs
// both of its segments; an empty unit is present in every shard.
__host__ __device__ inline bool unit_present(uint8_t b, uint32_t L, uint32_t g, bool pb)
{
    uint32_t base, len;
    unit_columns(L, g, pb, &base, &len);
    if (!len) return true;
    return pb ? ((b >> g) & (b >> (g + 4)) & 1) != 0 : ((b >> g) & 1) != 0;
}

struct ApplyParams {
    const uint8_t *src;            // stripe s source base = src + s*src_pitch
    uint8_t *dst;                  // stripe s output base = dst + s*dst_pitch
    unsigned long long src_pitch;  // bytes
    unsigned long long dst_pitch;
    const uint32_t *shard_len;  // device, nullable (=> stride); encode / verify: a length past the stride is malformed
    const StripePlan *plan;     // kModePlan
    uint32_t *mismatch;         // kModeVerify
    uint32_t *counter;          // dynamic scheduler, zero at launch: stripes (kModePlan) / work items (uniform modes)
    uint32_t stride;            // bytes between shards
    uint32_t n;                 // stripes
    uint32_t k;                 // sources
    uint32_t rows;              // outputs this pass (<= 4), uniform modes
    uint32_t row_off;           // first output row of this pass
    uint32_t items_per_stripe;  // ceil(ceil(stride/16)/32), uniform modes
    uint32_t row_bytes;         // 128: bytes per table row (a register operand keeps x*128 an IMAD)
    uint32_t use_tmap;          // 1: `tmap` is valid (uniform modes, TMA path)
    uint32_t rows_per_stripe;   // shards per stripe in `src` (k for encode, k+m for verify): tensor row of (s, j) = s*rows_per_stripe + j
    uint32_t half;              // kModePlan, PB contexts: plan indices are half-rows q = 2*shard + half (DESIGN.md 2.2)
    uint8_t coef[kRowsPerPass * kMaxK];  // uniform modes: coef[i*k + j]
    // kModeUnits: units[0] = work units, units[1 + w] = unit id s*U + g (U = 8, PB: 4); plan is per unit id.  It sits
    // in the padding before `tmap`, so the parameter block of the other modes keeps its size
    const uint32_t *units;
    // 2-D view of `src` for TMA: dim0 = stride/4 uint32 elements, dim1 = n*rows_per_stripe shards
    // (pitch `stride`), box = 128 elements (512 B = 32 columns) x k rows
    alignas(64) CUtensorMap tmap;
};
static_assert(sizeof(ApplyParams) == 384, "ApplyParams layout");

// ------------------------------------------------------------------ small device helpers
template <int I, int N, class F> __device__ __forceinline__ void static_for(F &&f)
{
    if constexpr (I < N) {
        f(std::integral_constant<int, I>{});
        static_for<I + 1, N>(f);
    }
}

__device__ __forceinline__ uint4 ldg_stream(const void *p)
{
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}
__device__ __forceinline__ void stg_stream(void *p, const uint4 &v)
{
    asm volatile("st.global.cs.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
                 "r"(v.w)
                 : "memory");
}
__device__ __forceinline__ uint32_t lds_u32(uint32_t addr)
{
    uint32_t r;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(r) : "r"(addr));
    return r;
}
__device__ __forceinline__ uint4 lds_v4(uint32_t addr)
{
    uint4 r;
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(addr) : "memory");
    return r;
}
// zero the bytes at positions >= nbytes (0 < nbytes < 16) of a 16-byte vector
__device__ __forceinline__ uint4 mask_tail(uint4 v, uint32_t nbytes)
{
    uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const int lo = 4 * i;
        if ((int)nbytes <= lo) w[i] = 0;
        else if ((int)nbytes < lo + 4) w[i] &= 0xffffffffu >> (8 * (lo + 4 - (int)nbytes));
    }
    return make_uint4(w[0], w[1], w[2], w[3]);
}

// ---- mbarrier + 1-D bulk async copy (TMA) ----------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init()
{
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity)
{
    asm volatile(
        "{\n"
        ".reg .pred P1;\n"
        "GEC_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
        "@P1 bra GEC_DONE;\n"
        "bra GEC_WAIT;\n"
        "GEC_DONE:\n"
        "}" ::"r"(bar),
        "r"(parity)
        : "memory");
}
// global -> this CTA's shared memory, completion counted in bytes on `bar`
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
                 "l"(src), "r"(bytes), "r"(bar)
                 : "memory");
}

// A warp reads its stage with LDS (generic proxy) and lane 0 then refills it with TMA (async proxy).  __syncwarp
// alone does not order the two proxies: the refill could overwrite rows whose LDS had not been serviced yet (seen
// on H100 as wrong parity in a few 32-column chunks of large encode / verify batches).  Every lane fences its reads
// against the async proxy before the warp lets lane 0 re-arm the stage.
__device__ __forceinline__ void stage_release()
{
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncwarp();
}

// 2-D tiled TMA: box (128 uint32 x K rows) at element column c0, row c1 of the tensor described by
// `tmap` -> dst (row r at dst + r*512); completes 512*K bytes on `bar` (also when the box sticks
// out of the tensor: out-of-bounds elements are filled with zeros and still counted)
__device__ __forceinline__ void tensor_g2s_2d(uint32_t dst, const CUtensorMap *tmap, uint32_t c0, uint32_t c1, uint32_t bar)
{
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(dst),
                 "l"(reinterpret_cast<uint64_t>(tmap)), "r"(c0), "r"(c1), "r"(bar)
                 : "memory");
}

// 4x4 byte transpose: a[p] holds {row0,row1,row2,row3} bytes of byte column p;
// returns r[i] = bytes of row i for columns 0..3.
__device__ __forceinline__ void transpose4x4(const uint32_t a0, const uint32_t a1, const uint32_t a2,
                                             const uint32_t a3, uint32_t &r0, uint32_t &r1,
                                             uint32_t &r2, uint32_t &r3)
{
    const uint32_t t0 = __byte_perm(a0, a1, 0x5140);  // a0.b0 a1.b0 a0.b1 a1.b1
    const uint32_t t1 = __byte_perm(a2, a3, 0x5140);
    const uint32_t t2 = __byte_perm(a0, a1, 0x7362);  // a0.b2 a1.b2 a0.b3 a1.b3
    const uint32_t t3 = __byte_perm(a2, a3, 0x7362);
    r0 = __byte_perm(t0, t1, 0x5410);
    r1 = __byte_perm(t0, t1, 0x7632);
    r2 = __byte_perm(t2, t3, 0x5410);
    r3 = __byte_perm(t2, t3, 0x7632);
}

// multiply four packed GF(2^8) bytes by alpha (= 2): shift left, reduce by 0x11D where bit 7 was set
__device__ __forceinline__ uint32_t xtime4(uint32_t v)
{
    const uint32_t hi = v & 0x80808080u;
    return ((v ^ hi) << 1) ^ ((hi >> 7) * 0x1du);
}

// ------------------------------------------------------------------ product tables
// Build the tables of `rows` (<= 4) coefficient rows coef[i*cstride + j], j < K, into one table
// buffer; slots >= K are zero.  Entry x of table j is XOR_{bit b of x} (packed column j)*alpha^b.
// Every lane owns one 16-byte bank quad (qd = lane & 7) of the rows x = 4*g + (lane >> 3): it
// keeps the eight powers of its quad's table(s) in registers and walks g in Gray-code order, so
// an entry costs ONE xor per table, and one STS.128 instruction of the warp writes 4 full rows
// (512 B over all 32 banks, the minimum 4 wavefronts).  Work unit = (group, 8 Gray steps);
// units are dealt round-robin to the `nw` participating warps (`w` = this warp's index).
template <class LAYC>
__device__ __forceinline__ void build_tables(uint32_t *tab, const uint8_t *coef, uint32_t cstride, uint32_t rows,
                                             uint32_t w, uint32_t nw, int K)
{
    constexpr TabLayout LAY = LAYC::kLay;
    const uint32_t lane = threadIdx.x & 31, qd = lane & 7, xs = lane >> 3;
    auto packed_col = [&](uint32_t j) -> uint32_t {
        uint32_t cur = 0;
        if (j < (uint32_t)K) {
#pragma unroll
            for (uint32_t i = 0; i < kRowsPerPass; i++)
                if (i < rows) cur |= (uint32_t)coef[i * cstride + j] << (8 * i);
        }
        return cur;
    };
    static_for<0, LAY.ngroups>([&](auto gc) {
        constexpr int g = decltype(gc)::value;
        constexpr int lg = LAY.lg[g];
        constexpr int NTQ = lg <= 3 ? 1 : (lg == 4 ? 2 : 4);  // tables inside one bank quad
        if (LAY.base[g] >= K && LAY.base[g] < LAYC::kK) return;  // plan mode, K = nsurv: no source of this group is read
        // does this warp own a unit of this group at all?
        bool any = false;
#pragma unroll
        for (int sg = 0; sg < 8; sg++) any |= ((uint32_t)(g * 8 + sg) % nw) == w;
        if (!any) return;
        uint32_t pw[NTQ][8];
#pragma unroll
        for (int t = 0; t < NTQ; t++) {
            // banks 4*qd + (4/NTQ)*t ... belong to table (bank >> (5 - lg)) of the group
            const uint32_t bank = 4 * qd + (4 / NTQ) * t;
            uint32_t cur = packed_col(LAY.base[g] + (bank >> (5 - lg)));
#pragma unroll
            for (int b = 0; b < 8; b++) {
                pw[t][b] = cur;
                cur = xtime4(cur);
            }
        }
#pragma unroll 1
        for (uint32_t sg = 0; sg < 8; sg++) {
            if (((uint32_t)(g * 8) + sg) % nw != w) continue;
            const uint32_t n0 = sg * 8;
            uint32_t gx = n0 ^ (n0 >> 1);  // Gray code of the first step of the segment
            uint32_t e[NTQ];
#pragma unroll
            for (int t = 0; t < NTQ; t++) {
                uint32_t v = 0;
                if (xs & 1) v ^= pw[t][0];
                if (xs & 2) v ^= pw[t][1];
#pragma unroll
                for (int b = 0; b < 6; b++)
                    if ((gx >> b) & 1) v ^= pw[t][2 + b];
                e[t] = v;
            }
#pragma unroll
            for (int i = 0; i < 8; i++) {
                const uint32_t x = gx * 4 + xs;
                uint4 v;
                if (NTQ == 1) v = make_uint4(e[0], e[0], e[0], e[0]);
                else if (NTQ == 2) v = make_uint4(e[0], e[0], e[NTQ - 1], e[NTQ - 1]);
                else v = make_uint4(e[0], e[1 % NTQ], e[2 % NTQ], e[3 % NTQ]);
                *reinterpret_cast<uint4 *>(tab + (size_t)g * (kGroupBytes / 4) + x * 32 + qd * 4) = v;
                if (i < 7) {
                    // Gray step n -> n+1 flips bit ctz(n+1); inside an aligned segment of 8 it only
                    // depends on i
                    const int c = (i & 1) == 0 ? 0 : ((i & 3) == 1 ? 1 : 2);
                    gx ^= 1u << c;
#pragma unroll
                    for (int t = 0; t < NTQ; t++) e[t] ^= pw[t][2 + c];
                }
            }
        }
    });
}

// 16 table lookups for one 16-byte vector; acc[4*w + p] ^= T[byte p of word w]
//   base = shared address of (group, this lane's bank for this phase); row_bytes = 128
// The streaming kernels sit at ~75-80 % issue and ~70 % alu-pipe utilisation (ncu, round 2), so
// the per-byte instruction count is what is left to win:
//  * GEC_DP4A: the table address  base + byte_p * 128  is ONE integer dot product,
//    dp4a(word, 0x80 << 8p, base) = base + 128 * byte_p, instead of PRMT (byte extract, alu pipe)
//    + IMAD (scale and add, fma pipe);
//  * GEC_XOR3: two sources are accumulated by one three-input LOP3 (a ^ b ^ c).
#ifndef GEC_DP4A
#define GEC_DP4A 1
#endif
#ifndef GEC_XOR3
#define GEC_XOR3 1
#endif
__device__ __forceinline__ uint32_t table_addr(uint32_t w, int p, uint32_t base, uint32_t row_bytes)
{
#if GEC_DP4A
    (void)row_bytes;
    return __dp4a(w, 0x80u << (8 * p), base);
#else
    const uint32_t x = __byte_perm(w, 0, 0x4440 + p);  // byte p, zero extended (alu pipe)
    return x * row_bytes + base;                        // IMAD (fma pipe)
#endif
}
__device__ __forceinline__ uint32_t xor3(uint32_t a, uint32_t b, uint32_t c)
{
    uint32_t d;
    asm("lop3.b32 %0, %1, %2, %3, 0x96;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}
template <bool kFirst>
__device__ __forceinline__ void lookup16(uint32_t (&acc)[16], const uint4 &d, uint32_t base,
                                         uint32_t row_bytes)
{
    const uint32_t w[4] = {d.x, d.y, d.z, d.w};
#pragma unroll
    for (int i = 0; i < 4; i++) {
#pragma unroll
        for (int p = 0; p < 4; p++) {
            const uint32_t v = lds_u32(table_addr(w[i], p, base, row_bytes));
            if (kFirst) acc[4 * i + p] = v;
            else acc[4 * i + p] ^= v;
        }
    }
}
// two sources at once: acc = acc ^ T_a[..] ^ T_b[..] in one LOP3
template <bool kFirst>
__device__ __forceinline__ void lookup16x2(uint32_t (&acc)[16], const uint4 &da, uint32_t base_a, const uint4 &db,
                                           uint32_t base_b, uint32_t row_bytes)
{
    const uint32_t wa[4] = {da.x, da.y, da.z, da.w}, wb[4] = {db.x, db.y, db.z, db.w};
#pragma unroll
    for (int i = 0; i < 4; i++) {
#pragma unroll
        for (int p = 0; p < 4; p++) {
            const uint32_t va = lds_u32(table_addr(wa[i], p, base_a, row_bytes));
            const uint32_t vb = lds_u32(table_addr(wb[i], p, base_b, row_bytes));
            if (kFirst) acc[4 * i + p] = va ^ vb;
            else acc[4 * i + p] = xor3(acc[4 * i + p], va, vb);
        }
    }
}

__device__ __forceinline__ void rows_from_acc(const uint32_t (&acc)[16], uint4 (&r)[4])
{
    uint32_t o[4][4];
#pragma unroll
    for (int i = 0; i < 4; i++)
        transpose4x4(acc[4 * i + 0], acc[4 * i + 1], acc[4 * i + 2], acc[4 * i + 3], o[0][i], o[1][i],
                     o[2][i], o[3][i]);
#pragma unroll
    for (int row = 0; row < 4; row++) r[row] = make_uint4(o[row][0], o[row][1], o[row][2], o[row][3]);
}

// Source shard read by this lane in slot u: slot u = phase p of group g; sub-warp q = lane / R
// of the group works on source base + (p xor q).
template <class CFG, int U> __device__ __forceinline__ uint32_t lane_source(uint32_t lane)
{
    constexpr TabLayout LAY = CFG::kLay;
    constexpr int g = slot_group(LAY, U);
    constexpr int lg = LAY.lg[g];
    constexpr int ph = U - LAY.base[g];
    return (uint32_t)LAY.base[g] + ((uint32_t)ph ^ (lg ? (lane >> (5 - lg)) : 0u));
}
template <class CFG, int U> __device__ __forceinline__ constexpr bool slot_may_pad()
{
    constexpr TabLayout LAY = CFG::kLay;
    constexpr int g = slot_group(LAY, U);
    return LAY.base[g] + (1 << LAY.lg[g]) > (int)CFG::kK;
}

// LDG: one 16-byte column of every source straight into registers.
//   sp     : address of this lane's column in source 0 (uniform modes) / shard 0 (plan mode)
//   kPlan  : source j lives at sp + src_off[j] (smem) instead of sp + j*stride
//   nsrc   : sources j >= nsrc read as zero (plan mode: an LRC local repair reads only its group)
template <class CFG, bool kPlan>
__device__ __forceinline__ void column_load(const uint8_t *sp, uint32_t stride, const uint32_t *src_off,
                                            uint32_t lane, uint4 (&d)[CFG::S], uint32_t nsrc = CFG::kK)
{
    static_for<0, CFG::S>([&](auto uc) {
        constexpr int u = decltype(uc)::value;
        const uint32_t j = lane_source<CFG, u>(lane);
        if ((!slot_may_pad<CFG, u>() || j < (uint32_t)CFG::kK) && (!kPlan || j < nsrc))
            d[u] = ldg_stream(sp + (kPlan ? src_off[j] : j * stride));
        else d[u] = make_uint4(0, 0, 0, 0);
    });
}
// TMA: the same vectors out of the warp's stage (row j = source j, 512 B per row)
// (rows j >= nsrc were not fetched: they read as zero, and entry 0 of every table is 0)
template <class CFG>
__device__ __forceinline__ void stage_read(uint32_t stage_lane_addr /* stage + lane*16 */, uint32_t lane,
                                           uint4 (&d)[CFG::S], uint32_t nsrc = CFG::kK)
{
    static_for<0, CFG::S>([&](auto uc) {
        constexpr int u = decltype(uc)::value;
        const uint32_t j = lane_source<CFG, u>(lane);
        if ((!slot_may_pad<CFG, u>() || j < (uint32_t)CFG::kK) && j < nsrc) d[u] = lds_v4(stage_lane_addr + j * kStageRowBytes);
        else d[u] = make_uint4(0, 0, 0, 0);
    });
}

// look up + transpose -> r[row] (uint4) for the slots of one column
//   tab_addr : shared address of the table buffer
template <class CFG>
__device__ __forceinline__ void column_compute(uint4 (&d)[CFG::S], uint32_t tab_addr, uint32_t lane,
                                               uint32_t row_bytes, uint32_t tail_bytes, uint4 (&r)[4])
{
    constexpr TabLayout LAY = CFG::kLay;
    uint32_t acc[16];
    if (tail_bytes) {
#pragma unroll
        for (int u = 0; u < CFG::S; u++) d[u] = mask_tail(d[u], tail_bytes);
    }
#if GEC_NULL_MATH
    (void)acc, (void)tab_addr, (void)lane, (void)row_bytes;
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const uint4 a = d[i % CFG::S], b = d[(i + 1) % CFG::S];
        r[i] = make_uint4(a.x ^ b.x, a.y ^ b.y, a.z ^ b.z, a.w ^ b.w);
    }
    return;
#endif
    // this lane's bank at phase ph of group g: lane xor ph*R
    auto slot_base = [&](auto uc) -> uint32_t {
        constexpr int u = decltype(uc)::value;
        constexpr int g = slot_group(LAY, u);
        constexpr int lg = LAY.lg[g];
        constexpr int ph = u - LAY.base[g];
        return tab_addr + (uint32_t)g * kGroupBytes + ((lane ^ ((uint32_t)ph << (lg ? 5 - lg : 0))) << 2);
    };
#if GEC_XOR3
    static_for<0, CFG::S / 2>([&](auto pc) {
        constexpr int u = 2 * decltype(pc)::value;
        lookup16x2<u == 0>(acc, d[u], slot_base(std::integral_constant<int, u>{}), d[u + 1],
                           slot_base(std::integral_constant<int, u + 1>{}), row_bytes);
    });
    if constexpr (CFG::S % 2 == 1)
        lookup16<CFG::S == 1>(acc, d[CFG::S - 1], slot_base(std::integral_constant<int, CFG::S - 1>{}), row_bytes);
#else
    static_for<0, CFG::S>([&](auto uc) {
        constexpr int u = decltype(uc)::value;
        lookup16<u == 0>(acc, d[u], slot_base(uc), row_bytes);
    });
#endif
    rows_from_acc(acc, r);
}

// ---- one table group at a time (split staging): rows of group g sit at stage rows 0..size-1
template <class CFG, int G>
__device__ __forceinline__ void group_read(uint32_t stage_lane_addr, uint32_t lane, uint4 (&d)[16], uint32_t nsrc = CFG::kK)
{
    constexpr TabLayout LAY = CFG::kLay;
    constexpr int lg = LAY.lg[G], n = 1 << lg;
    static_for<0, n>([&](auto pc) {
        constexpr int ph = decltype(pc)::value;
        const uint32_t row = (uint32_t)ph ^ (lg ? (lane >> (5 - lg)) : 0u);  // source base + row
        if ((LAY.base[G] + n <= (int)CFG::kK || (uint32_t)LAY.base[G] + row < (uint32_t)CFG::kK) && (uint32_t)LAY.base[G] + row < nsrc)
            d[ph] = lds_v4(stage_lane_addr + row * kStageRowBytes);
        else d[ph] = make_uint4(0, 0, 0, 0);
    });
}
template <class CFG, int G>
__device__ __forceinline__ void group_lookup(uint32_t (&acc)[16], uint4 (&d)[16], uint32_t tab_addr, uint32_t lane,
                                             uint32_t row_bytes, uint32_t tail_bytes)
{
    constexpr TabLayout LAY = CFG::kLay;
    constexpr int lg = LAY.lg[G], n = 1 << lg;
    if (tail_bytes) {
#pragma unroll
        for (int u = 0; u < n; u++) d[u] = mask_tail(d[u], tail_bytes);
    }
    auto base_of = [&](int ph) -> uint32_t {
        return tab_addr + (uint32_t)G * kGroupBytes + ((lane ^ ((uint32_t)ph << (lg ? 5 - lg : 0))) << 2);
    };
    if constexpr (n == 1) {
        if (G == 0) lookup16<true>(acc, d[0], base_of(0), row_bytes);
        else lookup16<false>(acc, d[0], base_of(0), row_bytes);
    } else {
        static_for<0, n / 2>([&](auto pc) {
            constexpr int u = 2 * decltype(pc)::value;
            if (G == 0 && u == 0) lookup16x2<true>(acc, d[u], base_of(u), d[u + 1], base_of(u + 1), row_bytes);
            else lookup16x2<false>(acc, d[u], base_of(u), d[u + 1], base_of(u + 1), row_bytes);
        });
    }
}

// ------------------------------------------------------------------ the streaming kernel
template <int K, int MODE> struct KernelCfg : StreamCfg<K, cfg_mode(MODE)> {
    static constexpr int kK = K;
};

template <int K, int MODE>
__global__ void __launch_bounds__(StreamCfg<K, cfg_mode(MODE)>::kThreads, 1) rs_apply_kernel(const __grid_constant__ ApplyParams p)
{
    using CFG = KernelCfg<K, MODE>;
    constexpr int S = CFG::S;
    constexpr int NW = CFG::kWarps;  // consumer warps
    constexpr bool TMA = CFG::kTma;
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    uint32_t *const tab = reinterpret_cast<uint32_t *>(smem_raw);
    const uint32_t tab_addr = (uint32_t)__cvta_generic_to_shared(smem_raw);
    const uint32_t stage_addr = tab_addr + CFG::kTabBytes + warp * (CFG::kStageRows * kStageRowBytes);
    PlanSlot *const slot = reinterpret_cast<PlanSlot *>(smem_raw + CFG::kTabBytes + CFG::kStageBytes);
    const uint32_t bars = tab_addr + CFG::kTabBytes + CFG::kStageBytes + 2 * (uint32_t)sizeof(PlanSlot);
    const uint32_t bar_full = bars, bar_empty = bars + 16, bar_stage = bars + 32 + warp * 8;  // full[2], empty[2], stage[NW]

    if (tid == 0) {
        mbar_init(bar_full, 32);
        mbar_init(bar_full + 8, 32);
        mbar_init(bar_empty, NW * 32);
        mbar_init(bar_empty + 8, NW * 32);
    }
    if (TMA && lane == 0 && warp < (uint32_t)NW) mbar_init(bar_stage, 1);
    mbar_fence_init();
    uint32_t stage_parity = 0;

    // TMA: lane 0 arms the warp's stage with `nrow` x `rb` bytes; the copies are issued by the caller
    if constexpr (cfg_mode(MODE) != kModePlan) {
        // ---- uniform coefficient matrix: build once, then warps stream items ----------------
        build_tables<CFG>(tab, p.coef, K, p.rows, warp, (uint32_t)NW, K);
        __syncthreads();

        const uint32_t ips = p.items_per_stripe;
        const uint32_t total = p.n * ips;  // host guarantees that total plus the claims past it stay < 2^32

        // Next work item of this warp.  Fixed stride: item = blockIdx.x * NW + warp, then + NW * gridDim.x.
        // Dynamic: the warp claims runs of GEC_CLAIM_RUN consecutive items from p.counter (zeroed on the stream
        // before the launch), so SMs that stream faster take more items and none idles at the end while another
        // still works through a fixed share.  Lane 0 claims the next run one run ahead, so the atomic's latency
        // hides behind the current run.  Either way a warp's items only grow.
        uint32_t run_next = CFG::kDynamic ? 0u : blockIdx.x * NW + warp, run_left = 0, run_ahead = 0;
        if (CFG::kDynamic && lane == 0) run_ahead = atomicAdd(p.counter, (uint32_t)GEC_CLAIM_RUN);
        auto claim = [&]() -> uint32_t {
            if constexpr (!CFG::kDynamic) {
                const uint32_t i = run_next;
                run_next += gridDim.x * NW;
                return i;
            } else {
                if (run_left == 0) {
                    run_next = __shfl_sync(0xffffffffu, run_ahead, 0);
                    run_left = GEC_CLAIM_RUN;
                    if (lane == 0) run_ahead = atomicAdd(p.counter, (uint32_t)GEC_CLAIM_RUN);
                }
                run_left--;
                return run_next++;
            }
        };

        // position of this lane's column for a work item (stripe, 32-column chunk)
        struct Pos {
            const uint8_t *sp;  // this lane's column in source 0
            uint32_t s, col, tail, rb;
            bool valid, any;  // this lane has a column / the warp has at least one
        };
        // A stripe whose shard_len exceeds the stride is malformed: none of its chunks has columns (encode writes
        // nothing of it) and verify sets every mismatch bit of this pass, once, from the stripe's first chunk.
        auto locate = [&](uint32_t item) -> Pos {
            Pos z;
            z.s = item / ips;
            const uint32_t c = item - z.s * ips;
            uint32_t len = p.shard_len ? __ldg(p.shard_len + z.s) : p.stride;
            if (len > p.stride) {
                if (MODE == kModeVerify && c == 0 && lane == 0) atomicOr(p.mismatch + z.s, ((1u << p.rows) - 1) << p.row_off);
                len = 0;
            }
            const uint32_t nvec = (len + 15) >> 4;
            z.col = c * 32 + lane;
            z.valid = z.col < nvec;
            z.any = c * 32 < nvec;
            z.tail = (z.col == nvec - 1) ? (len & 15) : 0;
            z.rb = z.any ? min(kStageRowBytes, (nvec - c * 32) * 16) : 0;
            z.sp = p.src + (unsigned long long)z.s * p.src_pitch + (size_t)z.col * 16;
            return z;
        };
        // TMA: arm the stage and bring in the staged rows (lane 0): one 2-D tensor copy for the K source
        // rows when the host supplied a tensor map, else one 1-D bulk copy per row
        auto issue = [&](const Pos &z) {
            if (!z.any || lane != 0) return;  // lane 0's column is the first of the chunk
            constexpr int NR = CFG::kStageRows;
            const uint32_t prow = MODE == kModeVerify ? p.rows : 0u;  // stored parity rows staged behind the sources
            if (GEC_TMAP && K >= GEC_TMAP_FROM_K && p.use_tmap) {
                mbar_arrive_expect_tx(bar_stage, kStageRowBytes * K + z.rb * prow);
                tensor_g2s_2d(stage_addr, &p.tmap, (z.col >> 5) * (kStageRowBytes / 4), z.s * p.rows_per_stripe, bar_stage);
            } else {
                mbar_arrive_expect_tx(bar_stage, z.rb * ((uint32_t)K + prow));
#pragma unroll
                for (int j = 0; j < K; j++) bulk_g2s(stage_addr + j * kStageRowBytes, z.sp + (size_t)j * p.stride, z.rb, bar_stage);
            }
#pragma unroll
            for (int j = K; j < NR; j++)
                if ((uint32_t)(j - K) < prow)
                    bulk_g2s(stage_addr + j * kStageRowBytes, z.sp + (size_t)(j + p.row_off) * p.stride, z.rb, bar_stage);
        };
        auto finish = [&](const Pos &z, const uint4 (&r)[4], const uint4 (&st)[4]) {
            uint32_t mm = 0;
            if (MODE == kModeEncode) {
                if (z.valid) {
                    uint8_t *dp = p.dst + (unsigned long long)z.s * p.dst_pitch + (size_t)z.col * 16;
#pragma unroll
                    for (int i = 0; i < 4; i++)
                        if (i < (int)p.rows) stg_stream(dp + (size_t)i * p.stride, r[i]);
                }
            } else {
                if (z.valid) {
#pragma unroll
                    for (int i = 0; i < 4; i++) {
                        if (i < (int)p.rows) {
                            uint4 sv = st[i];
                            if (z.tail) sv = mask_tail(sv, z.tail);
                            const uint32_t diff = (sv.x ^ r[i].x) | (sv.y ^ r[i].y) | (sv.z ^ r[i].z) | (sv.w ^ r[i].w);
                            if (diff) mm |= 1u << (p.row_off + i);
                        }
                    }
                }
                // warp-shuffle OR reduction of the per-lane mismatch bits, one atomic per warp
                mm = __reduce_or_sync(0xffffffffu, mm);
                if (mm && lane == 0) atomicOr(p.mismatch + z.s, mm);
            }
        };
        // stored parity rows of a verify item (they follow the k data shards of the same stripe)
        auto load_stored = [&](const Pos &z, uint4 (&st)[4]) {
            if (MODE != kModeVerify) return;
#pragma unroll
            for (int i = 0; i < 4; i++) {
                st[i] = make_uint4(0, 0, 0, 0);
                if (i < (int)p.rows && z.valid) {
                    if (TMA) st[i] = lds_v4(stage_addr + lane * 16 + (CFG::kSrcRows + i) * kStageRowBytes);
                    else st[i] = ldg_stream(z.sp + (size_t)(K + p.row_off + i) * p.stride);
                }
            }
        };

        uint32_t item = claim();
        if constexpr (CFG::kSplit) {
            // k > 16: one table group (<= 16 sources) per phase; the stage is refilled with the next group
            // (or the first group of the next item) as soon as the current one sits in registers
            constexpr TabLayout LAY = CFG::kLay;
            constexpr int NG = LAY.ngroups;
            auto issue_g = [&](const Pos &z, auto gc) {
                constexpr int g = decltype(gc)::value;
                constexpr int nrow = (LAY.base[g] + (1 << LAY.lg[g]) <= K) ? (1 << LAY.lg[g]) : (K - LAY.base[g]);
                if (!z.any || lane != 0) return;
                const uint32_t prow = (MODE == kModeVerify && g == NG - 1) ? p.rows : 0u;  // stored parity rides with the last group
                if (GEC_TMAP && p.use_tmap) {
                    // box = 16 rows: rows past this group are the next sources (or zero fill at the end of the
                    // tensor); they are fetched and ignored
                    mbar_arrive_expect_tx(bar_stage, kStageRowBytes * 16 + z.rb * prow);
                    tensor_g2s_2d(stage_addr, &p.tmap, (z.col >> 5) * (kStageRowBytes / 4),
                                  z.s * p.rows_per_stripe + LAY.base[g], bar_stage);
                } else {
                    mbar_arrive_expect_tx(bar_stage, z.rb * ((uint32_t)nrow + prow));
#pragma unroll 1  // fallback path (no tensor map: stride < 512 B): keep it out of the register budget
                    for (int r = 0; r < nrow; r++)
                        bulk_g2s(stage_addr + r * kStageRowBytes, z.sp + (size_t)(LAY.base[g] + r) * p.stride, z.rb, bar_stage);
                }
#pragma unroll 1
                for (uint32_t i = 0; i < prow; i++)
                    bulk_g2s(stage_addr + (CFG::kSrcRows + i) * kStageRowBytes, z.sp + (size_t)(K + p.row_off + i) * p.stride, z.rb,
                             bar_stage);
            };
            Pos nx;
            nx.valid = nx.any = false;
            if (item < total) {
                nx = locate(item);
                issue_g(nx, std::integral_constant<int, 0>{});
            }
            while (item < total) {
                const Pos cur = nx;
                if (!cur.any) {  // chunk past the end of a short stripe: nothing was staged for it
                    item = claim();
                    nx.valid = nx.any = false;
                    if (item < total) {
                        nx = locate(item);
                        issue_g(nx, std::integral_constant<int, 0>{});
                    }
                    continue;
                }
                uint32_t acc[16];
                uint4 st[4];
                static_for<0, NG>([&](auto gc) {
                    constexpr int g = decltype(gc)::value;
                    uint4 d[16];
                    mbar_wait(bar_stage, stage_parity);
                    stage_parity ^= 1;
                    group_read<CFG, g>(stage_addr + lane * 16, lane, d);
                    if (g == NG - 1) load_stored(cur, st);
                    stage_release();  // every lane has its vectors: the stage may be refilled
                    if constexpr (g + 1 < NG) {
                        issue_g(cur, std::integral_constant<int, g + 1>{});
                    } else {
                        item = claim();
                        nx.valid = nx.any = false;
                        if (item < total) {
                            nx = locate(item);
                            issue_g(nx, std::integral_constant<int, 0>{});
                        }
                    }
                    if (cur.valid) group_lookup<CFG, g>(acc, d, tab_addr, lane, p.row_bytes, cur.tail);
                });
                uint4 r[4];
                if (cur.valid) rows_from_acc(acc, r);
                finish(cur, r, st);
            }
        } else if constexpr (TMA) {
            Pos nx;
            nx.valid = nx.any = false;
            if (item < total) {
                nx = locate(item);
                issue(nx);
            }
            while (item < total) {
                const Pos cur = nx;
                uint4 d[S], st[4];
                if (cur.any) {
                    mbar_wait(bar_stage, stage_parity);
                    stage_parity ^= 1;
                    stage_read<CFG>(stage_addr + lane * 16, lane, d);
                    load_stored(cur, st);
                }
                stage_release();  // every lane has its vectors: the stage may be refilled
                item = claim();
                nx.valid = nx.any = false;
                if (item < total) {
                    nx = locate(item);
                    issue(nx);
                }
                uint4 r[4];
                if (cur.valid) column_compute<CFG>(d, tab_addr, lane, p.row_bytes, cur.tail, r);
                finish(cur, r, st);
            }
        } else {
            uint4 dn[S], stn[4];
            Pos nx;
            nx.valid = nx.any = false;
            if (item < total) {
                nx = locate(item);
                if (nx.valid) column_load<CFG, false>(nx.sp, p.stride, nullptr, lane, dn);
                load_stored(nx, stn);
            }
            while (item < total) {
                uint4 d[S], st[4];
#pragma unroll
                for (int u = 0; u < S; u++) d[u] = dn[u];
#pragma unroll
                for (int i = 0; i < 4; i++) st[i] = stn[i];
                const Pos cur = nx;
                item = claim();
                nx.valid = nx.any = false;
                if (item < total) {
                    nx = locate(item);
                    if (nx.valid) column_load<CFG, false>(nx.sp, p.stride, nullptr, lane, dn);
                    load_stored(nx, stn);
                }
                uint4 r[4];
                if (cur.valid) column_compute<CFG>(d, tab_addr, lane, p.row_bytes, cur.tail, r);
                finish(cur, r, st);
            }
        }
    } else {
        // ---- per-stripe matrices, no block-wide barrier after this one --------------------------
        // Sources past a plan's nsurv read as zero vectors, and the builder skips table groups that hold none of its
        // sources: those lookups hit row 0 of tables that may never have been built.  Row 0 of every table is 0.
        for (uint32_t i = tid; i < 2 * CFG::kLay.ngroups * 32; i += blockDim.x) tab[(i >> 5) * (kGroupBytes / 4) + (i & 31)] = 0;
        __syncthreads();  // mbarriers initialised, row 0 of the tables zeroed
        constexpr uint32_t kTabBuf = CFG::kTabBytes / 2;
        if (warp == (uint32_t)NW) {
            // ===== builder warp: claim work units, stage their plans, build their tables one unit
            // ahead of the consumers.  Unit sequence number i uses buffer / slot i & 1.
            // Unit u of the launch's counter: stripe u while u < whole, then the last stripes in GEC_TAIL_PARTS
            // chunk ranges each (4096 stripes on 132 SMs are 31.03 stripes per SM: with whole stripes only, a
            // few SMs streamed a 32nd stripe alone at the end).  The parts of a stripe have the same erasure
            // pattern: a table buffer that gets another part of the stripe it already holds skips the build.
            // kModeUnits: work unit w is unit units[1 + w], its plan p.plan[unit], its rows the unit's columns.
            // kModePlan compares with p.n itself below, not with nwork: a register copy of the count held across the
            // loop changes that mode's register allocation (RS(4, m) reconstruct's spills)
            constexpr bool kUnits = MODE == kModeUnits;
            const uint32_t nwork = kUnits ? __ldg(p.units) : p.n;
            const uint32_t whole = nwork > 2 * gridDim.x ? nwork - 2 * gridDim.x : 0;
            uint32_t claimed = 0;
            if (lane == 0) claimed = atomicAdd(p.counter, 1u);
            // pattern whose tables each buffer holds (scalars, not arrays: `b` is a run-time index)
            unsigned long long bp0 = ~0ull, bp1 = ~0ull, bo0 = ~0ull, bo1 = ~0ull;
            bool have0 = false, have1 = false;
            for (uint32_t i = 0;; i++) {
                const uint32_t b = i & 1, use = i >> 1;
                // every consumer warp has left the stripe that used this buffer and slot
                if (use >= 1) mbar_wait(bar_empty + 8 * b, (use - 1) & 1);
                PlanSlot &ps = slot[b];
                const uint32_t u = __shfl_sync(0xffffffffu, claimed, 0);
                if (lane == 0) claimed = atomicAdd(p.counter, 1u);  // consumed by the next iteration
                const bool in_tail = u >= whole;
                const uint32_t s = in_tail ? whole + (u - whole) / GEC_TAIL_PARTS : u;
                const uint32_t part = in_tail ? (u - whole) % GEC_TAIL_PARTS : 0u, parts = in_tail ? GEC_TAIL_PARTS : 1u;
                int rows = 0;
                uint32_t ns = 0;
                unsigned long long kp = 0, ko = 0;
                uint32_t sid = s, pid = s, ubase = 0, ulen = 0;  // kModeUnits: the unit's stripe, plan and columns
                if constexpr (kUnits) {
                    if (s < nwork) {
                        pid = __ldg(p.units + 1 + s);
                        sid = pid / (p.half ? 4u : 8u);
                    }
                }
                const uint32_t slen = s < (kUnits ? nwork : p.n) ? (p.shard_len ? __ldg(p.shard_len + sid) : p.stride) : 0;
                if constexpr (kUnits) unit_columns(slen, pid % (p.half ? 4u : 8u), p.half != 0, &ubase, &ulen);
                // source / output index -> byte offset: a shard, or (PB) the half-row q = 2*shard + half
                auto idx_off = [&](uint32_t i) -> uint32_t {
                    const uint32_t o = p.half ? (i >> 1) * p.stride + (i & 1) * (slen >> 1) : i * p.stride;
                    if constexpr (kUnits) return o + ubase;
                    else return o;
                };
                if (s < (kUnits ? nwork : p.n)) {
                    const StripePlan *pl = p.plan + pid;
                    rows = pl->unrecoverable ? 0 : min(kRowsPerPass, (int)pl->nrows - (int)p.row_off);
                    if (rows > 0) {
                        ns = pl->nsurv;
                        if (lane < ns) ps.src_off[lane] = idx_off(pl->surv[lane]);
                        if (lane < (uint32_t)rows) ps.dst_off[lane] = idx_off(pl->out_idx[p.row_off + lane]);
                        for (uint32_t e = lane; e < (uint32_t)rows * kMaxK; e += 32)
                            ps.coef[e] = pl->coef[p.row_off + e / kMaxK][e % kMaxK];
                        kp = pl->key_present;
                        ko = pl->key_out;
                    }
                }
                if (lane == 0) {
                    uint32_t len = p.half ? slen >> 1 : slen;  // PB: chunks of one half
                    if constexpr (kUnits) len = ulen;
                    const uint32_t nch = (((len + 15) >> 4) + 31) >> 5;  // 32-column chunks of the stripe
                    ps.sid = s;
                    if constexpr (kUnits) ps.sid = s < nwork ? sid : p.n;
                    ps.rows = rows;
                    ps.chunk_next = part * nch / parts;
                    ps.chunk_end = (part + 1) * nch / parts;
                    ps.len = len;
                    ps.nsurv = ns;
                }
                __syncwarp();
                const bool same = b ? (have1 && kp == bp1 && ko == bo1) : (have0 && kp == bp0 && ko == bo0);
                if (rows > 0 && !same) {
                    build_tables<CFG>(tab + b * (kTabBuf / 4), ps.coef, kMaxK, (uint32_t)rows, 0, 1, (int)ns);
                    if (b) {
                        bp1 = kp;
                        bo1 = ko;
                        have1 = true;
                    } else {
                        bp0 = kp;
                        bo0 = ko;
                        have0 = true;
                    }
                }
                mbar_arrive(bar_full + 8 * b);  // all 32 lanes: each lane's table stores are released by its own arrive
                if (s >= (kUnits ? nwork : p.n)) break;
            }
            return;
        }

        // ===== consumer warps
        constexpr uint32_t kNone = 0xffffffffu;
        uint32_t pos = 0;      // stripe sequence number the search is at
        bool entered = false;  // full[pos] has been waited for
        bool ended = false;    // the terminal slot (sid >= n) was seen
        uint32_t pend = kNone; // sequence number of the item whose lookups are still to run
        struct It {
            uint32_t seq, s, chunk, nvec, len, nsurv;
            int rows;
            bool valid;
        };
        // this warp will not touch tables / slot of sequence i again (every lane arrives: each
        // lane's own reads are ordered before its own release)
        auto leave = [&](uint32_t i) { mbar_arrive(bar_empty + 8 * (i & 1)); };
        // next work item of this warp; never waits for full[j] with j > lim (the builder may need
        // this warp's `leave` of an older stripe first)
        auto find = [&](uint32_t lim, It &it) {
            it.valid = false;
            while (!ended) {
                if (!entered) {
                    if (pos > lim) return;
                    mbar_wait(bar_full + 8 * (pos & 1), (pos >> 1) & 1);
                    entered = true;
                }
                PlanSlot &ps = slot[pos & 1];
                const uint32_t s = ps.sid;
                if (s >= p.n) {
                    ended = true;
                    return;
                }
                const int rows = ps.rows;
                if (rows > 0) {
                    const uint32_t len = ps.len, nvec = (len + 15) >> 4;
                    uint32_t c = 0;
                    if (lane == 0) c = atomicAdd(&ps.chunk_next, 1u);
                    c = __shfl_sync(0xffffffffu, c, 0);
                    if (c < ps.chunk_end) {
                        it.seq = pos;
                        it.s = s;
                        it.chunk = c;
                        it.nvec = nvec;
                        it.len = len;
                        it.nsurv = ps.nsurv;
                        it.rows = rows;
                        it.valid = true;
                        return;
                    }
                }
                if (pos != pend) leave(pos);  // else: deferred until the pending lookups are done
                pos++;
                entered = false;
            }
        };
        // start bringing in the columns of an item: TMA copies into the stage / LDG into dn
        uint4 dn[TMA ? 1 : S];
        // split staging: rows of table group g only (stage row r = source base_g + r)
        auto fetch_group = [&](const It &it, auto gc) {
            constexpr int g = decltype(gc)::value;
            constexpr TabLayout LAY = CFG::kLay;
            constexpr int nrow = (LAY.base[g] + (1 << LAY.lg[g]) <= K) ? (1 << LAY.lg[g]) : (K - LAY.base[g]);
            if (lane == 0) {
                const PlanSlot &ps = slot[it.seq & 1];
                const uint8_t *sbase = p.src + (unsigned long long)it.s * p.src_pitch + (size_t)it.chunk * kStageRowBytes;
                const uint32_t rb = min(kStageRowBytes, (it.nvec - it.chunk * 32) * 16);
                const uint32_t nr = it.nsurv > (uint32_t)LAY.base[g] ? min((uint32_t)nrow, it.nsurv - LAY.base[g]) : 0u;
                mbar_arrive_expect_tx(bar_stage, rb * nr);
#pragma unroll
                for (int r = 0; r < nrow; r++)
                    if ((uint32_t)r < nr) bulk_g2s(stage_addr + r * kStageRowBytes, sbase + ps.src_off[LAY.base[g] + r], rb, bar_stage);
            }
        };
        auto fetch = [&](const It &it) {
            const PlanSlot &ps = slot[it.seq & 1];
            const uint8_t *sbase = p.src + (unsigned long long)it.s * p.src_pitch;
            if constexpr (CFG::kSplit) {
                fetch_group(it, std::integral_constant<int, 0>{});
            } else if constexpr (TMA) {
                if (lane == 0) {
                    const uint32_t rb = min(kStageRowBytes, (it.nvec - it.chunk * 32) * 16);
                    mbar_arrive_expect_tx(bar_stage, rb * it.nsurv);
#pragma unroll
                    for (int j = 0; j < K; j++)
                        if ((uint32_t)j < it.nsurv)
                            bulk_g2s(stage_addr + j * kStageRowBytes, sbase + ps.src_off[j] + (size_t)it.chunk * kStageRowBytes, rb,
                                     bar_stage);
                }
            } else {
                const uint32_t col = it.chunk * 32 + lane;
                if (col < it.nvec) column_load<CFG, true>(sbase + (size_t)col * 16, p.stride, ps.src_off, lane, dn, it.nsurv);
            }
        };

        It nx;
        find(kNone, nx);
        if (nx.valid) fetch(nx);
        if constexpr (CFG::kSplit) {
            constexpr int NG = CFG::kLay.ngroups;
            while (nx.valid) {
                const It cur = nx;
                const uint32_t col = cur.chunk * 32 + lane;
                const bool have_col = col < cur.nvec;
                const uint32_t tail = (have_col && col == cur.nvec - 1) ? (cur.len & 15) : 0;
                uint32_t acc[16];
                static_for<0, NG>([&](auto gc) {
                    constexpr int g = decltype(gc)::value;
                    uint4 d[16];
                    mbar_wait(bar_stage, stage_parity);
                    stage_parity ^= 1;
                    group_read<CFG, g>(stage_addr + lane * 16, lane, d, cur.nsurv);
                    stage_release();  // every lane has its vectors: the stage may be refilled
                    if constexpr (g + 1 < NG) {
                        fetch_group(cur, std::integral_constant<int, g + 1>{});  // next group of the same item
                    } else {
                        pend = cur.seq;
                        find(cur.seq + 1, nx);
                        if (nx.valid) fetch(nx);  // first group of the next item
                    }
                    if (have_col) group_lookup<CFG, g>(acc, d, tab_addr + (cur.seq & 1) * kTabBuf, lane, p.row_bytes, tail);
                });
                if (have_col) {
                    const PlanSlot &ps = slot[cur.seq & 1];
                    uint4 r[4];
                    rows_from_acc(acc, r);
                    uint8_t *dbase = p.dst + (unsigned long long)cur.s * p.dst_pitch;
#pragma unroll
                    for (int i = 0; i < 4; i++)
                        if (i < cur.rows) stg_stream(dbase + ps.dst_off[i] + (size_t)col * 16, r[i]);
                }
                if (pos != cur.seq) leave(cur.seq);
                pend = kNone;
                if (!nx.valid && !ended) {
                    find(kNone, nx);
                    if (nx.valid) fetch(nx);
                }
            }
            return;
        }
        while (nx.valid) {
            const It cur = nx;
            uint4 d[S];
            if constexpr (TMA) {
                mbar_wait(bar_stage, stage_parity);
                stage_parity ^= 1;
                stage_read<CFG>(stage_addr + lane * 16, lane, d, cur.nsurv);
                stage_release();  // every lane has its vectors: the stage may be refilled
            } else {
#pragma unroll
                for (int u = 0; u < S; u++) d[u] = dn[u];
            }
            pend = cur.seq;
            find(cur.seq + 1, nx);
            if (nx.valid) fetch(nx);
            {
                const PlanSlot &ps = slot[cur.seq & 1];
                const uint32_t col = cur.chunk * 32 + lane;
                if (col < cur.nvec) {
                    const uint32_t tail = (col == cur.nvec - 1) ? (cur.len & 15) : 0;
                    uint4 r[4];
                    column_compute<CFG>(d, tab_addr + (cur.seq & 1) * kTabBuf, lane, p.row_bytes, tail, r);
                    uint8_t *dbase = p.dst + (unsigned long long)cur.s * p.dst_pitch;
#pragma unroll
                    for (int i = 0; i < 4; i++)
                        if (i < cur.rows) stg_stream(dbase + ps.dst_off[i] + (size_t)col * 16, r[i]);
                }
            }
            if (pos != cur.seq) leave(cur.seq);  // the search moved on while these lookups were pending
            pend = kNone;
            if (!nx.valid && !ended) {  // the look-ahead was not allowed to go further: continue now
                find(kNone, nx);
                if (nx.valid) fetch(nx);
            }
        }
    }
}

// ------------------------------------------------------------------ decode planning
struct PlanParams {
    const uint8_t *present;  // n*(k+m)
    const uint8_t *want;     // nullable
    int32_t *status;         // nullable, n
    StripePlan *plan;        // n
    uint32_t *counter;       // reset to 0 for the apply kernel's scheduler
    uint32_t n, k, m;
    uint32_t l;               // LRC local groups; 0 for RS and PB
    uint32_t pb;              // 1: PB(k, m), planned over half-rows
    uint32_t present_is_bad;  // 1: `present` holds "bad" flags (scrub): a shard is present iff flag == 0
    const uint32_t *shard_len;  // per stripe, nullable (=> stride); > stride (PB: or % 32 != 0) is malformed
    uint32_t stride;
    alignas(16) uint8_t P[kMaxM * kMaxK];  // parity rows, P[i*k + j] (16-byte aligned: staged with uint4 loads)
};

constexpr int kPlanWarps = 4;
static_assert(2 * kPbMaxM <= kMaxM && 2 * kPbMaxK <= kMaxK, "PB half-rows fit a StripePlan");

// Decode planning for every code (DESIGN.md section 4.2), one warp per stripe, lanes own the cols() <= 32 generator
// columns.  The survivors are a greedy rank basis, in row order, of PlanCode::candidate_rows; every wanted row is then
// expressed in that basis, or the stripe is unrecoverable.  h_read_plan (gf256.h) is the host twin.
// The basis is an incremental Gauss-Jordan: basis row b is stored reduced as [row | T_b], T_b giving it as a
// combination of the survivors, and a row is reduced against the basis rows in insertion order, which zeroes it at
// every earlier pivot.  The data rows come first and are identity rows, so the candidate data rows enter the basis
// as they are (pivot = their column, T = e_position), and reducing a row against all of them is one lane-parallel
// step.  Only parity rows and wanted rows are reduced serially, against the parity rows of the basis: fewer than the
// absent data columns and at most kMaxM.  A stripe whose shard_len exceeds the stride, or a PB stripe whose shard_len
// is not a multiple of 32 (no 16-byte aligned halves), is malformed: status GARAGE_EC_E_INVALID (-1), no rows, so the
// apply kernel reads and writes nothing of it.  16 CTAs per SM keep it at 32 registers, no spills.
__global__ void __launch_bounds__(kPlanWarps * 32, 16) plan_kernel(const __grid_constant__ PlanParams q)
{
    __shared__ __align__(16) uint8_t s_gf[sizeof(GfTables)];
    uint8_t *const s_exp = s_gf, *const s_log = s_gf + 512;
    __shared__ uint8_t s_R[kPlanWarps][kMaxM][2 * kMaxK];  // parity rows of the basis, [row | T]
    __shared__ uint8_t s_piv[kPlanWarps][kMaxM];
    __shared__ uint8_t s_surv[kPlanWarps][kMaxK];
    __shared__ __align__(16) uint8_t s_P[kMaxM * kMaxK];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    stage_gf_tables(s_gf);
    {  // parity rows: kernel parameter (constant bank) -> shared, warp-uniform 16-byte loads
        const uint4 *src = reinterpret_cast<const uint4 *>(q.P);
        for (uint32_t i = warp; i < sizeof(q.P) / 16; i += blockDim.x >> 5) {
            const uint4 v = src[i];
            if (lane < 4) reinterpret_cast<uint32_t *>(s_P)[i * 4 + lane] = lane == 0 ? v.x : (lane == 1 ? v.y : (lane == 2 ? v.z : v.w));
        }
    }
    if (blockIdx.x == 0 && tid == 0) *q.counter = 0;
    __syncthreads();
    auto mul = [&](uint32_t a, uint32_t b) -> uint32_t {
        return (a && b) ? s_exp[s_log[a] + s_log[b]] : 0u;
    };

    const uint32_t s = blockIdx.x * kPlanWarps + warp;
    if (s >= q.n) return;
    const uint32_t tot = q.k + q.m;
    StripePlan *pl = q.plan + s;
    const uint8_t *pr = q.present + (size_t)s * tot;
    const uint8_t *wn = q.want ? q.want + (size_t)s * tot : nullptr;

    // presence / wanted shard masks (tot <= 40: two ballot rounds)
    const bool inv = q.present_is_bad != 0;
    const bool p0 = lane < tot && ((pr[lane] != 0) != inv);
    const bool p1 = lane + 32 < tot && ((pr[lane + 32] != 0) != inv);
    const unsigned long long present =
        (unsigned long long)__ballot_sync(0xffffffffu, p0) | ((unsigned long long)__ballot_sync(0xffffffffu, p1) << 32);
    const bool w0 = lane < tot && !p0 && (!wn || wn[lane] != 0);
    const bool w1 = lane + 32 < tot && !p1 && (!wn || wn[lane + 32] != 0);
    const unsigned long long outmask =
        (unsigned long long)__ballot_sync(0xffffffffu, w0) | ((unsigned long long)__ballot_sync(0xffffffffu, w1) << 32);
    const uint32_t slen = q.shard_len ? q.shard_len[s] : q.stride;
    if (slen > q.stride || (q.pb && (slen & 31))) {
        if (lane == 0) {
            pl->key_present = present;
            pl->key_out = outmask;
            pl->nrows = 0;
            pl->unrecoverable = 1;
            pl->nsurv = 0;
            if (q.status) q.status[s] = -1;
        }
        return;
    }
    const PlanCode code{(int)q.k, (int)q.m, (int)q.l, q.pb != 0, s_P};
    const uint32_t K = (uint32_t)code.cols();
    const unsigned long long cand = code.candidate_rows(present, outmask);
    const unsigned long long wrows = code.below_k(present) ? 0ull : code.shard_rows(outmask);

    // the candidate data rows: basis positions 0..nd in column order
    const unsigned long long dmask = cand & ((1ull << K) - 1);
    const uint32_t nd = (uint32_t)__popcll(dmask);
    const bool dcol = (dmask >> lane) & 1;
    if (dcol) s_surv[warp][__popcll(dmask & ((1ull << lane) - 1))] = (uint8_t)lane;
    __syncwarp();
    const uint32_t dsrc = lane < nd ? s_surv[warp][lane] : 0u;  // the column of basis position `lane`
    uint8_t(*R)[2 * kMaxK] = s_R[warp];
    uint32_t np = 0;  // parity rows in the basis
    // v (lane = column) reduced against the basis, t accumulating the combination of survivors
    auto reduce = [&](uint32_t &v, uint32_t &t) {
        const uint32_t vd = __shfl_sync(0xffffffffu, v, dsrc);
        if (lane < nd) t ^= vd;
        if (dcol) v = 0;
        for (uint32_t b = 0; b < np; b++) {
            const uint32_t f = __shfl_sync(0xffffffffu, v, s_piv[warp][b]);
            if (f) {
                v ^= mul(f, R[b][lane]);
                t ^= mul(f, R[b][kMaxK + lane]);
            }
        }
    };
    uint32_t nsurv = nd;
    for (unsigned long long pm = cand & ~dmask; pm && nsurv < K; pm &= pm - 1) {
        const uint32_t c = (uint32_t)(__ffsll((long long)pm) - 1);
        uint32_t v = lane < K ? code.row((int)c, (int)lane) : 0u, t = lane == nsurv ? 1u : 0u;
        reduce(v, t);
        const uint32_t nz = __ballot_sync(0xffffffffu, v != 0);
        if (!nz) continue;  // in the span of the rows already chosen
        const uint32_t piv = __ffs(nz) - 1;
        const uint32_t iv = s_exp[255 - s_log[__shfl_sync(0xffffffffu, v, piv)]];
        R[np][lane] = (uint8_t)mul(v, iv);
        R[np][kMaxK + lane] = (uint8_t)mul(t, iv);
        if (lane == 0) {
            s_piv[warp][np] = (uint8_t)piv;
            s_surv[warp][nsurv] = (uint8_t)c;
        }
        __syncwarp();
        np++;
        nsurv++;
    }
    bool ok = !code.below_k(present);
    int nrows = 0;
    for (unsigned long long om = wrows; om && ok; om &= om - 1, nrows++) {
        const uint32_t o = (uint32_t)(__ffsll((long long)om) - 1);
        uint32_t v = lane < K ? code.row((int)o, (int)lane) : 0u, t = 0;
        reduce(v, t);
        ok = __ballot_sync(0xffffffffu, v != 0) == 0;  // else outside the span of the candidate rows
        // (while ok, nrows < kMaxM: RS and PB rebuild at most m shards, 2m <= kMaxM halves; LRC rows in the span of
        // fewer than k independent rows are at most l more than them)
        if (ok) pl->coef[nrows][lane] = (uint8_t)t;
    }
    if (lane < nsurv) pl->surv[lane] = s_surv[warp][lane];
    if (lane == 0) {
        int r = 0;
        if (ok)  // an unrecoverable stripe may have up to k+m-1 absent shards: out_idx holds kMaxM
            for (unsigned long long om = wrows; om; om &= om - 1, r++) pl->out_idx[r] = (uint8_t)(__ffsll((long long)om) - 1);
        pl->key_present = code.pb ? cand : present;  // with key_out, the apply kernel's table reuse key
        pl->key_out = wrows;
        pl->nrows = ok ? (uint8_t)nrows : 0;
        pl->unrecoverable = ok ? 0 : 1;
        pl->nsurv = (uint8_t)nsurv;
        if (q.status) q.status[s] = ok ? 0 : -4;
    }
}

// ---- reconstruct by adler8 unit (garage_ec_reconstruct_segments, DESIGN.md 2.10 / 4.13) -------------------------
// unit_prep_kernel turns the per-shard segment bits into one presence row per unit, plan_kernel plans the n*U rows,
// unit_fold_kernel gives each stripe its status and lists the units with work, and rs_apply_kernel<kModeUnits>
// rebuilds only those units' columns.
struct UnitParams {
    const uint8_t *seg_present;  // n*(k+m): bit g = segment g of shard i holds valid bytes
    const uint8_t *want;         // n*(k+m), nullable
    const uint32_t *shard_len;   // n, nullable (=> stride)
    uint8_t *unit_present;       // n*U*(k+m) out (prep)
    uint8_t *unit_want;          // n*U*(k+m) out (prep), when want != NULL
    const int32_t *unit_status;  // n*U, plan_kernel's verdict per unit (fold)
    const StripePlan *plan;      // n*U (fold)
    int32_t *status;             // n, nullable (fold)
    uint32_t *units;             // 1 + n*U (fold): units[0] = count (zero at launch), then unit ids
    uint32_t n, tot, stride, pb;
};
__host__ __device__ inline uint32_t units_per_stripe(bool pb) { return pb ? 4u : 8u; }
// A stripe whose L exceeds the stride, or a PB stripe whose L is not a multiple of 128, is malformed
__device__ __forceinline__ uint32_t unit_stripe_len(const UnitParams &q, uint32_t s, bool *bad)
{
    const uint32_t L = q.shard_len ? __ldg(q.shard_len + s) : q.stride;
    *bad = L > q.stride || (q.pb && (L & 127));
    return L;
}
// one thread per (unit, shard); a malformed stripe's units are all present (no work)
__global__ void __launch_bounds__(256) unit_prep_kernel(const __grid_constant__ UnitParams q)
{
    const uint32_t U = units_per_stripe(q.pb != 0);
    const size_t e = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (e >= (size_t)q.n * U * q.tot) return;
    const uint32_t unit = (uint32_t)(e / q.tot), i = (uint32_t)(e % q.tot), s = unit / U, g = unit % U;
    bool bad;
    const uint32_t L = unit_stripe_len(q, s, &bad);
    const size_t si = (size_t)s * q.tot + i;
    q.unit_present[e] = (bad || unit_present(__ldg(q.seg_present + si), L, g, q.pb != 0)) ? 1 : 0;
    if (q.want) q.unit_want[e] = __ldg(q.want + si);
}
// one thread per stripe: status, then the ids of its units that rebuild rows, appended to the work list (any order:
// every unit writes only its own columns)
__global__ void __launch_bounds__(256) unit_fold_kernel(const __grid_constant__ UnitParams q)
{
    const uint32_t s = blockIdx.x * 256 + threadIdx.x;
    if (s >= q.n) return;
    const uint32_t U = units_per_stripe(q.pb != 0);
    bool bad;
    (void)unit_stripe_len(q, s, &bad);
    int32_t st = bad ? GARAGE_EC_E_INVALID : 0;
    for (uint32_t g = 0; g < U && !st; g++)
        if (q.unit_status[(size_t)s * U + g] != 0) st = GARAGE_EC_E_UNRECOVERABLE;
    if (q.status) q.status[s] = st;
    if (st) return;
    uint32_t cnt = 0;
    for (uint32_t g = 0; g < U; g++) cnt += q.plan[(size_t)s * U + g].nrows > 0;
    if (!cnt) return;
    uint32_t w = atomicAdd(q.units, cnt);
    for (uint32_t g = 0; g < U; g++)
        if (q.plan[(size_t)s * U + g].nrows > 0) q.units[1 + w++] = s * U + g;
}

// ---- PB(k, m) encode / verify (DESIGN.md section 2.2) -----------------------------------------------------------
// The RS(k, m) product tables, built once.  A work item is 32 columns of the a-half and the same 32 columns of the
// b-half of every shard of a stripe, streamed through the warp's stage in two phases (a, then b) with k 1-D bulk
// copies each (+ m stored parity halves for verify): the b-phase copy flies while the a-rows are looked up, the next
// item's a-phase copy while the b-rows are.  Every data vector is looked up once; the piggybacks are plain XORs of
// the staged a-vectors of each group into the b-outputs.  HBM traffic is the RS(k, m) encode's, (k+m)*L per stripe.
// shard_len must be a multiple of 32 (16-byte aligned halves) and at most the stride: a malformed stripe gets every
// mismatch bit (verify) or no write at all (encode).
template <int K, int MODE> struct PbCfg {
    static constexpr int kK = K;
    static constexpr TabLayout kLay = make_layout(K, 5, 2);  // RS(10,4): 8 + 2 tables, 64 KB
    static constexpr int S = kLay.nslots;
    static constexpr uint32_t kTabBytes = (uint32_t)kLay.ngroups * kGroupBytes;
    static constexpr int kStageRows = K + (MODE == kModeVerify ? kRowsPerPass : 0);
    // register budget: S x 4 words of column data + piggybacks + stored rows + accumulators (12 warps: 168 registers)
    static constexpr int kWarps = cfg_fit_nw(K <= 8 ? 16 : 12, kTabBytes, kStageRows, false);
    static constexpr int kThreads = 32 * kWarps;
    static constexpr uint32_t kStageBytes = (uint32_t)kWarps * kStageRows * kStageRowBytes;
    static constexpr uint32_t kSmem = kTabBytes + kStageBytes + kAuxBytes;
    static_assert(K >= 1 && K <= kPbMaxK && kLay.nslots >= K, "no table layout for this k");
    static_assert(kSmem <= kSmemLimit, "shared memory budget exceeded");
};

template <int K, int MODE>
__global__ void __launch_bounds__(PbCfg<K, MODE>::kThreads, 1) pb_apply_kernel(const __grid_constant__ ApplyParams p)
{
    using CFG = PbCfg<K, MODE>;
    constexpr int S = CFG::S;
    constexpr int NW = CFG::kWarps;
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    uint32_t *const tab = reinterpret_cast<uint32_t *>(smem_raw);
    const uint32_t tab_addr = (uint32_t)__cvta_generic_to_shared(smem_raw);
    const uint32_t stage = tab_addr + CFG::kTabBytes + warp * (CFG::kStageRows * kStageRowBytes);
    const uint32_t bar = tab_addr + CFG::kTabBytes + CFG::kStageBytes + warp * 8;
    if (lane == 0) mbar_init(bar, 1);
    mbar_fence_init();
    build_tables<CFG>(tab, p.coef, K, p.rows, warp, (uint32_t)NW, K);
    __syncthreads();

    const uint32_t m = p.rows;  // 2..4: one pass
    const int gb2 = m > 2 ? pb_group_start(K, (int)m, 2) : K, gb3 = m > 3 ? pb_group_start(K, (int)m, 3) : K;
    const uint32_t ips = p.items_per_stripe, total = p.n * ips, step = gridDim.x * NW;
    struct Pos {
        const uint8_t *sp;  // chunk start in data shard 0, a-half
        uint32_t s, col, h, rb;
        bool valid;  // this lane has a column
    };
    // next item at or after `it` with columns to stream; malformed stripes are flagged (verify) and skipped
    auto advance = [&](uint32_t &it, Pos &z) -> bool {
        for (; it < total; it += step) {
            const uint32_t s = it / ips, c = it - s * ips;
            const uint32_t len = p.shard_len ? __ldg(p.shard_len + s) : p.stride;
            if ((len & 31) || len > p.stride) {
                if (MODE == kModeVerify && c == 0 && lane == 0) atomicOr(p.mismatch + s, (1u << m) - 1);
                continue;
            }
            const uint32_t nvec = len >> 5;  // 16-byte vectors per half
            if (c * 32 >= nvec) continue;
            z.s = s;
            z.h = len >> 1;
            z.col = c * 32 + lane;
            z.valid = z.col < nvec;
            z.rb = min(kStageRowBytes, (nvec - c * 32) * 16);
            z.sp = p.src + (unsigned long long)s * p.src_pitch + (size_t)c * kStageRowBytes;
            return true;
        }
        return false;
    };
    auto issue = [&](const Pos &z, uint32_t off) {
        if (lane != 0) return;
        const uint32_t prow = MODE == kModeVerify ? m : 0u;
        mbar_arrive_expect_tx(bar, z.rb * ((uint32_t)K + prow));
#pragma unroll
        for (int j = 0; j < K; j++) bulk_g2s(stage + j * kStageRowBytes, z.sp + (size_t)j * p.stride + off, z.rb, bar);
        for (uint32_t i = 0; i < prow; i++)
            bulk_g2s(stage + (K + i) * kStageRowBytes, z.sp + (size_t)(K + i) * p.stride + off, z.rb, bar);
    };
    auto load_stored = [&](uint4 (&st)[kRowsPerPass]) {
#pragma unroll
        for (int i = 0; i < kRowsPerPass; i++)
            st[i] = (MODE == kModeVerify && (uint32_t)i < m) ? lds_v4(stage + lane * 16 + (K + i) * kStageRowBytes) : make_uint4(0, 0, 0, 0);
    };
    auto finish = [&](const Pos &z, uint32_t off, const uint4 (&r)[4], const uint4 (&st)[kRowsPerPass], uint32_t &mm) {
        if (!z.valid) return;
        if (MODE == kModeEncode) {
            uint8_t *dp = p.dst + (unsigned long long)z.s * p.dst_pitch + off + (size_t)z.col * 16;
#pragma unroll
            for (int i = 0; i < kRowsPerPass; i++)
                if ((uint32_t)i < m) stg_stream(dp + (size_t)i * p.stride, r[i]);
        } else {
#pragma unroll
            for (int i = 0; i < kRowsPerPass; i++)
                if ((uint32_t)i < m && ((st[i].x ^ r[i].x) | (st[i].y ^ r[i].y) | (st[i].z ^ r[i].z) | (st[i].w ^ r[i].w))) mm |= 1u << i;
        }
    };

    uint32_t it = blockIdx.x * NW + warp, parity = 0;
    Pos cur;
    bool have = advance(it, cur);
    if (have) issue(cur, 0);
    while (have) {
        uint4 d[S], st[kRowsPerPass], pg[kPbMaxM - 1], r[4];
        uint32_t mm = 0;
        // ---- a-phase: look up the a-rows; keep the group XORs of the raw a-vectors for the piggybacks
        mbar_wait(bar, parity);
        parity ^= 1;
        stage_read<CFG>(stage + lane * 16, lane, d);
#pragma unroll
        for (int i = 0; i < kPbMaxM - 1; i++) pg[i] = make_uint4(0, 0, 0, 0);
#pragma unroll
        for (int j = 0; j < K; j++) {
            const uint4 v = lds_v4(stage + lane * 16 + j * kStageRowBytes);
            auto acc = [&](uint4 &g) { g = make_uint4(g.x ^ v.x, g.y ^ v.y, g.z ^ v.z, g.w ^ v.w); };
            if (j < gb2) acc(pg[0]);  // warp-uniform branches: pg stays in registers
            else if (j < gb3) acc(pg[1]);
            else acc(pg[2]);
        }
        load_stored(st);
        stage_release();
        issue(cur, cur.h);
        if (cur.valid) column_compute<CFG>(d, tab_addr, lane, p.row_bytes, 0, r);
        finish(cur, 0, r, st, mm);
        // ---- b-phase: RS value of the b-rows, then the piggybacks into parities 1..m-1
        mbar_wait(bar, parity);
        parity ^= 1;
        stage_read<CFG>(stage + lane * 16, lane, d);
        load_stored(st);
        stage_release();
        Pos nx;
        it += step;
        const bool have_next = advance(it, nx);
        if (have_next) issue(nx, 0);
        if (cur.valid) {
            column_compute<CFG>(d, tab_addr, lane, p.row_bytes, 0, r);
#pragma unroll
            for (int i = 1; i < kRowsPerPass; i++)
                r[i] = make_uint4(r[i].x ^ pg[i - 1].x, r[i].y ^ pg[i - 1].y, r[i].z ^ pg[i - 1].z, r[i].w ^ pg[i - 1].w);
        }
        finish(cur, cur.h, r, st, mm);
        if (MODE == kModeVerify) {
            mm = __reduce_or_sync(0xffffffffu, mm);
            if (mm && lane == 0) atomicOr(p.mismatch + cur.s, mm);
        }
        cur = nx;
        have = have_next;
    }
}

// ------------------------------------------------------------------ synthetic data
// splitmix64 counter stream of SURVEY.md 8(d) (the CPU checker generates the same stream).
__global__ void fill_random_kernel(unsigned long long *dst, size_t nwords, unsigned long long seed,
                                   unsigned long long first_idx)
{
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nwords;
         i += (size_t)gridDim.x * blockDim.x) {
        unsigned long long z = seed + (first_idx + i + 1) * 0x9E3779B97F4A7C15ull;
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
        z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
        dst[i] = z ^ (z >> 31);
    }
}

// ------------------------------------------------------------------ per-shard integrity (row f2)
// blake2sum (BLAKE2b-512 truncated to 32 bytes, src/util/data.rs:130-138) of every shard of a
// batch, one thread per shard.  BLAKE2b is sequential per message, so the parallelism is across
// the n * shards_per_stripe independent shards; compute-bound (~28 integer instructions per
// byte), not HBM-bound.  `expect` != NULL turns it into the scrub check: bad[i] = sum differs.
struct SumParams {
    const uint8_t *base;        // shard i at base + i * stride
    const uint32_t *shard_len;  // per stripe, nullable (=> stride)
    const uint8_t *expect;      // nullable: 32 bytes per shard to compare with
    uint8_t *sums;              // nullable: 32 bytes per shard out
    uint8_t *bad;               // nullable: 1 byte per shard out (only with expect)
    uint32_t stride;
    uint32_t per_stripe;        // shards per stripe (k, m or k+m)
    uint32_t n_shards;
    uint32_t out_per_stripe;    // sums/expect/bad are indexed (i / per_stripe) * out_per_stripe
    uint32_t out_off;           //                              + out_off + i % per_stripe
    // optional second segment (shards n_first.. of the launch): lets one launch hash the data
    // array AND the parity array of an encode batch (half the latency of two launches)
    const uint8_t *base2;
    uint32_t n_first;           // shards in the first segment (== n_shards when there is no second)
    uint32_t per_stripe2;
    uint32_t out_off2;
};

// where shard i of a launch lives, which stripe's length applies, and its slot in sums/expect/bad.  False for a shard
// whose length exceeds the stride: it is malformed, the kernels read none of it, check mode flags it bad and sums mode
// leaves its 32 bytes alone.
__device__ __forceinline__ bool locate_shard(const SumParams &q, uint32_t i, const uint8_t *&p, uint32_t &len,
                                             size_t &oi)
{
    uint32_t stripe;
    if (i < q.n_first) {
        stripe = i / q.per_stripe;
        p = q.base + (size_t)i * q.stride;
        oi = (size_t)stripe * q.out_per_stripe + q.out_off + (i - stripe * q.per_stripe);
    } else {
        const uint32_t j = i - q.n_first;
        stripe = j / q.per_stripe2;
        p = q.base2 + (size_t)j * q.stride;
        oi = (size_t)stripe * q.out_per_stripe + q.out_off2 + (j - stripe * q.per_stripe2);
    }
    len = q.shard_len ? __ldg(q.shard_len + stripe) : q.stride;
    return len <= q.stride;
}

__global__ void __launch_bounds__(128) blake2sum_shards_kernel(const __grid_constant__ SumParams q)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= q.n_shards) return;
    const uint8_t *p;
    uint32_t len;
    size_t oi;
    if (!locate_shard(q, i, p, len, oi)) {
        if (q.expect && q.bad) q.bad[oi] = 1;
        return;
    }
    Blake2bState S;
    blake2b_init512(S);
    uint64_t m[16];
    uint32_t off = 0;
    while (len - off > 128) {
#pragma unroll
        for (int w = 0; w < 8; w++) {
            const uint4 v = *reinterpret_cast<const uint4 *>(p + off + 16 * w);
            m[2 * w] = (uint64_t)v.x | ((uint64_t)v.y << 32);
            m[2 * w + 1] = (uint64_t)v.z | ((uint64_t)v.w << 32);
        }
        S.t += 128;
        blake2b_compress(S, m, false);
        off += 128;
    }
    const uint32_t rem = len - off;  // 0..128 bytes in the last block (0 only for an empty shard)
#pragma unroll
    for (int w = 0; w < 8; w++) {
        uint4 v = make_uint4(0, 0, 0, 0);
        if ((uint32_t)(16 * w) < rem) {
            v = *reinterpret_cast<const uint4 *>(p + off + 16 * w);  // within roundup16(len): readable
            if (rem - 16 * w < 16) v = mask_tail(v, rem - 16 * w);
        }
        m[2 * w] = (uint64_t)v.x | ((uint64_t)v.y << 32);
        m[2 * w + 1] = (uint64_t)v.z | ((uint64_t)v.w << 32);
    }
    S.t += rem;
    blake2b_compress(S, m, true);
    if (q.sums) {
        uint4 *o = reinterpret_cast<uint4 *>(q.sums + oi * 32);
        o[0] = make_uint4((uint32_t)S.h[0], (uint32_t)(S.h[0] >> 32), (uint32_t)S.h[1], (uint32_t)(S.h[1] >> 32));
        o[1] = make_uint4((uint32_t)S.h[2], (uint32_t)(S.h[2] >> 32), (uint32_t)S.h[3], (uint32_t)(S.h[3] >> 32));
    }
    if (q.expect && q.bad) {
        const unsigned long long *e = reinterpret_cast<const unsigned long long *>(q.expect + oi * 32);
        q.bad[oi] = (e[0] != S.h[0]) | (e[1] != S.h[1]) | (e[2] != S.h[2]) | (e[3] != S.h[3]);
    }
}


// ---- the same hash with FOUR lanes per shard --------------------------------------------------
// With a few ten-thousand shards per batch the one-thread-per-shard kernel leaves most of the GPU
// idle (28 672 shards = 1.5 warps per scheduler).  BLAKE2b's four column G functions and four
// diagonal G functions are independent, so a quad of lanes shares one message: lane c owns
// column c of the 4x4 state (a,b,c,d = v[c], v[4+c], v[8+c], v[12+c]); the diagonal step is the
// column step after rotating rows 1,2,3 by 1,2,3 lanes inside the quad (quad-masked shuffles).
// The 128-byte message block sits in shared memory (32 B loaded per lane, coalesced per quad); the
// per-round word selection sigma[r] is four byte offsets packed in one register per round.
// ~1.5x the instructions of the scalar kernel for 4x the parallelism.
__constant__ uint8_t c_b2_sigma[12][16] = {
    {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15}, {14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3},
    {11, 8, 12, 0, 5, 2, 15, 13, 10, 14, 3, 6, 7, 1, 9, 4}, {7, 9, 3, 1, 13, 12, 11, 14, 2, 6, 5, 10, 4, 0, 15, 8},
    {9, 0, 5, 7, 2, 4, 10, 15, 14, 1, 11, 12, 6, 8, 3, 13}, {2, 12, 6, 10, 0, 11, 8, 3, 4, 13, 7, 5, 15, 14, 1, 9},
    {12, 5, 1, 15, 14, 13, 4, 10, 0, 7, 6, 3, 9, 2, 8, 11}, {13, 11, 7, 14, 12, 1, 3, 9, 5, 0, 15, 4, 8, 6, 2, 10},
    {6, 15, 14, 9, 11, 3, 0, 8, 12, 2, 13, 7, 1, 4, 10, 5}, {10, 2, 8, 4, 7, 6, 1, 5, 15, 11, 9, 14, 3, 12, 13, 0},
    {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15}, {14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3}};

__device__ __forceinline__ uint64_t shfl64(uint32_t mask, uint64_t v, uint32_t src)
{
    const uint32_t lo = __shfl_sync(mask, (uint32_t)v, src), hi = __shfl_sync(mask, (uint32_t)(v >> 32), src);
    return (uint64_t)lo | ((uint64_t)hi << 32);
}
__device__ __forceinline__ uint64_t lds_u64(uint32_t addr)
{
    uint64_t r;
    asm volatile("ld.shared.u64 %0, [%1];" : "=l"(r) : "r"(addr));
    return r;
}

constexpr int kQuadThreads = 128;  // 32 shards per block

// BLAKE2b-512 of a len-byte message by one quad; lane c = threadIdx.x & 3 returns h[c], bytes 8c..8c+7 of the digest.
// load32(o, x, y) gives this lane's 32 message bytes at o + 32c, zero beyond len; it is called for o = 0, 128, ...
// in order, one block ahead of the compression.  s_row: the quad's 128-byte message row in shared memory.
template <class Load32>
__device__ __forceinline__ uint64_t blake2b_quad(uint32_t len, uint8_t *s_row, Load32 load32)
{
    const uint32_t lane = threadIdx.x & 31, c = threadIdx.x & 3;
    const uint32_t qmask = 0xFu << (lane & ~3u), qbase = lane & ~3u;
    const uint32_t msg = (uint32_t)__cvta_generic_to_shared(s_row);

    // per-round message offsets for this lane: {col x, col y, diag x, diag y} * 8 bytes
    uint32_t off[12];
#pragma unroll
    for (int r = 0; r < 12; r++)
        off[r] = ((uint32_t)c_b2_sigma[r][2 * c] << 3) | ((uint32_t)c_b2_sigma[r][2 * c + 1] << 11) |
                 ((uint32_t)c_b2_sigma[r][8 + 2 * c] << 19) | ((uint32_t)c_b2_sigma[r][8 + 2 * c + 1] << 27);
    const uint64_t IV[8] = {0x6a09e667f3bcc908ull, 0xbb67ae8584caa73bull, 0x3c6ef372fe94f82bull, 0xa54ff53a5f1d36f1ull,
                            0x510e527fade682d1ull, 0x9b05688c2b3e6c1full, 0x1f83d9abfb41bd6bull, 0x5be0cd19137e2179ull};
    const uint64_t ivlo = c == 0 ? IV[0] : (c == 1 ? IV[1] : (c == 2 ? IV[2] : IV[3]));
    const uint64_t ivhi = c == 0 ? IV[4] : (c == 1 ? IV[5] : (c == 2 ? IV[6] : IV[7]));
    uint64_t h0 = ivlo ^ (c == 0 ? 0x01010040ull : 0ull), h1 = ivhi;  // h[c], h[4+c]

    uint4 nx, ny;
    load32(0, nx, ny);
    uint32_t o = 0;
    for (;;) {
        const bool last = len - o <= 128;  // also true for an empty message
        __syncwarp(qmask);                  // previous block's words are no longer needed
        *reinterpret_cast<uint4 *>(s_row + 32 * c) = nx;
        *reinterpret_cast<uint4 *>(s_row + 32 * c + 16) = ny;
        __syncwarp(qmask);
        if (!last) load32(o + 128, nx, ny);  // prefetch the next block
        const uint64_t t = last ? (uint64_t)len : (uint64_t)o + 128;
        uint64_t va = h0, vb = h1, vc = ivlo, vd = ivhi;
        if (c == 0) vd ^= t;
        if (c == 2 && last) vd = ~vd;
#pragma unroll
        for (int r = 0; r < 12; r++) {
            const uint32_t f = off[r];
            uint64_t mx = lds_u64(msg + (f & 0xff)), my = lds_u64(msg + ((f >> 8) & 0xff));
            GEC_B2_G(va, vb, vc, vd, mx, my);
            vb = shfl64(qmask, vb, qbase + ((c + 1) & 3));
            vc = shfl64(qmask, vc, qbase + ((c + 2) & 3));
            vd = shfl64(qmask, vd, qbase + ((c + 3) & 3));
            mx = lds_u64(msg + ((f >> 16) & 0xff));
            my = lds_u64(msg + (f >> 24));
            GEC_B2_G(va, vb, vc, vd, mx, my);
            vb = shfl64(qmask, vb, qbase + ((c + 3) & 3));
            vc = shfl64(qmask, vc, qbase + ((c + 2) & 3));
            vd = shfl64(qmask, vd, qbase + ((c + 1) & 3));
        }
        h0 ^= va ^ vc;
        h1 ^= vb ^ vd;
        if (last) break;
        o += 128;
    }
    return h0;
}

__global__ void __launch_bounds__(kQuadThreads) blake2sum_shards_quad_kernel(const __grid_constant__ SumParams q)
{
    // 144-byte pitch: consecutive quads start 4 banks apart (a 128-byte pitch puts the same word
    // of all 8 quads of a warp in the same bank: 8-way conflicts on every message load)
    __shared__ __align__(16) uint8_t s_msg[kQuadThreads / 4][144];
    const uint32_t tid = threadIdx.x, lane = tid & 31, c = tid & 3;
    const uint32_t i = blockIdx.x * (kQuadThreads / 4) + (tid >> 2);  // shard index
    if (i >= q.n_shards) return;                                      // whole quads leave together
    const uint32_t qmask = 0xFu << (lane & ~3u);
    const uint8_t *p;
    uint32_t len;
    size_t oi;
    if (!locate_shard(q, i, p, len, oi)) {  // the same for the whole quad: it leaves together
        if (c == 0 && q.expect && q.bad) q.bad[oi] = 1;
        return;
    }

    // this lane's 32 bytes of the shard starting at byte `o` (zero beyond len)
    auto load32 = [&](uint32_t o, uint4 &x, uint4 &y) {
        x = make_uint4(0, 0, 0, 0);
        y = make_uint4(0, 0, 0, 0);
        const uint32_t a0 = o + 32 * c;
        if (a0 < len) {
            x = *reinterpret_cast<const uint4 *>(p + a0);
            if (len - a0 < 16) x = mask_tail(x, len - a0);
        }
        if (a0 + 16 < len) {
            y = *reinterpret_cast<const uint4 *>(p + a0 + 16);
            if (len - a0 - 16 < 16) y = mask_tail(y, len - a0 - 16);
        }
    };
    const uint64_t h0 = blake2b_quad(len, &s_msg[tid >> 2][0], load32);
    if (q.sums) *reinterpret_cast<unsigned long long *>(q.sums + oi * 32 + 8 * c) = h0;
    if (q.expect && q.bad) {
        const unsigned long long e = *reinterpret_cast<const unsigned long long *>(q.expect + oi * 32 + 8 * c);
        const uint32_t diff = __ballot_sync(qmask, e != h0) & qmask;
        if (c == 0) q.bad[oi] = diff ? 1 : 0;
    }
}

// ---- blake2sum of whole blocks, read from their data shards (deep scrub, DESIGN.md 4.7) -------------------------
// The block is the first block_len bytes of data shards 0..k-1 concatenated (DESIGN.md 2.3): block byte o is byte
// o % L of shard o / L, L = code_shard_len.  One quad per stripe, as in blake2sum_shards_quad_kernel.  Bytes of a
// shard at [L, stride) are not part of the block and never enter the hash.
struct BlockSumParams {
    const uint8_t *shards;        // stripe s at shards + s*(k+m)*stride, shard i at + i*stride
    const uint32_t *block_len;    // per stripe
    const uint8_t *hashes;        // 32 bytes per stripe: the content address
    uint8_t *hash_bad;            // out: 1 iff the block's blake2sum differs from hashes[s]
    uint32_t *shard_len;          // out: L, or 0 for a stripe whose L does not fit its stride
    uint32_t *mismatch;           // out: 0, or every parity bit for such a stripe (the verify launch ORs into it)
    uint8_t *digest;              // out, nullable: 32 bytes per stripe, the block's blake2sum (hashes, hash_bad,
                                  // shard_len and mismatch are then nullable too)
    uint32_t stride, k, m, n, quantum;
};

// 16 block bytes at offset `off` of data shard `j`, `nvalid` of them valid (zero past that).  Inside one shard at a
// 16-byte aligned offset: one vector load; inside one shard elsewhere: five aligned 32-bit loads and funnel shifts
// (as in split_blocks_kernel; the words stay inside roundup4(off + 16) <= roundup16(L)); only the one vector that
// crosses into the next shard -- or several shards when L < 16 -- is gathered byte by byte.
__device__ __forceinline__ uint4 block_vec16(const uint8_t *stripe, uint32_t stride, uint32_t L, uint32_t j,
                                             uint32_t off, uint32_t nvalid)
{
    if (!nvalid) return make_uint4(0, 0, 0, 0);
    const uint8_t *p = stripe + (size_t)j * stride;
    uint4 v;
    if (off + 16 <= L) {
        if (!(off & 15)) {
            v = __ldg(reinterpret_cast<const uint4 *>(p + off));
        } else {
            const uint32_t sh = (off & 3u) * 8;
            const uint32_t *wp = reinterpret_cast<const uint32_t *>(p + (off & ~3u));
            const uint32_t w0 = __ldg(wp), w1 = __ldg(wp + 1), w2 = __ldg(wp + 2), w3 = __ldg(wp + 3),
                           w4 = sh ? __ldg(wp + 4) : 0;
            v = make_uint4(__funnelshift_r(w0, w1, sh), __funnelshift_r(w1, w2, sh), __funnelshift_r(w2, w3, sh),
                           __funnelshift_r(w3, w4, sh));
        }
        return nvalid < 16 ? mask_tail(v, nvalid) : v;
    }
    uint32_t wv[4] = {0, 0, 0, 0};
#pragma unroll
    for (int b = 0; b < 16; b++) {
        if ((uint32_t)b < nvalid) {
            uint32_t ob = off + b, jb = j;
            if (ob >= L) {  // crossed into the next shard(s)
                jb += ob / L;
                ob %= L;
            }
            wv[b >> 2] |= (uint32_t)stripe[(size_t)jb * stride + ob] << (8 * (b & 3));
        }
    }
    return make_uint4(wv[0], wv[1], wv[2], wv[3]);
}

__global__ void __launch_bounds__(kQuadThreads) blake2sum_blocks_kernel(const __grid_constant__ BlockSumParams q)
{
    __shared__ __align__(16) uint8_t s_msg[kQuadThreads / 4][144];  // 144-byte pitch: see the shard kernel
    const uint32_t tid = threadIdx.x, lane = tid & 31, c = tid & 3;
    const uint32_t s = blockIdx.x * (kQuadThreads / 4) + (tid >> 2);  // stripe index
    if (s >= q.n) return;                                             // whole quads leave together
    const uint32_t qmask = 0xFu << (lane & ~3u);
    const uint32_t len = __ldg(q.block_len + s);
    const uint64_t L64 = code_shard_len(len, (int)q.k, q.quantum);
    const bool bad_geo = L64 > q.stride;  // DEVICE mode reports it; nothing of the stripe is read
    const uint32_t L = bad_geo ? 0u : (uint32_t)L64;
    if (c == 0 && q.shard_len) {
        q.shard_len[s] = L;
        q.mismatch[s] = bad_geo ? (1u << q.m) - 1 : 0u;
    }
    if (bad_geo) {
        if (c == 0 && q.hash_bad) q.hash_bad[s] = 1;
        return;
    }
    const uint8_t *stripe = q.shards + (size_t)s * (q.k + q.m) * q.stride;
    // this lane's 32 block bytes at o + 32c, as two 16-byte vectors; zero past block_len
    auto load32 = [&](uint32_t o, uint4 &x, uint4 &y) {
        const uint32_t a0 = o + 32 * c;
        uint32_t j = 0, off = 0;
        if (a0 < len) {  // L >= 1 here
            j = a0 / L;
            off = a0 - j * L;
        }
        const uint32_t nx = a0 < len ? min(16u, len - a0) : 0u, ny = a0 + 16 < len ? min(16u, len - a0 - 16) : 0u;
        x = block_vec16(stripe, q.stride, L, j, off, nx);
        if (ny && off + 16 >= L) {  // the second vector starts in the next shard
            off = off + 16 - L;
            j++;
        } else {
            off += 16;
        }
        y = block_vec16(stripe, q.stride, L, j, off, ny);
    };
    const uint64_t h0 = blake2b_quad(len, &s_msg[tid >> 2][0], load32);
    if (q.digest) *reinterpret_cast<unsigned long long *>(q.digest + (size_t)s * 32 + 8 * c) = h0;
    if (!q.hashes) return;
    const unsigned long long e = *reinterpret_cast<const unsigned long long *>(q.hashes + (size_t)s * 32 + 8 * c);
    const uint32_t diff = __ballot_sync(qmask, e != h0) & qmask;
    if (c == 0) q.hash_bad[s] = diff ? 1 : 0;
}

// ------------------------------------------------------------------ block -> shard framing on the device
// rpc_put_block hands over a contiguous block (bytes::Bytes); the streaming kernels want k shards,
// `stride` apart and 16-byte aligned, the last one zero padded (DataBlock::from_buffer framing,
// src/block/block.rs:85-96; short last block src/api/s3/put.rs:583-617).  The block crosses PCIe as
// ONE contiguous copy (a pitched 2-D copy with an odd row width -- shard_len is rarely a multiple of
// 16 -- runs far below the link rate) and this kernel cuts it up at HBM speed: every thread
// produces one 16-byte vector of one shard from an arbitrarily aligned source position (five
// aligned 32-bit loads + funnel shifts), zero beyond the shard / the block.
struct SplitParams {
    const uint8_t *blocks;       // block s at blocks + s*block_pitch (16-byte aligned)
    const uint32_t *block_len;   // per block
    uint8_t *shards;             // shard j of block s at shards + (s*k + j)*stride
    unsigned long long block_pitch;
    uint32_t stride, k, n;
    uint32_t parts;              // CTAs per block: a dispatcher batch of a dozen blocks still has to fill every SM
    uint32_t quantum;            // shard length = ceil(len/k) rounded up to this (code_shard_len: PB 128, Clay 16*alpha)
};
__global__ void __launch_bounds__(256) split_blocks_kernel(const __grid_constant__ SplitParams q)
{
    for (uint32_t w = blockIdx.x; w < q.n * q.parts; w += gridDim.x) {
        const uint32_t s = w / q.parts, part = w - s * q.parts;
        const uint32_t len = __ldg(q.block_len + s);
        const uint32_t L = (uint32_t)code_shard_len(len, (int)q.k, q.quantum), nvec = (L + 15) >> 4;
        const uint8_t *src = q.blocks + (unsigned long long)s * q.block_pitch;
        uint8_t *dst = q.shards + (unsigned long long)s * q.k * q.stride;
        const uint32_t total = q.k * nvec, per = ((total + q.parts - 1) / q.parts + 255u) & ~255u;
        const uint32_t lo = part * per, hi = min(total, lo + per);
#pragma unroll 4
        for (uint32_t idx = lo + threadIdx.x; idx < hi; idx += 256) {
            const uint32_t j = idx / nvec, v = idx - j * nvec;
            const uint32_t pos = j * L + v * 16;  // first source byte of this vector
            // valid bytes: inside the shard and inside the block
            uint32_t nvalid = min(16u, L - v * 16);
            nvalid = pos >= len ? 0 : min(nvalid, len - pos);
            uint4 o = make_uint4(0, 0, 0, 0);
            if (nvalid) {
                const uint32_t a = pos & ~3u, sh = (pos & 3u) * 8;
                const uint32_t *wp = reinterpret_cast<const uint32_t *>(src + a);
                // words a .. a+16 hold bytes pos .. pos+15 (+ up to 3 on either side); the staging buffer is
                // padded so that reading one word past the block is always inside the allocation
                const uint32_t w0 = wp[0], w1 = wp[1], w2 = wp[2], w3 = wp[3], w4 = sh ? wp[4] : 0;
                o = make_uint4(__funnelshift_r(w0, w1, sh), __funnelshift_r(w1, w2, sh), __funnelshift_r(w2, w3, sh),
                               __funnelshift_r(w3, w4, sh));
                if (nvalid < 16) o = mask_tail(o, nvalid);
            }
            *reinterpret_cast<uint4 *>(dst + (size_t)j * q.stride + (size_t)v * 16) = o;
        }
    }
}

// ------------------------------------------------------------------ code conversion (DESIGN.md 2.3)
// A block stored under source code S is the first block_len bytes of S's data shards 0..k_s-1 concatenated (a whole
// block: k_s = 1, L_s = block_len).  The transcode to code D writes D's data shard j = block bytes [j*L_d, (j+1)*L_d),
// zero padded, gathered straight from the source data shards, and D's parities.
struct TranscodeParams {
    const uint8_t *src;          // source stripe s at src + s*src_pitch, data shard i at + i*src_stride
    const uint32_t *block_len;   // per stripe
    uint8_t *dst;                // destination shard i of stripe s at dst + s*dst_pitch + i*dst_stride
    uint32_t *src_len, *dst_len; // per stripe: L_s, L_d (0 for a stripe that is skipped)
    int32_t *geo;                // per stripe: GARAGE_EC_E_INVALID if a length does not fit its stride, else 0
    int32_t *status;             // per stripe, out
    const int32_t *rec_status;   // nullable: verdict of the source reconstruct (== status when set)
    unsigned long long src_pitch, dst_pitch;
    uint32_t src_stride, dst_stride;
    uint32_t ks, kd;             // data shards of the source (1: whole blocks) and destination codes
    uint32_t src_whole;          // 1: the source is the block itself, L_s = block_len
    uint32_t src_quantum, dst_quantum;  // code_shard_len rounding of each code (1 for RS and LRC)
    uint32_t n, parts;           // parts: reframe CTAs per stripe
};
// per-stripe lengths and their geometry verdict; runs before the source reconstruct, which needs L_s
__global__ void __launch_bounds__(256) transcode_lens_kernel(const __grid_constant__ TranscodeParams q)
{
    for (uint32_t s = blockIdx.x * blockDim.x + threadIdx.x; s < q.n; s += gridDim.x * blockDim.x) {
        const uint32_t len = __ldg(q.block_len + s);
        const uint64_t ls = q.src_whole ? len : code_shard_len(len, (int)q.ks, q.src_quantum);
        const uint64_t ld = code_shard_len(len, (int)q.kd, q.dst_quantum);
        const bool bad = ls > q.src_stride || ld > q.dst_stride;
        q.geo[s] = bad ? GARAGE_EC_E_INVALID : 0;
        q.src_len[s] = bad ? 0u : (uint32_t)ls;  // a reconstruct of an empty stripe touches nothing
        q.dst_len[s] = bad ? 0u : (uint32_t)ld;
        if (!q.rec_status) q.status[s] = q.geo[s];
    }
}
// Stripe s failed (geometry, or an unrecoverable source): true, and one caller (`first`) records it -- the status, and
// dst_len = 0, so that the encode and tag launches write nothing for the stripe.  No caller reads dst_len of a failed
// stripe.
__device__ __forceinline__ bool transcode_failed(const TranscodeParams &q, uint32_t s, bool first)
{
    const int32_t geo = q.geo[s];
    const int32_t verdict = geo ? geo : (q.rec_status ? q.rec_status[s] : 0);
    if (verdict && first) {
        if (geo) q.status[s] = geo;  // else status already holds the reconstruct's verdict
        q.dst_len[s] = 0;
    }
    return verdict != 0;
}
// Vector v of destination data row j of one stripe (src = the stripe's source base).  A vector inside one source
// piece comes from five aligned 32-bit loads and funnel shifts (as in split_blocks_kernel); one that crosses a piece
// boundary or ends the row is gathered byte by byte.
__device__ __forceinline__ uint4 transcode_gather(const uint8_t *src, uint32_t src_stride, uint32_t Ls, uint32_t Ld,
                                                  uint32_t len, uint32_t j, uint32_t v)
{
    const uint64_t pos = (uint64_t)j * Ld + v * 16;  // block offset of the vector's first byte
    uint32_t nvalid = min(16u, Ld - v * 16);
    nvalid = pos >= len ? 0 : (uint32_t)min((uint64_t)nvalid, len - pos);
    if (!nvalid) return make_uint4(0, 0, 0, 0);
    const uint32_t p32 = (uint32_t)pos;  // < block_len: 32-bit division
    const uint32_t i = p32 / Ls, off = p32 - i * Ls;
    if (nvalid == 16 && off + 16 <= Ls) {
        // words a .. a+16 stay inside roundup4(off + 16) <= roundup16(L_s): readable
        const uint32_t a = off & ~3u, sh = (off & 3u) * 8;
        const uint32_t *wp = reinterpret_cast<const uint32_t *>(src + (size_t)i * src_stride + a);
        const uint32_t w0 = __ldg(wp), w1 = __ldg(wp + 1), w2 = __ldg(wp + 2), w3 = __ldg(wp + 3), w4 = sh ? __ldg(wp + 4) : 0;
        return make_uint4(__funnelshift_r(w0, w1, sh), __funnelshift_r(w1, w2, sh), __funnelshift_r(w2, w3, sh),
                          __funnelshift_r(w3, w4, sh));
    }
    uint32_t wv[4] = {0, 0, 0, 0};
#pragma unroll
    for (int b = 0; b < 16; b++) {
        if ((uint32_t)b < nvalid) {
            const uint32_t ob = p32 + b;
            const uint32_t ib = ob / Ls, offb = ob - ib * Ls;
            wv[b >> 2] |= (uint32_t)src[(size_t)ib * src_stride + offb] << (8 * (b & 3));
        }
    }
    return make_uint4(wv[0], wv[1], wv[2], wv[3]);
}
// The destination data shards, one vector per thread; the destination's own encode follows (DESIGN.md 4.5: a one-pass
// kernel that also looked the gathered vectors up in the parity tables measured no faster).
__global__ void __launch_bounds__(256) transcode_reframe_kernel(const __grid_constant__ TranscodeParams q)
{
    for (uint32_t w = blockIdx.x; w < q.n * q.parts; w += gridDim.x) {
        const uint32_t s = w / q.parts, part = w - s * q.parts;
        if (transcode_failed(q, s, part == 0 && threadIdx.x == 0)) continue;
        const uint32_t len = __ldg(q.block_len + s), Ls = q.src_len[s], Ld = q.dst_len[s], nvec = (Ld + 15) >> 4;
        const uint8_t *src = q.src + (unsigned long long)s * q.src_pitch;
        uint8_t *dst = q.dst + (unsigned long long)s * q.dst_pitch;
        const uint32_t total = q.kd * nvec, per = ((total + q.parts - 1) / q.parts + 255u) & ~255u;
        const uint32_t lo = part * per, hi = min(total, lo + per);
#pragma unroll 4
        for (uint32_t idx = lo + threadIdx.x; idx < hi; idx += 256) {
            const uint32_t j = idx / nvec, v = idx - j * nvec;
            *reinterpret_cast<uint4 *>(dst + (size_t)j * q.dst_stride + (size_t)v * 16) =
                transcode_gather(src, q.src_stride, Ls, Ld, len, j, v);
        }
    }
}
// ---- fast per-shard integrity tag: 8 x Adler-32 ("adler8") -----------------------------------
// BLAKE2b is compute-bound on CUDA cores (~20 integer instructions per byte: at most ~1.3 TB/s,
// round 1 measured 0.45-0.6 TB/s), which capped the scrub sweep at 7 % of HBM bandwidth.  Scrub
// only has to catch bit rot (the block's content address stays Garage's blake2sum), so the shard
// files may carry a cheap tag instead: the shard is cut in 8 segments of
// seg = roundup16(ceil(len / 8)) bytes and the tag is the 8 little-endian zlib Adler-32 values of
// the segments (an empty segment has Adler-32 = 1) -- 32 bytes, the size of Garage's `Hash`.
// Adler-32 is a = 1 + sum d_i, b = n + sum (n - i) d_i (mod 65521): plain byte sums, 4 DP4A per 16
// bytes for each, so the kernel streams at HBM speed; one warp per shard, four 16-byte loads per
// lane in flight.  Pinned by python's zlib.adler32 (tests/test_blake2.py).
constexpr uint32_t kAdlerMod = 65521;

__global__ void __launch_bounds__(256) adler8_shards_kernel(const __grid_constant__ SumParams q)
{
    // (a block-per-segment variant, 256 threads on one contiguous ~20 KB region + a shared-memory reduction, measured
    // slower)
    // work unit = one SEGMENT of one shard per warp (8 units per shard): 8x the units of a warp-per-shard
    // split, so the persistent grid stays balanced down to a few hundred shards (ncu of the warp-per-shard
    // version: 50 % of DRAM peak with a 2-wave tail at 18 432 shards).  `bad` must be zero on entry when
    // `expect` is given (the host memsets it): segments OR their verdict into the shard's flag byte.
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t wpb = blockDim.x >> 5;
    const uint32_t units = q.n_shards * 8u;  // host guarantees n_shards < 2^29
    for (uint32_t u = blockIdx.x * wpb + (threadIdx.x >> 5); u < units; u += gridDim.x * wpb) {
        const uint32_t i = u >> 3, sgi = u & 7;
        const uint8_t *p;
        uint32_t len;
        size_t oi;
        const bool ok = locate_shard(q, i, p, len, oi);  // warp-uniform: one unit per warp
        const uint32_t seg = adler8_seg_bytes(len);
        const uint32_t start = sgi * seg;
        uint32_t tag = 1;  // Adler-32 of an empty segment
        if (ok && start < len) {
            const uint32_t end = min(len, start + seg), n = end - start;
            unsigned long long A = 0, B = 0, T = 0;
            // 8 vectors per lane in flight: rel = byte offset of the vector inside the segment
            for (uint32_t r0 = lane * 16; r0 < n; r0 += 8 * 512) {
                uint4 v[8];
#pragma unroll
                for (int k = 0; k < 8; k++) {
                    const uint32_t rel = r0 + k * 512;
                    v[k] = make_uint4(0, 0, 0, 0);
                    if (rel < n) {
                        v[k] = ldg_stream(p + start + rel);  // within roundup16(len): readable
                        if (n - rel < 16) v[k] = mask_tail(v[k], n - rel);
                    }
                }
#pragma unroll
                for (int k = 0; k < 8; k++) {
                    const uint32_t rel = r0 + k * 512;
                    uint32_t sm = __dp4a(v[k].x, 0x01010101u, 0u);
                    sm = __dp4a(v[k].y, 0x01010101u, sm);
                    sm = __dp4a(v[k].z, 0x01010101u, sm);
                    sm = __dp4a(v[k].w, 0x01010101u, sm);
                    uint32_t t = __dp4a(v[k].x, 0x03020100u, 0u);  // sum_j j * byte_j
                    t = __dp4a(v[k].y, 0x07060504u, t);
                    t = __dp4a(v[k].z, 0x0b0a0908u, t);
                    t = __dp4a(v[k].w, 0x0f0e0d0cu, t);
                    A += sm;
                    if (rel < n) B += (unsigned long long)(n - rel) * sm;
                    T += t;
                }
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                A += __shfl_xor_sync(0xffffffffu, A, o);
                B += __shfl_xor_sync(0xffffffffu, B, o);
                T += __shfl_xor_sync(0xffffffffu, T, o);
            }
            const uint32_t a = (uint32_t)((1 + A) % kAdlerMod);
            const uint32_t b = (uint32_t)((n + B - T) % kAdlerMod);  // B >= T: (n - rel) >= j + 1 for every byte
            tag = (b << 16) | a;
        }
        if (lane == 0) {
            if (ok && q.sums) reinterpret_cast<uint32_t *>(q.sums + oi * 32)[sgi] = tag;
            if (q.expect && q.bad && (!ok || reinterpret_cast<const uint32_t *>(q.expect + oi * 32)[sgi] != tag)) {
                // set byte `oi` of bad[] to 1 through the aligned 32-bit word that contains it
                const unsigned long long addr = reinterpret_cast<unsigned long long>(q.bad + oi);
                atomicOr(reinterpret_cast<unsigned int *>(addr & ~3ull), 1u << (8 * (unsigned)(addr & 3ull)));
            }
        }
    }
}

// ------------------------------------------------------------------ ranged reads (DESIGN.md 2.5)
// Block byte o is byte c = o % L of data shard o / L.  Every code here is column-local: byte c of a rebuilt shard
// depends on the survivors only at the bytes of the same window coordinate, c (RS, LRC), c mod L/2 (PB: a-half column
// c pairs with b-half column c) or c mod L/alpha (Clay: the in-layer column across all alpha layers).  With unit = L,
// L/2 or L/alpha, a shard is L/unit runs of `unit` bytes; the window [w0, w0 + w) is the smallest 16-byte aligned
// interval (capped at unit) covering the window coordinates of the range's bytes in absent data shards.  The
// sub-stripe holds the window of every run of every shard, run z at z*w: a stripe of shard length (L/unit)*w that the
// code's own decode rebuilds into exactly the window of the full decode.
struct RangeWindow {
    uint32_t L, unit, w0, w;  // w = 0: no touched data shard is absent
    uint64_t want;            // the absent touched data shards
};
__host__ __device__ inline uint32_t range_unit(uint32_t L, bool pb, uint32_t alpha)
{
    return pb ? L / 2 : L / alpha;  // alpha = 1 for RS, LRC and PB
}
// present: the stripe's k+m map; off + len <= block_len is the caller's check
__host__ __device__ inline RangeWindow range_window(uint32_t L, uint32_t unit, uint64_t off, uint64_t len,
                                                    const uint8_t *present)
{
    RangeWindow r{L, unit, 0, 0, 0};
    if (!len || !unit) return r;
    uint64_t lo = unit, hi = 0;
    const uint64_t end = off + len;
    for (uint64_t j = off / L; j * L < end; j++) {
        if (present[j]) continue;
        r.want |= 1ull << j;
        const uint64_t base = j * L, c0 = (off > base ? off : base) - base, c1 = (end < base + L ? end : base + L) - base;
        if (c1 - c0 >= unit || c0 / unit != (c1 - 1) / unit) {  // wraps around a run: every window coordinate
            lo = 0;
            hi = unit;
        } else {
            lo = c0 % unit < lo ? c0 % unit : lo;
            hi = (c1 - 1) % unit + 1 > hi ? (c1 - 1) % unit + 1 : hi;
        }
    }
    if (!r.want) return r;
    r.w0 = (uint32_t)(lo & ~15ull);
    const uint64_t w1 = (hi + 15) & ~15ull;
    r.w = (uint32_t)((w1 < unit ? w1 : unit) - r.w0);
    return r;
}

struct RangeParams {
    const uint8_t *shards;          // the caller's shard layout: request s reads stripe s >> shift at
                                    // shards + (s >> shift)*pitch, shard i at + i*stride
    uint8_t *sub;                   // the sub-stripes, same layout (a window never exceeds its shard)
    const uint8_t *present;         // n*(k+m)
    const uint32_t *block_len, *offset, *len;  // per request
    uint8_t *out;                   // request s at out + s*out_stride
    uint4 *geo;                     // per request: L, unit (0: invalid request), w0, w
    uint32_t *sub_len;              // per request: (L/unit)*w, the sub-stripe's shard length
    uint8_t *want;                  // n*(k+m): the absent touched data shards
    const int32_t *plan_status;     // the decode's status of the sub-stripes
    int32_t *status;                // nullable, out
    unsigned long long pitch, out_stride;
    uint32_t stride, k, m, n, quantum, alpha, pb, shift;
};

// one thread per request: the window, the decode's want map and sub-stripe length
__global__ void __launch_bounds__(256) range_geo_kernel(const __grid_constant__ RangeParams q)
{
    const uint32_t tot = q.k + q.m;
    for (uint32_t s = blockIdx.x * blockDim.x + threadIdx.x; s < q.n; s += gridDim.x * blockDim.x) {
        const uint32_t blen = __ldg(q.block_len + s), off = __ldg(q.offset + s), len = __ldg(q.len + s);
        const uint64_t L64 = code_shard_len(blen, (int)q.k, q.quantum);
        const bool bad = L64 > q.stride || (uint64_t)off + len > blen;
        RangeWindow r{0, 0, 0, 0, 0};
        if (!bad) {
            const uint32_t L = (uint32_t)L64;
            r = range_window(L, range_unit(L, q.pb != 0, q.alpha), off, len, q.present + (size_t)s * tot);
            r.unit = r.unit ? r.unit : 1u;  // a valid empty block
        }
        q.geo[s] = make_uint4(r.L, r.unit, r.w0, r.w);
        q.sub_len[s] = r.w ? (r.L / r.unit) * r.w : 0u;
        for (uint32_t i = 0; i < tot; i++) q.want[(size_t)s * tot + i] = (uint8_t)((r.want >> i) & 1);
    }
}

// The window runs of every present shard into the sub-stripes, one 16-byte vector per thread (window starts are
// 16-byte aligned; the last vector of an RS / LRC run may read past the window, inside roundup16(L) <= stride).
// CTAs walk the requests.
__global__ void __launch_bounds__(256) range_pack_kernel(const __grid_constant__ RangeParams q)
{
    const uint32_t tot = q.k + q.m;
    for (uint32_t s = blockIdx.x; s < q.n; s += gridDim.x) {
        const uint4 g = q.geo[s];
        if (!g.w) continue;
        const uint32_t nz = g.x / g.y, nv = (g.w + 15) >> 4, per = nz * nv;
        const uint8_t *src = q.shards + (s >> q.shift) * q.pitch, *pr = q.present + (size_t)s * tot;
        uint8_t *dst = q.sub + s * q.pitch;
        for (uint32_t idx = threadIdx.x; idx < tot * per; idx += blockDim.x) {
            const uint32_t i = idx / per, r = idx - i * per, z = r / nv, v = r - z * nv;
            if (!pr[i]) continue;
            const uint4 x = __ldg(reinterpret_cast<const uint4 *>(src + (size_t)i * q.stride + z * g.y + g.z + 16 * v));
            *reinterpret_cast<uint4 *>(dst + (size_t)i * q.stride + z * g.w + 16 * v) = x;
        }
    }
}

// Where block byte o of request s lives: in the caller's layout for a present shard, in the rebuilt sub-stripe for an
// absent one; *rem = the bytes from there to the end of that contiguous piece.
__device__ __forceinline__ const uint8_t *range_src(const RangeParams &q, uint32_t s, const uint4 &g, uint32_t o,
                                                    uint32_t *rem)
{
    const uint32_t j = o / g.x, c = o - j * g.x;
    if (q.present[(size_t)s * (q.k + q.m) + j]) {
        *rem = g.x - c;
        return q.shards + (s >> q.shift) * q.pitch + (size_t)j * q.stride + c;
    }
    const uint32_t z = c / g.y, cc = c - z * g.y;
    *rem = g.z + g.w - cc;
    return q.sub + s * q.pitch + (size_t)j * q.stride + z * g.w + (cc - g.z);
}

// Every request's bytes into out, 16 per thread, zero past len up to roundup16(len).  A vector inside one piece is one
// aligned vector load, or five aligned 32-bit loads and funnel shifts (as block_vec16: the words stay inside the
// piece's 16-byte rounding); a vector whose 16 bytes would run past the end of its piece -- one that crosses a shard,
// PB half or Clay layer edge, or the range's last vector near such an edge -- is gathered byte by byte.  status: invalid requests GARAGE_EC_E_INVALID, requests without an absent touched data
// shard 0, the others the decode's verdict; nothing is written for a failed request.
__global__ void __launch_bounds__(256) range_join_kernel(const __grid_constant__ RangeParams q)
{
    for (uint32_t s = blockIdx.x; s < q.n; s += gridDim.x) {
        const uint4 g = q.geo[s];
        const int32_t verdict = !g.y ? GARAGE_EC_E_INVALID : (g.w ? q.plan_status[s] : 0);
        if (threadIdx.x == 0 && q.status) q.status[s] = verdict;
        if (verdict) continue;
        const uint32_t off = __ldg(q.offset + s), len = __ldg(q.len + s);
        uint8_t *dst = q.out + s * q.out_stride;
        for (uint32_t v = threadIdx.x; v < (len + 15) >> 4; v += blockDim.x) {
            const uint32_t o = off + 16 * v, nvalid = min(16u, len - 16 * v);
            uint32_t rem;
            const uint8_t *p = range_src(q, s, g, o, &rem);
            uint4 x;
            if (rem >= 16) {
                if (!(reinterpret_cast<uintptr_t>(p) & 15)) {
                    x = __ldg(reinterpret_cast<const uint4 *>(p));
                } else {
                    const uint32_t sh = (uint32_t)(reinterpret_cast<uintptr_t>(p) & 3u) * 8;
                    const uint32_t *wp = reinterpret_cast<const uint32_t *>(reinterpret_cast<uintptr_t>(p) & ~(uintptr_t)3);
                    const uint32_t w0 = __ldg(wp), w1 = __ldg(wp + 1), w2 = __ldg(wp + 2), w3 = __ldg(wp + 3),
                                   w4 = sh ? __ldg(wp + 4) : 0;
                    x = make_uint4(__funnelshift_r(w0, w1, sh), __funnelshift_r(w1, w2, sh), __funnelshift_r(w2, w3, sh),
                                   __funnelshift_r(w3, w4, sh));
                }
                if (nvalid < 16) x = mask_tail(x, nvalid);
            } else {
                uint32_t wv[4] = {0, 0, 0, 0};
#pragma unroll
                for (int b = 0; b < 16; b++) {
                    if ((uint32_t)b < nvalid) {
                        uint32_t rb;
                        wv[b >> 2] |= (uint32_t)*range_src(q, s, g, o + b, &rb) << (8 * (b & 3));
                    }
                }
                x = make_uint4(wv[0], wv[1], wv[2], wv[3]);
            }
            *reinterpret_cast<uint4 *>(dst + 16 * (size_t)v) = x;
        }
    }
}

}  // namespace garage_ec
