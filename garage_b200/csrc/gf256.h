// gf256.h -- GF(2^8)/0x11D arithmetic shared by host (matrix construction) and device
// (table build, decode planning).  Product code: does NOT use anything under oracle/.
//
// Field definition: SURVEY.md section 8(c) / DESIGN.md "Field".  The reference has no
// counterpart (no RS code in deuxfleurs-org/garage); the framing it imposes is cited where
// it matters (rs_kernels.cuh, garage_ec.cu).
#pragma once
#include <stdint.h>

#include "gf256_tables.inc"

#define GARAGE_EC_MAX_K_HOST 32
#define GARAGE_EC_MAX_M_HOST 8

#ifdef __CUDACC__
#define GEC_GF_HD __host__ __device__
#else
#define GEC_GF_HD
#endif

namespace garage_ec {

// host copies
static const uint8_t h_gf_exp[512] = GARAGE_EC_GF_EXP_INIT;
static const uint8_t h_gf_log[256] = GARAGE_EC_GF_LOG_INIT;

inline uint8_t h_mul(uint8_t a, uint8_t b)
{
    return (a && b) ? h_gf_exp[h_gf_log[a] + h_gf_log[b]] : 0;
}
inline uint8_t h_inv(uint8_t a) { return h_gf_exp[255 - h_gf_log[a]]; }

// In-place Gauss-Jordan inversion of an n x n matrix; false if singular.
inline bool h_invert(uint8_t *M, int n)
{
    uint8_t w[GARAGE_EC_MAX_K_HOST * 2 * GARAGE_EC_MAX_K_HOST];
    const int W = 2 * n;
    for (int r = 0; r < n; r++)
        for (int c = 0; c < W; c++) w[r * W + c] = c < n ? M[r * n + c] : (uint8_t)(c - n == r);
    for (int c = 0; c < n; c++) {
        int piv = -1;
        for (int r = c; r < n; r++)
            if (w[r * W + c]) { piv = r; break; }
        if (piv < 0) return false;
        if (piv != c)
            for (int x = 0; x < W; x++) {
                uint8_t t = w[c * W + x];
                w[c * W + x] = w[piv * W + x];
                w[piv * W + x] = t;
            }
        const uint8_t iv = h_inv(w[c * W + c]);
        for (int x = 0; x < W; x++) w[c * W + x] = h_mul(w[c * W + x], iv);
        for (int r = 0; r < n; r++) {
            const uint8_t f = w[r * W + c];
            if (r == c || !f) continue;
            for (int x = 0; x < W; x++) w[r * W + x] ^= h_mul(f, w[c * W + x]);
        }
    }
    for (int r = 0; r < n; r++)
        for (int c = 0; c < n; c++) M[r * n + c] = w[r * W + n + c];
    return true;
}

// Parity rows P (m x k).  kind 0: systematic Vandermonde, V[r][c] = r^c (0^0 = 1),
// P = V[k..k+m) * inv(V[0..k)).  kind 1: Cauchy, P[i][j] = 1/((k+i)^j).
inline bool h_build_matrix(int k, int m, int kind, uint8_t *P)
{
    if (kind == 1) {
        for (int i = 0; i < m; i++)
            for (int j = 0; j < k; j++) P[i * k + j] = h_inv((uint8_t)((k + i) ^ j));
        return true;
    }
    if (kind != 0) return false;
    uint8_t V[(GARAGE_EC_MAX_K_HOST + GARAGE_EC_MAX_M_HOST) * GARAGE_EC_MAX_K_HOST];
    uint8_t T[GARAGE_EC_MAX_K_HOST * GARAGE_EC_MAX_K_HOST];
    for (int r = 0; r < k + m; r++) {
        uint8_t p = 1;
        for (int c = 0; c < k; c++) {
            V[r * k + c] = p;
            p = h_mul(p, (uint8_t)r);
        }
    }
    for (int i = 0; i < k * k; i++) T[i] = V[i];
    if (!h_invert(T, k)) return false;
    for (int i = 0; i < m; i++)
        for (int j = 0; j < k; j++) {
            uint8_t acc = 0;
            for (int x = 0; x < k; x++) acc ^= h_mul(V[(k + i) * k + x], T[x * k + j]);
            P[i * k + j] = acc;
        }
    return true;
}

// LRC(k, l, r) parity rows (DESIGN.md section 2): l local rows (row g = 1 on data [g*k/l, (g+1)*k/l)), then the
// r Cauchy rows of RS(k, r).  P is (l + r) x k.
inline bool h_build_lrc(int k, int l, int r, uint8_t *P)
{
    if (k < 1 || k > GARAGE_EC_MAX_K_HOST || l < 1 || r < 1 || k % l || l + r > GARAGE_EC_MAX_M_HOST) return false;
    const int gs = k / l;
    for (int g = 0; g < l; g++)
        for (int j = 0; j < k; j++) P[g * k + j] = (uint8_t)(j / gs == g);
    return h_build_matrix(k, r, 1, P + l * k);
}

// ---- piggybacked RS, PB(k, m) (DESIGN.md section 2.2) ------------------------------------------------------------
// The k data shards form m-1 contiguous groups G_1..G_{m-1}, sizes as equal as possible, larger groups first.  The
// b-half of parity i >= 1 carries the XOR of the a-halves of G_i on top of its RS value.
constexpr int kPbMaxK = 16, kPbMinM = 2, kPbMaxM = 4;
// first data shard of group g (1 <= g <= m-1); g = m gives k
GEC_GF_HD inline int pb_group_start(int k, int m, int g)
{
    const int ng = m - 1, base = k / ng, rem = k % ng, i = g - 1;
    return i * base + (i < rem ? i : rem);
}
GEC_GF_HD inline int pb_group_of(int k, int m, int j)
{
    int g = 1;
    while (g < m - 1 && j >= pb_group_start(k, m, g + 1)) g++;
    return g;
}
// shard length of a block: ceil(block_len / k) rounded up to 128 bytes, so that both halves are 16-byte aligned and
// each half is exactly 4 of the 8 adler8 segments.  64-bit: with k = 1 a block_len near 2^32 rounds past 32 bits.
// code_shard_len: the same for every code -- ceil(block_len / k) rounded up to the code's quantum: 1 for RS and LRC,
// 128 for PB, 16 * alpha for Clay (host and device share it).
constexpr uint32_t kPbQuantum = 128;
GEC_GF_HD inline uint64_t code_shard_len(uint32_t block_len, int k, uint32_t quantum)
{
    const uint64_t L = ((uint64_t)block_len + (unsigned)k - 1) / (unsigned)k;
    return (L + quantum - 1) / quantum * quantum;
}
inline uint64_t pb_shard_len(uint32_t block_len, int k) { return code_shard_len(block_len, k, kPbQuantum); }


// Generator over half-symbols: row q = 2*shard + half (0..2(k+m)), column c = 2*data + half (0..2k).
GEC_GF_HD inline uint8_t pb_grow(int k, int m, const uint8_t *P, int q, int c)
{
    const int sh = q >> 1, h = q & 1, j = c >> 1, hc = c & 1;
    if (sh < k) return (uint8_t)(q == c);
    const int i = sh - k;
    if (hc == h) return P[i * k + j];
    return (uint8_t)(h == 1 && i >= 1 && pb_group_of(k, m, j) == i);  // the piggyback: a_j in b of parity i
}
// ---- decode planning (DESIGN.md sections 2.1, 2.2) ---------------------------------------------------------------
GEC_GF_HD inline int ctz64(uint64_t x)
{
#ifdef __CUDA_ARCH__
    return __ffsll((long long)x) - 1;
#else
    return __builtin_ctzll(x);
#endif
}
GEC_GF_HD inline int popc64(uint64_t x)
{
#ifdef __CUDA_ARCH__
    return __popcll(x);
#else
    return __builtin_popcountll(x);
#endif
}

// ---- Clay codes, Clay(k, m) (DESIGN.md section 2.4) ---------------------------------------------------------------
// q = m, t = ceil((k+m)/q), n' = q*t nodes of which s = n' - k - m are virtual (always zero), alpha = q^t layers per
// shard.  Node i sits at (x, y) = (i mod q, i div q); data shard j is node j, parity shard j is node k+s+j.  Every
// layer's uncoupled bytes are a codeword of RS(k+s, m).  Accepted: m in {2, 3, 4}, k >= 2, alpha <= 256.
constexpr int kClayMaxAlpha = 256, kClayMaxNodes = 16;
struct ClayGeo {
    int q, t, n, s, alpha;
};
GEC_GF_HD inline bool clay_geometry(int k, int m, ClayGeo *g)
{
    if (m < 2 || m > 4 || k < 2 || k > GARAGE_EC_MAX_K_HOST) return false;
    const int q = m, t = (k + m + q - 1) / q;
    int alpha = 1;
    for (int i = 0; i < t; i++) {
        alpha *= q;
        if (alpha > kClayMaxAlpha) return false;
    }
    *g = ClayGeo{q, t, q * t, q * t - k - m, alpha};
    return true;
}
// node of real shard i and back (-1: a virtual node)
GEC_GF_HD inline int clay_node(int k, int s, int i) { return i < k ? i : i + s; }
GEC_GF_HD inline int clay_shard(int k, int s, int a) { return a < k ? a : (a < k + s ? -1 : a - s); }
// The shards one stripe's decode reads (bit i = shard i), given the present and the wanted absent shards: nothing if
// no wanted shard is absent; every present shard when exactly one shard is absent and wanted (repair: only the layers
// of clay_repair_runs); else the first k present shards.  False if fewer than k shards are present (as RS).
GEC_GF_HD inline bool clay_read_set(int k, int m, uint64_t present, uint64_t want, uint64_t *read)
{
    const uint64_t all = (1ull << (k + m)) - 1;
    present &= all;
    const uint64_t absent = all & ~present;
    want &= absent;
    *read = 0;
    if (popc64(present) < k) return false;
    if (!want) return true;
    if (popc64(absent) == 1) {
        *read = present;
        return true;
    }
    uint64_t r = 0;
    for (uint64_t p = present; p && popc64(r) < k; p &= p - 1) r |= p & (~p + 1);
    *read = r;
    return true;
}

// The code a stripe is planned for: RS (l = 0), LRC(k, l, m - l) or PB(k, m) (pb), with parity rows P (m x k).  The
// planner picks survivors among generator rows: shards, or for PB the half-rows q = 2*shard + half.  Row masks have
// bit q for row q.  Rows are taken in index order, and the data rows come first and are identity rows: row q < cols()
// is e_q.  plan_kernel and h_read_plan share everything here.
struct PlanCode {
    int k, m, l;
    bool pb;
    const uint8_t *P;

    GEC_GF_HD int cols() const { return pb ? 2 * k : k; }
    GEC_GF_HD uint8_t row(int q, int c) const
    {
        if (pb) return pb_grow(k, m, P, q, c);
        return q < k ? (uint8_t)(q == c) : P[(q - k) * k + c];
    }
    // shard mask -> row mask (PB: both halves of every shard)
    GEC_GF_HD uint64_t shard_rows(uint64_t shards) const
    {
        if (!pb) return shards;
        uint64_t r = 0;
        for (; shards; shards &= shards - 1) r |= 3ull << (2 * ctz64(shards));
        return r;
    }
    // The rows the survivors are picked from, given the present shards and the wanted absent shards: the present
    // rows, or only those of rule 1 when it applies.
    //   LRC (local repair): every wanted shard is a data shard or a local parity and the only absent member of its
    //     group (the group's data plus its local parity): the other members of those groups.  Holds for want = 0.
    //   PB (piggyback repair): the only wanted shard is a data shard j of G_i, every other data shard is present and
    //     so are parities 0 and i: the b-halves of the other data shards and of parities 0 and i, and the a-halves
    //     of G_i \ {j}, k + |G_i| halves (P[0][j] != 0 gives b_j).
    // RS has no rule 1.  Rule 1 rows are independent, so the greedy basis keeps them all.
    GEC_GF_HD uint64_t candidate_rows(uint64_t present, uint64_t want) const
    {
        if (l) {
            const int gs = k / l;
            uint64_t r = 0;
            for (uint64_t w = want; w; w &= w - 1) {
                const int o = ctz64(w);
                if (o >= k + l) return present;
                const int g = o < k ? o / gs : o - k;
                const uint64_t gm = (((1ull << gs) - 1) << (g * gs)) | (1ull << (k + g));
                if ((gm & ~present) != (1ull << o)) return present;
                r |= gm & ~(1ull << o);
            }
            return r;
        }
        const uint64_t all = shard_rows(present), data = (1ull << k) - 1;
        if (!pb || !want || (want & (want - 1)) || !(want & data)) return all;
        const int j = ctz64(want), g = pb_group_of(k, m, j);
        if ((present & data) != (data & ~want) || !((present >> k) & 1) || !((present >> (k + g)) & 1)) return all;
        uint64_t r = (1ull << (2 * k + 1)) | (1ull << (2 * (k + g) + 1));
        for (int x = 0; x < k; x++)
            if (x != j) r |= 1ull << (2 * x + 1);
        for (int x = pb_group_start(k, m, g); x < pb_group_start(k, m, g + 1); x++)
            if (x != j) r |= 1ull << (2 * x);
        return r;
    }
    // RS reports a stripe with fewer than k present shards unrecoverable even when nothing is wanted (garage_ec.h);
    // LRC and PB judge the wanted rows only.
    GEC_GF_HD bool below_k(uint64_t present) const { return !l && !pb && popc64(present) < k; }
};

// Survivors of one stripe, the host twin of plan_kernel (DESIGN.md section 2).  Bit i of present / want: shard i
// present / wanted (only absent wanted shards are rebuilt).  *rows = the rows to read: the greedy rank basis, in row
// order, of the candidate rows.  False if a wanted row is outside its span.
inline bool h_read_plan(const PlanCode &c, uint64_t present, uint64_t want, uint64_t *rows)
{
    static_assert(2 * kPbMaxK <= GARAGE_EC_MAX_K_HOST, "PB columns");
    const int K = c.cols();
    const uint64_t all = (1ull << (c.k + c.m)) - 1;
    present &= all;
    want &= all & ~present;
    uint8_t R[GARAGE_EC_MAX_K_HOST][GARAGE_EC_MAX_K_HOST], v[GARAGE_EC_MAX_K_HOST];
    int piv[GARAGE_EC_MAX_K_HOST], nb = 0;
    // row q reduced against the basis into v; returns its first nonzero column, K if it lies in the span
    auto reduce = [&](int q) {
        for (int j = 0; j < K; j++) v[j] = c.row(q, j);
        for (int b = 0; b < nb; b++) {
            const uint8_t f = v[piv[b]];
            if (f)
                for (int j = 0; j < K; j++) v[j] ^= h_mul(f, R[b][j]);
        }
        int p = 0;
        while (p < K && !v[p]) p++;
        return p;
    };
    *rows = 0;
    for (uint64_t cm = c.candidate_rows(present, want); cm && nb < K; cm &= cm - 1) {
        const int q = ctz64(cm), p = reduce(q);
        if (p == K) continue;
        const uint8_t iv = h_inv(v[p]);
        for (int j = 0; j < K; j++) R[nb][j] = h_mul(v[j], iv);
        piv[nb++] = p;
        *rows |= 1ull << q;
    }
    for (uint64_t wm = c.shard_rows(want); wm; wm &= wm - 1)
        if (reduce(ctz64(wm)) != K) return false;
    return !c.below_k(present);
}

}  // namespace garage_ec
