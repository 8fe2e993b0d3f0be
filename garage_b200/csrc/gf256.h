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

// Survivor set of one stripe, the host twin of the plan kernels (DESIGN.md section 2).  Bit i of present / want:
// shard i present / wanted (only absent wanted shards are rebuilt).  l = 0: RS, the first k present shards.
// l > 0: LRC rule 1 (local repair) if it applies, else rule 2 (greedy rank basis in index order).  Returns false
// if a wanted shard cannot be rebuilt; *read = the shards to read.
inline bool h_read_set(int k, int m, int l, const uint8_t *P, uint64_t present, uint64_t want, uint64_t *read)
{
    const int tot = k + m;
    const uint64_t all = tot >= 64 ? ~0ull : ((1ull << tot) - 1);
    present &= all;
    want &= all & ~present;
    *read = 0;
    if (l == 0) {
        int used = 0;
        for (int i = 0; i < tot && used < k; i++)
            if ((present >> i) & 1) {
                *read |= 1ull << i;
                used++;
            }
        return used == k;
    }
    const int gs = k / l;
    auto group_mask = [&](int g) { return (((1ull << gs) - 1) << (g * gs)) | (1ull << (k + g)); };
    bool local = true;
    uint64_t rmask = 0;
    for (int o = 0; o < tot && local; o++) {
        if (!((want >> o) & 1)) continue;
        if (o >= k + l) {
            local = false;
            break;
        }
        const uint64_t gm = group_mask(o < k ? o / gs : o - k);
        if ((gm & ~present) != (1ull << o)) local = false;
        rmask |= gm & ~(1ull << o);
    }
    if (local) {
        *read = rmask;
        return true;
    }
    auto row = [&](int c, int j) -> uint8_t { return c < k ? (uint8_t)(c == j) : P[(c - k) * k + j]; };
    uint8_t R[GARAGE_EC_MAX_K_HOST][GARAGE_EC_MAX_K_HOST];
    int piv[GARAGE_EC_MAX_K_HOST], nb = 0;
    auto reduce = [&](uint8_t *v) {
        for (int b = 0; b < nb; b++) {
            const uint8_t f = v[piv[b]];
            if (f)
                for (int j = 0; j < k; j++) v[j] ^= h_mul(f, R[b][j]);
        }
    };
    for (int c = 0; c < tot && nb < k; c++) {
        if (!((present >> c) & 1)) continue;
        uint8_t v[GARAGE_EC_MAX_K_HOST];
        for (int j = 0; j < k; j++) v[j] = row(c, j);
        reduce(v);
        int p = 0;
        while (p < k && !v[p]) p++;
        if (p == k) continue;
        const uint8_t iv = h_inv(v[p]);
        for (int j = 0; j < k; j++) R[nb][j] = h_mul(v[j], iv);
        piv[nb++] = p;
        *read |= 1ull << c;
    }
    for (int o = 0; o < tot; o++) {
        if (!((want >> o) & 1)) continue;
        uint8_t v[GARAGE_EC_MAX_K_HOST];
        for (int j = 0; j < k; j++) v[j] = row(o, j);
        reduce(v);
        for (int j = 0; j < k; j++)
            if (v[j]) return false;
    }
    return true;
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
// code_shard_len: the same for every code -- ceil(block_len / k), PB rounded as above (host and device share it).
GEC_GF_HD inline uint64_t code_shard_len(uint32_t block_len, int k, bool pb)
{
    const uint64_t L = ((uint64_t)block_len + (unsigned)k - 1) / (unsigned)k;
    return pb ? (L + 127) / 128 * 128 : L;
}
inline uint64_t pb_shard_len(uint32_t block_len, int k) { return code_shard_len(block_len, k, true); }
// Generator over half-symbols: row q = 2*shard + half (0..2(k+m)), column c = 2*data + half (0..2k).
GEC_GF_HD inline uint8_t pb_grow(int k, int m, const uint8_t *P, int q, int c)
{
    const int sh = q >> 1, h = q & 1, j = c >> 1, hc = c & 1;
    if (sh < k) return (uint8_t)(q == c);
    const int i = sh - k;
    if (hc == h) return P[i * k + j];
    return (uint8_t)(h == 1 && i >= 1 && pb_group_of(k, m, j) == i);  // the piggyback: a_j in b of parity i
}
// Half-row read plan of one PB stripe (host twin of pb_plan_kernel).  Bit i of present / want: shard i present /
// wanted.  *halves: bit 2i = a-half of shard i read, bit 2i+1 = b-half.  Rule 1 when the only wanted absent shard is
// a data shard j of G_i, every other data shard is present and so are parities 0 and i; rule 2 (greedy rank basis of
// the present half-rows in q order) otherwise.  False if a wanted shard cannot be rebuilt.
inline bool h_pb_read_plan(int k, int m, const uint8_t *P, uint64_t present, uint64_t want, uint64_t *halves)
{
    const int tot = k + m, K2 = 2 * k;
    const uint64_t all = (1ull << tot) - 1, data = (1ull << k) - 1;
    present &= all;
    want &= all & ~present;
    *halves = 0;
    uint64_t hp = 0;
    for (int i = 0; i < tot; i++)
        if ((present >> i) & 1) hp |= 3ull << (2 * i);
    if (want && !(want & (want - 1)) && (want & data)) {
        const int j = __builtin_ctzll(want), g = pb_group_of(k, m, j);
        if ((present & data) == (data & ~want) && ((present >> k) & 1) && ((present >> (k + g)) & 1)) {
            uint64_t r = (1ull << (2 * k + 1)) | (1ull << (2 * (k + g) + 1));
            for (int x = 0; x < k; x++)
                if (x != j) r |= 1ull << (2 * x + 1);
            for (int x = pb_group_start(k, m, g); x < pb_group_start(k, m, g + 1); x++)
                if (x != j) r |= 1ull << (2 * x);
            *halves = r;
            return true;
        }
    }
    uint8_t R[2 * kPbMaxK][2 * kPbMaxK];
    int piv[2 * kPbMaxK], nb = 0;
    auto reduce = [&](uint8_t *v) {
        for (int b = 0; b < nb; b++) {
            const uint8_t f = v[piv[b]];
            if (f)
                for (int c = 0; c < K2; c++) v[c] ^= h_mul(f, R[b][c]);
        }
    };
    for (int q = 0; q < 2 * tot && nb < K2; q++) {
        if (!((hp >> q) & 1)) continue;
        uint8_t v[2 * kPbMaxK];
        for (int c = 0; c < K2; c++) v[c] = pb_grow(k, m, P, q, c);
        reduce(v);
        int p = 0;
        while (p < K2 && !v[p]) p++;
        if (p == K2) continue;
        const uint8_t iv = h_inv(v[p]);
        for (int c = 0; c < K2; c++) R[nb][c] = h_mul(v[c], iv);
        piv[nb++] = p;
        *halves |= 1ull << q;
    }
    for (int q = 0; q < 2 * tot; q++) {
        if (!((want >> (q >> 1)) & 1)) continue;
        uint8_t v[2 * kPbMaxK];
        for (int c = 0; c < K2; c++) v[c] = pb_grow(k, m, P, q, c);
        reduce(v);
        for (int c = 0; c < K2; c++)
            if (v[c]) return false;
    }
    return true;
}

}  // namespace garage_ec
