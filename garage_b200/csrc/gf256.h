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

}  // namespace garage_ec
