/* sse_c_oracle.c -- scalar reference of SSE-C block sealing (test infrastructure only; DESIGN.md section 2.6).
 * AES-256 from FIPS-197 (S-box computed from its definition in 5.1.1, key expansion 5.2, cipher 5.1), GCM from
 * NIST SP 800-38D (GHASH by Algorithm 1, GCTR, 96-bit IVs), and the STREAM-LE31 chunking of Garage's SSE-C blocks:
 * B = N || C_0 || ... || C_{n-1}, chunk c sealed under nonce N || LE32(c | last << 31).  Byte at a time, no tables
 * beyond the S-box: slow and obvious. */
#include <stdint.h>
#include <stddef.h>
#include <string.h>

static uint8_t sbox[256];
static int sbox_ready;

static uint8_t xtime(uint8_t a) { return (uint8_t)((a << 1) ^ ((a & 0x80) ? 0x1b : 0)); }
static uint8_t gmul(uint8_t a, uint8_t b)
{
    uint8_t r = 0;
    while (b) {
        if (b & 1) r ^= a;
        a = xtime(a);
        b >>= 1;
    }
    return r;
}
static void init_sbox(void)
{
    if (sbox_ready) return;
    for (int x = 0; x < 256; x++) {
        uint8_t inv = 0;
        for (int y = 1; x && y < 256; y++)
            if (gmul((uint8_t)x, (uint8_t)y) == 1) inv = (uint8_t)y;
        uint8_t s = 0x63;
        for (int i = 0; i < 8; i++) {
            int bit = ((inv >> i) ^ (inv >> ((i + 4) & 7)) ^ (inv >> ((i + 5) & 7)) ^ (inv >> ((i + 6) & 7)) ^
                       (inv >> ((i + 7) & 7))) & 1;
            s ^= (uint8_t)(bit << i);
        }
        sbox[x] = s;
    }
    sbox_ready = 1;
}

/* round keys: 15 x 16 bytes */
void sse_oracle_aes256_expand(const uint8_t key[32], uint8_t rk[240])
{
    init_sbox();
    memcpy(rk, key, 32);
    uint8_t rcon = 1;
    for (int i = 8; i < 60; i++) {
        uint8_t t[4];
        memcpy(t, rk + 4 * (i - 1), 4);
        if (i % 8 == 0) {
            uint8_t u = t[0];
            t[0] = sbox[t[1]] ^ rcon;
            t[1] = sbox[t[2]];
            t[2] = sbox[t[3]];
            t[3] = sbox[u];
            rcon = xtime(rcon);
        } else if (i % 8 == 4) {
            for (int j = 0; j < 4; j++) t[j] = sbox[t[j]];
        }
        for (int j = 0; j < 4; j++) rk[4 * i + j] = rk[4 * (i - 8) + j] ^ t[j];
    }
}

void sse_oracle_aes256_encrypt(const uint8_t rk[240], const uint8_t in[16], uint8_t out[16])
{
    init_sbox();
    uint8_t s[16];
    for (int i = 0; i < 16; i++) s[i] = in[i] ^ rk[i];
    for (int r = 1; r <= 14; r++) {
        uint8_t t[16];
        for (int i = 0; i < 16; i++) t[i] = sbox[s[i]];                     /* SubBytes */
        for (int c = 0; c < 4; c++)                                          /* ShiftRows */
            for (int row = 0; row < 4; row++) s[4 * c + row] = t[4 * ((c + row) & 3) + row];
        if (r < 14)
            for (int c = 0; c < 4; c++) {                                    /* MixColumns */
                uint8_t a0 = s[4 * c], a1 = s[4 * c + 1], a2 = s[4 * c + 2], a3 = s[4 * c + 3];
                s[4 * c] = gmul(a0, 2) ^ gmul(a1, 3) ^ a2 ^ a3;
                s[4 * c + 1] = a0 ^ gmul(a1, 2) ^ gmul(a2, 3) ^ a3;
                s[4 * c + 2] = a0 ^ a1 ^ gmul(a2, 2) ^ gmul(a3, 3);
                s[4 * c + 3] = gmul(a0, 3) ^ a1 ^ a2 ^ gmul(a3, 2);
            }
        for (int i = 0; i < 16; i++) s[i] ^= rk[16 * r + i];
    }
    memcpy(out, s, 16);
}

/* X <- X * Y in GF(2^128), SP 800-38D Algorithm 1 */
static void gf_mul(uint8_t X[16], const uint8_t Y[16])
{
    uint8_t Z[16] = {0}, V[16];
    memcpy(V, Y, 16);
    for (int i = 0; i < 128; i++) {
        if ((X[i / 8] >> (7 - i % 8)) & 1)
            for (int j = 0; j < 16; j++) Z[j] ^= V[j];
        int lsb = V[15] & 1;
        for (int j = 15; j > 0; j--) V[j] = (uint8_t)((V[j] >> 1) | (V[j - 1] << 7));
        V[0] >>= 1;
        if (lsb) V[0] ^= 0xe1;
    }
    memcpy(X, Z, 16);
}

static void ghash_blocks(uint8_t Y[16], const uint8_t H[16], const uint8_t *p, size_t len)
{
    for (size_t o = 0; o < len; o += 16) {
        size_t n = len - o < 16 ? len - o : 16;
        for (size_t i = 0; i < n; i++) Y[i] ^= p[o + i];
        gf_mul(Y, H);
    }
}

/* AES-256-GCM: out = ciphertext (len bytes) || tag (16).  J0 = IV || 0^31 || 1 for a 96-bit IV, else
 * GHASH(IV || 0-pad || 0^64 || [len(IV)]_64) (SP 800-38D 7.1 step 2) */
void sse_oracle_gcm_seal(const uint8_t key[32], const uint8_t *iv, size_t iv_len, const uint8_t *aad, size_t aad_len,
                         const uint8_t *pt, size_t len, uint8_t *out)
{
    uint8_t rk[240], H[16] = {0}, J[16] = {0}, ks[16], Y[16] = {0}, lens[16];
    sse_oracle_aes256_expand(key, rk);
    sse_oracle_aes256_encrypt(rk, H, H);
    if (iv_len == 12) {
        memcpy(J, iv, 12);
        J[15] = 1;
    } else {
        uint64_t ibits = (uint64_t)iv_len * 8;
        ghash_blocks(J, H, iv, iv_len);
        memset(lens, 0, 8);
        for (int i = 0; i < 8; i++) lens[8 + i] = (uint8_t)(ibits >> (56 - 8 * i));
        ghash_blocks(J, H, lens, 16);
    }
    for (size_t o = 0; o < len; o += 16) {
        uint32_t ctr = (((uint32_t)J[12] << 24) | ((uint32_t)J[13] << 16) | ((uint32_t)J[14] << 8) | J[15]) +
                       (uint32_t)(o / 16) + 1;  /* inc32 of J0, then one per block */
        uint8_t cb[16];
        memcpy(cb, J, 12);
        cb[12] = (uint8_t)(ctr >> 24);
        cb[13] = (uint8_t)(ctr >> 16);
        cb[14] = (uint8_t)(ctr >> 8);
        cb[15] = (uint8_t)ctr;
        sse_oracle_aes256_encrypt(rk, cb, ks);
        for (size_t i = 0; i < 16 && o + i < len; i++) out[o + i] = pt[o + i] ^ ks[i];
    }
    ghash_blocks(Y, H, aad, aad_len);
    ghash_blocks(Y, H, out, len);
    uint64_t abits = (uint64_t)aad_len * 8, cbits = (uint64_t)len * 8;
    for (int i = 0; i < 8; i++) {
        lens[i] = (uint8_t)(abits >> (56 - 8 * i));
        lens[8 + i] = (uint8_t)(cbits >> (56 - 8 * i));
    }
    ghash_blocks(Y, H, lens, 16);
    sse_oracle_aes256_encrypt(rk, J, ks);
    for (int i = 0; i < 16; i++) out[len + i] = Y[i] ^ ks[i];
    memset(rk, 0, sizeof(rk));
}

/* 0 and the plaintext in out if the tag matches, else 1 (out untouched) */
int sse_oracle_gcm_open(const uint8_t key[32], const uint8_t iv[12], const uint8_t *ct, size_t len, const uint8_t tag[16],
                        uint8_t *out)
{
    uint8_t rk[240], H[16] = {0}, J[16], ks[16], Y[16] = {0}, lens[16];
    sse_oracle_aes256_expand(key, rk);
    sse_oracle_aes256_encrypt(rk, H, H);
    memcpy(J, iv, 12);
    J[12] = J[13] = J[14] = 0;
    J[15] = 1;
    ghash_blocks(Y, H, ct, len);
    uint64_t cbits = (uint64_t)len * 8;
    memset(lens, 0, 8);
    for (int i = 0; i < 8; i++) lens[8 + i] = (uint8_t)(cbits >> (56 - 8 * i));
    ghash_blocks(Y, H, lens, 16);
    sse_oracle_aes256_encrypt(rk, J, ks);
    uint8_t diff = 0;
    for (int i = 0; i < 16; i++) diff |= (uint8_t)(Y[i] ^ ks[i] ^ tag[i]);
    if (diff) return 1;
    for (size_t o = 0; o < len; o += 16) {
        uint32_t ctr = (uint32_t)(o / 16) + 2;
        uint8_t cb[16];
        memcpy(cb, J, 12);
        cb[12] = (uint8_t)(ctr >> 24);
        cb[13] = (uint8_t)(ctr >> 16);
        cb[14] = (uint8_t)(ctr >> 8);
        cb[15] = (uint8_t)ctr;
        sse_oracle_aes256_encrypt(rk, cb, ks);
        for (size_t i = 0; i < 16 && o + i < len; i++) out[o + i] = ct[o + i] ^ ks[i];
    }
    return 0;
}

size_t sse_oracle_sealed_len(size_t len) { return 8 + len + 16 * (len ? (len + 4095) / 4096 : 1); }

/* STREAM-LE31 seal of one block: out gets sse_oracle_sealed_len(len) bytes */
void sse_oracle_seal(const uint8_t key[32], const uint8_t nonce8[8], const uint8_t *pt, size_t len, uint8_t *out)
{
    size_t n = len ? (len + 4095) / 4096 : 1;
    memcpy(out, nonce8, 8);
    for (size_t c = 0; c < n; c++) {
        uint8_t iv[12];
        uint32_t w = (uint32_t)c | (c == n - 1 ? 0x80000000u : 0u);
        memcpy(iv, nonce8, 8);
        iv[8] = (uint8_t)w;
        iv[9] = (uint8_t)(w >> 8);
        iv[10] = (uint8_t)(w >> 16);
        iv[11] = (uint8_t)(w >> 24);
        size_t cl = c == n - 1 ? len - 4096 * c : 4096;
        sse_oracle_gcm_seal(key, iv, 12, NULL, 0, pt + 4096 * c, cl, out + 8 + 4112 * c);
    }
}

/* STREAM-LE31 open: the plaintext length, or -1 for a framing or tag failure */
long sse_oracle_open(const uint8_t key[32], const uint8_t *b, size_t blen, uint8_t *out)
{
    if (blen < 24 || ((blen - 8) % 4112 >= 1 && (blen - 8) % 4112 < 16)) return -1;
    size_t n = (blen - 8 + 4111) / 4112, len = blen - 8 - 16 * n;
    for (size_t c = 0; c < n; c++) {
        uint8_t iv[12];
        uint32_t w = (uint32_t)c | (c == n - 1 ? 0x80000000u : 0u);
        memcpy(iv, b, 8);
        iv[8] = (uint8_t)w;
        iv[9] = (uint8_t)(w >> 8);
        iv[10] = (uint8_t)(w >> 16);
        iv[11] = (uint8_t)(w >> 24);
        size_t cl = c == n - 1 ? len - 4096 * c : 4096;
        const uint8_t *ch = b + 8 + 4112 * c;
        if (sse_oracle_gcm_open(key, iv, ch, cl, ch + cl, out + 4096 * c)) return -1;
    }
    return (long)len;
}
