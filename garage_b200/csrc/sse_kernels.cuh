// sse_kernels.cuh -- SSE-C blocks on the device (DESIGN.md sections 2.6 and 4.9): AES-256-GCM in the STREAM-LE31
// chunk framing of Garage's EncryptionParams::encrypt_block, written straight into and read straight out of the
// shard layout.
//
// A plain block P of len bytes, key K, 8-byte nonce prefix N:  B = N || C_0 || ... || C_{n-1}, n = max(1,
// ceil(len / 4096)), C_c = AES-256-GCM(K, N || LE32(c | (c == n-1) << 31), P[4096c, 4096c + 4096)) = ciphertext ||
// 16-byte tag.  Chunk c starts at byte 8 + 4112c of B, 8 bytes off a 16-byte boundary, and B is cut into data shards
// of L bytes (data shard j = B[jL, (j+1)L)), so chunks straddle shards at arbitrary offsets.
//
// One warp per chunk.  The warp stages its chunk's bytes of B in shared memory: seal writes ciphertext and tag there
// and then stores them to the shard layout with 16-byte stores aligned in shard space (bytes a vector shares with
// the neighbouring chunk are stored one by one, so two warps never write the same byte); open loads the chunk's
// bytes of every shard it touches with aligned 16-byte loads.  No pass over HBM stages B anywhere else.
//
// GHASH is split across the lanes: the chunk's nb data blocks are right-aligned in 256 slots, lane l runs Horner's
// rule (4-bit tables of H) over slots [8l, 8l+8), and its partial sum is multiplied by H^(8(31-l)) -- the same power
// for every chunk length, precomputed per key -- before a warp reduction.  Open checks every tag in one launch and
// decrypts in a second one, so that no plaintext of a block is written unless all of its tags passed.
#pragma once

#include <stdint.h>

#include <type_traits>

namespace garage_ec {
namespace sse {

constexpr uint32_t kChunk = 4096;          // STREAM_ENC_PLAIN_CHUNK_SIZE
constexpr uint32_t kFrame = kChunk + 16;   // one sealed chunk: ciphertext + tag
constexpr uint32_t kPrefix = 8;            // the nonce prefix at the head of B
constexpr int kWarps = 8;                  // warps per CTA of the chunk kernel
constexpr uint32_t kStage = kFrame + kPrefix + 24;  // per-warp staging: [0, 8) nonce, [8, 8 + 4112) chunk, slack

// sealed length of a len-byte block (64-bit: the caller checks it fits 32 bits)
__host__ __device__ inline uint64_t sealed_len(uint64_t len)
{
    const uint64_t n = len ? (len + kChunk - 1) / kChunk : 1;
    return kPrefix + len + 16 * n;
}

// DESIGN.md 2.7: the chunks c0 .. c0 + nch - 1 that plaintext bytes [o, o + len) of a block sealed to S bytes lie in,
// and their run of B, [span_off, span_off + span_len).  0; -7 (GARAGE_EC_E_AUTH) for an S the framing cannot hold;
// -1 (GARAGE_EC_E_INVALID) for a range past the plaintext.  An empty range touches nothing: nch = span_len = 0.
__host__ __device__ inline int sealed_range(uint32_t S, uint32_t o, uint32_t len, uint32_t *span_off,
                                            uint32_t *span_len, uint32_t *c0, uint32_t *nch)
{
    if (S < kPrefix + 16) return -7;
    const uint32_t r = (S - kPrefix) % kFrame;
    if (r >= 1 && r < 16) return -7;
    const uint64_t n = ((uint64_t)S - kPrefix + kFrame - 1) / kFrame, P = S - kPrefix - 16 * n;
    if ((uint64_t)o + len > P) return -1;
    const uint64_t a = o / kChunk, b = len ? ((uint64_t)o + len - 1) / kChunk + 1 : a;
    const uint64_t s0 = kPrefix + kFrame * a, s1 = kPrefix + kFrame * b;
    *c0 = (uint32_t)a;
    *nch = (uint32_t)(b - a);
    *span_off = (uint32_t)(s0 < S ? s0 : S);
    *span_len = (uint32_t)((s1 < S ? s1 : S) - *span_off);
    return 0;
}

// Per-key material, built by sse_setup_kernel: the AES-256 round keys (FIPS-197 5.2), the 4-bit multiplication
// table of H = E_K(0^128) and H^(8(31-l)) for lane l.  Secret: zeroed on the stream after the call's last kernel.
struct SseKey {
    uint32_t rk[60];
    uint32_t pad[4];
    unsigned long long hh[16], hl[16];   // i * H, GCM bit order (hi, lo words big-endian)
    unsigned long long pw[32][2];        // lane powers
};
static_assert(sizeof(SseKey) == 1024, "SseKey layout");

struct SseTables {
    uint32_t te[4][256];
    uint8_t sbox[256];
    uint32_t r4[16];   // reduction of the four bits a 4-bit shift drops (Shoup's table)
};

__device__ __forceinline__ uint8_t gf8_mul(uint8_t a, uint8_t b)
{
    uint8_t r = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        if (b & 1) r ^= a;
        const uint8_t hi = a & 0x80;
        a = (uint8_t)(a << 1);
        if (hi) a ^= 0x1b;
        b >>= 1;
    }
    return r;
}

// the S-box (FIPS-197 5.1.1: inverse in GF(2^8) mod x^8+x^4+x^3+x+1, then the affine map) and the encryption T
// tables, built by the CTA's threads (blockDim.x >= 256)
__device__ __forceinline__ void build_tables(SseTables &t)
{
    const uint32_t x = threadIdx.x;
    if (x < 256) {
        uint8_t inv = 0;
        if (x) {  // x^254
            uint8_t r = 1, b = (uint8_t)x;
            for (int e = 254; e; e >>= 1) {
                if (e & 1) r = gf8_mul(r, b);
                b = gf8_mul(b, b);
            }
            inv = r;
        }
        uint32_t s = inv;
        s ^= ((inv << 1) | (inv >> 7)) ^ ((inv << 2) | (inv >> 6)) ^ ((inv << 3) | (inv >> 5)) ^
             ((inv << 4) | (inv >> 4)) ^ 0x63;
        s &= 0xff;
        t.sbox[x] = (uint8_t)s;
        const uint32_t s2 = gf8_mul((uint8_t)s, 2), s3 = s2 ^ s;
        const uint32_t w = (s2 << 24) | (s << 16) | (s << 8) | s3;
        t.te[0][x] = w;
        t.te[1][x] = (w >> 8) | (w << 24);
        t.te[2][x] = (w >> 16) | (w << 16);
        t.te[3][x] = (w >> 24) | (w << 8);
    }
    if (x < 16) {
        uint32_t r = 0;
        for (int b = 0; b < 4; b++)
            if (x & (1u << b)) r ^= 0xE100u >> (3 - b);
        t.r4[x] = r;
    }
}

__device__ __forceinline__ uint32_t sub_word(const SseTables &t, uint32_t w)
{
    return ((uint32_t)t.sbox[w >> 24] << 24) | ((uint32_t)t.sbox[(w >> 16) & 0xff] << 16) |
           ((uint32_t)t.sbox[(w >> 8) & 0xff] << 8) | (uint32_t)t.sbox[w & 0xff];
}

// one AES-256 block; state as four big-endian column words
__device__ __forceinline__ void aes256_encrypt(const SseTables &t, const uint32_t *rk, uint32_t &s0, uint32_t &s1,
                                               uint32_t &s2, uint32_t &s3)
{
    s0 ^= rk[0];
    s1 ^= rk[1];
    s2 ^= rk[2];
    s3 ^= rk[3];
#pragma unroll
    for (int r = 1; r < 14; r++) {
        const uint32_t t0 = t.te[0][s0 >> 24] ^ t.te[1][(s1 >> 16) & 0xff] ^ t.te[2][(s2 >> 8) & 0xff] ^
                            t.te[3][s3 & 0xff] ^ rk[4 * r];
        const uint32_t t1 = t.te[0][s1 >> 24] ^ t.te[1][(s2 >> 16) & 0xff] ^ t.te[2][(s3 >> 8) & 0xff] ^
                            t.te[3][s0 & 0xff] ^ rk[4 * r + 1];
        const uint32_t t2 = t.te[0][s2 >> 24] ^ t.te[1][(s3 >> 16) & 0xff] ^ t.te[2][(s0 >> 8) & 0xff] ^
                            t.te[3][s1 & 0xff] ^ rk[4 * r + 2];
        const uint32_t t3 = t.te[0][s3 >> 24] ^ t.te[1][(s0 >> 16) & 0xff] ^ t.te[2][(s1 >> 8) & 0xff] ^
                            t.te[3][s2 & 0xff] ^ rk[4 * r + 3];
        s0 = t0;
        s1 = t1;
        s2 = t2;
        s3 = t3;
    }
    const uint8_t *S = t.sbox;
    const uint32_t o0 = ((uint32_t)S[s0 >> 24] << 24) | ((uint32_t)S[(s1 >> 16) & 0xff] << 16) |
                        ((uint32_t)S[(s2 >> 8) & 0xff] << 8) | S[s3 & 0xff];
    const uint32_t o1 = ((uint32_t)S[s1 >> 24] << 24) | ((uint32_t)S[(s2 >> 16) & 0xff] << 16) |
                        ((uint32_t)S[(s3 >> 8) & 0xff] << 8) | S[s0 & 0xff];
    const uint32_t o2 = ((uint32_t)S[s2 >> 24] << 24) | ((uint32_t)S[(s3 >> 16) & 0xff] << 16) |
                        ((uint32_t)S[(s0 >> 8) & 0xff] << 8) | S[s1 & 0xff];
    const uint32_t o3 = ((uint32_t)S[s3 >> 24] << 24) | ((uint32_t)S[(s0 >> 16) & 0xff] << 16) |
                        ((uint32_t)S[(s1 >> 8) & 0xff] << 8) | S[s2 & 0xff];
    s0 = o0 ^ rk[56];
    s1 = o1 ^ rk[57];
    s2 = o2 ^ rk[58];
    s3 = o3 ^ rk[59];
}

// X * Y in GF(2^128), GCM bit order, bit by bit (NIST SP 800-38D, Algorithm 1)
__device__ __forceinline__ void gf128_mul_bits(unsigned long long &xh, unsigned long long &xl, unsigned long long yh,
                                               unsigned long long yl)
{
    unsigned long long zh = 0, zl = 0, vh = yh, vl = yl;
    for (int i = 0; i < 128; i++) {
        const unsigned long long bit = i < 64 ? (xh >> (63 - i)) & 1 : (xl >> (127 - i)) & 1;
        const unsigned long long msk = 0ull - bit;
        zh ^= vh & msk;
        zl ^= vl & msk;
        const unsigned long long lsb = vl & 1;
        vl = (vl >> 1) | (vh << 63);
        vh = (vh >> 1) ^ ((0ull - lsb) & 0xE100000000000000ull);
    }
    xh = zh;
    xl = zl;
}

// X * H by the 4-bit table of H (hh / hl: i * H for the nibble i read most significant bit first)
__device__ __forceinline__ void gf128_mul_h(const unsigned long long *hh, const unsigned long long *hl,
                                            const uint32_t *r4, unsigned long long &xh, unsigned long long &xl)
{
    unsigned long long zh = 0, zl = 0;
#pragma unroll
    for (int i = 31; i >= 0; i--) {  // nibbles from the last (x^124..x^127) to the first
        const uint32_t nib = (uint32_t)((i < 16 ? xh >> (60 - 4 * i) : xl >> (60 - 4 * (i - 16))) & 0xf);
        if (i != 31) {
            const uint32_t rem = (uint32_t)(zl & 0xf);
            zl = (zh << 60) | (zl >> 4);
            zh = (zh >> 4) ^ ((unsigned long long)r4[rem] << 48);
        }
        zh ^= hh[nib];
        zl ^= hl[nib];
    }
    xh = zh;
    xl = zl;
}

__device__ __forceinline__ unsigned long long load_be64(const uint8_t *p)
{
    unsigned long long v = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) v = (v << 8) | p[i];
    return v;
}
__device__ __forceinline__ uint32_t bswap32(uint32_t v) { return __byte_perm(v, 0, 0x0123); }
__device__ __forceinline__ unsigned long long bswap64(unsigned long long v)
{
    return ((unsigned long long)bswap32((uint32_t)v) << 32) | bswap32((uint32_t)(v >> 32));
}

// ---- key setup: one thread per block --------------------------------------------------------------------------
struct SetupParams {
    const uint8_t *keys;   // 32 bytes per block
    SseKey *ks;            // out
    uint32_t n;
};
__global__ void __launch_bounds__(256) sse_setup_kernel(const __grid_constant__ SetupParams q)
{
    __shared__ SseTables t;
    build_tables(t);
    __syncthreads();
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= q.n) return;
    SseKey &K = q.ks[s];
    uint32_t w[60];
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const uint8_t *k = q.keys + (size_t)s * 32 + 4 * i;
        w[i] = ((uint32_t)k[0] << 24) | ((uint32_t)k[1] << 16) | ((uint32_t)k[2] << 8) | k[3];
    }
    uint32_t rcon = 1;
#pragma unroll
    for (int i = 8; i < 60; i++) {
        uint32_t tmp = w[i - 1];
        if (i % 8 == 0) {
            tmp = sub_word(t, (tmp << 8) | (tmp >> 24)) ^ (rcon << 24);
            rcon = gf8_mul((uint8_t)rcon, 2);
        } else if (i % 8 == 4) {
            tmp = sub_word(t, tmp);
        }
        w[i] = w[i - 8] ^ tmp;
    }
#pragma unroll
    for (int i = 0; i < 60; i++) K.rk[i] = w[i];
    uint32_t h0 = 0, h1 = 0, h2 = 0, h3 = 0;
    aes256_encrypt(t, w, h0, h1, h2, h3);
#pragma unroll
    for (int i = 0; i < 60; i++) w[i] = 0;
    unsigned long long vh = ((unsigned long long)h0 << 32) | h1, vl = ((unsigned long long)h2 << 32) | h3;
    const unsigned long long Hh = vh, Hl = vl;
    // table: entry 8 = H, 4 = H*x, 2 = H*x^2, 1 = H*x^3 (x = a right shift in GCM order), then the sums
    K.hh[0] = K.hl[0] = 0;
    K.hh[8] = vh;
    K.hl[8] = vl;
    for (int i = 4; i > 0; i >>= 1) {
        const unsigned long long lsb = vl & 1;
        vl = (vl >> 1) | (vh << 63);
        vh = (vh >> 1) ^ ((0ull - lsb) & 0xE100000000000000ull);
        K.hh[i] = vh;
        K.hl[i] = vl;
    }
    for (int i = 2; i <= 8; i <<= 1)
        for (int j = 1; j < i; j++) {
            K.hh[i + j] = K.hh[i] ^ K.hh[j];
            K.hl[i + j] = K.hl[i] ^ K.hl[j];
        }
    // H^8, then lane 31-i gets H^(8i); lane 31: the identity (bit 0 set)
    unsigned long long p8h = Hh, p8l = Hl;
    for (int i = 0; i < 3; i++) gf128_mul_bits(p8h, p8l, p8h, p8l);
    unsigned long long ph = 1ull << 63, pl = 0;
    for (int i = 0; i < 32; i++) {
        K.pw[31 - i][0] = ph;
        K.pw[31 - i][1] = pl;
        gf128_mul_bits(ph, pl, p8h, p8l);
    }
}

// ---- the chunk kernel -----------------------------------------------------------------------------------------
// kRangeCheck / kRangeOpen: ranged opens (DESIGN.md 4.10).  Request s reads its nonce prefix from row 2s of `rows`
// and chunks c0 .. c1 of its range, back to back from a 16-byte boundary, from row 2s + 1; the open writes only the
// plaintext bytes [offset, offset + len) to plain_out + s*plain_stride, zero up to roundup16(len).
// kReseal: copies with re-encryption (DESIGN.md 4.11).  Work item (d, c) is chunk c of destination d: the warp
// decrypts the source CTR blocks its pieces cover straight into the stage, then seals the stage in place as kSeal does.
// kCrc (added to kSeal or kReseal): also the CRC32 / CRC32C of each block's plaintext, per q.crc_kind (DESIGN.md 4.12).
enum { kSeal = 0, kCheck = 1, kOpen = 2, kRangeCheck = 3, kRangeOpen = 4, kReseal = 5, kCrc = 8 };

struct ChunkParams {
    const uint8_t *plain_in;        // seal: block s at plain_in + s*plain_stride
    uint8_t *plain_out;             // open: block s at plain_out + s*plain_stride
    const uint8_t *rows;            // ranged: row r at rows + r*row_pitch
    const uint32_t *offset, *len;   // ranged: the plaintext range per request
    unsigned long long row_pitch;
    unsigned long long plain_stride;
    const uint32_t *plain_len;      // seal: per block
    uint32_t *plain_len_out;        // open: per block
    const uint32_t *blen;           // len(B) per block: sealed length (plain_len when unkeyed)
    const uint32_t *shard_len;      // L per block; 0 = nothing of the block is touched
    const uint8_t *nonces;          // seal: 8 bytes per block
    const SseKey *ks;               // nullable (seal only): B = P
    uint8_t *shards;                // stripe s at shards + s*(k+m)*stride, data shard j at + j*stride
    int32_t *status;                // check / open
    const int32_t *rec_status;      // check: verdict of the reconstruct (ranged: of the two row decodes, 2s and 2s + 1)
    const uint8_t *hash_bad;        // open: skip the block when set
    uint32_t stride, k, m, n;
    uint32_t cmax;                  // chunks per block this launch covers (work item = block * cmax + chunk; ranged:
                                    // + chunk - c0)
    // reseal: block s is destination s (plain_len = |Q_s|, blen its sealed length, shard_len 0 = not proven, ks its
    // key), made of pieces [piece_start[s], piece_start[s + 1]) = {src, offset, len} words of the sources
    const uint32_t *pieces, *piece_start;
    const uint8_t *src_shards;      // source i at src_shards + i*(k+m)*stride
    const uint32_t *src_len;        // stored length S_i
    const uint32_t *src_L;          // its L
    const SseKey *src_ks;           // nullable: the sources are plaintext
    // the kCrc instantiations: checksum kind per block (GARAGE_EC_CRC_*, 0 = none) and its accumulator (DESIGN.md 4.12)
    const uint8_t *crc_kind;
    uint32_t *crc_acc;
};

struct ChunkSmem {
    SseTables t;
    __align__(16) uint8_t stage[kWarps][kStage];
    uint32_t rk[kWarps][60];
    unsigned long long hh[kWarps][16], hl[kWarps][16];
};

// ---- CRC32 / CRC32C of the plaintext (DESIGN.md 2.9 and 4.12) ----------------------------------------------------
// Values mod P in the reflected order of zlib: bit 31 is the coefficient of x^0, bit 0 that of x^31.  Kind index t =
// GARAGE_EC_CRC_* - 1: 0 = CRC32 (0xEDB88320), 1 = CRC32C (0x82F63B78).  "raw" is the CRC with zero init and no final
// XOR, which is linear: raw(A || B) = raw(A) * x^(8|B|) + raw(B), and leading zero bytes leave it unchanged.
__host__ __device__ constexpr uint32_t crc_poly(int t) { return t ? 0x82F63B78u : 0xEDB88320u; }
__host__ __device__ constexpr uint32_t crc_mulx(uint32_t v, uint32_t poly) { return (v >> 1) ^ ((v & 1u) ? poly : 0u); }
// v / x: P has a constant term, so x is invertible
__host__ __device__ constexpr uint32_t crc_divx(uint32_t v, uint32_t poly)
{
    return (v >> 31) ? ((v ^ poly) << 1) | 1u : v << 1;
}
// a * b mod P, branch-free over the 32 coefficients of a
__host__ __device__ constexpr uint32_t crc_mul(uint32_t a, uint32_t b, uint32_t poly)
{
    uint32_t p = 0;
    for (int i = 0; i < 32; i++) {
        p ^= b & (0u - ((a >> (31 - i)) & 1u));
        b = crc_mulx(b, poly);
    }
    return p;
}

struct CrcConsts {
    uint32_t slice[2][2][256];  // slicing-by-2: slice[t][j][b] = raw(b followed by j zero bytes)
    uint32_t slot[2][257];      // x^(-128 j): a lane value whose 16-byte slots end j slots into the chunk's grid
    uint32_t chunk[2][256];     // x^(-32768 c): chunk c's place in the block's grid of 4096-byte chunks
    uint32_t chunk_hi[2][12];   // x^(-32768 * 256 * 2^i), for chunks from 256 on (a block has fewer than 2^20)
    uint32_t x8[2][64];         // x^(8 * 2^i): a shift by a byte count
};
constexpr CrcConsts make_crc_consts()
{
    CrcConsts c{};
    for (int t = 0; t < 2; t++) {
        const uint32_t P = crc_poly(t);
        for (uint32_t b = 0; b < 256; b++) {
            uint32_t v = b;
            for (int i = 0; i < 8; i++) v = crc_mulx(v, P);
            c.slice[t][0][b] = v;
        }
        for (uint32_t b = 0; b < 256; b++) c.slice[t][1][b] = (c.slice[t][0][b] >> 8) ^ c.slice[t][0][c.slice[t][0][b] & 0xff];
        uint32_t h = 0x80000000u;  // x^-128
        for (int i = 0; i < 128; i++) h = crc_divx(h, P);
        c.slot[t][0] = 0x80000000u;
        for (int j = 1; j <= 256; j++) c.slot[t][j] = crc_mul(c.slot[t][j - 1], h, P);
        c.chunk[t][0] = 0x80000000u;
        for (int j = 1; j < 256; j++) c.chunk[t][j] = crc_mul(c.chunk[t][j - 1], c.slot[t][256], P);
        c.chunk_hi[t][0] = crc_mul(c.chunk[t][255], c.slot[t][256], P);
        for (int i = 1; i < 12; i++) c.chunk_hi[t][i] = crc_mul(c.chunk_hi[t][i - 1], c.chunk_hi[t][i - 1], P);
        c.x8[t][0] = 0x00800000u;  // x^8
        for (int i = 1; i < 64; i++) c.x8[t][i] = crc_mul(c.x8[t][i - 1], c.x8[t][i - 1], P);
    }
    return c;
}
// global, not __constant__, memory: the constant bank layout of every other kernel stays as it was
__device__ const CrcConsts kCrcDev = make_crc_consts();
constexpr CrcConsts kCrcHost = make_crc_consts();

// v * x^(8n): square-and-multiply over x8
__host__ __device__ inline uint32_t crc_shift(const CrcConsts &c, int t, uint32_t v, unsigned long long n)
{
    for (int i = 0; n; i++, n >>= 1)
        if (n & 1) v = crc_mul(c.x8[t][i], v, crc_poly(t));
    return v;
}
// The CRC (init and final XOR 0xFFFFFFFF) of a len-byte message M from acc = raw(M) * x^(-8 len), the form the chunk
// kernel accumulates: the init's contribution is 0xFFFFFFFF * x^(8 len), so CRC = (acc + 0xFFFFFFFF) * x^(8 len) + 0xFFFFFFFF.
__host__ __device__ inline uint32_t crc_finish(const CrcConsts &c, int t, uint32_t acc, unsigned long long len)
{
    return crc_shift(c, t, acc ^ 0xFFFFFFFFu, len) ^ 0xFFFFFFFFu;
}

// 6152 bytes on top of ChunkSmem's 41984, under the 48 KiB of static shared memory a CTA may have: slicing-by-4
// tables for both kinds (8 KiB) would not fit (DESIGN.md 4.12)
struct CrcChunkSmem : ChunkSmem {
    uint32_t crc_slice[2][2][256];
    uint32_t crc_slot[2][257];
};

// one lane's raw CRC continued over 16 plaintext bytes (two little-endian words, zero past the chunk's end)
__device__ __forceinline__ uint32_t crc_block16(const uint32_t (*T)[256], uint32_t c, unsigned long long a,
                                                unsigned long long b)
{
    const uint32_t w[4] = {(uint32_t)a, (uint32_t)(a >> 32), (uint32_t)b, (uint32_t)(b >> 32)};
#pragma unroll
    for (int i = 0; i < 4; i++) {
        c ^= w[i];
        c = (c >> 16) ^ T[1][c & 0xff] ^ T[0][(c >> 8) & 0xff];
        c = (c >> 16) ^ T[1][c & 0xff] ^ T[0][(c >> 8) & 0xff];
    }
    return c;
}

// kReseal: plaintext bytes [x0, x1) of source i into to[0, x1 - x0), lanes splitting its 16-byte blocks.  Block g of a
// keyed source is decrypted from its ciphertext at B position 8 + 4112 (g / 256) + 16 (g mod 256), counter block
// N_i || LE32(c | last << 31) || BE32(g mod 256 + 2); an unkeyed source's block is B[16g, 16g + 16).  The source's
// round keys are read from its key material in global memory, so the mode needs no shared memory of its own.
__device__ __forceinline__ void reseal_piece(const ChunkParams &q, const SseTables &t, uint8_t *to, uint32_t i,
                                             uint32_t x0, uint32_t x1, uint32_t lane)
{
    const uint32_t S = q.src_len[i], L = q.src_L[i];
    const uint8_t *stripe = q.src_shards + (size_t)i * (q.k + q.m) * q.stride;
    const SseKey *K = q.src_ks ? q.src_ks + i : nullptr;
    uint32_t P = S, nch = 1, nw0 = 0, nw1 = 0;
    if (K) {  // framing checked by sse_reseal_lens_kernel
        nch = (S - kPrefix + kFrame - 1) / kFrame;
        P = S - kPrefix - 16 * nch;
        uint8_t nb8[8];
#pragma unroll
        for (int b = 0; b < 8; b++) nb8[b] = stripe[(size_t)(b / L) * q.stride + b % L];
        nw0 = ((uint32_t)nb8[0] << 24) | ((uint32_t)nb8[1] << 16) | ((uint32_t)nb8[2] << 8) | nb8[3];
        nw1 = ((uint32_t)nb8[4] << 24) | ((uint32_t)nb8[5] << 16) | ((uint32_t)nb8[6] << 8) | nb8[7];
    }
    const uint32_t g1 = (x1 + 15) / 16;
    for (uint32_t g = x0 / 16 + lane; g < g1; g += 32) {
        const uint32_t c = g >> 8, pos = K ? kPrefix + kFrame * c + 16 * (g & 255) : 16 * g, j = pos / L;
        const uint4 v = block_vec16(stripe, q.stride, L, j, pos - j * L, min(16u, P - 16 * g));
        unsigned long long a = ((unsigned long long)v.y << 32) | v.x, b = ((unsigned long long)v.w << 32) | v.z;
        if (K) {
            uint32_t k0 = nw0, k1 = nw1, k2 = bswap32(c | (c == nch - 1 ? 0x80000000u : 0u)), k3 = (g & 255) + 2;
            aes256_encrypt(t, K->rk, k0, k1, k2, k3);
            a ^= bswap64(((unsigned long long)k0 << 32) | k1);
            b ^= bswap64(((unsigned long long)k2 << 32) | k3);
        }
        const uint32_t lo = max(16 * g, x0), hi = min(16 * g + 16, x1);
        for (uint32_t x = lo; x < hi; x++) {
            const uint32_t o = x - 16 * g;
            to[x - x0] = (uint8_t)(o < 8 ? a >> (8 * o) : b >> (8 * (o - 8)));
        }
    }
}

// Launch bounds: the checksumming modes are held to the CTAs per SM that kSeal (4) and kReseal (3) reach by their
// register counts -- unbounded, ptxas gives the checksumming seal 92 registers and 2 CTAs per SM (DESIGN.md 4.12).  A
// minimum of 0 leaves the other modes as they were built before the checksums existed.
template <int KMODE>
__global__ void __launch_bounds__(kWarps * 32, KMODE == (kSeal | kCrc) ? 4 : KMODE == (kReseal | kCrc) ? 3 : 0)
    sse_chunk_kernel(const __grid_constant__ ChunkParams q)
{
    constexpr int MODE = KMODE & ~kCrc;
    constexpr bool crc = (KMODE & kCrc) != 0;
    static_assert(!crc || MODE == kSeal || MODE == kReseal, "checksums are computed by the sealing modes only");
    __shared__ std::conditional_t<crc, CrcChunkSmem, ChunkSmem> sm;
    build_tables(sm.t);
    if constexpr (crc) {
        for (uint32_t i = threadIdx.x; i < 2 * 2 * 256; i += blockDim.x) (&sm.crc_slice[0][0][0])[i] = (&kCrcDev.slice[0][0][0])[i];
        for (uint32_t i = threadIdx.x; i < 2 * 257; i += blockDim.x) (&sm.crc_slot[0][0])[i] = (&kCrcDev.slot[0][0])[i];
    }
    __syncthreads();
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint8_t *st = sm.stage[wid];
    const unsigned long long total = (unsigned long long)q.n * q.cmax;
    for (unsigned long long w = (unsigned long long)blockIdx.x * kWarps + wid; w < total;
         w += (unsigned long long)gridDim.x * kWarps) {
        constexpr bool ranged = MODE == kRangeCheck || MODE == kRangeOpen;
        constexpr bool checking = MODE == kCheck || MODE == kRangeCheck;
        constexpr bool sealing = MODE == kSeal || MODE == kReseal;
        const uint32_t s = (uint32_t)(w / q.cmax), ci = (uint32_t)(w - (unsigned long long)s * q.cmax);
        const uint32_t L = ranged ? 0u : q.shard_len[s];
        if (!ranged && !L) continue;
        const uint32_t ckind = crc ? q.crc_kind[s] : 0u;  // 0 or GARAGE_EC_CRC_*: other kinds were given L = 0
        uint32_t cv = 0;                                   // this lane's raw CRC of its slots
        const bool keyed = MODE != kSeal || q.ks;
        const uint32_t blen = q.blen[s];
        const uint32_t prefix = keyed ? kPrefix : 0, pitch = keyed ? kFrame : kChunk;
        uint32_t plen, nch, c = ci, off = 0, len = 0, c1 = 0;
        if (sealing) {
            plen = q.plain_len[s];
        } else {
            const int32_t rs = ranged ? (q.rec_status[2 * s] ? q.rec_status[2 * s] : q.rec_status[2 * s + 1])
                                      : q.rec_status[s];
            if (checking && ci == 0) {
                if (rs && lane == 0) q.status[s] = rs;  // an unrecoverable stripe reports that, not its framing
            }
            if (q.status[s] != 0 || rs != 0) continue;
            if (MODE == kOpen && q.hash_bad[s]) continue;
            const uint32_t nn = (blen - kPrefix + kFrame - 1) / kFrame;  // framing checked by sse_lens_kernel
            plen = blen - kPrefix - 16 * nn;
            if (ranged) {  // range checked by sse_range_lens_kernel
                off = q.offset[s];
                len = q.len[s];
                if (!len) continue;
                c = off / kChunk + ci;
                c1 = (off + len - 1) / kChunk;
                if (c > c1) continue;
            }
        }
        nch = plen ? (plen + kChunk - 1) / kChunk : 1;
        if (c >= nch) continue;
        const bool last = c == nch - 1;
        const uint32_t clen = last ? plen - kChunk * c : kChunk;  // plaintext bytes of this chunk
        const uint32_t nb = (clen + 15) >> 4;
        const uint32_t base = pitch * c;  // B position of stage[0]
        uint8_t *stripe = q.shards + (size_t)s * (q.k + q.m) * q.stride;
        const SseKey *K = keyed ? q.ks + s : nullptr;
        if (keyed) {
            for (uint32_t i = lane; i < 60; i += 32) sm.rk[wid][i] = K->rk[i];
            if (lane < 16) {
                sm.hh[wid][lane] = K->hh[lane];
                sm.hl[wid][lane] = K->hl[lane];
            }
        }
        uint32_t nw0 = 0, nw1 = 0;  // the nonce prefix, big-endian words
        if (keyed) {
            if (sealing) {
                const uint8_t *np = q.nonces + (size_t)s * 8;
                nw0 = ((uint32_t)np[0] << 24) | ((uint32_t)np[1] << 16) | ((uint32_t)np[2] << 8) | np[3];
                nw1 = ((uint32_t)np[4] << 24) | ((uint32_t)np[5] << 16) | ((uint32_t)np[6] << 8) | np[7];
            } else {
                // B[0, 8): byte i of B is byte i % L of data shard i / L (ranged: the first 8 bytes of row 2s)
                const uint8_t *row = q.rows + 2ull * s * q.row_pitch;
                uint8_t nb8[8];
#pragma unroll
                for (int i = 0; i < 8; i++) nb8[i] = ranged ? row[i] : stripe[(size_t)(i / L) * q.stride + i % L];
                nw0 = ((uint32_t)nb8[0] << 24) | ((uint32_t)nb8[1] << 16) | ((uint32_t)nb8[2] << 8) | nb8[3];
                nw1 = ((uint32_t)nb8[4] << 24) | ((uint32_t)nb8[5] << 16) | ((uint32_t)nb8[6] << 8) | nb8[7];
            }
        }
        const uint32_t nw2 = bswap32(c | (last ? 0x80000000u : 0u));  // LE32(c | last << 31) as a big-endian word

        if (ranged) {
            // the chunk's ciphertext and tag, 16-byte aligned in row 2s + 1, into stage[8..]; the row is zero past
            // the span up to its roundup16, and a vector past clen + 16 lands in the stage's slack
            const uint8_t *src = q.rows + (2ull * s + 1) * q.row_pitch + (size_t)kFrame * ci;
            for (uint32_t v = 16 * lane; v < clen + 16; v += 512) {
                const uint4 d = *reinterpret_cast<const uint4 *>(src + v);
                *reinterpret_cast<unsigned long long *>(st + kPrefix + v) = ((unsigned long long)d.y << 32) | d.x;
                *reinterpret_cast<unsigned long long *>(st + kPrefix + v + 8) = ((unsigned long long)d.w << 32) | d.z;
            }
        } else if (MODE == kReseal) {
            // destination bytes [X0, X1) of Q_s: the pieces' destination offsets are an exclusive scan of their
            // lengths, formed 32 pieces at a time; every piece that overlaps the chunk is decrypted by the whole warp
            const uint32_t X0 = kChunk * c, X1 = X0 + clen, p1 = q.piece_start[s + 1];
            uint32_t run = 0;
            for (uint32_t pb = q.piece_start[s]; pb < p1 && run < X1; pb += 32) {
                const uint32_t p = pb + lane;
                uint32_t src = 0, po = 0, pl = 0;
                if (p < p1) {
                    src = q.pieces[3 * (size_t)p];
                    po = q.pieces[3 * (size_t)p + 1];
                    pl = q.pieces[3 * (size_t)p + 2];
                }
                uint32_t incl = pl;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
                    if (lane >= (uint32_t)o) incl += v;
                }
                const uint32_t at = run + incl - pl;
                uint32_t hit = __ballot_sync(0xffffffffu, pl && at < X1 && at + pl > X0);
                run += __shfl_sync(0xffffffffu, incl, 31);
                while (hit) {
                    const int l = __ffs(hit) - 1;
                    hit &= hit - 1;
                    const uint32_t hs = __shfl_sync(0xffffffffu, src, l), ho = __shfl_sync(0xffffffffu, po, l),
                                   hl = __shfl_sync(0xffffffffu, pl, l), ha = __shfl_sync(0xffffffffu, at, l);
                    const uint32_t a = max(X0, ha), e = min(X1, ha + hl);
                    reseal_piece(q, sm.t, st + kPrefix + (a - X0), hs, ho + a - ha, ho + e - ha, lane);
                }
            }
        } else if (MODE != kSeal) {
            // load this chunk's ciphertext and tag, B[base + 8, base + 8 + clen + 16), into stage[8..]
            const uint32_t r0 = base + kPrefix, r1 = r0 + clen + 16;
            for (uint32_t j = r0 / L; j * L < r1 && j < q.k; j++) {
                const uint32_t x0 = max(r0, j * L) - j * L, x1 = min(r1, (j + 1) * L) - j * L;
                const uint8_t *sh = stripe + (size_t)j * q.stride;
                for (uint32_t v = (x0 & ~15u) + 16 * lane; v < x1; v += 512) {
                    const uint4 d = *reinterpret_cast<const uint4 *>(sh + v);
                    const uint32_t wds[4] = {d.x, d.y, d.z, d.w};
#pragma unroll
                    for (int b = 0; b < 16; b++) {
                        const uint32_t x = v + b;
                        if (x >= x0 && x < x1) st[j * L + x - base] = (uint8_t)(wds[b >> 2] >> (8 * (b & 3)));
                    }
                }
            }
        }
        __syncwarp();

        // this lane's slots: data blocks b = 8*lane + i - (256 - nb)
        unsigned long long yh = 0, yl = 0;
        if (MODE == kSeal && !keyed) {
            // B = P: copy the chunk into the stage
            const uint8_t *src = q.plain_in + (size_t)s * q.plain_stride + (size_t)kChunk * c;
            for (uint32_t b = lane; b < nb; b += 32)
                *reinterpret_cast<uint4 *>(st + 16 * b) = *reinterpret_cast<const uint4 *>(src + 16 * b);
            if constexpr (crc) {
                if (ckind) {  // the lane's slots, as the keyed path below visits them, back out of the stage
                    __syncwarp();
                    for (uint32_t i = 0; i < 8; i++) {
                        const int b = (int)(8 * lane + i) - (int)(256 - nb);
                        if (b < 0) continue;
                        const uint32_t valid = min(16u, clen - 16u * (uint32_t)b);
                        const unsigned long long ma = valid >= 8 ? ~0ull : ((1ull << (8 * valid)) - 1),
                                                 mb = valid >= 16 ? ~0ull : valid <= 8 ? 0ull : ((1ull << (8 * (valid - 8))) - 1);
                        cv = crc_block16(sm.crc_slice[ckind - 1], cv,
                                         *reinterpret_cast<const unsigned long long *>(st + 16 * b) & ma,
                                         *reinterpret_cast<const unsigned long long *>(st + 16 * b + 8) & mb);
                    }
                }
            }
        } else {
#pragma unroll 1
            for (uint32_t i = 0; i < 8; i++) {
                const int b = (int)(8 * lane + i) - (int)(256 - nb);
                if (b < 0) continue;
                // ranged open: only the counter blocks that overlap the range
                if (MODE == kRangeOpen && (kChunk * c + 16 * (uint32_t)b >= off + len || kChunk * c + 16 * (uint32_t)b + 16 <= off))
                    continue;
                const uint32_t valid = min(16u, clen - 16u * (uint32_t)b);
                unsigned long long ch, cl;
                if (checking) {
                    ch = *reinterpret_cast<const unsigned long long *>(st + kPrefix + 16 * b);
                    cl = *reinterpret_cast<const unsigned long long *>(st + kPrefix + 16 * b + 8);
                } else {
                    uint32_t k0 = nw0, k1 = nw1, k2 = nw2, k3 = (uint32_t)b + 2;
                    aes256_encrypt(sm.t, sm.rk[wid], k0, k1, k2, k3);
                    // keystream in memory byte order (little-endian 64-bit words of the block)
                    const unsigned long long ksa = bswap64(((unsigned long long)k0 << 32) | k1),
                                             ksb = bswap64(((unsigned long long)k2 << 32) | k3);
                    unsigned long long pa, pb;
                    if (MODE == kSeal) {
                        const uint4 p = *reinterpret_cast<const uint4 *>(q.plain_in + (size_t)s * q.plain_stride +
                                                                         (size_t)kChunk * c + 16 * b);
                        pa = ((unsigned long long)p.y << 32) | p.x;
                        pb = ((unsigned long long)p.w << 32) | p.z;
                    } else {
                        pa = *reinterpret_cast<const unsigned long long *>(st + kPrefix + 16 * b);
                        pb = *reinterpret_cast<const unsigned long long *>(st + kPrefix + 16 * b + 8);
                    }
                    // mask to the valid bytes
                    const unsigned long long ma = valid >= 8 ? ~0ull : ((1ull << (8 * valid)) - 1),
                                             mb = valid >= 16 ? ~0ull : valid <= 8 ? 0ull : ((1ull << (8 * (valid - 8))) - 1);
                    if constexpr (crc) {
                        if (ckind) cv = crc_block16(sm.crc_slice[ckind - 1], cv, pa & ma, pb & mb);
                    }
                    const unsigned long long oa = (pa ^ ksa) & ma, ob = (pb ^ ksb) & mb;
                    if (sealing || MODE == kRangeOpen) {
                        *reinterpret_cast<unsigned long long *>(st + kPrefix + 16 * b) = oa;
                        *reinterpret_cast<unsigned long long *>(st + kPrefix + 16 * b + 8) = ob;
                        if (MODE == kRangeOpen) continue;
                        ch = oa;
                        cl = ob;
                    } else {
                        uint8_t *dst = q.plain_out + (size_t)s * q.plain_stride + (size_t)kChunk * c + 16 * b;
                        *reinterpret_cast<uint4 *>(dst) =
                            make_uint4((uint32_t)oa, (uint32_t)(oa >> 32), (uint32_t)ob, (uint32_t)(ob >> 32));
                        continue;
                    }
                }
                if (checking && valid < 16) {  // zero-pad the last block for GHASH
                    const unsigned long long ma = valid >= 8 ? ~0ull : ((1ull << (8 * valid)) - 1),
                                             mb = valid <= 8 ? 0ull : ((1ull << (8 * (valid - 8))) - 1);
                    ch &= ma;
                    cl &= mb;
                }
                // Horner: Y = (Y ^ C_b) * H, blocks as big-endian 128-bit values
                yh ^= bswap64(ch);
                yl ^= bswap64(cl);
                gf128_mul_h(sm.hh[wid], sm.hl[wid], sm.t.r4, yh, yl);
            }
        }

        if constexpr (crc) {
            // Fold (DESIGN.md 4.12): lane l's slots end at slot j = nb - 8(31 - l) of the chunk, and the chunk's grid at
            // slot 256c of the block's, so its share of acc = raw(P) * x^(-8 len(P)) is cv * x^(-128 (256c + j)).
            if (ckind) {
                const int t = (int)ckind - 1;
                const uint32_t poly = crc_poly(t);
                const int j = (int)nb - 8 * (31 - (int)lane);  // <= 0: no slot of the lane holds a byte, cv = 0
                cv = crc_mul(sm.crc_slot[t][max(j, 0)], cv, poly);
#pragma unroll
                for (int o = 16; o; o >>= 1) cv ^= __shfl_xor_sync(0xffffffffu, cv, o);
                if (lane == 0) {
                    cv = crc_mul(kCrcDev.chunk[t][c & 255], cv, poly);
                    for (uint32_t h = c >> 8, i = 0; h; h >>= 1, i++)
                        if (h & 1) cv = crc_mul(kCrcDev.chunk_hi[t][i], cv, poly);
                    atomicXor(q.crc_acc + s, cv);  // XOR: the order in which the chunks finish does not matter
                }
            }
        }

        if (MODE != kOpen && MODE != kRangeOpen && keyed) {
            if (lane != 31) gf128_mul_bits(yh, yl, K->pw[lane][0], K->pw[lane][1]);
            __syncwarp();  // the last data block's zero tail is in the stage before lane 0 writes the tag over it
#pragma unroll
            for (int o = 16; o; o >>= 1) {
                yh ^= __shfl_xor_sync(0xffffffffu, yh, o);
                yl ^= __shfl_xor_sync(0xffffffffu, yl, o);
            }
            if (lane == 0) {
                // S = (D ^ lengths) * H; T = E_K(J0) ^ S, J0 = nonce || 1
                yl ^= (unsigned long long)clen * 8;
                gf128_mul_h(sm.hh[wid], sm.hl[wid], sm.t.r4, yh, yl);
                uint32_t j0 = nw0, j1 = nw1, j2 = nw2, j3 = 1;
                aes256_encrypt(sm.t, sm.rk[wid], j0, j1, j2, j3);
                const unsigned long long th = yh ^ (((unsigned long long)j0 << 32) | j1),
                                         tl = yl ^ (((unsigned long long)j2 << 32) | j3);
                uint8_t *tp = st + kPrefix + clen;
                if (sealing) {
#pragma unroll
                    for (int i = 0; i < 8; i++) {
                        tp[i] = (uint8_t)(th >> (56 - 8 * i));
                        tp[8 + i] = (uint8_t)(tl >> (56 - 8 * i));
                    }
                    if (c == 0) {
#pragma unroll
                        for (int i = 0; i < 4; i++) {
                            st[i] = (uint8_t)(nw0 >> (24 - 8 * i));
                            st[4 + i] = (uint8_t)(nw1 >> (24 - 8 * i));
                        }
                    }
                } else {
                    const unsigned long long gh = load_be64(tp), gl = load_be64(tp + 8);
                    if (gh != th || gl != tl) q.status[s] = -7;  // GARAGE_EC_E_AUTH
                }
            }
        }
        if (MODE == kOpen && c == 0 && lane == 0) q.plain_len_out[s] = plen;

        if (MODE == kRangeOpen) {
            __syncwarp();
            // out positions [a, e) come from this chunk; the last chunk also writes the zero tail up to roundup16(len).
            // A vector shared with the neighbouring chunk is stored byte by byte, so two warps never write one byte.
            const uint32_t cb = kChunk * c, a = max(off, cb) - off, e = min(off + len, cb + clen) - off;
            const uint32_t ew = c == c1 ? (len + 15) & ~15u : e;
            uint8_t *dst = q.plain_out + (size_t)s * q.plain_stride;
            auto byte_at = [&](uint32_t x) -> uint8_t { return x < len ? st[kPrefix + off + x - cb] : (uint8_t)0; };
            for (uint32_t v = (a & ~15u) + 16 * lane; v < ew; v += 512) {
                if (v >= a && v + 16 <= ew) {
                    uint32_t wds[4] = {0, 0, 0, 0};
#pragma unroll
                    for (int b = 0; b < 16; b++) wds[b >> 2] |= (uint32_t)byte_at(v + b) << (8 * (b & 3));
                    *reinterpret_cast<uint4 *>(dst + v) = make_uint4(wds[0], wds[1], wds[2], wds[3]);
                } else {
                    for (uint32_t x = max(v, a); x < min(v + 16, ew); x++) dst[x] = byte_at(x);
                }
            }
        }

        if (sealing) {
            __syncwarp();
            // store this chunk's part of B: [start, end) -- chunk 0 from 0 (the nonce), the last chunk to k*L (the
            // zero tail); bytes past L of a shard, up to roundup16(L), are zero and belong to the chunk that owns
            // the shard's last byte
            const uint32_t start = c == 0 ? 0 : prefix + pitch * c;
            const uint32_t end = last ? q.k * L : prefix + pitch * (c + 1);
            const uint32_t Lr = (L + 15) & ~15u;
            for (uint32_t j = start / L; j * L < end && j < q.k; j++) {
                const uint32_t x0 = max(start, j * L) - j * L;
                uint32_t x1 = min(end, (j + 1) * L) - j * L;
                if (x1 == L) x1 = Lr;
                uint8_t *sh = stripe + (size_t)j * q.stride;
                auto byte_at = [&](uint32_t x) -> uint8_t {
                    const uint32_t p = j * L + x;
                    return (x >= L || p >= blen) ? (uint8_t)0 : st[p - base];
                };
                for (uint32_t v = (x0 & ~15u) + 16 * lane; v < x1; v += 512) {
                    if (v >= x0 && v + 16 <= x1) {
                        uint32_t wds[4] = {0, 0, 0, 0};
                        if (j * L + v < blen && v < L) {
#pragma unroll
                            for (int b = 0; b < 16; b++) wds[b >> 2] |= (uint32_t)byte_at(v + b) << (8 * (b & 3));
                        }
                        *reinterpret_cast<uint4 *>(sh + v) = make_uint4(wds[0], wds[1], wds[2], wds[3]);
                    } else {
                        for (uint32_t x = max(v, x0); x < min(v + 16, x1); x++) sh[x] = byte_at(x);
                    }
                }
            }
        }
        __syncwarp();
    }
}

// ---- per-block lengths and framing ----------------------------------------------------------------------------
struct LensParams {
    const uint32_t *plain_len;   // seal: per block
    const uint32_t *sealed_in;   // open: per block
    uint32_t *blen;              // out: len(B) (seal)
    uint32_t *shard_len;         // out: L, 0 for a block that is skipped
    int32_t *status;             // open: out, 0 / GARAGE_EC_E_AUTH (framing) / GARAGE_EC_E_INVALID (geometry)
    uint8_t *want;               // open: out, (k+m) bytes per block, the data shards
    unsigned long long plain_stride;
    uint32_t stride, k, m, n, quantum, keyed, open;
};
__global__ void __launch_bounds__(256) sse_lens_kernel(const __grid_constant__ LensParams q)
{
    for (uint32_t s = blockIdx.x * blockDim.x + threadIdx.x; s < q.n; s += gridDim.x * blockDim.x) {
        if (!q.open) {
            const uint32_t len = q.plain_len[s];
            const uint64_t b = q.keyed ? sealed_len(len) : len;
            const uint64_t L = b > 0xffffffffull ? ~0ull : code_shard_len((uint32_t)b, (int)q.k, q.quantum);
            const bool bad = L > q.stride || len > q.plain_stride;
            q.blen[s] = bad ? 0u : (uint32_t)b;
            q.shard_len[s] = bad ? 0u : (uint32_t)L;
            continue;
        }
        const uint32_t b = q.sealed_in[s];
        const uint64_t L = code_shard_len(b, (int)q.k, q.quantum);
        const uint32_t r = (b - kPrefix) % kFrame;
        const bool framed = b >= kPrefix + 16 && !(r >= 1 && r < 16);
        uint64_t plen = 0;
        if (framed) plen = b - kPrefix - 16ull * ((b - kPrefix + kFrame - 1) / kFrame);
        const bool bad = L > q.stride || plen > q.plain_stride;
        q.status[s] = bad ? -1 /* GARAGE_EC_E_INVALID */ : framed ? 0 : -7 /* GARAGE_EC_E_AUTH */;
        q.shard_len[s] = bad ? 0u : (uint32_t)L;
        for (uint32_t i = 0; i < q.k + q.m; i++) q.want[(size_t)s * (q.k + q.m) + i] = i < q.k;
    }
}

// ---- ranged open: per-request framing and the two row decodes --------------------------------------------------
struct RangeLensParams {
    const uint32_t *sealed, *offset, *len;  // per request
    const uint8_t *present;                 // n*(k+m)
    int32_t *status;                        // out: 0 / GARAGE_EC_E_AUTH (framing) / GARAGE_EC_E_INVALID (geometry)
    uint32_t *blen2, *off2, *len2;          // out: decode 2s = the prefix B[0, 8), 2s + 1 = the span (empty if failed)
    uint8_t *present2;                      // out: 2n*(k+m), request s's map twice
    unsigned long long out_stride;
    uint32_t stride, k, m, n, quantum;
};
__global__ void __launch_bounds__(256) sse_range_lens_kernel(const __grid_constant__ RangeLensParams q)
{
    const uint32_t tot = q.k + q.m;
    for (uint32_t s = blockIdx.x * blockDim.x + threadIdx.x; s < q.n; s += gridDim.x * blockDim.x) {
        const uint32_t S = q.sealed[s], o = q.offset[s], len = q.len[s];
        uint32_t so = 0, sl = 0, c0, nch;
        int32_t st = code_shard_len(S, (int)q.k, q.quantum) > q.stride ? -1 : sealed_range(S, o, len, &so, &sl, &c0, &nch);
        if (!st && ((uint64_t)len + 15) / 16 * 16 > q.out_stride) st = -1;
        q.status[s] = st;
        const bool go = !st && len;
        q.blen2[2 * s] = q.blen2[2 * s + 1] = go ? S : 0u;
        q.off2[2 * s] = 0;
        q.len2[2 * s] = go ? kPrefix : 0u;
        q.off2[2 * s + 1] = go ? so : 0u;
        q.len2[2 * s + 1] = go ? sl : 0u;
        for (uint32_t i = 0; i < tot; i++)
            q.present2[(2 * (size_t)s) * tot + i] = q.present2[(2 * (size_t)s + 1) * tot + i] = q.present[(size_t)s * tot + i];
    }
}

// ---- reseal: source framing, piece lists and destination lengths (DESIGN.md 4.11) ---------------------------------
// plaintext length of a source stored as S bytes, or ~0u when a keyed S cannot be framed (no piece is checked then:
// the source fails with GARAGE_EC_E_AUTH)
__device__ __forceinline__ uint32_t reseal_src_plain(uint32_t S, bool keyed)
{
    if (!keyed) return S;
    const uint32_t r = (S - kPrefix) % kFrame;
    if (S < kPrefix + 16 || (r >= 1 && r < 16)) return ~0u;
    return S - kPrefix - 16 * ((S - kPrefix + kFrame - 1) / kFrame);
}

struct ResealLensParams {
    const uint32_t *src_len, *pieces, *piece_start;
    int32_t *src_status;        // out: 0 / GARAGE_EC_E_AUTH (framing) / GARAGE_EC_E_INVALID (L past stride)
    uint32_t *src_L;            // out: L, 0 for a source that is not read
    uint8_t *want;              // out: n_src*(k+m), the data shards
    int32_t *status;            // out: 0 / GARAGE_EC_E_INVALID (piece list, L' past stride)
    uint32_t *dst_plen, *dst_blen, *dst_L;  // out: |Q_d|, sealed_len(|Q_d|), L' (0 when invalid)
    uint32_t stride, k, m, n_src, n_dst, quantum, keyed;
};
__global__ void __launch_bounds__(256) sse_reseal_lens_kernel(const __grid_constant__ ResealLensParams q)
{
    const uint32_t tot = q.k + q.m;
    for (uint32_t x = blockIdx.x * blockDim.x + threadIdx.x; x < max(q.n_src, q.n_dst); x += gridDim.x * blockDim.x) {
        if (x < q.n_src) {
            const uint32_t S = q.src_len[x];
            const uint64_t L = code_shard_len(S, (int)q.k, q.quantum);
            const bool bad = L > q.stride;
            q.src_status[x] = bad ? -1 : reseal_src_plain(S, q.keyed) == ~0u ? -7 : 0;
            q.src_L[x] = bad ? 0u : (uint32_t)L;
            for (uint32_t i = 0; i < tot; i++) q.want[(size_t)x * tot + i] = i < q.k;
        }
        if (x < q.n_dst) {
            const uint32_t p0 = q.piece_start[x], p1 = q.piece_start[x + 1];
            bool ok = p1 > p0;
            uint64_t Q = 0;
            for (uint32_t p = p0; ok && p < p1; p++) {
                const uint32_t src = q.pieces[3 * (size_t)p], off = q.pieces[3 * (size_t)p + 1],
                               len = q.pieces[3 * (size_t)p + 2];
                ok = src < q.n_src && len > 0;
                if (ok) {
                    const uint32_t P = reseal_src_plain(q.src_len[src], q.keyed);
                    ok = P == ~0u || (uint64_t)off + len <= P;
                }
                Q += len;
            }
            const uint64_t B = sealed_len(Q);
            const uint64_t L = ok && B <= 0xffffffffull ? code_shard_len((uint32_t)B, (int)q.k, q.quantum) : ~0ull;
            ok = ok && L <= q.stride;
            q.status[x] = ok ? 0 : -1;
            q.dst_plen[x] = ok ? (uint32_t)Q : 0u;
            q.dst_blen[x] = ok ? (uint32_t)B : 0u;
            q.dst_L[x] = ok ? (uint32_t)L : 0u;
        }
    }
}

// A destination is resealed only if every source it names is proven: status[d] becomes GARAGE_EC_E_UNRECOVERABLE if
// one is unrecoverable or does not hash to its address, else GARAGE_EC_E_AUTH, else GARAGE_EC_E_INVALID (its own
// lens verdict or a named source's geometry).  A destination that fails gets L' = len(B') = 0, so that no later
// kernel writes its shards; one that passes gets dst_len_out.  Sources: the reconstruct's verdict joins src_status.
struct ResealVerdictParams {
    const uint32_t *pieces, *piece_start;
    const int32_t *rec;           // n_src: the reconstruct's status
    const uint8_t *hash_bad;
    int32_t *src_status, *status;
    uint32_t *dst_blen, *dst_L, *dst_len_out;
    uint32_t n_src, n_dst;
};
__device__ __forceinline__ int32_t reseal_src_verdict(const ResealVerdictParams &q, uint32_t i)
{
    const int32_t st = q.rec[i] ? q.rec[i] : q.src_status[i];
    return st == -1 ? -1 : q.hash_bad[i] ? -4 /* GARAGE_EC_E_UNRECOVERABLE */ : st;
}
__global__ void __launch_bounds__(256) sse_reseal_verdict_kernel(const __grid_constant__ ResealVerdictParams q)
{
    for (uint32_t x = blockIdx.x * blockDim.x + threadIdx.x; x < max(q.n_src, q.n_dst); x += gridDim.x * blockDim.x) {
        if (x < q.n_src && q.rec[x]) q.src_status[x] = q.rec[x];
        if (x >= q.n_dst) continue;
        bool unrec = false, auth = false, inval = q.status[x] != 0;
        for (uint32_t p = q.piece_start[x]; p < q.piece_start[x + 1]; p++) {
            const uint32_t i = q.pieces[3 * (size_t)p];
            if (i >= q.n_src) continue;  // the lens verdict already says GARAGE_EC_E_INVALID
            const int32_t v = reseal_src_verdict(q, i);
            unrec |= v == -4;
            auth |= v == -7;
            inval |= v == -1;
        }
        const int32_t st = unrec ? -4 : auth ? -7 : inval ? -1 : 0;
        q.status[x] = st;
        if (st) {
            q.dst_blen[x] = q.dst_L[x] = 0;
        } else {
            q.dst_len_out[x] = q.dst_blen[x];
        }
    }
}

// ---- checksums: before and after the kCrc chunk kernel (DESIGN.md 4.12) ------------------------------------------
// Before (final = 0): zero each block's accumulator, and make a block of unknown kind malformed as an L past the
// stride makes it -- seal: L = len(B) = 0; reseal (status != NULL, ahead of the verdict): GARAGE_EC_E_INVALID.
// After (final = 1): crcs[s] = the CRC of a written block with a kind, 0 for every other block.
struct CrcPassParams {
    const uint8_t *kind;
    uint32_t *acc;
    uint32_t *shard_len;        // L, 0 = not written
    uint32_t *blen;             // before, seal
    int32_t *status;            // before, reseal
    const uint32_t *plain_len;  // after
    uint32_t *crcs;             // after
    uint32_t n, final;
};
__global__ void __launch_bounds__(256) sse_crc_pass_kernel(const __grid_constant__ CrcPassParams q)
{
    for (uint32_t s = blockIdx.x * blockDim.x + threadIdx.x; s < q.n; s += gridDim.x * blockDim.x) {
        const uint32_t k = q.kind[s];
        if (!q.final) {
            q.acc[s] = 0;
            if (k > 2) {
                if (q.status) {
                    q.status[s] = -1;  // GARAGE_EC_E_INVALID
                } else {
                    q.shard_len[s] = 0;
                    q.blen[s] = 0;
                }
            }
        } else {
            q.crcs[s] = k && k <= 2 && q.shard_len[s] ? crc_finish(kCrcDev, (int)k - 1, q.acc[s], q.plain_len[s]) : 0u;
        }
    }
}

}  // namespace sse
}  // namespace garage_ec
