/* crc_oracle.c -- scalar reference of the S3 CRC32 / CRC32C checksums (DESIGN.md 2.9), for the tests only.
 *
 * Deliberately unlike the library: the CRC is bit by bit with no table, and combine shifts by len_b zero bytes with
 * zlib's GF(2) matrix squaring (an operator matrix for one zero bit, squared to 2, 4, 8 ... bits) rather than with
 * powers of x.  kind 1 = CRC32 (reflected 0xEDB88320), 2 = CRC32C (reflected 0x82F63B78); init and final XOR
 * 0xFFFFFFFF. */
#include <stddef.h>
#include <stdint.h>

static uint32_t poly_of(int kind) { return kind == 2 ? 0x82F63B78u : 0xEDB88320u; }

uint32_t crc_oracle(int kind, const uint8_t *p, size_t n)
{
    const uint32_t poly = poly_of(kind);
    uint32_t c = 0xFFFFFFFFu;
    for (size_t i = 0; i < n; i++) {
        c ^= p[i];
        for (int b = 0; b < 8; b++) c = (c & 1u) ? (c >> 1) ^ poly : c >> 1;
    }
    return c ^ 0xFFFFFFFFu;
}

static uint32_t mat_times(const uint32_t *m, uint32_t v)
{
    uint32_t s = 0;
    for (int i = 0; v; i++, v >>= 1)
        if (v & 1u) s ^= m[i];
    return s;
}

static void mat_square(uint32_t *sq, const uint32_t *m)
{
    for (int i = 0; i < 32; i++) sq[i] = mat_times(m, m[i]);
}

/* CRC(A || B) from CRC(A), CRC(B) and |B| */
uint32_t crc_oracle_combine(int kind, uint32_t crc_a, uint32_t crc_b, uint64_t len_b)
{
    uint32_t even[32], odd[32];
    if (len_b == 0) return crc_a;
    odd[0] = poly_of(kind);  /* the operator for one zero bit */
    for (int i = 1; i < 32; i++) odd[i] = 1u << (i - 1);
    mat_square(even, odd);   /* two zero bits */
    mat_square(odd, even);   /* four */
    do {
        mat_square(even, odd);  /* one zero byte, then 2, 4 ... */
        if (len_b & 1) crc_a = mat_times(even, crc_a);
        len_b >>= 1;
        if (!len_b) break;
        mat_square(odd, even);
        if (len_b & 1) crc_a = mat_times(odd, crc_a);
        len_b >>= 1;
    } while (len_b);
    return crc_a ^ crc_b;
}
