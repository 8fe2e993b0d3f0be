// shard_wire.cpp -- msgpack (rmp-serde struct-map) encoding of the erasure-coded PutBlock message,
// versioned like garage_util::migrate::Migrate (see include/garage_shard_wire.h for the layout and
// the reference file:line it mirrors).  Host code only.
#include "../../include/garage_shard_wire.h"

#include <string.h>

namespace {

struct Writer {
    uint8_t *p;
    size_t cap, n = 0;
    bool ok = true;
    void put(const void *src, size_t len)
    {
        if (n + len > cap) {
            ok = false;
            return;
        }
        memcpy(p + n, src, len);
        n += len;
    }
    void byte(uint8_t b) { put(&b, 1); }
    void str(const char *s)  // fixstr (all our keys / variant names are < 32 bytes)
    {
        const size_t len = strlen(s);
        byte((uint8_t)(0xa0 | len));
        put(s, len);
    }
    void bin32(const uint8_t *b)  // bin8, 32 bytes: how serde_bytes writes a FixedBytes32
    {
        byte(0xc4);
        byte(32);
        put(b, 32);
    }
    void uint(uint64_t v)  // smallest msgpack unsigned encoding, as rmp does
    {
        if (v < 128) {
            byte((uint8_t)v);
        } else if (v < 256) {
            byte(0xcc);
            byte((uint8_t)v);
        } else if (v < 65536) {
            byte(0xcd);
            byte((uint8_t)(v >> 8));
            byte((uint8_t)v);
        } else {
            byte(0xce);
            for (int s = 24; s >= 0; s -= 8) byte((uint8_t)(v >> s));
        }
    }
};

struct Reader {
    const uint8_t *p;
    size_t len, n = 0;
    bool ok = true;
    uint8_t byte()
    {
        if (n >= len) {
            ok = false;
            return 0;
        }
        return p[n++];
    }
    bool str(char *out, size_t cap)  // fixstr / str8
    {
        uint8_t t = byte();
        size_t l;
        if ((t & 0xe0) == 0xa0) l = t & 0x1f;
        else if (t == 0xd9) l = byte();
        else return ok = false;
        if (!ok || n + l > len || l + 1 > cap) return ok = false;
        memcpy(out, p + n, l);
        out[l] = 0;
        n += l;
        return true;
    }
    bool bin32(uint8_t *out)
    {
        if (byte() != 0xc4 || byte() != 32 || !ok || n + 32 > len) return ok = false;
        memcpy(out, p + n, 32);
        n += 32;
        return true;
    }
    bool uint(uint64_t &v)
    {
        uint8_t t = byte();
        if (!ok) return false;
        if (t < 128) {
            v = t;
            return true;
        }
        int nb = t == 0xcc ? 1 : (t == 0xcd ? 2 : (t == 0xce ? 4 : (t == 0xcf ? 8 : 0)));
        if (!nb) return ok = false;
        v = 0;
        for (int i = 0; i < nb; i++) v = (v << 8) | byte();
        return ok;
    }
};

const char *variant_name(int header) { return header == GARAGE_SHARD_HEADER_COMPRESSED ? "Compressed" : "Plain"; }

bool parse_variant(const char *s, uint8_t &out)
{
    if (!strcmp(s, "Plain")) out = GARAGE_SHARD_HEADER_PLAIN;
    else if (!strcmp(s, "Compressed")) out = GARAGE_SHARD_HEADER_COMPRESSED;
    else return false;
    return true;
}

// decode a struct map; `full` = the v1 field set is required
bool decode_map(const uint8_t *bytes, size_t len, garage_shard_header *h, bool full)
{
    Reader r{bytes, len};
    const uint8_t t = r.byte();
    if (!r.ok || (t & 0xf0) != 0x80) return false;  // fixmap
    const int nf = t & 0x0f;
    unsigned seen = 0;
    for (int f = 0; f < nf; f++) {
        char key[24], val[24];
        if (!r.str(key, sizeof(key))) return false;
        uint64_t v = 0;
        if (!strcmp(key, "hash")) {
            if (!r.bin32(h->hash)) return false;
            seen |= 1;
        } else if (!strcmp(key, "header")) {
            if (!r.str(val, sizeof(val)) || !parse_variant(val, h->header)) return false;
            seen |= 2;
        } else if (!strcmp(key, "sum")) {
            if (!r.bin32(h->sum)) return false;
            seen |= 4;
        } else {
            if (!r.uint(v)) return false;
            if (!strcmp(key, "k")) h->k = (uint8_t)v, seen |= 8;
            else if (!strcmp(key, "m")) h->m = (uint8_t)v, seen |= 16;
            else if (!strcmp(key, "index")) h->index = (uint8_t)v, seen |= 32;
            else if (!strcmp(key, "block_len")) h->block_len = (uint32_t)v, seen |= 64;
            else if (!strcmp(key, "shard_len")) h->shard_len = (uint32_t)v, seen |= 128;
            else if (!strcmp(key, "sum_kind")) h->sum_kind = (uint8_t)v, seen |= 256;
            else if (full && !strcmp(key, "l") && v > 0) h->l = (uint8_t)v, seen |= 512;
            else if (full && !strcmp(key, "pb") && v == 1) h->pb = 1, seen |= 1024;
            else if (full && !strcmp(key, "clay") && v == 1) h->clay = 1, seen |= 2048;
            else return false;  // unknown field: not this format
            if (v > 0xffffffffull) return false;
        }
    }
    if (r.n != len) return false;
    return full ? (seen & 511) == 511 : seen == 3;
}

}  // namespace

extern "C" {

size_t garage_shard_wire_encode(const garage_shard_header *h, uint8_t *out, size_t cap)
{
    if (!h || !out || h->k < 1 || h->index >= h->k + h->m || h->header > 1) return 0;
    if (h->l && (h->l >= h->m || h->k % h->l)) return 0;
    if (h->pb > 1 || (h->pb && (h->l || h->m < 2 || h->m > 4 || h->k > 16))) return 0;
    if (h->clay > 1 || (h->clay && (h->l || h->pb || h->m < 2 || h->m > 4))) return 0;
    Writer w{out, cap};
    w.put(GARAGE_SHARD_WIRE_MARKER, 8);
    w.byte((uint8_t)(0x89 + (h->l ? 1 : 0) + (h->pb ? 1 : 0) + (h->clay ? 1 : 0)));  // fixmap, 9 fields (+ "l", "pb", "clay"), in declaration order like serde
    w.str("hash");
    w.bin32(h->hash);
    w.str("header");
    w.str(variant_name(h->header));
    w.str("k");
    w.uint(h->k);
    w.str("m");
    w.uint(h->m);
    w.str("index");
    w.uint(h->index);
    w.str("block_len");
    w.uint(h->block_len);
    w.str("shard_len");
    w.uint(h->shard_len);
    w.str("sum_kind");
    w.uint(h->sum_kind);
    w.str("sum");
    w.bin32(h->sum);
    if (h->l) {  // skip_serializing_if = 0: RS messages keep their bytes
        w.str("l");
        w.uint(h->l);
    }
    if (h->pb) {  // likewise
        w.str("pb");
        w.uint(1);
    }
    if (h->clay) {
        w.str("clay");
        w.uint(1);
    }
    return w.ok ? w.n : 0;
}

size_t garage_shard_wire_encode_v0(const uint8_t hash[32], int header, uint8_t *out, size_t cap)
{
    if (!hash || !out) return 0;
    Writer w{out, cap};
    w.byte(0x82);
    w.str("hash");
    w.bin32(hash);
    w.str("header");
    w.str(variant_name(header));
    return w.ok ? w.n : 0;
}

int garage_shard_wire_decode(const uint8_t *bytes, size_t len, garage_shard_header *out)
{
    if (!bytes || !out) return -1;
    garage_shard_header h;
    memset(&h, 0, sizeof(h));
    // Migrate::decode: the marker and the current format first ...
    if (len > 8 && !memcmp(bytes, GARAGE_SHARD_WIRE_MARKER, 8) && decode_map(bytes + 8, len - 8, &h, true)) {
        if (h.k < 1 || h.index >= h.k + h.m || (h.l && (h.l >= h.m || h.k % h.l))) return -1;
        if (h.pb && (h.l || h.m < 2 || h.m > 4 || h.k > 16)) return -1;
        if (h.clay && (h.l || h.pb || h.m < 2 || h.m > 4)) return -1;
        *out = h;
        return 0;
    }
    // ... else the previous version, migrated: a replicated block is the single shard of a 1+0 code
    memset(&h, 0, sizeof(h));
    if (decode_map(bytes, len, &h, false)) {
        h.k = 1;
        h.m = 0;
        h.index = 0;
        h.migrated = 1;
        *out = h;
        return 0;
    }
    return -1;
}

}  // extern "C"
