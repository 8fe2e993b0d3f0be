"""Generates sse_c_kat.json: SSE-C sealed blocks (DESIGN.md 2.6) made with the `cryptography` package's AES-256-GCM,
chunked the way aead's StreamLE31 frames Garage's 4096-byte chunks: nonce N || LE32(c | last << 31) per chunk, B = N ||
chunks.  Plaintexts come from a seeded generator; each record keeps the sealed block (or its SHA-256 when large) and
its blake2sum, the block's content address.  Run: python tests/golden/make_sse_c_kat.py"""
import hashlib
import json
import os
import struct

from cryptography.hazmat.primitives.ciphers.aead import AESGCM

HERE = os.path.dirname(os.path.abspath(__file__))
LENS = [0, 1, 15, 16, 4095, 4096, 4097, 8192, (1 << 20) - 1, 1 << 20]


def plain(n, seed):
    out = bytearray()
    ctr = 0
    while len(out) < n:
        out += hashlib.sha256(b"sse-c-kat %d %d" % (seed, ctr)).digest()
        ctr += 1
    return bytes(out[:n])


def seal(key, nonce8, pt):
    g = AESGCM(key)
    n = max(1, -(-len(pt) // 4096))
    out = bytearray(nonce8)
    for c in range(n):
        iv = nonce8 + struct.pack("<I", c | ((c == n - 1) << 31))
        out += g.encrypt(iv, pt[4096 * c:4096 * (c + 1)], None)
    return bytes(out)


def main():
    recs = []
    for i, n in enumerate(LENS):
        key = hashlib.sha256(b"key %d" % i).digest()
        nonce = hashlib.sha256(b"nonce %d" % i).digest()[:8]
        b = seal(key, nonce, plain(n, i))
        r = {"len": n, "key": key.hex(), "nonce": nonce.hex(), "sealed_len": len(b),
             "blake2sum": hashlib.blake2b(b).digest()[:32].hex()}
        if len(b) <= 9000:
            r["sealed"] = b.hex()
        else:
            r["sealed_sha256"] = hashlib.sha256(b).hexdigest()
        recs.append(r)
    with open(os.path.join(HERE, "sse_c_kat.json"), "w") as f:
        json.dump({"plain": "sha256(b'sse-c-kat <index> <counter>') stream", "records": recs}, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
