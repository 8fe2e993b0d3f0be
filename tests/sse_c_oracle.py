"""ctypes loader for the scalar SSE-C oracle (oracle/sse_c_oracle.c -> oracle/libsse_c_oracle.so): AES-256 from
FIPS-197, GCM from NIST SP 800-38D and the STREAM-LE31 chunk framing of Garage's SSE-C blocks (DESIGN.md 2.6).
Test infrastructure only, like oracle_lib."""
import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "oracle", "sse_c_oracle.c")
SO = os.path.join(ROOT, "oracle", "libsse_c_oracle.so")


def build(force=False):
    if force or not os.path.exists(SO) or (os.path.exists(SRC) and os.path.getmtime(SRC) > os.path.getmtime(SO)):
        tmp = SO + ".tmp%d" % os.getpid()
        subprocess.run([os.environ.get("CC", "gcc"), "-O2", "-fPIC", "-shared", "-Wall", "-Wextra", "-std=c11",
                        "-o", tmp, SRC], check=True)
        os.replace(tmp, SO)
    return SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(SO)
        vp, sz = C.c_void_p, C.c_size_t
        L.sse_oracle_aes256_expand.argtypes = [vp, vp]
        L.sse_oracle_aes256_encrypt.argtypes = [vp, vp, vp]
        L.sse_oracle_gcm_seal.argtypes = [vp, vp, sz, vp, sz, vp, sz, vp]
        L.sse_oracle_gcm_open.argtypes = [vp, vp, vp, sz, vp, vp]
        L.sse_oracle_sealed_len.argtypes = [sz]
        L.sse_oracle_sealed_len.restype = sz
        L.sse_oracle_seal.argtypes = [vp, vp, vp, sz, vp]
        L.sse_oracle_open.argtypes = [vp, vp, sz, vp]
        L.sse_oracle_open.restype = C.c_long
        _lib = L
    return _lib


def _buf(b):
    a = np.frombuffer(bytes(b), dtype=np.uint8).copy() if not isinstance(b, np.ndarray) else np.ascontiguousarray(b)
    return a, (a.ctypes.data_as(C.c_void_p) if a.size else None)


def aes256_encrypt(key, block):
    k, kp = _buf(key)
    rk = np.zeros(240, dtype=np.uint8)
    lib().sse_oracle_aes256_expand(kp, rk.ctypes.data_as(C.c_void_p))
    b, bp = _buf(block)
    out = np.zeros(16, dtype=np.uint8)
    lib().sse_oracle_aes256_encrypt(rk.ctypes.data_as(C.c_void_p), bp, out.ctypes.data_as(C.c_void_p))
    return out.tobytes()


def gcm_seal(key, iv, pt, aad=b""):
    """AES-256-GCM (any IV length): ciphertext || 16-byte tag"""
    k, kp = _buf(key)
    v, vp_ = _buf(iv)
    a, ap = _buf(aad)
    p, pp = _buf(pt)
    out = np.zeros(len(p) + 16, dtype=np.uint8)
    lib().sse_oracle_gcm_seal(kp, vp_, len(v), ap, len(a), pp, len(p), out.ctypes.data_as(C.c_void_p))
    return out.tobytes()


def sealed_len(n):
    return int(lib().sse_oracle_sealed_len(n))


def seal(key, nonce8, pt):
    """the sealed block B of plaintext pt"""
    k, kp = _buf(key)
    nn, np_ = _buf(nonce8)
    p, pp = _buf(pt)
    out = np.zeros(sealed_len(len(p)), dtype=np.uint8)
    lib().sse_oracle_seal(kp, np_, pp, len(p), out.ctypes.data_as(C.c_void_p))
    return out.tobytes()


def open_(key, b):
    """plaintext of sealed block b, or None if it fails its framing or a tag"""
    k, kp = _buf(key)
    a, ap = _buf(b)
    out = np.zeros(max(len(a), 1), dtype=np.uint8)
    n = lib().sse_oracle_open(kp, ap, len(a), out.ctypes.data_as(C.c_void_p))
    return None if n < 0 else out[:n].tobytes()
