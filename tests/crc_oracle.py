"""ctypes loader for the scalar CRC oracle (oracle/crc_oracle.c -> oracle/libcrc_oracle.so): bitwise CRC32 / CRC32C and
a combine by zlib's GF(2) matrix squaring (DESIGN.md 2.9).  Test infrastructure only, like sse_c_oracle."""
import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "oracle", "crc_oracle.c")
SO = os.path.join(ROOT, "oracle", "libcrc_oracle.so")

CRC32, CRC32C = 1, 2


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
        L.crc_oracle.argtypes = [C.c_int, C.c_void_p, C.c_size_t]
        L.crc_oracle.restype = C.c_uint32
        L.crc_oracle_combine.argtypes = [C.c_int, C.c_uint32, C.c_uint32, C.c_uint64]
        L.crc_oracle_combine.restype = C.c_uint32
        _lib = L
    return _lib


def crc(kind, data):
    a = np.ascontiguousarray(np.frombuffer(bytes(data), dtype=np.uint8) if not isinstance(data, np.ndarray) else data,
                             dtype=np.uint8)
    return int(lib().crc_oracle(kind, a.ctypes.data_as(C.c_void_p) if a.size else None, a.size))


def combine(kind, crc_a, crc_b, len_b):
    return int(lib().crc_oracle_combine(kind, crc_a, crc_b, len_b))
