"""garage_b200 -- H100 (sm_90a) erasure-coding block path for Garage.

The product is ``libgarage_ec.so`` (CUDA kernels + the C ABI declared in
``include/garage_ec.h``).  This module is the thin ctypes harness the tests and the bench
drive it with; it mirrors the C ABI one to one (same names minus the ``garage_ec_`` prefix,
same argument meaning, same error codes) and adds nothing of its own.  There is no CPU
fallback: if the library cannot be loaded or no sm_90 device is present, calls raise.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from . import _build

__all__ = ["GarageEc", "EcError", "load_library", "lib_path", "ABI_SYMBOLS",
           "MEM_HOST", "MEM_DEVICE", "VANDERMONDE", "CAUCHY"]

OK = 0
E_INVALID, E_CUDA, E_NOMEM, E_UNRECOVERABLE, E_NODEVICE, E_ALIGN, E_AUTH = -1, -2, -3, -4, -5, -6, -7
VANDERMONDE, CAUCHY = 0, 1
MEM_HOST, MEM_DEVICE = 0, 1
MAX_K, MAX_M = 32, 8

# every symbol include/garage_ec.h declares (tests check the .so exports each one)
ABI_SYMBOLS = [
    "garage_ec_create", "garage_ec_create_with_matrix", "garage_ec_destroy", "garage_ec_matrix",
    "garage_ec_params", "garage_ec_strerror", "garage_ec_last_error", "garage_ec_abi_version",
    "garage_ec_shard_len", "garage_ec_stride_for", "garage_ec_encode", "garage_ec_reconstruct",
    "garage_ec_verify", "garage_ec_encode_blocks", "garage_ec_decode_blocks",
    "garage_ec_fill_random", "garage_ec_host_alloc", "garage_ec_host_alloc_wc", "garage_ec_host_free",
    "garage_ec_launch_count", "garage_ec_set_timing", "garage_ec_timing_read",
    "garage_ec_shard_sums", "garage_ec_check_sums", "garage_ec_blake2sum",
    "garage_ec_encode_blocks_with_sums", "garage_ec_scrub_repair",
    "garage_ec_numa_info", "garage_ec_bind_thread", "garage_ec_device_count", "garage_ec_debug_fail_after",
    "garage_ec_set_sum_kind", "garage_ec_set_wait_mode", "garage_ec_copy_for_dma", "garage_ec_shard_sum_host", "garage_ec_reconstruct_stripes",
    "garage_ec_create_lrc", "garage_ec_code_info", "garage_ec_read_set",
    "garage_ec_create_piggyback", "garage_ec_piggyback_info", "garage_ec_code_shard_len", "garage_ec_read_plan",
    "garage_ec_check_shard_half_host", "garage_ec_transcode",
    "garage_ec_create_clay", "garage_ec_clay_info", "garage_ec_read_ranges",
    "garage_ec_deep_check",
    "garage_ec_tag_span", "garage_ec_check_shard_span_host", "garage_ec_range_plan", "garage_ec_decode_range",
    "garage_ec_decode_range_stripes",
    "garage_ec_sealed_len", "garage_ec_seal", "garage_ec_seal_blocks", "garage_ec_open", "garage_ec_open_stripes",
    "garage_ec_sealed_range", "garage_ec_open_range_plan", "garage_ec_open_range", "garage_ec_open_range_stripes",
    "garage_ec_reseal", "garage_ec_reseal_stripes",
    "garage_ec_seal_crc", "garage_ec_seal_blocks_crc", "garage_ec_reseal_crc", "garage_ec_reseal_stripes_crc",
    "garage_ec_crc_combine",
    "garage_ec_reconstruct_segments", "garage_ec_reconstruct_segments_stripes", "garage_ec_segment_read_ranges",
]


class EcError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("garage_ec error %d: %s" % (code, msg))
        self.code = code


def lib_path():
    return _build.SO


_lib = None


def load_library(build=True):
    """Load libgarage_ec.so (building it in-tree first if sources are newer).  Raises if the
    CUDA extension is missing -- the product path never falls back to CPU code."""
    global _lib
    if _lib is not None:
        return _lib
    if build:
        try:
            _build.build()
        except Exception:
            if not os.path.exists(_build.SO):
                raise
    if not os.path.exists(_build.SO):
        raise RuntimeError("garage_b200: %s missing -- build it with __graft_entry__.build()" % _build.SO)
    L = C.CDLL(_build.SO)
    vp, sz, i32, u32, u64 = C.c_void_p, C.c_size_t, C.c_int, C.c_uint32, C.c_uint64
    L.garage_ec_create.argtypes = [C.POINTER(vp), i32, i32, i32, i32]
    L.garage_ec_create_with_matrix.argtypes = [C.POINTER(vp), i32, i32, i32, vp]
    L.garage_ec_destroy.argtypes = [vp]
    L.garage_ec_destroy.restype = None
    L.garage_ec_matrix.argtypes = [vp, vp]
    L.garage_ec_params.argtypes = [vp, C.POINTER(i32), C.POINTER(i32), C.POINTER(i32)]
    L.garage_ec_strerror.argtypes = [i32]
    L.garage_ec_strerror.restype = C.c_char_p
    L.garage_ec_last_error.argtypes = [vp]
    L.garage_ec_last_error.restype = C.c_char_p
    L.garage_ec_abi_version.restype = i32
    L.garage_ec_shard_len.argtypes = [u32, i32]
    L.garage_ec_shard_len.restype = u32
    L.garage_ec_stride_for.argtypes = [u32]
    L.garage_ec_stride_for.restype = sz
    L.garage_ec_encode.argtypes = [vp, vp, vp, vp, sz, sz, i32, vp]
    L.garage_ec_reconstruct.argtypes = [vp, vp, vp, vp, vp, vp, sz, sz, i32, vp]
    L.garage_ec_verify.argtypes = [vp, vp, vp, vp, sz, sz, i32, vp]
    L.garage_ec_encode_blocks.argtypes = [vp, vp, vp, sz, vp, sz]
    L.garage_ec_encode_blocks_with_sums.argtypes = [vp, vp, vp, sz, vp, vp, sz]
    L.garage_ec_scrub_repair.argtypes = [vp, vp, vp, vp, vp, vp, sz, sz, i32, vp]
    L.garage_ec_shard_sums.argtypes = [vp, vp, vp, sz, sz, i32, vp, i32, vp]
    L.garage_ec_check_sums.argtypes = [vp, vp, vp, vp, sz, sz, i32, vp, i32, vp]
    L.garage_ec_blake2sum.argtypes = [vp, sz, vp]
    L.garage_ec_blake2sum.restype = None
    L.garage_ec_decode_blocks.argtypes = [vp, vp, vp, vp, sz, sz, vp, vp]
    L.garage_ec_fill_random.argtypes = [vp, vp, sz, u64, u64, vp]
    L.garage_ec_host_alloc.argtypes = [vp, C.POINTER(vp), sz]
    L.garage_ec_host_alloc_wc.argtypes = [vp, C.POINTER(vp), sz]
    L.garage_ec_host_free.argtypes = [vp, vp]
    L.garage_ec_host_free.restype = None
    L.garage_ec_launch_count.argtypes = [vp]
    L.garage_ec_launch_count.restype = u64
    L.garage_ec_set_timing.argtypes = [vp, i32]
    L.garage_ec_timing_read.argtypes = [vp, C.POINTER(C.c_double), C.POINTER(u64)]
    L.garage_ec_numa_info.argtypes = [vp, C.POINTER(i32), C.POINTER(i32)]
    L.garage_ec_bind_thread.argtypes = [vp]
    L.garage_ec_device_count.argtypes = []
    L.garage_ec_debug_fail_after.argtypes = [vp, C.c_long]
    L.garage_ec_reconstruct_stripes.argtypes = [vp, vp, vp, vp, vp, vp, sz, sz]
    L.garage_ec_reconstruct_segments.argtypes = [vp, vp, vp, vp, vp, vp, sz, sz, i32, vp]
    L.garage_ec_reconstruct_segments_stripes.argtypes = [vp, vp, vp, vp, vp, vp, sz, sz]
    L.garage_ec_segment_read_ranges.argtypes = [vp, vp, vp, u32, vp, sz, C.POINTER(sz)]
    L.garage_ec_set_sum_kind.argtypes = [vp, i32]
    L.garage_ec_set_wait_mode.argtypes = [vp, i32]
    L.garage_ec_copy_for_dma.argtypes = [vp, vp, C.c_size_t]
    L.garage_ec_copy_for_dma.restype = None
    L.garage_ec_shard_sum_host.argtypes = [i32, vp, sz, vp]
    L.garage_ec_create_lrc.argtypes = [C.POINTER(vp), i32, i32, i32, i32]
    L.garage_ec_code_info.argtypes = [vp, C.POINTER(i32), C.POINTER(i32)]
    L.garage_ec_read_set.argtypes = [vp, vp, vp, vp]
    L.garage_ec_create_piggyback.argtypes = [C.POINTER(vp), i32, i32, i32, i32]
    L.garage_ec_piggyback_info.argtypes = [vp, C.POINTER(i32), vp]
    L.garage_ec_code_shard_len.argtypes = [vp, u32, C.POINTER(u32)]
    L.garage_ec_read_plan.argtypes = [vp, vp, vp, vp]
    L.garage_ec_check_shard_half_host.argtypes = [i32, vp, u32, i32, vp]
    L.garage_ec_transcode.argtypes = [vp, vp, vp, vp, vp, sz, vp, sz, vp, vp, sz, i32, vp]
    L.garage_ec_create_clay.argtypes = [C.POINTER(vp), i32, i32, i32, i32]
    L.garage_ec_clay_info.argtypes = [vp, C.POINTER(i32), C.POINTER(i32), C.POINTER(i32), C.POINTER(i32), vp]
    L.garage_ec_read_ranges.argtypes = [vp, vp, vp, u32, vp, sz, C.POINTER(sz)]
    L.garage_ec_deep_check.argtypes = [vp, vp, vp, vp, vp, vp, sz, sz, i32, vp]
    L.garage_ec_tag_span.argtypes = [i32, u32, u32, u32, C.POINTER(u32), C.POINTER(u32)]
    L.garage_ec_check_shard_span_host.argtypes = [i32, vp, u32, u32, u32, vp]
    L.garage_ec_range_plan.argtypes = [vp, vp, u32, u32, u32, vp, sz, C.POINTER(sz), C.POINTER(i32)]
    L.garage_ec_decode_range.argtypes = [vp, vp, vp, vp, vp, vp, sz, vp, sz, vp, sz, i32, vp]
    L.garage_ec_decode_range_stripes.argtypes = [vp, vp, vp, vp, vp, vp, sz, vp, vp, sz]
    L.garage_ec_sealed_len.argtypes = [u32, C.POINTER(u32)]
    L.garage_ec_seal.argtypes = [vp, vp, sz, vp, vp, vp, vp, sz, vp, vp, sz, i32, vp]
    L.garage_ec_seal_blocks.argtypes = [vp, vp, vp, vp, vp, vp, sz, vp, vp, sz]
    L.garage_ec_open.argtypes = [vp, vp, vp, vp, vp, vp, vp, sz, vp, vp, vp, sz, sz, i32, vp]
    L.garage_ec_open_stripes.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, sz, sz]
    L.garage_ec_sealed_range.argtypes = [u32, u32, u32, C.POINTER(u32), C.POINTER(u32), C.POINTER(u32), C.POINTER(u32)]
    L.garage_ec_open_range_plan.argtypes = [vp, vp, u32, u32, u32, vp, sz, C.POINTER(sz), C.POINTER(i32)]
    L.garage_ec_open_range.argtypes = [vp, vp, vp, vp, vp, vp, vp, sz, vp, sz, vp, sz, i32, vp]
    L.garage_ec_open_range_stripes.argtypes = [vp, vp, vp, vp, vp, vp, vp, sz, vp, vp, sz]
    L.garage_ec_reseal.argtypes = [vp, vp, vp, vp, vp, vp, sz, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, sz, sz, i32, vp]
    L.garage_ec_reseal_stripes.argtypes = [vp, vp, vp, vp, vp, vp, sz, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, sz, sz]
    L.garage_ec_seal_crc.argtypes = [vp, vp, sz, vp, vp, vp, vp, sz, vp, vp, vp, vp, sz, i32, vp]
    L.garage_ec_seal_blocks_crc.argtypes = [vp, vp, vp, vp, vp, vp, sz, vp, vp, vp, vp, sz]
    L.garage_ec_reseal_crc.argtypes = [vp, vp, vp, vp, vp, vp, sz, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, sz,
                                       sz, i32, vp]
    L.garage_ec_reseal_stripes_crc.argtypes = [vp, vp, vp, vp, vp, vp, sz, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp,
                                               vp, sz, sz]
    L.garage_ec_crc_combine.argtypes = [i32, u32, u32, u64, C.POINTER(u32)]
    _lib = L
    return L


# S3 checksum kinds of the _crc seal and reseal forms (DESIGN.md 2.9)
CRC_NONE, CRC32, CRC32C = 0, 1, 2


def crc_combine(kind, crc_a, crc_b, len_b) -> int:
    """garage_ec_crc_combine (host only): the CRC of A || B from CRC(A), CRC(B) and len(B)"""
    v = C.c_uint32(0)
    rc = load_library().garage_ec_crc_combine(kind, crc_a, crc_b, len_b, C.byref(v))
    if rc:
        raise EcError(rc, "crc_combine")
    return v.value


def sealed_len(plain_len) -> int:
    """garage_ec_sealed_len: 8 + plain_len + 16 * max(1, ceil(plain_len / 4096))"""
    v = C.c_uint32(0)
    rc = load_library().garage_ec_sealed_len(plain_len, C.byref(v))
    if rc:
        raise EcError(rc, "sealed_len")
    return v.value


def blake2sum(data) -> bytes:
    """Garage's blake2sum (BLAKE2b-512 truncated to 32 bytes) through the library's host code."""
    L = load_library()
    a = np.frombuffer(bytes(data), dtype=np.uint8) if not isinstance(data, np.ndarray) else np.ascontiguousarray(data)
    out = np.zeros(32, dtype=np.uint8)
    L.garage_ec_blake2sum(C.c_void_p(a.ctypes.data) if a.size else None, a.size, C.c_void_p(out.ctypes.data))
    return out.tobytes()


SUM_BLAKE2, SUM_ADLER8 = 0, 1


def shard_sum_host(kind, data) -> bytes:
    """the 32-byte per-shard tag of `kind` computed by the library's host code"""
    L = load_library()
    a = np.frombuffer(bytes(data), dtype=np.uint8) if not isinstance(data, np.ndarray) else np.ascontiguousarray(data)
    out = np.zeros(32, dtype=np.uint8)
    rc = L.garage_ec_shard_sum_host(kind, C.c_void_p(a.ctypes.data) if a.size else None, a.size, C.c_void_p(out.ctypes.data))
    if rc:
        raise EcError(rc, "shard_sum_host")
    return out.tobytes()


def check_shard_half_host(kind, half, shard_len, which, tag) -> int:
    """garage_ec_check_shard_half_host: 0 if `half` (shard_len/2 bytes, which = 0 a-half / 1 b-half) matches its 4
    Adler-32 values in the 32-byte adler8 tag `tag`, 1 if not, or an E_* code"""
    L = load_library()
    a = np.frombuffer(bytes(half), dtype=np.uint8) if not isinstance(half, np.ndarray) else np.ascontiguousarray(half)
    t = np.frombuffer(bytes(tag), dtype=np.uint8)
    return L.garage_ec_check_shard_half_host(kind, C.c_void_p(a.ctypes.data) if a.size else None, shard_len, which,
                                             C.c_void_p(t.ctypes.data))


def tag_span(kind, shard_len, off, length):
    """garage_ec_tag_span: (span_off, span_len) of the whole tag segments covering [off, off + length) of a shard"""
    L = load_library()
    a, b = C.c_uint32(0), C.c_uint32(0)
    rc = L.garage_ec_tag_span(kind, shard_len, off, length, C.byref(a), C.byref(b))
    if rc:
        raise EcError(rc, "tag_span")
    return a.value, b.value


def check_shard_span_host(kind, span, shard_len, span_off, tag) -> int:
    """garage_ec_check_shard_span_host: 0 if `span` (the bytes of a tag span at span_off) matches the 32-byte tag,
    1 if not, or an E_* code"""
    L = load_library()
    a = np.frombuffer(bytes(span), dtype=np.uint8) if not isinstance(span, np.ndarray) else np.ascontiguousarray(span)
    t = np.frombuffer(bytes(tag), dtype=np.uint8)
    return L.garage_ec_check_shard_span_host(kind, C.c_void_p(a.ctypes.data) if a.size else None, shard_len, span_off,
                                             a.size, C.c_void_p(t.ctypes.data))


def copy_for_dma(dst, src):
    """copy `src` into `dst` (numpy uint8 views, dst normally pinned) with non-temporal stores: garage_ec_copy_for_dma"""
    assert dst.dtype == np.uint8 and src.dtype == np.uint8 and dst.size >= src.size
    load_library().garage_ec_copy_for_dma(C.c_void_p(dst.ctypes.data), C.c_void_p(src.ctypes.data), src.size)


def _ptr(x):
    """device tensor / numpy array / int / None -> void*"""
    if x is None:
        return None
    if isinstance(x, int):
        return C.c_void_p(x)
    if isinstance(x, np.ndarray):
        return C.c_void_p(x.ctypes.data)
    if hasattr(x, "data_ptr"):
        return C.c_void_p(x.data_ptr())
    raise TypeError(type(x))


def _is_device(x):
    return hasattr(x, "data_ptr") and getattr(x, "is_cuda", False)


class GarageEc:
    """One context = (GPU, k, m, matrix): mirrors ``garage_ec_ctx``.

    Buffers are torch CUDA uint8 tensors (DEVICE mode: enqueued on torch's current stream)
    or numpy uint8 arrays (HOST mode: synchronous, staged through the library's lanes).
    """

    def __init__(self, device=0, k=10, m=4, kind=VANDERMONDE, matrix=None, _lrc=None, _pb=False, _clay=False):
        self._L = load_library()
        h = C.c_void_p()
        if _clay:
            rc = self._L.garage_ec_create_clay(C.byref(h), device, k, m, kind)
        elif _pb:
            rc = self._L.garage_ec_create_piggyback(C.byref(h), device, k, m, kind)
        elif _lrc is not None:
            l, r = _lrc
            m = l + r
            rc = self._L.garage_ec_create_lrc(C.byref(h), device, k, l, r)
        elif matrix is not None:
            mat = np.ascontiguousarray(matrix, dtype=np.uint8)
            if mat.shape != (m, k):
                raise ValueError("matrix must be m x k")
            rc = self._L.garage_ec_create_with_matrix(C.byref(h), device, k, m, _ptr(mat))
        else:
            rc = self._L.garage_ec_create(C.byref(h), device, k, m, kind)
        if rc != OK:
            raise EcError(rc, self._L.garage_ec_strerror(rc).decode())
        self._h = h
        self.device, self.k, self.m = device, k, m

    @classmethod
    def lrc(cls, device=0, k=10, l=2, r=2):
        """LRC(k, l, r) context: l local XOR parities (one per group of k/l data shards), then r Cauchy parities"""
        return cls(device, k, l + r, _lrc=(l, r))

    @classmethod
    def piggyback(cls, device=0, k=10, m=4, kind=VANDERMONDE):
        """PB(k, m) context: RS(k, m) over two half-shards, b-halves of parities 1..m-1 carry the group XORs of a"""
        return cls(device, k, m, kind, _pb=True)

    @classmethod
    def clay(cls, device=0, k=10, m=4, kind=VANDERMONDE):
        """Clay(k, m) context: alpha = m^ceil((k+m)/m) coupled layers of RS(k+s, m); one lost shard is rebuilt from
        1/m of every other shard"""
        return cls(device, k, m, kind, _clay=True)

    # -- lifecycle
    def close(self):
        if getattr(self, "_h", None):
            self._L.garage_ec_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def _check(self, rc, allow=()):
        if rc != OK and rc not in allow:
            msg = self._L.garage_ec_strerror(rc).decode()
            if rc == E_CUDA:
                msg += " (" + self._L.garage_ec_last_error(self._h).decode() + ")"
            raise EcError(rc, msg)
        return rc

    def _stream(self, *bufs):
        if any(_is_device(b) for b in bufs):
            import torch

            return MEM_DEVICE, C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
        return MEM_HOST, None

    # -- introspection
    def matrix(self):
        out = np.zeros((self.m, self.k), dtype=np.uint8)
        self._check(self._L.garage_ec_matrix(self._h, _ptr(out)))
        return out

    def code_info(self):
        """(local groups, global parities): (l, r) for LRC, (0, m) for RS"""
        a, b = C.c_int(0), C.c_int(0)
        self._check(self._L.garage_ec_code_info(self._h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def read_set(self, present, want=None):
        """shards to fetch to rebuild the wanted absent shards of one stripe: (k+m,) uint8 array, or None if
        they cannot be rebuilt"""
        pr = np.ascontiguousarray(present, dtype=np.uint8)
        wn = None if want is None else np.ascontiguousarray(want, dtype=np.uint8)
        assert pr.shape == (self.k + self.m,) and (wn is None or wn.shape == pr.shape)
        out = np.zeros(self.k + self.m, dtype=np.uint8)
        rc = self._check(self._L.garage_ec_read_set(self._h, _ptr(pr), _ptr(wn), _ptr(out)), (E_UNRECOVERABLE,))
        return None if rc == E_UNRECOVERABLE else out

    def piggyback_info(self):
        """(groups, group_of): m-1 and the group (1..m-1) of every data shard for PB, (0, zeros) otherwise"""
        g = C.c_int(0)
        out = np.zeros(self.k, dtype=np.uint8)
        self._check(self._L.garage_ec_piggyback_info(self._h, C.byref(g), _ptr(out)))
        return g.value, out

    def read_plan(self, present, want=None):
        """halves to fetch per shard (bit 0 a-half, bit 1 b-half): (k+m,) uint8 array, or None if unrecoverable"""
        pr = np.ascontiguousarray(present, dtype=np.uint8)
        wn = None if want is None else np.ascontiguousarray(want, dtype=np.uint8)
        assert pr.shape == (self.k + self.m,) and (wn is None or wn.shape == pr.shape)
        out = np.zeros(self.k + self.m, dtype=np.uint8)
        rc = self._check(self._L.garage_ec_read_plan(self._h, _ptr(pr), _ptr(wn), _ptr(out)), (E_UNRECOVERABLE,))
        return None if rc == E_UNRECOVERABLE else out

    def clay_info(self):
        """(q, t, alpha, virtual nodes, m x (k+s) base rows) of a Clay context; (0, 0, 1, 0, None) otherwise"""
        v = [C.c_int(0) for _ in range(4)]
        rows = np.zeros(self.m * self.k + self.m * 4, dtype=np.uint8)
        self._check(self._L.garage_ec_clay_info(self._h, *[C.byref(x) for x in v], _ptr(rows)))
        q, t, alpha, s = (x.value for x in v)
        return q, t, alpha, s, (rows[: self.m * (self.k + s)].reshape(self.m, self.k + s) if q else None)

    def read_ranges(self, present, shard_len, want=None):
        """[(shard, offset, len)] byte runs to fetch for one stripe, or None if unrecoverable"""
        pr = np.ascontiguousarray(present, dtype=np.uint8)
        wn = None if want is None else np.ascontiguousarray(want, dtype=np.uint8)
        assert pr.shape == (self.k + self.m,) and (wn is None or wn.shape == pr.shape)
        cap = (self.k + self.m) * 256
        out = np.zeros(cap * 3, dtype=np.uint32)
        n = C.c_size_t(0)
        rc = self._check(self._L.garage_ec_read_ranges(self._h, _ptr(pr), _ptr(wn), shard_len, _ptr(out), cap,
                                                       C.byref(n)), (E_UNRECOVERABLE,))
        if rc == E_UNRECOVERABLE:
            return None
        return [tuple(int(v) for v in out[3 * i:3 * i + 3]) for i in range(n.value)]

    def segment_read_ranges(self, seg_present, shard_len, want=None, cap=None):
        """[(shard, offset, len)] byte runs reconstruct_segments reads to complete one stripe's wanted shards, or None
        if a unit is unrecoverable (DESIGN.md section 2.10)"""
        sp = np.ascontiguousarray(seg_present, dtype=np.uint8)
        wn = None if want is None else np.ascontiguousarray(want, dtype=np.uint8)
        assert sp.shape == (self.k + self.m,) and (wn is None or wn.shape == sp.shape)
        cap = (self.k + self.m) * 8 if cap is None else cap
        out = np.zeros(max(1, cap) * 3, dtype=np.uint32)
        n = C.c_size_t(0)
        rc = self._check(self._L.garage_ec_segment_read_ranges(self._h, _ptr(sp), _ptr(wn), shard_len, _ptr(out), cap,
                                                               C.byref(n)), (E_UNRECOVERABLE,))
        if rc == E_UNRECOVERABLE:
            return None
        return [tuple(int(v) for v in out[3 * i:3 * i + 3]) for i in range(n.value)]

    def range_plan(self, present, block_len, offset, length):
        """(runs [(shard, offset, len)], needs_gpu) for bytes [offset, offset + length) of one block, or (None,
        needs_gpu) if the absent touched data shards cannot be rebuilt"""
        pr = np.ascontiguousarray(present, dtype=np.uint8)
        assert pr.shape == (self.k + self.m,)
        cap = (self.k + self.m) * 512
        out = np.zeros(cap * 3, dtype=np.uint32)
        n, g = C.c_size_t(0), C.c_int(0)
        rc = self._check(self._L.garage_ec_range_plan(self._h, _ptr(pr), block_len, offset, length, _ptr(out), cap,
                                                      C.byref(n), C.byref(g)), (E_UNRECOVERABLE,))
        if rc == E_UNRECOVERABLE:
            return None, g.value
        return [tuple(int(v) for v in out[3 * i:3 * i + 3]) for i in range(n.value)], g.value

    def decode_range(self, shards, present, block_len, offset, length, stride, out, out_stride, status=None):
        """garage_ec_decode_range of n = len(block_len) requests (uint32 arrays, numpy or device tensors)"""
        kind, st = self._stream(shards)
        return self._check(self._L.garage_ec_decode_range(self._h, _ptr(shards), _ptr(present), _ptr(block_len),
                                                          _ptr(offset), _ptr(length), stride, _ptr(out), out_stride,
                                                          _ptr(status), len(block_len), kind, st),
                           (E_UNRECOVERABLE,))

    def decode_range_stripes(self, stripes, present, block_len, offset, length, stride, outs, status=None):
        """gather form: `stripes` / `outs` are lists of numpy arrays, one per request"""
        n = len(stripes)
        sp = (C.c_void_p * n)(*[a.ctypes.data for a in stripes])
        op = (C.c_void_p * n)(*[a.ctypes.data for a in outs])
        return self._check(self._L.garage_ec_decode_range_stripes(self._h, C.cast(sp, C.c_void_p), _ptr(present),
                                                                  _ptr(block_len), _ptr(offset), _ptr(length), stride,
                                                                  C.cast(op, C.c_void_p), _ptr(status), n),
                           (E_UNRECOVERABLE,))

    def code_shard_len(self, block_len):
        """shard length of a block under this context's code (PB: rounded up to 128 bytes)"""
        v = C.c_uint32(0)
        self._check(self._L.garage_ec_code_shard_len(self._h, block_len, C.byref(v)))
        return v.value

    def shard_len(self, block_len):
        return int(self._L.garage_ec_shard_len(block_len, self.k))

    def stride_for(self, shard_len):
        return int(self._L.garage_ec_stride_for(shard_len))

    def launch_count(self):
        return int(self._L.garage_ec_launch_count(self._h))

    def set_timing(self, on=True):
        self._check(self._L.garage_ec_set_timing(self._h, 1 if on else 0))

    def timing_read(self):
        ms, n = C.c_double(0), C.c_uint64(0)
        self._check(self._L.garage_ec_timing_read(self._h, C.byref(ms), C.byref(n)))
        return ms.value, n.value

    # -- the three batch operations (shard layout; see include/garage_ec.h)
    def encode(self, data, parity, stride, n, shard_len=None):
        kind, st = self._stream(data, parity)
        return self._check(self._L.garage_ec_encode(self._h, _ptr(data), _ptr(parity), _ptr(shard_len),
                                                    stride, n, kind, st))

    def reconstruct(self, shards, present, stride, n, want=None, status=None, shard_len=None,
                    allow_unrecoverable=True):
        kind, st = self._stream(shards)
        allow = (E_UNRECOVERABLE,) if allow_unrecoverable else ()
        return self._check(self._L.garage_ec_reconstruct(self._h, _ptr(shards), _ptr(present), _ptr(want),
                                                         _ptr(status), _ptr(shard_len), stride, n, kind, st),
                           allow)

    def reconstruct_stripes(self, stripes, present, stride, want=None, status=None, shard_len=None):
        """gather form: `stripes` is a list of numpy arrays, one (k+m)*stride buffer per stripe"""
        n = len(stripes)
        ptrs = (C.c_void_p * n)(*[a.ctypes.data for a in stripes])
        return self._check(self._L.garage_ec_reconstruct_stripes(self._h, C.cast(ptrs, C.c_void_p), _ptr(present),
                                                                 _ptr(want), _ptr(status), _ptr(shard_len), stride, n),
                           (E_UNRECOVERABLE,))

    def reconstruct_segments(self, shards, seg_present, stride, n, want=None, status=None, shard_len=None):
        """garage_ec_reconstruct_segments: seg_present holds one byte per shard, bit g = adler8 segment g is valid.
        `shards` a list of numpy arrays: the gather form (one (k+m)*stride buffer per stripe)"""
        if isinstance(shards, list):
            ptrs = (C.c_void_p * n)(*[a.ctypes.data for a in shards])
            return self._check(self._L.garage_ec_reconstruct_segments_stripes(
                self._h, C.cast(ptrs, C.c_void_p), _ptr(seg_present), _ptr(want), _ptr(status), _ptr(shard_len),
                stride, n), (E_UNRECOVERABLE,))
        kind, st = self._stream(shards)
        return self._check(self._L.garage_ec_reconstruct_segments(self._h, _ptr(shards), _ptr(seg_present), _ptr(want),
                                                                  _ptr(status), _ptr(shard_len), stride, n, kind, st),
                           (E_UNRECOVERABLE,))

    def verify(self, shards, mismatch, stride, n, shard_len=None):
        kind, st = self._stream(shards)
        return self._check(self._L.garage_ec_verify(self._h, _ptr(shards), _ptr(mismatch), _ptr(shard_len),
                                                    stride, n, kind, st))

    def deep_check(self, shards, block_len, hashes, hash_bad, mismatch, stride, n):
        """garage_ec_deep_check: hash_bad[s] = the block read from the data shards does not hash to hashes[s];
        mismatch[s] = garage_ec_verify's parity bits with the code's shard length"""
        kind, st = self._stream(shards)
        return self._check(self._L.garage_ec_deep_check(self._h, _ptr(shards), _ptr(block_len), _ptr(hashes),
                                                        _ptr(hash_bad), _ptr(mismatch), stride, n, kind, st))

    # -- per-shard integrity (blake2sum of every shard)
    def shard_sums(self, shards, sums_out, stride, n, per_stripe, shard_len=None):
        kind, st = self._stream(shards)
        return self._check(self._L.garage_ec_shard_sums(self._h, _ptr(shards), _ptr(shard_len), stride, n,
                                                        per_stripe, _ptr(sums_out), kind, st))

    def check_sums(self, shards, expect, bad_out, stride, n, per_stripe, shard_len=None):
        kind, st = self._stream(shards)
        return self._check(self._L.garage_ec_check_sums(self._h, _ptr(shards), _ptr(expect), _ptr(shard_len),
                                                        stride, n, per_stripe, _ptr(bad_out), kind, st))

    def scrub_repair(self, shards, expect_sums, bad_out, stride, n, status=None, shard_len=None):
        """config-5 sweep: hash every shard, rebuild the corrupt ones in place."""
        kind, st = self._stream(shards)
        return self._check(self._L.garage_ec_scrub_repair(self._h, _ptr(shards), _ptr(expect_sums), _ptr(bad_out),
                                                          _ptr(status), _ptr(shard_len), stride, n, kind, st),
                           (E_UNRECOVERABLE,))

    # -- block-level host API
    def encode_blocks(self, blocks, parity_out, stride, sums_out=None):
        """blocks: list of 1-D uint8 numpy arrays; parity_out: numpy (n*m*stride);
        sums_out: optional numpy n*(k+m)*32 for the per-shard blake2sums."""
        n = len(blocks)
        ptrs = (C.c_void_p * n)(*[b.ctypes.data for b in blocks])
        lens = np.array([b.size for b in blocks], dtype=np.uint32)
        return self._check(self._L.garage_ec_encode_blocks_with_sums(self._h, C.cast(ptrs, C.c_void_p), _ptr(lens),
                                                                     n, _ptr(parity_out), _ptr(sums_out), stride))

    def decode_blocks(self, shards, present, block_lens, stride, blocks_out, status=None):
        n = len(blocks_out)
        ptrs = (C.c_void_p * n)(*[b.ctypes.data for b in blocks_out])
        lens = np.ascontiguousarray(block_lens, dtype=np.uint32)
        return self._check(self._L.garage_ec_decode_blocks(self._h, _ptr(shards), _ptr(present), _ptr(lens), n,
                                                           stride, C.cast(ptrs, C.c_void_p), _ptr(status)),
                           (E_UNRECOVERABLE,))

    # -- code conversion
    def transcode(self, src, src_shards, block_lens, src_stride, dst_shards, dst_stride, n, src_present=None,
                  dst_sums=None, status=None):
        """garage_ec_transcode: rewrite n blocks stored under `src` (a GarageEc, or None for whole blocks
        `src_stride` apart) as this context's code; returns 0 or E_UNRECOVERABLE (HOST mode)"""
        kind, st = self._stream(src_shards, dst_shards)
        return self._check(self._L.garage_ec_transcode(self._h, src._h if src is not None else None, _ptr(src_shards),
                                                       _ptr(src_present), _ptr(block_lens), src_stride, _ptr(dst_shards),
                                                       dst_stride, _ptr(dst_sums), _ptr(status), n, kind, st),
                           (E_UNRECOVERABLE,))

    # -- SSE-C (AES-256-GCM STREAM chunks, DESIGN.md 2.6)
    def seal(self, plain, plain_stride, plain_len, keys, nonces, shards, stride, hashes, sums=None, n=None,
             crc_kind=None, crcs=None):
        """garage_ec_seal of n = len(plain_len) blocks; keys = nonces = None stores them as plaintext.  crc_kind (one
        uint8 CRC_* per block) and crcs (uint32 per block): also the plaintext checksums (garage_ec_seal_crc)"""
        kind, st = self._stream(plain, shards)
        n = len(plain_len) if n is None else n
        return self._check(self._L.garage_ec_seal_crc(self._h, _ptr(plain), plain_stride, _ptr(plain_len), _ptr(keys),
                                                      _ptr(nonces), _ptr(shards), stride, _ptr(hashes), _ptr(sums),
                                                      _ptr(crc_kind), _ptr(crcs), n, kind, st))

    def seal_blocks(self, blocks, keys, nonces, shards, stride, hashes, sums=None, crc_kind=None, crcs=None):
        """HOST gather form: `blocks` is a list of 1-D uint8 numpy arrays"""
        n = len(blocks)
        ptrs = (C.c_void_p * n)(*[b.ctypes.data if b.size else None for b in blocks])
        lens = np.array([b.size for b in blocks], dtype=np.uint32)
        return self._check(self._L.garage_ec_seal_blocks_crc(self._h, C.cast(ptrs, C.c_void_p), _ptr(lens), _ptr(keys),
                                                             _ptr(nonces), _ptr(shards), stride, _ptr(hashes),
                                                             _ptr(sums), _ptr(crc_kind), _ptr(crcs), n))

    def open(self, shards, present, sealed_len, hashes, keys, plain, plain_stride, plain_len_out, hash_bad, status,
             stride, n=None):
        """garage_ec_open; returns 0, E_UNRECOVERABLE or E_AUTH (HOST mode)"""
        kind, st = self._stream(shards)
        n = len(sealed_len) if n is None else n
        return self._check(self._L.garage_ec_open(self._h, _ptr(shards), _ptr(present), _ptr(sealed_len), _ptr(hashes),
                                                  _ptr(keys), _ptr(plain), plain_stride, _ptr(plain_len_out),
                                                  _ptr(hash_bad), _ptr(status), stride, n, kind, st),
                           (E_UNRECOVERABLE, E_AUTH))

    def open_stripes(self, stripes, present, sealed_len, hashes, keys, plains, plain_len_out, hash_bad, status, stride):
        """HOST gather form: `stripes` / `plains` are lists of numpy arrays, one per block"""
        n = len(stripes)
        sp = (C.c_void_p * n)(*[a.ctypes.data for a in stripes])
        op = (C.c_void_p * n)(*[a.ctypes.data for a in plains])
        return self._check(self._L.garage_ec_open_stripes(self._h, C.cast(sp, C.c_void_p), _ptr(present),
                                                          _ptr(sealed_len), _ptr(hashes), _ptr(keys),
                                                          C.cast(op, C.c_void_p), _ptr(plain_len_out), _ptr(hash_bad),
                                                          _ptr(status), stride, n),
                           (E_UNRECOVERABLE, E_AUTH))

    # -- SSE-C ranged opens (DESIGN.md 2.7)
    @staticmethod
    def sealed_range(sealed_len, offset, length):
        """garage_ec_sealed_range (host only, no context): (span_off, span_len, c0, n_chunks) of plaintext bytes
        [offset, offset + length) of a block sealed to sealed_len bytes; raises EcError (E_AUTH / E_INVALID)"""
        v = [C.c_uint32(0) for _ in range(4)]
        rc = load_library().garage_ec_sealed_range(sealed_len, offset, length, *[C.byref(x) for x in v])
        if rc:
            raise EcError(rc, "sealed_range")
        return tuple(x.value for x in v)

    def open_range_plan(self, present, sealed_len, offset, length):
        """(runs [(shard, offset, len)], needs_gpu) for the prefix and span of a plaintext range of one sealed block,
        or (None, needs_gpu) if an absent touched data shard cannot be rebuilt"""
        pr = np.ascontiguousarray(present, dtype=np.uint8)
        assert pr.shape == (self.k + self.m,)
        cap = (self.k + self.m) * 1024
        out = np.zeros(cap * 3, dtype=np.uint32)
        n, g = C.c_size_t(0), C.c_int(0)
        rc = self._check(self._L.garage_ec_open_range_plan(self._h, _ptr(pr), sealed_len, offset, length, _ptr(out),
                                                           cap, C.byref(n), C.byref(g)), (E_UNRECOVERABLE,))
        if rc == E_UNRECOVERABLE:
            return None, g.value
        return [tuple(int(v) for v in out[3 * i:3 * i + 3]) for i in range(n.value)], g.value

    def open_range(self, shards, present, sealed_len, keys, offset, length, stride, out, out_stride, status):
        """garage_ec_open_range of n = len(sealed_len) requests; returns 0, E_UNRECOVERABLE or E_AUTH (HOST mode)"""
        kind, st = self._stream(shards)
        return self._check(self._L.garage_ec_open_range(self._h, _ptr(shards), _ptr(present), _ptr(sealed_len),
                                                        _ptr(keys), _ptr(offset), _ptr(length), stride, _ptr(out),
                                                        out_stride, _ptr(status), len(sealed_len), kind, st),
                           (E_UNRECOVERABLE, E_AUTH))

    def open_range_stripes(self, stripes, present, sealed_len, keys, offset, length, stride, outs, status):
        """HOST gather form: `stripes` / `outs` are lists of numpy arrays, one per request"""
        n = len(stripes)
        sp = (C.c_void_p * n)(*[a.ctypes.data for a in stripes])
        op = (C.c_void_p * n)(*[a.ctypes.data for a in outs])
        return self._check(self._L.garage_ec_open_range_stripes(self._h, C.cast(sp, C.c_void_p), _ptr(present),
                                                                _ptr(sealed_len), _ptr(keys), _ptr(offset),
                                                                _ptr(length), stride, C.cast(op, C.c_void_p),
                                                                _ptr(status), n),
                           (E_UNRECOVERABLE, E_AUTH))

    # -- SSE-C copies with re-encryption (DESIGN.md 2.8)
    def reseal(self, src_shards, src_present, src_len, src_hashes, src_keys, pieces, piece_start, dst_keys, dst_nonces,
               dst_shards, dst_hashes, dst_len_out, src_hash_bad, src_status, status, stride, dst_sums=None,
               n_src=None, n_dst=None, crc_kind=None, crcs=None):
        """garage_ec_reseal: destination d = the pieces [piece_start[d], piece_start[d+1]) of `pieces` ((src, offset,
        len) uint32 triples), sealed under dst_keys / dst_nonces; src_keys = None: plaintext sources.  crc_kind / crcs
        per destination: also the checksums of their plaintext (garage_ec_reseal_crc).  Returns 0, E_UNRECOVERABLE or
        E_AUTH (HOST mode)"""
        kind, st = self._stream(src_shards, dst_shards)
        n_src = len(src_len) if n_src is None else n_src
        n_dst = len(piece_start) - 1 if n_dst is None else n_dst
        return self._check(self._L.garage_ec_reseal_crc(self._h, _ptr(src_shards), _ptr(src_present), _ptr(src_len),
                                                        _ptr(src_hashes), _ptr(src_keys), n_src, _ptr(pieces),
                                                        _ptr(piece_start), _ptr(dst_keys), _ptr(dst_nonces),
                                                        _ptr(dst_shards), _ptr(dst_hashes), _ptr(dst_sums),
                                                        _ptr(dst_len_out), _ptr(src_hash_bad), _ptr(src_status),
                                                        _ptr(status), _ptr(crc_kind), _ptr(crcs), stride, n_dst, kind,
                                                        st),
                           (E_UNRECOVERABLE, E_AUTH))

    def reseal_stripes(self, src_stripes, src_present, src_len, src_hashes, src_keys, pieces, piece_start, dst_keys,
                       dst_nonces, dst_shards, dst_hashes, dst_len_out, src_hash_bad, src_status, status, stride,
                       dst_sums=None, crc_kind=None, crcs=None):
        """HOST gather form: `src_stripes` is a list of numpy arrays, one (k+m)*stride stripe per source"""
        n = len(src_stripes)
        sp = (C.c_void_p * max(n, 1))(*[a.ctypes.data for a in src_stripes])
        return self._check(self._L.garage_ec_reseal_stripes_crc(self._h, C.cast(sp, C.c_void_p), _ptr(src_present),
                                                                _ptr(src_len), _ptr(src_hashes), _ptr(src_keys), n,
                                                                _ptr(pieces), _ptr(piece_start), _ptr(dst_keys),
                                                                _ptr(dst_nonces), _ptr(dst_shards), _ptr(dst_hashes),
                                                                _ptr(dst_sums), _ptr(dst_len_out), _ptr(src_hash_bad),
                                                                _ptr(src_status), _ptr(status), _ptr(crc_kind),
                                                                _ptr(crcs), stride, len(piece_start) - 1),
                           (E_UNRECOVERABLE, E_AUTH))

    # -- harness utilities
    def fill_random(self, dst, nbytes, seed, offset=0):
        import torch

        st = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
        return self._check(self._L.garage_ec_fill_random(self._h, _ptr(dst), nbytes, seed, offset, st))

    def host_alloc(self, nbytes, write_combined=False):
        """pinned host buffer as a numpy uint8 array (freed with host_free)."""
        p = C.c_void_p()
        fn = self._L.garage_ec_host_alloc_wc if write_combined else self._L.garage_ec_host_alloc
        self._check(fn(self._h, C.byref(p), nbytes))
        arr = np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(nbytes,))
        return arr, p

    def host_free(self, p):
        self._L.garage_ec_host_free(self._h, p)

    def numa_info(self):
        """(NUMA node of the GPU, node the last host_alloc landed on); -1 = unknown"""
        a, b = C.c_int(-1), C.c_int(-1)
        self._check(self._L.garage_ec_numa_info(self._h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def bind_thread(self):
        """pin the calling thread to the CPUs of the GPU's NUMA node; True if bound"""
        return self._L.garage_ec_bind_thread(self._h) == 0

    def set_wait_mode(self, blocking):
        """HOST-mode calls wait by sleeping on an event (True) instead of spinning in the driver (False, default)"""
        self._check(self._L.garage_ec_set_wait_mode(self._h, 1 if blocking else 0))

    def set_sum_kind(self, kind):
        self._check(self._L.garage_ec_set_sum_kind(self._h, kind))

    def debug_fail_after(self, n_calls):
        self._check(self._L.garage_ec_debug_fail_after(self._h, n_calls))
