"""ctypes binding of include/garage_placement.h (SURVEY.md section 8 row f4: placement and quorums for
erasure-coded blocks).  Pure host code inside libgarage_block.so; no GPU needed.

Reference surface mirrored: LayoutVersion::nodes_of / partition_of (src/rpc/layout/version.rs:101-137),
try_write_many_sets + QuorumSetResultTracker (src/rpc/rpc_helper.rs:432-538, 664-760),
block_read_nodes_of + request_order (src/rpc/rpc_helper.rs:570-660), write_quorum
(src/rpc/replication_mode.rs:52-60)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import block_manager as _bm

NB_PARTITIONS = 256
OK, E_INVALID, E_INFEASIBLE, E_NOMEM, E_DUPLICATE, E_GATEWAY, E_ZONES, E_ZONE_LOAD, E_CAPACITY = 0, -1, -2, -3, -4, -5, -6, -7, -8
CONSISTENT, DEGRADED, DANGEROUS = 0, 1, 2
QUORUM_PENDING, QUORUM_OK, QUORUM_FAILED = 0, 1, -1

PLACEMENT_SYMBOLS = [
    "garage_layout_compute", "garage_layout_from_ring", "garage_layout_free", "garage_layout_partition_of",
    "garage_layout_nodes_of", "garage_layout_ring", "garage_layout_replication_factor", "garage_layout_version",
    "garage_layout_partition_size", "garage_layout_check", "garage_layout_transition", "garage_ec_write_quorum",
    "garage_ec_read_quorum", "garage_layout_write_plan", "garage_quorum_tracker_new", "garage_quorum_tracker_register",
    "garage_quorum_tracker_state", "garage_quorum_tracker_free", "garage_layout_read_plan",
]


class LayoutStats(C.Structure):
    _fields_ = [("min_zones_per_partition", C.c_int32), ("max_shards_per_zone", C.c_int32),
                ("min_partitions_per_node", C.c_int32), ("max_partitions_per_node", C.c_int32),
                ("storage_nodes", C.c_int32), ("zones", C.c_int32)]


class ShardRequest(C.Structure):
    _fields_ = [("node", C.c_int32), ("index", C.c_int32), ("set_mask", C.c_uint32)]


class ShardSource(C.Structure):
    _fields_ = [("node", C.c_int32), ("index", C.c_int32), ("version", C.c_int32)]


class PlacementError(RuntimeError):
    def __init__(self, code, what):
        super().__init__("%s: code %d" % (what, code))
        self.code = code


_bound = False


def _lib():
    global _bound
    L = _bm.load_library()
    if not _bound:
        vp, i32, u64 = C.c_void_p, C.c_int, C.c_uint64
        L.garage_layout_compute.argtypes = [C.POINTER(vp), u64, i32, vp, vp, i32, i32, i32, vp]
        L.garage_layout_from_ring.argtypes = [C.POINTER(vp), u64, i32, vp, vp, i32, vp]
        L.garage_layout_free.argtypes = [vp]
        L.garage_layout_free.restype = None
        L.garage_layout_partition_of.argtypes = [vp]
        L.garage_layout_nodes_of.argtypes = [vp, vp, vp]
        L.garage_layout_ring.argtypes = [vp, vp]
        L.garage_layout_replication_factor.argtypes = [vp]
        L.garage_layout_version.argtypes = [vp]
        L.garage_layout_version.restype = u64
        L.garage_layout_partition_size.argtypes = [vp]
        L.garage_layout_partition_size.restype = u64
        L.garage_layout_check.argtypes = [vp, i32, i32, C.POINTER(LayoutStats)]
        L.garage_layout_transition.argtypes = [vp, vp, i32, vp, vp, vp]
        L.garage_ec_write_quorum.argtypes = [i32, i32, i32]
        L.garage_ec_read_quorum.argtypes = [i32, i32, i32]
        L.garage_layout_write_plan.argtypes = [vp, i32, vp, C.POINTER(ShardRequest), i32]
        L.garage_quorum_tracker_new.argtypes = [C.POINTER(vp), C.POINTER(ShardRequest), i32, i32, i32]
        L.garage_quorum_tracker_register.argtypes = [vp, i32, i32]
        L.garage_quorum_tracker_state.argtypes = [vp]
        L.garage_quorum_tracker_free.argtypes = [vp]
        L.garage_quorum_tracker_free.restype = None
        L.garage_layout_read_plan.argtypes = [vp, i32, vp, i32, vp, i32, i32, vp, C.POINTER(ShardSource), i32]
        _bound = True
    return L


def _hash_ptr(h):
    b = bytes(h)
    assert len(b) == 32
    return (C.c_uint8 * 32).from_buffer_copy(b)


def partition_of(hash32) -> int:
    return _lib().garage_layout_partition_of(_hash_ptr(hash32))


def write_quorum(k, m, mode=CONSISTENT) -> int:
    return _lib().garage_ec_write_quorum(k, m, mode)


def read_quorum(k, m, mode=CONSISTENT) -> int:
    return _lib().garage_ec_read_quorum(k, m, mode)


class Layout:
    """one layout version: 256 partitions x replication_factor (= k+m) nodes, shard i on the i-th node"""

    def __init__(self, handle, zones, capacities):
        self._h = handle
        self.zones = list(zones)
        self.capacities = list(capacities)

    @classmethod
    def compute(cls, zones, capacities, replication_factor, zone_redundancy=0, max_per_zone=0, previous=None, version=1):
        z = np.asarray(zones, dtype=np.int32)
        c = np.asarray(capacities, dtype=np.uint64)
        assert z.size == c.size
        h = C.c_void_p()
        rc = _lib().garage_layout_compute(C.byref(h), version, z.size, z.ctypes.data, c.ctypes.data, replication_factor,
                                          zone_redundancy, max_per_zone, previous._h if previous else None)
        if rc:
            raise PlacementError(rc, "garage_layout_compute")
        return cls(h, z, c)

    @classmethod
    def from_ring(cls, zones, capacities, replication_factor, ring, version=1):
        z = np.asarray(zones, dtype=np.int32)
        c = np.asarray(capacities, dtype=np.uint64)
        r = np.ascontiguousarray(ring, dtype=np.uint8).reshape(-1)
        assert r.size == NB_PARTITIONS * replication_factor
        h = C.c_void_p()
        rc = _lib().garage_layout_from_ring(C.byref(h), version, z.size, z.ctypes.data, c.ctypes.data, replication_factor,
                                            r.ctypes.data)
        if rc:
            raise PlacementError(rc, "garage_layout_from_ring")
        return cls(h, z, c)

    def close(self):
        if self._h:
            _lib().garage_layout_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def replication_factor(self):
        return _lib().garage_layout_replication_factor(self._h)

    @property
    def version(self):
        return _lib().garage_layout_version(self._h)

    @property
    def partition_size(self):
        return _lib().garage_layout_partition_size(self._h)

    def ring(self):
        rf = self.replication_factor
        out = np.zeros(NB_PARTITIONS * rf, dtype=np.uint8)
        _lib().garage_layout_ring(self._h, out.ctypes.data)
        return out.reshape(NB_PARTITIONS, rf)

    def nodes_of(self, hash32):
        out = np.zeros(self.replication_factor, dtype=np.int32)
        rc = _lib().garage_layout_nodes_of(self._h, _hash_ptr(hash32), out.ctypes.data)
        if rc:
            raise PlacementError(rc, "garage_layout_nodes_of")
        return out.tolist()

    def check(self, zone_redundancy=0, max_per_zone=0):
        st = LayoutStats()
        rc = _lib().garage_layout_check(self._h, zone_redundancy, max_per_zone, C.byref(st))
        return rc, {n: getattr(st, n) for n, _ in LayoutStats._fields_}

    def transition_to(self, new, partition=-1):
        """partition >= 0: list of (index, from_node, to_node); partition < 0: number of shards that move overall"""
        rf = self.replication_factor
        idx, a, b = (np.zeros(rf, dtype=np.int32) for _ in range(3))
        n = _lib().garage_layout_transition(self._h, new._h, partition, idx.ctypes.data, a.ctypes.data, b.ctypes.data)
        if n < 0:
            raise PlacementError(n, "garage_layout_transition")
        if partition < 0:
            return n
        return [(int(idx[j]), int(a[j]), int(b[j])) for j in range(n)]


def _handles(layouts):
    return (C.c_void_p * max(len(layouts), 1))(*[l._h for l in layouts])


def write_plan(versions, hash32):
    """unique (node, index) requests of a PUT over the active versions (oldest first) -> list of (node, index, set_mask)"""
    cap = sum(v.replication_factor for v in versions)
    out = (ShardRequest * cap)()
    n = _lib().garage_layout_write_plan(_handles(versions), len(versions), _hash_ptr(hash32), out, cap)
    if n < 0:
        raise PlacementError(n, "garage_layout_write_plan")
    return [(out[i].node, out[i].index, out[i].set_mask) for i in range(n)]


class QuorumTracker:
    def __init__(self, requests, n_sets, quorum):
        arr = (ShardRequest * len(requests))(*[ShardRequest(n, i, m) for n, i, m in requests])
        self._h = C.c_void_p()
        rc = _lib().garage_quorum_tracker_new(C.byref(self._h), arr, len(requests), n_sets, quorum)
        if rc:
            raise PlacementError(rc, "garage_quorum_tracker_new")

    def register(self, request, ok) -> int:
        return _lib().garage_quorum_tracker_register(self._h, request, 1 if ok else 0)

    @property
    def state(self) -> int:
        return _lib().garage_quorum_tracker_state(self._h)

    def close(self):
        if self._h:
            _lib().garage_quorum_tracker_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def read_plan(active, hash32, k, our_node=-1, ping_us=None, old=()):
    """ordered (node, index, version) sources of a GET: see garage_layout_read_plan"""
    cap = sum(v.replication_factor for v in list(active) + list(old))
    out = (ShardSource * cap)()
    ping = None
    if ping_us is not None:
        ping = np.asarray(ping_us, dtype=np.uint32)
    n = _lib().garage_layout_read_plan(_handles(active), len(active), _handles(old) if old else None, len(old),
                                       _hash_ptr(hash32), k, our_node, ping.ctypes.data if ping is not None else None,
                                       out, cap)
    if n < 0:
        raise PlacementError(n, "garage_layout_read_plan")
    return [(out[i].node, out[i].index, out[i].version) for i in range(n)]


# ---- drive layout (DESIGN.md section 5.7): a node's files over several data directories ----------
DRIVE_NPART = 1024
DRIVE_MAX_DIRS = 16
DRIVE_SYMBOLS = [
    "garage_drive_partition_of", "garage_drive_layout_init", "garage_drive_layout_update",
    "garage_drive_layout_drop_secondaries", "garage_drive_layout_n_dirs", "garage_drive_layout_primary",
    "garage_drive_layout_secondaries", "garage_drive_layout_serialize", "garage_drive_layout_deserialize",
    "garage_drive_layout_free",
]
_drive_bound = False


def _dlib():
    global _drive_bound
    L = _lib()
    if not _drive_bound:
        vp, i32 = C.c_void_p, C.c_int
        L.garage_drive_partition_of.argtypes = [vp]
        L.garage_drive_layout_init.argtypes = [C.POINTER(vp), i32, vp, vp]
        L.garage_drive_layout_update.argtypes = [C.POINTER(vp), vp, vp, i32, vp, vp]
        L.garage_drive_layout_drop_secondaries.argtypes = [C.POINTER(vp), vp]
        L.garage_drive_layout_n_dirs.argtypes = [vp]
        L.garage_drive_layout_primary.argtypes = [vp, i32]
        L.garage_drive_layout_secondaries.argtypes = [vp, i32, vp, i32]
        L.garage_drive_layout_serialize.argtypes = [vp, vp, C.c_size_t]
        L.garage_drive_layout_serialize.restype = C.c_size_t
        L.garage_drive_layout_deserialize.argtypes = [C.POINTER(vp), vp, C.c_size_t]
        L.garage_drive_layout_free.argtypes = [vp]
        L.garage_drive_layout_free.restype = None
        _drive_bound = True
    return L


def drive_partition_of(hash32) -> int:
    return _dlib().garage_drive_partition_of(_hash_ptr(hash32))


class DriveLayout:
    """a node's drive layout: per partition a primary directory and ordered secondary directories.  capacity 0 marks
    a read-only directory; non_empty[i]: directory i holds a garage-marker or a hex-named subdirectory."""

    def __init__(self, handle):
        self._h = handle

    @staticmethod
    def _arrays(capacity, non_empty):
        c = np.ascontiguousarray(capacity, dtype=np.uint64)
        ne = np.ascontiguousarray(non_empty if non_empty is not None else np.zeros(c.size), dtype=np.uint8)
        return c, ne

    @classmethod
    def init(cls, capacity, non_empty=None):
        c, ne = cls._arrays(capacity, non_empty)
        h = C.c_void_p()
        rc = _dlib().garage_drive_layout_init(C.byref(h), c.size, c.ctypes.data, ne.ctypes.data)
        if rc:
            raise PlacementError(rc, "garage_drive_layout_init")
        return cls(h)

    def update(self, prev_index, capacity, non_empty=None):
        c, ne = self._arrays(capacity, non_empty)
        pi = np.ascontiguousarray(prev_index, dtype=np.int32)
        assert pi.size == c.size
        h = C.c_void_p()
        rc = _dlib().garage_drive_layout_update(C.byref(h), self._h, pi.ctypes.data, c.size, c.ctypes.data, ne.ctypes.data)
        if rc:
            raise PlacementError(rc, "garage_drive_layout_update")
        return DriveLayout(h)

    def drop_secondaries(self):
        h = C.c_void_p()
        rc = _dlib().garage_drive_layout_drop_secondaries(C.byref(h), self._h)
        if rc:
            raise PlacementError(rc, "garage_drive_layout_drop_secondaries")
        return DriveLayout(h)

    @property
    def n_dirs(self):
        return _dlib().garage_drive_layout_n_dirs(self._h)

    def primary(self, part):
        return _dlib().garage_drive_layout_primary(self._h, part)

    def secondaries(self, part):
        out = (C.c_uint8 * DRIVE_MAX_DIRS)()
        n = _dlib().garage_drive_layout_secondaries(self._h, part, out, DRIVE_MAX_DIRS)
        return list(out[:n])

    def primaries(self):
        return [self.primary(p) for p in range(DRIVE_NPART)]

    def all_secondaries(self):
        return [self.secondaries(p) for p in range(DRIVE_NPART)]

    def serialize(self) -> bytes:
        n = _dlib().garage_drive_layout_serialize(self._h, None, 0)
        buf = (C.c_uint8 * n)()
        _dlib().garage_drive_layout_serialize(self._h, buf, n)
        return bytes(buf)

    @classmethod
    def deserialize(cls, data: bytes):
        b = (C.c_uint8 * max(1, len(data))).from_buffer_copy(data or b"\0")
        h = C.c_void_p()
        rc = _dlib().garage_drive_layout_deserialize(C.byref(h), b, len(data))
        if rc:
            raise PlacementError(rc, "garage_drive_layout_deserialize")
        return cls(h)

    def __del__(self):
        try:
            if self._h:
                _dlib().garage_drive_layout_free(self._h)
                self._h = None
        except Exception:
            pass
