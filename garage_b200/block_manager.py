"""ctypes view of libgarage_block.so -- the C++ host-side mirror of Garage's BlockManager for
the erasure-coded path (include/garage_block_manager.h).  Harness only; the logic is C++."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _build

OK = 0
E_CORRUPT_DATA, E_MISSING_BLOCK, E_MESSAGE, E_QUORUM = -10, -11, -12, -13

SYMBOLS = [
    "garage_bm_default_config", "garage_bm_create", "garage_bm_destroy", "garage_bm_blake2sum",
    "garage_bm_rpc_put_block", "garage_bm_rpc_get_block", "garage_bm_resync_block", "garage_bm_resync_all",
    "garage_bm_repair_enqueue_missing", "garage_bm_scrub", "garage_bm_set_node_up", "garage_bm_corrupt_shard",
    "garage_bm_drop_shard", "garage_bm_node_shard_index", "garage_bm_storage_nodes_of", "garage_bm_get_metrics",
    "garage_bm_block_incref", "garage_bm_block_decref", "garage_bm_get_block_rc", "garage_bm_scrub_step",
    "garage_bm_bench", "garage_bm_corrupt_shard_header", "garage_bm_plant_stale_shard", "garage_bm_set_node_readonly",
    "garage_bm_convert_step", "garage_bm_debug_convert_stop_after", "garage_bm_apply_layout", "garage_bm_layout_sync_step",
    "garage_bm_layout_versions", "garage_bm_deep_scrub_step", "garage_bm_rpc_get_block_range",
    "garage_bm_get_range_metrics", "garage_bm_stripe_repair_step", "garage_bm_get_stripe_repair_metrics",
    "garage_bm_get_salvage_metrics", "garage_bm_get_segment_repair_metrics",
    "garage_bm_set_data_dirs", "garage_bm_rebalance_step", "garage_bm_get_drive_metrics", "garage_bm_create_with_drives",
    "garage_bm_resync_step", "garage_bm_list_resync_errors", "garage_bm_resync_retry_now", "garage_bm_block_info",
    "garage_bm_debug_set_clock_ms", "garage_bm_get_resync_metrics",
    "garage_bm_rpc_put_block_sealed", "garage_bm_rpc_get_block_opened", "garage_bm_get_sealed_metrics",
    "garage_bm_rpc_get_block_range_opened", "garage_bm_get_sealed_range_metrics",
    "garage_bm_rpc_put_block_resealed", "garage_bm_get_reseal_metrics",
    "garage_bm_rpc_put_block_sealed_crc", "garage_bm_rpc_put_block_resealed_crc",
    "garage_bm_create_on_devices", "garage_bm_get_device_metrics",
]
MAX_DEVICES = 16
MAX_PIECES = 64
CRC_NONE, CRC32, CRC32C = 0, 1, 2  # checksum kinds of the _crc writes (DESIGN.md 2.9)
SUM_BLAKE2, SUM_ADLER8 = 0, 1


class Code(C.Structure):
    """garage_bm_code: a code the store may still hold shards of"""
    _fields_ = [("k", C.c_int), ("m", C.c_int), ("local_groups", C.c_int), ("piggyback", C.c_int), ("clay", C.c_int)]


class LayoutSpec(C.Structure):
    """garage_bm_layout_spec: one layout version over the manager's n_nodes node stores"""
    _fields_ = [("zone", C.POINTER(C.c_int32)), ("capacity", C.POINTER(C.c_uint64)), ("zone_redundancy", C.c_int),
                ("max_per_zone", C.c_int)]


def _layout_spec(zone, capacity, zone_redundancy=0, max_per_zone=0):
    """-> (LayoutSpec, the arrays it points into: keep them alive while the spec is used)"""
    z = (C.c_int32 * max(1, len(zone)))(*map(int, zone))
    c = (C.c_uint64 * max(1, len(capacity)))(*map(int, capacity))
    return LayoutSpec(C.cast(z, C.POINTER(C.c_int32)), C.cast(c, C.POINTER(C.c_uint64)), zone_redundancy, max_per_zone), (z, c)


class DataDir(C.Structure):
    """garage_bm_data_dir: one drive of a node, path relative to the node directory"""
    _fields_ = [("path", C.c_char_p), ("capacity", C.c_uint64), ("read_only", C.c_int)]


def _data_dirs(dirs):
    """(path, capacity) / (path, capacity, read_only) tuples or dicts -> (DataDir array or None, n)"""
    rows = []
    for d in dirs:
        if isinstance(d, dict):
            rows.append((d["path"], d.get("capacity", 0), d.get("read_only", False)))
        else:
            rows.append((d[0], d[1], d[2] if len(d) > 2 else False))
    arr = (DataDir * max(1, len(rows)))(*[DataDir(p.encode() if isinstance(p, str) else p, int(c), int(bool(ro)))
                                          for p, c, ro in rows])
    return arr, len(rows)


class Config(C.Structure):
    _fields_ = [("data_shards", C.c_int), ("parity_shards", C.c_int), ("cuda_device", C.c_int),
                ("n_nodes", C.c_int), ("block_size", C.c_uint32), ("block_ram_buffer_max", C.c_uint64),
                ("batch_max_blocks", C.c_uint32), ("batch_linger_us", C.c_uint32), ("data_dir", C.c_char_p),
                ("shard_sum_kind", C.c_int), ("verify_content_hash", C.c_int), ("data_fsync", C.c_int),
                ("block_gc_delay_ms", C.c_uint32), ("local_groups", C.c_int), ("piggyback", C.c_int),
                ("previous_codes", C.POINTER(Code)), ("n_previous_codes", C.c_int), ("legacy_replicas", C.c_int),
                ("layout", C.POINTER(LayoutSpec)), ("clay", C.c_int), ("clay_layout", C.c_int)]


class Metrics(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in (
        "bytes_written", "bytes_read", "corruption_counter", "resync_counter", "resync_error_counter",
        "resync_recv_counter", "delete_counter", "put_calls", "put_batches", "reconstruct_calls",
        "reconstruct_batches", "scrub_shards_checked", "scrub_corruptions", "resync_queue_length",
        "encode_call_us", "reconstruct_call_us", "corrupt_data_errors", "write_errors", "resync_shards_read", "resync_bytes_read",
        "convert_blocks", "convert_bytes_read", "convert_bytes_written", "convert_errors", "convert_call_us", "legacy_gets",
        "legacy_deleted", "layout_shards_copied", "layout_shards_rebuilt", "layout_bytes_read", "layout_bytes_written",
        "layout_deleted", "layout_sync_errors", "layout_version", "resync_bytes_fetched", "deep_scrub_blocks",
        "deep_scrub_skipped", "deep_scrub_parity_bad", "deep_scrub_content_errors", "deep_check_call_us",
        "layout_bytes_fetched")]


class RangeMetrics(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("range_gets", "range_degraded", "range_bytes_read", "range_bytes_fetched")]


class DriveMetrics(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in (
        "rebalance_files_moved", "rebalance_bytes_moved", "rebalance_errors", "drive_marker_errors")]


class StripeRepairMetrics(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in (
        "stripe_repairs", "stripe_repair_shards", "stripe_repair_bytes_read", "stripe_repair_bytes_fetched",
        "stripe_repair_bytes_written", "stripe_repair_errors", "stripe_repair_call_us")]


class SalvageMetrics(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in (
        "salvage_attempts", "salvage_blocks", "salvage_failures", "salvage_units_rebuilt", "salvage_quarantined_segments",
        "salvage_bytes_read", "salvage_call_us")]


class SegmentRepairMetrics(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in (
        "repairs", "units_rebuilt", "bytes_read", "bytes_fetched", "fallbacks", "call_us")]


class ResyncMetrics(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in (
        "resync_error_entries", "resync_deferred", "resync_steps", "resync_retry_nows", "resync_failed_bytes_read")]


class SealedMetrics(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in (
        "sealed_puts", "sealed_batches", "opened_gets", "opened_auth_failures", "opened_fallbacks", "seal_call_us",
        "open_call_us")]


class SealedRangeMetrics(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in (
        "gets", "degraded_gets", "bytes_read", "bytes_fetched", "auth_failures", "fallbacks", "call_us",
        "open_range_call_us")]


class ResealMetrics(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in (
        "calls", "batches", "sources_gathered", "bytes_read", "auth_failures", "fallbacks", "call_us", "reseal_call_us")]


class DeviceMetrics(C.Structure):
    """garage_bm_device_metrics: one dispatcher group"""
    _fields_ = [("cuda_device", C.c_int), ("numa_node", C.c_int)] + [(n, C.c_uint64) for n in (
        "batches", "blocks", "bytes", "routed_local", "routed_remote")] + [("pool_numa_node", C.c_int)]


class Piece(C.Structure):
    """garage_bm_piece: plaintext bytes [offset, offset + len) of stored block `hash`"""
    _fields_ = [("hash", C.c_uint8 * 32), ("offset", C.c_uint32), ("len", C.c_uint32)]


class ResyncError(C.Structure):
    """garage_bm_resync_error: one entry of a node's resync error table"""
    _fields_ = [("node", C.c_int32), ("hash", C.c_uint8 * 32), ("rc", C.c_longlong), ("errors", C.c_uint64),
                ("last_try_ms", C.c_uint64), ("next_try_ms", C.c_uint64), ("last_status", C.c_int32)]


# garage_bm_block_status.state values
SHARD_VALID, SHARD_ABSENT, SHARD_DOWN, SHARD_BAD_HEADER, SHARD_BAD_TAG, SHARD_QUARANTINED, SHARD_PREVIOUS = range(7)
MAX_SHARDS = 40


class BlockStatus(C.Structure):
    """garage_bm_block_status: what garage_bm_block_info reports of one block"""
    _fields_ = [("rc", C.c_longlong), ("code", Code), ("block_len", C.c_uint32), ("n_shards", C.c_int32),
                ("node", C.c_int32 * MAX_SHARDS), ("state", C.c_int32 * MAX_SHARDS),
                ("resync_errors", C.c_uint64 * MAX_SHARDS), ("recoverable", C.c_int32),
                ("read_set", C.c_uint8 * MAX_SHARDS)]


_lib = None


def load_library():
    global _lib
    if _lib is None:
        _build.build_block_manager()
        L = C.CDLL(_build.BM_SO)
        vp, i32, sz = C.c_void_p, C.c_int, C.c_size_t
        L.garage_bm_default_config.argtypes = [C.POINTER(Config)]
        L.garage_bm_default_config.restype = None
        L.garage_bm_create.argtypes = [C.POINTER(vp), C.POINTER(Config)]
        L.garage_bm_destroy.argtypes = [vp]
        L.garage_bm_destroy.restype = None
        L.garage_bm_blake2sum.argtypes = [vp, sz, vp]
        L.garage_bm_blake2sum.restype = None
        L.garage_bm_rpc_put_block.argtypes = [vp, vp, vp, sz]
        L.garage_bm_rpc_get_block.argtypes = [vp, vp, vp, sz, C.POINTER(sz)]
        L.garage_bm_resync_block.argtypes = [vp, i32, vp]
        L.garage_bm_block_incref.argtypes = [vp, vp]
        L.garage_bm_block_decref.argtypes = [vp, vp]
        L.garage_bm_get_block_rc.argtypes = [vp, vp]
        L.garage_bm_get_block_rc.restype = C.c_longlong
        L.garage_bm_resync_all.argtypes = [vp, i32, i32, C.POINTER(C.c_uint64)]
        L.garage_bm_repair_enqueue_missing.argtypes = [vp, i32, C.POINTER(C.c_uint64)]
        L.garage_bm_scrub.argtypes = [vp, i32, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
        L.garage_bm_scrub_step.argtypes = [vp, i32, vp, sz, vp, C.POINTER(i32), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
        L.garage_bm_set_node_up.argtypes = [vp, i32, i32]
        L.garage_bm_corrupt_shard.argtypes = [vp, i32, vp, sz]
        L.garage_bm_drop_shard.argtypes = [vp, i32, vp]
        L.garage_bm_node_shard_index.argtypes = [vp, i32, vp]
        L.garage_bm_storage_nodes_of.argtypes = [vp, vp, C.POINTER(i32)]
        L.garage_bm_get_metrics.argtypes = [vp, C.POINTER(Metrics)]
        L.garage_bm_get_range_metrics.argtypes = [vp, C.POINTER(RangeMetrics)]
        L.garage_bm_get_range_metrics.restype = None
        L.garage_bm_rpc_get_block_range.argtypes = [vp, vp, C.c_uint32, C.c_uint32, vp, sz, C.POINTER(sz)]
        L.garage_bm_get_metrics.restype = None
        L.garage_bm_bench.argtypes = [vp, i32, i32, C.c_uint32, i32, C.c_uint64, C.POINTER(C.c_double), C.POINTER(C.c_uint64)]
        L.garage_bm_corrupt_shard_header.argtypes = [vp, i32, vp, i32]
        L.garage_bm_plant_stale_shard.argtypes = [vp, i32, vp]
        L.garage_bm_set_node_readonly.argtypes = [vp, i32, i32]
        L.garage_bm_convert_step.argtypes = [vp, i32, vp, sz, vp, C.POINTER(i32), C.POINTER(C.c_uint64)]
        L.garage_bm_debug_convert_stop_after.argtypes = [vp, C.c_long]
        L.garage_bm_apply_layout.argtypes = [vp, C.POINTER(LayoutSpec), C.POINTER(C.c_uint64)]
        L.garage_bm_layout_sync_step.argtypes = [vp, i32, vp, sz, vp, C.POINTER(i32), C.POINTER(C.c_uint64)]
        L.garage_bm_layout_versions.argtypes = [vp, C.POINTER(C.c_uint64), i32]
        L.garage_bm_deep_scrub_step.argtypes = [vp, i32, vp, sz, vp, C.POINTER(i32), C.POINTER(C.c_uint64),
                                                C.POINTER(C.c_uint64)]
        L.garage_bm_stripe_repair_step.argtypes = [vp, i32, vp, sz, i32, vp, C.POINTER(i32), C.POINTER(C.c_uint64),
                                                   C.POINTER(C.c_uint64)]
        L.garage_bm_get_stripe_repair_metrics.argtypes = [vp, C.POINTER(StripeRepairMetrics)]
        L.garage_bm_get_stripe_repair_metrics.restype = None
        L.garage_bm_get_salvage_metrics.argtypes = [vp, C.POINTER(SalvageMetrics)]
        L.garage_bm_get_salvage_metrics.restype = None
        L.garage_bm_get_segment_repair_metrics.argtypes = [vp, C.POINTER(SegmentRepairMetrics)]
        L.garage_bm_get_segment_repair_metrics.restype = None
        L.garage_bm_create_with_drives.argtypes = [C.POINTER(vp), C.POINTER(Config), C.POINTER(DataDir), i32]
        L.garage_bm_create_on_devices.argtypes = [C.POINTER(vp), C.POINTER(Config), C.POINTER(DataDir), i32,
                                                  C.POINTER(C.c_int), i32]
        L.garage_bm_get_device_metrics.argtypes = [vp, C.POINTER(DeviceMetrics), i32, C.POINTER(i32)]
        L.garage_bm_set_data_dirs.argtypes = [vp, i32, C.POINTER(DataDir), i32]
        L.garage_bm_rebalance_step.argtypes = [vp, i32, vp, sz, vp, C.POINTER(i32), C.POINTER(C.c_uint64)]
        L.garage_bm_get_drive_metrics.argtypes = [vp, C.POINTER(DriveMetrics)]
        L.garage_bm_get_drive_metrics.restype = None
        u64p = C.POINTER(C.c_uint64)
        L.garage_bm_resync_step.argtypes = [vp, i32, i32, sz, u64p, u64p, u64p, C.POINTER(C.c_int64)]
        L.garage_bm_list_resync_errors.argtypes = [vp, i32, C.POINTER(ResyncError), sz, C.POINTER(sz)]
        L.garage_bm_resync_retry_now.argtypes = [vp, i32, vp, u64p]
        L.garage_bm_block_info.argtypes = [vp, vp, i32, C.POINTER(BlockStatus)]
        L.garage_bm_debug_set_clock_ms.argtypes = [vp, C.c_uint64]
        L.garage_bm_get_resync_metrics.argtypes = [vp, C.POINTER(ResyncMetrics)]
        L.garage_bm_get_resync_metrics.restype = None
        L.garage_bm_rpc_put_block_sealed.argtypes = [vp, vp, vp, sz, vp]
        L.garage_bm_rpc_get_block_opened.argtypes = [vp, vp, vp, vp, sz, C.POINTER(sz)]
        L.garage_bm_get_sealed_metrics.argtypes = [vp, C.POINTER(SealedMetrics)]
        L.garage_bm_get_sealed_metrics.restype = None
        L.garage_bm_rpc_get_block_range_opened.argtypes = [vp, vp, vp, C.c_uint32, C.c_uint32, vp, sz, C.POINTER(sz)]
        L.garage_bm_get_sealed_range_metrics.argtypes = [vp, C.POINTER(SealedRangeMetrics)]
        L.garage_bm_get_sealed_range_metrics.restype = None
        L.garage_bm_rpc_put_block_resealed.argtypes = [vp, vp, C.c_int, vp, vp, vp, C.POINTER(C.c_uint32)]
        L.garage_bm_get_reseal_metrics.argtypes = [vp, C.POINTER(ResealMetrics)]
        L.garage_bm_get_reseal_metrics.restype = None
        L.garage_bm_rpc_put_block_sealed_crc.argtypes = [vp, vp, vp, sz, C.c_uint8, vp, C.POINTER(C.c_uint32)]
        L.garage_bm_rpc_put_block_resealed_crc.argtypes = [vp, vp, C.c_int, vp, vp, C.c_uint8, vp,
                                                           C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
        _lib = L
    return _lib


def blake2sum(data) -> bytes:
    L = load_library()
    a = np.frombuffer(bytes(data), dtype=np.uint8) if not isinstance(data, np.ndarray) else np.ascontiguousarray(data)
    out = np.zeros(32, dtype=np.uint8)
    L.garage_bm_blake2sum(C.c_void_p(a.ctypes.data) if a.size else None, a.size, C.c_void_p(out.ctypes.data))
    return out.tobytes()


class BlockManagerError(RuntimeError):
    def __init__(self, code):
        super().__init__("garage_bm error %d" % code)
        self.code = code


class BlockManager:
    """Same method names as garage_block::manager::BlockManager where they exist."""

    def __init__(self, k=10, m=4, n_nodes=None, cuda_device=0, batch_max_blocks=64, batch_linger_us=100,
                 block_ram_buffer_max=256 << 20, data_dir=None, shard_sum_kind=SUM_ADLER8, verify_content_hash=True,
                 data_fsync=False, block_gc_delay_ms=0, local_groups=0, piggyback=False, previous_codes=(),
                 legacy_replicas=0, layout=None, clay=False, clay_layout=False, data_dirs=None, cuda_devices=None):
        """block_gc_delay_ms defaults to 0 HERE (tests delete at once); the library's default is the
        reference's BLOCK_GC_DELAY of 10 minutes.  local_groups > 0: LRC(k, local_groups, m - local_groups).
        piggyback: PB(k, m), half-shard repair reads.  clay: Clay(k, m), a lost shard rebuilt from 1/m of the others; clay_layout: that store may change its
        layout.  previous_codes: (k, m, local_groups, piggyback[, clay]) tuples of codes the store may still hold; legacy_replicas: replication factor of a previous replicated layout.
        layout: None (partition p on nodes (p mod n_nodes) + i) or a dict with zone, capacity and optionally
        zone_redundancy, max_per_zone: version 1 of the cluster layout.  data_dirs: None (one directory per node) or a list
        of (path, capacity[, read_only]) tuples or {path, capacity, read_only} dicts, paths relative to each node's
        directory: the drives every node spreads its files over.  cuda_devices: None (cuda_device alone) or the list of
        devices to run one dispatcher group each on (garage_bm_create_on_devices; a device may repeat)."""
        self._L = load_library()
        cfg = Config()
        self._L.garage_bm_default_config(C.byref(cfg))
        cfg.data_shards, cfg.parity_shards, cfg.cuda_device = k, m, cuda_device
        cfg.n_nodes = n_nodes or (k + m)
        cfg.batch_max_blocks, cfg.batch_linger_us = batch_max_blocks, batch_linger_us
        cfg.block_ram_buffer_max = block_ram_buffer_max
        cfg.shard_sum_kind, cfg.verify_content_hash = shard_sum_kind, 1 if verify_content_hash else 0
        cfg.data_fsync, cfg.block_gc_delay_ms = 1 if data_fsync else 0, block_gc_delay_ms
        cfg.local_groups = local_groups
        cfg.piggyback = 1 if piggyback else 0
        cfg.clay = 1 if clay else 0
        cfg.clay_layout = int(clay_layout)
        self._prev = (Code * max(1, len(previous_codes)))(*[Code(*map(int, c)) for c in previous_codes])  # kept alive
        cfg.previous_codes = C.cast(self._prev, C.POINTER(Code)) if previous_codes else None
        cfg.n_previous_codes, cfg.legacy_replicas = len(previous_codes), legacy_replicas
        self._dir = data_dir.encode() if data_dir else None  # keep the bytes alive
        cfg.data_dir = self._dir
        if layout is not None:
            self._spec, self._spec_arrays = _layout_spec(**layout)  # kept alive
            cfg.layout = C.pointer(self._spec)
        h = C.c_void_p()
        if cuda_devices is not None:
            devs = (C.c_int * max(1, len(cuda_devices)))(*map(int, cuda_devices))
            drives, n = _data_dirs(data_dirs) if data_dirs is not None else (None, 0)
            rc = self._L.garage_bm_create_on_devices(C.byref(h), C.byref(cfg), drives, n, devs, len(cuda_devices))
        elif data_dirs is None:
            rc = self._L.garage_bm_create(C.byref(h), C.byref(cfg))
        else:
            drives, n = _data_dirs(data_dirs)
            rc = self._L.garage_bm_create_with_drives(C.byref(h), C.byref(cfg), drives, n)
        if rc != OK:
            raise BlockManagerError(rc)
        self._h, self.k, self.m, self.n_nodes = h, k, m, cfg.n_nodes
        self._down = set()  # nodes set down through set_node_up

    def close(self):
        if getattr(self, "_h", None):
            self._L.garage_bm_destroy(self._h)
            self._h = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @staticmethod
    def _hp(hash32):
        return C.c_char_p(bytes(hash32))

    def rpc_put_block(self, hash32, data):
        a = np.ascontiguousarray(data, dtype=np.uint8)
        return self._L.garage_bm_rpc_put_block(self._h, self._hp(hash32), C.c_void_p(a.ctypes.data), a.size)

    def rpc_get_block(self, hash32, cap=(1 << 20) + 64):
        out = np.empty(cap, dtype=np.uint8)
        n = C.c_size_t(0)
        rc = self._L.garage_bm_rpc_get_block(self._h, self._hp(hash32), C.c_void_p(out.ctypes.data), cap, C.byref(n))
        return rc, (out[: n.value].copy() if rc == OK else None)

    def rpc_put_block_sealed(self, key32, data):
        """(rc, content address) of an SSE-C PUT; key32 None stores the block as plaintext"""
        a = np.ascontiguousarray(data, dtype=np.uint8)
        h = (C.c_uint8 * 32)()
        rc = self._L.garage_bm_rpc_put_block_sealed(self._h, None if key32 is None else C.c_char_p(bytes(key32)),
                                                    C.c_void_p(a.ctypes.data) if a.size else None, a.size, h)
        return rc, bytes(h)

    def rpc_put_block_sealed_crc(self, key32, data, crc_kind):
        """(rc, content address, CRC) of an SSE-C PUT that also returns the S3 checksum of kind crc_kind (CRC_*) of
        the plaintext"""
        a = np.ascontiguousarray(data, dtype=np.uint8)
        h = (C.c_uint8 * 32)()
        crc = C.c_uint32(0)
        rc = self._L.garage_bm_rpc_put_block_sealed_crc(self._h, None if key32 is None else C.c_char_p(bytes(key32)),
                                                        C.c_void_p(a.ctypes.data) if a.size else None, a.size,
                                                        crc_kind, h, C.byref(crc))
        return rc, bytes(h), crc.value

    def rpc_get_block_opened(self, hash32, key32, cap=1 << 20):
        """(rc, plaintext or None) of an SSE-C GET"""
        out = np.empty(max(cap, 1), dtype=np.uint8)
        n = C.c_size_t(0)
        rc = self._L.garage_bm_rpc_get_block_opened(self._h, self._hp(hash32), C.c_char_p(bytes(key32)),
                                                    C.c_void_p(out.ctypes.data), cap, C.byref(n))
        return rc, (out[: n.value].copy() if rc == OK else None)

    def sealed_metrics(self):
        mt = SealedMetrics()
        self._L.garage_bm_get_sealed_metrics(self._h, C.byref(mt))
        return {n: getattr(mt, n) for n, _ in SealedMetrics._fields_}

    def rpc_get_block_range_opened(self, hash32, key32, offset, length):
        """(rc, plaintext bytes [offset, offset + length) of an SSE-C block or None)"""
        out = np.empty(max(length, 1), dtype=np.uint8)
        n = C.c_size_t(0)
        rc = self._L.garage_bm_rpc_get_block_range_opened(self._h, self._hp(hash32), C.c_char_p(bytes(key32)), offset,
                                                          length, C.c_void_p(out.ctypes.data), length, C.byref(n))
        return rc, (out[: n.value].copy() if rc == OK else None)

    def get_sealed_range_metrics(self):
        mt = SealedRangeMetrics()
        self._L.garage_bm_get_sealed_range_metrics(self._h, C.byref(mt))
        return {n: getattr(mt, n) for n, _ in SealedRangeMetrics._fields_}

    def put_block_resealed(self, pieces, src_key32, dst_key32):
        """(rc, content address, stored length) of a copy with re-encryption: `pieces` is a list of (hash, offset,
        len) plaintext ranges of stored blocks, sealed into one new block under dst_key32; src_key32 None: the sources
        are plaintext blocks"""
        arr = (Piece * max(1, len(pieces)))()
        for i, (h, off, n) in enumerate(pieces):
            arr[i].hash[:] = list(bytes(h))
            arr[i].offset, arr[i].len = off, n
        h = (C.c_uint8 * 32)()
        ln = C.c_uint32(0)
        rc = self._L.garage_bm_rpc_put_block_resealed(
            self._h, arr, len(pieces), None if src_key32 is None else C.c_char_p(bytes(src_key32)),
            None if dst_key32 is None else C.c_char_p(bytes(dst_key32)), h, C.byref(ln))
        return rc, bytes(h), ln.value

    def put_block_resealed_crc(self, pieces, src_key32, dst_key32, crc_kind):
        """put_block_resealed that also returns the S3 checksum of kind crc_kind (CRC_*) of the new block's plaintext:
        (rc, content address, stored length, CRC)"""
        arr = (Piece * max(1, len(pieces)))()
        for i, (h, off, n) in enumerate(pieces):
            arr[i].hash[:] = list(bytes(h))
            arr[i].offset, arr[i].len = off, n
        h = (C.c_uint8 * 32)()
        ln, crc = C.c_uint32(0), C.c_uint32(0)
        rc = self._L.garage_bm_rpc_put_block_resealed_crc(
            self._h, arr, len(pieces), None if src_key32 is None else C.c_char_p(bytes(src_key32)),
            None if dst_key32 is None else C.c_char_p(bytes(dst_key32)), crc_kind, h, C.byref(ln), C.byref(crc))
        return rc, bytes(h), ln.value, crc.value

    def reseal_metrics(self):
        mt = ResealMetrics()
        self._L.garage_bm_get_reseal_metrics(self._h, C.byref(mt))
        return {n: getattr(mt, n) for n, _ in ResealMetrics._fields_}

    def rpc_get_block_range(self, hash32, offset, length):
        """(rc, bytes [offset, offset + length) of the block or None)"""
        out = np.empty(max(length, 1), dtype=np.uint8)
        n = C.c_size_t(0)
        rc = self._L.garage_bm_rpc_get_block_range(self._h, self._hp(hash32), offset, length, C.c_void_p(out.ctypes.data),
                                                   length, C.byref(n))
        return rc, (out[: n.value].copy() if rc == OK else None)

    def block_incref(self, hash32):
        return self._L.garage_bm_block_incref(self._h, self._hp(hash32))

    def block_decref(self, hash32):
        return self._L.garage_bm_block_decref(self._h, self._hp(hash32))

    def get_block_rc(self, hash32):
        return int(self._L.garage_bm_get_block_rc(self._h, self._hp(hash32)))

    def resync_block(self, node, hash32):
        return self._L.garage_bm_resync_block(self._h, node, self._hp(hash32))

    def resync_all(self, node, workers=8):
        done = C.c_uint64(0)
        failed = self._L.garage_bm_resync_all(self._h, node, workers, C.byref(done))
        return failed, done.value

    def resync_step(self, node, workers=8, max_blocks=0):
        """one ResyncWorker pass over node's due entries -> (rc, resynced, failed, deferred, wait_ms)"""
        a, b, c, w = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0), C.c_int64(0)
        rc = self._L.garage_bm_resync_step(self._h, node, workers, max_blocks, C.byref(a), C.byref(b), C.byref(c),
                                           C.byref(w))
        return rc, a.value, b.value, c.value, w.value

    def list_resync_errors(self, node=-1):
        """-> (rc, [dict of node, hash, rc, errors, last_try_ms, next_try_ms, last_status]) in node then hash order"""
        n = C.c_size_t(0)
        rc = self._L.garage_bm_list_resync_errors(self._h, node, None, 0, C.byref(n))  # the size query
        if rc != OK:
            return rc, []
        arr = (ResyncError * max(1, n.value))()
        rc = self._L.garage_bm_list_resync_errors(self._h, node, arr, len(arr), C.byref(n))
        out = [{"node": e.node, "hash": bytes(e.hash), "rc": e.rc, "errors": e.errors, "last_try_ms": e.last_try_ms,
                "next_try_ms": e.next_try_ms, "last_status": e.last_status} for e in arr[:min(n.value, len(arr))]]
        return rc, out

    def resync_retry_now(self, node, hash32=None):
        """clear_backoff of hash32 (None: every error entry of node) -> (rc, entries made due)"""
        n = C.c_uint64(0)
        rc = self._L.garage_bm_resync_retry_now(self._h, node, self._hp(hash32) if hash32 is not None else None,
                                                C.byref(n))
        return rc, n.value

    def block_info(self, hash32, check_tags=False):
        """-> (rc, dict of rc, code, block_len, node, state, resync_errors (per index), recoverable, read_set)"""
        st = BlockStatus()
        rc = self._L.garage_bm_block_info(self._h, self._hp(hash32), 1 if check_tags else 0, C.byref(st))
        n = st.n_shards
        return rc, {"rc": st.rc, "code": (st.code.k, st.code.m, st.code.local_groups, st.code.piggyback, st.code.clay),
                    "block_len": st.block_len, "node": list(st.node[:n]), "state": list(st.state[:n]),
                    "resync_errors": list(st.resync_errors[:n]), "recoverable": bool(st.recoverable),
                    "read_set": list(st.read_set[:n])}

    def debug_set_clock_ms(self, now_ms):
        return self._L.garage_bm_debug_set_clock_ms(self._h, now_ms)

    def resync_metrics(self):
        mt = ResyncMetrics()
        self._L.garage_bm_get_resync_metrics(self._h, C.byref(mt))
        return {n: getattr(mt, n) for n, _ in ResyncMetrics._fields_}

    def repair_enqueue_missing(self, node):
        n = C.c_uint64(0)
        self._L.garage_bm_repair_enqueue_missing(self._h, node, C.byref(n))
        return n.value

    def scrub(self, node):
        a, b = C.c_uint64(0), C.c_uint64(0)
        rc = self._L.garage_bm_scrub(self._h, node, C.byref(a), C.byref(b))
        return rc, a.value, b.value

    def scrub_step(self, node, cursor=None, max_shards=0):
        """-> (rc, cursor_out bytes, finished, checked, corrupt)"""
        out = C.create_string_buffer(32)
        fin, a, b = C.c_int(0), C.c_uint64(0), C.c_uint64(0)
        rc = self._L.garage_bm_scrub_step(self._h, node, C.c_char_p(bytes(cursor)) if cursor else None, max_shards,
                                          C.cast(out, C.c_void_p), C.byref(fin), C.byref(a), C.byref(b))
        return rc, out.raw, bool(fin.value), a.value, b.value

    def deep_scrub_step(self, node, cursor=None, max_blocks=0):
        """-> (rc, cursor_out bytes, finished, blocks checked, shards quarantined)"""
        out = C.create_string_buffer(32)
        fin, a, b = C.c_int(0), C.c_uint64(0), C.c_uint64(0)
        rc = self._L.garage_bm_deep_scrub_step(self._h, node, C.c_char_p(bytes(cursor)) if cursor else None, max_blocks,
                                               C.cast(out, C.c_void_p), C.byref(fin), C.byref(a), C.byref(b))
        return rc, out.raw, bool(fin.value), a.value, b.value

    def stripe_repair_step(self, node, cursor=None, max_blocks=0, min_missing=0):
        """-> (rc, cursor_out bytes, finished, stripes repaired, shards rebuilt)"""
        out = C.create_string_buffer(32)
        fin, a, b = C.c_int(0), C.c_uint64(0), C.c_uint64(0)
        rc = self._L.garage_bm_stripe_repair_step(self._h, node, C.c_char_p(bytes(cursor)) if cursor else None, max_blocks,
                                                  min_missing, C.cast(out, C.c_void_p), C.byref(fin), C.byref(a),
                                                  C.byref(b))
        return rc, out.raw, bool(fin.value), a.value, b.value

    def stripe_repair_all(self, min_missing=0):
        """one full stripe_repair_step sweep of every node that is up -> (stripes repaired, shards rebuilt); an error
        from a node that is up raises BlockManagerError"""
        repaired = rebuilt = 0
        for node in range(self.n_nodes):
            if node in self._down:
                continue
            rc, _, finished, a, b = self.stripe_repair_step(node, min_missing=min_missing)
            if rc != OK:
                raise BlockManagerError(rc)
            assert finished
            repaired, rebuilt = repaired + a, rebuilt + b
        return repaired, rebuilt

    def stripe_repair_metrics(self):
        mt = StripeRepairMetrics()
        self._L.garage_bm_get_stripe_repair_metrics(self._h, C.byref(mt))
        return {n: getattr(mt, n) for n, _ in StripeRepairMetrics._fields_}

    def salvage_metrics(self):
        """garage_bm_salvage_metrics (DESIGN.md section 5.14) as a dict"""
        mt = SalvageMetrics()
        self._L.garage_bm_get_salvage_metrics(self._h, C.byref(mt))
        return {n: getattr(mt, n) for n, _ in SalvageMetrics._fields_}

    def segment_repair_metrics(self):
        """garage_bm_segment_repair_metrics (DESIGN.md section 5.15) as a dict"""
        mt = SegmentRepairMetrics()
        self._L.garage_bm_get_segment_repair_metrics(self._h, C.byref(mt))
        return {n: getattr(mt, n) for n, _ in SegmentRepairMetrics._fields_}

    def set_data_dirs(self, node, dirs):
        """node restarts with this data_dir list ((path, capacity[, read_only]) tuples or dicts) -> rc; a failed marker
        check (E_MESSAGE) leaves the node down, success brings it up"""
        arr, n = _data_dirs(dirs)
        rc = self._L.garage_bm_set_data_dirs(self._h, node, C.cast(arr, C.POINTER(DataDir)) if n else None, n)
        if rc == OK:
            self._down.discard(node)
        elif rc == E_MESSAGE:
            self._down.add(node)
        return rc

    def rebalance_step(self, node, cursor=None, max_files=0):
        """-> (rc, cursor_out bytes, finished, files moved)"""
        out = C.create_string_buffer(32)
        fin, n = C.c_int(0), C.c_uint64(0)
        rc = self._L.garage_bm_rebalance_step(self._h, node, C.c_char_p(bytes(cursor)) if cursor else None, max_files,
                                              C.cast(out, C.c_void_p), C.byref(fin), C.byref(n))
        return rc, out.raw, bool(fin.value), n.value

    def rebalance_all(self, nodes=None):
        """one full rebalance_step pass over every node that is up (or over `nodes`) -> files moved; an error from a
        node that is up raises BlockManagerError"""
        total = 0
        for node in (range(self.n_nodes) if nodes is None else nodes):
            if node in self._down:
                continue
            rc, _, finished, n = self.rebalance_step(node)
            if rc != OK:
                raise BlockManagerError(rc)
            assert finished
            total += n
        return total

    def device_metrics(self):
        """one dict per dispatcher group, in the order the devices were listed"""
        n = C.c_int(0)
        arr = (DeviceMetrics * MAX_DEVICES)()
        rc = self._L.garage_bm_get_device_metrics(self._h, arr, MAX_DEVICES, C.byref(n))
        if rc != OK:
            raise BlockManagerError(rc)
        return [{f: getattr(arr[i], f) for f, _ in DeviceMetrics._fields_} for i in range(n.value)]

    def drive_metrics(self):
        mt = DriveMetrics()
        self._L.garage_bm_get_drive_metrics(self._h, C.byref(mt))
        return {n: getattr(mt, n) for n, _ in DriveMetrics._fields_}

    def convert_step(self, node, cursor=None, max_blocks=0):
        """-> (rc, cursor_out bytes, finished, converted)"""
        out = C.create_string_buffer(32)
        fin, n = C.c_int(0), C.c_uint64(0)
        rc = self._L.garage_bm_convert_step(self._h, node, C.c_char_p(bytes(cursor)) if cursor else None, max_blocks,
                                            C.cast(out, C.c_void_p), C.byref(fin), C.byref(n))
        return rc, out.raw, bool(fin.value), n.value

    def convert_all(self):
        """one full convert_step sweep over every node -> blocks converted"""
        total = 0
        for node in range(self.n_nodes):
            rc, _, finished, n = self.convert_step(node)
            if rc == OK:
                assert finished
                total += n
        return total

    def debug_convert_stop_after(self, n_ops):
        return self._L.garage_bm_debug_convert_stop_after(self._h, n_ops)

    def apply_layout(self, zone, capacity, zone_redundancy=0, max_per_zone=0):
        """-> (rc, new version)"""
        spec, keep = _layout_spec(zone, capacity, zone_redundancy, max_per_zone)
        v = C.c_uint64(0)
        rc = self._L.garage_bm_apply_layout(self._h, C.byref(spec), C.byref(v))
        del keep
        return rc, v.value

    def layout_sync_step(self, node, cursor=None, max_blocks=0):
        """-> (rc, cursor_out bytes, finished, shards moved)"""
        out = C.create_string_buffer(32)
        fin, n = C.c_int(0), C.c_uint64(0)
        rc = self._L.garage_bm_layout_sync_step(self._h, node, C.c_char_p(bytes(cursor)) if cursor else None, max_blocks,
                                                C.cast(out, C.c_void_p), C.byref(fin), C.byref(n))
        return rc, out.raw, bool(fin.value), n.value

    def layout_sync_all(self, nodes=None):
        """one full layout_sync_step pass over every node that is up (or over `nodes`) -> shards moved; an error from
        a node that is up raises BlockManagerError"""
        total = 0
        for node in (range(self.n_nodes) if nodes is None else nodes):
            if node in self._down:
                continue
            rc, _, finished, n = self.layout_sync_step(node)
            if rc != OK:
                raise BlockManagerError(rc)
            assert finished
            total += n
        return total

    def layout_versions(self):
        out = (C.c_uint64 * 8)()
        n = self._L.garage_bm_layout_versions(self._h, out, 8)
        return list(out[:n])

    def set_node_up(self, node, up):
        rc = self._L.garage_bm_set_node_up(self._h, node, 1 if up else 0)
        if rc == OK:
            (self._down.discard if up else self._down.add)(node)
        return rc

    def corrupt_shard(self, node, hash32, byte_off=0):
        return self._L.garage_bm_corrupt_shard(self._h, node, self._hp(hash32), byte_off)

    def corrupt_shard_header(self, node, hash32, what):
        return self._L.garage_bm_corrupt_shard_header(self._h, node, self._hp(hash32), what)

    def plant_stale_shard(self, node, hash32):
        return self._L.garage_bm_plant_stale_shard(self._h, node, self._hp(hash32))

    def set_node_readonly(self, node, readonly):
        return self._L.garage_bm_set_node_readonly(self._h, node, 1 if readonly else 0)

    def bench(self, threads, blocks_per_thread, block_len=1 << 20, mode=0, seed=1):
        """native closed-loop load generator: -> (rc, GiB/s, errors)"""
        g, e = C.c_double(0), C.c_uint64(0)
        rc = self._L.garage_bm_bench(self._h, threads, blocks_per_thread, block_len, mode, seed, C.byref(g), C.byref(e))
        return rc, g.value, e.value

    def drop_shard(self, node, hash32):
        return self._L.garage_bm_drop_shard(self._h, node, self._hp(hash32))

    def node_shard_index(self, node, hash32):
        return self._L.garage_bm_node_shard_index(self._h, node, self._hp(hash32))

    def storage_nodes_of(self, hash32):
        out = (C.c_int * (self.k + self.m))()
        self._L.garage_bm_storage_nodes_of(self._h, self._hp(hash32), out)
        return list(out)

    def metrics(self):
        mt = Metrics()
        self._L.garage_bm_get_metrics(self._h, C.byref(mt))
        rm = RangeMetrics()
        self._L.garage_bm_get_range_metrics(self._h, C.byref(rm))
        out = {n: getattr(mt, n) for n, _ in Metrics._fields_}
        out.update({n: getattr(rm, n) for n, _ in RangeMetrics._fields_})
        return out


# ---- shard wire format (include/garage_shard_wire.h) ---------------------------------------------
class ShardHeader(C.Structure):
    _fields_ = [("hash", C.c_uint8 * 32), ("header", C.c_uint8), ("k", C.c_uint8), ("m", C.c_uint8),
                ("index", C.c_uint8), ("sum_kind", C.c_uint8), ("migrated", C.c_uint8),
                ("block_len", C.c_uint32), ("shard_len", C.c_uint32), ("sum", C.c_uint8 * 32), ("l", C.c_uint8),
                ("pb", C.c_uint8), ("clay", C.c_uint8)]

    def as_dict(self):
        d = {"hash": bytes(self.hash), "header": int(self.header), "k": int(self.k), "m": int(self.m),
             "index": int(self.index), "sum_kind": int(self.sum_kind), "migrated": int(self.migrated),
             "block_len": int(self.block_len), "shard_len": int(self.shard_len), "sum": bytes(self.sum)}
        if self.l:  # like the wire: only LRC shards carry it
            d["l"] = int(self.l)
        if self.pb:  # only PB shards carry it
            d["pb"] = int(self.pb)
        if self.clay:  # only Clay shards carry it
            d["clay"] = int(self.clay)
        return d


WIRE_SYMBOLS = ["garage_shard_wire_encode", "garage_shard_wire_decode", "garage_shard_wire_encode_v0"]


def _wire():
    L = load_library()
    L.garage_shard_wire_encode.argtypes = [C.POINTER(ShardHeader), C.c_void_p, C.c_size_t]
    L.garage_shard_wire_encode.restype = C.c_size_t
    L.garage_shard_wire_decode.argtypes = [C.c_void_p, C.c_size_t, C.POINTER(ShardHeader)]
    L.garage_shard_wire_encode_v0.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t]
    L.garage_shard_wire_encode_v0.restype = C.c_size_t
    return L


def wire_encode(hash32, header, k, m, index, block_len, shard_len, sum_kind, sum32, l=0, pb=0, clay=0) -> bytes:
    h = ShardHeader()
    C.memmove(h.hash, bytes(hash32), 32)
    C.memmove(h.sum, bytes(sum32), 32)
    h.header, h.k, h.m, h.index, h.sum_kind = header, k, m, index, sum_kind
    h.block_len, h.shard_len, h.l, h.pb, h.clay = block_len, shard_len, l, pb, clay
    buf = (C.c_uint8 * 256)()
    n = _wire().garage_shard_wire_encode(C.byref(h), buf, 256)
    return bytes(buf[:n])


def wire_encode_v0(hash32, header) -> bytes:
    buf = (C.c_uint8 * 128)()
    hb = (C.c_uint8 * 32).from_buffer_copy(bytes(hash32))
    n = _wire().garage_shard_wire_encode_v0(hb, header, buf, 128)
    return bytes(buf[:n])


def wire_decode(data: bytes):
    h = ShardHeader()
    b = (C.c_uint8 * len(data)).from_buffer_copy(data) if data else None
    rc = _wire().garage_shard_wire_decode(b, len(data), C.byref(h))
    return None if rc else h.as_dict()
