"""ctypes binding of libdint_b200.so (include/dint_b200.h): the GPU-resident stand-in for one
reference server process (`server <threads>` / `server_shard <id> <threads>`).

There is no CPU implementation behind this class: if the CUDA library cannot be built/loaded, or no
CUDA device is present, construction raises.
"""
import ctypes as C
import os

import numpy as np

from . import _build
from .wire import MSG_SIZE, LOG_ENTRY_SIZE, KIND_NAMES

DINT_OK, DINT_EPROTO = 0, -71
# dint_cfg.flags bit (tatp): keep the holder's key beside every lock bit, so that a refused kAcquireLock is answered
# kRejectLockSameKey (28) or kRejectLock (8, false sharing) as tatp/ebpf/lock_kern.c:289-298 does
DINT_CFG_LOCK_HOLDER_KEYS = 1
# dint_cfg.flags bits 1-2 (store): answer as the reference's eBPF store server, with its per-bucket cache tier in front of
# the table (store/ebpf/store_kern.c, store_wb_kern.c, store_wt_kern.c); see include/dint_b200.h
DINT_CFG_STORE_EBPF_WB_BLOOM, DINT_CFG_STORE_EBPF_WB, DINT_CFG_STORE_EBPF_WT = 1 << 1, 2 << 1, 3 << 1
DINT_CFG_STORE_EBPF_MASK = 3 << 1
STORE_EBPF_VARIANTS = {"wb_bloom": DINT_CFG_STORE_EBPF_WB_BLOOM, "wb": DINT_CFG_STORE_EBPF_WB, "wt": DINT_CFG_STORE_EBPF_WT}
STORE_CACHE_ENTRY_BYTES = 232      # struct cache_entry, store/ebpf/utils.h:58-66
STORE_CACHE_STATS = ("hits", "bloom_negatives", "table", "write_backs", "installs")
# dint_cfg.flags bit 3 (tatp): answer as the reference's eBPF TATP shard server (tatp/ebpf/shard_kern.c; with
# lock_holder_keys, lock_kern.c): a write-back cache set with a bloom word per bucket in front of chained tables
DINT_CFG_TATP_EBPF = 1 << 3
TATP_CHAIN_REC = np.dtype([("key", "<u8", (4,)), ("ver", "<u4", (4,)), ("valid", "u1", (4,)), ("val", "u1", (4, 40))])
TATP_CACHE_STATS = STORE_CACHE_STATS + ("allocated", "reused", "freed", "failed")
# dint_cfg.flags bit 4 (smallbank): answer as the reference's eBPF SmallBank shard server (smallbank/ebpf/shard_kern.c):
# a write-back cache set per bucket of both tables in front of them, warmed by dint_populate as its client warms it
DINT_CFG_SMALLBANK_EBPF = 1 << 4
SMALLBANK_CACHE_ENTRY_BYTES = 96   # struct cache_entry, smallbank/ebpf/utils.h:82-89
SMALLBANK_CACHE_STATS = ("hits", "table", "write_backs", "installs")


class DintCfg(C.Structure):
    _fields_ = [("lock_slots", C.c_uint32), ("log_ring", C.c_uint32), ("subs_sizing", C.c_uint32),
                ("subs_populate", C.c_uint32), ("accts_sizing", C.c_uint32), ("accts_populate", C.c_uint32),
                ("n_shards", C.c_uint32), ("shard_id", C.c_uint32), ("chunk", C.c_uint32),
                ("kv_capacity_log2", C.c_uint32 * 5), ("flags", C.c_uint32), ("txn_shards", C.c_uint32),
                ("txn_shard_id", C.c_uint32), ("reserved", C.c_uint32 * 2)]


class DintStats(C.Structure):
    _fields_ = [("requests", C.c_uint64), ("chunks", C.c_uint64), ("kernel_launches", C.c_uint64),
                ("conflicted", C.c_uint64), ("max_run", C.c_uint64), ("errors", C.c_uint64),
                ("h2d_bytes", C.c_uint64), ("d2h_bytes", C.c_uint64), ("kv_rebuilds", C.c_uint64),
                ("ordered_fallbacks", C.c_uint64), ("bucket_split_tasks", C.c_uint64), ("writerless_chunks", C.c_uint64)]


class DintPeerPtrs(C.Structure):
    _fields_ = [("p", C.c_uint64 * 8)]

    @classmethod
    def of(cls, ptrs):
        o = cls()
        for i, v in enumerate(ptrs):
            o.p[i] = int(v)
        return o


class DintClientsCfg(C.Structure):
    _fields_ = [("n_clients", C.c_uint32), ("n_keys", C.c_uint32), ("seed", C.c_uint64), ("zipf_theta", C.c_double),
                ("read_pct", C.c_uint32), ("set_pct", C.c_uint32), ("store_subscribers", C.c_uint32),
                ("store_hot", C.c_uint32), ("reserved", C.c_uint32 * 4)]


class DintKernelTime(C.Structure):
    _fields_ = [("name", C.c_char * 32), ("launches", C.c_uint64), ("total_ms", C.c_double)]


_lib = None

# every symbol include/dint_b200.h declares
ABI_SYMBOLS = [
    "dint_msg_size", "dint_default_cfg", "dint_create", "dint_destroy", "dint_populate", "dint_load",
    "dint_submit", "dint_submit_device", "dint_route_owner", "dint_route_partition", "dint_route_unpermute", "dint_route_tile_records", "dint_route_dispatch", "dint_route_combine", "dint_p2p_wait", "dint_p2p_signal", "dint_shard_create", "dint_shard_destroy", "dint_shard_submit_many", "dint_shard_submit_host", "dint_shard_submit_many_v", "dint_shard_flags", "dint_cluster_create", "dint_cluster_populate", "dint_cluster_submit", "dint_cluster_engine", "dint_cluster_size", "dint_cluster_overflow_retries", "dint_shard_recover", "dint_cluster_destroy", "dint_clients_create", "dint_clients_create_cfg", "dint_clients_run", "dint_clients_stats", "dint_clients_stats_all", "dint_clients_peek", "dint_clients_destroy", "dint_txn_clients_create", "dint_txn_clients_run", "dint_txn_clients_stats", "dint_txn_clients_peek", "dint_txn_clients_times", "dint_txn_clients_lock_stats", "dint_txn_clients_destroy", "dint_cluster_clients_create", "dint_cluster_clients_run", "dint_cluster_clients_stats", "dint_cluster_clients_peek", "dint_cluster_clients_times", "dint_cluster_clients_destroy", "dint_snapshot_create", "dint_snapshot_restore", "dint_snapshot_destroy", "dint_image_save", "dint_image_open", "dint_cluster_image_save", "dint_cluster_image_open", "dint_image_times", "dint_cluster_reshard", "dint_reshard_times", "dint_cluster_rebuild", "dint_cluster_image_open_rebuild", "dint_rebuild_times", "dint_cluster_clients_rebind", "dint_cluster_reshard_txn", "dint_txn_clients_drain", "dint_txn_clients_rebind", "dint_sync", "dint_kv_get", "dint_store_cache_set", "dint_store_cache_stats", "dint_tatp_cache_set", "dint_tatp_chain", "dint_tatp_cache_stats", "dint_smallbank_cache_set", "dint_smallbank_cache_stats", "dint_kv_count", "dint_lock_state", "dint_lock_holder",
    "dint_lock_slot", "dint_dump_log", "dint_log_entry_size", "dint_get_stats", "dint_reset_stats",
    "dint_profile", "dint_kernel_times", "dint_last_error", "dint_host_alloc", "dint_host_free",
    "dint_test_fasthash64", "dint_test_fastmod", "dint_test_rebuild_source", "dint_test_txn_reshard_dests", "dint_test_host_slices",
]


def lib():
    """Load (building first if the sources are newer) libdint_b200.so.  Raises if that is impossible."""
    global _lib
    if _lib is not None:
        return _lib
    path = _build.LIB
    if _build.find_nvcc() is not None:
        _build.build()
    if not os.path.exists(path):
        raise RuntimeError(f"{path} is missing and nvcc is not available: dint_b200 has no CPU fallback")
    L = C.CDLL(path)
    vp, u32, u64, i32 = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int
    L.dint_msg_size.restype = u32; L.dint_msg_size.argtypes = [i32]
    L.dint_default_cfg.restype = None; L.dint_default_cfg.argtypes = [i32, C.POINTER(DintCfg)]
    L.dint_create.restype = i32; L.dint_create.argtypes = [i32, C.POINTER(DintCfg), i32, C.POINTER(vp)]
    L.dint_destroy.restype = None; L.dint_destroy.argtypes = [vp]
    L.dint_populate.restype = i32; L.dint_populate.argtypes = [vp]
    L.dint_load.restype = i32; L.dint_load.argtypes = [vp, i32, vp, vp, u64]
    L.dint_submit.restype = i32; L.dint_submit.argtypes = [vp, vp, u64, vp]
    L.dint_submit_device.restype = i32; L.dint_submit_device.argtypes = [vp, vp, u64, vp, vp]
    L.dint_route_owner.restype = i32; L.dint_route_owner.argtypes = [vp, vp, u64, vp, vp]
    L.dint_route_partition.restype = i32; L.dint_route_partition.argtypes = [vp, vp, vp, u64, u32, vp, vp, vp, vp]
    pp = C.POINTER(DintPeerPtrs)
    L.dint_route_tile_records.restype = u32; L.dint_route_tile_records.argtypes = [vp]
    L.dint_route_dispatch.restype = i32; L.dint_route_dispatch.argtypes = [vp, vp, vp, u64, u32, u32, u32, pp, pp, u32, vp, vp, vp, vp]
    L.dint_route_combine.restype = i32; L.dint_route_combine.argtypes = [vp, pp, vp, vp, u64, u32, u32, vp, vp]
    L.dint_p2p_wait.restype = i32; L.dint_p2p_wait.argtypes = [vp, vp, u32, u32, vp, vp]
    L.dint_p2p_signal.restype = i32; L.dint_p2p_signal.argtypes = [vp, pp, u32, u32, u32, vp]
    L.dint_shard_create.restype = i32; L.dint_shard_create.argtypes = [vp, u32, u32, u32, u32, pp, pp, pp, u64, C.POINTER(vp)]
    L.dint_shard_submit_many_v.restype = i32; L.dint_shard_submit_many_v.argtypes = [vp, u32, C.POINTER(vp), C.POINTER(vp), C.POINTER(u64), C.POINTER(u32), C.POINTER(vp), vp]
    L.dint_shard_submit_host.restype = i32; L.dint_shard_submit_host.argtypes = [vp, u32, C.POINTER(vp), C.POINTER(vp), u64, C.POINTER(vp)]
    L.dint_cluster_create.restype = i32; L.dint_cluster_create.argtypes = [i32, C.POINTER(DintCfg), i32, C.POINTER(i32), u64, C.POINTER(vp)]
    L.dint_cluster_populate.restype = i32; L.dint_cluster_populate.argtypes = [vp]
    L.dint_cluster_submit.restype = i32; L.dint_cluster_submit.argtypes = [vp, vp, u64, vp, vp]
    L.dint_cluster_engine.restype = vp; L.dint_cluster_engine.argtypes = [vp, i32]
    L.dint_cluster_size.restype = u32; L.dint_cluster_size.argtypes = [vp]
    L.dint_cluster_overflow_retries.restype = u64; L.dint_cluster_overflow_retries.argtypes = [vp]
    L.dint_shard_recover.restype = i32; L.dint_shard_recover.argtypes = [vp, u32, C.POINTER(u32)]
    L.dint_cluster_destroy.restype = None; L.dint_cluster_destroy.argtypes = [vp]
    L.dint_clients_create.restype = i32; L.dint_clients_create.argtypes = [vp, u32, u64, u32, C.c_double, u32, C.POINTER(vp)]
    L.dint_clients_create_cfg.restype = i32; L.dint_clients_create_cfg.argtypes = [vp, C.POINTER(DintClientsCfg), C.POINTER(vp)]
    L.dint_clients_run.restype = i32; L.dint_clients_run.argtypes = [vp, u32, vp]
    L.dint_clients_stats.restype = i32; L.dint_clients_stats.argtypes = [vp, C.POINTER(u64)]
    L.dint_clients_stats_all.restype = i32; L.dint_clients_stats_all.argtypes = [vp, C.POINTER(u64)]
    L.dint_clients_peek.restype = i32; L.dint_clients_peek.argtypes = [vp, vp, vp]
    L.dint_clients_destroy.restype = None; L.dint_clients_destroy.argtypes = [vp]
    L.dint_txn_clients_create.restype = i32; L.dint_txn_clients_create.argtypes = [vp, u32, u32, u32, C.POINTER(vp)]
    L.dint_txn_clients_run.restype = i32; L.dint_txn_clients_run.argtypes = [vp, u32]
    L.dint_txn_clients_stats.restype = i32; L.dint_txn_clients_stats.argtypes = [vp, C.POINTER(u64)]
    L.dint_txn_clients_peek.restype = i32; L.dint_txn_clients_peek.argtypes = [vp, vp, vp, C.POINTER(u64), vp, C.POINTER(u64)]
    L.dint_txn_clients_times.restype = i32; L.dint_txn_clients_times.argtypes = [vp, C.POINTER(C.c_double)]
    L.dint_txn_clients_lock_stats.restype = i32; L.dint_txn_clients_lock_stats.argtypes = [vp, C.POINTER(u64)]
    L.dint_txn_clients_destroy.restype = None; L.dint_txn_clients_destroy.argtypes = [vp]
    L.dint_txn_clients_drain.restype = i32; L.dint_txn_clients_drain.argtypes = [vp, u32, C.POINTER(u32)]
    L.dint_txn_clients_rebind.restype = i32; L.dint_txn_clients_rebind.argtypes = [vp, vp]
    L.dint_cluster_clients_create.restype = i32; L.dint_cluster_clients_create.argtypes = [vp, C.POINTER(DintClientsCfg), C.POINTER(vp)]
    L.dint_cluster_clients_run.restype = i32; L.dint_cluster_clients_run.argtypes = [vp, u32]
    L.dint_cluster_clients_stats.restype = i32; L.dint_cluster_clients_stats.argtypes = [vp, C.POINTER(u64)]
    L.dint_cluster_clients_peek.restype = i32; L.dint_cluster_clients_peek.argtypes = [vp, vp, vp]
    L.dint_cluster_clients_times.restype = i32; L.dint_cluster_clients_times.argtypes = [vp, C.POINTER(C.c_double)]
    L.dint_cluster_clients_destroy.restype = None; L.dint_cluster_clients_destroy.argtypes = [vp]
    L.dint_snapshot_create.restype = i32; L.dint_snapshot_create.argtypes = [vp, C.POINTER(vp)]
    L.dint_snapshot_restore.restype = i32; L.dint_snapshot_restore.argtypes = [vp, vp]
    L.dint_snapshot_destroy.restype = None; L.dint_snapshot_destroy.argtypes = [vp]
    L.dint_image_save.restype = i32; L.dint_image_save.argtypes = [vp, C.c_char_p]
    L.dint_image_open.restype = i32; L.dint_image_open.argtypes = [C.c_char_p, i32, C.POINTER(vp)]
    L.dint_cluster_image_save.restype = i32; L.dint_cluster_image_save.argtypes = [vp, C.c_char_p]
    L.dint_cluster_image_open.restype = i32; L.dint_cluster_image_open.argtypes = [C.c_char_p, i32, C.POINTER(i32), u64, C.POINTER(vp)]
    L.dint_image_times.restype = i32; L.dint_image_times.argtypes = [C.POINTER(C.c_double)]
    L.dint_cluster_reshard.restype = i32; L.dint_cluster_reshard.argtypes = [vp, i32, C.POINTER(i32), u64, C.POINTER(vp)]
    L.dint_reshard_times.restype = i32; L.dint_reshard_times.argtypes = [C.POINTER(C.c_double)]
    L.dint_cluster_reshard_txn.restype = i32; L.dint_cluster_reshard_txn.argtypes = [vp, i32, C.POINTER(i32), u64, C.POINTER(vp)]
    L.dint_cluster_rebuild.restype = i32; L.dint_cluster_rebuild.argtypes = [vp, u32]
    L.dint_cluster_image_open_rebuild.restype = i32
    L.dint_cluster_image_open_rebuild.argtypes = [C.c_char_p, i32, C.POINTER(i32), u64, C.POINTER(u32), C.POINTER(vp)]
    L.dint_rebuild_times.restype = i32; L.dint_rebuild_times.argtypes = [C.POINTER(C.c_double)]
    L.dint_cluster_clients_rebind.restype = i32; L.dint_cluster_clients_rebind.argtypes = [vp, vp]
    L.dint_shard_destroy.restype = None; L.dint_shard_destroy.argtypes = [vp]
    L.dint_shard_submit_many.restype = i32; L.dint_shard_submit_many.argtypes = [vp, u32, C.POINTER(vp), C.POINTER(vp), u64, C.POINTER(vp), vp]
    L.dint_shard_flags.restype = i32; L.dint_shard_flags.argtypes = [vp, C.POINTER(u32)]
    L.dint_route_unpermute.restype = i32; L.dint_route_unpermute.argtypes = [vp, vp, vp, u64, vp, vp]
    L.dint_sync.restype = i32; L.dint_sync.argtypes = [vp]
    L.dint_kv_get.restype = i32; L.dint_kv_get.argtypes = [vp, i32, u64, vp, C.POINTER(u32)]
    L.dint_store_cache_set.restype = i32; L.dint_store_cache_set.argtypes = [vp, u32, vp]
    L.dint_store_cache_stats.restype = i32; L.dint_store_cache_stats.argtypes = [vp, C.POINTER(u64)]
    L.dint_tatp_cache_set.restype = i32; L.dint_tatp_cache_set.argtypes = [vp, i32, u32, vp]
    L.dint_tatp_chain.restype = i32; L.dint_tatp_chain.argtypes = [vp, i32, u32, vp, u32, C.POINTER(u32)]
    L.dint_tatp_cache_stats.restype = i32; L.dint_tatp_cache_stats.argtypes = [vp, C.POINTER(u64)]
    L.dint_smallbank_cache_set.restype = i32; L.dint_smallbank_cache_set.argtypes = [vp, i32, u32, vp]
    L.dint_smallbank_cache_stats.restype = i32; L.dint_smallbank_cache_stats.argtypes = [vp, C.POINTER(u64)]
    L.dint_kv_count.restype = C.c_int64; L.dint_kv_count.argtypes = [vp, i32]
    L.dint_lock_state.restype = i32; L.dint_lock_state.argtypes = [vp, i32, u32, C.POINTER(u32)]
    L.dint_lock_holder.restype = i32; L.dint_lock_holder.argtypes = [vp, i32, u32, C.POINTER(u64)]
    L.dint_lock_slot.restype = u32; L.dint_lock_slot.argtypes = [vp, i32, u64]
    L.dint_dump_log.restype = i32; L.dint_dump_log.argtypes = [vp, vp, C.POINTER(u64)]
    L.dint_log_entry_size.restype = u32; L.dint_log_entry_size.argtypes = [i32]
    L.dint_get_stats.restype = i32; L.dint_get_stats.argtypes = [vp, C.POINTER(DintStats)]
    L.dint_reset_stats.restype = None; L.dint_reset_stats.argtypes = [vp]
    L.dint_profile.restype = i32; L.dint_profile.argtypes = [vp, i32]
    L.dint_kernel_times.restype = i32; L.dint_kernel_times.argtypes = [vp, C.POINTER(DintKernelTime), i32]
    L.dint_last_error.restype = C.c_char_p; L.dint_last_error.argtypes = []
    L.dint_host_alloc.restype = vp; L.dint_host_alloc.argtypes = [C.c_size_t]
    L.dint_host_free.restype = None; L.dint_host_free.argtypes = [vp]
    L.dint_test_fasthash64.restype = u64; L.dint_test_fasthash64.argtypes = [u64, i32]
    L.dint_test_fastmod.restype = u32; L.dint_test_fastmod.argtypes = [u64, u32]
    L.dint_test_rebuild_source.restype = i32; L.dint_test_rebuild_source.argtypes = [u64, u32, u32]
    L.dint_test_txn_reshard_dests.restype = u32; L.dint_test_txn_reshard_dests.argtypes = [u64, u32, u32, u32]
    _lib = L
    return L


class DintError(RuntimeError):
    def __init__(self, code, what):
        msg = lib().dint_last_error().decode(errors="replace")
        super().__init__(f"{what}: error {code} ({msg})")
        self.code = code


def default_cfg(kind, **over):
    """dint_default_cfg() with fields overridden by name; lock_holder_keys=True sets DINT_CFG_LOCK_HOLDER_KEYS;
    store_ebpf="wb_bloom" | "wb" | "wt" (or None) sets the DINT_CFG_STORE_EBPF_* variant; tatp_ebpf=True sets
    DINT_CFG_TATP_EBPF; smallbank_ebpf=True sets DINT_CFG_SMALLBANK_EBPF."""
    cfg = DintCfg()
    lib().dint_default_cfg(kind, C.byref(cfg))
    for k, v in over.items():
        if k == "kv_capacity_log2":
            for i, x in enumerate(v):
                cfg.kv_capacity_log2[i] = x
        elif k == "lock_holder_keys":
            if v:
                cfg.flags |= DINT_CFG_LOCK_HOLDER_KEYS
        elif k == "tatp_ebpf":
            if v:
                cfg.flags |= DINT_CFG_TATP_EBPF
        elif k == "smallbank_ebpf":
            if v:
                cfg.flags |= DINT_CFG_SMALLBANK_EBPF
        elif k == "store_ebpf":
            if v is not None:
                if v not in STORE_EBPF_VARIANTS:
                    raise ValueError(f"store_ebpf must be one of {sorted(STORE_EBPF_VARIANTS)}, not {v!r}")
                cfg.flags = (cfg.flags & ~DINT_CFG_STORE_EBPF_MASK) | STORE_EBPF_VARIANTS[v]
        else:
            setattr(cfg, k, v)
    return cfg


IMAGE_HEADER_BYTES = 144          # include/dint_b200.h, "State images"
CLUSTER_MANIFEST_BYTES = 104


def read_image_header(path):
    """The header of a state image (or, for a directory, of its cluster manifest): kind, cfg, and for a file the
    saved KV capacities and region count."""
    if os.path.isdir(path):
        with open(os.path.join(path, "manifest"), "rb") as f:
            b = f.read(CLUSTER_MANIFEST_BYTES)
        kind, shards = np.frombuffer(b, "<u4", 2, 12)
        return {"magic": b[:8], "kind": int(kind), "shards": int(shards), "cfg": DintCfg.from_buffer_copy(b, 24)}
    with open(path, "rb") as f:
        b = f.read(IMAGE_HEADER_BYTES)
    version, kind = np.frombuffer(b, "<u4", 2, 8)
    return {"magic": b[:8], "version": int(version), "kind": int(kind), "cfg": DintCfg.from_buffer_copy(b, 16),
            "n_regions": int(np.frombuffer(b, "<u4", 1, 92)[0]), "kv_capacity": [int(x) for x in np.frombuffer(b, "<u8", 5, 96)]}


def reshard_times():
    """Seconds spent by this thread's last GpuCluster.reshard: wall, re-shard kernels (CUDA events), key count +
    allocation of the destination (dint_reshard_times)."""
    out = (C.c_double * 3)()
    lib().dint_reshard_times(out)
    return {"wall_s": out[0], "kernel_s": out[1], "count_alloc_s": out[2]}


def rebuild_times():
    """Seconds spent by this thread's last rebuild (GpuCluster.rebuild, or GpuCluster.open_image with rebuild=True): wall,
    rebuild kernels (CUDA events), row count + allocation of the new engines (dint_rebuild_times)."""
    out = (C.c_double * 3)()
    lib().dint_rebuild_times(out)
    return {"wall_s": out[0], "kernel_s": out[1], "count_alloc_s": out[2]}


def image_times():
    """Seconds spent by this thread's last image call: wall, pack / unpack kernels, copies, file (dint_image_times)."""
    out = (C.c_double * 4)()
    lib().dint_image_times(out)
    return {"wall_s": out[0], "kernel_s": out[1], "copy_s": out[2], "file_s": out[3]}


class PinnedBuffer:
    """Page-locked host buffer exposed as a numpy uint8 array (dint_host_alloc)."""

    def __init__(self, nbytes):
        self.nbytes = max(int(nbytes), 1)
        self.ptr = lib().dint_host_alloc(self.nbytes)
        if not self.ptr:
            raise MemoryError("dint_host_alloc failed")
        self.array = np.ctypeslib.as_array(C.cast(self.ptr, C.POINTER(C.c_uint8)), shape=(self.nbytes,))

    def close(self):
        if self.ptr:
            self.array = None
            lib().dint_host_free(self.ptr)
            self.ptr = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Engine:
    """One GPU-resident server of the given kind.

    submit() has the semantics of feeding the requests, in order, to ONE thread of the reference
    server and collecting its replies (see include/dint_b200.h).
    """

    def __init__(self, kind, device=0, populate=False, **cfg_over):
        self.kind = kind
        self.msg = MSG_SIZE[kind]
        self.cfg = default_cfg(kind, **cfg_over)
        self.device = device
        h = C.c_void_p()
        rc = lib().dint_create(kind, C.byref(self.cfg), device, C.byref(h))
        if rc != 0:
            raise DintError(rc, f"dint_create({KIND_NAMES[kind]})")
        self.h = h
        if populate:
            self.populate()

    def close(self):
        if getattr(self, "h", None):
            lib().dint_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    # -- population ------------------------------------------------------------------------------
    def populate(self):
        rc = lib().dint_populate(self.h)
        if rc != 0:
            raise DintError(rc, "dint_populate")

    def load(self, table, keys, vals):
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        vals = np.ascontiguousarray(vals, dtype=np.uint8)
        rc = lib().dint_load(self.h, table, keys.ctypes.data, vals.ctypes.data, keys.size)
        if rc != 0:
            raise DintError(rc, "dint_load")

    # -- request path ----------------------------------------------------------------------------
    def submit(self, req, out=None, check=True):
        """Host path: req is a uint8 array of n*msg bytes (or structured wire records)."""
        raw = np.ascontiguousarray(req).view(np.uint8).reshape(-1)
        n = raw.size // self.msg
        if raw.size != n * self.msg:
            raise ValueError("request buffer is not a whole number of wire records")
        if out is None:
            out = np.empty_like(raw)
        rc = lib().dint_submit(self.h, raw.ctypes.data, n, out.ctypes.data)
        if rc != 0 and (check or rc != DINT_EPROTO):
            raise DintError(rc, "dint_submit")
        return out

    def submit_device(self, req_ptr, n, resp_ptr, stream=0):
        """Device path: raw device pointers (16-byte aligned), asynchronous on `stream`."""
        rc = lib().dint_submit_device(self.h, C.c_void_p(req_ptr), n, C.c_void_p(resp_ptr),
                                      C.c_void_p(stream) if stream else None)
        if rc != 0:
            raise DintError(rc, "dint_submit_device")

    def submit_tensor(self, req, out=None, stream=None):
        """Device path on torch CUDA uint8 tensors; runs on the current torch stream by default."""
        import torch
        assert req.is_cuda and req.dtype == torch.uint8 and req.is_contiguous()
        n = req.numel() // self.msg
        if out is None:
            out = torch.empty_like(req)
        s = stream if stream is not None else torch.cuda.current_stream(req.device).cuda_stream
        self.submit_device(req.data_ptr(), n, out.data_ptr(), s)
        return out

    def route_owner(self, req, stream=None):
        """owner shard (uint8 CUDA tensor) of every wire record in the CUDA uint8 tensor `req`."""
        import torch
        n = req.numel() // self.msg
        owner = torch.empty(n, dtype=torch.uint8, device=req.device)
        s = stream if stream is not None else torch.cuda.current_stream(req.device).cuda_stream
        rc = lib().dint_route_owner(self.h, C.c_void_p(req.data_ptr()), n, C.c_void_p(owner.data_ptr()),
                                    C.c_void_p(s) if s else None)
        if rc != 0:
            raise DintError(rc, "dint_route_owner")
        return owner

    def route_partition(self, req, owner, n_shards):
        """Stable partition of the CUDA uint8 tensor `req` by `owner` (uint8 tensor): returns (sorted, perm, counts)."""
        import torch
        n = owner.numel()
        out = torch.empty_like(req)
        perm = torch.empty(n, dtype=torch.int32, device=req.device)
        counts = torch.empty(n_shards, dtype=torch.int32, device=req.device)
        s = torch.cuda.current_stream(req.device).cuda_stream
        rc = lib().dint_route_partition(self.h, C.c_void_p(req.data_ptr()), C.c_void_p(owner.data_ptr()), n, n_shards,
                                        C.c_void_p(out.data_ptr()), C.c_void_p(perm.data_ptr()), C.c_void_p(counts.data_ptr()),
                                        C.c_void_p(s) if s else None)
        if rc != 0:
            raise DintError(rc, "dint_route_partition")
        return out, perm, counts

    def route_state(self, n, device):
        """Buffers the dispatch fills for the combine: (owner uint8 [n], tilebase int32 [tiles * 8])."""
        import torch
        tr = lib().dint_route_tile_records(self.h)
        tiles = (n + tr - 1) // tr
        return (torch.empty(max(n, 1), dtype=torch.uint8, device=device),
                torch.empty(max(tiles, 1) * 8, dtype=torch.int32, device=device))

    def route_dispatch(self, req, n, n_shards, rank, cap, slab_ptrs, flags, owner_in=None, sig_ptrs=None, epoch=0, state=None,
                       stream=None):
        """Fused stable partition of n records into per-shard slabs (see dint_route_dispatch).  slab_ptrs /
        sig_ptrs: DintPeerPtrs; flags: int32 CUDA tensor (>= 2).  Returns the (owner, tilebase) state."""
        import torch
        if state is None:
            state = self.route_state(n, req.device)
        s = stream if stream is not None else torch.cuda.current_stream(req.device).cuda_stream
        rc = lib().dint_route_dispatch(self.h, C.c_void_p(req.data_ptr()), C.c_void_p(owner_in.data_ptr()) if owner_in is not None else None,
                                       n, n_shards, rank, cap, C.byref(slab_ptrs), C.byref(sig_ptrs) if sig_ptrs is not None else None,
                                       epoch, C.c_void_p(state[0].data_ptr()), C.c_void_p(state[1].data_ptr()),
                                       C.c_void_p(flags.data_ptr()), C.c_void_p(s) if s else None)
        if rc != 0:
            raise DintError(rc, "dint_route_dispatch")
        return state

    def route_combine(self, reply_ptrs, state, n, n_shards, cap, out, stream=None):
        import torch
        s = stream if stream is not None else torch.cuda.current_stream(out.device).cuda_stream
        rc = lib().dint_route_combine(self.h, C.byref(reply_ptrs), C.c_void_p(state[0].data_ptr()), C.c_void_p(state[1].data_ptr()),
                                      n, n_shards, cap, C.c_void_p(out.data_ptr()), C.c_void_p(s) if s else None)
        if rc != 0:
            raise DintError(rc, "dint_route_combine")
        return out

    @staticmethod
    def slab_ptrs(base_ptr, n_shards, stride_bytes):
        """DintPeerPtrs for slabs laid out back to back in one local buffer."""
        return DintPeerPtrs.of([base_ptr + o * stride_bytes for o in range(n_shards)])

    def route_unpermute(self, sorted_resp, perm, out=None):
        import torch
        n = perm.numel()
        if out is None:
            out = torch.empty_like(sorted_resp)     # pass `out` (n_original * msg bytes) when perm has padding slots
        s = torch.cuda.current_stream(sorted_resp.device).cuda_stream
        rc = lib().dint_route_unpermute(self.h, C.c_void_p(sorted_resp.data_ptr()), C.c_void_p(perm.data_ptr()), n,
                                        C.c_void_p(out.data_ptr()), C.c_void_p(s) if s else None)
        if rc != 0:
            raise DintError(rc, "dint_route_unpermute")
        return out

    def snapshot(self):
        """Device-to-device copy of the whole server state; returns a handle for restore()."""
        h = C.c_void_p()
        rc = lib().dint_snapshot_create(self.h, C.byref(h))
        if rc != 0:
            raise DintError(rc, "dint_snapshot_create")
        return h

    def restore(self, snap, stream=None):
        """Asynchronous on the current torch stream (or `stream`): order it between submit calls."""
        if stream is None:
            import torch
            stream = torch.cuda.current_stream().cuda_stream
        rc = lib().dint_snapshot_restore(snap, C.c_void_p(stream) if stream else None)
        if rc != 0:
            raise DintError(rc, "dint_snapshot_restore")

    def free_snapshot(self, snap):
        lib().dint_snapshot_destroy(snap)

    def save_image(self, path):
        """Write the whole server state to the image file `path` (dint_image_save; waits for the engine to be idle)."""
        rc = lib().dint_image_save(self.h, os.fsencode(path))
        if rc != 0:
            raise DintError(rc, f"dint_image_save({path})")

    @classmethod
    def open_image(cls, path, device=0):
        """A new engine on `device` holding the state saved in the image file `path` (dint_image_open)."""
        h = C.c_void_p()
        rc = lib().dint_image_open(os.fsencode(path), device, C.byref(h))
        if rc != 0:
            raise DintError(rc, f"dint_image_open({path})")
        hdr = read_image_header(path)
        e = cls.__new__(cls)
        e.kind, e.msg, e.cfg, e.device, e.h = hdr["kind"], MSG_SIZE[hdr["kind"]], hdr["cfg"], device, h
        return e

    def sync(self, check=True):
        rc = lib().dint_sync(self.h)
        if rc != 0 and (check or rc != DINT_EPROTO):
            raise DintError(rc, "dint_sync")
        return rc

    # -- inspection ------------------------------------------------------------------------------
    def kv_get(self, table, key):
        val = (C.c_uint8 * 40)()
        ver = C.c_uint32(0)
        rc = lib().dint_kv_get(self.h, table, key, val, C.byref(ver))
        if rc < 0:
            raise DintError(rc, "dint_kv_get")
        return None if rc == 1 else (bytes(val), ver.value)

    def kv_count(self, table):
        return lib().dint_kv_count(self.h, table)

    def store_cache_set(self, bucket):
        """store with store_ebpf: cache set `bucket` as the reference's struct cache_entry (232 uint8; lock = 0)."""
        out = np.zeros(STORE_CACHE_ENTRY_BYTES, dtype=np.uint8)
        rc = lib().dint_store_cache_set(self.h, bucket, out.ctypes.data)
        if rc != 0:
            raise DintError(rc, "dint_store_cache_set")
        return out

    def store_cache_stats(self):
        """store with store_ebpf: the tier's counters since create, keyed by STORE_CACHE_STATS."""
        out = (C.c_uint64 * 5)()
        rc = lib().dint_store_cache_stats(self.h, out)
        if rc != 0:
            raise DintError(rc, "dint_store_cache_stats")
        return {k: int(out[i]) for i, k in enumerate(STORE_CACHE_STATS)}

    def tatp_cache_set(self, table, bucket):
        """tatp with tatp_ebpf: cache set `bucket` of `table` as the reference's struct cache_entry (232 uint8)."""
        out = np.zeros(STORE_CACHE_ENTRY_BYTES, dtype=np.uint8)
        rc = lib().dint_tatp_cache_set(self.h, table, bucket, out.ctypes.data)
        if rc != 0:
            raise DintError(rc, "dint_tatp_cache_set")
        return out

    def tatp_chain(self, table, bucket, max_entries=64):
        """tatp with tatp_ebpf: the chained table's entries of `bucket` of `table`, head first (TATP_CHAIN_REC)."""
        out = np.zeros(max_entries, dtype=TATP_CHAIN_REC)
        n = C.c_uint32(0)
        rc = lib().dint_tatp_chain(self.h, table, bucket, out.ctypes.data, max_entries, C.byref(n))
        if rc != 0:
            raise DintError(rc, "dint_tatp_chain")
        if n.value > max_entries:
            return self.tatp_chain(table, bucket, n.value)
        return out[:n.value]

    def tatp_cache_stats(self):
        """tatp with tatp_ebpf: the tier's counters since create, keyed by TATP_CACHE_STATS."""
        out = (C.c_uint64 * 9)()
        rc = lib().dint_tatp_cache_stats(self.h, out)
        if rc != 0:
            raise DintError(rc, "dint_tatp_cache_stats")
        return {k: int(out[i]) for i, k in enumerate(TATP_CACHE_STATS)}

    def smallbank_cache_set(self, table, bucket):
        """smallbank with smallbank_ebpf: cache set `bucket` of `table` as the reference's struct cache_entry (96 uint8)."""
        out = np.zeros(SMALLBANK_CACHE_ENTRY_BYTES, dtype=np.uint8)
        rc = lib().dint_smallbank_cache_set(self.h, table, bucket, out.ctypes.data)
        if rc != 0:
            raise DintError(rc, "dint_smallbank_cache_set")
        return out

    def smallbank_cache_stats(self):
        """smallbank with smallbank_ebpf: the tier's counters since create, keyed by SMALLBANK_CACHE_STATS."""
        out = (C.c_uint64 * 4)()
        rc = lib().dint_smallbank_cache_stats(self.h, out)
        if rc != 0:
            raise DintError(rc, "dint_smallbank_cache_stats")
        return {k: int(out[i]) for i, k in enumerate(SMALLBANK_CACHE_STATS)}

    def lock_slot(self, table, key):
        return lib().dint_lock_slot(self.h, table, key)

    def lock_state(self, table, slot):
        out = (C.c_uint32 * 2)()
        rc = lib().dint_lock_state(self.h, table, slot, out)
        if rc != 0:
            raise DintError(rc, "dint_lock_state")
        return out[0], out[1]

    def lock_holder(self, table, slot):
        """tatp with lock_holder_keys: the key the last granted kAcquireLock left in the slot (stale once the slot is
        free)."""
        out = C.c_uint64(0)
        rc = lib().dint_lock_holder(self.h, table, slot, C.byref(out))
        if rc != 0:
            raise DintError(rc, "dint_lock_holder")
        return out.value

    def dump_log(self):
        es = LOG_ENTRY_SIZE[self.kind]
        n = self.cfg.log_ring
        out = np.zeros((n, es), dtype=np.uint8)
        appended = C.c_uint64(0)
        rc = lib().dint_dump_log(self.h, out.ctypes.data, C.byref(appended))
        if rc != 0:
            raise DintError(rc, "dint_dump_log")
        return out, appended.value

    def stats(self):
        s = DintStats()
        rc = lib().dint_get_stats(self.h, C.byref(s))
        if rc != 0:
            raise DintError(rc, "dint_get_stats")
        return {k: getattr(s, k) for k, _ in DintStats._fields_ if k != "reserved"}

    def reset_stats(self):
        lib().dint_reset_stats(self.h)

    PROF_CLASSIFY, PROF_LOG_SCAN, PROF_APPLY, PROF_ORDERED, PROF_LOAD = 1, 2, 4, 8, 16

    def profile(self, enable=True):
        """True/1 = time every kernel with CUDA events, False/0 = off, or a mask of Engine.PROF_*."""
        rc = lib().dint_profile(self.h, int(enable))
        if rc != 0:
            raise DintError(rc, "dint_profile")

    def kernel_times(self):
        arr = (DintKernelTime * 16)()
        k = lib().dint_kernel_times(self.h, arr, 16)
        return {arr[i].name.decode(): (arr[i].launches, arr[i].total_ms) for i in range(max(k, 0))}


class GpuClients:
    """Closed-loop clients resident on the GPU next to `engine` (dint_clients_*), of the engine's kind: lock_2pl,
    lock_fasst, log_server or store.  The keyword arguments are those of workloads.Workload, so one dict of them
    drives the GPU clients and the host clients alike."""

    def __init__(self, engine, n_clients, seed=20230, n_keys=24_000_000, zipf_theta=0.0, read_pct=80, set_pct=0,
                 store_subscribers=2_000_000, store_hot=False):
        self.engine, self.n, self.kind = engine, n_clients, engine.kind
        self.msg = MSG_SIZE[self.kind]
        cfg = DintClientsCfg(n_clients=n_clients, n_keys=n_keys, seed=seed, zipf_theta=zipf_theta, read_pct=read_pct,
                             set_pct=set_pct, store_subscribers=store_subscribers, store_hot=1 if store_hot else 0)
        h = C.c_void_p()
        rc = lib().dint_clients_create_cfg(engine.h, C.byref(cfg), C.byref(h))
        if rc != 0:
            raise DintError(rc, "dint_clients_create_cfg")
        self.h = h

    def run(self, rounds, stream=None):
        if stream is None:
            import torch
            stream = torch.cuda.current_stream().cuda_stream
        rc = lib().dint_clients_run(self.h, rounds, C.c_void_p(stream) if stream else None)
        if rc != 0:
            raise DintError(rc, "dint_clients_run")

    def stats(self):
        """the counters of workloads.Workload.stats(), under the same keys"""
        out = (C.c_uint64 * 6)()
        rc = lib().dint_clients_stats_all(self.h, out)
        if rc != 0:
            raise DintError(rc, "dint_clients_stats_all")
        keys = ["requests", "committed", "validation_aborts", "lock_rejects", "not_exist", "rounds"]
        return dict(zip(keys, [int(x) for x in out]))

    def peek(self):
        """(the requests the clients send next, the replies they absorbed last): uint8 arrays of n_clients * msg bytes"""
        rq = np.empty(self.n * self.msg, dtype=np.uint8)
        rs = np.empty(self.n * self.msg, dtype=np.uint8)
        rc = lib().dint_clients_peek(self.h, rq.ctypes.data, rs.ctypes.data)
        if rc != 0:
            raise DintError(rc, "dint_clients_peek")
        return rq, rs

    def close(self):
        if getattr(self, "h", None):
            lib().dint_clients_destroy(self.h)
            self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class GpuCluster:
    """G shard engines driven by ONE process (dint_cluster_*): the C-level multi-GPU server.  devices: CUDA ordinals,
    all distinct (NVLink peer access) or all the same (several shards resident on one GPU)."""

    def __init__(self, kind, n_shards, devices=None, max_batch=0, populate=False, **cfg_over):
        self.kind, self.msg, self.G = kind, MSG_SIZE[kind], n_shards
        cfg = self.cfg = default_cfg(kind, **cfg_over)
        dv = (C.c_int * n_shards)(*devices) if devices is not None else None
        h = C.c_void_p()
        rc = lib().dint_cluster_create(kind, C.byref(cfg), n_shards, dv, max_batch, C.byref(h))
        if rc != 0:
            raise DintError(rc, f"dint_cluster_create({KIND_NAMES[kind]}, {n_shards})")
        self.h = h
        if populate:
            rc = lib().dint_cluster_populate(self.h)
            if rc != 0:
                raise DintError(rc, "dint_cluster_populate")

    def submit(self, req, dst=None, out=None, check=True):
        raw = np.ascontiguousarray(req).view(np.uint8).reshape(-1)
        n = raw.size // self.msg
        if out is None:
            out = np.empty_like(raw)
        d = None if dst is None else np.ascontiguousarray(dst, dtype=np.uint8)
        rc = lib().dint_cluster_submit(self.h, raw.ctypes.data, n, None if d is None else d.ctypes.data, out.ctypes.data)
        if rc != 0 and (check or rc != DINT_EPROTO):
            raise DintError(rc, "dint_cluster_submit")
        return out

    def overflow_retries(self):
        return int(lib().dint_cluster_overflow_retries(self.h))

    def save_image(self, path):
        """Write every shard's state to directory `path`: a manifest and one image per shard (dint_cluster_image_save)."""
        rc = lib().dint_cluster_image_save(self.h, os.fsencode(path))
        if rc != 0:
            raise DintError(rc, f"dint_cluster_image_save({path})")

    @classmethod
    def open_image(cls, path, devices=None, max_batch=0, rebuild=False):
        """A new cluster holding the state saved in directory `path` (dint_cluster_image_open); one shard per entry of
        `devices` (default: as many shards as were saved, on devices 0..G-1).  rebuild=True (tatp / smallbank,
        dint_cluster_image_open_rebuild): a shard image that is missing, short or corrupt is rebuilt from the other
        shards' replicas, and `.rebuilt` lists the shards rebuilt.  To repair a directory, save the result to ANOTHER
        one: a save removes the manifest before it rewrites shards."""
        if not isinstance(rebuild, bool):
            raise TypeError("rebuild must be True or False")
        if devices is not None:
            n = len(devices)
        else:                                   # as many shards as were saved; an unreadable manifest is the C call's to refuse
            try:
                n = read_image_header(path)["shards"]
            except (OSError, ValueError):
                n = 0
        dv = (C.c_int * n)(*devices) if devices is not None else None
        h = C.c_void_p()
        mask = C.c_uint32(0)
        if rebuild:
            rc = lib().dint_cluster_image_open_rebuild(os.fsencode(path), n, dv, max_batch, C.byref(mask), C.byref(h))
        else:
            rc = lib().dint_cluster_image_open(os.fsencode(path), n, dv, max_batch, C.byref(h))
        if rc != 0:
            raise DintError(rc, f"dint_cluster_image_open{'_rebuild' if rebuild else ''}({path})")
        hdr = read_image_header(path)
        cl = cls.__new__(cls)
        cl.kind, cl.msg, cl.G, cl.cfg, cl.h = hdr["kind"], MSG_SIZE[hdr["kind"]], n, hdr["cfg"], h
        if rebuild:
            cl.rebuilt = [r for r in range(n) if (mask.value >> r) & 1]
        return cl

    def rebuild(self, shards):
        """Rebuild the listed shards of this tatp / smallbank cluster in place from the surviving replicas
        (dint_cluster_rebuild): each gets a new engine holding, for every key it replicates, the row of the key's
        surviving replica with the lowest role; lock state, the log ring and statistics start empty.  No GPU
        transaction clients may be attached.  On failure the cluster is unchanged."""
        if isinstance(shards, (int, np.integer)):
            raise TypeError("shards: a list of shard indices")
        shards = list(shards)
        if not shards or any(isinstance(s, bool) or not isinstance(s, (int, np.integer)) for s in shards):
            raise ValueError(f"shards: a non-empty list of shard indices, not {shards!r}")
        if len(set(shards)) != len(shards) or any(not 0 <= s < self.G for s in shards):
            raise ValueError(f"shards {shards}: distinct indices in [0, {self.G}) expected")
        mask = sum(1 << int(s) for s in shards)
        rc = lib().dint_cluster_rebuild(self.h, mask)
        if rc != 0:
            raise DintError(rc, f"dint_cluster_rebuild({KIND_NAMES[self.kind]}, shards {sorted(shards)})")

    def reshard(self, n_shards, devices=None, max_batch=0):
        """A new cluster of `n_shards` shards holding this one's state (dint_cluster_reshard): it answers every later
        request exactly as this one would.  lock_2pl / lock_fasst / store only; this cluster is not changed and stays
        usable.  devices / max_batch as for GpuCluster; peak device memory is both clusters."""
        dv = (C.c_int * n_shards)(*devices) if devices is not None else None
        h = C.c_void_p()
        rc = lib().dint_cluster_reshard(self.h, n_shards, dv, max_batch, C.byref(h))
        if rc != 0:
            raise DintError(rc, f"dint_cluster_reshard({KIND_NAMES[self.kind]}, {self.G} -> {n_shards})")
        cl = GpuCluster.__new__(GpuCluster)
        cl.kind, cl.msg, cl.G, cl.cfg, cl.h = self.kind, self.msg, n_shards, self.cfg, h
        return cl

    def reshard_txn(self, n_shards, devices=None, max_batch=0):
        """A new tatp / smallbank cluster of `n_shards` shards (1 or 3..8) on which every row sits on its replicas under
        the new placement, copied with its version from the key's old primary (dint_cluster_reshard_txn).  Lock state,
        the log ring and statistics start empty, and no lock may be held: drain the GpuTxnClients first.  This cluster
        is not changed and stays usable.  devices / max_batch as for GpuCluster; peak device memory is both clusters."""
        dv = (C.c_int * n_shards)(*devices) if devices is not None else None
        h = C.c_void_p()
        rc = lib().dint_cluster_reshard_txn(self.h, n_shards, dv, max_batch, C.byref(h))
        if rc != 0:
            raise DintError(rc, f"dint_cluster_reshard_txn({KIND_NAMES[self.kind]}, {self.G} -> {n_shards})")
        cl = GpuCluster.__new__(GpuCluster)
        cl.kind, cl.msg, cl.G, cl.cfg, cl.h = self.kind, self.msg, n_shards, self.cfg, h
        return cl

    def engine(self, shard):
        """A non-owning Engine view of one shard (state inspection)."""
        e = Engine.__new__(Engine)
        e.kind, e.msg, e.device, e.cfg = self.kind, self.msg, None, self.cfg
        e.h = C.c_void_p(lib().dint_cluster_engine(self.h, shard))
        e.close = lambda: None
        return e

    def close(self):
        if getattr(self, "h", None):
            lib().dint_cluster_destroy(self.h)
            self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class GpuTxnClients:
    """TATP or SmallBank closed-loop clients resident on the GPUs of `cluster` (a GpuCluster of that kind;
    dint_txn_clients_*): the state machines of TxnWorkload, draw for draw, with every round emitted on the devices
    and served by one exchange step.  subscribers: kSubscriberNum (tatp) or kAccountNum (smallbank) of the key
    generators, as in TxnWorkload -- it must match the servers' population.  Keep the cluster open while these
    clients exist."""

    def __init__(self, cluster, n_clients, subscribers=None, gid0=0):
        from .wire import TATP
        if subscribers is None:
            subscribers = 7_000_000 if cluster.kind == TATP else 24_000_000
        self.cluster, self.kind, self.msg, self.n = cluster, cluster.kind, cluster.msg, n_clients
        h = C.c_void_p()
        rc = lib().dint_txn_clients_create(cluster.h, n_clients, gid0, subscribers, C.byref(h))
        if rc != 0:
            raise DintError(rc, "dint_txn_clients_create")
        self.h = h

    def run(self, rounds, check=True):
        """Serve `rounds` closed-loop rounds; returns when they are served."""
        rc = lib().dint_txn_clients_run(self.h, rounds)
        if rc != 0 and (check or rc != DINT_EPROTO):
            raise DintError(rc, "dint_txn_clients_run")
        return rc

    def stats(self):
        """TxnWorkload.stats()'s dict (requests and rounds count what was served) plus fallback_rounds, the rounds
        served in pieces because they did not fit the cluster's slabs or batch size."""
        from .txn_workloads import SMALLBANK_TXN_NAMES, TATP_TXN_NAMES
        from .wire import TATP
        out = (C.c_uint64 * 19)()
        rc = lib().dint_txn_clients_stats(self.h, out)
        if rc != 0:
            raise DintError(rc, "dint_txn_clients_stats")
        d = {"requests": int(out[0]), "txns": int(out[1]), "committed": int(out[2]), "rounds": int(out[3])}
        names = TATP_TXN_NAMES if self.kind == TATP else SMALLBANK_TXN_NAMES
        d["by_type"] = {n: (int(out[4 + i]), int(out[11 + i])) for i, n in enumerate(names)}
        d["fallback_rounds"] = int(out[18])
        return d

    def lock_stats(self):
        """TxnWorkload.lock_stats()'s dict, counted on the devices."""
        out = (C.c_uint64 * 3)()
        rc = lib().dint_txn_clients_lock_stats(self.h, out)
        if rc != 0:
            raise DintError(rc, "dint_txn_clients_lock_stats")
        return {"locks": int(out[0]), "reject_sharing": int(out[1]), "reject_same_key": int(out[2])}

    def peek(self):
        """(next_req, next_dst, last_resp) in global client order: the pending round's requests and destination
        shards, and the replies the clients absorbed last."""
        cap = self.n * 9
        rq = np.empty(cap * self.msg, dtype=np.uint8)
        dst = np.empty(cap, dtype=np.uint8)
        rs = np.empty(cap * self.msg, dtype=np.uint8)
        nn, nl = C.c_uint64(), C.c_uint64()
        rc = lib().dint_txn_clients_peek(self.h, rq.ctypes.data, dst.ctypes.data, C.byref(nn), rs.ctypes.data, C.byref(nl))
        if rc != 0:
            raise DintError(rc, "dint_txn_clients_peek")
        return rq[: nn.value * self.msg], dst[: nn.value], rs[: nl.value * self.msg]

    def drain(self, max_rounds=64):
        """Serve rounds until every client has finished the transaction it was in and started no new one; returns the
        rounds served (dint_txn_clients_drain).  The clients stay idle until the next run(), peek() or stats(), which
        resumes them, possibly on another cluster (rebind)."""
        n = C.c_uint32(0)
        rc = lib().dint_txn_clients_drain(self.h, max_rounds, C.byref(n))
        if rc != 0:
            raise DintError(rc, "dint_txn_clients_drain")
        return int(n.value)

    def rebind(self, cluster):
        """Move drained clients (or clients that have never run) to `cluster`, a GpuCluster of the same kind (e.g. from
        GpuCluster.reshard_txn): each client's state and the counters carry over (dint_txn_clients_rebind).  The old
        cluster may then be closed."""
        rc = lib().dint_txn_clients_rebind(self.h, cluster.h)
        if rc != 0:
            raise DintError(rc, "dint_txn_clients_rebind")
        self.cluster = cluster

    def times(self):
        """Rounds timed by run(), their host wall time and the CUDA-event time of their device work (rank 0), in s."""
        out = (C.c_double * 3)()
        rc = lib().dint_txn_clients_times(self.h, out)
        if rc != 0:
            raise DintError(rc, "dint_txn_clients_times")
        return {"rounds": int(out[0]), "wall_s": out[1], "device_s": out[2]}

    def close(self):
        if getattr(self, "h", None):
            lib().dint_txn_clients_destroy(self.h)
            self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class GpuClusterClients:
    """lock_2pl, lock_fasst, store or log_server closed-loop clients resident on the GPUs of `cluster` (a GpuCluster of
    that kind; dint_cluster_clients_*): GpuClients' state machines, split over the ranks in contiguous blocks, every
    round served by one exchange step.  The keyword arguments are those of GpuClients and workloads.Workload, and the
    clients send and absorb, round for round, what GpuClients with the same clients on one engine would.  Keep the
    cluster open while these clients exist."""

    def __init__(self, cluster, n_clients, seed=20230, n_keys=24_000_000, zipf_theta=0.0, read_pct=80, set_pct=0,
                 store_subscribers=2_000_000, store_hot=False):
        self.cluster, self.n, self.kind, self.msg = cluster, n_clients, cluster.kind, cluster.msg
        cfg = DintClientsCfg(n_clients=n_clients, n_keys=n_keys, seed=seed, zipf_theta=zipf_theta, read_pct=read_pct,
                             set_pct=set_pct, store_subscribers=store_subscribers, store_hot=1 if store_hot else 0)
        h = C.c_void_p()
        rc = lib().dint_cluster_clients_create(cluster.h, C.byref(cfg), C.byref(h))
        if rc != 0:
            raise DintError(rc, "dint_cluster_clients_create")
        self.h = h

    def run(self, rounds, check=True):
        """Serve `rounds` closed-loop rounds; returns when they are served."""
        rc = lib().dint_cluster_clients_run(self.h, rounds)
        if rc != 0 and (check or rc != DINT_EPROTO):
            raise DintError(rc, "dint_cluster_clients_run")
        return rc

    def stats(self):
        """GpuClients.stats()'s dict (rounds counted once, not once per rank) plus fallback_rounds, the rounds served
        in pieces because some (rank, shard) count exceeded the cluster's slab capacity."""
        out = (C.c_uint64 * 7)()
        rc = lib().dint_cluster_clients_stats(self.h, out)
        if rc != 0:
            raise DintError(rc, "dint_cluster_clients_stats")
        keys = ["requests", "committed", "validation_aborts", "lock_rejects", "not_exist", "rounds", "fallback_rounds"]
        return dict(zip(keys, [int(x) for x in out]))

    def peek(self):
        """(the requests the clients send next, the replies they absorbed last) in global client order: uint8 arrays of
        n_clients * msg bytes"""
        rq = np.empty(self.n * self.msg, dtype=np.uint8)
        rs = np.empty(self.n * self.msg, dtype=np.uint8)
        rc = lib().dint_cluster_clients_peek(self.h, rq.ctypes.data, rs.ctypes.data)
        if rc != 0:
            raise DintError(rc, "dint_cluster_clients_peek")
        return rq, rs

    def rebind(self, cluster):
        """Move the clients to `cluster`, a GpuCluster of the same kind (e.g. from GpuCluster.reshard): their state, the
        pending round and the counters carry over (dint_cluster_clients_rebind).  The old cluster may then be closed."""
        rc = lib().dint_cluster_clients_rebind(self.h, cluster.h)
        if rc != 0:
            raise DintError(rc, "dint_cluster_clients_rebind")
        self.cluster = cluster

    def times(self):
        """Rounds timed by run(), their host wall time and the CUDA-event time of their device work (rank 0), in s."""
        out = (C.c_double * 3)()
        rc = lib().dint_cluster_clients_times(self.h, out)
        if rc != 0:
            raise DintError(rc, "dint_cluster_clients_times")
        return {"rounds": int(out[0]), "wall_s": out[1], "device_s": out[2]}

    def close(self):
        if getattr(self, "h", None):
            lib().dint_cluster_clients_destroy(self.h)
            self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
