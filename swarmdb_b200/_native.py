"""ctypes binding of the C ABI in include/swarmdb_b200.h (the drop-in boundary).

`Shard` is one GPU-resident queue shard (one handle, one GPU).  There is no CPU
implementation behind it: if the CUDA library is missing or no device is present, loading /
construction fails loudly - it never falls back.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path
from typing import Optional, Tuple

import numpy as np

_CSRC = Path(__file__).resolve().parent / "csrc"
LIB_PATH = _CSRC / "libswarmdb_b200.so"

LOAD_DTYPE = np.dtype([("received", "<u4"), ("pending", "<u4"), ("pending_by_prio", "<u4", (4,)), ("pending_granules", "<u4"),
                       ("reserved", "<u4")])
QSTATS_FIELDS = ["agents_with_pending", "pending", "p0", "p1", "p2", "p3", "pending_granules", "received", "max_pending",
                 "max_pending_agent"]
HDR_DTYPE = np.dtype([("seq", "<u8"), ("timestamp", "<f8"), ("sender", "<u4"), ("receiver", "<u4"),
                      ("group", "<u4"), ("len", "<u2"), ("prio", "u1"), ("type", "u1")])
assert HDR_DTYPE.itemsize == 32
# compact receive format (sdb_recv_entry / sdb_recv_send): one entry per record, one row per distinct payload image
ENTRY_DTYPE = np.dtype([("seq", "<u8"), ("send", "<u4"), ("receiver", "<u4")])
SEND_DTYPE = np.dtype([("timestamp", "<f8"), ("payload_off", "<u8"), ("sender", "<u4"), ("group", "<u4"),
                       ("len", "<u2"), ("prio", "u1"), ("type", "u1"), ("reserved", "<u4")])
assert ENTRY_DTYPE.itemsize == 16 and SEND_DTYPE.itemsize == 32
# one exported lease (sdb_lease_meta): its id on the exporting handle, deadline, agent, delivery count and state
META_DTYPE = np.dtype([("id", "<u8"), ("deadline", "<f8"), ("agent", "<u4"), ("deliveries", "<u4"), ("state", "<u4"),
                       ("reserved", "<u4")])
assert META_DTYPE.itemsize == 32
LEASE_STATE_LIVE, LEASE_STATE_DEAD = 0, 3

NO_GROUP = 0xFFFFFFFF
NO_RECEIVER = 0xFFFFFFFF
RECV_PRIORITY = 1
RECV_PEEK = 2
RECV_ASYNC = 4
RECV_OWNED = 8
EXPIRE_ALL = 16
WHERE_DROP = 32
LEASE_ACK = 0                   # sdb_lease_settle ops
LEASE_RENEW = 1
LEASE_ALL = 1                   # sdb_lease_sweep flag: every live lease is due
FILTER_SENDER, FILTER_RECEIVER, FILTER_GROUP, FILTER_TYPE = 1, 2, 4, 8
FILTER_PRIO, FILTER_TIME, FILTER_SEQ, FILTER_KEYWORD, FILTER_ICASE, FILTER_IDS = 16, 32, 64, 128, 256, 512
FILTER_MAX_KEYWORD = 256
FILTER_MAX_IDS = 1 << 22
TYPEF_JSON = 0x08
TYPEF_EXTRAS = 0x10
TYPEF_SUPERSEDE = 0x20
TYPEF_TOKENS = 0x40
TYPE_MASK = 0x07

STATUS_NAMES = {0: "SDB_OK", -1: "SDB_EINVAL", -2: "SDB_ECUDA", -3: "SDB_ENOMEM", -4: "SDB_ERING_OVERFLOW",
                -5: "SDB_EARENA_FULL", -6: "SDB_ECAPACITY", -7: "SDB_ENOTFOUND", -8: "SDB_EOUTPUT"}


def shared_payload_enabled() -> bool:
    """Mirror of the library's SDB_SHARED_PAYLOAD switch (csrc/sdb_api.cu, sdb_create): group sends above the pull
    threshold keep ONE payload per send in the arena log instead of one per recipient."""
    return os.environ.get("SDB_SHARED_PAYLOAD", "1") != "0"


class SdbError(RuntimeError):
    def __init__(self, code: int, msg: str) -> None:
        super().__init__(f"{STATUS_NAMES.get(code, code)}: {msg}")
        self.code = code


class SdbConfig(C.Structure):
    _fields_ = [("struct_bytes", C.c_uint32), ("device", C.c_int32), ("shard_id", C.c_uint32),
                ("num_shards", C.c_uint32), ("max_agents", C.c_uint32), ("ring_slots", C.c_uint32),
                ("arena_bytes", C.c_uint64), ("max_payload_bytes", C.c_uint32), ("max_groups", C.c_uint32),
                ("member_pool_entries", C.c_uint64), ("max_backends", C.c_uint32), ("max_batch_sends", C.c_uint32),
                ("max_batch_payload", C.c_uint64), ("max_recv_records", C.c_uint64), ("max_recv_payload", C.c_uint64),
                ("list_pool_entries", C.c_uint64), ("fanout_variant", C.c_uint32), ("flags", C.c_uint32)]


class SdbFilter(C.Structure):
    """sdb_filter (include/swarmdb_b200.h): the clauses named in `fields` are ANDed; make_filter() builds one."""
    _fields_ = [("struct_bytes", C.c_uint32), ("fields", C.c_uint32), ("sender", C.c_uint32), ("receiver", C.c_uint32),
                ("group", C.c_uint32), ("type_mask", C.c_uint8), ("prio_mask", C.c_uint8), ("keyword_len", C.c_uint16),
                ("after", C.c_double), ("before", C.c_double), ("seq_lo", C.c_uint64), ("seq_hi", C.c_uint64),
                ("keyword", C.c_void_p), ("n_ids", C.c_uint64), ("ids", C.c_void_p), ("id_hits", C.c_void_p),
                ("id_agent", C.c_void_p)]


def make_filter(sender=None, receiver=None, group=None, types=None, prios=None, after=None, before=None, seq=None,
                keyword=None, icase=False, ids=None) -> SdbFilter:
    """A filter for Shard.receive_where.  Each argument that is not None adds its clause: sender / receiver / group are
    indices (NO_RECEIVER selects broadcast copies, NO_GROUP non-group sends); types / prios are iterables of type codes
    (0..7) and priorities (0..3); after / before bound the timestamp strictly (either may be None: unbounded); seq is a
    half-open range (lo, hi); keyword (bytes or str, UTF-8) must occur in the content bytes, ASCII case folded with
    icase; ids (an iterable of sequence numbers or a u64 array; duplicates allowed, empty matches nothing) selects the
    records whose seq is listed.  The keyword bytes and the id array are kept alive by the returned object."""
    f = SdbFilter()
    f.struct_bytes = C.sizeof(SdbFilter)
    fields = 0
    if sender is not None:
        fields |= FILTER_SENDER; f.sender = int(sender)
    if receiver is not None:
        fields |= FILTER_RECEIVER; f.receiver = int(receiver)
    if group is not None:
        fields |= FILTER_GROUP; f.group = int(group)
    if types is not None:
        fields |= FILTER_TYPE; f.type_mask = sum(1 << (int(t) & TYPE_MASK) for t in set(types))
    if prios is not None:
        fields |= FILTER_PRIO; f.prio_mask = sum(1 << int(p) for p in set(prios))
    if after is not None or before is not None:
        fields |= FILTER_TIME
        f.after = float("-inf") if after is None else float(after)
        f.before = float("inf") if before is None else float(before)
    if seq is not None:
        fields |= FILTER_SEQ; f.seq_lo, f.seq_hi = int(seq[0]), int(seq[1])
    if keyword is not None:
        kw = keyword.encode("utf-8") if isinstance(keyword, str) else bytes(keyword)
        fields |= FILTER_KEYWORD
        f._kw = C.create_string_buffer(kw, max(len(kw), 1))
        f.keyword = C.cast(f._kw, C.c_void_p)
        f.keyword_len = len(kw) if len(kw) <= 0xFFFF else 0xFFFF
    if icase:
        fields |= FILTER_ICASE
    if ids is not None:
        a = ids if isinstance(ids, np.ndarray) else np.fromiter((int(x) for x in ids), np.uint64)
        f._ids = np.ascontiguousarray(a, np.uint64)
        if f._ids.ndim != 1:
            raise ValueError("ids must be one-dimensional")
        fields |= FILTER_IDS
        f.n_ids = len(f._ids)
        f.ids = f._ids.ctypes.data                                 # never NULL: the library refuses NULL ids
    f.fields = fields
    return f


class SdbStats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("next_seq", "enqueued", "delivered", "ring_overflow", "skipped_sender",
                                          "arena_tail_bytes", "arena_floor_bytes", "n_agents", "kernel_launches",
                                          "backend_picks")]


class SdbLeaseSummary(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("live", "acked_unreclaimed", "redelivered_total", "acked_total", "entries_used",
                                          "entries_reserved", "payload_used", "payload_reserved")]


class SdbLeasePolicySummary(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("max_deliveries", "dead", "dead_total", "ledger_used", "ledger_cap",
                                          "held_by_ledger_total")]


class SdbDedupSummary(C.Structure):
    _fields_ = [("capacity", C.c_uint64), ("live", C.c_uint64), ("used", C.c_uint64), ("window", C.c_double)] + \
        [(n, C.c_uint64) for n in ("accepted_total", "duplicate_total", "expired_total", "forgotten_total", "rebuilds")]


DEDUP_CONTENT = 1
KEY_DTYPE = np.dtype([("lo", "<u8"), ("hi", "<u8")])     # sdb_dedup_key; {0,0}: not deduplicated


class SdbRelocateSummary(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("agents", "records", "moved_bytes", "skipped_bytes", "floor_before", "floor_after",
                                          "tail_after")]


EXPORTS = ["sdb_abi_version", "sdb_create", "sdb_destroy", "sdb_set_stream", "sdb_sync", "sdb_last_error",
           "sdb_get_stats", "sdb_debug_set_arena_pos", "sdb_advance_seq", "sdb_profile", "sdb_profile_read", "sdb_profile_read_n", "sdb_register_agents", "sdb_deregister_agents", "sdb_create_group", "sdb_send_batch",
           "sdb_send_group_batch", "sdb_send_list_batch", "sdb_send_mixed_batch", "sdb_stage_batch", "sdb_submit_staged", "sdb_free_staged",
           "sdb_receive_batch", "sdb_receive_compact", "sdb_receive_budget", "sdb_receive_compact_budget", "sdb_receive_tokens", "sdb_receive_compact_tokens", "sdb_pending_tokens", "sdb_restore_compact", "sdb_expire", "sdb_trim", "sdb_supersede", "sdb_receive_where", "sdb_receive_where_budget", "sdb_latency_server", "sdb_last_receive_dev", "sdb_last_receive_totals",
           "sdb_digest_reset", "sdb_digest_fold", "sdb_digest_read", "sdb_wire_bytes", "sdb_set_agent_shards",
           "sdb_export_group_batch", "sdb_export_mixed_batch", "sdb_export_mixed_batch_seq", "sdb_import_wire_batches", "sdb_wire_alloc", "sdb_wire_open",
           "sdb_wire_close", "sdb_import_wire_ptrs", "sdb_wire_wait_done", "sdb_wire_publish", "sdb_import_wire_ptrs_async", "sdb_import_prefetch", "sdb_overflow_log", "sdb_set_backends", "sdb_get_backend_loads",
           "sdb_release_backends", "sdb_select_backend_batch", "sdb_agent_loads", "sdb_queue_stats",
           "sdb_assign_agent_backends", "sdb_backend_loads_from_queues", "sdb_lease_reserve", "sdb_receive_leased", "sdb_receive_leased_select",
           "sdb_lease_settle", "sdb_lease_sweep", "sdb_lease_stats", "sdb_lease_set_policy", "sdb_lease_deliveries",
           "sdb_lease_dead_letters", "sdb_lease_policy_stats", "sdb_arena_relocate", "sdb_lease_export",
           "sdb_lease_import", "sdb_lease_ledger_export", "sdb_lease_ledger_import", "sdb_dedup_reserve",
           "sdb_send_mixed_batch_dedup", "sdb_dedup_forget", "sdb_dedup_stats"]

_lib = None


def _keys(keys, n: Optional[int]) -> np.ndarray:
    """Keys as a contiguous KEY_DTYPE array: from KEY_DTYPE or an (n, 2) array of (lo, hi)."""
    k = np.asarray(keys)
    if k.dtype != KEY_DTYPE:
        k = np.ascontiguousarray(np.asarray(keys, np.uint64).reshape(-1, 2)).view(KEY_DTYPE).reshape(-1)
    k = np.ascontiguousarray(k)
    if n is not None and len(k) != n:
        raise ValueError(f"{len(k)} keys for {n} sends")
    return k


def load_library() -> C.CDLL:
    """dlopen the in-tree CUDA library.  Raises if it has not been built (no fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    path = Path(os.environ.get("SWARMDB_B200_LIB", str(LIB_PATH)))
    if not path.exists():
        raise ImportError(f"{path} not built - run `python -c 'import __graft_entry__ as g; g.build()'` "
                          f"(or make -C swarmdb_b200/csrc). swarmdb_b200 has no CPU fallback.")
    L = C.CDLL(str(path))
    vp, u32, u64, i32 = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int
    L.sdb_abi_version.restype = i32
    L.sdb_create.restype = i32; L.sdb_create.argtypes = [C.POINTER(SdbConfig), C.POINTER(vp)]
    L.sdb_destroy.restype = i32; L.sdb_destroy.argtypes = [vp]
    L.sdb_set_stream.restype = i32; L.sdb_set_stream.argtypes = [vp, vp]
    L.sdb_sync.restype = i32; L.sdb_sync.argtypes = [vp]
    L.sdb_last_error.restype = C.c_char_p; L.sdb_last_error.argtypes = [vp]
    L.sdb_get_stats.restype = i32; L.sdb_get_stats.argtypes = [vp, C.POINTER(SdbStats)]
    L.sdb_debug_set_arena_pos.restype = i32; L.sdb_debug_set_arena_pos.argtypes = [vp, u64]
    L.sdb_advance_seq.restype = i32; L.sdb_advance_seq.argtypes = [vp, u64]
    L.sdb_profile.restype = i32; L.sdb_profile.argtypes = [vp, i32]
    L.sdb_profile_read.restype = i32; L.sdb_profile_read.argtypes = [vp, vp, vp]
    L.sdb_profile_read_n.restype = i32; L.sdb_profile_read_n.argtypes = [vp, u32, vp, vp]
    L.sdb_register_agents.restype = i32; L.sdb_register_agents.argtypes = [vp, u32, vp]
    L.sdb_deregister_agents.restype = i32; L.sdb_deregister_agents.argtypes = [vp, u32, vp]
    L.sdb_create_group.restype = i32; L.sdb_create_group.argtypes = [vp, u32, u32, vp]
    L.sdb_send_batch.restype = i32; L.sdb_send_batch.argtypes = [vp, u32] + [vp] * 7 + [u64, vp, vp]
    L.sdb_send_group_batch.restype = i32; L.sdb_send_group_batch.argtypes = [vp, u32] + [vp] * 7 + [u64, vp, vp]
    L.sdb_send_list_batch.restype = i32; L.sdb_send_list_batch.argtypes = [vp, u32] + [vp] * 8 + [u64, vp, vp]
    L.sdb_send_mixed_batch.restype = i32
    L.sdb_send_mixed_batch.argtypes = [vp, u32, vp, vp, vp, u32] + [vp] * 7 + [u64, vp, vp]
    L.sdb_send_mixed_batch_dedup.restype = i32
    L.sdb_send_mixed_batch_dedup.argtypes = [vp, u32, vp, vp, vp, u32] + [vp] * 7 + [u64, vp, vp, u32, C.c_double, vp, vp, vp, vp]
    L.sdb_dedup_reserve.restype = i32; L.sdb_dedup_reserve.argtypes = [vp, u64, C.c_double]
    L.sdb_dedup_forget.restype = i32; L.sdb_dedup_forget.argtypes = [vp, u64, vp, vp]
    L.sdb_dedup_stats.restype = i32; L.sdb_dedup_stats.argtypes = [vp, C.POINTER(SdbDedupSummary)]
    L.sdb_stage_batch.restype = i32; L.sdb_stage_batch.argtypes = [vp, u32, u32] + [vp] * 7 + [u64, vp, C.POINTER(vp)]
    L.sdb_submit_staged.restype = i32; L.sdb_submit_staged.argtypes = [vp, vp, vp]
    L.sdb_free_staged.restype = i32; L.sdb_free_staged.argtypes = [vp, vp]
    L.sdb_receive_batch.restype = i32
    L.sdb_receive_batch.argtypes = [vp, u32, vp, u32, u32, vp, vp, u64, vp, u64, vp, vp]
    L.sdb_receive_compact.restype = i32
    L.sdb_receive_compact.argtypes = [vp, u32, vp, u32, u32, vp, vp, u64, vp, u64, vp, u64, vp, vp, vp]
    L.sdb_receive_budget.restype = i32
    L.sdb_receive_budget.argtypes = [vp, u32, vp, u32, u64, u32, vp, vp, u64, vp, u64, vp, vp]
    L.sdb_receive_compact_budget.restype = i32
    L.sdb_receive_compact_budget.argtypes = [vp, u32, vp, u32, u64, u32, vp, vp, u64, vp, u64, vp, u64, vp, vp, vp]
    L.sdb_receive_tokens.restype = i32
    L.sdb_receive_tokens.argtypes = [vp, u32, vp, u32, u64, u64, u32, vp, vp, u64, vp, u64, vp, vp]
    L.sdb_receive_compact_tokens.restype = i32
    L.sdb_receive_compact_tokens.argtypes = [vp, u32, vp, u32, u64, u64, u32, vp, vp, u64, vp, u64, vp, u64, vp, vp, vp]
    L.sdb_pending_tokens.restype = i32; L.sdb_pending_tokens.argtypes = [vp, u32, vp, vp]
    L.sdb_restore_compact.restype = i32
    L.sdb_restore_compact.argtypes = [vp, u32, vp, vp, vp, u64, vp, u64, vp, u64, u32, vp, vp]
    L.sdb_lease_reserve.restype = i32; L.sdb_lease_reserve.argtypes = [vp, u64, u64]
    L.sdb_receive_leased.restype = i32
    L.sdb_receive_leased.argtypes = [vp, u32, vp, u32, u32, C.c_double, vp, vp, u64, vp, u64, vp, u64, vp, vp, vp, vp]
    L.sdb_receive_leased_select.restype = i32
    L.sdb_receive_leased_select.argtypes = [vp, u32, vp, u32, u64, u64, vp, u32, C.c_double, vp, vp, u64, vp, u64, vp, u64,
                                            vp, vp, vp, vp]
    L.sdb_lease_settle.restype = i32; L.sdb_lease_settle.argtypes = [vp, u64, vp, u32, C.c_double, vp, vp]
    L.sdb_lease_sweep.restype = i32; L.sdb_lease_sweep.argtypes = [vp, C.c_double, u32, vp, vp, vp]
    L.sdb_lease_stats.restype = i32; L.sdb_lease_stats.argtypes = [vp, C.POINTER(SdbLeaseSummary)]
    L.sdb_lease_set_policy.restype = i32; L.sdb_lease_set_policy.argtypes = [vp, u32, u64]
    L.sdb_lease_deliveries.restype = i32; L.sdb_lease_deliveries.argtypes = [vp, u64, vp, vp]
    L.sdb_lease_dead_letters.restype = i32
    L.sdb_lease_dead_letters.argtypes = [vp, u32, vp, u32, vp, vp, u64, vp, u64, vp, u64, vp, vp, vp, vp]
    L.sdb_lease_policy_stats.restype = i32; L.sdb_lease_policy_stats.argtypes = [vp, C.POINTER(SdbLeasePolicySummary)]
    L.sdb_lease_export.restype = i32
    L.sdb_lease_export.argtypes = [vp, u64, u32, vp, u64, vp, u64, vp, u64, vp, vp, vp, vp, vp]
    L.sdb_lease_import.restype = i32; L.sdb_lease_import.argtypes = [vp, u64, vp, vp, u64, vp, u64, vp, u32, vp]
    L.sdb_lease_ledger_export.restype = i32; L.sdb_lease_ledger_export.argtypes = [vp, u64, vp, vp, vp, vp]
    L.sdb_lease_ledger_import.restype = i32; L.sdb_lease_ledger_import.argtypes = [vp, u64, vp, vp, vp, vp]
    L.sdb_arena_relocate.restype = i32; L.sdb_arena_relocate.argtypes = [vp, u64, u32, C.POINTER(SdbRelocateSummary)]
    L.sdb_expire.restype = i32
    L.sdb_expire.argtypes = [vp, u32, vp, C.c_double, u32, vp, vp, u64, vp, u64, vp, u64, vp, vp, vp]
    L.sdb_trim.restype = i32
    L.sdb_trim.argtypes = [vp, u32, vp, u32, u64, u32, vp, vp, u64, vp, u64, vp, u64, vp, vp, vp]
    L.sdb_supersede.restype = i32
    L.sdb_supersede.argtypes = [vp, u32, vp, u32, vp, vp, u64, vp, u64, vp, u64, vp, vp, vp]
    L.sdb_receive_where.restype = i32
    L.sdb_receive_where.argtypes = [vp, u32, vp, u32, u32, C.POINTER(SdbFilter), vp, vp, u64, vp, u64, vp, vp]
    L.sdb_receive_where_budget.restype = i32
    L.sdb_receive_where_budget.argtypes = [vp, u32, vp, u32, u64, u64, u32, C.POINTER(SdbFilter), vp, vp, u64, vp, u64, vp, vp]
    L.sdb_latency_server.restype = i32; L.sdb_latency_server.argtypes = [vp, i32]
    L.sdb_last_receive_dev.restype = i32; L.sdb_last_receive_dev.argtypes = [vp, vp, vp, vp]
    L.sdb_last_receive_totals.restype = i32; L.sdb_last_receive_totals.argtypes = [vp, vp, vp]
    L.sdb_digest_reset.restype = i32; L.sdb_digest_reset.argtypes = [vp]
    L.sdb_digest_fold.restype = i32; L.sdb_digest_fold.argtypes = [vp]
    L.sdb_digest_read.restype = i32; L.sdb_digest_read.argtypes = [vp, u32, vp, vp]
    L.sdb_wire_bytes.restype = u64; L.sdb_wire_bytes.argtypes = [vp, u32, u64]
    L.sdb_set_agent_shards.restype = i32; L.sdb_set_agent_shards.argtypes = [vp, u32, vp]
    L.sdb_export_group_batch.restype = i32; L.sdb_export_group_batch.argtypes = [vp, u32] + [vp] * 7 + [u64, vp, vp, u64]
    L.sdb_export_mixed_batch.restype = i32
    L.sdb_export_mixed_batch.argtypes = [vp, u32, vp, vp, vp, u32] + [vp] * 7 + [u64, vp, vp, u64]
    L.sdb_export_mixed_batch_seq.restype = i32
    L.sdb_export_mixed_batch_seq.argtypes = [vp, u64, u32, vp, vp, vp, u32] + [vp] * 7 + [u64, vp, vp, u64]
    L.sdb_wire_alloc.restype = i32; L.sdb_wire_alloc.argtypes = [vp, u64, C.POINTER(vp), vp]
    L.sdb_wire_open.restype = i32; L.sdb_wire_open.argtypes = [vp, vp, C.POINTER(vp)]
    L.sdb_wire_close.restype = i32; L.sdb_wire_close.argtypes = [vp, vp, i32]
    L.sdb_import_wire_ptrs.restype = i32; L.sdb_import_wire_ptrs.argtypes = [vp, u32, vp, vp]
    L.sdb_wire_wait_done.restype = i32; L.sdb_wire_wait_done.argtypes = [vp, u32, vp, u64, u32]
    L.sdb_wire_publish.restype = i32; L.sdb_wire_publish.argtypes = [vp, vp, u64, u32]
    L.sdb_import_wire_ptrs_async.restype = i32; L.sdb_import_wire_ptrs_async.argtypes = [vp, u32, vp, u64, u32]
    L.sdb_import_prefetch.restype = i32; L.sdb_import_prefetch.argtypes = [vp, u32, vp, u64, u32]
    L.sdb_overflow_log.restype = i32; L.sdb_overflow_log.argtypes = [vp, u32, vp, vp, vp, vp]
    L.sdb_import_wire_batches.restype = i32; L.sdb_import_wire_batches.argtypes = [vp, u32, vp, u64, vp]
    L.sdb_set_backends.restype = i32; L.sdb_set_backends.argtypes = [vp, u32, vp, vp]
    L.sdb_get_backend_loads.restype = i32; L.sdb_get_backend_loads.argtypes = [vp, u32, vp]
    L.sdb_release_backends.restype = i32; L.sdb_release_backends.argtypes = [vp, u32, vp, vp]
    L.sdb_select_backend_batch.restype = i32; L.sdb_select_backend_batch.argtypes = [vp, u32, vp, u32, u64, vp]
    L.sdb_agent_loads.restype = i32; L.sdb_agent_loads.argtypes = [vp, u32, vp, vp]
    L.sdb_queue_stats.restype = i32; L.sdb_queue_stats.argtypes = [vp, vp]
    L.sdb_assign_agent_backends.restype = i32; L.sdb_assign_agent_backends.argtypes = [vp, u32, vp, vp]
    L.sdb_backend_loads_from_queues.restype = i32; L.sdb_backend_loads_from_queues.argtypes = [vp]
    if L.sdb_abi_version() != 1:
        raise ImportError("swarmdb_b200 ABI version mismatch")
    _lib = L
    return L


def _p(a):
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        return a.ctypes.data_as(C.c_void_p)
    if isinstance(a, int):
        return C.c_void_p(a)
    raise TypeError(type(a))


def _arr(x, dt) -> np.ndarray:
    return np.ascontiguousarray(x, dtype=dt)


def pad32(n):
    return (n + 31) & ~31


def recv_capacity(cfg) -> int:
    """Records of the maximum size one receive call takes under `cfg` (a GpuConfig or SdbConfig):
    min(max_recv_records, max_recv_payload / pad32(max_payload_bytes)), at least 1.  The library divides
    max_recv_payload rounded up to 32 bytes, so it may allow a call more records than this, never fewer."""
    payload = int(cfg.max_recv_payload) or int(cfg.max_recv_records) * 256
    return max(1, min(int(cfg.max_recv_records), payload // pad32(int(cfg.max_payload_bytes))))


# kernel variant used when the caller does not choose one (SDB_FANOUT_VARIANT overrides, for A/B runs)
DEFAULT_FANOUT_VARIANT = int(os.environ.get("SDB_FANOUT_VARIANT", "2"))


class Shard:
    """One GPU-resident shard: per-agent rings + message arena + backend table on one device."""

    def __init__(self, max_agents: int, ring_slots: int = 64, arena_bytes: int = 1 << 28,
                 max_payload_bytes: int = 256, max_groups: int = 1, member_pool_entries: int = 0,
                 max_backends: int = 256, max_batch_sends: int = 65536, max_batch_payload: int = 0,
                 max_recv_records: int = 1 << 20, max_recv_payload: int = 0, list_pool_entries: int = 0,
                 device: int = 0, shard_id: int = 0, num_shards: int = 1, fanout_variant: Optional[int] = None) -> None:
        self._L = load_library()
        cfg = SdbConfig()
        cfg.struct_bytes = C.sizeof(SdbConfig)
        cfg.device, cfg.shard_id, cfg.num_shards = device, shard_id, num_shards
        cfg.max_agents, cfg.ring_slots, cfg.arena_bytes = max_agents, ring_slots, arena_bytes
        cfg.max_payload_bytes, cfg.max_groups = max_payload_bytes, max_groups
        cfg.member_pool_entries = member_pool_entries or max(1024, 2 * max_agents)
        cfg.max_backends, cfg.max_batch_sends, cfg.max_batch_payload = max_backends, max_batch_sends, max_batch_payload
        cfg.max_recv_records, cfg.max_recv_payload, cfg.list_pool_entries = max_recv_records, max_recv_payload, list_pool_entries
        cfg.fanout_variant = DEFAULT_FANOUT_VARIANT if fanout_variant is None else fanout_variant
        self.cfg = cfg
        self.max_agents = max_agents
        self._h = C.c_void_p()
        rc = self._L.sdb_create(C.byref(cfg), C.byref(self._h))
        if rc != 0:
            msg = self._L.sdb_last_error(self._h).decode() if self._h else "sdb_create failed"
            if self._h:
                self._L.sdb_destroy(self._h)
                self._h = C.c_void_p()
            raise SdbError(rc, msg)
        self.max_recv_records = int(cfg.max_recv_records) or (1 << 20)
        self._keep = None          # keeps the last payload buffer alive while its H2D copy is in flight
        # pinned-or-pageable host output buffers, grown on demand
        self._out_hdr = np.zeros(0, HDR_DTYPE)
        self._out_pay = np.zeros(0, np.uint8)
        self._nb = 0

    # ------------------------------------------------------------------ plumbing
    def _check(self, rc: int) -> None:
        if rc != 0:
            raise SdbError(rc, self._L.sdb_last_error(self._h).decode())

    def close(self) -> None:
        if getattr(self, "_h", None):
            self._L.sdb_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_stream(self, cuda_stream: int) -> None:
        self._check(self._L.sdb_set_stream(self._h, C.c_void_p(cuda_stream)))

    def sync(self) -> None:
        self._check(self._L.sdb_sync(self._h))

    def stats(self) -> dict:
        s = SdbStats()
        self._check(self._L.sdb_get_stats(self._h, C.byref(s)))
        return {n: int(getattr(s, n)) for n, _ in SdbStats._fields_}

    def debug_set_arena_pos(self, granules: int) -> None:
        self._check(self._L.sdb_debug_set_arena_pos(self._h, granules))

    def advance_seq(self, next_seq: int) -> None:
        """Move the handle's sequence counter forward (ids of a refused batch are never reissued)."""
        self._check(self._L.sdb_advance_seq(self._h, next_seq))

    # the SDB_PK_N classes sdb_profile_read fills, then the classes only sdb_profile_read_n reports (SDB_PK_ALL in all)
    PROFILE_KINDS = ["p2p", "fanout", "commit", "recv_count", "recv_scan", "recv_select", "recv_gather",
                     "arena_floor", "pick", "xshard", "index", "xwait", "recv_compact", "expire", "where", "restore"]
    PROFILE_KINDS_ALL = PROFILE_KINDS + ["lease"]
    PROFILE_CLASSES = PROFILE_KINDS_ALL + ["dedup"]      # SDB_PK_CLASSES: every class sdb_profile_read_n reports

    def profile(self, enable: bool) -> None:
        self._check(self._L.sdb_profile(self._h, 1 if enable else 0))

    def profile_read(self) -> dict:
        """{kernel class: (total ms, launches)} over PROFILE_CLASSES, measured with CUDA events on the launching stream."""
        n = len(self.PROFILE_CLASSES)
        ms = np.zeros(n, np.float64)
        cnt = np.zeros(n, np.uint64)
        self._check(self._L.sdb_profile_read_n(self._h, n, _p(ms), _p(cnt)))
        return {k: (float(ms[i]), int(cnt[i])) for i, k in enumerate(self.PROFILE_CLASSES)}

    # ------------------------------------------------------------------ registry / groups
    def register(self, idx) -> None:
        a = _arr(np.atleast_1d(idx), np.uint32)
        self._check(self._L.sdb_register_agents(self._h, len(a), _p(a)))

    def deregister(self, idx) -> None:
        a = _arr(np.atleast_1d(idx), np.uint32)
        self._check(self._L.sdb_deregister_agents(self._h, len(a), _p(a)))

    def create_group(self, g: int, members) -> None:
        m = _arr(members, np.uint32)
        self._check(self._L.sdb_create_group(self._h, g, len(m), _p(m)))

    # ------------------------------------------------------------------ enqueue
    @staticmethod
    def _common(n, prio, typ, lens, payload_off, payload, ts):
        prio = None if prio is None else _arr(prio, np.uint8)
        typ = None if typ is None else _arr(typ, np.uint8)
        lens = _arr(lens, np.uint16)
        payload_off = _arr(payload_off, np.uint64)
        payload = _arr(payload, np.uint8)
        ts = None if ts is None else _arr(ts, np.float64)
        assert len(lens) == n and len(payload_off) == n
        return prio, typ, lens, payload_off, payload, ts

    def send_batch(self, sender, receiver, prio, typ, lens, payload_off, payload, ts=None) -> int:
        s, r = _arr(sender, np.uint32), _arr(receiver, np.uint32)
        prio, typ, lens, po, pl, ts = self._common(len(s), prio, typ, lens, payload_off, payload, ts)
        base = C.c_uint64(0)
        self._keep = pl
        self._check(self._L.sdb_send_batch(self._h, len(s), _p(s), _p(r), _p(prio), _p(typ), _p(lens), _p(po), _p(pl),
                                           pl.nbytes, _p(ts), C.cast(C.byref(base), C.c_void_p)))
        return base.value

    def send_group_batch(self, sender, group, prio, typ, lens, payload_off, payload, ts=None) -> int:
        s, g = _arr(sender, np.uint32), _arr(group, np.uint32)
        prio, typ, lens, po, pl, ts = self._common(len(s), prio, typ, lens, payload_off, payload, ts)
        base = C.c_uint64(0)
        self._keep = pl
        self._check(self._L.sdb_send_group_batch(self._h, len(s), _p(s), _p(g), _p(prio), _p(typ), _p(lens), _p(po),
                                                 _p(pl), pl.nbytes, _p(ts), C.cast(C.byref(base), C.c_void_p)))
        return base.value

    def send_list_batch(self, sender, list_off, list_idx, prio, typ, lens, payload_off, payload, ts=None) -> int:
        s = _arr(sender, np.uint32)
        lo, li = _arr(list_off, np.uint64), _arr(list_idx, np.uint32)
        prio, typ, lens, po, pl, ts = self._common(len(s), prio, typ, lens, payload_off, payload, ts)
        base = C.c_uint64(0)
        self._keep = pl
        self._check(self._L.sdb_send_list_batch(self._h, len(s), _p(s), _p(lo), _p(li), _p(prio), _p(typ), _p(lens),
                                                _p(po), _p(pl), pl.nbytes, _p(ts), C.cast(C.byref(base), C.c_void_p)))
        return base.value

    def send_mixed_batch(self, sender, kind, target, list_off, list_idx, prio, typ, lens, payload_off, payload,
                         ts=None) -> int:
        """kind[i]: 0 p2p (target = receiver), 1 group (target = group), 2 list (target = list number)."""
        s, k, t = _arr(sender, np.uint32), _arr(kind, np.uint8), _arr(target, np.uint32)
        lo = _arr(list_off if list_off is not None else [0], np.uint64)
        li = _arr(list_idx if list_idx is not None else [], np.uint32)
        prio, typ, lens, po, pl, ts = self._common(len(s), prio, typ, lens, payload_off, payload, ts)
        base = C.c_uint64(0)
        self._keep = pl
        self._check(self._L.sdb_send_mixed_batch(self._h, len(s), _p(s), _p(k), _p(t), len(lo) - 1, _p(lo), _p(li),
                                                 _p(prio), _p(typ), _p(lens), _p(po), _p(pl), pl.nbytes, _p(ts),
                                                 C.cast(C.byref(base), C.c_void_p)))
        return base.value

    def send_mixed_batch_dedup(self, sender, kind, target, list_off, list_idx, prio, typ, lens, payload_off, payload,
                               ts=None, keys=None, content: bool = False, now: float = 0.0):
        """send_mixed_batch with deduplication (include/swarmdb_b200.h "deduplicated sends").  keys: KEY_DTYPE[n] or a
        (n, 2) uint64 array of (lo, hi), None for all {0,0}.  Returns (seq_base, dup_of uint64[n], keys KEY_DTYPE[n]):
        dup_of[i] is the first seq of the send i duplicates (0: accepted), keys the keys used."""
        s, k, t = _arr(sender, np.uint32), _arr(kind, np.uint8), _arr(target, np.uint32)
        lo = _arr(list_off if list_off is not None else [0], np.uint64)
        li = _arr(list_idx if list_idx is not None else [], np.uint32)
        prio, typ, lens, po, pl, ts = self._common(len(s), prio, typ, lens, payload_off, payload, ts)
        kin = None if keys is None else _keys(keys, len(s))
        kout = np.zeros(len(s), KEY_DTYPE)
        dup = np.zeros(len(s), np.uint64)
        base, ndup = C.c_uint64(0), C.c_uint32(0)
        self._keep = pl
        self._check(self._L.sdb_send_mixed_batch_dedup(
            self._h, len(s), _p(s), _p(k), _p(t), len(lo) - 1, _p(lo), _p(li), _p(prio), _p(typ), _p(lens), _p(po), _p(pl),
            pl.nbytes, _p(ts), None if kin is None else _p(kin), DEDUP_CONTENT if content else 0, float(now), _p(kout),
            _p(dup), C.cast(C.byref(ndup), C.c_void_p), C.cast(C.byref(base), C.c_void_p)))
        return base.value, dup, kout

    def dedup_reserve(self, entries: int, window: float = 300.0) -> None:
        """Allocate (or clear) the deduplication table; 0 entries frees it."""
        self._check(self._L.sdb_dedup_reserve(self._h, int(entries), float(window)))

    def dedup_forget(self, keys) -> np.ndarray:
        """Kill the entries of the given keys; returns removed uint8[n] (1 where the entry was live)."""
        kin = _keys(keys, None)
        out = np.zeros(len(kin), np.uint8)
        self._check(self._L.sdb_dedup_forget(self._h, len(kin), _p(kin), _p(out)))
        return out

    def dedup_stats(self) -> dict:
        st = SdbDedupSummary()
        self._check(self._L.sdb_dedup_stats(self._h, C.byref(st)))
        return {n: (float(getattr(st, n)) if n == "window" else int(getattr(st, n))) for n, _ in SdbDedupSummary._fields_}

    def stage(self, kind: int, sender, second, prio, typ, lens, payload_off, payload, ts=None) -> int:
        """Copy a p2p (kind 0) or group (kind 1) batch to device memory; returns a staged handle."""
        s, g = _arr(sender, np.uint32), _arr(second, np.uint32)
        prio, typ, lens, po, pl, ts = self._common(len(s), prio, typ, lens, payload_off, payload, ts)
        out = C.c_void_p()
        self._check(self._L.sdb_stage_batch(self._h, kind, len(s), _p(s), _p(g), _p(prio), _p(typ), _p(lens), _p(po),
                                            _p(pl), pl.nbytes, _p(ts), C.byref(out)))
        return out.value

    def submit(self, staged: int) -> int:
        base = C.c_uint64(0)
        self._check(self._L.sdb_submit_staged(self._h, C.c_void_p(staged), C.cast(C.byref(base), C.c_void_p)))
        return base.value

    def free_staged(self, staged: int) -> None:
        self._check(self._L.sdb_free_staged(self._h, C.c_void_p(staged)))

    # ------------------------------------------------------------------ cross-shard
    def wire_bytes(self, max_sends: int, max_payload: int) -> int:
        return int(self._L.sdb_wire_bytes(self._h, max_sends, max_payload))

    def set_agent_shards(self, shard_of) -> None:
        s = _arr(shard_of, np.uint8)
        self._check(self._L.sdb_set_agent_shards(self._h, len(s), _p(s)))
        full = np.full(self.max_agents, int(self.cfg.shard_id), np.uint8)
        full[: len(s)] = s
        self.n_owned = int((full == int(self.cfg.shard_id)).sum()) if int(self.cfg.num_shards) > 1 else None

    def export_group_batch(self, sender, group, prio, typ, lens, payload_off, payload, wire_dev: int, wire_cap: int,
                           ts=None) -> None:
        """Write this rank's batch of group sends as one wire batch into device memory at `wire_dev`."""
        s, g = _arr(sender, np.uint32), _arr(group, np.uint32)
        prio, typ, lens, po, pl, ts = self._common(len(s), prio, typ, lens, payload_off, payload, ts)
        self._keep = pl
        self._check(self._L.sdb_export_group_batch(self._h, len(s), _p(s), _p(g), _p(prio), _p(typ), _p(lens), _p(po),
                                                   _p(pl), pl.nbytes, _p(ts), C.c_void_p(wire_dev), wire_cap))

    def export_mixed_batch(self, sender, kind, target, list_off, list_idx, prio, typ, lens, payload_off, payload,
                           wire_dev: int, wire_cap: int, ts=None, seq_base: int = 0) -> None:
        """seq_base != 0: the exporter numbers its own sends from that (composite) sequence number."""
        s, k, t = _arr(sender, np.uint32), _arr(kind, np.uint8), _arr(target, np.uint32)
        lo = _arr(list_off if list_off is not None else [0], np.uint64)
        li = _arr(list_idx if list_idx is not None else [], np.uint32)
        prio, typ, lens, po, pl, ts = self._common(len(s), prio, typ, lens, payload_off, payload, ts)
        self._keep = pl
        if seq_base:
            self._check(self._L.sdb_export_mixed_batch_seq(self._h, seq_base, len(s), _p(s), _p(k), _p(t), len(lo) - 1, _p(lo),
                                                           _p(li), _p(prio), _p(typ), _p(lens), _p(po), _p(pl), pl.nbytes,
                                                           _p(ts), C.c_void_p(wire_dev), wire_cap))
            return
        self._check(self._L.sdb_export_mixed_batch(self._h, len(s), _p(s), _p(k), _p(t), len(lo) - 1, _p(lo), _p(li),
                                                   _p(prio), _p(typ), _p(lens), _p(po), _p(pl), pl.nbytes, _p(ts),
                                                   C.c_void_p(wire_dev), wire_cap))

    def wire_alloc(self, nbytes: int):
        """Device export buffer + its 64-byte CUDA-IPC handle (bytes) for the peer-memory transport."""
        dev = C.c_void_p()
        handle = C.create_string_buffer(64)
        self._check(self._L.sdb_wire_alloc(self._h, nbytes, C.byref(dev), C.cast(handle, C.c_void_p)))
        return dev.value, handle.raw

    def wire_open(self, ipc_handle: bytes) -> int:
        dev = C.c_void_p()
        buf = C.create_string_buffer(ipc_handle, 64)
        self._check(self._L.sdb_wire_open(self._h, C.cast(buf, C.c_void_p), C.byref(dev)))
        return dev.value

    def wire_close(self, dev: int, opened: bool) -> None:
        self._check(self._L.sdb_wire_close(self._h, C.c_void_p(dev), 1 if opened else 0))

    def import_wire_ptrs(self, ptrs) -> int:
        """Import one wire batch per source rank from a table of device pointers (rank order)."""
        arr = (C.c_void_p * len(ptrs))(*[C.c_void_p(int(x)) for x in ptrs])
        base = C.c_uint64(0)
        self._check(self._L.sdb_import_wire_ptrs(self._h, len(ptrs), C.cast(arr, C.c_void_p), C.cast(C.byref(base), C.c_void_p)))
        return base.value

    # flag-synchronised, host-asynchronous peer transport (see include/swarmdb_b200.h)
    @staticmethod
    def _ptr_table(ptrs):
        return (C.c_void_p * len(ptrs))(*[C.c_void_p(int(x)) for x in ptrs])

    def wire_wait_done(self, ptrs, wire_bytes: int, step: int) -> None:
        """Stream-ordered wait until the owner of every listed buffer has finished importing `step`."""
        arr = self._ptr_table(ptrs)
        self._check(self._L.sdb_wire_wait_done(self._h, len(ptrs), C.cast(arr, C.c_void_p), wire_bytes, step))

    def wire_publish(self, wire_dev: int, wire_bytes: int, step: int) -> None:
        """Stream-ordered: this buffer now holds the complete export of `step`."""
        self._check(self._L.sdb_wire_publish(self._h, C.c_void_p(wire_dev), wire_bytes, step))

    def overflow_log(self, cap: int = 4096):
        """(agents, seqs, dropped): the records that found their receiver's ring full since the last call
        (include/swarmdb_b200.h: sdb_overflow_log); reading clears the log."""
        ag = np.zeros(cap, np.uint32); sq = np.zeros(cap, np.uint64)
        n = C.c_uint32(0); dropped = C.c_uint64(0)
        self._check(self._L.sdb_overflow_log(self._h, cap, _p(ag), _p(sq), C.cast(C.byref(n), C.c_void_p),
                                             C.cast(C.byref(dropped), C.c_void_p)))
        return ag[:n.value].copy(), sq[:n.value].copy(), int(dropped.value)

    def import_prefetch(self, ptrs, wire_bytes: int, step: int) -> None:
        """Run the flag wait + localize pass of `step` on the handle's prefetch stream, beside what is enqueued next
        (include/swarmdb_b200.h: sdb_import_prefetch); the following import_wire_ptrs_async(step) only places it."""
        arr = (C.c_void_p * len(ptrs))(*ptrs)
        self._check(self._L.sdb_import_prefetch(self._h, len(ptrs), C.cast(arr, C.c_void_p), wire_bytes, step))

    def import_wire_ptrs_async(self, ptrs, wire_bytes: int, step: int) -> None:
        """Wait on the device for every source's `step`, import without a host round trip, report done."""
        arr = self._ptr_table(ptrs)
        self._check(self._L.sdb_import_wire_ptrs_async(self._h, len(ptrs), C.cast(arr, C.c_void_p), wire_bytes, step))

    def import_wire_batches(self, n_src: int, wire_dev_all: int, stride: int) -> int:
        """Expand the wire batches of `n_src` ranks (rank order, `stride` bytes apart) for the agents this shard owns."""
        base = C.c_uint64(0)
        self._check(self._L.sdb_import_wire_batches(self._h, n_src, C.c_void_p(wire_dev_all), stride,
                                                    C.cast(C.byref(base), C.c_void_p)))
        return base.value

    # ------------------------------------------------------------------ dequeue
    def receive_batch(self, agents, max_messages: int, flags: int = 0, copy_out: bool = True,
                      out_hdr: Optional[np.ndarray] = None, out_payload: Optional[np.ndarray] = None, wait: bool = True):
        """Returns (counts[n_agents], headers[total], payload bytes) - views into reusable buffers
        unless explicit output arrays are given.  copy_out=False leaves results on the device and returns
        (None, total, payload_bytes); with wait=False the call only enqueues the receive (SDB_RECV_ASYNC,
        totals later through last_receive_totals()) and returns (None, None, None)."""
        if not wait:
            if copy_out:
                raise ValueError("wait=False needs copy_out=False")
            flags |= RECV_ASYNC
        a, n, counts = self._agents_arg(agents, copy_out)
        total, pbytes = C.c_uint64(0), C.c_uint64(0)
        hdr = pay = None
        hdr_cap = pay_cap = 0
        if copy_out:
            hdr = out_hdr if out_hdr is not None else self._grow_hdr()
            pay = out_payload if out_payload is not None else self._grow_pay()
            hdr_cap, pay_cap = len(hdr), pay.nbytes
        self._check(self._L.sdb_receive_batch(self._h, n, _p(a), max_messages, flags, _p(counts), _p(hdr), hdr_cap,
                                              _p(pay), pay_cap, C.cast(C.byref(total), C.c_void_p),
                                              C.cast(C.byref(pbytes), C.c_void_p)))
        if not wait:
            return None, None, None
        if not copy_out:
            return None, total.value, pbytes.value
        if agents is None:
            counts = self._served_counts(counts, flags)
        return counts, hdr[: total.value], pay[: pbytes.value]

    def receive_budget(self, agents, max_messages: int, max_agent_bytes: int, flags: int = 0,
                       out_hdr: Optional[np.ndarray] = None, out_payload: Optional[np.ndarray] = None):
        """receive_batch by byte budget (include/swarmdb_b200.h: sdb_receive_budget): each agent takes the longest prefix
        of its delivery order with at most max_messages records and sum(pad32(len)) <= max_agent_bytes (0: no byte
        limit; an oversized first record is taken alone), and the call fills its buffers exactly by bytes instead of
        by max_payload_bytes.  Returns (counts[n_agents], headers[total], payload bytes) as receive_batch does."""
        a, n, counts = self._agents_arg(agents)
        hdr = out_hdr if out_hdr is not None else self._grow_hdr()
        pay = out_payload if out_payload is not None else self._grow_pay()
        total, pbytes = C.c_uint64(0), C.c_uint64(0)
        self._check(self._L.sdb_receive_budget(self._h, n, _p(a), max_messages, int(max_agent_bytes), flags, _p(counts),
                                               _p(hdr), len(hdr), _p(pay), pay.nbytes, C.cast(C.byref(total), C.c_void_p),
                                               C.cast(C.byref(pbytes), C.c_void_p)))
        if agents is None:
            counts = self._served_counts(counts, flags)
        return counts, hdr[: total.value], pay[: pbytes.value]

    def receive_compact(self, agents, max_messages: int, flags: int = 0, out_entries: Optional[np.ndarray] = None,
                        out_sends: Optional[np.ndarray] = None, out_payload: Optional[np.ndarray] = None,
                        max_agent_bytes: Optional[int] = None):
        """The records receive_batch would return, in the compact format (include/swarmdb_b200.h:
        sdb_receive_compact): (counts[n_agents], entries[total] ENTRY_DTYPE, sends[n_sends] SEND_DTYPE, payload bytes),
        each distinct payload once.  Views into reusable buffers unless explicit (e.g. pinned) arrays are given;
        expand_compact() turns them into receive_batch's (headers, payload).  With max_agent_bytes (0: no per-agent
        limit) the call takes receive_budget's records (sdb_receive_compact_budget)."""
        a, n, counts = self._agents_arg(agents)
        ent, snd, pay = self._compact_outputs(out_entries, out_sends, out_payload)
        total, n_sends, pbytes = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
        tail = (_p(counts), _p(ent), len(ent), _p(snd), len(snd), _p(pay), pay.nbytes, C.cast(C.byref(total), C.c_void_p),
                C.cast(C.byref(n_sends), C.c_void_p), C.cast(C.byref(pbytes), C.c_void_p))
        if max_agent_bytes is None:
            self._check(self._L.sdb_receive_compact(self._h, n, _p(a), max_messages, flags, *tail))
        else:
            self._check(self._L.sdb_receive_compact_budget(self._h, n, _p(a), max_messages, int(max_agent_bytes), flags, *tail))
        if agents is None:
            counts = self._served_counts(counts, flags)
        return counts, ent[: total.value], snd[: n_sends.value], pay[: pbytes.value]

    def receive_tokens(self, agents, max_messages: int, max_agent_tokens: int, max_agent_bytes: int = 0, flags: int = 0,
                       out_hdr: Optional[np.ndarray] = None, out_payload: Optional[np.ndarray] = None):
        """receive_budget by token budget (include/swarmdb_b200.h: sdb_receive_tokens): each agent's take is also cut
        at the longest prefix of its delivery order whose token weights (the u32 count at the start of a TYPEF_TOKENS
        payload, 0 for other records) sum to at most max_agent_tokens (0: no token limit; a heavier first record is
        taken alone).  Returns (counts[n_agents], headers[total], payload bytes) as receive_batch does."""
        a, n, counts = self._agents_arg(agents)
        hdr = out_hdr if out_hdr is not None else self._grow_hdr()
        pay = out_payload if out_payload is not None else self._grow_pay()
        total, pbytes = C.c_uint64(0), C.c_uint64(0)
        self._check(self._L.sdb_receive_tokens(self._h, n, _p(a), max_messages, int(max_agent_bytes), int(max_agent_tokens),
                                               flags, _p(counts), _p(hdr), len(hdr), _p(pay), pay.nbytes,
                                               C.cast(C.byref(total), C.c_void_p), C.cast(C.byref(pbytes), C.c_void_p)))
        if agents is None:
            counts = self._served_counts(counts, flags)
        return counts, hdr[: total.value], pay[: pbytes.value]

    def receive_compact_tokens(self, agents, max_messages: int, max_agent_tokens: int, max_agent_bytes: int = 0,
                               flags: int = 0, out_entries: Optional[np.ndarray] = None,
                               out_sends: Optional[np.ndarray] = None, out_payload: Optional[np.ndarray] = None):
        """receive_tokens' records in the compact format (sdb_receive_compact_tokens); returns what receive_compact
        returns."""
        a, n, counts = self._agents_arg(agents)
        ent, snd, pay = self._compact_outputs(out_entries, out_sends, out_payload)
        total, n_sends, pbytes = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
        self._check(self._L.sdb_receive_compact_tokens(
            self._h, n, _p(a), max_messages, int(max_agent_bytes), int(max_agent_tokens), flags, _p(counts), _p(ent),
            len(ent), _p(snd), len(snd), _p(pay), pay.nbytes, C.cast(C.byref(total), C.c_void_p),
            C.cast(C.byref(n_sends), C.c_void_p), C.cast(C.byref(pbytes), C.c_void_p)))
        if agents is None:
            counts = self._served_counts(counts, flags)
        return counts, ent[: total.value], snd[: n_sends.value], pay[: pbytes.value]

    def pending_tokens(self, agents=None, n: Optional[int] = None) -> np.ndarray:
        """uint64 per agent: the token weights of its pending records, summed (sdb_pending_tokens).  agents None: every
        agent below the registration watermark (or the first n)."""
        if agents is None:
            a, cnt = None, int(n if n is not None else self.stats_n_agents())
        else:
            a = _arr(agents, np.uint32)
            cnt = len(a)
        out = np.zeros(cnt, np.uint64)
        self._check(self._L.sdb_pending_tokens(self._h, cnt, _p(a), _p(out)))
        return out

    def restore_compact(self, agents, counts, entries, sends, payload, flags: int = 0) -> Tuple[int, int]:
        """Append records in the compact receive format behind what each listed agent has pending, with their own
        sequence numbers (include/swarmdb_b200.h: sdb_restore_compact): agent i takes the next counts[i] entries.  All
        or nothing.  Returns (records restored, next sequence number)."""
        a, c = _arr(agents, np.uint32), _arr(counts, np.uint32)
        if len(a) != len(c):
            raise ValueError("agents and counts differ in length")
        ent, snd = np.ascontiguousarray(entries, ENTRY_DTYPE), np.ascontiguousarray(sends, SEND_DTYPE)
        pay = np.ascontiguousarray(payload, np.uint8)
        restored, seq_end = C.c_uint64(0), C.c_uint64(0)
        self._check(self._L.sdb_restore_compact(self._h, len(a), _p(a), _p(c), _p(ent), len(ent), _p(snd), len(snd),
                                                _p(pay), pay.nbytes, flags, C.cast(C.byref(restored), C.c_void_p),
                                                C.cast(C.byref(seq_end), C.c_void_p)))
        return int(restored.value), int(seq_end.value)

    # ------------------------------------------------------------------ leases (include/swarmdb_b200.h: sdb_lease_*)
    def lease_reserve(self, max_records: int, max_payload_bytes: int) -> None:
        """Allocate the device lease store (0 records frees it); refused while it holds live leases."""
        self._check(self._L.sdb_lease_reserve(self._h, int(max_records), int(max_payload_bytes)))

    def receive_leased(self, agents, max_messages: int, deadline: float, flags: int = 0,
                       out_entries: Optional[np.ndarray] = None, out_sends: Optional[np.ndarray] = None,
                       out_payload: Optional[np.ndarray] = None, max_agent_bytes: int = 0, max_agent_tokens: int = 0,
                       filt: Optional[SdbFilter] = None):
        """receive_compact's records and result, each also kept in the lease store with `deadline` until it is acked or
        redelivered.  Returns (counts, entries, sends, payload, lease_base): entry r holds lease lease_base + r.
        max_agent_bytes / max_agent_tokens (0: no limit) cut each agent's take as receive_budget / receive_tokens do,
        and `filt` (make_filter()) leases only the matching records, as receive_where takes them
        (include/swarmdb_b200.h: sdb_receive_leased_select)."""
        a, n, counts = self._agents_arg(agents)
        ent, snd, pay = self._compact_outputs(out_entries, out_sends, out_payload)
        total, n_sends, pbytes, base = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
        tail = (float(deadline), _p(counts), _p(ent), len(ent), _p(snd), len(snd), _p(pay), pay.nbytes,
                C.cast(C.byref(total), C.c_void_p), C.cast(C.byref(n_sends), C.c_void_p),
                C.cast(C.byref(pbytes), C.c_void_p), C.cast(C.byref(base), C.c_void_p))
        if max_agent_bytes or max_agent_tokens or filt is not None:
            self._check(self._L.sdb_receive_leased_select(self._h, n, _p(a), max_messages, int(max_agent_bytes),
                                                          int(max_agent_tokens),
                                                          None if filt is None else C.cast(C.byref(filt), C.c_void_p),
                                                          flags, *tail))
        else:
            self._check(self._L.sdb_receive_leased(self._h, n, _p(a), max_messages, flags, *tail))
        if agents is None:
            counts = self._served_counts(counts, flags)
        return counts, ent[: total.value], snd[: n_sends.value], pay[: pbytes.value], int(base.value)

    def lease_settle(self, lease_ids, op: int, deadline: float = 0.0) -> Tuple[np.ndarray, int]:
        """Ack (LEASE_ACK) or renew (LEASE_RENEW, new deadline) leases.  Returns (settled[n] uint8: 1 where the lease was
        live, number settled)."""
        ids = _arr(np.atleast_1d(lease_ids), np.uint64)
        out = np.zeros(len(ids), np.uint8)
        n = C.c_uint64(0)
        self._check(self._L.sdb_lease_settle(self._h, len(ids), _p(ids), op, float(deadline), _p(out),
                                             C.cast(C.byref(n), C.c_void_p)))
        return out, int(n.value)

    def lease_sweep(self, now: float, flags: int = 0) -> Tuple[int, int, int]:
        """Redeliver due leases (one compact receive's capacity per call).  Returns (redelivered, blocked agents,
        due records left for the next call)."""
        red, blk, left = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
        self._check(self._L.sdb_lease_sweep(self._h, float(now), flags, C.cast(C.byref(red), C.c_void_p),
                                            C.cast(C.byref(blk), C.c_void_p), C.cast(C.byref(left), C.c_void_p)))
        return int(red.value), int(blk.value), int(left.value)

    def lease_stats(self) -> dict:
        s = SdbLeaseSummary()
        self._check(self._L.sdb_lease_stats(self._h, C.byref(s)))
        return {n: int(getattr(s, n)) for n, _ in SdbLeaseSummary._fields_}

    def lease_set_policy(self, max_deliveries: int, ledger_entries: int) -> None:
        """Redelivery limit and ledger size (include/swarmdb_b200.h: sdb_lease_set_policy); (0, 0) turns it off."""
        self._check(self._L.sdb_lease_set_policy(self._h, int(max_deliveries), int(ledger_entries)))

    def lease_deliveries(self, lease_ids) -> np.ndarray:
        """Delivery count of each live or dead lease (uint32), 0 for unknown, acked or redelivered ids."""
        ids = _arr(np.atleast_1d(lease_ids), np.uint64)
        out = np.zeros(len(ids), np.uint32)
        self._check(self._L.sdb_lease_deliveries(self._h, len(ids), _p(ids), _p(out)))
        return out

    def lease_dead_letters(self, agents, flags: int = 0, out_entries: Optional[np.ndarray] = None,
                           out_sends: Optional[np.ndarray] = None, out_payload: Optional[np.ndarray] = None):
        """The listed agents' dead letters in receive_compact's shape (PEEK leaves them in the store).  Returns
        (counts, entries, sends, payload, deliveries); the first four are valid restore_compact input as they stand."""
        a, n, counts = self._agents_arg(agents)
        ent, snd, pay = self._compact_outputs(out_entries, out_sends, out_payload)
        deliv = np.zeros(len(ent), np.uint32)
        total, n_sends, pbytes = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
        self._check(self._L.sdb_lease_dead_letters(self._h, n, _p(a), flags, _p(counts), _p(ent), len(ent), _p(snd),
                                                   len(snd), _p(pay), pay.nbytes, _p(deliv),
                                                   C.cast(C.byref(total), C.c_void_p), C.cast(C.byref(n_sends), C.c_void_p),
                                                   C.cast(C.byref(pbytes), C.c_void_p)))
        if agents is None:
            counts = counts[: self.stats_n_agents()]
        return counts, ent[: total.value], snd[: n_sends.value], pay[: pbytes.value], deliv[: total.value]

    def lease_policy_stats(self) -> dict:
        s = SdbLeasePolicySummary()
        self._check(self._L.sdb_lease_policy_stats(self._h, C.byref(s)))
        return {n: int(getattr(s, n)) for n, _ in SdbLeasePolicySummary._fields_}

    def lease_export(self, start_id: int = 0, out_entries: Optional[np.ndarray] = None,
                     out_sends: Optional[np.ndarray] = None, out_payload: Optional[np.ndarray] = None,
                     out_meta: Optional[np.ndarray] = None):
        """One chunk of the store's live leases and dead letters with id >= start_id, in lease-id order, without changing
        anything (include/swarmdb_b200.h: sdb_lease_export).  Returns (entries, sends, payload, meta META_DTYPE, next_id);
        loop from next_id until entries is empty.  Views into reusable buffers unless explicit arrays are given; out_meta
        holds as many records as out_entries."""
        ent, snd, pay = self._compact_outputs(out_entries, out_sends, out_payload)
        meta = out_meta
        if meta is None:
            if len(getattr(self, "_out_meta", ())) < len(ent):
                self._out_meta = np.zeros(len(ent), META_DTYPE)
            meta = self._out_meta
        if len(meta) < len(ent):
            raise ValueError("out_meta holds fewer records than out_entries")
        total, n_sends, pbytes, nxt = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
        self._check(self._L.sdb_lease_export(self._h, int(start_id), 0, _p(ent), len(ent), _p(snd), len(snd), _p(pay),
                                             pay.nbytes, _p(meta), C.cast(C.byref(total), C.c_void_p),
                                             C.cast(C.byref(n_sends), C.c_void_p), C.cast(C.byref(pbytes), C.c_void_p),
                                             C.cast(C.byref(nxt), C.c_void_p)))
        return ent[: total.value], snd[: n_sends.value], pay[: pbytes.value], meta[: total.value], int(nxt.value)

    def lease_import(self, entries, sends, payload, meta, flags: int = 0) -> int:
        """Append exported leases behind what the store holds, with their deadlines, states and counts
        (include/swarmdb_b200.h: sdb_lease_import).  All or nothing.  Returns the lease id of the first record."""
        ent, snd = np.ascontiguousarray(entries, ENTRY_DTYPE), np.ascontiguousarray(sends, SEND_DTYPE)
        pay, met = np.ascontiguousarray(payload, np.uint8), np.ascontiguousarray(meta, META_DTYPE)
        if len(met) != len(ent):
            raise ValueError("entries and meta differ in length")
        base = C.c_uint64(0)
        self._check(self._L.sdb_lease_import(self._h, len(ent), _p(ent), _p(snd), len(snd), _p(pay), pay.nbytes, _p(met),
                                             flags, C.cast(C.byref(base), C.c_void_p)))
        return int(base.value)

    def ledger_export(self) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        """The redelivery ledger's counts of records still pending, as (agent uint32, seq uint64, count uint32) arrays in
        no particular order (include/swarmdb_b200.h: sdb_lease_ledger_export)."""
        n = C.c_uint64(0)
        rc = self._L.sdb_lease_ledger_export(self._h, 0, None, None, None, C.cast(C.byref(n), C.c_void_p))
        if rc not in (0, -8):                                       # -8 (SDB_EOUTPUT): n holds the size
            self._check(rc)
        while True:
            k = int(n.value)
            a, s, c = np.zeros(k, np.uint32), np.zeros(k, np.uint64), np.zeros(k, np.uint32)
            rc = self._L.sdb_lease_ledger_export(self._h, k, _p(a), _p(s), _p(c), C.cast(C.byref(n), C.c_void_p))
            if rc != -8:
                self._check(rc)
                return a[: n.value], s[: n.value], c[: n.value]

    def ledger_import(self, agent, seq, count) -> int:
        """Give each (agent, seq) triple's oldest pending record the delivery count `count` in the ledger, as if a sweep
        had redelivered it (include/swarmdb_b200.h: sdb_lease_ledger_import).  Returns the triples matched."""
        a, s, c = _arr(agent, np.uint32), _arr(seq, np.uint64), _arr(count, np.uint32)
        if not len(a) == len(s) == len(c):
            raise ValueError("agent, seq and count differ in length")
        matched = C.c_uint64(0)
        self._check(self._L.sdb_lease_ledger_import(self._h, len(a), _p(a), _p(s), _p(c), C.cast(C.byref(matched), C.c_void_p)))
        return int(matched.value)

    def relocate(self, floor_bytes: int, peek: bool = False) -> dict:
        """Move the pending records of every agent with one below `floor_bytes` to the arena tail, in place in their
        rings (include/swarmdb_b200.h: sdb_arena_relocate); peek=True is a dry run.  Returns the summary."""
        s = SdbRelocateSummary()
        self._check(self._L.sdb_arena_relocate(self._h, int(floor_bytes), RECV_PEEK if peek else 0, C.byref(s)))
        return {n: int(getattr(s, n)) for n, _ in SdbRelocateSummary._fields_}

    def expire(self, agents, older_than: float, flags: int = 0, archive: bool = True,
               out_entries: Optional[np.ndarray] = None, out_sends: Optional[np.ndarray] = None,
               out_payload: Optional[np.ndarray] = None):
        """Retire pending records older than `older_than` (every pending record with EXPIRE_ALL) without delivering them
        (include/swarmdb_b200.h: sdb_expire).  archive=True returns the expired records in receive_compact's shape,
        (counts, entries, sends, payload) - what does not fit stays queued, so loop until no entry comes back;
        archive=False drops them on the device and returns (counts, total)."""
        a, n, counts = self._agents_arg(agents)
        total, n_sends, pbytes = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
        ent = snd = pay = None
        if archive:
            ent, snd, pay = self._compact_outputs(out_entries, out_sends, out_payload)
        self._check(self._L.sdb_expire(self._h, n, _p(a), float(older_than), flags, _p(counts),
                                       _p(ent), 0 if ent is None else len(ent), _p(snd), 0 if snd is None else len(snd),
                                       _p(pay), 0 if pay is None else pay.nbytes,
                                       C.cast(C.byref(total), C.c_void_p), C.cast(C.byref(n_sends), C.c_void_p),
                                       C.cast(C.byref(pbytes), C.c_void_p)))
        if agents is None:
            counts = self._served_counts(counts, flags)
        if not archive:
            return counts, int(total.value)
        return counts, ent[: total.value], snd[: n_sends.value], pay[: pbytes.value]

    def trim(self, agents, max_records: int = 0, max_bytes: int = 0, flags: int = 0, archive: bool = True,
             out_entries: Optional[np.ndarray] = None, out_sends: Optional[np.ndarray] = None,
             out_payload: Optional[np.ndarray] = None):
        """Cap each agent's pending queue at max_records records and max_bytes payload bytes (sum of pad32(len); 0: no
        limit) by retiring its oldest records, or with RECV_PRIORITY its lowest-priority ones first, without delivering
        them (include/swarmdb_b200.h: sdb_trim).  Returns expire's shapes: archive=True gives the trimmed records as
        (counts, entries, sends, payload) - loop until no entry comes back; archive=False drops them: (counts, total)."""
        a, n, counts = self._agents_arg(agents)
        total, n_sends, pbytes = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
        ent = snd = pay = None
        if archive:
            ent, snd, pay = self._compact_outputs(out_entries, out_sends, out_payload)
        self._check(self._L.sdb_trim(self._h, n, _p(a), int(max_records), int(max_bytes), flags, _p(counts),
                                     _p(ent), 0 if ent is None else len(ent), _p(snd), 0 if snd is None else len(snd),
                                     _p(pay), 0 if pay is None else pay.nbytes,
                                     C.cast(C.byref(total), C.c_void_p), C.cast(C.byref(n_sends), C.c_void_p),
                                     C.cast(C.byref(pbytes), C.c_void_p)))
        if agents is None:
            counts = self._served_counts(counts, flags)
        if not archive:
            return counts, int(total.value)
        return counts, ent[: total.value], snd[: n_sends.value], pay[: pbytes.value]

    def supersede(self, agents, flags: int = 0, archive: bool = True, out_entries: Optional[np.ndarray] = None,
                  out_sends: Optional[np.ndarray] = None, out_payload: Optional[np.ndarray] = None):
        """Keep, per agent and key (sender, group, type & TYPE_MASK) of the pending records sent with TYPEF_SUPERSEDE,
        only the newest one (largest seq, the later in the ring on a tie) and retire the others without delivering them
        (include/swarmdb_b200.h: sdb_supersede).  Returns trim's shapes: archive=True gives the superseded records as
        (counts, entries, sends, payload) - loop until no entry comes back; archive=False drops them: (counts, total)."""
        a, n, counts = self._agents_arg(agents)
        total, n_sends, pbytes = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
        ent = snd = pay = None
        if archive:
            ent, snd, pay = self._compact_outputs(out_entries, out_sends, out_payload)
        self._check(self._L.sdb_supersede(self._h, n, _p(a), flags, _p(counts),
                                          _p(ent), 0 if ent is None else len(ent), _p(snd), 0 if snd is None else len(snd),
                                          _p(pay), 0 if pay is None else pay.nbytes,
                                          C.cast(C.byref(total), C.c_void_p), C.cast(C.byref(n_sends), C.c_void_p),
                                          C.cast(C.byref(pbytes), C.c_void_p)))
        if agents is None:
            counts = self._served_counts(counts, flags)
        if not archive:
            return counts, int(total.value)
        return counts, ent[: total.value], snd[: n_sends.value], pay[: pbytes.value]

    def receive_where(self, agents, max_messages: int, flags: int = 0, filt: Optional[SdbFilter] = None,
                      drop: bool = False, out_hdr: Optional[np.ndarray] = None, out_payload: Optional[np.ndarray] = None,
                      id_hits: Optional[np.ndarray] = None, id_agent: Optional[np.ndarray] = None,
                      max_agent_bytes: int = 0, max_agent_tokens: int = 0):
        """Take (or with RECV_PEEK, only look at) the first max_messages pending records per agent that match `filt`
        (make_filter(); None matches every record), in delivery order (include/swarmdb_b200.h: sdb_receive_where).
        Returns receive_batch's (counts, headers, payload); what does not fit stays queued, so loop until nothing
        comes back.  drop=True retires the matches on the device without returning them: (counts, total).
        With an id clause (make_filter(ids=...)), id_hits / id_agent (u32 arrays, one per listed id) receive each id's
        matching records, counted before max_messages and the capacity cut, and the smallest agent holding one
        (NO_RECEIVER: none).  max_agent_bytes / max_agent_tokens (0: no limit) also cut each agent's take of the matches
        as receive_budget / receive_tokens cut a plain one (sdb_receive_where_budget)."""
        if filt is None:
            filt = make_filter()
        n_ids = int(filt.n_ids) if filt.fields & FILTER_IDS else 0
        for name, out in (("id_hits", id_hits), ("id_agent", id_agent)):
            if out is not None and (out.dtype != np.uint32 or out.shape != (n_ids,) or not out.flags.c_contiguous):
                raise ValueError(f"{name} must be a contiguous uint32 array of one entry per id ({n_ids})")
        a, n, counts = self._agents_arg(agents)
        total, pbytes = C.c_uint64(0), C.c_uint64(0)
        hdr = pay = None
        if drop:
            flags |= WHERE_DROP
        else:
            hdr = out_hdr if out_hdr is not None else self._grow_hdr()
            pay = out_payload if out_payload is not None else self._grow_pay()
        filt.id_hits, filt.id_agent = _p(id_hits), _p(id_agent)
        tail = (_p(counts), _p(hdr), 0 if hdr is None else len(hdr), _p(pay), 0 if pay is None else pay.nbytes,
                C.cast(C.byref(total), C.c_void_p), C.cast(C.byref(pbytes), C.c_void_p))
        try:
            if max_agent_bytes or max_agent_tokens:
                self._check(self._L.sdb_receive_where_budget(self._h, n, _p(a), max_messages, int(max_agent_bytes),
                                                             int(max_agent_tokens), flags, C.byref(filt), *tail))
            else:
                self._check(self._L.sdb_receive_where(self._h, n, _p(a), max_messages, flags, C.byref(filt), *tail))
        finally:
            filt.id_hits = filt.id_agent = None                    # the filter does not keep the caller's arrays
        if agents is None:
            counts = self._served_counts(counts, flags)
        if drop:
            return counts, int(total.value)
        return counts, hdr[: total.value], pay[: pbytes.value]

    def latency_server(self, enable: bool) -> None:
        """Start / stop the persistent low-latency dequeue server (single-agent receives then skip launch, sync and D2H)."""
        self._check(self._L.sdb_latency_server(self._h, 1 if enable else 0))

    def last_receive_totals(self):
        """(records, payload bytes) of the last receive call; waits for it."""
        total, pbytes = C.c_uint64(0), C.c_uint64(0)
        self._check(self._L.sdb_last_receive_totals(self._h, C.cast(C.byref(total), C.c_void_p), C.cast(C.byref(pbytes), C.c_void_p)))
        return total.value, pbytes.value

    # stream digests (definition in include/swarmdb_b200.h): order + content of every agent's stream, on the device
    def digest_reset(self) -> None:
        self._check(self._L.sdb_digest_reset(self._h))

    def digest_fold(self) -> None:
        """Fold the records of the last bulk receive (still on the device) into the per-agent digests."""
        self._check(self._L.sdb_digest_fold(self._h))

    def digest_read(self, agents=None) -> np.ndarray:
        if agents is None:
            a, n = None, self.max_agents
        else:
            a = _arr(agents, np.uint32)
            n = len(a)
        out = np.zeros(n, np.uint64)
        self._check(self._L.sdb_digest_read(self._h, n, _p(a), _p(out)))
        return out

    def receive_one(self, agent: int, max_messages: int = 100, flags: int = 0):
        """Latency path for a single agent (one kernel launch, one D2H): returns (headers, payload)
        views into reusable buffers.  Pre-built ctypes arguments keep the Python overhead minimal."""
        st = getattr(self, "_one", None)
        if st is None:
            mp = pad32(max(int(self.cfg.max_payload_bytes), 1))
            cap = max(1, min(1024, (1 << 22) // mp))          # records per call: a 4 MiB payload window
            hdr = np.zeros(cap, HDR_DTYPE)
            pay = np.zeros(cap * mp, np.uint8)
            a = np.zeros(1, np.uint32); cnt = np.zeros(1, np.uint32)
            total, pbytes = C.c_uint64(0), C.c_uint64(0)
            st = self._one = (a, cnt, hdr, pay, total, pbytes, _p(a), _p(cnt), _p(hdr), _p(pay),
                              C.cast(C.byref(total), C.c_void_p), C.cast(C.byref(pbytes), C.c_void_p), cap, pay.nbytes)
        a, cnt, hdr, pay, total, pbytes, pa, pc, ph, pp, pt, pb, cap, pcap = st
        a[0] = agent
        k = max_messages if max_messages <= cap else cap
        rc = self._L.sdb_receive_batch(self._h, 1, pa, k, flags, pc, ph, cap, pp, pcap, pt, pb)
        if rc != 0:
            self._check(rc)
        return hdr[: total.value], pay[: pbytes.value], k

    def stats_n_agents(self) -> int:
        return self.stats()["n_agents"]

    def _grow_hdr(self) -> np.ndarray:
        if len(self._out_hdr) < self.max_recv_records:
            self._out_hdr = np.zeros(self.max_recv_records, HDR_DTYPE)
        return self._out_hdr

    def _grow_pay(self) -> np.ndarray:
        need = int(self.cfg.max_recv_payload) or self.max_recv_records * 256
        if self._out_pay.nbytes < need:
            self._out_pay = np.zeros(need, np.uint8)
        return self._out_pay

    def _compact_outputs(self, out_entries, out_sends, out_payload):
        """(entries, sends, payload) output arrays of a compact-format call: the caller's, else reusable buffers."""
        if out_entries is None or out_sends is None:
            cur = getattr(self, "_out_ent", None)
            if cur is None or len(cur[0]) < self.max_recv_records:
                self._out_ent = (np.zeros(self.max_recv_records, ENTRY_DTYPE), np.zeros(self.max_recv_records, SEND_DTYPE))
        return (out_entries if out_entries is not None else self._out_ent[0],
                out_sends if out_sends is not None else self._out_ent[1],
                out_payload if out_payload is not None else self._grow_pay())

    def _agents_arg(self, agents, with_counts: bool = True):
        """(agent array or None, n_agents, zeroed counts) of a receive-family call; None means every agent."""
        if agents is None:
            return None, 0, np.zeros(self.max_agents, np.uint32) if with_counts else None
        a = _arr(agents, np.uint32)
        return a, len(a), np.zeros(len(a), np.uint32) if with_counts else None

    def _served_counts(self, counts, flags: int):
        """counts of a call without an agent list, cut to the agents it served: this shard's own with RECV_OWNED on a
        sharded handle, else every agent below the registration watermark."""
        owned = (flags & RECV_OWNED) and getattr(self, "n_owned", None) is not None
        return counts[: self.n_owned if owned else self.stats_n_agents()]

    def last_receive_dev(self) -> Tuple[int, int, int]:
        c, h, p = C.c_void_p(), C.c_void_p(), C.c_void_p()
        self._check(self._L.sdb_last_receive_dev(self._h, C.byref(c), C.byref(h), C.byref(p)))
        return c.value, h.value, p.value

    # ------------------------------------------------------------------ inbox / load queries from the rings (N3)
    def agent_loads(self, agents=None, n: Optional[int] = None) -> np.ndarray:
        """Per-agent `received` (inbox size), `pending` (unread) and its priority histogram, computed on the device."""
        if agents is None:
            a, cnt = None, int(n if n is not None else self.stats_n_agents())
        else:
            a = _arr(agents, np.uint32)
            cnt = len(a)
        out = np.zeros(cnt, LOAD_DTYPE)
        self._check(self._L.sdb_agent_loads(self._h, cnt, _p(a), _p(out)))
        return out

    def queue_stats(self) -> dict:
        raw = np.zeros(10, np.uint64)
        self._check(self._L.sdb_queue_stats(self._h, _p(raw)))
        d = {k: int(v) for k, v in zip(QSTATS_FIELDS, raw)}
        d["pending_by_prio"] = [d.pop("p0"), d.pop("p1"), d.pop("p2"), d.pop("p3")]
        return d

    def assign_agent_backends(self, agents, backends) -> None:
        a, b = _arr(agents, np.uint32), _arr(backends, np.uint32)
        self._check(self._L.sdb_assign_agent_backends(self._h, len(a), _p(a), _p(b)))

    def backend_loads_from_queues(self) -> None:
        """load[b] = pending records of the agents assigned to backend b (stream-ordered, no host round trip)."""
        self._check(self._L.sdb_backend_loads_from_queues(self._h))

    # ------------------------------------------------------------------ backends
    def set_backends(self, weight, load0=None) -> None:
        w = _arr(weight, np.uint32)
        l0 = None if load0 is None else _arr(load0, np.uint64)
        self._check(self._L.sdb_set_backends(self._h, len(w), _p(w), _p(l0)))
        self._nb = len(w)

    def backend_loads(self) -> np.ndarray:
        out = np.zeros(self._nb, np.uint64)
        self._check(self._L.sdb_get_backend_loads(self._h, self._nb, _p(out)))
        return out

    def release_backends(self, backend, cost=None) -> None:
        b = _arr(backend, np.uint32)
        c = None if cost is None else _arr(cost, np.uint32)
        self._check(self._L.sdb_release_backends(self._h, len(b), _p(b), _p(c)))

    def select_backends(self, n_req: int, cost=None, mode: int = 0, seed: int = 0) -> np.ndarray:
        c = None if cost is None else _arr(cost, np.uint32)
        out = np.zeros(n_req, np.uint32)
        self._check(self._L.sdb_select_backend_batch(self._h, n_req, _p(c), mode, seed, _p(out)))
        return out


def expand_compact(entries: np.ndarray, sends: np.ndarray, payload: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """(headers, payload) in receive_batch's format from a compact receive's (entries, sends, payload): record r takes
    seq and receiver from its entry, every other header field and its padded payload from row sends[entry.send]."""
    entries = np.asarray(entries, ENTRY_DTYPE)
    sends = np.asarray(sends, SEND_DTYPE)
    payload = np.asarray(payload, np.uint8)
    row = sends[entries["send"].astype(np.int64)]
    hdr = np.empty(len(entries), HDR_DTYPE)
    hdr["seq"], hdr["receiver"] = entries["seq"], entries["receiver"]
    for f in ("timestamp", "sender", "group", "len", "prio", "type"):
        hdr[f] = row[f]
    # padded payloads are whole 32-byte granules: granule k of record r is granule row.payload_off / 32 + k of the
    # compact payload, so one gather over granules builds the full stream
    glen = pad32(row["len"].astype(np.int64)) >> 5
    total = int(glen.sum())
    out = np.empty(total * 32, np.uint8)
    if total:
        dst_start = np.zeros(len(glen), np.int64)
        np.cumsum(glen[:-1], out=dst_start[1:])
        src = np.repeat((row["payload_off"].astype(np.int64) >> 5) - dst_start, glen) + np.arange(total, dtype=np.int64)
        gran = np.ascontiguousarray(payload[: len(payload) & ~31]).view("V32")
        out.view("V32")[:] = gran[src]
    return hdr, out


def payload_offsets(hdr: np.ndarray) -> np.ndarray:
    """Byte offset of each record's payload inside the packed payload stream of a receive."""
    pl = pad32(hdr["len"].astype(np.int64))
    off = np.zeros(len(hdr), np.int64)
    if len(hdr) > 1:
        np.cumsum(pl[:-1], out=off[1:])
    return off
