"""`SwarmsDB` - the reference's Python surface over GPU-resident per-agent rings.

Mirrors the public interface of the reference class (/root/reference/swarmdb/" main.py", tag
`M:`; signatures in SURVEY.md section 8b(i)): same method names, argument meaning, defaults, return
values and error behaviour for the hot path

    register_agent / deregister_agent   M:314-372
    send_message                        M:393-519
    receive_messages                    M:521-601
    broadcast_message                   M:810-850
    add_agent_group (= create_group)    M:1208-1227
    send_to_group                       M:1229-1279
    set_llm_load_balancing / assign_llm_backend / get_llm_backend   M:1281-1325

What changed underneath: the Kafka producer/consumer pair (M:192-204, M:334-345) and the
JSON envelope (M:466, M:575-576) are gone.  Sends are staged in a host buffer (the role of
the producer's `linger.ms` batching, M:197) and flushed as one mixed batch through the C ABI
(`swarmdb_b200._native.Shard` -> libswarmdb_b200.so -> sm_90a kernels); receives pop the
agent's ring on the device and decode the returned bytes.  There is no CPU fallback.

Bulk entry points for index-level traffic (`send_to_group_batch`, `send_batch`,
`receive_batch`, `select_llm_backends`) bypass per-message Python objects entirely.
"""
from __future__ import annotations

import bisect
import datetime
import hashlib
import heapq
import json
import os
import secrets
import time
import uuid
from dataclasses import dataclass
from enum import Enum
from pathlib import Path
from typing import Any, Callable, Dict, Iterable, List, Optional, Set, Tuple, Union

import numpy as np
from pydantic import BaseModel, Field

from . import _native
from ._native import (EXPIRE_ALL, FILTER_MAX_IDS, FILTER_MAX_KEYWORD, NO_GROUP, RECV_PEEK, RECV_PRIORITY, TYPE_MASK, TYPEF_EXTRAS, TYPEF_JSON, TYPEF_SUPERSEDE, TYPEF_TOKENS,
                      SdbError, Shard, make_filter, pad32, recv_capacity)


class RingOverflow(SdbError):
    """Some records of a flushed batch found their receiver's ring full.  `exact` tells whether the lost messages were
    identified (only they are FAILED) or the whole batch had to be marked."""
    exact = False


try:  # the reference logs through loguru; keep the same logger object when it is installed
    from loguru import logger
except Exception:  # pragma: no cover
    import logging

    logger = logging.getLogger("swarmdb_b200")


# ----------------------------------------------------------------------------- vocabularies (M:23-51)
class MessageType(str, Enum):
    CHAT = "chat"
    COMMAND = "command"
    FUNCTION_CALL = "function_call"
    FUNCTION_RESULT = "function_result"
    SYSTEM = "system"
    ERROR = "error"
    STATUS = "status"


class MessagePriority(int, Enum):
    LOW = 0
    NORMAL = 1
    HIGH = 2
    CRITICAL = 3


class MessageStatus(str, Enum):
    PENDING = "pending"
    DELIVERED = "delivered"
    READ = "read"
    PROCESSED = "processed"
    FAILED = "failed"


_TYPE_CODE = {t: i for i, t in enumerate(MessageType)}
_TYPE_BY_CODE = list(MessageType)


class Message(BaseModel):
    """Same eleven fields and defaults as the reference model (M:54-82)."""

    id: str = Field(default_factory=lambda: str(uuid.uuid4()))
    sender_id: str
    receiver_id: Optional[str] = None
    content: Union[str, Dict[str, Any], List[Any]]
    type: MessageType = MessageType.CHAT
    priority: MessagePriority = MessagePriority.NORMAL
    timestamp: float = Field(default_factory=time.time)
    status: MessageStatus = MessageStatus.PENDING
    metadata: Dict[str, Any] = Field(default_factory=dict)
    token_count: Optional[int] = None
    visible_to: List[str] = Field(default_factory=list)

    def to_dict(self) -> Dict[str, Any]:
        """Plain dict with enum fields flattened to their values (the intent of M:91-98)."""
        d = self.model_dump()
        d["type"], d["priority"], d["status"] = self.type.value, self.priority.value, self.status.value
        return d

    @classmethod
    def from_dict(cls, data: Dict[str, Any]) -> "Message":
        d = dict(data)
        if isinstance(d.get("type"), str):
            d["type"] = MessageType(d["type"])
        if isinstance(d.get("priority"), int):
            d["priority"] = MessagePriority(d["priority"])
        if isinstance(d.get("status"), str):
            d["status"] = MessageStatus(d["status"])
        return cls(**d)


@dataclass
class KafkaConfig:
    """Accepted for drop-in compatibility (M:114-127).  Only `num_partitions` has a meaning
    here (informational: the shard count comes from the process group); the other knobs
    configured librdkafka and are ignored."""

    bootstrap_servers: str = "localhost:9092"
    group_id: str = "agent_messaging_system"
    auto_offset_reset: str = "earliest"
    num_partitions: int = 3
    replication_factor: int = 1
    retention_ms: int = 604800000          # default cutoff of expire_pending()
    max_poll_interval_ms: int = 300000
    session_timeout_ms: int = 30000
    heartbeat_interval_ms: int = 10000
    consumer_timeout_ms: int = 1000


@dataclass
class GpuConfig:
    """Sizing of the GPU-resident queue (replaces broker-side capacity planning)."""

    device: int = 0
    max_agents: int = 1 << 16
    ring_slots: int = 256                 # pending messages per agent (power of two)
    arena_bytes: int = 1 << 28            # message log (power of two)
    max_payload_bytes: int = 32768
    max_groups: int = 4096
    member_pool_entries: int = 0          # 0: 4 x max_agents
    max_backends: int = 256
    flush_threshold: int = 4096           # buffered sends before an automatic flush
    max_recv_records: int = 1 << 16
    max_recv_payload: int = 1 << 26
    priority_dequeue: bool = False        # True: receive in (priority desc, arrival) order - extension
    deterministic_ids: bool = False       # True: ids are uuid.UUID(int=seq) (tests / reproducibility)
    id_nonce: Optional[int] = None        # high 64 bits of every id (must match across the ranks of a sharded deployment)
    fanout_variant: Optional[int] = None      # None: the library default (_native.DEFAULT_FANOUT_VARIANT)
    shard_id: int = 0                     # multi-GPU: this process's shard / total shards (see sharded.ShardedSwarmsDB)
    num_shards: int = 1
    lease_records: int = 0                # leased receives: device lease store entries (0: no store, no memory)
    lease_payload_bytes: int = 0          # ... and payload bytes (0: lease_records x pad32(max_payload_bytes))
    lease_max_deliveries: int = 0         # dead letters: deliveries after which a leased message is parked (0: no limit,
                                          # no counts); needs lease_records
    lease_ledger_entries: int = 0         # ... and the device ledger of redelivered records' counts (0: lease_records)
    arena_relocate: bool = False          # a flush the arena refuses relocates the agents that pin the log and retries once
    dedup_entries: int = 0                # deduplicated sends: device table of this many keys (0: off, no memory)
    dedup_window: float = 300.0           # ... seconds a key stays live after its send
    dedup_content: bool = False           # ... sends without a dedup_id are keyed by their content
    queue_max_messages: int = 0           # bounded queues: after every flush each agent keeps its newest this many
                                          # pending messages (0: no count cap)
    queue_max_bytes: int = 0              # ... and pending payload bytes, sum of pad32(len) (0: no byte cap)
    queue_trim_priority: bool = False     # ... dropping the lowest priority first (oldest first within a level)


def _check_lease_policy(g: GpuConfig) -> None:
    """The dead-letter settings of a GpuConfig, checked before any device work."""
    if not 0 <= g.lease_max_deliveries <= 0xFFFFFFFF:
        raise ValueError(f"GpuConfig.lease_max_deliveries={g.lease_max_deliveries} is outside [0, 2^32 - 1]")
    if not 0 <= g.lease_ledger_entries < (1 << 31):
        raise ValueError(f"GpuConfig.lease_ledger_entries={g.lease_ledger_entries} is outside [0, 2^31)")
    if g.lease_max_deliveries and not g.lease_records:
        raise ValueError("GpuConfig.lease_max_deliveries needs a lease store (GpuConfig.lease_records)")
    if g.lease_ledger_entries and not g.lease_max_deliveries:
        raise ValueError("GpuConfig.lease_ledger_entries is used only with GpuConfig.lease_max_deliveries")


def _check_queue_caps(g: GpuConfig) -> None:
    """The bounded-queue settings of a GpuConfig, checked before any device work."""
    if not isinstance(g.queue_max_messages, int) or not 0 <= g.queue_max_messages <= 0xFFFFFFFF:
        raise ValueError(f"GpuConfig.queue_max_messages={g.queue_max_messages!r} is not an integer in [0, 2^32 - 1]")
    if not isinstance(g.queue_max_bytes, int) or not 0 <= g.queue_max_bytes < (1 << 64):
        raise ValueError(f"GpuConfig.queue_max_bytes={g.queue_max_bytes!r} is not an integer in [0, 2^64)")
    if not isinstance(g.queue_trim_priority, bool):
        raise ValueError(f"GpuConfig.queue_trim_priority={g.queue_trim_priority!r} is not a bool")


def _trim_limits(max_messages: Optional[int], max_bytes: Optional[int]) -> Tuple[int, int]:
    """The (max_records, max_agent_bytes) of sdb_trim for trim_queues' arguments (None: no limit)."""
    for name, v, top in (("max_messages", max_messages, 0xFFFFFFFF), ("max_bytes", max_bytes, (1 << 64) - 1)):
        if v is not None and (isinstance(v, bool) or not isinstance(v, int) or not 1 <= v <= top):
            raise ValueError(f"{name}={v!r} is not None or an integer in [1, {top}]")
    if max_messages is None and max_bytes is None:
        raise ValueError("trim_queues needs max_messages or max_bytes (expire_pending or deregister_agent(purge=True) "
                         "empties queues)")
    return max_messages or 0, max_bytes or 0


def _check_supersede(supersede: Any) -> None:
    if not isinstance(supersede, bool):
        raise TypeError(f"supersede={supersede!r} is not a bool")


def _flagged(typ, n: int) -> np.ndarray:
    """Which of n index-level sends carry TYPEF_SUPERSEDE in their type (typ None: none)."""
    if typ is None:
        return np.zeros(n, bool)
    return np.broadcast_to((np.asarray(typ, np.int64) & TYPEF_SUPERSEDE) != 0, (n,))


def _encode_content(content: Any) -> (bytes, int):
    if isinstance(content, str):
        return content.encode("utf-8"), 0
    return json.dumps(content).encode("utf-8"), TYPEF_JSON


def _check_token_count(n: Any) -> None:
    if isinstance(n, bool) or not isinstance(n, (int, np.integer)) or not 0 <= n < (1 << 32):
        raise ValueError(f"token_count={n!r} is not an integer in [0, 2^32): the device carries it as a u32")


def _encode_payload(body: bytes, flags: int, extras: Dict[str, Any], token_count: Optional[int]) -> Tuple[bytes, int]:
    """Wire form of a message and its type flags: the content bytes, or with JSON extras (metadata, visibility)
    u32 content length | content | extras (TYPEF_EXTRAS); a token count goes in front of either as a u32 (TYPEF_TOKENS),
    where the device reads it."""
    if extras:
        payload = len(body).to_bytes(4, "little") + body + json.dumps(extras).encode("utf-8")
        flags |= TYPEF_EXTRAS
    else:
        payload = body
    if token_count is not None:
        payload = int(token_count).to_bytes(4, "little") + payload
        flags |= TYPEF_TOKENS
    return payload, flags


def _renumber_rows(entries, sends) -> Tuple[np.ndarray, np.ndarray]:
    """Rows of a compact-format result reordered by their smallest seq (unreferenced rows last), entries remapped.  A
    restore lays rows out in row order, so records restored in stream order then take the arena positions, and share the
    payloads, they had when they were sent."""
    ent = np.array(entries, _native.ENTRY_DTYPE)
    snd = np.asarray(sends, _native.SEND_DTYPE)
    rows = np.ascontiguousarray(ent["send"])                       # contiguous: ufunc.at over strided fields is ~20x slower
    smallest = np.full(len(snd), np.iinfo(np.uint64).max, np.uint64)
    np.minimum.at(smallest, rows, np.ascontiguousarray(ent["seq"]))
    order = np.argsort(smallest, kind="stable")
    inv = np.empty(len(order), np.uint32)
    inv[order] = np.arange(len(order), dtype=np.uint32)
    ent["send"] = inv[rows]
    return ent, snd[order]


def _compact_rows(entries, sends, payload) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """Only the rows `entries` name, in row order, with their padded payloads packed back to back."""
    ent = np.array(entries, _native.ENTRY_DTYPE)
    used, inv = np.unique(ent["send"].astype(np.int64), return_inverse=True)
    ent["send"] = inv.astype(np.uint32)
    snd = np.array(sends[used], _native.SEND_DTYPE)
    glen = pad32(snd["len"].astype(np.int64)) >> 5
    start = np.zeros(len(snd), np.int64)
    if len(snd) > 1:
        np.cumsum(glen[:-1], out=start[1:])
    src = np.repeat((snd["payload_off"].astype(np.int64) >> 5) - start, glen) + np.arange(int(glen.sum()), dtype=np.int64)
    pay = np.ascontiguousarray(payload[: len(payload) & ~31]).view("V32")[src].view(np.uint8).copy()
    snd["payload_off"] = (start << 5).astype(np.uint64)
    return ent, snd, pay


class _TransportAdmin:
    """What callers probe through `db.admin_client` (the REST health check lists topics as a liveness test,
    api.py:798): here the "topic" is the device queue and its "partitions" are the shards."""

    def __init__(self, db: "SwarmsDB") -> None:
        self._db = db

    def list_topics(self, timeout: Optional[float] = None):
        from types import SimpleNamespace
        self._db.shard.stats()                     # raises if the device transport is gone
        parts = {i: SimpleNamespace(id=i) for i in range(max(1, self._db.gpu_config.num_shards))}
        return SimpleNamespace(topics={self._db.base_topic: SimpleNamespace(partitions=parts)})


class SwarmsDB:
    """Agent message queue + LLM-backend balancer; reference-compatible surface (see module doc)."""

    def __init__(
        self,
        base_topic: str = "agent_messaging",
        config: Optional[KafkaConfig] = None,
        save_dir: Optional[Union[str, Path]] = None,
        auto_save: bool = True,
        save_interval: int = 300,
        max_messages_per_file: int = 10000,
        token_counter: Optional[Callable[[str], int]] = None,
        gpu_config: Optional[GpuConfig] = None,
        _shard: Any = None,
    ):
        self.base_topic = base_topic
        self.config = config or KafkaConfig()
        self.gpu_config = gpu_config or GpuConfig()
        g = self.gpu_config
        _check_lease_policy(g)
        _check_queue_caps(g)
        # the transport: constructing it fails loudly when the CUDA library or a device is missing
        self.shard = _shard if _shard is not None else Shard(
            max_agents=g.max_agents, ring_slots=g.ring_slots, arena_bytes=g.arena_bytes,
            max_payload_bytes=g.max_payload_bytes, max_groups=g.max_groups,
            member_pool_entries=g.member_pool_entries or 4 * g.max_agents, max_backends=g.max_backends,
            max_batch_sends=max(g.flush_threshold, 1), max_batch_payload=max(1 << 22, 2 * pad32(g.max_payload_bytes)),
            max_recv_records=g.max_recv_records, max_recv_payload=g.max_recv_payload, device=g.device,
            fanout_variant=g.fanout_variant, shard_id=g.shard_id, num_shards=g.num_shards)

        # local state, same names as the reference (M:210-233)
        self.messages: Dict[str, Message] = {}
        self.agent_inbox: Dict[str, List[str]] = {}
        self.message_count = 0
        self.registered_agents: Set[str] = set()
        self.metadata: Dict[str, Any] = {}
        self.token_counter = token_counter
        self.llm_load_balancing = False

        self.save_dir = Path(save_dir) if save_dir else Path(os.getcwd()) / "message_history"
        self.save_dir.mkdir(parents=True, exist_ok=True)
        self.auto_save = auto_save
        self.save_interval = save_interval
        self.max_messages_per_file = max_messages_per_file
        self.last_save_time = time.time()

        # index maps (the device only knows dense indices)
        self._agent_idx: Dict[str, int] = {}
        self._agent_name: List[str] = []
        self._group_idx: Dict[str, int] = {}
        self._group_name: List[str] = []
        self._group_snapshot: List[List[str]] = []
        self._backend_idx: Dict[str, int] = {}
        self._backend_name: List[str] = []
        self._id_hi = 0 if g.deterministic_ids else (((g.id_nonce if g.id_nonce is not None else secrets.randbits(63)) & ((1 << 63) - 1)) << 64)
        self._next_seq = 1                      # mirror of the handle's sequence counter
        self._list_cap = 2 * g.max_agents + 1024 - 8      # the handle's default list_pool_entries, minus slack
        self._seq_to_id: Dict[int, str] = {}
        # leased receives: message id -> [(agent index, lease id)] (a broadcast is leased by each of its receivers under
        # one id), and a heap of the deadlines set, so a receive sweeps only once one may have passed
        self._leases: Dict[str, List[Tuple[int, int]]] = {}
        self._lease_deadlines: List[float] = []
        if g.lease_records:
            self.shard.lease_reserve(g.lease_records, g.lease_payload_bytes or g.lease_records * pad32(g.max_payload_bytes))
        if g.lease_max_deliveries:
            self.shard.lease_set_policy(g.lease_max_deliveries, g.lease_ledger_entries or g.lease_records)
        # deduplicated sends: duplicate id -> the id of the message it matched, and the dedup_id of each keyed message
        self._dup_of: Dict[str, str] = {}
        self._dedup_ids: Dict[str, str] = {}
        if g.dedup_entries:
            if not g.dedup_window > 0:
                raise ValueError(f"GpuConfig.dedup_window={g.dedup_window} must be > 0 seconds")
            self.shard.dedup_reserve(g.dedup_entries, g.dedup_window)
        self._trimmed = 0                       # records the automatic queue caps dropped (get_stats()["trimmed"])
        self._superseded = 0                    # records superseding sends retired (get_stats()["superseded"])
        self._supersedes = False                # a flagged record was staged, sent or restored: passes after re-enqueues
        self._reset_buffer()
        self._closed = False
        self.admin_client = _TransportAdmin(self)          # M:202-204: callers only list topics through it
        logger.info(f"SwarmsDB (H100) initialized with base topic: {base_topic}")

    # ------------------------------------------------------------------ helpers
    def _reset_buffer(self) -> None:
        self._b_sender: List[int] = []
        self._b_kind: List[int] = []
        self._b_target: List[int] = []
        self._b_prio: List[int] = []
        self._b_type: List[int] = []
        self._b_len: List[int] = []
        self._b_off: List[int] = []
        self._b_ts: List[float] = []
        self._b_payload = bytearray()
        self._b_list_off: List[int] = [0]
        self._b_list_idx: List[int] = []
        self._b_msgs: List[Message] = []
        self._b_key: List[Tuple[int, int]] = []          # dedup key of each send, (0, 0): none
        self._b_seq0: List[int] = []                     # first seq of each send
        self._b_supersede: Set[int] = set()              # receivers of the buffered superseding sends
        self._b_first_seq = self._next_seq

    def _index(self, agent_id: str) -> int:
        i = self._agent_idx.get(agent_id)
        if i is None:
            i = len(self._agent_name)
            if i >= self.gpu_config.max_agents:
                raise RuntimeError(f"agent capacity exhausted (GpuConfig.max_agents={self.gpu_config.max_agents})")
            self._agent_idx[agent_id] = i
            self._agent_name.append(agent_id)
        return i

    def agent_index(self, agent_id: str) -> int:
        """Dense device index of an agent id (assigned on first mention)."""
        return self._index(agent_id)

    def _make_id(self, seq: int) -> str:
        h = "%032x" % (self._id_hi | seq)                 # same text as str(uuid.UUID(int=...)), 4x cheaper
        return f"{h[:8]}-{h[8:12]}-{h[12:16]}-{h[16:20]}-{h[20:]}"

    def _count_tokens(self, content: Any) -> int:          # M:295-307
        if self.token_counter is None:
            return 0
        text = json.dumps(content) if isinstance(content, (dict, list)) else str(content)
        return self.token_counter(text)

    def _stage(self, kind: int, sender: int, target: int, prio: int, type_code: int, payload: bytes, ts: float,
               key: Tuple[int, int] = (0, 0)) -> None:
        if len(payload) > self.gpu_config.max_payload_bytes:
            raise ValueError(f"encoded message is {len(payload)} bytes; GpuConfig.max_payload_bytes="
                             f"{self.gpu_config.max_payload_bytes}")
        self._b_key.append(key); self._b_seq0.append(self._next_seq)
        self._b_sender.append(sender); self._b_kind.append(kind); self._b_target.append(target)
        self._b_prio.append(prio); self._b_type.append(type_code); self._b_len.append(len(payload))
        self._b_off.append(len(self._b_payload)); self._b_ts.append(ts)
        self._b_payload += payload
        self._b_payload += b"\0" * (pad32(len(payload)) - len(payload))

    def flush(self) -> None:
        """Push every buffered send to the device (one mixed batch, call order preserved)."""
        n = len(self._b_sender)
        if n == 0:
            return
        msgs = self._b_msgs
        superseding = self._b_supersede
        keys = None                             # the keys the device used (deduplicated sends only)
        try:
            payload = np.frombuffer(bytes(self._b_payload) + b"\0" * 32, dtype=np.uint8)
            batch = (np.asarray(self._b_sender, np.uint32), np.asarray(self._b_kind, np.uint8),
                     np.asarray(self._b_target, np.uint32), np.asarray(self._b_list_off, np.uint64),
                     np.asarray(self._b_list_idx, np.uint32), np.asarray(self._b_prio, np.uint8),
                     np.asarray(self._b_type, np.uint8), np.asarray(self._b_len, np.uint16),
                     np.asarray(self._b_off, np.uint64), payload, np.asarray(self._b_ts, np.float64))
            g = self.gpu_config
            now = time.time()

            def send():
                if not g.dedup_entries:
                    return self.shard.send_mixed_batch(*batch), None, None
                return self.shard.send_mixed_batch_dedup(*batch, keys=np.asarray(self._b_key, np.uint64).reshape(-1, 2),
                                                         content=g.dedup_content, now=now)
            try:
                base, dup_of, keys = send()
            except SdbError as e:
                # a refused batch takes no sequence numbers and writes nothing (nor stores a key), so it can be sent
                # again as it is and gets the same verdicts
                if e.code != -5 or not self.gpu_config.arena_relocate:
                    raise
                self.relocate_pinned(self._batch_bound())
                base, dup_of, keys = send()
            if base != self._b_first_seq:
                raise RuntimeError(f"sequence mirror out of step: device {base}, host {self._b_first_seq}")
            if dup_of is not None:
                self._settle_duplicates(msgs, dup_of)
            st = self.shard.stats()
            if st["ring_overflow"] > getattr(self, "_seen_overflow", 0):
                lost = st["ring_overflow"] - getattr(self, "_seen_overflow", 0)
                self._seen_overflow = st["ring_overflow"]
                err = RingOverflow(-4, f"{lost} message(s) not enqueued: a receiver's ring is full "
                                       f"(GpuConfig.ring_slots={self.gpu_config.ring_slots})")
                err.exact = self._mark_overflowed(msgs, str(err))
                raise err
        except Exception as e:                  # M:501-519: mark FAILED, keep the error, re-raise
            if not (isinstance(e, RingOverflow) and e.exact):      # the device said which records were lost: only those failed
                for m in msgs:
                    m.status = MessageStatus.FAILED
                    m.metadata["error"] = str(e)
            if keys is not None:                # forget the keys of failed sends, so that a resend is accepted
                self._forget_failed(msgs, keys, dup_of)
            # ids already handed out stay used: the device counter moves up to the host's, never the other way
            self.shard.advance_seq(self._next_seq)
            self._reset_buffer()
            if isinstance(e, RingOverflow):     # the device took the batch but some records: they may supersede
                self._supersede_receivers(superseding)
            raise
        self._reset_buffer()
        self._supersede_receivers(superseding)
        self._apply_queue_caps()

    def _supersede_receivers(self, receivers) -> None:
        """The pass after a send: over the receivers of its superseding sends, nothing when there were none."""
        if receivers:
            self._supersede_pass(np.fromiter(sorted(receivers), dtype=np.uint32, count=len(receivers)))

    def _supersede_pass(self, agents: Optional[np.ndarray]) -> int:
        """sdb_supersede over `agents` (None: every agent below the watermark) in archive mode, call after call until
        nothing comes back.  Each retired copy that has a host record leaves its receiver's inbox and adds the receiver
        to metadata["superseded_for"]; the record stays in `messages` with its status.  Returns the records retired."""
        total = 0
        while True:
            cnt, ent, _, _ = self.shard.supersede(agents)
            if len(ent) == 0:
                break
            idx = agents if agents is not None else np.arange(len(cnt), dtype=np.uint32)
            for a, seq in zip(np.repeat(idx, cnt.astype(np.int64)).tolist(), ent["seq"].tolist()):
                m = self.messages.get(self._make_id(int(seq)))
                if m is None:
                    continue
                name = self._agent_name[a] if a < len(self._agent_name) else None
                inbox = self.agent_inbox.get(name)
                if inbox and m.id in inbox:
                    inbox.remove(m.id)
                m.metadata.setdefault("superseded_for", []).append(name)
            total += len(ent)
        self._superseded += total
        return total

    def _supersede_after_restore(self, flagged: bool = False) -> None:
        """The pass over every agent after a call that put records back (flagged: those records include one)."""
        self._supersedes = self._supersedes or bool(flagged)
        if self._supersedes:
            self._supersede_pass(None)

    def supersede_pending(self, agent_ids: Optional[Iterable[str]] = None) -> int:
        """Keep, per agent (default: every agent) and per (sender, group, message type), only the newest pending message
        among those sent with supersede=True, and drop the others without delivering them.  Host records are updated as
        after a flush: a dropped copy leaves its receiver's inbox and names it in metadata["superseded_for"].  Returns
        the number of records dropped."""
        agents = None if agent_ids is None else self._expire_scope(agent_ids)[0]
        self._pre_read()
        if agents is not None and len(agents) == 0:
            return 0
        return self._supersede_pass(agents)

    def _apply_queue_caps(self) -> None:
        """GpuConfig.queue_max_messages / queue_max_bytes: one drop-mode trim of every agent this instance serves."""
        g = self.gpu_config
        if g.queue_max_messages or g.queue_max_bytes:
            agents, flags = self._expire_scope(None)
            flags |= RECV_PRIORITY if g.queue_trim_priority else 0
            self._trimmed += self.shard.trim(agents, g.queue_max_messages, g.queue_max_bytes, flags, archive=False)[1]

    def _dedup_key(self, sender_id: str, dedup_id: Optional[str]) -> Tuple[int, int]:
        """The device key of a send: a 128-bit blake2b of sender_id NUL dedup_id (a dedup_id is scoped to its sender)."""
        if dedup_id is None:
            return (0, 0)
        if not self.gpu_config.dedup_entries:
            raise ValueError("dedup_id needs deduplication (GpuConfig.dedup_entries > 0)")
        d = hashlib.blake2b(f"{sender_id}\0{dedup_id}".encode("utf-8"), digest_size=16).digest()
        lo, hi = int.from_bytes(d[:8], "little"), int.from_bytes(d[8:], "little")
        return (lo, hi) if lo or hi else (1, 0)

    def _send_of(self, m: Message) -> int:
        """Index in the flushed batch of the send that carries message m."""
        return bisect.bisect_right(self._b_seq0, self._seq_of_id(m.id)) - 1

    def _settle_duplicates(self, msgs: List[Message], dup_of: np.ndarray) -> None:
        """The device wrote nothing for a duplicate send: its messages leave `messages` and the inboxes, and each names
        the message it matched (member j of a group send matches member j of the original)."""
        for m in msgs:
            i = self._send_of(m)
            d = int(dup_of[i])
            if not d:
                continue
            orig = self._make_id(d + self._seq_of_id(m.id) - self._b_seq0[i])
            self._dup_of[m.id] = orig
            m.metadata["duplicate_of"] = orig
            if self.messages.pop(m.id, None) is not None:
                self.message_count -= 1
            for a in ([m.receiver_id] if m.receiver_id is not None else list(self.agent_inbox)):
                inbox = self.agent_inbox.get(a)
                if inbox and m.id in inbox:
                    inbox.remove(m.id)

    def _forget_failed(self, msgs: List[Message], keys: np.ndarray, dup_of: np.ndarray) -> None:
        failed = sorted({self._send_of(m) for m in msgs if m.status == MessageStatus.FAILED})
        sel = [i for i in failed if not dup_of[i] and (keys["lo"][i] or keys["hi"][i])]
        if sel:
            self.shard.dedup_forget(keys[sel])

    def original_id(self, message_id: str) -> Optional[str]:
        """The id of the message a duplicate send matched (GpuConfig.dedup_entries), else None."""
        return self._dup_of.get(message_id)

    def _batch_bound(self) -> int:
        """Arena bytes the buffered batch can take at most: one header and one padded payload per copy."""
        total = 0
        for kind, target, n in zip(self._b_kind, self._b_target, self._b_len):
            if kind == 0:
                copies = 1
            elif kind == 1:
                copies = len(self._group_snapshot[target] or ())
            else:
                copies = self._b_list_off[target + 1] - self._b_list_off[target]
            total += copies * (32 + pad32(n))
        return total

    def relocate_pinned(self, free_bytes: int) -> dict:
        """Make room for at least `free_bytes` more at the arena tail by moving the queued messages of the agents that pin
        the log (idle, slow, crashed or deregistered receivers) to the tail, without delivering or dropping any
        (include/swarmdb_b200.h: sdb_arena_relocate).  Finds the lowest cut that leaves the room with dry runs, then
        relocates once and returns the device's summary.  Raises SdbError -5 (SDB_EARENA_FULL) and changes nothing when no
        cut does: the arena then holds too many live messages, and only receiving or expiring them frees it."""
        arena = int(self.gpu_config.arena_bytes)
        need = int(free_bytes)

        def short(tail: int, floor: int) -> int:           # bytes missing for `need` behind `tail` (the wrap rule included)
            skip = arena - tail % arena if tail % arena + need > arena else 0
            return tail + skip + need - floor - arena

        tail = self.shard.stats()["arena_tail_bytes"]
        cut = max(0, short(tail, 0))
        for step in range(8):
            # each step moves the cut to the floor the last dry run would have needed; the last one is at the tail
            cut = tail if step == 7 else min(cut, tail)
            s = self.shard.relocate(cut, peek=True)
            missing = short(s["tail_after"], s["floor_after"])
            if missing <= 0:
                return self.shard.relocate(cut)
            if cut >= tail:
                break
            cut = s["floor_after"] + missing
        raise SdbError(-5, f"relocation cannot free {need} bytes of the message arena: it is full of live messages "
                           f"(receive or expire them, or enlarge GpuConfig.arena_bytes)")

    def _mark_overflowed(self, msgs: List[Message], error: str) -> bool:
        """Delivery report for a batch that overflowed rings (M:374-391): the device logs (receiver, sequence number)
        of every dropped record (sdb_overflow_log).  Point-to-point and group messages have one record each (id <->
        sequence number): exactly those are marked FAILED, the rest of the batch stays DELIVERED.  A broadcast is one
        message with many copies: it stays DELIVERED, names the receivers that missed it in
        metadata["undelivered_to"] and leaves their inboxes (it is not unread for an agent that never got it).  Returns False when the log could not name every dropped record (more than its
        capacity in one batch): the caller then fails the whole batch, as before."""
        agents, seqs, dropped = self.shard.overflow_log()
        if dropped != len(seqs):
            return False
        in_batch = {id(m) for m in msgs}
        for a, sq in zip(agents.tolist(), seqs.tolist()):
            m = self.messages.get(self._make_id(int(sq)))
            if m is None or id(m) not in in_batch:
                return False
            if m.receiver_id is None:
                name = self._agent_name[a] if a < len(self._agent_name) else a
                m.metadata.setdefault("undelivered_to", []).append(name)
                inbox = self.agent_inbox.get(name)
                if inbox and m.id in inbox:          # never queued for this receiver: not unread there
                    inbox.remove(m.id)
            else:
                m.status = MessageStatus.FAILED
                m.metadata["error"] = error
        return True

    # ------------------------------------------------------------------ registry
    def register_agent(self, agent_id: str) -> None:
        if agent_id in self.registered_agents:
            return
        self.registered_agents.add(agent_id)
        self.agent_inbox.setdefault(agent_id, [])
        self.shard.register(self._index(agent_id))
        logger.debug(f"Agent {agent_id} registered with messaging system")

    def register_agents(self, agent_ids: Iterable[str]) -> np.ndarray:
        """Bulk registration; returns the dense indices."""
        idx = np.fromiter((self._index(a) for a in agent_ids), dtype=np.uint32)
        for a in agent_ids:
            if a not in self.registered_agents:
                self.registered_agents.add(a)
                self.agent_inbox.setdefault(a, [])
        if len(idx):
            self.shard.register(idx)
        return idx

    def deregister_agent(self, agent_id: str, purge: bool = False) -> None:
        """purge=True also drops every message still queued for the agent on the device, so that a departed agent
        stops pinning the message arena (the ring itself is kept, like the Kafka consumer-group offset)."""
        if agent_id not in self.registered_agents:
            logger.warning(f"Agent {agent_id} not registered")
            return
        self.registered_agents.remove(agent_id)
        self.shard.deregister(self._index(agent_id))
        if purge:
            agents, flags = self._expire_scope([agent_id])
            if len(agents):
                self._pre_read()
                self.shard.expire(agents, 0.0, flags | EXPIRE_ALL, archive=False)

    # ------------------------------------------------------------------ send
    def send_message(
        self,
        sender_id: str,
        content: Union[str, Dict[str, Any], List[Any]],
        receiver_id: Optional[str] = None,
        message_type: MessageType = MessageType.CHAT,
        priority: MessagePriority = MessagePriority.NORMAL,
        metadata: Optional[Dict[str, Any]] = None,
        visible_to: Optional[List[str]] = None,
        _group: int = NO_GROUP,
        dedup_id: Optional[str] = None,
        supersede: bool = False,
    ) -> str:
        """dedup_id: with GpuConfig.dedup_entries, a second send of the same sender with the same dedup_id inside the
        window is not queued; after the flush, original_id() names the message it matched.
        supersede: a later superseding send of the same sender and message type to the same receiver replaces this one
        while both are pending (a last-value queue for status reports, heartbeats, plans); each flush keeps the newest."""
        _check_supersede(supersede)
        key = self._dedup_key(sender_id, dedup_id)
        if sender_id not in self.registered_agents:
            self.register_agent(sender_id)
        if receiver_id is not None and receiver_id not in self.registered_agents:
            self.register_agent(receiver_id)
        token_count = self._count_tokens(content) if self.token_counter else None
        if token_count is not None:
            _check_token_count(token_count)

        seq = self._next_seq
        if not isinstance(content, (str, dict, list)):
            raise TypeError("content must be str, dict or list")
        # fields are normalised here, so pydantic's per-field validation (14 % of the reference's send cost) is skipped
        message = Message.model_construct(
            id=self._make_id(seq), sender_id=str(sender_id), receiver_id=receiver_id, content=content,
            type=MessageType(message_type), priority=MessagePriority(priority), timestamp=time.time(),
            status=MessageStatus.PENDING, metadata=dict(metadata or {}), token_count=token_count,
            visible_to=list(visible_to or []))
        if receiver_id is None and not message.visible_to:
            message.visible_to = list(self.registered_agents)           # M:449-450

        self.messages[message.id] = message
        self.message_count += 1
        if receiver_id is not None:
            if receiver_id in self.agent_inbox:
                self.agent_inbox[receiver_id].append(message.id)
        else:
            for agent_id in self.registered_agents:                      # M:461-463
                self.agent_inbox[agent_id].append(message.id)

        # wire form: content bytes (+ JSON extras for metadata / visible_to, + the token count)
        body, flags = _encode_content(content)
        extras: Dict[str, Any] = {}
        md = dict(message.metadata)
        if _group != NO_GROUP:
            md.pop("group", None)                                        # travels as header.group
        if md:
            extras["m"] = md
        if message.visible_to:
            extras.update(self._encode_visibility(message.visible_to))
        payload, flags = _encode_payload(body, flags, extras, token_count)
        type_code = _TYPE_CODE[MessageType(message_type)] | flags | (TYPEF_SUPERSEDE if supersede else 0)
        prio = int(MessagePriority(priority))
        sender = self._index(sender_id)
        recips: List[int] = []
        try:
            if receiver_id is not None:
                deliverable = (not message.visible_to) or (receiver_id in message.visible_to)    # M:579-585
                if deliverable:
                    recips = [self._index(receiver_id)]
                    self._stage(0, sender, recips[0], prio, type_code, payload, message.timestamp, key)
                else:      # in the log, matched by no consumer: an empty recipient list
                    self._stage_list(sender, [], prio, type_code, payload, message.timestamp, key)
            else:
                seen: Set[int] = set()
                for a in message.visible_to:
                    i = self._index(a)
                    if i not in seen:
                        seen.add(i); recips.append(i)
                self._stage_list(sender, recips, prio, type_code, payload, message.timestamp, key)
        except Exception as e:
            message.status = MessageStatus.FAILED
            message.metadata["error"] = str(e)
            raise
        self._next_seq += 1
        self._b_msgs.append(message)
        if supersede:
            self._supersedes = True
            self._b_supersede.update(recips)
        if dedup_id is not None:
            self._dedup_ids[message.id] = dedup_id
        message.status = MessageStatus.DELIVERED                          # delivery report, M:374-391
        self._after_send()
        return message.id

    def _encode_visibility(self, visible_to: List[str]) -> Dict[str, Any]:
        """How `visible_to` (M:82) travels inside each copy's payload.  Short lists go as names ("v").  A broadcast
        to (nearly) everybody would put O(agents) bytes into every one of O(agents) copies, so long lists travel
        as their COMPLEMENT over the dense agent indices known at send time: "vc" = [n, [indices < n that are NOT
        visible]] (sender, excluded and not-yet/no-longer registered agents).  Indices agree on every rank of a
        sharded deployment (the registry is replicated), so any receiver reconstructs the exact set."""
        if len(visible_to) <= 32:
            return {"v": visible_to}
        n = len(self._agent_name)
        vis = {self._agent_idx[a] for a in visible_to if a in self._agent_idx}
        if len(vis) != len(set(visible_to)):                  # names the registry has never seen: keep them literal
            return {"v": visible_to}
        comp = [i for i in range(n) if i not in vis]
        if len(comp) >= len(visible_to):
            return {"v": visible_to}
        return {"vc": [n, comp]}

    def _decode_visibility(self, extras: Dict[str, Any]) -> List[str]:
        if "vc" in extras:
            n, comp = extras["vc"]
            skip = set(comp)
            return [self._agent_name[i] for i in range(min(n, len(self._agent_name))) if i not in skip]
        return list(extras.get("v", []))

    def _stage_list(self, sender: int, recips: List[int], prio: int, type_code: int, payload: bytes, ts: float,
                    key: Tuple[int, int] = (0, 0)) -> None:
        # recipient lists (and the one-entry lists of buffered point-to-point sends) share the device's per-batch
        # list pool: flush first if this list would not fit beside what is already buffered
        if self._b_sender and len(self._b_list_idx) + len(recips) + len(self._b_sender) + 1 > self._list_cap:
            self.flush()
        self._stage(2, sender, len(self._b_list_off) - 1, prio, type_code, payload, ts, key)
        self._b_list_idx.extend(recips)
        self._b_list_off.append(len(self._b_list_idx))

    def _after_send(self) -> None:
        if len(self._b_sender) >= self.gpu_config.flush_threshold or len(self._b_payload) >= (1 << 21):
            self.flush()
        if self.auto_save and (time.time() - self.last_save_time > self.save_interval
                               or self.message_count % self.max_messages_per_file == 0):
            self.save_message_history()

    def broadcast_message(
        self,
        sender_id: str,
        content: Union[str, Dict[str, Any], List[Any]],
        message_type: MessageType = MessageType.CHAT,
        priority: MessagePriority = MessagePriority.NORMAL,
        metadata: Optional[Dict[str, Any]] = None,
        exclude_agents: Optional[List[str]] = None,
        dedup_id: Optional[str] = None,
        supersede: bool = False,
    ) -> str:
        excluded = set(exclude_agents or [])
        visible = [a for a in self.registered_agents if a != sender_id and a not in excluded]
        return self.send_message(sender_id=sender_id, content=content, receiver_id=None, message_type=message_type,
                                 priority=priority, metadata=metadata, visible_to=visible, dedup_id=dedup_id,
                                 supersede=supersede)

    # ------------------------------------------------------------------ groups
    def add_agent_group(self, group_name: str, agent_ids: List[str]) -> None:
        groups = self.metadata.setdefault("agent_groups", {})
        groups[group_name] = agent_ids                    # the caller's list object, like M:1223
        self._sync_group(group_name)
        logger.debug(f"Agent group '{group_name}' created with {len(agent_ids)} agents")

    create_group = add_agent_group

    def _sync_group(self, group_name: str) -> int:
        """Upload the group's member list if it is new or was mutated by the caller."""
        members = self.metadata["agent_groups"][group_name]
        g = self._group_idx.get(group_name)
        if g is None:
            g = len(self._group_name)
            if g >= self.gpu_config.max_groups:
                raise RuntimeError("group capacity exhausted (GpuConfig.max_groups)")
            self._group_idx[group_name] = g
            self._group_name.append(group_name)
            self._group_snapshot.append(None)
        if self._group_snapshot[g] != members:
            self.flush()                                   # earlier sends used the old membership
            self.shard.create_group(g, np.fromiter((self._index(a) for a in members), dtype=np.uint32,
                                                   count=len(members)))
            self._group_snapshot[g] = list(members)
        return g

    def send_to_group(
        self,
        sender_id: str,
        group_name: str,
        content: Union[str, Dict[str, Any], List[Any]],
        message_type: MessageType = MessageType.CHAT,
        priority: MessagePriority = MessagePriority.NORMAL,
        metadata: Optional[Dict[str, Any]] = None,
        dedup_id: Optional[str] = None,
        supersede: bool = False,
    ) -> List[str]:
        """supersede: as in send_message, per member: the newest pending superseding send of this sender and message
        type to the group is the one each member keeps."""
        _check_supersede(supersede)
        key = self._dedup_key(sender_id, dedup_id)
        groups = self.metadata.get("agent_groups", {})
        if group_name not in groups:
            logger.warning(f"Agent group '{group_name}' not found")
            return []
        members = groups[group_name]
        msg_metadata = metadata or {}
        msg_metadata["group"] = group_name               # mutates a non-empty caller dict, like M:1263-1264
        g = self._sync_group(group_name)

        if sender_id not in self.registered_agents:
            self.register_agent(sender_id)
        token_count = self._count_tokens(content) if self.token_counter else None
        if token_count is not None:
            _check_token_count(token_count)
        body, flags = _encode_content(content)
        md = {k: v for k, v in msg_metadata.items() if k != "group"}
        extras: Dict[str, Any] = {}
        if md:
            extras["m"] = md
        payload, flags = _encode_payload(body, flags, extras, token_count)
        base = self._next_seq
        now = time.time()
        mtype, mprio = MessageType(message_type), MessagePriority(priority)
        if not isinstance(content, (str, dict, list)):
            raise TypeError("content must be str, dict or list")
        ids: List[str] = []
        staged = False
        for j, agent_id in enumerate(members):
            if agent_id == sender_id:
                continue
            if agent_id not in self.registered_agents:
                self.register_agent(agent_id)
            m = Message.model_construct(
                id=self._make_id(base + j), sender_id=str(sender_id), receiver_id=agent_id, content=content,
                type=mtype, priority=mprio, metadata=dict(msg_metadata), token_count=token_count,
                timestamp=now, status=MessageStatus.DELIVERED, visible_to=[])
            self.messages[m.id] = m
            self.message_count += 1
            self.agent_inbox[agent_id].append(m.id)
            self._b_msgs.append(m)
            ids.append(m.id)
            staged = True
        if staged or members:
            self._stage(1, self._index(sender_id), g, int(MessagePriority(priority)),
                        _TYPE_CODE[MessageType(message_type)] | flags | (TYPEF_SUPERSEDE if supersede else 0), payload, now,
                        key)
            self._next_seq += len(members)
            if supersede:
                self._supersedes = True
                self._b_supersede.update(self._index(a) for a in members if a != sender_id)
        if ids:
            self._after_send()
        return ids

    # ------------------------------------------------------------------ receive
    def receive_messages(self, agent_id: str, max_messages: int = 100, timeout: float = 1.0,
                         max_bytes: Optional[int] = None, max_tokens: Optional[int] = None) -> List[Message]:
        """Pop up to `max_messages` pending messages for `agent_id` in stream order (or priority
        order with GpuConfig.priority_dequeue).  Never blocks: `timeout` is accepted for
        compatibility (the reference spins up to `timeout` when fewer are available, M:553-556).
        max_bytes bounds the encoded payload bytes returned: the longest run of pending messages, in delivery order,
        whose encoded payloads (each rounded up to 32 bytes) fit max_bytes, or the first message alone when it is
        larger.  max_tokens bounds their token counts the same way: as many pending messages as fit max_tokens tokens
        of a model's context, counted with the token_counter the messages were sent with (a message sent without a
        count weighs 0, so max_bytes is what bounds those).  The two combine: the shorter run wins.  One such call
        returns at most GpuConfig.max_recv_records messages and max_recv_payload bytes."""
        self._prepare_receive(agent_id)
        return self._receive_local(agent_id, max_messages, max_bytes, max_tokens)

    def _prepare_receive(self, agent_id: str) -> bool:
        """Before a receive for `agent_id`: register it if needed and push buffered sends (a sharded front-end checks
        ownership instead).  False when the agent can have nothing queued."""
        if agent_id not in self.registered_agents:
            logger.warning(f"Agent {agent_id} not registered, registering now")
            self.register_agent(agent_id)
        self.flush()
        return True

    @staticmethod
    def _budget_limits(max_bytes: Optional[int], max_tokens: Optional[int]) -> Tuple[int, int]:
        """The device's per-agent (byte, token) limits for max_bytes / max_tokens, 0 for None (no limit)."""
        if max_bytes is not None and max_bytes < 0:
            raise ValueError("max_bytes must be >= 0")
        if max_tokens is not None and not 0 < max_tokens < (1 << 64):
            raise ValueError("max_tokens must be positive (None: no token limit)")
        # the device reads 0 as "no limit"; a 1-byte limit takes the same records as a 0-byte one (sizes are multiples of 32)
        return (0 if max_bytes is None else max(int(max_bytes), 1)), (0 if max_tokens is None else int(max_tokens))

    def _receive_budget_one(self, agent_id: str, max_messages: int, max_bytes: Optional[int], flags: int,
                            max_tokens: Optional[int] = None):
        """(headers, payload) of one byte- and/or token-budget receive for one agent (Shard.receive_budget,
        Shard.receive_tokens)."""
        nbytes, _ = self._budget_limits(max_bytes, max_tokens)
        k = min(max_messages, self.shard.max_recv_records)
        if max_tokens is not None:
            _, hdr, pay = self.shard.receive_tokens([self._index(agent_id)], k, int(max_tokens), nbytes, flags)
        else:
            _, hdr, pay = self.shard.receive_budget([self._index(agent_id)], k, nbytes, flags)
        return hdr, pay

    def _receive_local(self, agent_id: str, max_messages: int, max_bytes: Optional[int] = None,
                       max_tokens: Optional[int] = None) -> List[Message]:
        if max_messages <= 0:
            return []
        flags = RECV_PRIORITY if self.gpu_config.priority_dequeue else 0
        if max_bytes is not None or max_tokens is not None:
            hdr, pay = self._receive_budget_one(agent_id, max_messages, max_bytes, flags, max_tokens)
            return self._decode(hdr, pay, agent_id)
        out: List[Message] = []
        a = self._index(agent_id)
        remaining = max_messages
        while remaining > 0:
            hdr, pay, k = self.shard.receive_one(a, remaining, flags)   # single-launch latency path of the C ABI
            if len(hdr) == 0:
                break
            out.extend(self._decode(hdr, pay, agent_id))
            remaining -= len(hdr)
            if len(hdr) < k:
                break
        return out

    # ------------------------------------------------------------------ leased receive (at-least-once delivery)
    def receive_messages_leased(self, agent_id: str, max_messages: int = 100, visibility_timeout: float = 30.0,
                                max_bytes: Optional[int] = None, max_tokens: Optional[int] = None) -> List[Message]:
        """receive_messages with at-least-once delivery: the messages read READ, and each stays owed until it is acked
        (ack_messages, mark_message_as_processed).  One not acked within `visibility_timeout` seconds goes back behind
        what the agent has pending and is delivered again, with its id (an SQS visibility timeout).  Expired leases are
        swept back first, so they are visible to this call.  max_bytes and max_tokens bound the take as in
        receive_messages (one call, at most GpuConfig.max_recv_records messages): an agent that builds a model's
        context from its queue gets as many messages as fit, and each comes back if the model call fails.  Needs
        GpuConfig.lease_records."""
        self._prepare_receive(agent_id)
        return self._receive_leased_local(agent_id, max_messages, visibility_timeout, max_bytes, max_tokens)

    def _receive_leased_local(self, agent_id: str, max_messages: int, visibility_timeout: float,
                              max_bytes: Optional[int] = None, max_tokens: Optional[int] = None,
                              filt=None) -> List[Message]:
        """Leased receives for one agent with the bookkeeping of receive_messages_leased; with a limit one call, else
        a loop until max_messages or nothing more.  `filt`: leases only the matching messages (Shard.receive_leased)."""
        limited = max_bytes is not None or max_tokens is not None
        nbytes, ntokens = self._budget_limits(max_bytes, max_tokens)
        now = time.time()
        self._sweep_due(now)
        if max_messages <= 0:
            return []
        flags = RECV_PRIORITY if self.gpu_config.priority_dequeue else 0
        a = self._index(agent_id)
        deadline = now + visibility_timeout
        select = {} if filt is None and not limited else {"max_agent_bytes": nbytes, "max_agent_tokens": ntokens, "filt": filt}
        out: List[Message] = []
        remaining = max_messages
        while remaining > 0:
            k = min(remaining, self.shard.max_recv_records) if limited else remaining
            try:
                _, ent, snd, pay, base = self.shard.receive_leased([a], k, deadline, flags, **select)
            except SdbError as e:
                if out and e.code == -6:                   # SDB_ECAPACITY
                    break                                  # the store is full: what was leased so far is returned
                raise
            if len(ent) == 0:
                break
            hdr, full = _native.expand_compact(ent, snd, pay)
            msgs = self._decode(hdr, full, agent_id)
            if self.gpu_config.lease_max_deliveries:       # one lookup per chunk: how often each message was delivered
                counts = self.shard.lease_deliveries(np.arange(base, base + len(ent), dtype=np.uint64)).tolist()
                for m, c in zip(msgs, counts):
                    m.metadata["delivery_count"] = int(c)
            for j, m in enumerate(msgs):
                self._leases.setdefault(m.id, []).append((a, base + j))
            out += msgs
            remaining -= len(ent)
            if limited:
                break
        if out:
            heapq.heappush(self._lease_deadlines, deadline)
        return out

    def receive_batch_leased(self, agent_idx=None, max_messages: int = 100, visibility_timeout: float = 30.0,
                             priority: Optional[bool] = None, max_bytes: Optional[int] = None,
                             max_tokens: Optional[int] = None, filt=None, **kw):
        """receive_batch_compact, leased (Shard.receive_leased): (counts, entries, sends, payload, lease_base); entry r
        holds lease lease_base + r, for settle_leases.  Index-level: no host message records.  max_bytes and
        max_tokens bound each agent's take as in receive_batch; `filt` (make_filter()) leases only matching records."""
        nbytes, ntokens = self._budget_limits(max_bytes, max_tokens)
        if max_bytes is not None or max_tokens is not None or filt is not None:
            kw.update(max_agent_bytes=nbytes, max_agent_tokens=ntokens, filt=filt)
        self.flush()
        pr = self.gpu_config.priority_dequeue if priority is None else priority
        deadline = time.time() + visibility_timeout
        res = self.shard.receive_leased(agent_idx, max_messages, deadline, RECV_PRIORITY if pr else 0, **kw)
        if len(res[1]):
            heapq.heappush(self._lease_deadlines, deadline)
        return res

    def settle_leases(self, lease_ids, op: int = _native.LEASE_ACK, deadline: float = 0.0) -> np.ndarray:
        """Bulk settle by lease id: op LEASE_ACK, or LEASE_RENEW with a new deadline (-inf: due now).  Returns one flag
        per id, 1 where the lease was live."""
        if op == _native.LEASE_RENEW:
            heapq.heappush(self._lease_deadlines, float(deadline))
        return self.shard.lease_settle(lease_ids, op, deadline)[0]

    def _agent_leases(self, agent_id: str, message_ids: Iterable[str]) -> List[int]:
        a = self._agent_idx.get(agent_id)
        return [lid for mid in message_ids for (x, lid) in self._leases.get(mid, []) if x == a]

    def _forget(self, agent_idx: Optional[int], message_ids: Iterable[str]) -> None:
        for mid in message_ids:
            left = [(x, lid) for (x, lid) in self._leases.get(mid, []) if agent_idx is not None and x != agent_idx]
            if left:
                self._leases[mid] = left
            else:
                self._leases.pop(mid, None)

    def ack_messages(self, agent_id: str, message_ids: Iterable[str]) -> int:
        """The agent is done with these messages: their leases are settled and never redelivered.  Returns how many were
        still leased (a message already redelivered, or never leased, counts 0)."""
        message_ids = list(message_ids)
        ids = self._agent_leases(agent_id, message_ids)
        n = int(self.shard.lease_settle(ids, _native.LEASE_ACK)[1]) if ids else 0
        self._forget(self._agent_idx.get(agent_id), message_ids)
        for mid in message_ids:
            if mid in self.messages:
                self.messages[mid].status = MessageStatus.PROCESSED
        return n

    def nack_messages(self, agent_id: str, message_ids: Iterable[str]) -> int:
        """Give the messages back now: the next sweep (the next leased receive, or redeliver_expired) redelivers them."""
        return self.extend_leases(agent_id, message_ids, visibility_timeout=-np.inf)

    def extend_leases(self, agent_id: str, message_ids: Iterable[str], visibility_timeout: float = 30.0) -> int:
        """Move the deadline of the agent's live leases on these messages to now + visibility_timeout."""
        ids = self._agent_leases(agent_id, message_ids)
        if not ids:
            return 0
        deadline = time.time() + visibility_timeout
        heapq.heappush(self._lease_deadlines, deadline)
        return int(self.shard.lease_settle(ids, _native.LEASE_RENEW, deadline)[1])

    def redeliver_expired(self, now: Optional[float] = None, all: bool = False) -> int:
        """Sweep every lease whose deadline has passed (all=True: every live lease) back to its agent's queue, behind
        what is pending.  Returns the messages redelivered; agents whose queue is full keep theirs leased."""
        self.flush()
        now = time.time() if now is None else now
        total = 0
        while True:
            red, blocked, left = self.shard.lease_sweep(now, _native.LEASE_ALL if all else 0)
            total += red
            if left == 0 or red == 0:
                break
        if not all and not blocked:
            while self._lease_deadlines and self._lease_deadlines[0] <= now:
                heapq.heappop(self._lease_deadlines)
        if total:
            self._supersede_after_restore()
        return total

    # ------------------------------------------------------------------ dead letters (GpuConfig.lease_max_deliveries)
    def _dead_letter_agents(self, agent_ids) -> Optional[np.ndarray]:
        if not self.gpu_config.lease_max_deliveries:
            raise SdbError(-1, "dead letters need GpuConfig.lease_max_deliveries")
        self.flush()
        return None if agent_ids is None else np.array([self._index(a) for a in agent_ids], np.uint32)

    def dead_letters(self, agent_id: Optional[str] = None, max_messages: int = 100, peek: bool = False) -> List[Message]:
        """Messages parked after GpuConfig.lease_max_deliveries deliveries without an ack, oldest lease first (agent by
        agent when agent_id is None): status FAILED and metadata["delivery_count"].  peek=False takes them out of the
        device store and marks the host's records FAILED, so resend_failed_messages sends them again as new messages;
        redrive_dead_letters puts them back with their ids instead."""
        agents = self._dead_letter_agents(None if agent_id is None else [agent_id])
        out: List[Message] = []
        while len(out) < max_messages:
            k = min(max_messages - len(out), self.shard.max_recv_records)
            cnt, ent, snd, pay, deliv = self.shard.lease_dead_letters(
                agents, _native.RECV_PEEK if peek else 0, out_entries=np.zeros(k, _native.ENTRY_DTYPE),
                out_sends=np.zeros(k, _native.SEND_DTYPE))
            if len(ent) == 0:
                break
            hdr, full = _native.expand_compact(ent, snd, pay)
            who = np.repeat(agents if agents is not None else np.arange(len(cnt), dtype=np.uint32), cnt.astype(np.int64))
            msgs = self._decode(hdr, full, agent_id or "", record=False, status=MessageStatus.FAILED)
            for m, c, a in zip(msgs, deliv.tolist(), who.tolist()):
                m.metadata["delivery_count"] = int(c)
                if not peek:
                    if m.id in self.messages:
                        self.messages[m.id].status = MessageStatus.FAILED
                    else:
                        self.messages[m.id] = m
                    self._forget(a, [m.id])
            out += msgs
            if peek:
                break
        return out

    def redrive_dead_letters(self, agent_ids: Optional[Iterable[str]] = None) -> int:
        """Put dead letters back behind what their agents have pending, with their ids (a redrive); their delivery counts
        start again at 1.  Each chunk is restored before it leaves the dead-letter store, so a refused restore (a full
        ring) loses nothing.  Returns the messages redriven."""
        agents = self._dead_letter_agents(None if agent_ids is None else list(agent_ids))
        total = 0
        while True:
            cnt, ent, snd, pay, _ = self.shard.lease_dead_letters(agents, _native.RECV_PEEK)
            if len(ent) == 0:
                return total
            idx = agents if agents is not None else np.arange(len(cnt), dtype=np.uint32)
            ids = [self._make_id(int(x)) for x in ent["seq"].tolist()]
            who = np.repeat(idx, cnt.astype(np.int64)).tolist()
            n, seq_end = self.shard.restore_compact(idx, cnt, ent, snd, pay)
            self._next_seq = max(self._next_seq, seq_end); self._b_first_seq = self._next_seq
            taken = self.shard.lease_dead_letters(agents, 0)[1]
            assert len(taken) == n, (len(taken), n)                 # the same chunk: nothing changed the store between
            for a, mid in zip(who, ids):
                self._forget(a, [mid])
            total += n
            self._supersede_after_restore()

    def _sweep_due(self, now: float) -> None:
        if self._lease_deadlines and self._lease_deadlines[0] <= now:
            self.redeliver_expired(now)

    def _pre_read(self) -> None:
        """Make buffered sends visible before a read (a sharded front-end reads only what earlier collective
        flushes delivered, so it overrides this with a no-op)."""
        self.flush()

    def peek_messages(self, agent_id: str, max_messages: int = 100, max_bytes: Optional[int] = None,
                      max_tokens: Optional[int] = None) -> List[Message]:
        """What `receive_messages` (with the same max_bytes and max_tokens) would return next, without consuming it
        (device PEEK receive)."""
        self._pre_read()
        flags = RECV_PEEK | (RECV_PRIORITY if self.gpu_config.priority_dequeue else 0)
        if max_bytes is not None or max_tokens is not None:
            if max_messages <= 0:
                return []
            hdr, pay = self._receive_budget_one(agent_id, max_messages, max_bytes, flags, max_tokens)
        else:
            hdr, pay, _ = self.shard.receive_one(self._index(agent_id), max_messages, flags)
        return self._decode(hdr, pay, agent_id, record=False, status=MessageStatus.DELIVERED)

    def _where_filter(self, sender_id=None, receiver_idx=None, message_type=None, min_priority=None, group_name=None,
                      after_timestamp=None, before_timestamp=None, keyword=None, case_sensitive=True, message_ids=None):
        """The device filter (make_filter) for these host-level clauses, or None when an unknown sender or group, or
        message ids none of which this instance issued, make it match nothing."""
        kw = {}
        if message_ids is not None:
            seqs = [s for s in map(self._seq_of_id, message_ids) if s is not None]
            if not seqs:
                return None
            kw["ids"] = np.array(seqs, np.uint64)
        if sender_id is not None:
            if sender_id not in self._agent_idx:
                return None
            kw["sender"] = self._agent_idx[sender_id]
        if receiver_idx is not None:
            kw["receiver"] = receiver_idx
        if message_type is not None:
            kw["types"] = [_TYPE_CODE[MessageType(message_type)]]
        if min_priority is not None:
            kw["prios"] = range(int(MessagePriority(min_priority)), 4)
        if group_name is not None:
            if group_name not in self._group_idx:
                return None
            kw["group"] = self._group_idx[group_name]
        if after_timestamp is not None or before_timestamp is not None:
            kw["after"], kw["before"] = after_timestamp, before_timestamp
        if keyword is not None:
            kw["keyword"], kw["icase"] = keyword, not case_sensitive
        return make_filter(**kw)

    def receive_matching(self, agent_id: str, max_messages: int = 100, *, sender_id: Optional[str] = None,
                         message_type: Optional[MessageType] = None, min_priority: Optional[MessagePriority] = None,
                         group_name: Optional[str] = None, after_timestamp: Optional[float] = None,
                         before_timestamp: Optional[float] = None, keyword: Optional[str] = None,
                         case_sensitive: bool = False, message_ids: Optional[Iterable[str]] = None,
                         max_bytes: Optional[int] = None, max_tokens: Optional[int] = None, leased: bool = False,
                         visibility_timeout: float = 30.0) -> List[Message]:
        """A selective receive_messages: pop up to `max_messages` of the agent's pending messages that match every
        given clause, in stream order (priority order with GpuConfig.priority_dequeue), with receive_messages'
        bookkeeping; the other messages stay queued in their order.  The timestamp bounds are strict.  `keyword` must
        occur in the message content (its UTF-8 text; JSON content as json.dumps gives it), at most 256 bytes; the
        case-insensitive compare folds ASCII letters only.  `message_ids` takes those specific messages (ids this
        instance did not issue match nothing).  max_bytes and max_tokens bound the take of the matches as in
        receive_messages (one call, at most GpuConfig.max_recv_records messages).  leased=True takes the matches with
        receive_messages_leased's at-least-once delivery and `visibility_timeout`."""
        limits = self._budget_limits(max_bytes, max_tokens)
        limited = max_bytes is not None or max_tokens is not None
        if message_ids is not None:
            message_ids = list(message_ids)
            if len(message_ids) > FILTER_MAX_IDS:
                raise ValueError(f"more than {FILTER_MAX_IDS} message ids")
        if keyword is not None and len(keyword.encode("utf-8")) > FILTER_MAX_KEYWORD:
            raise ValueError(f"keyword longer than {FILTER_MAX_KEYWORD} bytes")     # taken records cannot be re-checked
        if not self._prepare_receive(agent_id):
            return []
        filt = self._where_filter(sender_id, None, message_type, min_priority, group_name, after_timestamp,
                                  before_timestamp, keyword, case_sensitive, message_ids)
        if max_messages <= 0 or filt is None:
            return []
        if leased:
            return self._receive_leased_local(agent_id, max_messages, visibility_timeout, max_bytes, max_tokens, filt)
        flags = RECV_PRIORITY if self.gpu_config.priority_dequeue else 0
        a = np.array([self._index(agent_id)], np.uint32)
        if limited:
            _, hdr, pay = self.shard.receive_where(a, min(max_messages, self.shard.max_recv_records), flags, filt,
                                                   max_agent_bytes=limits[0], max_agent_tokens=limits[1])
            return self._decode(hdr, pay, agent_id)
        out: List[Message] = []
        while len(out) < max_messages:
            _, hdr, pay = self.shard.receive_where(a, max_messages - len(out), flags, filt)
            if len(hdr) == 0:
                break
            out.extend(self._decode(hdr, pay, agent_id))
        return out

    def _device_agents(self) -> np.ndarray:
        """Indices of the agents whose device queues this instance reads (a sharded rank: the ones it owns)."""
        agents, _ = self._expire_scope(self._agent_name)
        return agents

    def _device_matches(self, filt, need: int, accept: Callable[[Message], bool],
                        agents: Optional[np.ndarray] = None) -> List[Message]:
        """The newest (highest sequence number) `need` device-pending messages that match `filt` (PEEK receives: nothing
        is consumed), pass `accept` and have no host record (a host record wins over its device copy), one per id (the
        copies of a broadcast share one).  Each call's records are decoded newest first and only until `need` of them
        are taken: a message among the overall newest `need` is also among the newest `need` taken from its own call,
        so the Python work is bounded by `need` and the rejected candidates, not by the number of matches."""
        self._pre_read()
        if filt is None or need <= 0:
            return []
        found: Dict[int, Message] = {}
        seen = set()
        for part, cap in self._pending_chunks(self._device_agents() if agents is None else agents, 1 << 31):
            _, hdr, pay = self.shard.receive_where(part, cap, RECV_PEEK, filt)
            offs = _native.payload_offsets(hdr)
            seqs = hdr["seq"]
            taken = 0
            for i in np.argsort(seqs, kind="stable")[::-1].tolist():
                seq = int(seqs[i])
                if seq in seen:
                    continue
                seen.add(seq)
                m = self._decode(hdr[i:i + 1], pay[int(offs[i]):], "", record=False, status=MessageStatus.DELIVERED)[0]
                if m.id in self.messages or not accept(m):
                    continue
                found[seq] = m
                taken += 1
                if taken >= need:
                    break
        return [found[k] for k in sorted(found, reverse=True)[:need]]

    def pending_snapshot(self, per_agent: int = 1024) -> Dict[str, List[Message]]:
        """Every message still queued on the device, per agent, in delivery order (non-destructive).
        This is the D2H ring dump behind `save_message_history(include_device=True)`."""
        self._pre_read()
        n = len(self._agent_name)
        out: Dict[str, List[Message]] = {}
        if n == 0:
            return out
        flags = RECV_PEEK | (RECV_PRIORITY if self.gpu_config.priority_dequeue else 0)
        for part, cap in self._pending_chunks(np.arange(n, dtype=np.uint32), per_agent):
            counts, hdr, pay = self.shard.receive_batch(part, min(per_agent, cap), flags)
            offs = _native.payload_offsets(hdr)
            pos = 0
            for a, c in zip(part, counts):
                c = int(c)
                if c:
                    name = self._agent_name[int(a)]
                    sub_pay = pay[int(offs[pos]):] if pos < len(offs) else pay[:0]
                    out[name] = self._decode(hdr[pos:pos + c], sub_pay, name, record=False, status=MessageStatus.DELIVERED)
                pos += c
        return out

    def _pending_chunks(self, agents: np.ndarray, per_agent: int):
        """Yield (agent list, record capacity): consecutive parts of `agents` whose pending messages (at most per_agent
        each) fit one receive call.  A call holds min(max_recv_records, max_recv_payload / padded payload) records and
        leaves out whole agents beyond that; a PEEK consumes nothing, so a fixed chunking would silently skip them.  The
        parts are packed from the agents' pending counts instead (one device query)."""
        cap = recv_capacity(self.gpu_config)
        if len(agents) == 0:
            return
        pending = np.minimum(self.shard.agent_loads(agents)["pending"][: len(agents)].astype(np.int64), per_agent)
        busy = np.nonzero(pending)[0]
        b = 0
        while b < len(busy):
            e, room = b, cap
            while e < len(busy) and (pending[busy[e]] <= room or e == b):
                room -= int(pending[busy[e]]); e += 1
            if e == b + 1 and pending[busy[b]] > cap:
                logger.warning(f"agent {self._agent_name[int(agents[busy[b]])]} has more pending messages than one receive "
                               f"call holds ({cap}); only the first {cap} are read")
            yield agents[busy[b:e]].astype(np.uint32), cap
            b = e

    def _decode(self, hdr: np.ndarray, pay: np.ndarray, agent_id: str, record: bool = True,
                status: MessageStatus = MessageStatus.READ) -> List[Message]:
        msgs: List[Message] = []
        n = len(hdr)
        if n == 0:
            return msgs
        offs = _native.payload_offsets(hdr).tolist()
        raw = pay.tobytes()
        # column-wise conversion once: per-record structured-array field access dominates otherwise
        seqs, lens, types, prios = hdr["seq"].tolist(), hdr["len"].tolist(), hdr["type"].tolist(), hdr["prio"].tolist()
        senders, receivers, groups, stamps = (hdr["sender"].tolist(), hdr["receiver"].tolist(), hdr["group"].tolist(),
                                              hdr["timestamp"].tolist())
        names = self._agent_name
        for k in range(n):
            blob = raw[offs[k]: offs[k] + lens[k]]
            t = types[k]
            tokens = None
            if t & TYPEF_TOKENS:
                tokens, blob = int.from_bytes(blob[:4], "little"), blob[4:]
            extras: Dict[str, Any] = {}
            if t & TYPEF_EXTRAS:
                clen = int.from_bytes(blob[:4], "little")
                body, extras = blob[4:4 + clen], json.loads(blob[4 + clen:].decode("utf-8"))
            else:
                body = blob
            content: Any = json.loads(body.decode("utf-8")) if t & TYPEF_JSON else body.decode("utf-8")
            metadata = dict(extras.get("m", {})) if extras else {}
            grp = groups[k]
            if grp != NO_GROUP:
                metadata["group"] = self._group_name[grp]
            receiver = receivers[k]
            m = Message.model_construct(
                id=self._make_id(seqs[k]), sender_id=names[senders[k]],
                receiver_id=None if receiver == _native.NO_RECEIVER else names[receiver],
                content=content, type=_TYPE_BY_CODE[t & TYPE_MASK], priority=MessagePriority(prios[k]),
                timestamp=stamps[k], status=status, metadata=metadata,
                token_count=tokens if tokens is not None else (extras.get("t") if extras else None), visible_to=self._decode_visibility(extras) if extras else [])
            if record:
                self.messages[m.id] = m                    # M:587-588
            msgs.append(m)
        return msgs

    # ------------------------------------------------------------------ bulk (index-level) API
    def send_batch(self, sender_idx, receiver_idx, prio, typ, lens, payload_off, payload, ts=None) -> int:
        self.flush()
        base = self.shard.send_batch(sender_idx, receiver_idx, prio, typ, lens, payload_off, payload, ts)
        self._next_seq = base + len(np.atleast_1d(sender_idx)); self._b_first_seq = self._next_seq
        flagged = _flagged(typ, len(np.atleast_1d(sender_idx)))
        if flagged.any():
            self._supersedes = True
            self._supersede_receivers(set(np.broadcast_to(np.asarray(receiver_idx, np.int64), flagged.shape)[flagged].tolist()))
        return base

    def send_to_group_batch(self, sender_idx, group_idx, prio, typ, lens, payload_off, payload, ts=None) -> int:
        self.flush()
        base = self.shard.send_group_batch(sender_idx, group_idx, prio, typ, lens, payload_off, payload, ts)
        self._next_seq = self.shard.stats()["next_seq"]; self._b_first_seq = self._next_seq
        flagged = _flagged(typ, len(np.atleast_1d(sender_idx)))
        if flagged.any():
            self._supersedes = True
            groups = set(np.broadcast_to(np.asarray(group_idx, np.int64), flagged.shape)[flagged].tolist())
            known = [self._group_snapshot[k] for k in groups if k < len(self._group_snapshot)]
            if len(known) == len(groups) and all(m is not None for m in known):
                self._supersede_receivers({self._agent_idx[a] for m in known for a in m if a in self._agent_idx})
            else:                               # a group this instance did not create: every agent
                self._supersede_pass(None)
        return base

    def receive_batch(self, agent_idx=None, max_messages: int = 100, priority: Optional[bool] = None,
                      max_bytes: Optional[int] = None, max_tokens: Optional[int] = None, **kw):
        """max_bytes: each agent takes at most that many encoded payload bytes (each payload rounded up to 32 bytes; an
        oversized first message alone; 0: no per-agent limit) and the call is sized by the bytes it selects
        (Shard.receive_budget).  max_tokens: each agent's take is also cut where its token counts would pass
        max_tokens (a heavier first message alone; messages without a count weigh 0; 0: no token limit;
        Shard.receive_tokens).  None for both keeps the plain receive."""
        self.flush()
        pr = self.gpu_config.priority_dequeue if priority is None else priority
        if max_tokens is not None:
            return self.shard.receive_tokens(agent_idx, max_messages, int(max_tokens), int(max_bytes or 0),
                                             RECV_PRIORITY if pr else 0, **kw)
        if max_bytes is not None:
            return self.shard.receive_budget(agent_idx, max_messages, int(max_bytes), RECV_PRIORITY if pr else 0, **kw)
        return self.shard.receive_batch(agent_idx, max_messages, RECV_PRIORITY if pr else 0, **kw)

    def receive_batch_compact(self, agent_idx=None, max_messages: int = 100, priority: Optional[bool] = None,
                              max_bytes: Optional[int] = None, max_tokens: Optional[int] = None, **kw):
        """receive_batch's records in the compact format: (counts, entries, sends, payload) with each distinct
        payload once (Shard.receive_compact; _native.expand_compact gives receive_batch's (headers, payload)).
        max_bytes and max_tokens as in receive_batch; bytes are counted per message, shared payloads included."""
        self.flush()
        pr = self.gpu_config.priority_dequeue if priority is None else priority
        if max_tokens is not None:
            return self.shard.receive_compact_tokens(agent_idx, max_messages, int(max_tokens), int(max_bytes or 0),
                                                     RECV_PRIORITY if pr else 0, **kw)
        return self.shard.receive_compact(agent_idx, max_messages, RECV_PRIORITY if pr else 0,
                                          max_agent_bytes=None if max_bytes is None else int(max_bytes), **kw)

    def requeue_batch_compact(self, counts, entries, sends, payload, agent_idx) -> int:
        """The nack of receive_batch_compact: put what a compact receive took (or any input of that shape: agent_idx[i]
        owns the next counts[i] entries) back behind what each agent has pending, with the original message ids.  Rows are
        renumbered by their smallest seq first, so records requeued in stream order share payloads as they did.
        All or nothing (Shard.restore_compact).  Returns the records requeued."""
        self.flush()
        ent, snd = _renumber_rows(entries, sends)
        n, seq_end = self.shard.restore_compact(agent_idx, counts, ent, snd, payload)
        self._next_seq = max(self._next_seq, seq_end); self._b_first_seq = self._next_seq
        self._supersede_after_restore(bool(np.any(np.asarray(snd["type"]) & TYPEF_SUPERSEDE)))
        return n

    # ------------------------------------------------------------------ queue snapshots (restart persistence)
    SNAPSHOT_VERSION = 1
    SNAPSHOT_VERSION_IN_FLIGHT = 2          # format 1 + the lease store and the redelivery ledger

    def save_queue_snapshot(self, path: Union[str, Path], in_flight: bool = False) -> Path:
        """Write every message pending on the device to one .npz file (no pickle) that load_queue_snapshot puts back
        into a fresh instance: the agent and group tables in index order, the id nonce, the sequence counter and the
        pending records as PEEK compact receives in stream order (rows renumbered by smallest seq).  Nothing is
        consumed.  An agent with more pending records than one receive call holds raises: a snapshot is complete or it
        is not written.  Leased messages not yet acked are in flight, not pending, and are not in the snapshot: call
        redeliver_expired(all=True) first to include them.

        in_flight=True (needs GpuConfig.lease_records) writes format 2 instead: the same, plus every live lease and dead
        letter with its deadline and delivery count, and the delivery counts of redelivered messages still pending, so a
        restart keeps at-least-once delivery: leases not yet acked can still be acked or are redelivered when due, dead
        letters stay parked, and counts continue.  Nothing on the device changes."""
        self.flush()
        g = self.gpu_config
        if in_flight and not g.lease_records:
            raise ValueError("save_queue_snapshot(in_flight=True) needs a lease store (GpuConfig.lease_records)")
        if g.lease_records and not in_flight:
            live = self.shard.lease_stats()["live"]
            if live:
                logger.warning(f"queue snapshot leaves out {live} leased messages in flight "
                               f"(redeliver_expired(all=True) first to include them)")
            dead = self.shard.lease_policy_stats()["dead"] if g.lease_max_deliveries else 0
            if dead:
                logger.warning(f"queue snapshot leaves out {dead} dead letters (redrive_dead_letters() first to include them)")
        cap = recv_capacity(g)
        agents = np.arange(len(self._agent_name), dtype=np.uint32)
        parts: List[Tuple[np.ndarray, ...]] = []
        if len(agents):
            pending = self.shard.agent_loads(agents)["pending"][: len(agents)].astype(np.int64)
            deep = np.nonzero(pending > cap)[0]
            if len(deep):
                raise RuntimeError(f"agent {self._agent_name[int(agents[deep[0]])]} has {int(pending[deep[0]])} pending "
                                   f"messages, more than one receive call holds ({cap}): no snapshot written")
            for part, _ in self._pending_chunks(agents, cap):
                cnt, ent, snd, pay = self.shard.receive_compact(part, cap, RECV_PEEK)
                ent, snd = _renumber_rows(ent, snd)
                parts.append((part, cnt.astype(np.uint32), ent, snd, pay.copy()))
        off = np.zeros((len(parts) + 1, 4), np.uint64)          # chunk k: agents, entries, rows, payload bytes
        for k, (a, _, e, s, p) in enumerate(parts):
            off[k + 1] = off[k] + [len(a), len(e), len(s), len(p)]
        snd_all = np.concatenate([s for *_, s, _ in parts]) if parts else np.zeros(0, _native.SEND_DTYPE)
        ent_all = np.concatenate([e for _, _, e, _, _ in parts]) if parts else np.zeros(0, _native.ENTRY_DTYPE)
        if parts:                 # entries index the whole row table, rows the whole payload: add each chunk's offsets
            snd_all["payload_off"] += np.repeat(off[:-1, 3], [len(s) for *_, s, _ in parts])
            ent_all["send"] += np.repeat(off[:-1, 2], [len(e) for _, _, e, _, _ in parts]).astype(np.uint32)
        members = [[self._agent_idx[a] for a in (self._group_snapshot[k] or [])] for k in range(len(self._group_name))]
        moff = np.zeros(len(members) + 1, np.uint64)
        moff[1:] = np.cumsum([len(m) for m in members]) if members else []
        extra = self._in_flight_arrays() if in_flight else {}
        path = Path(path)
        with open(path, "wb") as f:
            np.savez(f, version=np.uint32(self.SNAPSHOT_VERSION_IN_FLIGHT if in_flight else self.SNAPSHOT_VERSION), **extra,
                     shard=np.array([g.shard_id, max(1, g.num_shards)], np.uint32),
                     id_nonce=np.uint64(self._id_hi >> 64), next_seq=np.uint64(self._next_seq),
                     agent_names=np.array(self._agent_name, dtype=np.str_),
                     registered=np.array([a in self.registered_agents for a in self._agent_name], bool),
                     group_names=np.array(self._group_name, dtype=np.str_), group_off=moff,
                     group_members=np.array([x for m in members for x in m], np.uint32),
                     chunk_off=off,
                     agents=np.concatenate([p[0] for p in parts]).astype(np.uint32) if parts else np.zeros(0, np.uint32),
                     counts=np.concatenate([p[1] for p in parts]) if parts else np.zeros(0, np.uint32),
                     entries=ent_all,
                     sends=snd_all,
                     payload=np.concatenate([p[4] for p in parts]) if parts else np.zeros(0, np.uint8))
        return path

    def _in_flight_arrays(self) -> Dict[str, np.ndarray]:
        """The lease section (export chunks concatenated, rows and payload rebased per chunk as the pending chunks are)
        and the ledger section of a format-2 snapshot."""
        parts: List[Tuple[np.ndarray, ...]] = []
        start = 0
        while True:
            ent, snd, pay, meta, start = self.shard.lease_export(start)
            if len(ent) == 0:
                break
            parts.append((ent.copy(), snd.copy(), pay.copy(), meta.copy()))
        off = np.zeros((len(parts) + 1, 3), np.uint64)          # chunk k: entries, rows, payload bytes
        for k, (e, s, p, _) in enumerate(parts):
            off[k + 1] = off[k] + [len(e), len(s), len(p)]
        ent_all = np.concatenate([p[0] for p in parts]) if parts else np.zeros(0, _native.ENTRY_DTYPE)
        snd_all = np.concatenate([p[1] for p in parts]) if parts else np.zeros(0, _native.SEND_DTYPE)
        if parts:
            ent_all["send"] += np.repeat(off[:-1, 1], [len(p[0]) for p in parts]).astype(np.uint32)
            snd_all["payload_off"] += np.repeat(off[:-1, 2], [len(p[1]) for p in parts])
        M = self.gpu_config.lease_max_deliveries
        if M:
            la, ls, lc = self.shard.ledger_export()
        else:
            la, ls, lc = np.zeros(0, np.uint32), np.zeros(0, np.uint64), np.zeros(0, np.uint32)
        return dict(lease_entries=ent_all, lease_sends=snd_all,
                    lease_payload=np.concatenate([p[2] for p in parts]) if parts else np.zeros(0, np.uint8),
                    lease_meta=np.concatenate([p[3] for p in parts]) if parts else np.zeros(0, _native.META_DTYPE),
                    lease_chunk_off=off, ledger_agent=la, ledger_seq=ls, ledger_count=lc,
                    ledger_max_deliveries=np.uint32(M))

    @staticmethod
    def _read_snapshot(path: Union[str, Path]) -> Dict[str, np.ndarray]:
        with np.load(Path(path), allow_pickle=False) as z:
            snap = {k: z[k] for k in z.files}
        known = (SwarmsDB.SNAPSHOT_VERSION, SwarmsDB.SNAPSHOT_VERSION_IN_FLIGHT)
        if int(snap["version"]) not in known:
            raise ValueError(f"{path}: queue snapshot format {int(snap['version'])}, expected one of {known}")
        return snap

    def _lease_parts(self, snap: Dict[str, np.ndarray]) -> List[Tuple[np.ndarray, ...]]:
        """The lease section as import calls: each chunk split where this instance's receive capacity is smaller, each
        part with only the rows it names and their payloads packed (entries, sends, payload, meta)."""
        cap = recv_capacity(self.gpu_config)
        off = snap["lease_chunk_off"].astype(np.int64)
        ent, snd, pay, meta = snap["lease_entries"], snap["lease_sends"], snap["lease_payload"], snap["lease_meta"]
        out = []
        for k in range(len(off) - 1):
            for i in range(int(off[k, 0]), int(off[k + 1, 0]), cap):
                j = min(i + cap, int(off[k + 1, 0]))
                out.append(_compact_rows(ent[i:j], snd, pay) + (meta[i:j],))
        return out

    def _check_in_flight_fits(self, snap: Dict[str, np.ndarray], parts) -> None:
        """Refuse a format-2 snapshot this fresh instance cannot hold, before anything of it is adopted."""
        g = self.gpu_config
        if not g.lease_records:
            raise RuntimeError("snapshot holds in-flight leases: loading it needs a lease store (GpuConfig.lease_records)")
        meta = snap["lease_meta"]
        dead = int(np.count_nonzero(meta["state"] == _native.LEASE_STATE_DEAD))
        counted = len(snap["ledger_agent"]) or int(np.count_nonzero(meta["deliveries"] > 1))
        if (dead or counted) and not g.lease_max_deliveries:
            raise RuntimeError(f"snapshot holds {dead} dead letters and delivery counts: loading it needs "
                               f"GpuConfig.lease_max_deliveries")
        ls = self.shard.lease_stats()
        entries, rows = sum(len(p[0]) for p in parts), sum(len(p[1]) for p in parts)
        pbytes = sum(pad32(len(p[2])) for p in parts)
        if max(entries, rows) > ls["entries_reserved"] - ls["entries_used"] or pbytes > ls["payload_reserved"] - ls["payload_used"]:
            raise RuntimeError(f"snapshot holds {entries} leases ({pbytes} payload bytes), more than the lease store's free "
                               f"room (GpuConfig.lease_records={g.lease_records})")
        if g.lease_max_deliveries:
            room = self.shard.lease_policy_stats()["ledger_cap"]
            if len(snap["ledger_agent"]) > room:
                raise RuntimeError(f"snapshot holds {len(snap['ledger_agent'])} delivery counts, more than the ledger holds "
                                   f"({room})")

    def _load_in_flight(self, snap: Dict[str, np.ndarray], parts) -> None:
        """The ledger (it looks records up in the rings, so after the restore), then the leases; rebuilds the host's
        lease map and deadline heap so acks, nacks, renewals, sweeps and dead letters work on leases from before."""
        if len(snap["ledger_agent"]):
            self.shard.ledger_import(snap["ledger_agent"], snap["ledger_seq"], snap["ledger_count"])
        deadlines = set()
        for ent, snd, pay, meta in parts:
            base = self.shard.lease_import(ent, snd, pay, meta)
            for k, (seq, a, st, d) in enumerate(zip(ent["seq"].tolist(), meta["agent"].tolist(), meta["state"].tolist(),
                                                    meta["deadline"].tolist())):
                self._leases.setdefault(self._make_id(seq), []).append((a, base + k))
                if st == _native.LEASE_STATE_LIVE:
                    deadlines.add(d)
        for d in deadlines:
            heapq.heappush(self._lease_deadlines, d)

    def _check_fresh(self) -> None:
        st = self.shard.stats()
        if self._agent_name or self._group_name or len(self._b_sender) or st["enqueued"] or st["next_seq"] != 1:
            raise RuntimeError("load_queue_snapshot needs a fresh instance (no agent, group or send yet)")

    def _adopt_tables(self, snap: Dict[str, np.ndarray]) -> None:
        """Agents and groups in the snapshot's index order (indices keep their meaning: payloads of long visible_to
        lists hold dense agent indices), the id nonce and the sequence counter."""
        nonce = int(snap["id_nonce"])
        g = self.gpu_config
        if not g.deterministic_ids:
            if g.id_nonce is not None and (g.id_nonce & ((1 << 63) - 1)) != nonce:
                raise ValueError(f"GpuConfig.id_nonce={g.id_nonce:#x} differs from the snapshot's id nonce {nonce:#x}")
            self._id_hi = nonce << 64
        names = [str(x) for x in snap["agent_names"]]
        for a in names:
            self._index(a)
        reg = [a for a, r in zip(names, snap["registered"].tolist()) if r]
        if reg:
            self.register_agents(reg)
        moff, mem = snap["group_off"].astype(np.int64), snap["group_members"]
        for k, gname in enumerate(str(x) for x in snap["group_names"]):
            self.add_agent_group(gname, [names[int(i)] for i in mem[moff[k]:moff[k + 1]]])
        nxt = int(snap["next_seq"])
        self.shard.advance_seq(nxt)
        self._next_seq = max(self._next_seq, nxt); self._b_first_seq = self._next_seq

    def _check_snapshot_fits(self, snap: Dict[str, np.ndarray]) -> None:
        """Refuse a snapshot this instance cannot hold before anything of it is adopted: the instance is fresh, so every
        ring is empty and an agent's records fit exactly when they number at most ring_slots (and one restore call).
        A refusal found chunk by chunk would leave the earlier chunks restored and the instance no longer fresh."""
        agents, counts = snap["agents"].astype(np.int64), snap["counts"].astype(np.int64)
        if not len(agents):
            return
        per_agent = np.bincount(agents, weights=counts).astype(np.int64)
        worst = int(np.argmax(per_agent))
        cap = recv_capacity(self.gpu_config)
        if counts.max() > cap:
            raise RuntimeError(f"snapshot agent with {int(counts.max())} records does not fit one restore call ({cap})")
        if per_agent[worst] > self.gpu_config.ring_slots:
            raise SdbError(-4, f"snapshot agent {snap['agent_names'][worst]} has {int(per_agent[worst])} records, more than "
                               f"its ring holds "
                               f"(GpuConfig.ring_slots={self.gpu_config.ring_slots}): nothing restored")

    def _restore_chunks(self, snap: Dict[str, np.ndarray]) -> int:
        """Restore every chunk of a snapshot, split by whole agents where this instance's receive capacity is smaller;
        returns the largest sequence number + 1 seen."""
        cap = recv_capacity(self.gpu_config)
        off = snap["chunk_off"].astype(np.int64)
        agents, counts, ent, snd, pay = snap["agents"], snap["counts"], snap["entries"], snap["sends"], snap["payload"]
        seq_end = self._next_seq
        for k in range(len(off) - 1):
            a0, a1, e0 = off[k, 0], off[k + 1, 0], off[k, 1]
            ca = counts[a0:a1].astype(np.int64)
            first = e0 + np.concatenate([[0], np.cumsum(ca)])
            i = 0
            while i < len(ca):
                j = i
                while j < len(ca) and first[j + 1] - first[i] <= cap:
                    j += 1
                part_ent, part_snd, part_pay = _compact_rows(ent[first[i]:first[j]], snd, pay)
                _, se = self.shard.restore_compact(agents[a0 + i:a0 + j], ca[i:j], part_ent, part_snd, part_pay)
                seq_end = max(seq_end, se)
                i = j
        return seq_end

    def load_queue_snapshot(self, path: Union[str, Path]) -> None:
        """Put a snapshot written by save_queue_snapshot back into this instance, which must be fresh: the agents and
        groups are re-created in the snapshot's index order, its id nonce is adopted (GpuConfig.id_nonce, when set, must
        equal it) and every pending record is restored with its id, to be delivered as if it had never left.  A snapshot
        this instance cannot hold is refused before anything of it is adopted, and the instance stays fresh: an agent
        with more records than one receive call holds raises RuntimeError (checked first), one with more records than
        its ring holds raises SdbError (code -4).  A format-2 snapshot (save_queue_snapshot(in_flight=True)) also puts the
        delivery counts, the leases and the dead letters back, in that order after the pending records; it is refused
        (RuntimeError) by an instance without a lease store, with too little free store or ledger room, or without
        GpuConfig.lease_max_deliveries when it holds dead letters or counts.  Leases keep their deadlines, so one that
        passed during the restart is due at the next sweep; the messages keep their ids."""
        self._check_fresh()
        snap = self._read_snapshot(path)
        self._check_snapshot_fits(snap)
        in_flight = int(snap["version"]) == self.SNAPSHOT_VERSION_IN_FLIGHT
        parts = self._lease_parts(snap) if in_flight else []
        if in_flight:
            self._check_in_flight_fits(snap, parts)
        self._adopt_tables(snap)
        seq_end = self._restore_chunks(snap)
        self._next_seq = max(self._next_seq, seq_end); self._b_first_seq = self._next_seq
        if in_flight:
            self._load_in_flight(snap, parts)
        self._supersede_after_restore(bool(np.any(snap["sends"]["type"] & TYPEF_SUPERSEDE)))

    # ------------------------------------------------------------------ LLM backends (M:1281-1325 + real balancer)
    def set_llm_load_balancing(self, enabled: bool = True) -> None:
        self.llm_load_balancing = enabled

    def assign_llm_backend(self, agent_id: str, backend_id: str) -> None:
        self.metadata.setdefault("llm_backends", {})[agent_id] = backend_id
        b = self._backend_idx.get(backend_id)
        if b is not None and agent_id in self._agent_idx:      # device copy of the sticky map: backs queue-fed loads
            self.shard.assign_agent_backends([self._agent_idx[agent_id]], [b])

    def get_llm_backend(self, agent_id: str) -> Optional[str]:
        return self.metadata.get("llm_backends", {}).get(agent_id)

    def register_llm_backends(self, backend_ids: List[str], weights: Optional[List[int]] = None,
                              loads: Optional[List[int]] = None) -> None:
        """Declare the backend pool the balancer picks from (weight = relative capacity)."""
        self._backend_name = list(backend_ids)
        self._backend_idx = {b: i for i, b in enumerate(self._backend_name)}
        self.shard.set_backends(np.asarray(weights if weights is not None else [1] * len(backend_ids), np.uint32),
                                None if loads is None else np.asarray(loads, np.uint64))

    def select_llm_backends(self, n_requests: int, cost=None, mode: str = "least_load", seed: int = 0) -> np.ndarray:
        """Batched pick: backend index per request (see include/swarmdb_b200.h for the definition)."""
        return self.shard.select_backends(n_requests, cost, 0 if mode == "least_load" else 1, seed)

    def select_llm_backend(self, agent_id: Optional[str] = None, cost: int = 1) -> Optional[str]:
        """Sticky assignment if the agent has one (M:1303-1307), else a balanced pick when
        load balancing is enabled; the pick is remembered as the agent's assignment."""
        if agent_id is not None:
            b = self.get_llm_backend(agent_id)
            if b is not None:
                return b
        if not self.llm_load_balancing or not self._backend_name:
            return None
        b = self._backend_name[int(self.shard.select_backends(1, np.array([cost], np.uint32), 0, 0)[0])]
        if agent_id is not None:
            self.assign_llm_backend(agent_id, b)
        return b

    def release_llm_backend(self, backend_id: str, cost: int = 1) -> None:
        self.shard.release_backends([self._backend_idx[backend_id]], [cost])

    def refresh_llm_backend_loads(self) -> Dict[str, int]:
        """Set every backend's load to the backlog of the agents assigned to it - the reference's only load signal is
        get_agent_load (M:1049-1094); here it is one pass over the ring headers on the device."""
        self._pre_read()
        self.shard.backend_loads_from_queues()
        return self.llm_backend_loads()

    def llm_backend_loads(self) -> Dict[str, int]:
        return {b: int(l) for b, l in zip(self._backend_name, self.shard.backend_loads())}

    # ------------------------------------------------------------------ host-side bookkeeping (M:603-808, 973-1206)
    def get_message(self, message_id: str, include_device: bool = False) -> Optional[Message]:
        """The host record of `message_id` (M:603-613).  include_device=True also looks the id up on the device queue
        when there is no host record (bulk sends, other ranks' traffic, messages sent before a load_message_history,
        restored or redelivered records): one counting pass over every agent's queue finds the first agent holding
        it, then one PEEK of that agent returns it, status DELIVERED.  Only pending messages are found (not leased or
        dead-lettered ones), and only ids this instance issued."""
        m = self.messages.get(message_id)
        if m is None and message_id in self._dup_of:           # a duplicate send: the message it matched
            m = self.messages.get(self._dup_of[message_id])
        if m is not None or not include_device:
            return m
        return self.get_messages([message_id], include_device=True)[0]

    def get_messages(self, message_ids: Iterable[str], include_device: bool = False) -> List[Optional[Message]]:
        """get_message for many ids, in input order (None: not found).  With include_device=True the ids without a host
        record are looked up on the device in one counting pass over every agent's queue, then one PEEK per part of
        the agents that hold them; a host record wins over its device copy."""
        ids = list(message_ids)
        out: List[Optional[Message]] = [self.messages.get(mid) for mid in ids]
        if not include_device:
            return out
        want = {}
        for k, mid in enumerate(ids):
            seq = self._seq_of_id(mid) if out[k] is None else None
            if seq is not None:
                want.setdefault(seq, []).append(k)
        if not want:
            return out
        if len(want) > FILTER_MAX_IDS:
            raise ValueError(f"more than {FILTER_MAX_IDS} distinct message ids")
        self._pre_read()
        filt = make_filter(ids=np.fromiter(want, np.uint64, count=len(want)))
        where = np.empty(len(want), np.uint32)
        agents, flags = self._expire_scope(None)
        self.shard.receive_where(agents, 1, flags | RECV_PEEK, filt, drop=True, id_agent=where)
        holders = np.unique(where[where != _native.NO_RECEIVER])
        found: Dict[int, Message] = {}
        for part, cap in self._pending_chunks(holders.astype(np.uint32), 1 << 31):
            _, hdr, pay = self.shard.receive_where(part, cap, RECV_PEEK, filt)
            for m, seq in zip(self._decode(hdr, pay, "", record=False, status=MessageStatus.DELIVERED), hdr["seq"].tolist()):
                found.setdefault(seq, m)
        for seq, ks in want.items():
            for k in ks:
                out[k] = found.get(seq)
        return out

    def get_agent_messages(self, agent_id: str, status: Optional[MessageStatus] = None, limit: int = 100,
                           skip: int = 0) -> List[Message]:
        picked: List[Message] = []
        for pos, mid in enumerate(reversed(self.agent_inbox.get(agent_id, []))):
            if pos < skip:
                continue
            if len(picked) >= limit:
                break
            m = self.messages.get(mid)
            if m is not None and (status is None or m.status == status):
                picked.append(m)
        return picked

    def mark_message_as_processed(self, message_id: str) -> bool:
        leased = [lid for _, lid in self._leases.pop(message_id, [])]
        if leased:                                     # a leased message is done: every live lease on it is acked
            self.shard.lease_settle(leased, _native.LEASE_ACK)
        m = self.messages.get(message_id)
        if m is None:
            return False
        m.status = MessageStatus.PROCESSED
        return True

    def query_messages(self, sender_id: Optional[str] = None, receiver_id: Optional[str] = None,
                       message_type: Optional[MessageType] = None, status: Optional[MessageStatus] = None,
                       after_timestamp: Optional[float] = None, before_timestamp: Optional[float] = None,
                       limit: int = 100, include_device: bool = False) -> List[Message]:
        """Host records that match, newest first (M:671-700).  include_device=True adds the matching messages still
        queued on the device that have no host record (bulk sends, other ranks' traffic, messages sent before a
        load_message_history), newest first, after the host hits; they read as DELIVERED, so a `status` other than
        DELIVERED adds none.  receiver_id reads that agent's queue and, as the host rule does, leaves broadcasts out."""
        def keep(m: Message) -> bool:
            return ((sender_id is None or m.sender_id == sender_id)
                    and (receiver_id is None or m.receiver_id == receiver_id)
                    and (message_type is None or m.type == message_type)
                    and (status is None or m.status == status)
                    and (after_timestamp is None or m.timestamp > after_timestamp)
                    and (before_timestamp is None or m.timestamp < before_timestamp))
        hits: List[Message] = []
        for m in reversed(list(self.messages.values())):
            if len(hits) >= limit:
                break
            if keep(m):
                hits.append(m)
        if include_device and len(hits) < limit and status in (None, MessageStatus.DELIVERED):
            agents = None
            if receiver_id is not None:
                owned = self._expire_scope([receiver_id])[0] if receiver_id in self._agent_idx else []
                if len(owned) == 0:
                    return hits
                agents = owned
            filt = self._where_filter(sender_id, None if agents is None else int(agents[0]), message_type, None, None,
                                      after_timestamp, before_timestamp)
            hits += self._device_matches(filt, limit - len(hits), keep, agents)
        return hits

    def search_messages(self, keyword: str, case_sensitive: bool = False, limit: int = 100,
                        include_device: bool = False) -> List[Message]:
        """Host records whose content contains `keyword`, newest first (M:702-740).  include_device=True adds the
        matching device-queued messages without a host record, newest first, after the host hits.  On the device the
        content bytes are searched for the keyword's first 256 UTF-8 bytes with ASCII-only case folding, then every
        candidate is checked with the host rule; a message that matches only under Unicode case folding beyond ASCII
        (e.g. the Kelvin sign against "k") is not found on the device."""
        needle = keyword if case_sensitive else keyword.lower()

        def keep(m: Message) -> bool:
            text = json.dumps(m.content) if isinstance(m.content, (dict, list)) else str(m.content)
            return needle in (text if case_sensitive else text.lower())
        hits: List[Message] = []
        for m in reversed(list(self.messages.values())):
            if len(hits) >= limit:
                break
            if keep(m):
                hits.append(m)
        if include_device and len(hits) < limit:
            kw = keyword.encode("utf-8")[:FILTER_MAX_KEYWORD]
            filt = make_filter(keyword=kw, icase=not case_sensitive)
            hits += self._device_matches(filt, limit - len(hits), keep)
        return hits

    def get_conversation(self, agent_id_1: str, agent_id_2: str, limit: int = 100,
                         include_device: bool = False) -> List[Message]:
        half = limit // 2
        return (self.query_messages(sender_id=agent_id_1, receiver_id=agent_id_2, limit=half, include_device=include_device)
                + self.query_messages(sender_id=agent_id_2, receiver_id=agent_id_1, limit=half, include_device=include_device))

    def get_unread_message_count(self, agent_id: str) -> int:
        return sum(1 for mid in self.agent_inbox.get(agent_id, [])
                   if mid in self.messages and self.messages[mid].status == MessageStatus.DELIVERED)

    def get_agent_load(self, agent_id: str) -> Dict[str, Any]:
        if agent_id not in self.registered_agents:
            return {"registered": False, "message_count": 0, "inbox_size": 0, "unread_count": 0, "processing_rate": 0}
        horizon = time.time() - 60
        involved = recent = 0
        for m in self.messages.values():
            if m.receiver_id == agent_id or m.sender_id == agent_id:
                involved += 1
            if m.receiver_id == agent_id and m.timestamp > horizon:
                recent += 1
        return {"registered": True, "message_count": involved, "inbox_size": len(self.agent_inbox.get(agent_id, [])),
                "unread_count": self.get_unread_message_count(agent_id), "processing_rate": recent / 60}

    def get_agent_queue_load(self, agent_id: str) -> Dict[str, Any]:
        """get_agent_load's inbox_size / unread_count (M:1076-1080) answered by the device queue itself: works for
        traffic that never had a host-side record (bulk index-level sends, messages ingested by other ranks)."""
        if agent_id not in self._agent_idx:
            return {"registered": False, "inbox_size": 0, "unread_count": 0, "unread_by_priority": [0, 0, 0, 0], "unread_bytes": 0}
        self._pre_read()
        ld = self.shard.agent_loads([self._agent_idx[agent_id]])[0]
        return {"registered": agent_id in self.registered_agents, "inbox_size": int(ld["received"]),
                "unread_count": int(ld["pending"]), "unread_by_priority": [int(x) for x in ld["pending_by_prio"]],
                "unread_bytes": int(ld["pending_granules"]) * 32}

    def get_stats(self) -> Dict[str, Any]:
        by_type = {t.value: 0 for t in MessageType}
        by_status = {s.value: 0 for s in MessageStatus}
        sent: Dict[str, int] = {}
        recv: Dict[str, int] = {}
        for m in self.messages.values():
            by_type[m.type.value] += 1
            by_status[m.status.value] += 1
            sent[m.sender_id] = sent.get(m.sender_id, 0) + 1
            if m.receiver_id is not None:
                recv[m.receiver_id] = recv.get(m.receiver_id, 0) + 1
        by_agent = {a: {"sent": sent.get(a, 0), "received": recv.get(a, 0), "total": sent.get(a, 0) + recv.get(a, 0)}
                    for a in self.registered_agents}
        out = {"total_messages": self.message_count, "active_agents": len(self.registered_agents),
               "messages_by_type": by_type, "messages_by_status": by_status, "messages_by_agent": by_agent,
               "last_save_time": self.last_save_time, "device": self.shard.stats(),
               "queue": self.shard.queue_stats()}             # pending totals / priority histogram / deepest inbox, computed on the device
        if self.gpu_config.lease_records:
            out["leases"] = self.shard.lease_stats()
        if self.gpu_config.lease_max_deliveries:
            out["dead_letters"] = self.shard.lease_policy_stats()["dead"]
        if self.gpu_config.dedup_entries:
            out["dedup"] = self.shard.dedup_stats()
        if self.gpu_config.queue_max_messages or self.gpu_config.queue_max_bytes:
            out["trimmed"] = self._trimmed                 # messages the queue caps dropped, never delivered
        out["superseded"] = self._superseded               # records newer superseding sends replaced, never delivered
        return out

    def resend_failed_messages(self) -> List[str]:
        resent: List[str] = []
        for m in [x for x in self.messages.values() if x.status == MessageStatus.FAILED]:
            new_id = self.send_message(sender_id=m.sender_id, content=m.content, receiver_id=m.receiver_id,
                                       message_type=m.type, priority=m.priority, metadata=m.metadata,
                                       visible_to=m.visible_to, dedup_id=self._dedup_ids.get(m.id))
            self.messages[new_id].metadata["resent_from"] = m.id
            resent.append(new_id)
        return resent

    def delete_message(self, message_id: str, include_device: bool = False) -> bool:
        """Delete the host record (M:1132-1157).  include_device=True also drops every device-queued copy of the
        message (all copies of a broadcast), so it is never delivered; only ids this instance issued are looked up
        there.  True when anything was deleted."""
        return self.delete_messages([message_id], include_device)[0]

    def delete_messages(self, message_ids: Iterable[str], include_device: bool = False) -> List[bool]:
        """delete_message for many ids, in input order: True where anything of that id was deleted.  With
        include_device=True one device call drops every pending copy of every listed id (only ids this instance
        issued are looked up there).  A leased (in flight) or dead-lettered copy is not pending and stays: a deleted
        id that is leased elsewhere comes back only through its lease."""
        ids = list(message_ids)
        host = {}
        for mid in dict.fromkeys(ids):
            host[mid] = self.messages.pop(mid, None) is not None
            if host[mid]:
                for inbox in self.agent_inbox.values():
                    if mid in inbox:
                        inbox.remove(mid)
        out = [host[mid] for mid in ids]
        if not include_device:
            return out
        seq_of = {mid: self._seq_of_id(mid) for mid in host}
        seqs = list(dict.fromkeys(s for s in seq_of.values() if s is not None))
        if not seqs:
            return out
        if len(seqs) > FILTER_MAX_IDS:
            raise ValueError(f"more than {FILTER_MAX_IDS} distinct message ids")
        self._pre_read()
        agents, flags = self._expire_scope(None)
        # at most one copy per id and agent, as a send leaves it.  One id is the range [seq, seq + 1): the call's total
        # answers it, with no id table to build; several ids take the id clause and its per-id hit counts.
        if len(seqs) == 1:
            _, n = self.shard.receive_where(agents, 1, flags, make_filter(seq=(seqs[0], seqs[0] + 1)), drop=True)
            dropped = set(seqs) if n else set()
        else:
            hits = np.empty(len(seqs), np.uint32)
            self.shard.receive_where(agents, len(seqs), flags, make_filter(ids=np.array(seqs, np.uint64)), drop=True,
                                     id_hits=hits)
            dropped = {s for s, h in zip(seqs, hits.tolist()) if h}
        return [o or seq_of[mid] in dropped for o, mid in zip(out, ids)]

    def _seq_of_id(self, message_id: str) -> Optional[int]:
        """The sequence number behind an id this instance issued (_make_id), else None."""
        try:
            v = int(message_id.replace("-", ""), 16)
        except ValueError:
            return None
        seq = v & ((1 << 64) - 1)
        return seq if (v ^ seq) == self._id_hi and 0 < seq and self._make_id(seq) == message_id else None

    def flush_old_messages(self, older_than: Optional[float] = None, include_device: bool = False) -> int:
        """Archive every message older than the cutoff to archives/archive_{ts}.json and delete it (M:1159-1206).
        include_device=True also expires the messages still queued on the device (device-only traffic included) and
        archives them with the rest: a host record wins over its device copy, a broadcast is one entry.  Returns the
        number of distinct messages archived."""
        cutoff = older_than if older_than is not None else time.time() - 7 * 24 * 3600
        old = [mid for mid, m in self.messages.items() if m.timestamp < cutoff]
        archived = {mid: self.messages[mid].to_dict() for mid in old}
        if include_device:
            for m in self._expire_device_archive(cutoff):
                if m.id not in archived:
                    host = self.messages.get(m.id)
                    archived[m.id] = (host if host is not None else m).to_dict()
        if archived:
            path = self.save_dir / "archives" / f"archive_{int(time.time())}.json"
            path.parent.mkdir(parents=True, exist_ok=True)
            path.write_text(json.dumps(archived))
            for mid in archived:
                self.delete_message(mid)
        return len(archived)

    # ------------------------------------------------------------------ retention (sdb_expire)
    def _expire_scope(self, agent_ids: Optional[Iterable[str]]):
        """(agent indices or None = every agent below the watermark, flags) an expiry acts on.  Unknown agents have
        nothing queued and are left out, as are repeats (the device refuses an agent listed twice)."""
        if agent_ids is None:
            return None, 0
        idx = dict.fromkeys(self._agent_idx[a] for a in agent_ids if a in self._agent_idx)
        return np.fromiter(idx, dtype=np.uint32, count=len(idx)), 0

    def expire_pending(self, older_than: Optional[float] = None, agent_ids: Optional[Iterable[str]] = None) -> int:
        """Drop the device-queued messages whose timestamp is older than the cutoff (default: now - retention_ms)
        without delivering them, and return how many records went.  Messages sent without a timestamp (bulk sends)
        carry 0.0 and go with any positive cutoff.  Host records are not touched (flush_old_messages archives those)."""
        self._pre_read()
        cutoff = older_than if older_than is not None else time.time() - self.config.retention_ms / 1000.0
        agents, flags = self._expire_scope(agent_ids)
        if agents is not None and len(agents) == 0:
            return 0
        return self.shard.expire(agents, cutoff, flags, archive=False)[1]

    def trim_queues(self, max_messages: Optional[int] = None, max_bytes: Optional[int] = None,
                    agent_ids: Optional[Iterable[str]] = None, by_priority: bool = False) -> int:
        """Cap the device queues: each agent (default: every agent) keeps at most max_messages pending messages and
        max_bytes pending payload bytes (sum of pad32(len)); None is no limit.  The oldest messages go first, or with
        by_priority=True the lowest priority first (oldest first within a level); they are dropped without being
        delivered.  Returns the number of records dropped.  Host records are not touched, as in expire_pending."""
        limits = _trim_limits(max_messages, max_bytes)
        self._pre_read()
        agents, flags = self._expire_scope(agent_ids)
        if agents is not None and len(agents) == 0:
            return 0
        return self.shard.trim(agents, *limits, flags | (RECV_PRIORITY if by_priority else 0), archive=False)[1]

    def pending_tokens(self, agent_ids: Optional[Iterable[str]] = None) -> Dict[str, int]:
        """Per agent (default: every agent this instance serves), the token counts of its device-pending messages,
        summed; messages sent without a count weigh 0 and in-flight leases are not pending.  Unknown agents read 0."""
        self._pre_read()
        names = list(self._agent_name) if agent_ids is None else list(dict.fromkeys(agent_ids))
        agents, _ = self._expire_scope(names)
        out = dict.fromkeys(names, 0) if agent_ids is not None else {}
        if len(agents):
            for a, t in zip(agents.tolist(), self.shard.pending_tokens(agents).tolist()):
                out[self._agent_name[a]] = int(t)
        return out

    def _expire_device_archive(self, cutoff: float) -> List[Message]:
        """Expire the device-queued records older than the cutoff in archive mode, call after call until none is left,
        and decode them (one Message per record: the copies of a broadcast share one id)."""
        self._pre_read()
        agents, flags = self._expire_scope(None)
        out: List[Message] = []
        while True:
            _, ent, snd, pay = self.shard.expire(agents, cutoff, flags, archive=True)
            if len(ent) == 0:
                return out
            hdr, p = _native.expand_compact(ent, snd, pay)
            out.extend(self._decode(hdr, p, "", record=False, status=MessageStatus.DELIVERED))

    # ------------------------------------------------------------------ history (schema of M:878-884)
    def _history(self, include_device: bool = False) -> Dict[str, Any]:
        messages = {mid: m.to_dict() for mid, m in self.messages.items()}
        inbox = self.agent_inbox
        if include_device:
            # messages that only exist on the device (bulk index-level sends have no host record): add the
            # pending ones to the same schema (M:878-884) so a history file is complete
            inbox = {a: list(v) for a, v in self.agent_inbox.items()}
            for agent, pend in self.pending_snapshot().items():
                box = inbox.setdefault(agent, [])
                have = set(box)
                for m in pend:
                    if m.id not in messages:
                        messages[m.id] = m.to_dict()
                    if m.id not in have:
                        box.append(m.id); have.add(m.id)
        return {"messages": messages, "agent_inbox": inbox, "registered_agents": list(self.registered_agents),
                "timestamp": time.time(), "message_count": max(self.message_count, len(messages))}

    def save_message_history(self, filename: Optional[str] = None, include_device: bool = False) -> None:
        if not filename:
            stamp = datetime.datetime.now().strftime("%Y%m%d_%H%M%S")
            filename = f"message_history_{stamp}_{self.message_count}.json"
        try:
            with open(self.save_dir / filename, "w") as f:
                json.dump(self._history(include_device), f, indent=2)
            self.last_save_time = time.time()
        except Exception as e:
            logger.error(f"Failed to save message history: {e}")

    def load_message_history(self, filepath: Union[str, Path]) -> None:
        path = Path(filepath)
        if not path.exists():
            logger.error(f"Message history file {path} does not exist")
            return
        try:
            history = json.loads(path.read_text())
            self.messages = {mid: Message.from_dict(d) for mid, d in history["messages"].items()}
            self.agent_inbox = history["agent_inbox"]
            for a in history["registered_agents"]:
                self.register_agent(a)
            self.message_count = history["message_count"]
        except Exception as e:
            logger.error(f"Failed to load message history: {e}")

    def export_as_yaml(self, filepath: Union[str, Path]) -> None:
        try:
            import yaml
            with open(Path(filepath), "w") as f:
                yaml.dump(self._history(), f, sort_keys=False)
        except Exception as e:
            logger.error(f"Failed to export message history as YAML: {e}")

    def auto_scale_partitions(self) -> None:
        """Kafka partition growth (M:1327-1365) has no analogue: shards are the GPUs of the box."""
        return None

    # ------------------------------------------------------------------ lifecycle (M:1367-1394)
    def close(self) -> None:
        if self._closed:
            return
        try:
            self.flush()
            if self.auto_save:
                self.save_message_history()
        finally:
            self.shard.close()
            self._closed = True

    def __enter__(self) -> "SwarmsDB":
        return self

    def __exit__(self, exc_type, exc_val, exc_tb) -> None:
        self.close()
