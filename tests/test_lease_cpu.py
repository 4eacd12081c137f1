"""The lease model (tests/lease_ref.py) on the CPU oracle, the SwarmsDB lease surface over an oracle-backed stand-in
shard, and the sharded refusals.  No GPU: tests/test_gpu_lease.py holds the device to the same model."""
import math

import numpy as np
import pytest

from tests.fake_shard import OracleShard
from tests.lease_ref import LeaseModel
from tests.ring_ref import BoundedOracle

A, G, R = 16, 2, 8
ROOT = __import__("pathlib").Path(__file__).resolve().parent.parent


def test_header_declares_lease_calls_and_profiler_slot():
    """The lease entry points and their profiler class: slot 16, past the SDB_PK_N = 16 entries sdb_profile_read fills
    (the array size of ABI-1 callers), so it is read with sdb_profile_read_n (SDB_PK_ALL = 17 classes)."""
    import ctypes as C
    import re
    h = (ROOT / "include" / "swarmdb_b200.h").read_text()
    assert re.search(r"int sdb_receive_leased\(sdb_handle h, uint32_t n_agents, const uint32_t\* agent_idx", h)
    assert "SDB_PK_N = 16" in h and "SDB_PK_LEASE = 16" in h and "SDB_PK_ALL = 17" in h
    assert re.search(r"int sdb_profile_read_n\(sdb_handle h, uint32_t n, double\* ms_out", h)
    from swarmdb_b200._native import EXPORTS, SdbLeaseSummary, Shard
    for name in ("sdb_lease_reserve", "sdb_receive_leased", "sdb_lease_settle", "sdb_lease_sweep", "sdb_lease_stats",
                 "sdb_profile_read_n"):
        assert name in EXPORTS
    assert len(Shard.PROFILE_KINDS) == 16 and Shard.PROFILE_KINDS_ALL[:16] == Shard.PROFILE_KINDS
    assert Shard.PROFILE_KINDS_ALL[16] == "lease" and len(Shard.PROFILE_KINDS_ALL) == 17
    assert C.sizeof(SdbLeaseSummary) == 64


def _oracle_with_traffic(seed=0, n=40, ring_slots=64):
    """An oracle bounded by rings of `ring_slots` (tests/ring_ref.py) and some p2p and group traffic."""
    from oracle.cpu_ref import CpuOracle
    rng = np.random.default_rng(seed)
    c = BoundedOracle(CpuOracle(A, G), G, ring_slots)
    groups = {0: np.arange(0, 4, dtype=np.uint32), 1: np.arange(4, 8, dtype=np.uint32)}
    for g, m in groups.items():
        c.create_group(g, m)
    c.register(np.arange(A, dtype=np.uint32))
    lens = rng.integers(0, 64, n).astype(np.uint16)
    off = np.arange(n, dtype=np.uint64) * 64
    buf = rng.integers(33, 127, n * 64 + 64).astype(np.uint8)
    c.send_batch(rng.integers(0, A, n), rng.integers(8, A, n), rng.integers(0, 4, n), None, lens, off, buf)
    c.send_group_batch(rng.integers(8, A, 2), [0, 1], [1, 2], None, lens[:2], off[:2], buf)
    return c, groups, rng


def _pending(c):
    return c.agent_loads(np.arange(A, dtype=np.uint32))["pending"].astype(np.int64)


def test_lease_ids_acks_renew_and_sweep_order():
    c, groups, _ = _oracle_with_traffic()
    before = _pending(c)
    m = LeaseModel(c, groups, rec_cap=1 << 10, cap=1 << 10)
    cnt, hdr, pay, base = m.lease(None, 2, 10.0)
    assert base == 0 and len(hdr) == int(cnt.sum()) > 0
    ids = np.arange(len(hdr), dtype=np.uint64)
    assert m.settle(ids[:3], 0)[1] == 3
    assert m.settle(ids[:3], 0)[1] == 0                              # already acked
    assert m.settle([10 ** 9], 0)[1] == 0                            # unknown
    out, n = m.settle([ids[3], ids[3]], 1, -math.inf)                # repeated in one call: 1 each time, settled once
    assert out.tolist() == [1, 1] and n == 2
    assert m.sweep(math.nan) == (0, 0, 0)                            # NaN: nothing due
    assert m.sweep(5.0) == (1, 0, 0)                                 # the nack only
    assert m.settle([ids[3]], 0)[1] == 0                             # late ack after redelivery
    red, blocked, left = m.sweep(10.0)
    assert red == len(hdr) - 4 and blocked == 0 and left == 0
    assert np.array_equal(_pending(c), before - _acked(cnt, 3, A))      # only the acked records are gone
    assert m.stats()["live"] == 0 and m.stats()["entries_used"] == 0 and m.stats()["acked_total"] == 3


def _acked(cnt, k, n_agents):
    """Per agent, how many of the first k leased records it owned (those are gone for good)."""
    who = np.repeat(np.arange(n_agents), cnt.astype(np.int64))[:k]
    return np.bincount(who, minlength=n_agents)


def test_redelivery_goes_behind_newer_records_in_lease_order():
    c, groups, rng = _oracle_with_traffic(1)
    m = LeaseModel(c, groups, rec_cap=1 << 10, cap=1 << 10)
    _, hdr, _, _ = m.lease([9], 100, 1.0)
    assert len(hdr) > 1
    c.send_batch([3], [9], [1], None, [5], [0], np.full(64, 65, np.uint8))
    m.sweep(1.0)
    _, again, _ = c.receive_batch([9], 100)
    assert again["seq"].tolist()[1:] == hdr["seq"].tolist()          # the newer record first, then the leased ones
    assert again["seq"][0] > hdr["seq"].max()


def test_all_flag_chunks_and_blocked_agents():
    c, groups, rng = _oracle_with_traffic(2, n=120, ring_slots=R)
    m = LeaseModel(c, groups, rec_cap=5, cap=1 << 10)
    total = 0
    while True:
        got = m.lease(None, 1 << 10, math.inf)[1]
        if len(got) == 0:
            break
        total += len(got)
    assert m.sweep(1e300) == (0, 0, 0)                               # infinite deadlines are never due ...
    # fill agent 9's ring with newer records: its leases stay in the store while every other agent is served
    n9 = sum(1 for r in m.recs if r["agent"] == 9)
    assert n9 > 0
    k = c.capacity(9)
    c.send_batch([3] * k, [9] * k, [1] * k, None, [1] * k, np.zeros(k, np.uint64), np.full(64, 65, np.uint8))
    red_total, blocked_seen, calls = 0, 0, 0
    while True:
        red, blocked, left = m.sweep(0.0, all_=True)                 # ... but ALL takes them, 5 per call
        assert red <= 5
        red_total, calls = red_total + red, calls + 1
        blocked_seen = max(blocked_seen, blocked)
        if red == 0:                                                 # done, or a chunk of agent 9's records only
            break
    assert blocked_seen >= 1 and calls > 2
    assert sum(1 for r in m.recs if r["agent"] == 9) == n9          # blocked records stay leased
    for _ in range(100):                                             # room again: the rest comes back
        if not m.stats()["live"]:
            break
        c.receive_batch(None, R)
        while m.sweep(0.0, all_=True)[0]:
            pass
    assert m.stats()["live"] == 0 and m.stats()["redelivered_total"] == total


class LeaseShard(OracleShard):
    """OracleShard plus the lease calls, answered by tests/lease_ref.py in the compact format (one row per record)."""

    def __init__(self, max_agents, max_groups, rank, world):
        super().__init__(max_agents, max_groups, rank, world)
        self.max_groups = max_groups
        self.model = None

    def lease_reserve(self, max_records, max_payload_bytes):
        if max_records and not isinstance(self.o, BoundedOracle):
            self.o = BoundedOracle(self.o, self.max_groups, 64, self.groups)
        self.model = LeaseModel(self.o, self.groups, 1 << 16, max_records) if max_records else None

    def receive_leased(self, agents, max_messages, deadline, flags=0):
        from swarmdb_b200._native import ENTRY_DTYPE, SEND_DTYPE
        cnt, hdr, pay, base = self.model.lease(agents, max_messages, deadline, flags)
        ent = np.zeros(len(hdr), ENTRY_DTYPE)
        snd = np.zeros(len(hdr), SEND_DTYPE)
        ent["seq"], ent["send"], ent["receiver"] = hdr["seq"], np.arange(len(hdr)), hdr["receiver"]
        for f in ("timestamp", "sender", "group", "len", "prio", "type"):
            snd[f] = hdr[f]
        pl = (hdr["len"].astype(np.int64) + 31) & ~31
        if len(pl) > 1:
            snd["payload_off"][1:] = np.cumsum(pl)[:-1]
        return cnt, ent, snd, pay, base

    def lease_settle(self, ids, op, deadline=0.0):
        return self.model.settle(np.atleast_1d(ids), op, deadline)

    def lease_sweep(self, now, flags=0):
        return self.model.sweep(now, bool(flags & 1))

    def lease_stats(self):
        return self.model.stats()


def _db(tmp_path, lease_records=256):
    import swarmdb_b200 as sdb
    return sdb.SwarmsDB(save_dir=str(tmp_path), auto_save=False, _shard=LeaseShard(64, 4, 0, 1),
                        gpu_config=sdb.GpuConfig(max_agents=64, max_groups=4, deterministic_ids=True,
                                                 lease_records=lease_records))


def test_surface_ack_nack_extend_and_redelivery(tmp_path):
    from swarmdb_b200.core import MessageStatus
    db = _db(tmp_path)
    for a in ("a", "b", "c"):
        db.register_agent(a)
    ids = [db.send_message("a", f"m{k}", receiver_id="b") for k in range(5)]
    got = db.receive_messages_leased("b", 10, visibility_timeout=60.0)
    assert [m.id for m in got] == ids and all(m.status == MessageStatus.READ for m in got)
    assert db.receive_messages_leased("b", 10) == []                 # leased: not visible
    assert db.ack_messages("b", ids[:2]) == 2
    assert db.ack_messages("b", ids[:1]) == 0                        # already acked
    assert db.nack_messages("b", [ids[2]]) == 1
    assert db.extend_leases("b", [ids[3]], visibility_timeout=3600.0) == 1
    again = db.receive_messages_leased("b", 10, visibility_timeout=60.0)   # the nack is swept back first
    assert [m.id for m in again] == [ids[2]]
    assert db.mark_message_as_processed(ids[2])                      # acks its lease too
    assert db.get_stats()["leases"]["live"] == 2                     # ids[3] (extended) and ids[4]
    assert db.redeliver_expired(all=True) == 2
    assert [m.id for m in db.receive_messages("b", 10)] == [ids[3], ids[4]]
    db.close()


def test_surface_broadcast_leased_by_several_agents(tmp_path):
    db = _db(tmp_path)
    for a in ("a", "b", "c"):
        db.register_agent(a)
    mid = db.broadcast_message("a", "hello")
    assert [m.id for m in db.receive_messages_leased("b")] == [mid]
    assert [m.id for m in db.receive_messages_leased("c")] == [mid]
    assert db.ack_messages("b", [mid]) == 1                          # c's lease stays
    assert db.redeliver_expired(all=True) == 1
    assert [m.id for m in db.receive_messages("c")] == [mid]
    assert db.receive_messages("b") == []
    db.close()


def test_surface_without_a_store_changes_nothing(tmp_path):
    db = _db(tmp_path, lease_records=0)
    db.register_agent("a")
    mid = db.send_message("a", "x", receiver_id="a")
    assert "leases" not in db.get_stats()
    assert [m.id for m in db.receive_messages("a")] == [mid]
    assert db.mark_message_as_processed(mid)
    db.close()


def test_sharded_front_end_refuses_leases(tmp_path):
    import swarmdb_b200 as sdb
    from swarmdb_b200 import sharded

    class Ex:
        def __init__(self, *a): pass
        def close(self): pass
    db = sharded.ShardedSwarmsDB(0, 1, exchange_factory=Ex, shard=OracleShard(64, 4, 0, 1), save_dir=str(tmp_path),
                                 auto_save=False, gpu_config=sdb.GpuConfig(max_agents=64, max_groups=4))
    for call in (lambda: db.receive_messages_leased("a"), lambda: db.receive_batch_leased(None),
                 lambda: db.ack_messages("a", []), lambda: db.nack_messages("a", []),
                 lambda: db.extend_leases("a", []), lambda: db.redeliver_expired(),
                 lambda: db.settle_leases([0]), lambda: db.requeue_batch_compact([], [], [], [], [])):
        with pytest.raises(NotImplementedError):
            call()
    with pytest.raises(NotImplementedError):
        sharded.ShardedSwarmsDB(0, 1, exchange_factory=Ex, shard=OracleShard(64, 4, 0, 1), save_dir=str(tmp_path),
                                auto_save=False, gpu_config=sdb.GpuConfig(max_agents=64, max_groups=4, lease_records=16))
