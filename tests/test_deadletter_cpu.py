"""The dead-letter model (tests/deadletter_ref.py) on the CPU oracle, the ABI of the policy calls, and the GpuConfig
checks of the Python surface.  No GPU: tests/test_gpu_dead_letter.py holds the device to the same model."""
import ctypes as C
import math

import numpy as np
import pytest

from tests.deadletter_ref import DEAD, DeadLetterModel
from tests.lease_ref import LeaseModel
from tests.test_lease_cpu import A, _oracle_with_traffic


def test_abi_declares_the_policy_calls():
    from swarmdb_b200._native import EXPORTS, SdbLeasePolicySummary
    for name in ("sdb_lease_set_policy", "sdb_lease_deliveries", "sdb_lease_dead_letters", "sdb_lease_policy_stats"):
        assert name in EXPORTS
    assert C.sizeof(SdbLeasePolicySummary) == 48
    assert [n for n, _ in SdbLeasePolicySummary._fields_] == ["max_deliveries", "dead", "dead_total", "ledger_used",
                                                              "ledger_cap", "held_by_ledger_total"]


def _step(rng, m, now):
    op = int(rng.integers(0, 5))
    if op == 0:
        m.lease(None if rng.random() < 0.3 else rng.choice(A, int(rng.integers(1, A)), replace=False), int(rng.integers(1, 4)),
                now + float(rng.integers(0, 3)))
    elif op == 1 and m.recs:
        ids = [r["id"] for r in m.recs]
        m.settle(rng.choice(ids, min(len(ids), 3)), 0)
    elif op == 2 and m.recs:
        ids = [r["id"] for r in m.recs]
        m.settle(rng.choice(ids, min(len(ids), 3)), 1, -math.inf)
    elif op == 3:
        m.sweep(now, bool(rng.random() < 0.2))
    else:
        m.o.receive_batch(rng.choice(A, 2, replace=False), 1)
    return m.stats()


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_no_policy_equals_the_lease_model_step_for_step(seed):
    c1, g1, _ = _oracle_with_traffic(seed)
    c2, g2, _ = _oracle_with_traffic(seed)
    a, b = LeaseModel(c1, g1, 16, 64), DeadLetterModel(c2, g2, 16, 64)
    r1, r2 = np.random.default_rng(seed + 10), np.random.default_rng(seed + 10)
    for t in range(40):
        assert _step(r1, a, float(t)) == _step(r2, b, float(t))
        assert [r["id"] for r in a.recs] == [r["id"] for r in b.recs]
        snap1, snap2 = c1.snapshot(), c2.snapshot()
        assert {k: [int(h["seq"]) for h, _ in v] for k, v in snap1.items()} == \
               {k: [int(h["seq"]) for h, _ in v] for k, v in snap2.items()}


def _lease_one(m, a):
    cnt, hdr, _, base = m.lease([a], 100, 0.0)
    return hdr, base


def test_counts_follow_nack_sweep_cycles_and_die_at_the_limit():
    c, groups, _ = _oracle_with_traffic(3)
    m = DeadLetterModel(c, groups, rec_cap=1 << 10, cap=1 << 10, max_deliveries=3, ledger_entries=64)
    hdr, base = _lease_one(m, 9)
    n = len(hdr)
    assert n > 1
    for k in (1, 2, 3):
        ids = np.arange(base, base + n)
        assert m.deliveries(ids).tolist() == [k] * n
        red, blocked, left = m.sweep(0.0)
        if k < 3:
            assert (red, blocked, left) == (n, 0, 0) and len(m.ledger) == n
            hdr2, base = _lease_one(m, 9)
            assert hdr2["seq"].tolist() == hdr["seq"].tolist()
        else:
            assert (red, blocked, left) == (0, 0, 0)
    assert m.policy_stats()["dead"] == n and m.deliveries(np.arange(base, base + n)).tolist() == [3] * n
    assert m.settle(np.arange(base, base + n), 0)[1] == 0                 # dead letters are not live
    cnt, ent, snd, pay, deliv = m.dead_letters([9], 1 << 10, peek=True)
    assert cnt.tolist() == [n] and deliv.tolist() == [3] * n and ent["seq"].tolist() == hdr["seq"].tolist()
    cnt, ent, snd, pay, deliv = m.dead_letters([9], 1 << 10)
    assert m.policy_stats()["dead"] == 0 and not m.recs
    m.redrive([9], cnt, ent, snd, pay)
    hdr3, base = _lease_one(m, 9)
    assert hdr3["seq"].tolist() == hdr["seq"].tolist()
    assert m.deliveries(np.arange(base, base + n)).tolist() == [1] * n   # a redrive restarts the count


def test_a_record_consumed_elsewhere_and_requeued_restarts_at_one():
    """The ledger's stale test: a plain receive takes the redelivered record, a restore puts the same seq back; the
    untouched neighbour inherits its count."""
    from oracle.cpu_ref import HDR_DTYPE  # noqa: F401
    from swarmdb_b200._native import ENTRY_DTYPE, SEND_DTYPE
    c, groups, _ = _oracle_with_traffic(4)
    m = DeadLetterModel(c, groups, rec_cap=1 << 10, cap=1 << 10, max_deliveries=10, ledger_entries=64)
    hdr, base = _lease_one(m, 10)
    assert len(hdr) >= 2
    m.sweep(0.0)
    cc, taken, tp = c.receive_batch([10], 1)                          # the first redelivered record leaves by a plain receive
    assert taken["seq"][0] == hdr["seq"][0]
    h = taken[0]
    ent = np.array([(h["seq"], 0, h["receiver"])], ENTRY_DTYPE)
    snd = np.array([(h["timestamp"], 0, h["sender"], h["group"], h["len"], h["prio"], h["type"], 0)], SEND_DTYPE)
    m.redrive([10], [1], ent, snd, tp)                                 # and comes back with the same seq
    _, base2 = _lease_one(m, 10)
    got = {int(r["hdr"]["seq"]): r["deliveries"] for r in m.recs if r["id"] >= base2}
    assert got[int(hdr["seq"][0])] == 1 and all(got[int(s)] == 2 for s in hdr["seq"][1:])


def test_a_full_ledger_holds_due_leases_in_the_store():
    c, groups, _ = _oracle_with_traffic(5)
    m = DeadLetterModel(c, groups, rec_cap=1 << 10, cap=1 << 10, max_deliveries=5, ledger_entries=2)
    hdr, base = _lease_one(m, 11)
    n = len(hdr)
    assert n > 2
    assert m.sweep(0.0) == (2, 0, n - 2)
    assert m.sweep(0.0) == (0, 0, n - 2)                              # the ledger is full until the records are taken
    assert m.policy_stats()["held_by_ledger_total"] == 2 * (n - 2)
    c.receive_batch([11], 100)                                        # taken by a plain receive: the entries go stale
    assert m.sweep(0.0) == (2, 0, n - 4)


def test_sweep_all_kills_only_leases_at_the_limit():
    c, groups, _ = _oracle_with_traffic(6)
    m = DeadLetterModel(c, groups, rec_cap=1 << 10, cap=1 << 10, max_deliveries=1, ledger_entries=8)
    _, hdr, _, _ = m.lease([12, 13], 100, 50.0)
    assert m.sweep(0.0) == (0, 0, 0) and m.policy_stats()["dead"] == 0     # not due yet
    assert m.sweep(0.0, True) == (0, 0, 0) and m.policy_stats()["dead"] == len(hdr)
    assert all(r["state"] == DEAD for r in m.recs)


@pytest.mark.parametrize("kw", [dict(lease_max_deliveries=-1, lease_records=8), dict(lease_max_deliveries=1 << 32, lease_records=8),
                                dict(lease_max_deliveries=2), dict(lease_ledger_entries=4, lease_records=8),
                                dict(lease_max_deliveries=2, lease_records=8, lease_ledger_entries=-1)])
def test_surface_refuses_bad_policy_settings_before_any_device_work(kw, tmp_path):
    import swarmdb_b200
    from swarmdb_b200.core import GpuConfig, SwarmsDB

    class Boom:
        def __getattr__(self, name):
            raise AssertionError("the shard was touched")

    with pytest.raises(ValueError):
        SwarmsDB(save_dir=tmp_path, auto_save=False, gpu_config=GpuConfig(**kw), _shard=Boom())
    assert swarmdb_b200.SwarmsDB is SwarmsDB


def test_sharded_front_end_refuses_a_redelivery_limit():
    from swarmdb_b200.core import GpuConfig
    from swarmdb_b200.sharded import ShardedSwarmsDB
    with pytest.raises(NotImplementedError):
        ShardedSwarmsDB(0, 1, gpu_config=GpuConfig(lease_max_deliveries=2, lease_records=8), shard=object())
    assert ShardedSwarmsDB.dead_letters is ShardedSwarmsDB.redrive_dead_letters


def _lg_slot_np(agent, seq, slots):
    """lg_slot in numpy's wrapping uint64 arithmetic: an independent restatement of the Python integer one."""
    u = np.uint64
    with np.errstate(over="ignore"):
        x = u(seq) ^ (u(agent) * u(0x9E3779B97F4A7C15))
        x ^= x >> u(33); x *= u(0xFF51AFD7ED558CCD); x ^= x >> u(33); x *= u(0xC4CEB9FE1A85EC53); x ^= x >> u(33)
    return (int(x) * slots) >> 64


def test_crafted_ledger_keys_collide_under_the_restated_hash():
    """The keys tests/test_gpu_lease_edges.py sends: every seq of a wrap case probes from the index's last slot, and
    the pair of the bit-32 case shares its first probe."""
    from tests.deadletter_ref import lg_slot, seqs_at_slot
    a = 8 * 64
    for N in (2, 4):
        slots = 2 * N
        seqs = seqs_at_slot(a + 7, slots, slots - 1, 1000, N + 1)
        assert seqs == sorted(set(seqs)) and len(seqs) == N + 1
        assert all(lg_slot(a + 7, q, slots) == _lg_slot_np(a + 7, q, slots) == slots - 1 for q in seqs)
    s = (1 << 33) + 1
    while lg_slot(a + 5, s, 4) != lg_slot(a + 5, s + (1 << 32), 4):
        s += 1
    assert s < (1 << 33) + 64 and _lg_slot_np(a + 5, s, 4) == _lg_slot_np(a + 5, s + (1 << 32), 4)
    # the hash spreads keys over the slots and reads the seq's high word and the agent
    rng = np.random.default_rng(1)
    for _ in range(200):
        ag, q, n = int(rng.integers(0, 1 << 32)), int(rng.integers(0, 1 << 63)), int(rng.integers(1, 1 << 31))
        assert lg_slot(ag, q, n) == _lg_slot_np(ag, q, n) < n
    hits = np.bincount([lg_slot(3, q, 16) for q in range(4096)], minlength=16)
    assert hits.min() > 160
    assert len({lg_slot(5, q << 32, 1 << 20) for q in range(64)}) > 60
    assert len({lg_slot(ag, 77, 1 << 20) for ag in range(64)}) > 60
