"""Snapshots of the lease store and the redelivery ledger on the device (sdb_lease_export / sdb_lease_import /
sdb_lease_ledger_export / sdb_lease_ledger_import) against tests/lease_snapshot_ref.py, in both arena layouts.

An export must equal the model byte for byte and change nothing.  A fresh handle given the pending records, the ledger and
the lease chunks must then behave like the original: the same operations on both, with lease ids mapped by position, give
the same results, delivery counts included, and the same drains on every receive path.
"""
import math
from types import SimpleNamespace

import numpy as np
import pytest

from tests.lease_snapshot_ref import SnapshotModel
from tests.ring_ref import BoundedOracle
from tests.test_gpu_compact_receive import Rig
from tests.test_gpu_dead_letter import _dead, _lease, _nack_all, _sweep
from tests.test_gpu_restore import _every_path, _fresh, _groups, _loads_equal, _renumber

pytestmark = pytest.mark.gpu

BIG = 1 << 20


@pytest.fixture(params=["1", "0"])
def shared(request, monkeypatch):
    monkeypatch.setenv("SDB_SHARED_PAYLOAD", request.param)
    return request.param == "1"


def _attach(g, c, rig, shared, M, ledger, cap=BIG):
    """A lease store and policy on g, and the snapshot model over the oracle c (wrapped in the ring model)."""
    from swarmdb_b200._native import recv_capacity
    g.lease_reserve(cap, cap * 256)
    g.lease_set_policy(M, ledger)
    bc = c if isinstance(c, BoundedOracle) else BoundedOracle(c, rig.G, int(g.cfg.ring_slots), _groups(rig), rig.A)
    return bc, SnapshotModel(bc, _groups(rig), recv_capacity(g.cfg), cap, shared, M, ledger)


def _history(rig, m):
    """Leases, acks, renewals, nacks, sweeps and kills: the store ends with live leases of several counts and three
    deadlines, dead letters at the limit, and the ledger with counts of redelivered records still pending."""
    from swarmdb_b200._native import LEASE_ACK, LEASE_RENEW
    from tests.test_gpu_shared_layout import _payloads
    poison = rig.idx[-6:]                                              # non-members: p2p records only, all leased each round
    lens, off, buf = _payloads(rig.rng, 24, 100)
    r, snd = np.repeat(poison, 4), rig.rng.integers(0, rig.A, 24)
    assert rig.c.send_batch(snd, r, None, None, lens, off, buf) == rig.g.send_batch(snd, r, None, None, lens, off, buf)
    for k in range(m.M):
        ids = _lease(rig, m, None, 2, 10.0)
        third = ids[: len(ids) // 3]
        assert np.array_equal(rig.g.lease_settle(third, LEASE_ACK)[0], m.settle(third, LEASE_ACK)[0])
        later = ids[len(ids) // 3: len(ids) // 2]
        assert np.array_equal(rig.g.lease_settle(later, LEASE_RENEW, 20.0)[0], m.settle(later, LEASE_RENEW, 20.0)[0])
        _nack_all(rig, m, ids[len(ids) // 2:])
        _sweep(rig, m, 0.0)
    for k in range(m.M):                                               # the poison agents' records die at the limit
        ids = _lease(rig, m, poison, 1000, 10.0)
        _nack_all(rig, m, ids)
        _sweep(rig, m, 0.0)
    _lease(rig, m, rig.idx[::3], 1, 10.0)                              # counts of redelivered records continue
    assert m.policy_stats()["dead"] > 0 and m.live > 0 and m.ledger


def _state(g, idx):
    st = g.stats()
    st.pop("kernel_launches")
    return st, g.lease_stats(), g.lease_policy_stats(), g.agent_loads(idx).tobytes()


def _export_all(g, start=0, cap=None):
    from swarmdb_b200._native import ENTRY_DTYPE, META_DTYPE, SEND_DTYPE
    kw = {}
    if cap:
        kw = dict(out_entries=np.zeros(cap, ENTRY_DTYPE), out_sends=np.zeros(cap, SEND_DTYPE),
                  out_meta=np.zeros(cap, META_DTYPE))
    chunks = []
    while True:
        ent, snd, pay, meta, start = g.lease_export(start, **kw)
        if len(ent) == 0:
            return chunks
        chunks.append((ent.copy(), snd.copy(), pay.copy(), meta.copy()))


@pytest.mark.parametrize("M", [2, 3])
def test_chunked_export_equals_the_model_and_changes_nothing(shared, M):
    from swarmdb_b200._native import recv_capacity
    rig = Rig(np.random.default_rng(10 + M), G=8, F=64, extra=64)
    rig.check_advance = False
    rig.mixed(2)
    rig.c, m = _attach(rig.g, rig.c, rig, shared, M, 1 << 16)
    _history(rig, m)
    before = _state(rig.g, rig.idx)
    ids = [r["id"] for r in m.recs]
    for start, cap in ((0, None), (ids[len(ids) // 2], 7), (ids[len(ids) // 2] + 1, 64), (ids[-1] + 1, 7)):
        got = _export_all(rig.g, start, cap)
        want, s = [], start
        while True:
            w = m.export(s, min(cap or BIG, recv_capacity(rig.g.cfg)))
            if len(w[0]) == 0:
                break
            want.append(w[:4])
            s = w[4]
        assert len(got) == len(want) and (cap is None or len(got) > 1 or start > ids[-1])
        for x, y in zip(got, want):
            for a, b, name in zip(x, y, ("entries", "sends", "payload", "meta")):
                assert a.tobytes() == b.tobytes(), (start, cap, name)
    assert _state(rig.g, rig.idx) == before
    _every_path(rig, rig.g, rig.c, shared, rig.rng)
    rig.close()


def _copy_to_fresh(rig, shared, M, ledger_entries=1 << 16):
    """A fresh handle and model: the pending PEEK restored, the ledger imported, the lease chunks imported.  Returns the
    new side and the map old lease id -> new lease id."""
    from swarmdb_b200._native import RECV_PEEK
    cnt, ent, snd, pay = rig.g.receive_compact(None, BIG, RECV_PEEK)
    ent, snd = _renumber(ent, snd)
    pay = pay.copy()
    g2, c2 = _fresh(rig)
    c2, m2 = _attach(g2, c2, rig, shared, M, ledger_entries)
    assert g2.restore_compact(rig.idx, cnt, ent, snd, pay)[0] == len(ent)
    m2.redrive(rig.idx, cnt, ent, snd, pay)
    a, s, c = rig.g.ledger_export()
    assert set(zip(a.tolist(), s.tolist(), c.tolist())) == rig.m.ledger_triples()
    assert g2.ledger_import(a, s, c) == m2.ledger_import(a, s, c) == len(a)
    idmap = {}
    for ent, snd, pay, meta in _export_all(rig.g, 0, 100):
        base = g2.lease_import(ent, snd, pay, meta)
        assert base == m2.import_(ent, snd, pay, meta)
        idmap.update(zip(meta["id"].tolist(), range(base, base + len(ent))))
    other = SimpleNamespace(g=g2, c=c2, idx=rig.idx, rng=rig.rng, A=rig.A, G=rig.G)
    _loads_equal(g2, c2, rig.idx, "after the copy")
    return other, m2, idmap


def _leased_counts(sides, agents, k):
    """A leased receive on each (side, model): the delivery counts, equal on every side."""
    outs = [side.g.lease_deliveries(_lease(side, m, agents, k, 10.0)) for side, m in sides]
    for x in outs[1:]:
        assert np.array_equal(outs[0], x)
    return outs[0]


def test_round_trip_runs_in_lockstep(shared):
    from swarmdb_b200._native import LEASE_ACK, LEASE_RENEW
    M = 3
    rig = Rig(np.random.default_rng(21), G=8, F=64, extra=64)
    rig.check_advance = False
    rig.mixed(2)
    rig.c, rig.m = _attach(rig.g, rig.c, rig, shared, M, 1 << 16)
    _history(rig, rig.m)
    new, m2, idmap = _copy_to_fresh(rig, shared, M)
    one = SimpleNamespace(g=rig.g, c=rig.c, idx=rig.idx, rng=rig.rng, A=rig.A, G=rig.G)
    ls1, ls2 = rig.g.lease_stats(), new.g.lease_stats()
    assert ls1["live"] == ls2["live"] and ls1["entries_used"] - ls1["acked_unreclaimed"] == ls2["entries_used"]
    assert rig.g.lease_policy_stats()["dead"] == new.g.lease_policy_stats()["dead"]
    old = np.array(sorted(idmap), np.uint64)
    pairs = [(one, rig.m, old), (new, m2, np.array([idmap[i] for i in old.tolist()], np.uint64))]

    def each(fn):
        """fn on both sides: the device results must agree with each other."""
        outs = [fn(*p) for p in pairs]
        for a, b in zip(outs[0], outs[1]):
            assert np.asarray(a).tobytes() == np.asarray(b).tobytes(), fn
        return outs[0]

    def settle(side, m, ids, op, deadline=0.0):
        got = side.g.lease_settle(ids, op, deadline)[0]
        assert np.array_equal(got, m.settle(ids, op, deadline)[0])
        return (got,)

    def deliveries(side, m, ids):
        got = side.g.lease_deliveries(ids)
        assert np.array_equal(got, m.deliveries(ids))
        return (got,)

    each(deliveries)
    each(lambda side, m, ids: settle(side, m, ids[: len(ids) // 4], LEASE_ACK))
    each(lambda side, m, ids: settle(side, m, ids[len(ids) // 4: len(ids) // 2], LEASE_RENEW, 30.0))
    each(lambda side, m, ids: _sweep(side, m, 15.0))                  # the 10.0 and 20.0 deadlines come due
    got = each(lambda side, m, ids: (lambda new_ids: (new_ids - new_ids[0], side.g.lease_deliveries(new_ids)))(
        _lease(side, m, None, 3, 40.0)))
    assert 2 in got[1].tolist()                                        # counts carried by the imported ledger and store
    each(lambda side, m, ids: _sweep(side, m, 0.0, True))            # LEASE_ALL: kills at the limit, redelivers the rest
    each(lambda side, m, ids: _dead(side, m, None, peek=True))
    each(lambda side, m, ids: _dead(side, m, side.idx[::2]))
    each(lambda side, m, ids: (side.g.lease_stats()["live"], side.g.lease_policy_stats()["dead"]))
    _every_path(rig, rig.g, rig.c, shared, rig.rng)
    _every_path(rig, new.g, new.c, shared, rig.rng)
    new.g.close()
    rig.close()


def test_ledger_counts_continue_and_pairs_without_a_record_are_dropped(shared):
    from swarmdb_b200._native import SdbError
    rig = Rig(np.random.default_rng(31), G=8, F=64, extra=64)
    rig.check_advance = False
    rig.mixed(1)
    rig.c, rig.m = _attach(rig.g, rig.c, rig, shared, 10, 1 << 16)
    for _ in range(3):                                                 # counts 1, 2, 3 wait in the ledger
        ids = _lease(rig, rig.m, rig.idx[::2], 1000, 10.0)
        _nack_all(rig, rig.m, ids)
        _sweep(rig, rig.m, 0.0)
    gone = rig.idx[:64:2]                                              # these agents' redelivered records are consumed
    rig.g.receive_batch(gone, 1000)
    rig.c.receive_batch(gone, 1000)
    a, s, c = rig.g.ledger_export()
    assert set(zip(a.tolist(), s.tolist(), c.tolist())) == rig.m.ledger_triples() and set(c.tolist()) == {3}
    assert not np.isin(a, gone).any()
    extra_a = np.array([int(gone[0]), int(rig.idx[1])], np.uint32)    # one consumed pair, one that never existed
    extra_s = np.array([1, 1 << 40], np.uint64)
    new, m2, _ = _copy_to_fresh(rig, shared, 10)
    before = new.g.lease_policy_stats()
    assert new.g.ledger_import(extra_a, extra_s, [4, 4]) == m2.ledger_import(extra_a, extra_s, [4, 4]) == 0
    assert new.g.lease_policy_stats() == before
    got = _leased_counts([(rig, rig.m), (new, m2)], rig.idx[::2], 1000)
    assert len(got) and set(got.tolist()) == {4}                       # k + 1 for a record redelivered with count k
    # above the free room: refused, nothing changes
    g3, c3 = _fresh(rig)
    c3, m3 = _attach(g3, c3, rig, shared, 10, max(1, len(a) - 1))
    with pytest.raises(SdbError) as e:
        g3.ledger_import(a, s, c)
    assert e.value.code == -6 and g3.lease_policy_stats()["ledger_used"] == 0
    g3.close()
    _every_path(rig, new.g, new.c, shared, rig.rng)
    new.g.close()
    rig.close()


def test_refusals_change_nothing(shared):
    from swarmdb_b200._native import SdbError, Shard
    rig = Rig(np.random.default_rng(41), G=8, F=64, extra=64)
    rig.check_advance = False
    rig.mixed(1)
    rig.c, rig.m = _attach(rig.g, rig.c, rig, shared, 3, 1 << 16)
    _history(rig, rig.m)
    ent, snd, pay, meta = _export_all(rig.g)[0]                      # the whole store in one chunk
    assert len(ent) > 63 and (meta["state"] == 3).any() and (meta["state"] == 0).any()
    g2, c2 = _fresh(rig)
    c2, m2 = _attach(g2, c2, rig, shared, 3, 1 << 16)

    def refused(code, change=None, g=g2, flags=0):
        e, s, p, t = ent.copy(), snd.copy(), pay.copy(), meta.copy()
        if change:
            change(e, s, p, t)
        before = _state(g, rig.idx)
        with pytest.raises(SdbError) as err:
            g.lease_import(e, s, p, t, flags)
        assert err.value.code == code, (change, err.value)
        assert _state(g, rig.idx) == before

    def bad_send(e, s, p, t): e["send"][5] = len(s)
    def bad_agent(e, s, p, t): t["agent"][3] = rig.A
    def bad_receiver(e, s, p, t): e["receiver"][0] = (int(t["agent"][0]) + 1) % rig.A
    def bad_len(e, s, p, t): s["len"][-1] = 257
    def bad_prio(e, s, p, t): s["prio"][0] = 4
    def misaligned(e, s, p, t): s["payload_off"][1] += 8
    def past(e, s, p, t):
        r = int(np.nonzero(s["len"] > 0)[0][-1])
        s["payload_off"][r] = len(p) - 16
    def bad_state(e, s, p, t): t["state"][2] = 1

    refused(-1, flags=1)
    for change in (bad_send, bad_agent, bad_receiver, bad_len, bad_prio, misaligned, past, bad_state):
        refused(-1, change)
    nopol = Shard(max_agents=rig.A, max_groups=rig.G, ring_slots=512)
    nopol.lease_reserve(BIG, BIG * 256)
    refused(-1, g=nopol)                                               # dead letters on a handle without a policy
    small = Shard(max_agents=rig.A, max_groups=rig.G, ring_slots=512, max_recv_records=32)
    small.lease_reserve(BIG, BIG * 256)
    small.lease_set_policy(3, 1 << 10)
    refused(-6, g=small)                                               # more than one compact receive holds
    full = Shard(max_agents=rig.A, max_groups=rig.G, ring_slots=512)
    full.lease_reserve(63, 63 * 256)
    full.lease_set_policy(3, 1 << 10)
    refused(-6, g=full)                                                # lease store full
    with pytest.raises(SdbError):
        Shard(max_agents=8).lease_export(0)                            # no store
    for bad in (([rig.A], [1], [1]), ([0], [1], [0])):
        with pytest.raises(SdbError):
            g2.ledger_import(*bad)
    with pytest.raises(SdbError):
        nopol.ledger_import([0], [1], [1])
    with pytest.raises(SdbError):
        nopol.ledger_export()
    assert g2.lease_import(ent, snd, pay, meta) == m2.import_(ent, snd, pay, meta) == 0
    assert g2.lease_stats()["live"] == m2.live and g2.lease_policy_stats()["dead"] == int((meta["state"] == 3).sum())
    for x in (nopol, small, full, g2):
        x.close()
    rig.close()


def test_sequence_numbers_past_2_pow_32(shared):
    """Seqs straddle 2^32: the ledger and the store keep all 64 bits through export and import."""
    rig = Rig(np.random.default_rng(51), G=4, F=64, extra=64)
    rig.check_advance = False
    for g in rig.gs:
        g.advance_seq((1 << 32) - 300)
    rig.c.next_seq = (1 << 32) - 300
    rig.mixed(1)
    assert rig.g.stats()["next_seq"] > 1 << 32
    rig.c, rig.m = _attach(rig.g, rig.c, rig, shared, 4, 1 << 16)
    _history(rig, rig.m)
    new, m2, idmap = _copy_to_fresh(rig, shared, 4)
    got = _leased_counts([(rig, rig.m), (new, m2)], None, 1000)
    assert 3 in got.tolist()
    _every_path(rig, new.g, new.c, shared, rig.rng)
    new.g.close()
    rig.close()


def test_surface_snapshot_keeps_leases_dead_letters_and_counts(tmp_path, monkeypatch):
    monkeypatch.setenv("SDB_SHARED_PAYLOAD", "1")
    from swarmdb_b200.core import GpuConfig, SwarmsDB
    cfg = dict(max_agents=64, max_groups=4, arena_bytes=1 << 24, max_payload_bytes=1024, max_recv_records=1 << 12,
               max_recv_payload=1 << 20, lease_records=1 << 10, lease_max_deliveries=3, deterministic_ids=True)
    db = SwarmsDB(save_dir=tmp_path, auto_save=False, gpu_config=GpuConfig(**cfg))
    for a in "abcd":
        db.register_agent(a)
    acked = [db.send_message("a", f"ack {i}", receiver_id="b") for i in range(4)]
    again = [db.send_message("a", f"again {i}", receiver_id="b") for i in range(3)]
    poison = db.send_message("a", "poison", receiver_id="c")
    kept = [db.send_message("a", f"kept {i}", receiver_id="d") for i in range(5)]
    assert [m.id for m in db.receive_messages_leased("b", 10, visibility_timeout=600.0)] == acked + again
    assert db.ack_messages("b", acked[:2]) == 2
    assert db.nack_messages("b", again) == 3
    assert db.redeliver_expired() == 3
    got = db.receive_messages_leased("b", 10, visibility_timeout=600.0)
    assert [m.id for m in got] == again and {m.metadata["delivery_count"] for m in got} == {2}
    for _ in range(3):
        db.receive_messages_leased("c", 10, visibility_timeout=-1.0)
        db.redeliver_expired()
    assert db.get_stats()["dead_letters"] == 1
    db.receive_messages_leased("d", 2, visibility_timeout=600.0)
    db.nack_messages("d", kept[1:2])
    assert db.redeliver_expired() == 1                                 # pending again, its count in the ledger
    path = db.save_queue_snapshot(tmp_path / "q.npz", in_flight=True)
    db.close()

    db2 = SwarmsDB(save_dir=tmp_path, auto_save=False, gpu_config=GpuConfig(**cfg))
    db2.load_queue_snapshot(path)
    assert db2.ack_messages("b", acked) == 2                           # the two acked before the restart count 0
    assert db2.ack_messages("d", kept[:1]) == 1
    assert db2.nack_messages("b", again[:1]) == 1
    assert db2.redeliver_expired(now=math.inf) == 3                    # every live lease is due at +inf: again[0..2]
    back = db2.receive_messages_leased("b", 10, visibility_timeout=600.0)
    assert [m.id for m in back] == again and {m.metadata["delivery_count"] for m in back} == {3}
    dead = db2.dead_letters(peek=True)
    assert [m.id for m in dead] == [poison] and dead[0].metadata["delivery_count"] == 3
    rest = db2.receive_messages_leased("d", 10)                         # kept[1] was redelivered once before the restart
    assert [m.id for m in rest] == kept[2:] + kept[1:2]
    assert [m.metadata["delivery_count"] for m in rest] == [1, 1, 1, 2]
    db2.close()

    bare = SwarmsDB(save_dir=tmp_path, auto_save=False, gpu_config=GpuConfig(max_agents=64, max_groups=4))
    with pytest.raises(RuntimeError):
        bare.load_queue_snapshot(path)
    bare._check_fresh()
    bare.close()
