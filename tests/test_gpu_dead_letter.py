"""Dead letters of leased receives on the device (sdb_lease_set_policy / sdb_lease_deliveries / sdb_lease_dead_letters)
against tests/deadletter_ref.py, byte for byte, in both arena layouts.

Every leased receive must equal the model's receive and its delivery counts; every sweep the model's result, store
bookkeeping and policy stats; every dead-letter readout the model's compact result and counts.  Cases end by draining
every receive path (tests/test_gpu_restore.py::_every_path) against the oracle.
"""
import math

import numpy as np
import pytest

from tests.deadletter_ref import DeadLetterModel
from tests.ring_ref import BoundedOracle
from tests.test_gpu_compact_receive import Rig, _same
from tests.test_gpu_restore import _every_path, _expand, _groups, _loads_equal

pytestmark = pytest.mark.gpu

BIG = 1 << 20


@pytest.fixture(params=["1", "0"])
def shared(request, monkeypatch):
    monkeypatch.setenv("SDB_SHARED_PAYLOAD", request.param)
    return request.param == "1"


def _rig(seed, **kw):
    rig = Rig(np.random.default_rng(seed), G=8, F=64, extra=64, **kw)
    rig.check_advance = False
    rig.mixed(2)
    return rig


def _model(rig, shared, M, ledger, cap=BIG):
    from swarmdb_b200._native import recv_capacity
    rig.g.lease_reserve(cap, cap * 256)
    rig.g.lease_set_policy(M, ledger)
    if not isinstance(rig.c, BoundedOracle):
        rig.c = BoundedOracle(rig.c, rig.G, int(rig.g.cfg.ring_slots), _groups(rig), rig.A)
    return DeadLetterModel(rig.c, _groups(rig), recv_capacity(rig.g.cfg), cap, shared, M, ledger)


def _lease(rig, m, agents, k, deadline, flags=0):
    cnt, ent, snd, pay, base = rig.g.receive_leased(agents, k, deadline, flags)
    got = _expand((cnt, ent.copy(), snd.copy(), pay.copy()))
    want = m.lease(agents, k, deadline, flags, rows=ent["send"])
    _same(got, want[:3], "leased receive")
    assert base == want[3]
    ids = np.arange(base, base + len(ent), dtype=np.uint64)
    assert np.array_equal(rig.g.lease_deliveries(ids), m.deliveries(ids))
    return ids


def _sweep(rig, m, now, all_=False):
    from swarmdb_b200._native import LEASE_ALL
    st0 = rig.g.stats()
    got = rig.g.lease_sweep(now, LEASE_ALL if all_ else 0)
    want = m.sweep(now, all_)
    assert got == want, (got, want)
    st1 = rig.g.stats()
    assert st1["enqueued"] - st0["enqueued"] == got[0] and st1["next_seq"] == st0["next_seq"]
    assert st1["arena_tail_bytes"] - st0["arena_tail_bytes"] == 32 * m.last_granules, \
        (st1["arena_tail_bytes"] - st0["arena_tail_bytes"], 32 * m.last_granules)
    _loads_equal(rig.g, rig.c, rig.idx, "after sweep")
    ls, ps = rig.g.lease_stats(), rig.g.lease_policy_stats()
    for k, v in m.stats().items():
        assert ls[k] == v, (k, ls[k], v)
    for k, v in m.policy_stats().items():
        assert ps[k] == v, (k, ps[k], v)
    return got


def _dead(rig, m, agents, peek=False, cap=None):
    from swarmdb_b200._native import ENTRY_DTYPE, RECV_PEEK, SEND_DTYPE, recv_capacity
    kw = {}
    if cap is not None:
        kw = dict(out_entries=np.zeros(cap, ENTRY_DTYPE), out_sends=np.zeros(cap, SEND_DTYPE))
    cnt, ent, snd, pay, dl = rig.g.lease_dead_letters(agents, RECV_PEEK if peek else 0, **kw)
    got = tuple(x.copy() for x in (cnt, ent, snd, pay, dl))
    want = m.dead_letters(agents, min(cap or BIG, recv_capacity(rig.g.cfg)), peek)
    assert np.array_equal(got[0], want[0][: len(got[0])]) and not want[0][len(got[0]):].any()
    for x, y, name in zip(got[1:], want[1:], ("entries", "sends", "payload", "deliveries")):
        assert x.tobytes() == y.tobytes(), name
    return got


def _nack_all(rig, m, ids):
    from swarmdb_b200._native import LEASE_RENEW
    got = rig.g.lease_settle(ids, LEASE_RENEW, -math.inf)
    want = m.settle(ids, LEASE_RENEW, -math.inf)
    assert np.array_equal(got[0], want[0])


def _to_the_limit(rig, m, agents, k=1000, rounds=16):
    """Lease, nack and sweep until the agents have nothing pending and no lease is live: every record of theirs ends
    as a dead letter."""
    for _ in range(rounds):
        ids = _lease(rig, m, agents, k, 10.0)
        if len(ids):
            _nack_all(rig, m, ids)
        elif m.live == 0:
            break
        _sweep(rig, m, 0.0)
    assert m.live == 0 and rig.g.lease_stats()["live"] == 0
    assert not rig.g.agent_loads(agents)["pending"].any()


def test_counts_rise_to_the_limit_then_the_sweep_dead_letters(shared):
    from swarmdb_b200._native import RECV_PRIORITY
    M = 3
    rig = _rig(1)
    m = _model(rig, shared, M, 1 << 16)
    ids = _lease(rig, m, None, 1000, 10.0)                            # everything: redeliveries then come back alone
    assert len(ids) > 0
    for k in range(1, M + 1):
        assert set(rig.g.lease_deliveries(ids).tolist()) == {k}
        _nack_all(rig, m, ids)
        red, blocked, left = _sweep(rig, m, 0.0)
        if k < M:
            assert red == len(ids) and blocked == 0 and left == 0
            assert rig.g.lease_policy_stats()["ledger_used"] == len(ids)
            ids = _lease(rig, m, None, 1000, 10.0, RECV_PRIORITY if k == 1 else 0)
        else:
            assert red == 0 and rig.g.lease_policy_stats()["dead"] == len(ids)
    ls = rig.g.lease_stats()
    assert ls["live"] == 0 and ls["entries_used"] == len(ids)       # dead letters keep their space
    assert rig.g.lease_settle(ids, 0)[1] == 0                          # and are not live
    a = _dead(rig, m, None, peek=True)
    b = _dead(rig, m, None, peek=True)
    assert all(x.tobytes() == y.tobytes() for x, y in zip(a, b))
    assert set(a[4].tolist()) == {M}
    first = np.unique(a[1]["send"], return_index=True)[1]
    assert np.array_equal(np.sort(first), first)                       # rows numbered by first appearance
    # take agent by agent in a listed order, then redrive through restore_compact
    agents = rig.rng.permutation(rig.idx)[:200].astype(np.uint32)
    cnt, ent, snd, pay, _ = _dead(rig, m, agents)
    assert rig.g.restore_compact(agents, cnt, ent, snd, pay)[0] == len(ent)
    m.redrive(agents, cnt, ent, snd, pay)
    while True:
        cnt, ent, snd, pay, _ = _dead(rig, m, None)
        if len(ent) == 0:
            break
        idx = np.arange(len(cnt), dtype=np.uint32)
        assert rig.g.restore_compact(idx, cnt, ent, snd, pay)[0] == len(ent)
        m.redrive(idx, cnt, ent, snd, pay)
    assert rig.g.lease_stats()["entries_used"] == 0 and rig.g.lease_policy_stats()["dead"] == 0
    ids = _lease(rig, m, None, 2, 10.0)
    assert set(rig.g.lease_deliveries(ids).tolist()) <= {1, 2}       # redriven records restart at 1
    _every_path(rig, rig.g, rig.c, shared, rig.rng)
    rig.close()


def test_dead_letter_capacity_keeps_the_lead_agent_rule(shared):
    rig = _rig(2)
    m = _model(rig, shared, 1, 64)
    ids = _lease(rig, m, None, 6, 10.0)
    _sweep(rig, m, 0.0, True)
    assert rig.g.lease_policy_stats()["dead"] == len(ids)
    agents = rig.rng.permutation(rig.idx)[:300].astype(np.uint32)
    total = 0
    while True:
        cnt, ent, *_ = _dead(rig, m, agents, cap=4)                   # at most 4 records: a lead agent with 6 gets 4
        if len(ent) == 0:
            break
        assert len(ent) <= 4
        total += len(ent)
    assert total > 0
    _every_path(rig, rig.g, rig.c, shared, rig.rng)
    rig.close()


def test_the_ledger_is_exact_after_other_paths_consume_a_redelivered_record(shared):
    from swarmdb_b200._native import EXPIRE_ALL, WHERE_DROP, make_filter
    rig = _rig(3)
    m = _model(rig, shared, 100, 1 << 12)
    agents = rig.idx[rig.G * rig.F: rig.G * rig.F + 3].astype(np.uint32)  # non-members with p2p and broadcast traffic
    ids = _lease(rig, m, agents, 1000, 10.0)                          # everything they have: only redeliveries stay
    assert len(ids) >= 6
    _nack_all(rig, m, ids)
    _sweep(rig, m, 0.0)
    # agent 0: a plain receive takes its oldest redelivered record; agent 1: expiry; agent 2: a WHERE_DROP by seq
    seqs = {}
    for a in agents.tolist():
        pend = rig.g.receive_compact([a], 1, 2)[1]                     # PEEK: the oldest pending record
        if len(pend) == 0:
            continue
        seqs[a] = int(pend["seq"][0])
    a0, a1, a2 = agents.tolist()
    took = {}
    if a0 in seqs:
        cnt, ent, snd, pay = (x.copy() for x in rig.g.receive_compact([a0], 1))
        rig.c.receive_batch([a0], 1)
        took[a0] = (cnt, ent, snd, pay)
    if a1 in seqs:
        cnt, ent, snd, pay = (x.copy() for x in rig.g.expire([a1], math.inf, EXPIRE_ALL))
        rig.c.expire([a1], math.inf, EXPIRE_ALL)
        took[a1] = (cnt, ent, snd, pay)
    if a2 in seqs:
        f = make_filter(seq=(seqs[a2], seqs[a2] + 1))
        rig.g.receive_where([a2], 1, WHERE_DROP, f, drop=True)
        rig.c.receive_where([a2], 1, 0, f, drop=True)
    for a, (cnt, ent, snd, pay) in took.items():                        # requeued with the same seqs
        assert rig.g.restore_compact([a], cnt, ent, snd, pay)[0] == len(ent)
        m.redrive([a], cnt, ent, snd, pay)
    ids = _lease(rig, m, agents, 100, 10.0)                             # counts: model (1 for the requeued, 2 for the rest)
    d = rig.g.lease_deliveries(ids)
    assert 1 in d.tolist() and 2 in d.tolist()
    _every_path(rig, rig.g, rig.c, shared, rig.rng)
    rig.close()


def test_a_full_ledger_holds_records_until_the_redelivered_ones_are_received(shared):
    rig = _rig(4)
    m = _model(rig, shared, 10, 5)
    ids = _lease(rig, m, None, 2, 10.0)
    assert len(ids) > 10
    _nack_all(rig, m, ids)
    red, _, left = _sweep(rig, m, 0.0)
    assert red == 5 and left == len(ids) - 5
    assert _sweep(rig, m, 0.0) == (0, 0, len(ids) - 5)
    _lease(rig, m, None, 1000, 10.0)                                    # takes the redelivered records' ledger entries
    red, _, left = _sweep(rig, m, 0.0)
    assert red == 5 and left == len(ids) - 10
    _every_path(rig, rig.g, rig.c, shared, rig.rng)
    rig.close()


def test_a_blocked_ring_under_a_policy(shared):
    """Agents x < y < z < w with 4 leases each, a ring of 16 slots, a limit of 3 and a ledger of 12 entries: the first
    sweep takes 12 due records (w's 4 are held by the ledger), y's refilled ring blocks it, z's ring has exactly the
    room for its 4.  The ledger numbers x's and z's entries densely across y's dropped run."""
    from tests.test_gpu_shared_layout import _payloads
    R = 16
    rig = Rig(np.random.default_rng(9), G=8, F=64, extra=64, ring_slots=R)
    rig.check_advance = False
    x, y, z, w = (rig.G * rig.F + k for k in (1, 2, 3, 4))

    def send_to(receivers):
        r = np.asarray(receivers, np.uint32)
        lens, off, buf = _payloads(rig.rng, len(r), 100)
        s = rig.rng.integers(0, rig.A, len(r))
        assert rig.c.send_batch(s, r, None, None, lens, off, buf) == rig.g.send_batch(s, r, None, None, lens, off, buf)

    send_to([x] * 4 + [y] * 4 + [z] * 4 + [w] * 4)
    send_to(rig.rng.integers(0, x, 100))
    m = _model(rig, shared, 3, 12)
    agents = [x, y, z, w]
    ids = _lease(rig, m, agents, 100, 10.0)
    assert len(ids) == 16
    y_ids = ids[4:8]
    _nack_all(rig, m, ids)
    send_to([y] * (R - 3) + [z] * (R - 4))                             # y: 3 free slots for 4 records, z: 4 for 4
    assert rig.c.capacity(y) == 3 and rig.c.capacity(z) == 4
    assert _sweep(rig, m, 0.0) == (8, 1, 4)
    ps = rig.g.lease_policy_stats()
    assert ps["held_by_ledger_total"] == 4 and ps["ledger_used"] == 8
    assert rig.g.lease_stats()["live"] == 8
    assert rig.g.lease_deliveries(y_ids).tolist() == [1] * 4          # y's leases stay live with their counts
    _same(rig.g.receive_batch([y], 100), rig.c.receive_batch([y], 100), "y's newer records")
    assert _sweep(rig, m, 0.0) == (4, 0, 4)                            # y's records come back; w's wait for room
    _to_the_limit(rig, m, agents)                                      # counts continue to the limit
    assert rig.g.lease_policy_stats()["dead"] == 16 + R - 4            # z's newer records too
    cnt, ent, snd, pay, dl = _dead(rig, m, agents, peek=True)
    assert set(dl.tolist()) == {3}
    cnt, ent, snd, pay, _ = _dead(rig, m, agents[::-1])
    assert rig.g.restore_compact(agents[::-1], cnt, ent, snd, pay)[0] == len(ent)
    m.redrive(agents[::-1], cnt, ent, snd, pay)
    assert rig.g.lease_policy_stats()["dead"] == 0
    _every_path(rig, rig.g, rig.c, shared, rig.rng)
    rig.close()


def test_lease_all_kills_only_leases_at_the_limit(shared):
    rig = _rig(5)
    m = _model(rig, shared, 2, 1 << 12)
    ids = _lease(rig, m, None, 1000, 10.0)
    _sweep(rig, m, 0.0, True)                                          # count 1: every live lease is redelivered
    ids2 = _lease(rig, m, rig.idx[: len(rig.idx) // 2], 1000, 10.0)    # half of them leased again: count 2
    assert set(rig.g.lease_deliveries(ids2).tolist()) <= {1, 2} and 2 in rig.g.lease_deliveries(ids2).tolist()
    _lease(rig, m, rig.idx[len(rig.idx) // 2:], 1000, 10.0)
    _sweep(rig, m, 0.0, True)                                          # LEASE_ALL: count-2 leases die, the rest redeliver
    assert rig.g.lease_policy_stats()["dead"] > 0 and len(ids) > 0
    _every_path(rig, rig.g, rig.c, shared, rig.rng)
    rig.close()


def test_arena_full_sweep_leaves_store_and_ledger_unchanged(shared):
    from swarmdb_b200._native import SdbError
    rig = _rig(6, arena_bytes=1 << 24)
    m = _model(rig, shared, 3, 1 << 12)
    ids = _lease(rig, m, None, 1000, 10.0)
    _nack_all(rig, m, ids)
    _sweep(rig, m, 0.0)
    ids = _lease(rig, m, None, 1000, 10.0)
    _nack_all(rig, m, ids)
    while True:                                                        # fill the arena with pending traffic
        try:
            rig.p2p(400)
        except SdbError:
            break
    before = (rig.g.lease_stats(), rig.g.lease_policy_stats(), rig.g.stats()["enqueued"])
    with pytest.raises(SdbError) as e:
        rig.g.lease_sweep(0.0)
    assert e.value.code == -5
    assert before == (rig.g.lease_stats(), rig.g.lease_policy_stats(), rig.g.stats()["enqueued"])
    assert set(rig.g.lease_deliveries(ids).tolist()) == {2}
    rig.close()


def test_refusals_zero_outputs_and_change_nothing():
    from swarmdb_b200._native import SdbError
    rig = _rig(7)
    g = rig.g
    with pytest.raises(SdbError):
        g.lease_set_policy(2, 16)                                      # no store
    g.lease_reserve(BIG, BIG * 256)
    with pytest.raises(SdbError):
        g.lease_deliveries([0])                                        # no policy
    with pytest.raises(SdbError):
        g.lease_dead_letters(None)
    with pytest.raises(SdbError):
        g.lease_set_policy(2, 0)                                       # a limit without a ledger
    g.lease_set_policy(2, 16)
    g.receive_leased(None, 1, 10.0)
    with pytest.raises(SdbError):
        g.lease_set_policy(3, 16)                                      # live leases
    with pytest.raises(SdbError):
        g.lease_dead_letters([1, 1])
    with pytest.raises(SdbError):
        g.lease_dead_letters(None, 4)                                  # an unknown flag bit
    st = (g.lease_stats(), g.lease_policy_stats())
    assert st[1]["max_deliveries"] == 2 and st[1]["ledger_cap"] == 16
    assert rig.g.lease_deliveries([10 ** 9]).tolist() == [0]
    rig.close()


def test_a_policy_turned_off_behaves_like_no_policy(shared):
    from swarmdb_b200._native import LEASE_ACK, LEASE_RENEW
    rig = _rig(8, twins=2)
    for g in rig.gs:
        g.lease_reserve(BIG, BIG * 256)
    rig.gs[1].lease_set_policy(2, 64)
    rig.gs[1].lease_set_policy(0, 0)
    launches = []
    outs = []
    for g in rig.gs:
        k0 = g.stats()["kernel_launches"]
        res = [x.copy() for x in g.receive_leased(None, 3, 10.0)[:4]]
        base = g.receive_leased(None, 1, 10.0)[4]
        g.lease_settle(np.arange(0, base, 2, dtype=np.uint64), LEASE_ACK)
        g.lease_settle(np.arange(1, base, 2, dtype=np.uint64), LEASE_RENEW, -math.inf)
        res.append(np.array(g.lease_sweep(0.0)))
        res += [x.copy() for x in g.receive_compact(None, 100)]
        outs.append(res)
        launches.append(g.stats()["kernel_launches"] - k0)
    assert all(x.tobytes() == y.tobytes() for x, y in zip(*outs))
    assert launches[0] == launches[1]
    rig.close()


def test_surface_dead_letters_and_redrive(tmp_path, monkeypatch):
    monkeypatch.setenv("SDB_SHARED_PAYLOAD", "1")
    from swarmdb_b200.core import GpuConfig, MessageStatus, SwarmsDB
    db = SwarmsDB(save_dir=tmp_path, auto_save=False,
                  gpu_config=GpuConfig(max_agents=64, max_groups=4, arena_bytes=1 << 24, max_payload_bytes=1024,
                                       max_recv_records=1 << 12, max_recv_payload=1 << 20, lease_records=1 << 10,
                                       lease_max_deliveries=2, deterministic_ids=True))
    db.register_agent("a"); db.register_agent("b")
    mid = db.send_message("a", "poison", receiver_id="b")
    for k in (1, 2):
        got = db.receive_messages_leased("b", 10, visibility_timeout=-1.0)
        assert [m.id for m in got] == [mid] and got[0].metadata["delivery_count"] == k
        db.redeliver_expired()
    assert db.get_stats()["dead_letters"] == 1
    assert db.receive_messages_leased("b", 10) == []
    peek = db.dead_letters(peek=True)
    assert [m.id for m in peek] == [mid] and peek[0].status == MessageStatus.FAILED
    assert peek[0].metadata["delivery_count"] == 2
    assert db.redrive_dead_letters() == 1 and db.get_stats()["dead_letters"] == 0
    again = db.receive_messages_leased("b", 10, visibility_timeout=-1.0)
    assert [m.id for m in again] == [mid] and again[0].metadata["delivery_count"] == 1
    db.redeliver_expired()
    db.receive_messages_leased("b", 10, visibility_timeout=-1.0)
    db.redeliver_expired()
    taken = db.dead_letters("b")
    assert [m.id for m in taken] == [mid] and db.messages[mid].status == MessageStatus.FAILED
    assert db.dead_letters() == [] and db.get_stats()["dead_letters"] == 0
    db.close()
