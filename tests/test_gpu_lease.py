"""Leased receives on the device (sdb_receive_leased / sdb_lease_settle / sdb_lease_sweep) against tests/lease_ref.py,
byte for byte.

Every leased receive must equal the oracle's receive (and, on a twin handle, sdb_receive_compact's bytes); every settle
and sweep must return what the model returns; after each sweep stats, agent loads, the arena advance and the store's
bookkeeping must agree, and at the end of a case every receive path (tests/test_gpu_restore.py::_every_path) must
deliver what the oracle delivers.  Each case runs in both arena layouts.
"""
import math

import numpy as np
import pytest

from tests.lease_ref import LeaseModel
from tests.ring_ref import BoundedOracle
from tests.test_gpu_compact_receive import Rig, _same
from tests.test_gpu_restore import _every_path, _expand, _groups, _loads_equal

pytestmark = pytest.mark.gpu

BIG = 1 << 20


def _model(rig, cap, shared, rec_cap=None):
    """The lease model over the rig's oracle, bounded by the handle's rings from here on (the rig has only sent so
    far: its windows are contiguous)."""
    from swarmdb_b200._native import recv_capacity
    if not isinstance(rig.c, BoundedOracle):
        rig.c = BoundedOracle(rig.c, rig.G, int(rig.g.cfg.ring_slots), _groups(rig), rig.A)
    return LeaseModel(rig.c, _groups(rig), rec_cap or recv_capacity(rig.g.cfg), cap, shared)


def _lease(rig, m, agents, k, deadline, flags=0):
    st0 = rig.g.stats()
    cnt, ent, snd, pay, base = rig.g.receive_leased(agents, k, deadline, flags)
    got = _expand((cnt, ent.copy(), snd.copy(), pay.copy()))
    want = m.lease(agents, k, deadline, flags, rows=ent["send"])
    _same(got, want[:3], "leased receive")
    assert base == want[3]
    assert rig.g.stats()["delivered"] - st0["delivered"] == len(ent)
    _loads_equal(rig.g, rig.c, rig.idx, "after lease")
    return ent, base


def _settle(rig, m, ids, op, deadline=0.0):
    got = rig.g.lease_settle(ids, op, deadline)
    want = m.settle(ids, op, deadline)
    assert np.array_equal(got[0], want[0]) and got[1] == want[1]
    return got[1]


def _sweep(rig, m, now, all_=False):
    from swarmdb_b200._native import LEASE_ALL
    st0 = rig.g.stats()
    got = rig.g.lease_sweep(now, LEASE_ALL if all_ else 0)
    want = m.sweep(now, all_)
    assert got == want, (got, want)
    st1 = rig.g.stats()
    assert st1["enqueued"] - st0["enqueued"] == got[0] and st1["delivered"] == st0["delivered"]
    assert st1["next_seq"] == st0["next_seq"]
    if got[0]:
        assert st1["arena_tail_bytes"] - st0["arena_tail_bytes"] == 32 * m.last_granules
    _loads_equal(rig.g, rig.c, rig.idx, "after sweep")
    ls = rig.g.lease_stats()
    for k, v in m.stats().items():
        assert ls[k] == v, (k, ls[k], v)
    return got


def _drain_sweeps(rig, m, now, all_=False):
    total = 0
    while True:
        red, _, left = _sweep(rig, m, now, all_)
        total += red
        if left == 0 or red == 0:
            return total


@pytest.fixture(params=["1", "0"])
def shared(request, monkeypatch):
    monkeypatch.setenv("SDB_SHARED_PAYLOAD", request.param)
    return request.param == "1"


def _rig(seed, **kw):
    rig = Rig(np.random.default_rng(seed), G=8, F=64, extra=64, **kw)
    rig.check_advance = False
    rig.mixed(2)
    return rig


def test_leased_receive_equals_compact_receive_on_a_twin(shared):
    from swarmdb_b200._native import RECV_PRIORITY
    rig = _rig(1, twins=2)
    rig.g.lease_reserve(BIG, BIG * 256)
    for agents, k, flags in ((rig.idx[:300], 3, 0), (rig.idx[100:700], 2, RECV_PRIORITY), (None, 5, 0)):
        a = rig.g.receive_leased(agents, k, 1.0, flags)
        b = rig.gs[1].receive_compact(agents, k, flags)
        for x, y in zip(a[:4], b):
            assert x.tobytes() == y.tobytes()
    rig.close()


def test_ack_all_then_sweep_redelivers_nothing(shared):
    from swarmdb_b200._native import LEASE_ACK
    rig = _rig(2)
    rig.g.lease_reserve(BIG, BIG * 256)
    m = _model(rig, BIG, shared)
    ent, base = _lease(rig, m, None, 4, 5.0)
    n = len(ent)
    assert n > 0
    ids = np.arange(base, base + n, dtype=np.uint64)
    assert _settle(rig, m, ids, LEASE_ACK) == n
    assert _settle(rig, m, ids[:10], LEASE_ACK) == 0               # already acked
    assert _sweep(rig, m, 0.0, True) == (0, 0, 0)
    assert rig.g.lease_stats()["entries_used"] == 0 and rig.g.lease_stats()["acked_total"] == n
    _every_path(rig, rig.g, rig.c, shared, rig.rng)
    rig.close()


def test_deadline_nack_extend_and_partial_acks(shared):
    from swarmdb_b200._native import LEASE_ACK, LEASE_RENEW
    rig = _rig(3)
    rig.g.lease_reserve(BIG, BIG * 256)
    m = _model(rig, BIG, shared)
    ent, base = _lease(rig, m, None, 6, 10.0)
    ids = np.arange(base, base + len(ent), dtype=np.uint64)
    rig.mixed(1)                                                      # newer pending records: redelivery goes behind them
    assert _sweep(rig, m, 9.5)[0] == 0                               # before the deadline
    rng = rig.rng
    perm = rng.permutation(ids)
    acked, nacked, extended = perm[: len(ids) // 3], perm[len(ids) // 3: len(ids) // 2], perm[len(ids) // 2: 2 * len(ids) // 3]
    _settle(rig, m, acked, LEASE_ACK)                                # partial acks, group rows shared with unacked records
    _settle(rig, m, nacked, LEASE_RENEW, -math.inf)
    _settle(rig, m, extended, LEASE_RENEW, 100.0)
    _settle(rig, m, np.array([ids[-1] + 7, acked[0], acked[0]], np.uint64), LEASE_ACK)   # unknown, late, repeated
    red = _drain_sweeps(rig, m, -1.0)                                # only the nacks
    assert red == len(nacked)
    late = _settle(rig, m, nacked[:5], LEASE_ACK)                    # acks after redelivery read 0
    assert late == 0
    red = _drain_sweeps(rig, m, 10.0)                                # at the deadline: the rest but the extended ones
    assert red == len(ids) - len(acked) - len(nacked) - len(extended)
    assert rig.g.lease_stats()["live"] == len(extended)
    _drain_sweeps(rig, m, math.nan)                                  # NaN: nothing due
    assert rig.g.lease_stats()["live"] == len(extended)
    _drain_sweeps(rig, m, 100.0)
    assert rig.g.lease_stats()["live"] == 0
    _every_path(rig, rig.g, rig.c, shared, rig.rng)
    rig.close()


def test_priority_leases_broadcasts_and_private_images(shared):
    from swarmdb_b200._native import RECV_PRIORITY, LEASE_ACK
    rig = _rig(4)
    rig.broadcast(20)
    rig.g.lease_reserve(BIG, BIG * 256)
    m = _model(rig, BIG, shared)
    ent, base = _lease(rig, m, None, 5, 1.0, RECV_PRIORITY)
    ent2, base2 = _lease(rig, m, rig.idx[::3], 3, 2.0)
    _settle(rig, m, np.arange(base, base + len(ent), 5, dtype=np.uint64), LEASE_ACK)
    rig.mixed(1)
    _drain_sweeps(rig, m, 1.5)
    _drain_sweeps(rig, m, 0.0, True)
    _every_path(rig, rig.g, rig.c, shared, rig.rng)
    rig.close()


def test_store_caps_the_receive_and_space_returns_after_a_sweep(shared):
    from swarmdb_b200._native import LEASE_ACK, SdbError
    rig = _rig(5)
    cap = 700
    rig.g.lease_reserve(cap, BIG * 256)
    m = _model(rig, cap, shared)
    ent, base = _lease(rig, m, None, 50, 1.0)
    while rig.g.lease_stats()["entries_used"] < cap:                 # the lead agent takes what is left
        assert len(_lease(rig, m, None, 50, 1.0)[0]) > 0
    assert rig.g.lease_stats()["entries_used"] == cap
    st = rig.g.stats()
    with pytest.raises(SdbError) as e:
        rig.g.receive_leased(None, 50, 1.0)
    assert e.value.code == -6 and "lease store full" in str(e.value)
    assert rig.g.stats() == st
    _settle(rig, m, np.arange(base, base + 300, dtype=np.uint64), LEASE_ACK)
    assert _sweep(rig, m, 0.5)[0] == 0                               # reclaims the acked entries
    assert rig.g.lease_stats()["entries_used"] == cap - 300
    ent, base = _lease(rig, m, None, 50, 2.0)
    assert 0 < len(ent) <= 300
    _drain_sweeps(rig, m, 0.0, True)
    _every_path(rig, rig.g, rig.c, shared, rig.rng)
    rig.close()


def test_more_due_records_than_one_call_holds(shared):
    rig = _rig(6, max_recv_records=256)
    rig.g.lease_reserve(BIG, BIG * 256)
    m = _model(rig, BIG, shared)
    for _ in range(6):
        _lease(rig, m, rig.idx, 1, 1.0)
    calls = 0
    while True:
        red, blocked, left = _sweep(rig, m, 1.0)
        calls += 1
        if left == 0:
            break
    assert calls > 2
    while True:                                                      # drain at this handle's capacity
        got = rig.g.receive_batch(None, 1 << 20)
        _same(got, m._receive(rig.idx, 1 << 20, 0, 256), "drain")
        if len(got[1]) == 0:
            break
    rig.close()


def test_full_ring_blocks_only_its_agent(shared):
    R = 128
    rig = _rig(7, ring_slots=R)
    rig.g.lease_reserve(BIG, BIG * 256)
    m = _model(rig, BIG, shared)
    _lease(rig, m, None, R, 1.0)
    a = int(rig.G * rig.F)                                           # a non-member agent
    assert any(rec["agent"] == a for rec in m.recs)
    from tests.test_gpu_shared_layout import _payloads
    lens, off, buf = _payloads(rig.rng, R, 64)
    s = np.full(R, 1, np.uint32)
    r = np.full(R, a, np.uint32)
    assert rig.c.send_batch(s, r, None, None, lens, off, buf) == rig.g.send_batch(s, r, None, None, lens, off, buf)
    red, blocked, left = _sweep(rig, m, 1.0)
    assert blocked == 1 and red > 0
    assert rig.g.lease_stats()["live"] == sum(1 for rec in m.recs if rec["agent"] == a) > 0
    _same(rig.g.receive_batch([a], R), rig.c.receive_batch([a], R), "full ring")
    _drain_sweeps(rig, m, 1.0)
    assert rig.g.lease_stats()["live"] == 0
    _every_path(rig, rig.g, rig.c, shared, rig.rng)
    rig.close()


def test_stream_order_group_lease_comes_back_in_the_sends_arena_bytes(shared):
    from tests.test_gpu_shared_layout import _arena_advance
    rng = np.random.default_rng(8)
    rig = Rig(rng, G=8, F=64, extra=64)
    rig.check_advance = False
    rig.g.lease_reserve(BIG, BIG * 256)
    m = _model(rig, BIG, shared)
    n = 300
    s, grp, prio = rng.integers(rig.G * rig.F, rig.A, n), rng.integers(0, rig.G, n), rng.integers(0, 4, n)
    from tests.test_gpu_shared_layout import _payloads
    lens, off, buf = _payloads(rng, n, 256)
    t0 = rig.g.stats()["arena_tail_bytes"]
    base = rig.c.send_group_batch(s, grp, prio, None, lens, off, buf)[0]
    assert rig.g.send_group_batch(s, grp, prio, None, lens, off, buf) == base
    sent = rig.g.stats()["arena_tail_bytes"] - t0
    assert sent == _arena_advance(rig.F, lens)
    ent, _ = _lease(rig, m, None, 1 << 20, 1.0)                     # stream order: the whole batch
    assert len(ent) == n * rig.F
    t1 = rig.g.stats()["arena_tail_bytes"]
    assert _drain_sweeps(rig, m, 1.0) == n * rig.F
    assert rig.g.stats()["arena_tail_bytes"] - t1 == sent            # the same layout: F headers + one payload per send
    # ... and the compact receive finds the sends' rows again: one row per send
    cnt, ent2, snd2, pay2 = rig.g.receive_compact(None, 1 << 20)
    assert len(snd2) == (n if shared else n * rig.F)
    rig.c.receive_batch(rig.idx, 1 << 20, rec_cap=1 << 21)
    rig.close()


def test_arena_full_leaves_store_and_rings_unchanged(shared):
    from swarmdb_b200._native import SdbError
    rng = np.random.default_rng(9)
    rig = Rig(rng, G=2, F=16, extra=32, arena_bytes=1 << 16)
    rig.check_advance = False
    rig.g.lease_reserve(BIG, BIG * 256)
    m = _model(rig, BIG, shared)
    rig.p2p(100, 128)
    _lease(rig, m, None, 1 << 20, 1.0)
    # fill the arena with newer records nobody receives
    from tests.test_gpu_shared_layout import _payloads
    while True:
        lens, off, buf = _payloads(rng, 16, 256)
        lens[:] = 256
        s, r = rng.integers(0, rig.A, 16), rng.integers(0, rig.A, 16)
        try:
            rig.g.send_batch(s, r, None, None, lens, off, buf)
        except SdbError as e:
            assert e.code == -5
            break
        rig.c.send_batch(s, r, None, None, lens, off, buf)
    st, ls, loads = rig.g.stats(), rig.g.lease_stats(), rig.g.agent_loads(rig.idx)
    with pytest.raises(SdbError) as e:
        rig.g.lease_sweep(0.0, 1)
    assert e.value.code == -5
    st2 = rig.g.stats()
    for k in ("kernel_launches", "arena_floor_bytes"):               # the failed reservation may recompute the floor
        st2[k] = st[k]
    assert st2 == st and rig.g.lease_stats() == ls
    assert rig.g.agent_loads(rig.idx).tobytes() == loads.tobytes()
    rig.g.receive_batch(None, 1 << 20)
    rig.c.receive_batch(rig.idx, 1 << 20, rec_cap=1 << 21)
    assert _drain_sweeps(rig, m, 0.0, True) > 0
    _same(rig.g.receive_batch(None, 1 << 20), rig.c.receive_batch(rig.idx, 1 << 20, rec_cap=1 << 21), "after the sweep")
    rig.close()


def test_refusals_leave_outputs_zero_and_state_unchanged():
    from swarmdb_b200._native import LEASE_ACK, RECV_ASYNC, RECV_PEEK, SdbError
    rig = _rig(10)
    g = rig.g
    st, loads = g.stats(), g.agent_loads(rig.idx)

    def refused(fn, code=-1):
        with pytest.raises(SdbError) as e:
            fn()
        assert e.value.code == code
        s2 = g.stats()
        s2["kernel_launches"] = st["kernel_launches"]
        assert s2 == st and g.agent_loads(rig.idx).tobytes() == loads.tobytes()

    refused(lambda: g.receive_leased(None, 4, 1.0))                 # no store
    refused(lambda: g.lease_settle([0], LEASE_ACK))
    refused(lambda: g.lease_sweep(0.0))
    g.lease_reserve(1024, 1 << 20)
    refused(lambda: g.receive_leased(None, 4, 1.0, RECV_PEEK))
    refused(lambda: g.receive_leased(None, 4, 1.0, RECV_ASYNC))
    refused(lambda: g.receive_leased(None, 4, 1.0, 64))
    refused(lambda: g.lease_settle([0], 7))
    refused(lambda: g.lease_sweep(0.0, 2))
    refused(lambda: g.receive_leased([1, 1], 4, 1.0))
    g.lease_reserve(8, 100)                                          # a store smaller than one maximum-size record
    refused(lambda: g.receive_leased(None, 4, 1.0), -6)
    g.lease_reserve(1024, 1 << 20)
    m = _model(rig, 1024, True)
    _lease(rig, m, rig.idx[:10], 2, 1.0)
    with pytest.raises(SdbError) as e:
        g.lease_reserve(2048, 1 << 20)                               # live leases
    assert e.value.code == -1
    assert g.lease_stats()["live"] == m.live > 0
    rig.close()


def test_swarmsdb_surface_on_the_device(tmp_path):
    """receive_messages_leased / ack / nack / extend / mark_message_as_processed / redeliver_expired on a real shard."""
    import swarmdb_b200 as sdb
    from swarmdb_b200.core import MessageStatus
    cfg = sdb.GpuConfig(max_agents=64, max_groups=4, deterministic_ids=True, lease_records=1024)
    db = sdb.SwarmsDB(save_dir=str(tmp_path), auto_save=False, gpu_config=cfg)
    for a in ("a", "b", "c"):
        db.register_agent(a)
    ids = [db.send_message("a", f"m{k}", receiver_id="b") for k in range(5)]
    bid = db.broadcast_message("a", "all")
    got = db.receive_messages_leased("b", 10, visibility_timeout=60.0)
    assert [m.id for m in got] == ids + [bid] and all(m.status == MessageStatus.READ for m in got)
    assert [m.content for m in got] == [f"m{k}" for k in range(5)] + ["all"]
    assert db.receive_messages_leased("b", 10) == []
    assert [m.id for m in db.receive_messages_leased("c", 10)] == [bid]
    assert db.ack_messages("b", ids[:2]) == 2 and db.ack_messages("b", ids[:1]) == 0
    assert db.nack_messages("b", [ids[2]]) == 1
    assert db.extend_leases("b", [ids[3]], visibility_timeout=3600.0) == 1
    assert [m.id for m in db.receive_messages_leased("b", 10, visibility_timeout=60.0)] == [ids[2]]
    assert db.mark_message_as_processed(ids[2]) and db.mark_message_as_processed(bid)   # b's and c's leases of bid
    st = db.get_stats()["leases"]
    assert st["live"] == 2 and st["acked_total"] == 5
    assert db.redeliver_expired(all=True) == 2
    assert [m.id for m in db.receive_messages("b", 10)] == [ids[3], ids[4]]
    assert db.get_stats()["leases"]["live"] == 0 and db.receive_messages("c", 10) == []
    db.close()


def test_lease_kernel_time_is_read_past_the_abi1_slots():
    """sdb_profile_read writes SDB_PK_N = 16 entries and no more; the lease class (16) comes through sdb_profile_read_n."""
    import ctypes as C
    rig = _rig(11)
    g = rig.g
    g.lease_reserve(BIG, BIG * 256)
    g.profile(True)
    g.receive_leased(None, 4, 1.0)
    ms, cnt = np.full(17, -1.0), np.full(17, 7, np.uint64)           # entry 16 is a sentinel
    assert g._L.sdb_profile_read(g._h, ms.ctypes.data_as(C.c_void_p), cnt.ctypes.data_as(C.c_void_p)) == 0
    assert ms[16] == -1.0 and cnt[16] == 7
    assert cnt[12] >= 1                                              # the receive's compact class (12) is reported
    g.profile(True)
    g.receive_leased(None, 4, 1.0)
    prof = g.profile_read()
    assert prof["lease"][1] == 1 and prof["lease"][0] > 0 and prof["recv_compact"][1] >= 1
    g.profile(False)
    rig.close()
