"""Bounded queues on the device (sdb_trim) against tests/trim_ref.py, byte for byte.

Trimmed records are returned (archive mode) in the compact receive format; expanded they must equal the model's trim:
counts, every header field and the padded payload bytes.  Afterwards every receive path must deliver what the oracle
delivers after the same trim, i.e. what it would have delivered had the trimmed records never been enqueued.
"""
import math

import numpy as np
import pytest

from tests.budget_ref import agent_take
from tests.ring_ref import RingModel
from tests.test_gpu_compact_receive import Rig, _check_format, _same
from tests.test_gpu_expire import _loads_equal, _sends_with_ts
from tests.test_gpu_shared_layout import _payloads
from tests.trim_ref import TrimmingOracle

pytestmark = pytest.mark.gpu

CAPS = [(3, 0), (0, 300), (4, 500)]            # (max_records, max_agent_bytes): by count, by bytes, by both


def _rig(rng, **kw):
    rig = Rig(rng, **kw)
    rig.check_advance = False
    rig.c = TrimmingOracle(rig.c, rig.G, dict(enumerate(rig.members)), rig.A)
    return rig


def _trim_all_calls(g, agents, n, b, flags=0, shared=True, **kw):
    """Archive-mode calls until nothing comes back; (summed counts, expanded headers, payload, calls)."""
    from swarmdb_b200._native import HDR_DTYPE
    total_cnt, hdrs, pays, calls = None, [], [], 0
    while True:
        cnt, hdr, pay = _check_format(g.trim(agents, n, b, flags, **kw), shared)
        calls += 1
        total_cnt = cnt.astype(np.int64) if total_cnt is None else total_cnt + cnt
        if len(hdr) == 0:
            break
        hdrs.append(hdr); pays.append(pay)
    hdr = np.concatenate(hdrs) if hdrs else np.zeros(0, HDR_DTYPE)
    pay = np.concatenate(pays) if pays else np.zeros(0, np.uint8)
    return total_cnt.astype(np.uint32), hdr, pay, calls


def _every_path(rig, shared, what):
    """Stream, priority, few-agent, compact, budget and filtered receives, then a digest drain, against the oracle."""
    from swarmdb_b200._native import RECV_PEEK, RECV_PRIORITY, make_filter
    rng = rig.rng
    sel = rng.choice(rig.A, 300, replace=False).astype(np.uint32)
    _same(rig.g.receive_batch(sel[:100], 2, RECV_PRIORITY), rig.c.receive_batch(sel[:100], 2, RECV_PRIORITY), what + " priority")
    _same(rig.g.receive_batch(sel[100:200], 2), rig.c.receive_batch(sel[100:200], 2), what + " stream")
    for flags in (0, RECV_PRIORITY):
        _same(rig.g.receive_batch(sel[200:208], 1, flags), rig.c.receive_batch(sel[200:208], 1, flags), what + " <= 8 agents")
    _same(_check_format(rig.g.receive_compact(sel[208:260], 2), shared),
          rig.c.receive_batch(sel[208:260], 2, 0, rec_cap=1 << 21), what + " compact")
    for a in sel[260:280].tolist():                # byte budget: the model's take of the oracle's pending lengths
        _, hdr, _ = rig.c.receive_batch([a], 1000, RECV_PEEK)
        k = max(agent_take([int(x) for x in hdr["len"]], 1000, 600), 1)
        _same(rig.g.receive_budget([a], 1000, 600), rig.c.receive_batch([a], k), what + " budget")
    f = make_filter(prios=[2, 3])
    got = rig.g.receive_where(sel[280:], 3, 0, f)
    _same(got, rig.c.receive_where(sel[280:], 3, 0, f), what + " filtered")
    _loads_equal(rig, what + " loads")
    rig.g.digest_reset(); rig.c.digest_enable()
    while True:
        _, total, _ = rig.g.receive_batch(None, 64, copy_out=False)
        rig.g.digest_fold()
        rig.c.receive_counts(None, 64)
        if total == 0:
            break
    assert np.array_equal(rig.g.digest_read(), rig.c.digest_read()), what


@pytest.mark.parametrize("shared", ["1", "0"])
@pytest.mark.parametrize("prio", [False, True])
def test_trim_matches_the_model_then_every_receive_path(shared, prio, monkeypatch):
    from swarmdb_b200._native import RECV_PEEK, RECV_PRIORITY, make_filter
    monkeypatch.setenv("SDB_SHARED_PAYLOAD", shared)
    rng = np.random.default_rng(61 + prio)
    rig = _rig(rng, G=8, F=64, extra=64)
    _sends_with_ts(rig)
    # holes in the windows: a priority receive and a filtered take
    some = rng.choice(rig.A, 120, replace=False).astype(np.uint32)
    _same(rig.g.receive_batch(some[:60], 2, RECV_PRIORITY), rig.c.receive_batch(some[:60], 2, RECV_PRIORITY), "holes")
    f = make_filter(prios=[1])
    _same(rig.g.receive_where(some[60:], 1, 0, f), rig.c.receive_where(some[60:], 1, 0, f), "filtered holes")
    flags = RECV_PRIORITY if prio else 0
    st0 = rig.g.stats()
    perm = rng.permutation(rig.A).astype(np.uint32)
    parts = np.array_split(perm, len(CAPS) + 1)
    for (n, b), agents in zip(CAPS, parts):
        p1 = _check_format(rig.g.trim(agents, n, b, flags | RECV_PEEK), shared == "1")
        p2 = _check_format(rig.g.trim(agents, n, b, flags | RECV_PEEK), shared == "1")
        _same(p1, p2, "peek twice")
        _loads_equal(rig, "after peek")
        want = rig.c.trim(agents, n, b, flags)
        assert len(want[1]) > 0
        _same(p1, want, f"peek vs model {n} {b}")
        got = _trim_all_calls(rig.g, agents, n, b, flags, shared=shared == "1")
        _same(got[:3], want, f"trimmed set {n} {b}")
        _loads_equal(rig, f"after trim {n} {b}")
        ld = rig.g.agent_loads(agents)
        assert (n == 0 or ld["pending"].max() <= n) and (b == 0 or ld["pending_granules"].max() * 32 <= b)
        assert rig.g.trim(agents, n, b, flags, archive=False)[1] == 0          # within the caps: nothing more
    # drop mode on the last part
    cnt, total = rig.g.trim(parts[-1], 2, 200, flags, archive=False)
    cc, tc = rig.c.trim(parts[-1], 2, 200, flags, materialise=False)
    assert total == tc > 0 and np.array_equal(cnt, cc)
    st1 = rig.g.stats()
    assert {k: st1[k] for k in ("enqueued", "delivered")} == {k: st0[k] for k in ("enqueued", "delivered")}
    _every_path(rig, shared == "1", "after trim")
    rig.close()


def test_trim_capacity_partial_first_agent_and_caller_caps():
    from swarmdb_b200._native import ENTRY_DTYPE, RECV_PEEK, RECV_PRIORITY, SEND_DTYPE, SdbError
    rng = np.random.default_rng(7)
    rig = _rig(rng, G=4, F=64, extra=64, max_recv_records=64)
    _sends_with_ts(rig, 1)
    n = 300                                      # agent 7: far more than 64 records over the cap
    s, prio = rng.integers(0, rig.A, n), rng.integers(0, 4, n)
    lens, off, buf = _payloads(rng, n, 100)
    r = np.full(n, 7)
    rig.c.send_batch(s, r, prio, None, lens, off, buf); rig.g.send_batch(s, r, prio, None, lens, off, buf)
    agents = np.concatenate([[7], rng.permutation(np.setdiff1d(rig.idx, [7]))]).astype(np.uint32)
    for flags in (0, RECV_PRIORITY):
        # the first call: agent 7 alone, the first 64 records of its eviction order
        c1 = _check_format(rig.g.trim(agents, 2, 0, flags | RECV_PEEK))
        assert c1[0][0] == 64 and int(c1[0][1:].sum()) == 0
        _same(c1, rig.c.trim(agents, 2, 0, flags | RECV_PEEK, rec_cap=64), "partial first agent")
    # repeated calls with a caller cap of 10 entries give what one drop call gives: the same digests after
    twin = Rig(np.random.default_rng(7), G=4, F=64, extra=64, max_recv_records=64)
    twin.check_advance = False
    _sends_with_ts(twin, 1)
    twin.g.send_batch(s, r, prio, None, lens, off, buf)
    want = rig.c.trim(agents, 2, 300, RECV_PRIORITY, materialise=False)
    ent, snd = np.zeros(10, ENTRY_DTYPE), np.zeros(10, SEND_DTYPE)
    got = _trim_all_calls(rig.g, agents, 2, 300, RECV_PRIORITY, out_entries=ent, out_sends=snd)
    assert got[3] > 30 and np.array_equal(got[0], want[0])
    assert twin.g.trim(agents, 2, 300, RECV_PRIORITY, archive=False)[1] == want[1]
    _loads_equal(rig, "after capped trim")
    for x in (rig.g, twin.g):
        x.digest_reset()
        while x.receive_batch(None, 1000, copy_out=False)[1]:
            x.digest_fold()
    assert np.array_equal(rig.g.digest_read(), twin.g.digest_read())
    twin.close()
    # argument checks
    with pytest.raises(SdbError) as e:
        rig.g.trim(agents, 2, 0, out_entries=np.zeros(0, ENTRY_DTYPE), out_sends=np.zeros(0, SEND_DTYPE))
    assert e.value.code == -8
    for bad_flags in (4, 16, 32):
        with pytest.raises(SdbError) as e:
            rig.g.trim(agents, 2, 0, bad_flags)
        assert e.value.code == -1
    with pytest.raises(SdbError) as e:
        rig.g.trim(agents, 0, 0, archive=False)
    assert e.value.code == -1
    for bad in ([1, 2, 1], [rig.A]):
        with pytest.raises(SdbError) as e:
            rig.g.trim(np.array(bad, np.uint32), 2, 0, archive=False)
        assert e.value.code == -1
    rig.close()


def test_trim_frees_exactly_the_ring_room_the_model_predicts():
    from swarmdb_b200._native import RECV_PRIORITY, Shard
    R = 16
    g = Shard(max_agents=4, ring_slots=R, arena_bytes=1 << 20, max_payload_bytes=64)
    g.register(np.arange(4, dtype=np.uint32))
    m = RingModel(R)
    lens, off, buf = np.full(R, 40, np.uint16), np.arange(R, dtype=np.uint64) * 64, np.full(R * 64 + 64, 7, np.uint8)
    prio = np.array([0, 1, 2, 0, 3, 1, 0, 2, 1, 0, 3, 0, 1, 2, 0, 1], np.uint8)
    base = g.send_batch(np.ones(R), np.zeros(R), prio, None, lens, off, buf)
    m.append(0, range(base, base + R))
    hdr = g.receive_batch([0], 2, RECV_PRIORITY)[1]                 # the two level-3 records: holes at 4 and 10
    m.retire(0, hdr["seq"])
    assert g.trim([0], 3, 0, archive=False)[1] == R - 2 - 3
    pend = g.receive_batch([0], 100, 2)[1]["seq"]                   # PEEK
    m.retire_to(0, pend)
    room = m.capacity(0)
    assert room == 13                                                # head at position 13: the oldest record kept
    ovf = g.stats()["ring_overflow"]
    g.send_batch(np.ones(room), np.zeros(room), None, None, lens[:room], off[:room], buf)
    assert g.stats()["ring_overflow"] == ovf
    g.send_batch(np.ones(1), np.zeros(1), None, None, lens[:1], off[:1], buf)
    assert g.stats()["ring_overflow"] == ovf + 1
    g.close()


def test_idle_agent_pinning_the_arena_is_unpinned_by_a_cap():
    from swarmdb_b200._native import SdbError, Shard
    A = 64
    g = Shard(max_agents=A, ring_slots=4096, arena_bytes=1 << 20, max_payload_bytes=256)
    g.register(np.arange(A, dtype=np.uint32))
    lens, off = np.full(64, 200, np.uint16), np.arange(64, dtype=np.uint64) * 256
    buf = np.full(64 * 256 + 64, 65, np.uint8)
    g.send_batch([1, 1], [0, 0], None, None, lens[:2], off[:2], buf)           # agent 0 never receives
    with pytest.raises(SdbError) as e:
        for _ in range(10000):
            g.send_batch(np.ones(64), np.full(64, 5), None, None, lens, off, buf)
            assert len(g.receive_batch([5], 1000)[1]) == 64
    assert e.value.code == -5
    floor0 = g.stats()["arena_floor_bytes"]
    assert g.trim(None, 1, 0, archive=False)[1] == 1                # the older record of agent 0 goes
    assert g.trim(None, 0, 100, archive=False)[1] == 1              # 200 B > 100 B on its own: it goes too
    assert g.stats()["arena_floor_bytes"] == floor0
    g.send_batch(np.ones(64), np.full(64, 5), None, None, lens, off, buf)
    assert g.stats()["arena_floor_bytes"] > floor0
    assert len(g.receive_batch([5], 1000)[1]) == 64 and g.queue_stats()["pending"] == 0
    g.close()


def test_trim_near_the_handle_wrap():
    from oracle.cpu_ref import CpuOracle
    from swarmdb_b200._native import RECV_PRIORITY, Shard
    A = 256
    rng = np.random.default_rng(3)
    g, c = Shard(max_agents=A, ring_slots=256, arena_bytes=1 << 22, max_payload_bytes=256), CpuOracle(A, 1)
    g.register(np.arange(A, dtype=np.uint32)); c.register(np.arange(A))
    c = TrimmingOracle(c, 1, watermark=A)
    g.debug_set_arena_pos((1 << 32) - 300)
    for _ in range(6):
        n = 200
        s, r, prio = rng.integers(0, A, n), rng.integers(0, A, n), rng.integers(0, 4, n)
        lens, off, buf = _payloads(rng, n, 200)
        c.send_batch(s, r, prio, None, lens, off, buf); g.send_batch(s, r, prio, None, lens, off, buf)
    assert g.stats()["arena_tail_bytes"] > (1 << 32) * 32
    want = c.trim(None, 2, 200, RECV_PRIORITY)
    got = _trim_all_calls(g, None, 2, 200, RECV_PRIORITY)
    _same(got[:3], want, "handle wrap")
    _same(g.receive_batch(None, 1000), c.receive_batch(None, 1000), "drain")
    g.close(); c.close()


def test_leases_are_neither_counted_nor_touched_and_a_trimmed_redelivery_keeps_no_count():
    from swarmdb_b200._native import LEASE_RENEW, Shard
    g = Shard(max_agents=8, ring_slots=64, arena_bytes=1 << 22, max_payload_bytes=64)
    g.register(np.arange(8, dtype=np.uint32))
    g.lease_reserve(256, 256 * 64)
    g.lease_set_policy(10, 256)
    lens, off, buf = np.full(6, 40, np.uint16), np.arange(6, dtype=np.uint64) * 64, np.arange(6 * 64 + 64, dtype=np.uint8)
    g.send_batch(np.ones(6), np.zeros(6), None, None, lens, off, buf)
    _, ent, _, _, lb = g.receive_leased([0], 4, 10.0)                # 4 in flight, 2 pending
    ids = np.arange(lb, lb + len(ent), dtype=np.uint64)
    assert g.trim([0], 2, 0, archive=False)[1] == 0                  # leases are not counted
    assert g.trim([0], 1, 0, archive=False)[1] == 1
    assert g.lease_stats()["live"] == 4 and g.agent_loads([0])["pending"][0] == 1
    g.lease_settle(ids, LEASE_RENEW, -math.inf)
    assert g.lease_sweep(0.0)[0] == 4                                 # redelivered: 5 pending, 4 of them counted once
    cnt, ent, snd, pay = (x.copy() for x in g.trim([0], 2, 0))       # the 3 oldest go, redelivered ones among them
    assert cnt[0] == 3
    assert g.restore_compact([0], cnt, ent, snd, pay)[0] == 3        # requeued with the same seqs
    _, ent2, _, _, lb2 = g.receive_leased([0], 100, 10.0)
    d = dict(zip(ent2["seq"].tolist(), g.lease_deliveries(np.arange(lb2, lb2 + len(ent2), dtype=np.uint64)).tolist()))
    assert all(d[s] == 1 for s in ent["seq"].tolist())               # a trimmed record passes on no count
    assert sorted(v for s, v in d.items() if s not in set(ent["seq"].tolist())) == [2, 2]
    g.close()


def test_sharded_handle_owned_agents():
    from oracle.cpu_ref import CpuOracle
    from swarmdb_b200._native import RECV_OWNED, RECV_PRIORITY
    from tests.test_gpu_xshard import _async_cluster
    rng = np.random.default_rng(19)
    A, G, F, S = 2048, 32, 64, 300
    perm = rng.permutation(A)
    groups = [perm[k * F:(k + 1) * F] for k in range(G)]
    smap, shards, wb, bufs = _async_cluster(1, A, G, S, groups)
    s = shards[0]
    s.register(np.arange(A, dtype=np.uint32))
    o = CpuOracle(A, G)
    for k, m in enumerate(groups):
        o.create_group(k, m)
    o.register(np.arange(A))
    o = TrimmingOracle(o, G, dict(enumerate(groups)), A)
    for step in (1, 2):
        sender, grp, prio = rng.integers(0, A, S), rng.integers(0, G, S), rng.integers(0, 4, S)
        lens, off, buf = _payloads(rng, S, 256)
        ts = rng.uniform(0, 10, S)                   # distinct per send: _check_format tells the sends apart by it
        s.export_group_batch(sender, grp, prio, None, lens, off, buf, bufs[step & 1][0], wb, ts)
        s.wire_publish(bufs[step & 1][0], wb, step)
        s.import_wire_ptrs_async(bufs[step & 1], wb, step)
        o.send_group_batch(sender, grp, prio, None, lens, off, buf, ts)
    cnt, total = s.trim(None, 4, 0, RECV_OWNED, archive=False)
    cc, tc = o.trim(None, 4, 0, materialise=False)
    assert total == tc > 0 and len(cnt) == A and np.array_equal(cnt, cc[:A])
    got = _trim_all_calls(s, None, 2, 300, RECV_OWNED | RECV_PRIORITY)
    want = o.trim(None, 2, 300, RECV_PRIORITY)
    _same(got[:3], (want[0][:A],) + want[1:], "owned archive")
    _same(s.receive_batch(np.arange(A, dtype=np.uint32), 1000), o.receive_batch(np.arange(A), 1000), "drain")
    s.close(); o.close()


def _survivors(grp, sizes, prio, G, cap_n, cap_b, by_prio):
    """Per send of a c2 batch, whether it survives the trim: every member of a group holds the same records."""
    keep = np.ones(len(grp), bool)
    order = np.argsort(grp, kind="stable")
    bounds = np.searchsorted(grp[order], np.arange(G + 1))
    for k in range(G):
        idx = order[bounds[k]:bounds[k + 1]]
        if by_prio:
            idx = idx[np.argsort(prio[idx], kind="stable")]
        n_left, b_left = len(idx), int(sizes[idx].sum())
        for i in idx:
            if (not cap_n or n_left <= cap_n) and (not cap_b or b_left <= cap_b):
                break
            keep[i] = False
            n_left -= 1
            b_left -= int(sizes[i])
    return keep


@pytest.mark.parametrize("cap", ["count2", "bytes512_priority"])
def test_c2_backlog_drop_mode_matches_oracle_digests(cap):
    """The 1M-agent c2 backlog (65,536 group sends x 64 = 4,194,304 pending records), one drop-mode trim, then the full
    drain's digests and the queue statistics against an oracle that was only ever sent the surviving sends."""
    from bench import Workload
    from oracle.cpu_ref import CpuOracle
    from swarmdb_b200._native import RECV_PRIORITY, Shard
    wl = Workload()
    g = Shard(max_agents=wl.A, ring_slots=64, arena_bytes=1 << 31, max_payload_bytes=wl.L, max_groups=wl.G,
              member_pool_entries=wl.A + 1024, max_batch_sends=wl.S, max_batch_payload=wl.S * wl.L,
              max_recv_records=1 << 23, max_recv_payload=(1 << 23) * wl.L)
    surv = CpuOracle(wl.A, wl.G)
    g.register(np.arange(wl.A, dtype=np.uint32))
    surv.register(np.arange(wl.A))
    for k in range(wl.G):
        g.create_group(k, wl.members(k)); surv.create_group(k, wl.members(k))
    b = wl.batch(var_len=cap != "count2")
    sender, grp, prio, typ, lens, off, pay = b
    base = g.send_group_batch(*b)
    n, nb, flags = (2, 0, 0) if cap == "count2" else (0, 512, RECV_PRIORITY)
    keep = _survivors(grp, (lens.astype(np.int64) + 31) & ~31, prio, wl.G, n, nb, flags != 0)
    assert 0 < keep.sum() < wl.S
    surv.send_group_seq(sender[keep], grp[keep], prio[keep], typ[keep], lens[keep], off[keep], pay,
                        base + wl.F * np.nonzero(keep)[0].astype(np.uint64))
    cnt, total = g.trim(None, n, nb, flags, archive=False)
    assert total == wl.F * int((~keep).sum())
    qg, qs = g.queue_stats(), surv.queue_stats(wl.A)
    assert {k: qg[k] for k in ("pending", "pending_by_prio", "pending_granules", "agents_with_pending")} == \
        {k: qs[k] for k in ("pending", "pending_by_prio", "pending_granules", "agents_with_pending")}
    g.digest_reset(); surv.digest_enable()
    _, tot, _ = g.receive_batch(None, 100, copy_out=False)
    g.digest_fold()
    surv.receive_counts(None, 100)
    assert tot == wl.S * wl.F - total
    assert np.array_equal(g.digest_read(), surv.digest_read())
    g.close(); surv.close()


def _db(tmp_path, **kw):
    import swarmdb_b200 as sdb
    return sdb.SwarmsDB(save_dir=str(tmp_path), auto_save=False,
                        gpu_config=sdb.GpuConfig(max_agents=64, ring_slots=64, arena_bytes=1 << 22, max_payload_bytes=1024,
                                                 deterministic_ids=True, **kw))


def test_swarmsdb_automatic_caps_keep_the_newest(tmp_path):
    from swarmdb_b200 import MessagePriority
    db = _db(tmp_path, queue_max_messages=3)
    db.register_agent("a"); db.register_agent("b")
    for i in range(10):
        db.send_message("a", f"m{i}", receiver_id="b")
    db.flush()
    assert db.get_stats()["trimmed"] == 7
    assert [m.content for m in db.receive_messages("b")] == ["m7", "m8", "m9"]
    for i in range(5):                               # two flushes of 2 and 3: only what goes over the cap is dropped
        db.send_message("a", f"n{i}", receiver_id="b")
        if i in (1, 4):
            db.flush()
    assert db.get_stats()["trimmed"] == 9
    assert [m.content for m in db.receive_messages("b")] == ["n2", "n3", "n4"]
    db.close()
    db = _db(tmp_path, queue_max_messages=3, queue_trim_priority=True)
    db.register_agent("a"); db.register_agent("b")
    prios = [MessagePriority.CRITICAL, MessagePriority.LOW, MessagePriority.NORMAL, MessagePriority.CRITICAL,
             MessagePriority.HIGH, MessagePriority.LOW, MessagePriority.NORMAL, MessagePriority.HIGH,
             MessagePriority.LOW, MessagePriority.NORMAL]
    for i, p in enumerate(prios):
        db.send_message("a", f"m{i}", receiver_id="b", priority=p)
    db.flush()
    assert db.get_stats()["trimmed"] == 7
    assert sorted(m.content for m in db.receive_messages("b")) == ["m0", "m3", "m7"]     # both CRITICAL and the newest HIGH
    assert db.trim_queues(max_messages=1) == 0
    db.close()
    db = _db(tmp_path)
    assert "trimmed" not in db.get_stats()
    db.register_agent("a"); db.register_agent("b")
    for i in range(10):
        db.send_message("a", f"m{i}", receiver_id="b", priority=MessagePriority.LOW if i % 2 else MessagePriority.HIGH)
    assert db.trim_queues(max_messages=4, agent_ids=["b", "nobody"], by_priority=True) == 6
    assert [m.content for m in db.receive_messages("b")] == ["m2", "m4", "m6", "m8"]
    db.close()
