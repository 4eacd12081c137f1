"""Retention on the device (sdb_expire) against the CPU oracle, byte for byte.

The oracle side of an expiry is tests/expire_ref.py: the survivors are replayed into a fresh oracle that never saw the
expired records.

Expired records are returned (archive mode) in the compact receive format; expanded they must equal the oracle's
expiry: counts, every header field and the padded payload bytes.  Afterwards every receive path must deliver what the
oracle delivers after the same expiry, i.e. what it would have delivered had the expired records never been enqueued.
"""
import numpy as np
import pytest

from tests.expire_ref import ExpiringOracle
from tests.test_gpu_compact_receive import Rig, _check_format, _same
from tests.test_gpu_shared_layout import _payloads

pytestmark = pytest.mark.gpu


def _sends_with_ts(rig, rounds=2):
    """p2p, shared-layout group and broadcast sends, each with a non-monotonic uniform timestamp in [0, 10)."""
    rng = rig.rng
    for _ in range(rounds):
        n = 400
        s, r, prio = rng.integers(0, rig.A, n), rng.integers(0, rig.A, n), rng.integers(0, 4, n)
        lens, off, buf = _payloads(rng, n, 200)
        ts = rng.uniform(0, 10, n)
        base = rig.c.send_batch(s, r, prio, None, lens, off, buf, ts)
        assert rig.g.send_batch(s, r, prio, None, lens, off, buf, ts) == base
        n = 300
        s = rng.integers(rig.G * rig.F, rig.A, n)
        grp, prio = rng.integers(0, rig.G, n), rng.integers(0, 4, n)
        lens, off, buf = _payloads(rng, n, 256)
        ts = rng.uniform(0, 10, n)
        base = rig.c.send_group_batch(s, grp, prio, None, lens, off, buf, ts)[0]
        assert rig.g.send_group_batch(s, grp, prio, None, lens, off, buf, ts) == base
        n = 6
        lists = [rng.choice(rig.A, size=int(rng.integers(1, 200)), replace=False) for _ in range(n)]
        lo = np.zeros(n + 1, np.uint64); lo[1:] = np.cumsum([len(x) for x in lists])
        li = np.concatenate(lists).astype(np.uint32)
        s, prio = rng.integers(0, rig.A, n), rng.integers(0, 4, n)
        lens, off, buf = _payloads(rng, n, 200)
        ts = rng.uniform(0, 10, n)
        base = rig.c.send_list_batch(s, lo, li, prio, None, lens, off, buf, ts)
        assert rig.g.send_list_batch(s, lo, li, prio, None, lens, off, buf, ts) == base


def _expire_all_calls(g, agents, cutoff, flags=0, shared=True, **kw):
    """Archive-mode calls until nothing comes back; (summed counts, expanded headers, payload) of all of them."""
    total_cnt, hdrs, pays, calls = None, [], [], 0
    while True:
        cnt, hdr, pay = _check_format(g.expire(agents, cutoff, flags, **kw), shared)
        calls += 1
        total_cnt = cnt.astype(np.int64) if total_cnt is None else total_cnt + cnt
        if len(hdr) == 0:
            break
        hdrs.append(hdr); pays.append(pay)
    from swarmdb_b200._native import HDR_DTYPE
    hdr = np.concatenate(hdrs) if hdrs else np.zeros(0, HDR_DTYPE)
    pay = np.concatenate(pays) if pays else np.zeros(0, np.uint8)
    return total_cnt.astype(np.uint32), hdr, pay, calls


def _rig(rng, **kw):
    rig = Rig(rng, **kw)
    rig.check_advance = False
    rig.c = ExpiringOracle(rig.c, rig.G, dict(enumerate(rig.members)), rig.A)
    return rig


def _loads_equal(rig, what):
    lg, lc = rig.g.agent_loads(rig.idx), rig.c.agent_loads(rig.idx)
    for f in ("received", "pending", "pending_by_prio", "pending_granules"):
        assert np.array_equal(lg[f], lc[f]), (what, f)


@pytest.mark.parametrize("shared", ["1", "0"])
def test_expire_matches_oracle_then_every_receive_path(shared, monkeypatch):
    from swarmdb_b200._native import RECV_PEEK, RECV_PRIORITY
    monkeypatch.setenv("SDB_SHARED_PAYLOAD", shared)
    rng = np.random.default_rng(41)
    rig = _rig(rng, G=8, F=64, extra=64)
    _sends_with_ts(rig)
    # holes in the middle of windows: priority receives on some agents
    some = rng.choice(rig.A, 100, replace=False).astype(np.uint32)
    _same(rig.g.receive_batch(some, 3, RECV_PRIORITY), rig.c.receive_batch(some, 3, RECV_PRIORITY), "holes")
    st0 = rig.g.stats()
    agents = rng.permutation(rig.A)[: rig.A * 3 // 4].astype(np.uint32)
    # PEEK twice: the same answer, nothing retired
    p1 = _check_format(rig.g.expire(agents, 5.0, RECV_PEEK), shared == "1")
    p2 = _check_format(rig.g.expire(agents, 5.0, RECV_PEEK), shared == "1")
    _same(p1, p2, "peek twice")
    _loads_equal(rig, "after peek")
    want = rig.c.expire(agents, 5.0)
    _same(p1, want, "peek vs oracle expiry")
    got = _expire_all_calls(rig.g, agents, 5.0, shared=shared == "1")
    _same(got[:3], want, "expired set")
    st1 = rig.g.stats()
    assert {k: st1[k] for k in ("enqueued", "delivered")} == {k: st0[k] for k in ("enqueued", "delivered")}
    assert st1["arena_floor_bytes"] == st0["arena_floor_bytes"]
    _loads_equal(rig, "after expire")
    # drop mode on the rest of the agents, at a different cutoff
    rest = np.setdiff1d(rig.idx, agents).astype(np.uint32)
    cnt, total = rig.g.expire(rest, 3.0, archive=False)
    cc, tc = rig.c.expire(rest, 3.0, materialise=False)
    assert total == tc and np.array_equal(cnt, cc)
    _loads_equal(rig, "after drop")
    # every receive path delivers what the oracle delivers after the same expiry
    sel = rng.choice(rig.A, 300, replace=False).astype(np.uint32)
    _same(rig.g.receive_batch(sel, 2, RECV_PRIORITY), rig.c.receive_batch(sel, 2, RECV_PRIORITY), "priority pipeline")
    _same(rig.g.receive_batch(sel, 2), rig.c.receive_batch(sel, 2), "stream plan")
    eight = sel[:8]
    for flags in (0, RECV_PRIORITY):
        _same(rig.g.receive_batch(eight, 3, flags), rig.c.receive_batch(eight, 3, flags), "<= 8 agents")
    rig.g.latency_server(True)
    for a in sel[8:20]:
        for flags in (0, RECV_PRIORITY):
            h, p, _ = rig.g.receive_one(int(a), 2, flags)
            _, hc, pc = rig.c.receive_batch([a], 2, flags)
            assert h.tobytes() == hc.tobytes() and p.tobytes() == pc.tobytes(), ("latency server", a)
    # an expire while the server runs, then the server still answers
    cnt, total = rig.g.expire(sel[20:40], 7.0, archive=False)
    assert total == rig.c.expire(sel[20:40], 7.0, materialise=False)[1]
    h, p, _ = rig.g.receive_one(int(sel[20]), 5)
    _, hc, pc = rig.c.receive_batch([sel[20]], 5)
    assert h.tobytes() == hc.tobytes() and p.tobytes() == pc.tobytes()
    rig.g.latency_server(False)
    _same(_check_format(rig.g.receive_compact(None, 2), shared == "1"), rig.c.receive_batch(rig.idx, 2, 0, rec_cap=1 << 21),
          "compact")
    # full drain through the digests
    rig.g.digest_reset(); rig.c.digest_enable()
    while True:
        _, total, _ = rig.g.receive_batch(None, 64, copy_out=False)
        rig.g.digest_fold()
        rig.c.receive_counts(None, 64)
        if total == 0:
            break
    assert np.array_equal(rig.g.digest_read(), rig.c.digest_read())
    assert rig.g.queue_stats()["pending"] == 0 == rig.c.queue_stats()["pending"]
    rig.close()


def test_expire_capacity_partial_first_agent_and_caller_caps():
    from swarmdb_b200._native import ENTRY_DTYPE, EXPIRE_ALL, RECV_PEEK, SEND_DTYPE, SdbError
    rng = np.random.default_rng(5)
    rig = _rig(rng, G=4, F=64, extra=64, max_recv_records=64)
    _sends_with_ts(rig, 1)
    # one agent with far more than 64 matches: the partial first agent
    n = 300
    s, prio = rng.integers(0, rig.A, n), rng.integers(0, 4, n)
    lens, off, buf = _payloads(rng, n, 100)
    ts = rng.uniform(0, 10, n)
    r = np.full(n, 7)
    rig.c.send_batch(s, r, prio, None, lens, off, buf, ts); rig.g.send_batch(s, r, prio, None, lens, off, buf, ts)
    agents = np.concatenate([[7], rng.permutation(np.setdiff1d(rig.idx, [7]))]).astype(np.uint32)
    want_all = rig.c.expire(agents, 6.0, RECV_PEEK)
    # first call: agent 7 alone, its first 64 matches
    c1 = _check_format(rig.g.expire(agents, 6.0, RECV_PEEK))
    assert c1[0][0] == 64 and int(c1[0][1:].sum()) == 0
    # the whole set through repeated calls, with a caller cap of 10 entries
    ent, snd = np.zeros(10, ENTRY_DTYPE), np.zeros(10, SEND_DTYPE)
    got = _expire_all_calls(rig.g, agents, 6.0, out_entries=ent, out_sends=snd)
    assert got[3] > 30
    _same(got[:3], want_all, "repeated capped calls")
    rig.c.expire(agents, 6.0)
    _loads_equal(rig, "after capped expiry")
    with pytest.raises(SdbError) as e:
        rig.g.expire(agents, 6.0, out_entries=np.zeros(0, ENTRY_DTYPE), out_sends=np.zeros(0, SEND_DTYPE))
    assert e.value.code == -8
    for bad_flags in (1, 4, 32):
        with pytest.raises(SdbError) as e:
            rig.g.expire(agents, 6.0, bad_flags)
        assert e.value.code == -1
    for bad in ([1, 2, 1], [rig.A]):
        with pytest.raises(SdbError) as e:
            rig.g.expire(np.array(bad, np.uint32), 6.0, archive=False)
        assert e.value.code == -1
    # purge: everything of the listed agents, timestamps not read
    cnt, total = rig.g.expire(agents[:50], 0.0, EXPIRE_ALL, archive=False)
    cc, tc = rig.c.expire(agents[:50], 0.0, EXPIRE_ALL, materialise=False)
    assert total == tc and np.array_equal(cnt, cc)
    _loads_equal(rig, "after purge")
    for k in range(0, 64, 8):                  # max_recv_records = 64: eight agents x 5 records per call always fit
        _same(rig.g.receive_batch(agents[k:k + 8], 5), rig.c.receive_batch(agents[k:k + 8], 5), "after purge")
    rig.close()


@pytest.mark.parametrize("how", ["expire", "purge"])
def test_idle_agent_pins_the_arena_until_expired(how):
    from swarmdb_b200._native import EXPIRE_ALL, SdbError, Shard
    A = 64
    g = Shard(max_agents=A, ring_slots=4096, arena_bytes=1 << 20, max_payload_bytes=256)
    g.register(np.arange(A, dtype=np.uint32))
    lens, off = np.full(64, 200, np.uint16), np.arange(64, dtype=np.uint64) * 256
    buf = np.full(64 * 256 + 64, 65, np.uint8)
    g.send_batch([1], [0], None, None, lens[:1], off[:1], buf, np.array([1.0]))           # agent 0 never receives
    t = 2.0
    with pytest.raises(SdbError) as e:
        for _ in range(10000):
            g.send_batch(np.ones(64), np.full(64, 5), None, None, lens, off, buf, np.full(64, t))
            assert len(g.receive_batch([5, 6, 7, 8, 9, 10, 11, 12, 13], 1000)[1]) == 64
            t += 1.0
    assert e.value.code == -5
    floor0 = g.stats()["arena_floor_bytes"]
    if how == "expire":
        assert g.expire(None, 1.5, archive=False)[1] == 1
    else:
        assert g.expire([0], 0.0, EXPIRE_ALL, archive=False)[1] == 1
    assert g.stats()["arena_floor_bytes"] == floor0                   # the call itself does not move the floor
    g.send_batch(np.ones(64), np.full(64, 5), None, None, lens, off, buf, np.full(64, t))
    assert g.stats()["arena_floor_bytes"] > floor0
    assert len(g.receive_batch([5], 1000)[1]) == 64 and g.queue_stats()["pending"] == 0
    g.close()


def test_partially_expired_group_send_keeps_its_shared_payload_through_arena_wraps():
    from swarmdb_b200._native import EXPIRE_ALL
    rng = np.random.default_rng(8)
    rig = _rig(rng, G=8, F=64, extra=64, arena_bytes=1 << 21, max_payload_bytes=256)
    ex = np.arange(rig.G * rig.F, rig.A)

    def pump(to_bytes):
        while rig.g.stats()["arena_tail_bytes"] < to_bytes:
            s, r = rng.choice(ex, 64), rng.choice(ex, 64)
            lens, off, buf = _payloads(rng, 64, 256)
            rig.c.send_batch(s, r, None, None, lens, off, buf); rig.g.send_batch(s, r, None, None, lens, off, buf)
            _same(rig.g.receive_batch(ex.astype(np.uint32), 1000), rig.c.receive_batch(ex.astype(np.uint32), 1000), "pump")
    pump(1100 << 10)                                                    # the group batch (~0.7 MB) lands near the end
    rig.shared_batch(300)
    half = np.concatenate([m[:32] for m in rig.members]).astype(np.uint32)
    cnt, total = rig.g.expire(half, 0.0, EXPIRE_ALL, archive=False)
    assert total == rig.c.expire(half, 0.0, EXPIRE_ALL, materialise=False)[1] > 0
    pump((1 << 21) + (300 << 10))                                       # the write position wraps round below the pinned batch
    keep = np.concatenate([m[32:] for m in rig.members]).astype(np.uint32)
    _same(rig.g.receive_batch(keep, 1000), rig.c.receive_batch(keep, 1000), "remaining members")
    rig.close()


def test_expire_near_the_handle_wrap():
    from swarmdb_b200._native import Shard
    from oracle.cpu_ref import CpuOracle
    A = 256
    rng = np.random.default_rng(3)
    g, c = Shard(max_agents=A, ring_slots=256, arena_bytes=1 << 22, max_payload_bytes=256), CpuOracle(A, 1)
    g.register(np.arange(A, dtype=np.uint32)); c.register(np.arange(A))
    c = ExpiringOracle(c, 1, watermark=A)
    g.debug_set_arena_pos((1 << 32) - 300)
    for _ in range(6):
        n = 200
        s, r = rng.integers(0, A, n), rng.integers(0, A, n)
        lens, off, buf = _payloads(rng, n, 200)
        ts = rng.uniform(0, 10, n)
        c.send_batch(s, r, None, None, lens, off, buf, ts); g.send_batch(s, r, None, None, lens, off, buf, ts)
    assert g.stats()["arena_tail_bytes"] > (1 << 32) * 32
    want = c.expire(None, 5.0)
    got = _expire_all_calls(g, None, 5.0)
    _same(got[:3], want, "handle wrap")
    _same(g.receive_batch(None, 1000), c.receive_batch(None, 1000), "drain")
    g.close(); c.close()


def test_sharded_handle_owned_agents_and_async_import_ordering():
    """A sharded handle (one GPU, loopback) with SDB_RECV_OWNED; expire right after import_wire_ptrs_async and between
    import_prefetch(step) and its import."""
    from oracle.cpu_ref import CpuOracle
    from swarmdb_b200._native import RECV_OWNED
    from tests.test_gpu_xshard import _async_cluster
    rng = np.random.default_rng(17)
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
    o = ExpiringOracle(o, G, dict(enumerate(groups)), A)

    def export(step):
        sender, grp = rng.integers(0, A, S), rng.integers(0, G, S)
        lens, off, buf = _payloads(rng, S, 256)
        ts = rng.uniform(0, 10, S)
        s.export_group_batch(sender, grp, None, None, lens, off, buf, bufs[step & 1][0], wb, ts)
        s.wire_publish(bufs[step & 1][0], wb, step)
        return lambda: o.send_group_batch(sender, grp, None, None, lens, off, buf, ts)    # the oracle's copy, when imported

    export(1)()
    s.import_wire_ptrs_async(bufs[1], wb, 1)
    cnt, total = s.expire(None, 3.0, RECV_OWNED, archive=False)            # right after the asynchronous import
    cc, tc = o.expire(None, 3.0, materialise=False)
    assert total == tc > 0 and len(cnt) == A and np.array_equal(cnt, cc[:A])
    oracle_send = export(2)
    s.import_prefetch(bufs[0], wb, 2)
    cnt, total = s.expire(None, 6.0, RECV_OWNED, archive=False)            # between the prefetch and its import
    assert total == o.expire(None, 6.0, materialise=False)[1] > 0
    s.import_wire_ptrs_async(bufs[0], wb, 2)
    oracle_send()
    got = _expire_all_calls(s, None, 8.0, RECV_OWNED)
    want = o.expire(None, 8.0)
    _same(got[:3], (want[0][:A],) + want[1:], "owned archive")
    _same(s.receive_batch(np.arange(A, dtype=np.uint32), 1000), o.receive_batch(np.arange(A), 1000), "drain")
    s.close(); o.close()


def test_c2_backlog_drop_at_the_median_matches_oracle_digests():
    """The 1M-agent c2 backlog (65,536 group sends x 64 = 4,194,304 pending records, a seeded uniform timestamp per
    send), drop mode at the median cutoff, then the full drain's digests against an oracle that was only ever sent the
    surviving sends (same sequence numbers), and the queue statistics against it."""
    from bench import Workload
    from oracle.cpu_ref import CpuOracle
    from swarmdb_b200._native import Shard
    wl = Workload()
    g = Shard(max_agents=wl.A, ring_slots=64, arena_bytes=1 << 31, max_payload_bytes=wl.L, max_groups=wl.G,
              member_pool_entries=wl.A + 1024, max_batch_sends=wl.S, max_batch_payload=wl.S * wl.L,
              max_recv_records=1 << 23, max_recv_payload=(1 << 23) * wl.L)
    full, surv = CpuOracle(wl.A, wl.G), CpuOracle(wl.A, wl.G)
    g.register(np.arange(wl.A, dtype=np.uint32))
    for o in (full, surv):
        o.register(np.arange(wl.A))
    for k in range(wl.G):
        g.create_group(k, wl.members(k)); full.create_group(k, wl.members(k)); surv.create_group(k, wl.members(k))
    b = wl.batch()
    ts = np.random.default_rng(99).uniform(0.0, 1.0, wl.S)
    base = g.send_group_batch(*b, ts=ts)
    full.send_group_batch(*b, ts=ts)
    cut = float(np.median(ts))
    keep = ~(ts < cut)
    sender, grp, prio, typ, lens, off, pay = b
    # every group has F members and no sender is in its own group: send i numbers its members from base + F i
    surv.send_group_seq(sender[keep], grp[keep], prio[keep], typ[keep], lens[keep], off[keep], pay,
                        base + wl.F * np.nonzero(keep)[0].astype(np.uint64), ts[keep])
    cnt, total = g.expire(None, cut, archive=False)
    lf, ls = full.agent_loads(None, wl.A), surv.agent_loads(None, wl.A)
    assert total == wl.F * int((~keep).sum())
    assert np.array_equal(cnt.astype(np.int64), lf["pending"].astype(np.int64) - ls["pending"])
    qg, qs = g.queue_stats(), surv.queue_stats(wl.A)
    assert {k: qg[k] for k in ("pending", "pending_by_prio", "pending_granules", "agents_with_pending")} == \
        {k: qs[k] for k in ("pending", "pending_by_prio", "pending_granules", "agents_with_pending")}
    assert qg["received"] == full.queue_stats(wl.A)["received"]
    full.close()
    g.digest_reset(); surv.digest_enable()
    _, tot, _ = g.receive_batch(None, 100, copy_out=False)
    g.digest_fold()
    surv.receive_counts(None, 100)
    assert tot == wl.S * wl.F - total
    assert np.array_equal(g.digest_read(), surv.digest_read())
    g.close(); surv.close()
