"""Relocation of pinned queues on the device (sdb_arena_relocate).

Most cases run one seeded program on two handles: A has a small arena and relocates whenever a send would not fit, B has
a large arena and never relocates.  Relocation changes only where records sit in HBM, so every result of A must equal
B's byte for byte: receives on every path, agent loads, queue stats, digests and delivery counts.
"""
import numpy as np
import pytest

from tests.test_gpu_shared_layout import _payloads

pytestmark = pytest.mark.gpu

A, G, F = 1024, 8, 64                     # agents; groups of F members over the first G x F agents (exclusive)


def _shard(arena, **kw):
    from swarmdb_b200._native import Shard
    s = Shard(max_agents=A, max_groups=G, ring_slots=1024, arena_bytes=arena, max_payload_bytes=256,
              max_recv_records=1 << 18, **kw)
    s.register(np.arange(A, dtype=np.uint32))
    for g in range(G):
        s.create_group(g, np.arange(g * F, (g + 1) * F, dtype=np.uint32))
    return s


def _eq(ra, rb, what):
    assert len(ra) == len(rb), what
    for x, y in zip(ra, rb):
        if isinstance(x, np.ndarray):
            assert x.tobytes() == y.tobytes(), what
        else:
            assert x == y, what


def _expanded(res):
    """A compact-format result with its rows expanded: relocation may split a send's shared image in two (the moved
    members' copy and the original), which changes the rows but never the records."""
    from swarmdb_b200._native import expand_compact
    return (res[0].copy(), *expand_compact(res[1], res[2], res[3])) + tuple(res[4:])


def _loads_eq(a, b, what):
    assert a.agent_loads(np.arange(A, dtype=np.uint32)).tobytes() == b.agent_loads(np.arange(A, dtype=np.uint32)).tobytes(), what
    assert a.queue_stats() == b.queue_stats(), what


class Twin:
    def __init__(self, small, large=1 << 28, **kw):
        self.a, self.b = _shard(small, **kw), _shard(large, **kw)
        self.relocations = []

    def both(self, fn, what):
        ra = fn(self.a)
        ra = tuple(x.copy() if isinstance(x, np.ndarray) else x for x in ra) if isinstance(ra, tuple) else ra
        rb = fn(self.b)
        if isinstance(ra, tuple):
            _eq(ra, rb, what)
        else:
            assert ra == rb, what
        return ra

    def relocate(self, cut):
        """One relocation of A at `cut`, held to the contract: dry run = real call, counters, floor, idempotence."""
        a = self.a
        st0 = a.stats()
        dry = a.relocate(cut, peek=True)
        assert {k: v for k, v in a.stats().items() if k != "kernel_launches"} == \
            {k: v for k, v in st0.items() if k != "kernel_launches"}  # the dry run writes nothing
        s = a.relocate(cut)
        assert s == dry
        st1 = a.stats()
        moved = {k: st1[k] - st0[k] for k in st0 if k not in ("arena_tail_bytes", "arena_floor_bytes", "kernel_launches")}
        assert all(v == 0 for v in moved.values()), moved
        if s["records"]:
            assert st1["arena_tail_bytes"] == st0["arena_tail_bytes"] + s["skipped_bytes"] + s["moved_bytes"] == s["tail_after"]
        assert st1["arena_floor_bytes"] == s["floor_after"] >= min(cut, st0["arena_tail_bytes"])
        assert s["moved_bytes"] >= 32 * s["records"] and (s["records"] == 0) == (s["agents"] == 0)
        again = a.relocate(min(cut, st0["arena_tail_bytes"]))
        assert again["records"] == 0 and again["moved_bytes"] == 0 and a.stats()["arena_tail_bytes"] == st1["arena_tail_bytes"]
        _loads_eq(self.a, self.b, "loads after a relocation")
        self.relocations.append(s)
        return s

    def send(self, fn, what):
        """fn on A, then on B.  A relocates what pins the lower part of its log once half of it is in use, and
        everything when a send still does not fit."""
        from swarmdb_b200._native import SdbError
        st = self.a.stats()
        tail, arena = st["arena_tail_bytes"], int(self.a.cfg.arena_bytes)
        if tail - st["arena_floor_bytes"] > arena // 2:
            self.relocate(tail - arena // 4)
        try:
            ba = fn(self.a)
        except SdbError as e:
            assert e.code == -5, (what, str(e))
            self.relocate(self.a.stats()["arena_tail_bytes"])
            ba = fn(self.a)
        assert fn(self.b) == ba, what

    def close(self):
        self.a.close(); self.b.close()


def _program(t, rng, rounds):
    """Sends of every kind, partial stream and priority receives, filtered takes, expiry and requeue, on idle agents too."""
    from swarmdb_b200._native import RECV_PEEK, RECV_PRIORITY, make_filter
    idle = np.arange(0, A, 31, dtype=np.uint32)                       # never received by plain receives
    busy = np.setdiff1d(np.arange(A), idle).astype(np.uint32)
    ts = [0.0]
    for rnd in range(rounds):
        n = 200
        s, r, prio = rng.integers(0, A, n), rng.integers(0, A, n), rng.integers(0, 4, n)
        lens, off, buf = _payloads(rng, n, 256)
        tsv = ts[0] + rng.uniform(0, 1, n)
        t.send(lambda x: x.send_batch(s, r, prio, None, lens, off, buf, tsv), "p2p")
        n = 300 if rnd % 2 == 0 else 40                               # 300 x 64 records: shared layout; 40: per recipient
        s, grp, prio = rng.integers(G * F, A, n), rng.integers(0, G, n), rng.integers(0, 4, n)
        lens, off, buf = _payloads(rng, n, 256)
        lens[: n // 10] = 0                                           # zero-length shared payloads too
        tsv = ts[0] + rng.uniform(0, 1, n)
        t.send(lambda x: x.send_group_batch(s, grp, prio, None, lens, off, buf, tsv), "group")
        n = 5
        lists = [rng.choice(A, size=int(rng.integers(1, 300)), replace=False) for _ in range(n)]
        lo = np.zeros(n + 1, np.uint64); lo[1:] = np.cumsum([len(x) for x in lists])
        li = np.concatenate(lists).astype(np.uint32)
        s, prio = rng.integers(0, A, n), rng.integers(0, 4, n)
        lens, off, buf = _payloads(rng, n, 256)
        t.send(lambda x: x.send_list_batch(s, lo, li, prio, None, lens, off, buf), "broadcast")
        n = 60
        s, kind, prio = rng.integers(0, A, n), rng.integers(0, 3, n).astype(np.uint8), rng.integers(0, 4, n)
        ml = [rng.choice(A, size=int(rng.integers(1, 40)), replace=False) for _ in range(n)]
        mlo = np.zeros(n + 1, np.uint64); mlo[1:] = np.cumsum([len(x) for x in ml])
        mli = np.concatenate(ml).astype(np.uint32)
        target = np.where(kind == 0, rng.integers(0, A, n), np.where(kind == 1, rng.integers(0, G, n), np.arange(n))).astype(np.uint32)
        lens, off, buf = _payloads(rng, n, 256)
        t.send(lambda x: x.send_mixed_batch(s, kind, target, mlo, mli, prio, None, lens, off, buf), "mixed")
        ts[0] += 1.0
        sub = rng.choice(busy, 400, replace=False).astype(np.uint32)
        t.both(lambda x: x.receive_batch(sub, 2), "stream receive")
        sub = rng.choice(busy, 300, replace=False).astype(np.uint32)
        t.both(lambda x: x.receive_batch(sub, 3, RECV_PRIORITY), "priority receive")
        sub = rng.choice(A, 200, replace=False).astype(np.uint32)
        f = make_filter(prios=[3])
        t.both(lambda x: x.receive_where(sub, 2, 0, f), "filtered take (tombstones)")
        t.both(lambda x: x.receive_batch(busy, 1024), "the busy agents catch up")
        if rnd % 3 == 2:
            sub = rng.choice(A, 100, replace=False).astype(np.uint32)
            t.both(lambda x: x.expire(sub, ts[0] - 1.5, archive=False), "expiry")
            sub = rng.choice(busy, 50, replace=False).astype(np.uint32)
            taken = {}
            t.both(lambda x: _expanded(taken.setdefault(id(x), tuple(y.copy() for y in x.receive_compact(sub, 4)))),
                   "compact take")
            t.send(lambda x: x.restore_compact(sub, *taken[id(x)]), "requeue")
        t.both(lambda x: _expanded(x.receive_compact(idle[:64], 1000, RECV_PEEK)), "compact peek of idle agents")


def _drain(t):
    from swarmdb_b200._native import RECV_PEEK, RECV_PRIORITY
    every = np.arange(A, dtype=np.uint32)
    for flags in (RECV_PRIORITY | RECV_PEEK, RECV_PEEK):
        t.both(lambda x: x.receive_batch(every, 1024, flags), "peek drain")
    for x in (t.a, t.b):
        x.digest_reset()
    while True:
        got = t.both(lambda x: (x.receive_batch(every, 1024), x.digest_fold())[0], "drain")
        if len(got[1]) == 0:
            break
    assert np.array_equal(t.a.digest_read(every), t.b.digest_read(every))
    assert t.a.queue_stats()["pending"] == 0


@pytest.mark.parametrize("shared", ["1", "0"])
def test_twin_handles_agree_through_relocations(shared, monkeypatch):
    monkeypatch.setenv("SDB_SHARED_PAYLOAD", shared)
    rng = np.random.default_rng(71)
    t = Twin(1 << (23 if shared == "1" else 25))
    _program(t, rng, 14)
    assert len(t.relocations) >= 2 and any(s["agents"] for s in t.relocations), t.relocations
    _drain(t)
    t.close()


@pytest.mark.parametrize("shared", ["1", "0"])
def test_pinned_arena_keeps_the_idle_agents_record(shared, monkeypatch):
    """The expiry test's scenario, but the pinned record is kept: one relocation lets the refused send through."""
    monkeypatch.setenv("SDB_SHARED_PAYLOAD", shared)
    from swarmdb_b200._native import SdbError, Shard
    g = Shard(max_agents=64, ring_slots=4096, arena_bytes=1 << 20, max_payload_bytes=256)
    g.register(np.arange(64, dtype=np.uint32))
    lens, off = np.full(64, 200, np.uint16), np.arange(64, dtype=np.uint64) * 256
    buf = np.full(64 * 256 + 64, 65, np.uint8)
    buf[:200] = np.arange(200) % 251
    g.send_batch([1], [0], None, None, lens[:1], off[:1], buf, np.array([1.0]))           # agent 0 never receives
    _, want_h, want_p = (x.copy() for x in g.receive_batch([0], 1, 2))                   # PEEK
    t = 2.0
    with pytest.raises(SdbError) as e:
        for _ in range(10000):
            g.send_batch(np.ones(64), np.full(64, 5), None, None, lens, off, buf, np.full(64, t))
            assert len(g.receive_batch([5], 1000)[1]) == 64
            t += 1.0
    assert e.value.code == -5
    tail = g.stats()["arena_tail_bytes"]
    s = g.relocate(tail - (1 << 19))
    assert s["agents"] == 1 and s["records"] == 1 and s["moved_bytes"] == 32 * 8
    g.send_batch(np.ones(64), np.full(64, 5), None, None, lens, off, buf, np.full(64, t))
    assert len(g.receive_batch([5], 1000)[1]) == 64
    _, h, p = g.receive_batch([0], 10)
    assert h.tobytes() == want_h.tobytes() and p.tobytes() == want_p.tobytes()
    g.close()


@pytest.mark.parametrize("shared", ["1", "0"])
def test_exact_size_records_and_floor(shared, monkeypatch):
    """Agents that got the first phase's traffic are selected at a cut between the phases; moved_bytes is the PEEK
    compact identity over them and records their pending counts.  A cut at the tail moves every pending record."""
    monkeypatch.setenv("SDB_SHARED_PAYLOAD", shared)
    from swarmdb_b200._native import RECV_PEEK, make_filter
    rng = np.random.default_rng(5)
    t = Twin(1 << 26)
    first = np.arange(0, 4 * F, dtype=np.uint32)                      # groups 0..3 and p2p / broadcast to their members
    second = np.arange(4 * F, A, dtype=np.uint32)
    for agents, groups in ((first, np.arange(0, 4)), (second, np.arange(4, G))):
        n = 300
        s, grp = rng.integers(0, A, n), rng.choice(groups, n)
        lens, off, buf = _payloads(rng, n, 256)
        lens[:20] = 0
        t.send(lambda x: x.send_group_batch(s, grp, None, None, lens, off, buf), "group")
        n = 300
        s, r = rng.integers(0, A, n), rng.choice(agents, n)
        lens, off, buf = _payloads(rng, n, 256)
        t.send(lambda x: x.send_batch(s, r, None, None, lens, off, buf), "p2p")
        lo = np.array([0, 50], np.uint64); li = rng.choice(agents, 50, replace=False).astype(np.uint32)
        lens, off, buf = _payloads(rng, 1, 256)
        t.send(lambda x: x.send_list_batch([1], lo, li, None, None, lens, off, buf), "broadcast")
        if agents is first:
            cut = t.a.stats()["arena_tail_bytes"]
    t.both(lambda x: x.receive_batch(first[::3], 5), "take some")
    t.both(lambda x: x.receive_where(first[1::3], 3, 0, make_filter(prios=[1, 2])), "holes")
    pend = t.a.agent_loads(first)["pending"]
    sel = first[pend > 0]
    _, ent, snd, _ = t.a.receive_compact(sel, 1024, RECV_PEEK)
    want = 32 * (len(ent) + int(((snd["len"].astype(np.int64) + 31) // 32).sum()))
    s = t.relocate(cut)
    assert s["agents"] == len(sel) and s["records"] == int(pend.sum()) and s["moved_bytes"] == want
    pend_all = t.a.agent_loads(np.arange(A, dtype=np.uint32))["pending"]
    s = t.relocate(t.a.stats()["arena_tail_bytes"] + 12345)            # beyond the tail: a full compaction
    assert s["agents"] == int((pend_all > 0).sum()) and s["records"] == int(pend_all.sum())
    _drain(t)
    t.close()


@pytest.mark.parametrize("shared", ["1", "0"])
def test_dead_letter_counts_survive_a_relocation(shared, monkeypatch):
    monkeypatch.setenv("SDB_SHARED_PAYLOAD", shared)
    from swarmdb_b200._native import LEASE_ALL
    rng = np.random.default_rng(9)
    t = Twin(1 << 26)
    for x in (t.a, t.b):
        x.lease_reserve(1 << 14, (1 << 14) * 256)
        x.lease_set_policy(3, 1 << 14)
    n = 300
    s, grp = rng.integers(0, A, n), rng.integers(0, G, n)
    lens, off, buf = _payloads(rng, n, 256)
    t.send(lambda x: x.send_group_batch(s, grp, None, None, lens, off, buf), "group")
    s, r = rng.integers(0, A, n), rng.integers(0, A, n)
    lens, off, buf = _payloads(rng, n, 256)
    t.send(lambda x: x.send_batch(s, r, None, None, lens, off, buf), "p2p")
    sub = rng.choice(A, 300, replace=False).astype(np.uint32)
    for sweep in range(2):
        got = t.both(lambda x: _expanded(x.receive_leased(sub, 1024, 1.0)), "leased receive")
        ids = np.arange(got[3], got[3] + len(got[1]), dtype=np.uint64)
        t.both(lambda x: tuple(x.lease_deliveries(ids)), "counts")
        t.both(lambda x: x.lease_sweep(2.0, LEASE_ALL), "sweep")
    t.relocate(t.a.stats()["arena_tail_bytes"])
    got = t.both(lambda x: _expanded(x.receive_leased(sub, 1024, 1.0)), "leased receive after the relocation")
    ids = np.arange(got[3], got[3] + len(got[1]), dtype=np.uint64)
    d = t.both(lambda x: tuple(x.lease_deliveries(ids)), "counts after the relocation")
    assert max(d) == 3
    t.both(lambda x: x.lease_sweep(2.0, LEASE_ALL), "third sweep")
    assert t.a.lease_policy_stats()["dead"] == t.b.lease_policy_stats()["dead"] > 0
    t.both(lambda x: _expanded(x.lease_dead_letters(sub)), "dead letters")
    t.close()


def test_handle_wrap_and_physical_wrap():
    """A moved region that would cross the arena's end is placed after it (skipped_bytes > 0), and there its handles
    wrap at 2^32 granules; then the random program runs across the wrap."""
    rng = np.random.default_rng(13)
    t = Twin(1 << 23)
    p0 = (1 << 32) - 1000                                              # 1000 granules before the arena's end and the wrap
    for x in (t.a, t.b):
        x.debug_set_arena_pos(p0)
    assert t.a.relocate(0)["records"] == 0
    lens, off = np.full(50, 256, np.uint16), np.arange(50, dtype=np.uint64) * 256
    buf = rng.integers(0, 256, 50 * 256 + 64).astype(np.uint8)
    t.send(lambda x: x.send_batch(np.full(50, 3), np.arange(50), None, None, lens, off, buf), "50 pinned records")
    t.send(lambda x: x.send_batch(np.full(30, 3), np.full(30, 100), None, None, lens[:30], off[:30], buf), "to agent 100")
    t.both(lambda x: x.receive_batch([100], 100), "agent 100 receives")
    tail = t.a.stats()["arena_tail_bytes"]
    assert tail == 32 * (p0 + 720)
    s = t.relocate(tail)
    assert s["records"] == 50 and s["moved_bytes"] == 32 * 450 and s["skipped_bytes"] == 32 * 280
    assert s["tail_after"] == 32 * ((1 << 32) + 450) == s["floor_after"] + 32 * 450
    _program(t, rng, 8)
    _drain(t)
    t.close()


def test_refusals_change_nothing():
    from swarmdb_b200._native import RECV_PEEK, SdbError
    rng = np.random.default_rng(17)
    g = _shard(1 << 20)
    n = 100
    s, r = rng.integers(0, A, n), rng.integers(0, A, n)
    lens, off, buf = _payloads(rng, n, 256)
    while g.stats()["arena_tail_bytes"] < (3 << 18):
        g.send_batch(s, r, None, None, lens, off, buf)
    every = np.arange(A, dtype=np.uint32)
    before = (g.stats(), g.agent_loads(every).tobytes(), g.queue_stats(), g.receive_compact(every, 1024, RECV_PEEK)[1].tobytes())
    for peek in (True, False):
        with pytest.raises(SdbError) as e:
            g.relocate(g.stats()["arena_tail_bytes"], peek=peek)             # 3/4 of the arena is live: no room for a copy
        assert e.value.code == -5
    with pytest.raises(SdbError) as e:
        g._check(g._L.sdb_arena_relocate(g._h, 0, 1, None))
    assert e.value.code == -1
    after = (g.stats(), g.agent_loads(every).tobytes(), g.queue_stats(), g.receive_compact(every, 1024, RECV_PEEK)[1].tobytes())
    assert before[1:] == after[1:]
    assert {k: v for k, v in before[0].items() if k != "kernel_launches"} == \
        {k: v for k, v in after[0].items() if k != "kernel_launches"}
    g.close()


@pytest.mark.parametrize("relocate", [True, False])
def test_surface_keeps_sending_past_an_idle_agent(relocate, tmp_path):
    import swarmdb_b200 as sdb
    cfg = sdb.GpuConfig(arena_relocate=relocate, arena_bytes=1 << 20, max_agents=64, max_groups=4, max_payload_bytes=1024,
                        deterministic_ids=True, flush_threshold=64)
    db = sdb.SwarmsDB(save_dir=str(tmp_path), auto_save=False, gpu_config=cfg)
    db.register_agents(["idle", "busy", "src"])
    kept = []
    try:
        for k in range(3000):
            if k % 100 == 0:
                kept.append(db.send_message("src", f"for idle {k}", "idle"))
            db.send_message("src", "x" * 600, "busy")
            if k % 64 == 63:
                db.flush()
                db.receive_messages("busy", 1000)
    except sdb._native.SdbError as e:
        assert not relocate and e.code == -5
    else:
        assert relocate
        got = db.receive_messages("idle", 1000)
        assert [m.id for m in got] == kept and [m.content for m in got] == [f"for idle {k}" for k in range(0, 3000, 100)]
    db.close()


@pytest.mark.parametrize("shared", ["1", "0"])
def test_latency_server_receives_after_a_relocation(shared, monkeypatch):
    """Single-agent receives served by the persistent dequeue kernel after a relocation (whose first call allocates its
    scratch and so stops a running server).  Only A runs a server: a second handle's cudaFree in the same process would
    wait on it.  B answers the same requests through the ordinary single-agent path."""
    monkeypatch.setenv("SDB_SHARED_PAYLOAD", shared)
    from swarmdb_b200._native import RECV_PRIORITY
    rng = np.random.default_rng(19)
    t = Twin(1 << 24)
    t.a.latency_server(True)
    n = 300
    s, grp, prio = rng.integers(G * F, A, n), rng.integers(0, G, n), rng.integers(0, 4, n)
    lens, off, buf = _payloads(rng, n, 256)
    t.send(lambda x: x.send_group_batch(s, grp, prio, None, lens, off, buf), "group")
    s, r, prio = rng.integers(0, A, n), rng.integers(0, 32, n), rng.integers(0, 4, n)
    lens, off, buf = _payloads(rng, n, 256)
    t.send(lambda x: x.send_batch(s, r, prio, None, lens, off, buf), "p2p")
    t.both(lambda x: tuple(y.copy() for y in x.receive_one(40, 2, 0)[:2]), "served before the relocation")
    s = t.relocate(t.a.stats()["arena_tail_bytes"])                  # first call: allocates, stops the server
    assert s["records"] > 0
    for a in list(range(8)) + [64, 65, 130]:
        for flags in (0, RECV_PRIORITY):
            t.both(lambda x: tuple(y.copy() for y in x.receive_one(a, 3, flags)[:2]), "served after the relocation")
    s = t.relocate(t.a.stats()["arena_tail_bytes"])                  # the server runs through a later relocation
    for a in range(8, 16):
        t.both(lambda x: tuple(y.copy() for y in x.receive_one(a, 5, 0)[:2]), "served after a second relocation")
    t.a.latency_server(False)
    _drain(t)
    t.close()


@pytest.mark.parametrize("shared", ["1", "0"])
def test_async_import_after_a_relocation(shared, monkeypatch):
    """A num_shards = 1 asynchronous import whose localize pass was prefetched before a relocation and placed after it:
    it must land behind the moved region and deliver what the same steps deliver without the relocation."""
    monkeypatch.setenv("SDB_SHARED_PAYLOAD", shared)
    from tests.test_gpu_xshard import _async_cluster
    Aa, Ga, Fa, S = 4096, 64, 64, 200
    groups = [np.arange(g * Fa, (g + 1) * Fa) for g in range(Ga)]
    outs = []
    for relocate in (True, False):
        rng = np.random.default_rng(23)
        smap, shards, wb, bufs = _async_cluster(1, Aa, Ga, S, groups, arena_bytes=1 << 24)
        sh = shards[0]
        for step in (1, 2, 3):
            sender = rng.integers(0, Aa, S); grp = rng.integers(0, Ga, S)
            lens, off, buf = _payloads(rng, S, 256)
            sh.export_group_batch(sender, grp, None, None, lens, off, buf, bufs[step & 1][0], wb)
            sh.wire_publish(bufs[step & 1][0], wb, step)
            sh.import_prefetch(bufs[step & 1], wb, step)
            if relocate and step >= 2:
                tail = sh.stats()["arena_tail_bytes"]
                sm = sh.relocate(tail // 2)
                assert sm["records"] > 0 and sh.stats()["arena_tail_bytes"] == sm["tail_after"]
            sh.import_wire_ptrs_async(bufs[step & 1], wb, step)
            if relocate and step >= 2:
                st = sh.stats()
                assert st["arena_tail_bytes"] > sm["tail_after"] and st["arena_floor_bytes"] >= sm["floor_after"]
            if step == 2:                                              # a partial receive between the steps
                cnt, hdr, pay = sh.receive_batch(np.arange(0, Aa, 3, dtype=np.uint32), 4)
                outs.append((cnt.copy(), hdr.copy(), pay.copy()))
        cnt, hdr, pay = sh.receive_batch(np.arange(Aa, dtype=np.uint32), 1024)
        outs.append((cnt.copy(), hdr.copy(), pay.copy()))
        assert sh.queue_stats()["pending"] == 0
        sh.close()
    _eq(outs[0], outs[2], "partial receive with and without the relocation")
    _eq(outs[1], outs[3], "drain with and without the relocation")
