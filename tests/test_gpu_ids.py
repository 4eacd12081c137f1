"""The id clause of the filtered receive (SDB_FILTER_IDS) on the device, against tests/ids_ref.py byte for byte: one id
against the seq range it equals, id sets from empty to a million over every mode, order, agent list and kernel, the
per-id outputs (a broadcast queued at every agent included), the refusals, and the SwarmsDB surface."""
import ctypes as C

import numpy as np
import pytest

from tests.ids_ref import IdsOracle
from tests.test_gpu_compact_receive import Rig, _same
from tests.test_gpu_where import _loads_same, _traffic

pytestmark = pytest.mark.gpu


def _rig(seed, seq0=None, shared="1", monkeypatch=None, **kw):
    if monkeypatch is not None:
        monkeypatch.setenv("SDB_SHARED_PAYLOAD", shared)
    rig = Rig(np.random.default_rng(seed), G=8, F=64, extra=64, **kw)
    rig.check_advance = False
    if seq0 is not None:                                     # seqs past 2^32: the handle and the oracle move together
        rig.g.advance_seq(seq0)
        rig.c.next_seq = seq0
    rig.c = IdsOracle(rig.c, rig.G, dict(enumerate(rig.members)), rig.A)
    rig.d0 = rig.g.stats()["delivered"]
    return rig


def _seqs(rig):
    """Every pending seq, and how many copies of each (the oracle's PEEK of the whole queue)."""
    st = rig.c.snapshot()
    s = np.array([int(h["seq"]) for recs in st.values() for h, _ in recs], np.uint64)
    u, n = np.unique(s, return_counts=True)
    return u, n


def _where(rig, agents, k, flags, filt, what, drop=False, outputs=False):
    n_ids = int(filt.n_ids)
    hg, ag, hc, ac = (np.zeros(n_ids, np.uint32) for _ in range(4)) if outputs else (None,) * 4
    got = rig.g.receive_where(agents, k, flags, filt, drop=drop, id_hits=hg, id_agent=ag)
    want = rig.c.receive_where(agents, k, flags & ~32, filt, drop=drop, id_hits=hc, id_agent=ac)
    if drop:
        assert got[1] == want[1] and np.array_equal(got[0], want[0]), what
    else:
        _same(got, want, what)
    if outputs:
        assert np.array_equal(hg, hc) and np.array_equal(ag, ac), what
    _loads_same(rig.g, rig.c, rig.idx, what)
    return got


@pytest.mark.parametrize("shared,seq0", [("1", None), ("0", None), ("1", (1 << 32) - 500)])
def test_one_id_equals_the_seq_range(shared, seq0, monkeypatch):
    """For p2p, both group payload layouts, broadcast lists and seqs across 2^32: the id clause with one id returns,
    byte for byte, what SDB_FILTER_SEQ [s, s + 1) returns, in every mode; the queues then drain identically."""
    from swarmdb_b200._native import RECV_PEEK, RECV_PRIORITY, WHERE_DROP, make_filter
    rigs = [_rig(41, seq0, shared, monkeypatch) for _ in range(2)]
    for rig in rigs:
        _traffic(rig)
    u, n = _seqs(rigs[0])
    rng = np.random.default_rng(5)
    pick = list(rng.choice(u, 40, replace=False)) + [u[np.argmax(n)]] + ([1 << 32] if seq0 else [])
    for s in pick:
        s = int(s)
        fi, fs = make_filter(ids=[s]), make_filter(seq=(s, s + 1))
        for flags in (RECV_PEEK, RECV_PEEK | RECV_PRIORITY):
            a = rigs[0].g.receive_where(None, 1000, flags, fi)
            b = rigs[0].g.receive_where(None, 1000, flags, fs)
            _same(a, b, (s, flags))
        ci, ti = rigs[0].g.receive_where(None, 1000, WHERE_DROP | RECV_PEEK, fi, drop=True)
        cs, ts = rigs[0].g.receive_where(None, 1000, WHERE_DROP | RECV_PEEK, fs, drop=True)
        assert ti == ts and np.array_equal(ci, cs)
    # take on one twin, drop on the other, with the two clauses alternating
    for k, s in enumerate(pick[:20]):
        s = int(s)
        f = make_filter(ids=[s]) if k % 2 else make_filter(seq=(s, s + 1))
        g = make_filter(seq=(s, s + 1)) if k % 2 else make_filter(ids=[s])
        _where(rigs[0], None, 1000, RECV_PRIORITY if k % 3 else 0, f, ("take", s))
        _where(rigs[1], None, 1000, WHERE_DROP, g, ("drop", s), drop=True)
    for flags in (RECV_PRIORITY, 0):
        for rig in rigs:
            _same(rig.g.receive_batch(rig.idx, 100000, flags | RECV_PEEK),
                  rig.c.receive_batch(rig.idx, 100000, flags | RECV_PEEK), "rings")
    _same(rigs[0].g.receive_batch(rigs[0].idx, 100000), rigs[0].c.receive_batch(rigs[0].idx, 100000), "drain 0")
    _same(rigs[1].g.receive_batch(rigs[1].idx, 100000), rigs[1].c.receive_batch(rigs[1].idx, 100000), "drain 1")
    for rig in rigs:
        assert rig.g.queue_stats()["pending"] == 0
        rig.close()


def test_sets_every_mode_order_agent_list_and_kernel():
    """Sets of 0, 1, 1 k and 1 M ids (present, absent, duplicated, id 0) against the model: PEEK, take, drop and
    DROP | PEEK, stream and priority order, agent lists and NULL, the header and the keyword kernel, with the per-id
    outputs."""
    from swarmdb_b200._native import RECV_PEEK, RECV_PRIORITY, WHERE_DROP, make_filter
    rig = _rig(43)
    _traffic(rig, rounds=2)
    u, _ = _seqs(rig)
    rng = np.random.default_rng(9)
    big = np.concatenate([rng.choice(u, len(u) // 2, replace=False), rng.integers(1, 1 << 40, (1 << 20) - len(u) // 2 - 2,
                                                                                  dtype=np.uint64), [0, u[0]]]).astype(np.uint64)
    sets = {"empty": np.zeros(0, np.uint64), "one": u[:1], "1k": np.concatenate([rng.choice(u, 900), [0] * 4,
                                                                                rng.integers(1 << 33, 1 << 34, 96)]),
            "1M": rng.permutation(big)}
    agents = rng.permutation(rig.A).astype(np.uint32)
    for name, ids in sets.items():
        for extra in ({}, {"prios": [1, 2, 3]}, {"keyword": b"ab", "icase": True}):
            f = make_filter(ids=ids, **extra)
            for flags in (RECV_PEEK, RECV_PEEK | RECV_PRIORITY):
                for ag in (None, agents[:500]):
                    _where(rig, ag, 3, flags, f, (name, extra, flags), outputs=True)
            _where(rig, agents[:300], 1000, WHERE_DROP | RECV_PEEK, f, (name, extra, "dry"), drop=True, outputs=True)
    for name in ("1k", "one", "1M"):
        f = make_filter(ids=sets[name])
        _where(rig, agents[:700], 2, RECV_PRIORITY, f, (name, "take"), outputs=True)
        _where(rig, None, 1, 0, make_filter(ids=sets[name], keyword=b"a"), (name, "take kw"), outputs=True)
        _where(rig, agents[700:], 1000, WHERE_DROP, f, (name, "drop"), drop=True, outputs=True)
    _same(rig.g.receive_batch(rig.idx, 100000), rig.c.receive_batch(rig.idx, 100000), "drain")
    rig.close()


def test_broadcast_at_every_agent_sends_all_hits_to_one_slot():
    """One broadcast list to every agent: id_hits is the number of agents and id_agent the smallest, for the whole
    list, a part of it and with the keyword kernel; a drop then removes exactly those copies."""
    from swarmdb_b200._native import RECV_PEEK, WHERE_DROP, make_filter
    rig = _rig(47)
    _traffic(rig)
    A = rig.A
    buf = np.frombuffer(b"broadcast to all".ljust(64, b" "), np.uint8).copy()
    lo = np.array([0, A], np.uint64)
    base = rig.c.send_list_batch([3], lo, rig.idx, [2], [0], [16], [0], buf, [1.0])
    assert rig.g.send_list_batch([3], lo, rig.idx, [2], [0], [16], [0], buf, [1.0]) == base
    for ag, kw in ((None, None), (rig.idx[A // 2:][::-1].copy(), None), (None, b"ALL")):
        f = make_filter(ids=[base, 12345678, base], keyword=kw, icase=kw is not None)
        hits, first = np.zeros(3, np.uint32), np.zeros(3, np.uint32)
        rig.g.receive_where(ag, 1, RECV_PEEK | WHERE_DROP, f, drop=True, id_hits=hits, id_agent=first)
        n = A if ag is None else len(ag)
        lo_agent = 0 if ag is None else int(ag.min())
        assert hits[0] == hits[2] >= n - 1 and hits[1] == 0                 # the sender may hold no copy
        assert first[0] == first[2] <= lo_agent + 1 and first[1] == 0xFFFFFFFF
        _where(rig, ag, 1, RECV_PEEK | WHERE_DROP, f, ("bc", kw), drop=True, outputs=True)
    _where(rig, None, 1 << 20, WHERE_DROP, make_filter(ids=[base]), "drop bc", drop=True, outputs=True)
    _same(rig.g.receive_batch(rig.idx, 100000), rig.c.receive_batch(rig.idx, 100000), "drain")
    rig.close()


def test_refusals_leave_the_queue_alone():
    """The old struct_bytes still works without the clause; each refusal is SDB_EINVAL and moves nothing."""
    from swarmdb_b200._native import RECV_PEEK, SdbError, make_filter
    rig = _rig(53)
    _traffic(rig)
    u, _ = _seqs(rig)
    old = make_filter(prios=[1, 2])
    want = rig.g.receive_where(None, 5, RECV_PEEK, old)
    old.struct_bytes = 64
    _same(rig.g.receive_where(None, 5, RECV_PEEK, old), want, "old struct_bytes")
    before = rig.g.agent_loads(rig.idx).copy()
    bad = []
    f = make_filter(ids=u[:3]); f.struct_bytes = 64; bad.append((f, {}))
    f = make_filter(ids=u[:3]); f.ids = None; bad.append((f, {}))
    f = make_filter(ids=[]); f.ids = None; bad.append((f, {}))
    f = make_filter(ids=u[:3]); f.n_ids = (1 << 22) + 1; bad.append((f, {}))
    bad.append((make_filter(prios=[1]), {"id_hits": np.zeros(0, np.uint32)}))
    for f, kw in bad:
        hits = np.zeros(int(f.n_ids) if f.fields & 512 else 0, np.uint32) if kw else None
        f.id_hits = None if hits is None else hits.ctypes.data
        counts = np.zeros(rig.A, np.uint32)
        rc = rig.g._L.sdb_receive_where(rig.g._h, 0, None, 5, 0, C.byref(f), counts.ctypes.data_as(C.c_void_p), None, 0,
                                        None, 0, None, None)
        assert rc == -1, (f.fields, f.n_ids, kw)
    with pytest.raises(ValueError):
        rig.g.receive_where(None, 5, 0, make_filter(ids=u[:3]), id_hits=np.zeros(2, np.uint32))
    with pytest.raises(SdbError):
        rig.g.receive_where(None, 5, 0, make_filter(prios=[1]), id_agent=np.zeros(0, np.uint32))
    assert rig.g.agent_loads(rig.idx).tobytes() == before.tobytes()
    rig.close()


def test_owned_agents_of_a_sharded_handle():
    """SDB_RECV_OWNED with the id clause on two shards of one GPU: each shard's PEEK, outputs and drop equal the
    model's over its own agents."""
    from oracle.cpu_ref import CpuOracle
    from swarmdb_b200._native import RECV_OWNED, RECV_PEEK, WHERE_DROP, make_filter
    from tests.test_gpu_where import _payloads, _types
    from tests.test_gpu_xshard import _async_cluster
    rng = np.random.default_rng(59)
    A, G, F, S, world = 2048, 32, 64, 300, 2
    perm = rng.permutation(A)
    groups = [perm[k * F:(k + 1) * F] for k in range(G)]
    smap, shards, wb, bufs = _async_cluster(world, A, G, S, groups)
    o = CpuOracle(A, G)
    for k, m in enumerate(groups):
        o.create_group(k, m)
    o.register(np.arange(A))
    for s in shards:
        s.register(np.arange(A, dtype=np.uint32))
    o = IdsOracle(o, G, dict(enumerate(groups)), A)
    for r in range(world):
        sender, grp, prio, typ = rng.integers(0, A, S), rng.integers(0, G, S), rng.integers(0, 4, S), _types(rng, S)
        lens, off, buf = _payloads(rng, S, 256, typ)
        ts = rng.uniform(0, 10, S)
        shards[r].export_group_batch(sender, grp, prio, typ, lens, off, buf, bufs[1][r], wb, ts)
        shards[r].wire_publish(bufs[1][r], wb, 1)
        o.send_group_batch(sender, grp, prio, typ, lens, off, buf, ts)
    for s in shards:
        s.import_wire_ptrs_async(bufs[1], wb, 1)
    st = o.snapshot()
    u = np.unique([int(h["seq"]) for recs in st.values() for h, _ in recs]).astype(np.uint64)
    ids = np.concatenate([rng.choice(u, 200, replace=False), [0, 7 << 40]]).astype(np.uint64)
    for r, s in enumerate(shards):
        local = np.nonzero(smap == r)[0].astype(np.uint32)
        f = make_filter(ids=ids)
        hg, ag, hc, ac = (np.zeros(len(ids), np.uint32) for _ in range(4))
        cg, xg, pg = s.receive_where(None, 1000, RECV_OWNED | RECV_PEEK, f, id_hits=hg, id_agent=ag)
        cc, xc, pc = o.receive_where(local, 1000, RECV_PEEK, f, id_hits=hc, id_agent=ac)
        assert np.array_equal(cg, cc) and xg.tobytes() == xc.tobytes() and pg.tobytes() == pc.tobytes(), r
        assert np.array_equal(hg, hc) and np.array_equal(ag, ac), r
        cg, tg = s.receive_where(None, 1000, RECV_OWNED | WHERE_DROP, f, drop=True)
        cc, tc = o.receive_where(local, 1000, 0, f, drop=True)
        assert np.array_equal(cg, cc) and tg == tc > 0, r
        _loads_same(s, o, local, (r, "drop"))
    for s in shards:
        s.close()
    o.close()


def test_surface_get_delete_and_receive_matching(tmp_path):
    """get_message / get_messages with include_device, delete_messages and receive_matching(message_ids=) on a
    SwarmsDB over the device, for device-only bulk traffic and a broadcast whose host record was dropped."""
    import swarmdb_b200 as sdb
    db = sdb.SwarmsDB(save_dir=str(tmp_path), auto_save=False,
                      gpu_config=sdb.GpuConfig(max_agents=256, max_groups=4, deterministic_ids=True, ring_slots=256,
                                               arena_bytes=1 << 24, max_payload_bytes=512))
    names = [f"ag{i}" for i in range(200)]
    db.register_agents(names)
    n = 600
    rng = np.random.default_rng(61)
    bodies = [f"bulk {i}".encode() for i in range(n)]
    buf = b"".join(b.ljust(32, b" ") for b in bodies) + bytes(32)
    recv = rng.integers(0, 200, n)
    base = db.send_batch(rng.integers(0, 200, n), recv, None, None, np.array([len(b) for b in bodies], np.uint16),
                         np.arange(n, dtype=np.uint64) * 32, np.frombuffer(buf, np.uint8))
    bc = db.broadcast_message("ag0", "to everyone")
    host = db.send_message("ag1", "host copy", receiver_id="ag2")
    db.flush()
    ids = [db._make_id(base + i) for i in range(n)]
    assert db.get_message(ids[7]) is None
    m = db.get_message(ids[7], include_device=True)
    assert m.content == "bulk 7" and m.receiver_id == names[recv[7]] and m.status == sdb.MessageStatus.DELIVERED
    pick = [ids[i] for i in rng.choice(n, 300, replace=False)] + ["junk", host, ids[3]]
    got = db.get_messages(pick, include_device=True)
    at = {mid: i for i, mid in enumerate(ids)}
    assert [g.content for g in got[:300]] == [f"bulk {at[i]}" for i in pick[:300]]
    assert got[300] is None and got[301] is db.messages[host] and got[302].content == "bulk 3"
    db.messages.pop(bc)
    assert db.get_message(bc, include_device=True).content == "to everyone"
    pending0 = db.get_stats()["queue"]["pending"]
    gone = [ids[i] for i in range(0, n, 3)]
    res = db.delete_messages(gone + [bc, "junk", gone[0]], include_device=True)
    assert res == [True] * len(gone) + [True, False, True]
    assert db.get_stats()["queue"]["pending"] == pending0 - len(gone) - 199
    assert db.get_messages(gone + [bc], include_device=True) == [None] * (len(gone) + 1)
    assert db.delete_message(ids[1], include_device=True) and not db.delete_message(ids[1], include_device=True)
    who = names[recv[2]]
    mine = [ids[i] for i in range(n) if recv[i] == recv[2] and i % 3 and i != 1]
    got = db.receive_matching(who, message_ids=mine[::2] + [ids[0]])
    assert [g.id for g in got] == mine[::2] and all(g.id in db.messages for g in got)
    assert [g.id for g in db.receive_messages(who, max_messages=1000) if g.id in at] == mine[1::2]
    db.close()
