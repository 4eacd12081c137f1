"""Filtered receive on the device (sdb_receive_where) against the CPU oracle, byte for byte.

The oracle side is tests/where_ref.py: every record is decided in plain Python, the matches are selected with the
capacity rule, and the survivors are replayed into a fresh oracle.  After every call the counts, every header field and
the padded payloads are compared, and so are stats()["delivered"] and agent_loads(); afterwards every receive path
must deliver what the oracle delivers.
"""
import numpy as np
import pytest

from tests.test_gpu_compact_receive import Rig, _same
from tests.where_ref import WhereOracle, content_bytes, fold_ascii

pytestmark = pytest.mark.gpu

ALPHA = np.frombuffer(b"abcdeABCDE\xc3\xa9\xc3\x89 {}\"", np.uint8)


def _payloads(rng, n, max_len, typ):
    """Payloads over a small alphabet (so that short keywords hit), non-ASCII bytes included.  Records typed
    TYPEF_EXTRAS carry a plausible content length in their first 4 bytes 70 % of the time, a bogus one otherwise."""
    lens = rng.integers(0, max_len + 1, n).astype(np.uint16)
    stride = (max_len + 31) & ~31
    buf = rng.choice(ALPHA, n * stride + 64).astype(np.uint8)
    for i in np.nonzero(typ & 0x10)[0]:
        if lens[i] >= 4 and rng.random() < 0.7:
            buf[i * stride:i * stride + 4] = np.frombuffer(np.uint32(rng.integers(0, int(lens[i]) - 3)).tobytes(), np.uint8)
    return lens, np.arange(n, dtype=np.uint64) * stride, buf


def _types(rng, n):
    return (rng.integers(0, 7, n) | rng.choice([0, 0x08, 0x10, 0x18], n)).astype(np.uint8)


def _traffic(rig, rounds=1):
    """p2p, shared-layout group and broadcast sends with random types, priorities and timestamps."""
    rng = rig.rng
    for _ in range(rounds):
        n = 400
        s, r, prio, typ = rng.integers(0, rig.A, n), rng.integers(0, rig.A, n), rng.integers(0, 4, n), _types(rng, n)
        lens, off, buf = _payloads(rng, n, 200, typ)
        ts = rng.uniform(0, 10, n)
        base = rig.c.send_batch(s, r, prio, typ, lens, off, buf, ts)
        assert rig.g.send_batch(s, r, prio, typ, lens, off, buf, ts) == base
        n = 300
        s, grp = rng.integers(rig.G * rig.F, rig.A, n), rng.integers(0, rig.G, n)
        prio, typ = rng.integers(0, 4, n), _types(rng, n)
        lens, off, buf = _payloads(rng, n, 256, typ)
        ts = rng.uniform(0, 10, n)
        base = rig.c.send_group_batch(s, grp, prio, typ, lens, off, buf, ts)[0]
        assert rig.g.send_group_batch(s, grp, prio, typ, lens, off, buf, ts) == base
        n = 6
        lists = [rng.choice(rig.A, size=int(rng.integers(1, 200)), replace=False) for _ in range(n)]
        lo = np.zeros(n + 1, np.uint64); lo[1:] = np.cumsum([len(x) for x in lists])
        li = np.concatenate(lists).astype(np.uint32)
        s, prio, typ = rng.integers(0, rig.A, n), rng.integers(0, 4, n), _types(rng, n)
        lens, off, buf = _payloads(rng, n, 200, typ)
        ts = rng.uniform(0, 10, n)
        base = rig.c.send_list_batch(s, lo, li, prio, typ, lens, off, buf, ts)
        assert rig.g.send_list_batch(s, lo, li, prio, typ, lens, off, buf, ts) == base


def _rig(rng, **kw):
    rig = Rig(rng, **kw)
    rig.check_advance = False
    rig.c = WhereOracle(rig.c, rig.G, dict(enumerate(rig.members)), rig.A)
    rig.d0 = rig.g.stats()["delivered"]
    return rig


def _check(rig, what):
    """delivered and the per-agent loads against the oracle."""
    assert rig.g.stats()["delivered"] - rig.d0 == rig.c.delivered, what
    lg, lc = rig.g.agent_loads(rig.idx), rig.c.agent_loads(rig.idx)
    for f in ("received", "pending", "pending_by_prio", "pending_granules"):
        assert np.array_equal(lg[f], lc[f]), (what, f)


def _loads_same(g, c, idx, what):
    lg, lc = g.agent_loads(idx), c.agent_loads(idx)
    for f in ("received", "pending", "pending_by_prio", "pending_granules"):
        assert np.array_equal(lg[f], lc[f]), (what, f)


def _where(rig, agents, k, flags, filt, what, rec_cap=(1 << 64) - 1):
    _same(rig.g.receive_where(agents, k, flags, filt), rig.c.receive_where(agents, k, flags, filt, rec_cap=rec_cap), what)
    _check(rig, what)


def _filters(rig, seq_mid):
    from swarmdb_b200._native import NO_GROUP, NO_RECEIVER, make_filter as mf
    s0 = rig.G * rig.F + 5
    return {
        "all": mf(), "sender": mf(sender=s0), "receiver": mf(receiver=17), "broadcast": mf(receiver=NO_RECEIVER),
        "group": mf(group=3), "no_group": mf(group=NO_GROUP), "types": mf(types=[1, 4]), "prio3": mf(prios=[3]),
        "prio02": mf(prios=[0, 2]), "time": mf(after=2.5, before=7.5), "after": mf(after=8.0), "seq": mf(seq=(seq_mid, seq_mid + 5000)),
        "kw": mf(keyword=b"abc"), "kw_icase": mf(keyword=b"aBc", icase=True), "kw_utf8": mf(keyword="é".encode()),
        "kw_icase_utf8": mf(keyword="ÉA".encode(), icase=True), "kw_empty": mf(keyword=b""),
        "group_prio": mf(group=3, prios=[2, 3]), "sender_time_kw": mf(sender=s0, after=1.0, keyword=b"dE", icase=True),
        "types_seq": mf(types=[0, 2, 5], seq=(0, seq_mid)), "broadcast_kw": mf(receiver=NO_RECEIVER, keyword=b"e "),
    }


@pytest.mark.parametrize("shared", ["1", "0"])
def test_every_clause_matches_oracle_then_every_receive_path(shared, monkeypatch):
    from swarmdb_b200._native import RECV_PEEK, RECV_PRIORITY, WHERE_DROP, make_filter
    monkeypatch.setenv("SDB_SHARED_PAYLOAD", shared)
    rng = np.random.default_rng(7)
    rig = _rig(rng, G=8, F=64, extra=64)
    _traffic(rig)
    some = rng.choice(rig.A, 100, replace=False).astype(np.uint32)       # holes: priority receives on some agents
    _same(rig.g.receive_batch(some, 3, RECV_PRIORITY), rig.c.receive_batch(some, 3, RECV_PRIORITY), "holes")
    seq_mid = rig.g.stats()["next_seq"] // 2
    agents = rng.permutation(rig.A).astype(np.uint32)
    for name, filt in _filters(rig, seq_mid).items():
        for flags in (RECV_PEEK, RECV_PEEK | RECV_PRIORITY):
            for k in (3, 1000):
                _where(rig, agents, k, flags, filt, (name, flags, k))
    # the receiver clause maps to one ring: that agent's p2p and group copies, never broadcasts
    f17 = make_filter(receiver=17)
    got = rig.g.receive_where([17], 1000, RECV_PEEK, f17)
    assert (got[1]["receiver"] == 17).all()
    # take mode, both orders; then drop and drop | PEEK
    _where(rig, agents, 5, RECV_PRIORITY, make_filter(group=3, prios=[2, 3]), "take group prio")
    _where(rig, agents, 4, 0, make_filter(keyword=b"ab", icase=True), "take keyword")
    _where(rig, agents[:300], 2, RECV_PRIORITY, make_filter(types=[1, 2, 3]), "take types")
    filt = make_filter(after=4.0, before=6.0)
    peek = rig.g.receive_where(agents, 7, WHERE_DROP | RECV_PEEK, filt, drop=True)
    want = rig.c.receive_where(agents, 7, RECV_PEEK, filt, drop=True)
    assert peek[1] == want[1] and np.array_equal(peek[0], want[0])
    _check(rig, "drop peek")
    got = rig.g.receive_where(agents, 7, WHERE_DROP, filt, drop=True)
    want = rig.c.receive_where(agents, 7, 0, filt, drop=True)
    assert got[1] == want[1] > 0 and np.array_equal(got[0], want[0])
    _check(rig, "drop")
    # every receive path delivers what the oracle delivers after the same calls
    sel = rng.choice(rig.A, 300, replace=False).astype(np.uint32)
    _same(rig.g.receive_batch(sel, 2, RECV_PRIORITY), rig.c.receive_batch(sel, 2, RECV_PRIORITY), "priority pipeline")
    _same(rig.g.receive_batch(sel, 2), rig.c.receive_batch(sel, 2), "stream plan")
    for flags in (0, RECV_PRIORITY):
        _same(rig.g.receive_batch(sel[:8], 3, flags), rig.c.receive_batch(sel[:8], 3, flags), "k_recv_small")
    rig.g.latency_server(True)
    for a in sel[8:20]:
        for flags, k in ((0, 2), (RECV_PRIORITY, 2), (0, 40)):            # fast path, slow path (priority, > 32)
            h, p, _ = rig.g.receive_one(int(a), k, flags)
            _, hc, pc = rig.c.receive_batch([a], k, flags)
            assert h.tobytes() == hc.tobytes() and p.tobytes() == pc.tobytes(), ("latency server", a)
    _where(rig, sel[20:40], 3, 0, make_filter(prios=[1]), "while the server runs")
    rig.g.latency_server(False)
    _check(rig, "paths")
    _same(rig.g.receive_batch(rig.idx, 100000), rig.c.receive_batch(rig.idx, 100000), "drain")
    _check(rig, "drained")
    assert rig.g.queue_stats()["pending"] == 0
    rig.close()


@pytest.mark.parametrize("flags", [0, 1])
def test_max_messages_and_capacity_drains(flags):
    """max_messages at the warp and window thresholds on one deep ring, then capacity through max_recv_records,
    max_recv_payload and each caller buffer, drained call after call: every record arrives exactly once, in order."""
    from swarmdb_b200._native import HDR_DTYPE, RECV_PEEK, make_filter
    rng = np.random.default_rng(11 + flags)
    R = 512
    rig = _rig(rng, G=4, F=64, extra=64, max_recv_records=64, max_recv_payload=48 * 256)
    # agent 7: a full ring of p2p records (holes after a priority receive), agent 9 and others some records
    n = R
    s, prio, typ = rng.integers(0, rig.A, n), rng.integers(0, 4, n), _types(rng, n)
    lens, off, buf = _payloads(rng, n, 200, typ)
    ts = rng.uniform(0, 10, n)
    for r in (np.full(n, 7), rng.choice([9, 10, 11, 12], n)):
        rig.c.send_batch(s, r, prio, typ, lens, off, buf, ts); rig.g.send_batch(s, r, prio, typ, lens, off, buf, ts)
    assert rig.g.agent_loads([7])["pending"][0] == R
    filt = make_filter(prios=[0, 1, 3])
    for k in (1, 8, 9, 31, 32, 33, R - 1, R, 2 * R):
        _where(rig, [7], k, RECV_PEEK | flags, filt, ("k", k), rec_cap=48)
    _same(rig.g.receive_batch([7], 5, 1), rig.c.receive_batch([7], 5, 1), "holes")
    agents = np.array([7, 9, 3, 10, 11, 12], np.uint32)
    filt = make_filter(prios=[0, 1])                                         # each pass drains its own priorities
    for cap, rec_cap in (("device", 48), ("hdr", 10), ("payload", 7)):     # max_recv_payload / 256 binds on the device
        kw = {}
        if cap == "hdr":
            kw["out_hdr"] = np.zeros(10, HDR_DTYPE)
        if cap == "payload":
            kw["out_payload"] = np.zeros(7 * 256, np.uint8)
        want = rig.c.receive_where(agents, 1000, RECV_PEEK | flags, filt)
        got_c, hs, ps, calls = np.zeros(len(agents), np.int64), [], [], 0
        while True:
            c, h, p = rig.g.receive_where(agents, 1000, flags, filt, **kw)
            cc, hc, pc = rig.c.receive_where(agents, 1000, flags, filt, rec_cap=rec_cap)
            _same((c, h, p), (cc, hc, pc), (cap, calls))
            _check(rig, (cap, calls))
            calls += 1
            if len(h) == 0:
                break
            assert c[np.nonzero(c)[0][0]] > 0                              # progress: the lead agent always gives records
            got_c += c; hs.append(h.copy()); ps.append(p.tobytes())
        assert calls > 2 and np.array_equal(got_c, want[0])
        assert np.concatenate(hs).tobytes() == want[1].tobytes() and b"".join(ps) == want[2].tobytes()
        filt = make_filter(prios=[3]) if cap == "device" else make_filter(prios=[2], keyword=b"a")
    _same(rig.g.receive_batch(rig.idx, 64), rig.c.receive_batch(rig.idx, 64), "after")
    rig.close()


def test_keyword_edges():
    """Keyword at the first and last content byte, across 16-byte and staging-chunk boundaries, equal to the content,
    longer than it, 1 and 256 bytes, empty and 65504-byte payloads, EXTRAS slices, ASCII folding and exact non-ASCII."""
    from oracle.cpu_ref import CpuOracle
    from swarmdb_b200._native import RECV_PEEK, SdbError, Shard, make_filter
    rng = np.random.default_rng(3)
    A, L = 4, 65504
    g = Shard(max_agents=A, ring_slots=256, arena_bytes=1 << 24, max_payload_bytes=L, max_recv_records=256,
              max_recv_payload=256 * L)
    c = WhereOracle(CpuOracle(A, 1), 1, watermark=A)
    g.register(np.arange(A, dtype=np.uint32)); c.register(np.arange(A))
    kw = b"Needle"
    bodies = []
    for pos in (0, 10, 11, 14, 15, 16, 1018, 1019, 1020, 1024, 1900, 4096 - 3):
        b = bytearray(rng.choice(ALPHA[:10], 4100).tobytes()); b[pos:pos + len(kw)] = kw
        bodies.append((bytes(b[:pos + len(kw) + int(rng.integers(0, 3))]), 0))      # at / near the last byte too
    long_kw = bytes(rng.choice(ALPHA, 256).tobytes())
    bodies += [(kw, 0), (kw[:-1], 0), (b"", 0), (b"N", 0), (b"nEEDLE", 0), (b"x" * 100 + long_kw, 0), (long_kw[:-1], 0),
               ("É needle é".encode(), 0), (b"a" * (L - 6) + kw, 0), (b"a" * (L - 7) + kw + b"b", 0)]
    ext = lambda content, extras, clen=None: (np.uint32(len(content) if clen is None else clen).tobytes() + content + extras, 0x10)
    bodies += [ext(b"abc", b'{"m":"Needle"}'), ext(b"abcNee", b"dle"), ext(b"Needle", b"{}"), ext(kw, b"", 1 << 30),
               ext(b"xNeedle", b"zz", 3), ((3).to_bytes(4, "little")[:3], 0x10), (b"\x02\x00\x00\x00Ne", 0x10)]
    for body, t in bodies:
        pad = np.frombuffer(body + bytes(64), np.uint8)
        pr = [int(rng.integers(0, 4))]
        for o in (g, c):
            o.send_batch([1], [2], pr, [t], [len(body)], [0], pad)
    filters = [make_filter(keyword=kw), make_filter(keyword=kw, icase=True), make_filter(keyword=b"N"),
               make_filter(keyword=b"n", icase=True), make_filter(keyword=long_kw), make_filter(keyword=long_kw, icase=True),
               make_filter(keyword="é".encode(), icase=True), make_filter(keyword="É".encode()),
               make_filter(keyword=b"ee", icase=True), make_filter(keyword=b"needle \xc3", icase=True)]
    for filt in filters:
        for flags in (RECV_PEEK, RECV_PEEK | 1):
            cg, hg, pg = g.receive_where([2], 1000, flags, filt)
            cc, hc, pc = c.receive_where([2], 1000, flags, filt)
            assert np.array_equal(cg, cc) and hg.tobytes() == hc.tobytes() and pg.tobytes() == pc.tobytes()
            _loads_same(g, c, np.arange(A), "keyword peek")
    # the brute force agrees with the reference on what it found
    _, hc, pc = c.receive_where([2], 1000, RECV_PEEK, filters[1])
    off = 0
    for h in hc:
        n = (int(h["len"]) + 31) & ~31
        assert fold_ascii(kw) in fold_ascii(content_bytes(h, pc[off:off + n].tobytes())); off += n
    assert len(hc) >= 12
    cg, hg, pg = g.receive_where([2], 1000, 0, filters[0])
    cc, hc, pc = c.receive_where([2], 1000, 0, filters[0])
    assert np.array_equal(cg, cc) and hg.tobytes() == hc.tobytes() and pg.tobytes() == pc.tobytes()
    _loads_same(g, c, np.arange(A), "keyword take")
    assert g.stats()["delivered"] == c.delivered
    cg, hg, pg = g.receive_batch([2], 1000)
    cc, hc, pc = c.receive_batch([2], 1000)
    assert np.array_equal(cg, cc) and hg.tobytes() == hc.tobytes() and pg.tobytes() == pc.tobytes()
    # refusals
    bad = make_filter(keyword=b"x" * 257)
    for args in (dict(filt=bad), dict(filt=make_filter(), flags=4), dict(filt=make_filter(), flags=64),
                 dict(agents=[1, 2, 1]), dict(agents=[A])):
        with pytest.raises(SdbError) as e:
            a = args.pop("agents", [2])
            g.receive_where(a, 10, args.pop("flags", 0), args.pop("filt", make_filter()))
        assert e.value.code == -1, args
    f = make_filter(); f.struct_bytes = 60
    f2 = make_filter(); f2.fields = 512
    f3 = make_filter(); f3.fields = 128; f3.keyword_len = 3
    for ff in (f, f2, f3):
        with pytest.raises(SdbError) as e:
            g.receive_where([2], 10, 0, ff)
        assert e.value.code == -1
    import ctypes
    cnt = np.zeros(1, np.uint32); hdr = np.zeros(4, np.uint8)
    rc = g._L.sdb_receive_where(g._h, 1, np.array([2], np.uint32).ctypes.data_as(ctypes.c_void_p), 10, 32,
                                ctypes.byref(make_filter()), cnt.ctypes.data_as(ctypes.c_void_p),
                                hdr.ctypes.data_as(ctypes.c_void_p), 1, None, 0, None, None)
    assert rc == -1                                                          # drop mode with an output buffer
    with pytest.raises(SdbError) as e:
        g.receive_where([2], 10, 0, make_filter(), out_hdr=np.zeros(0, dtype=[("x", "V32")]))
    assert e.value.code == -8
    g.digest_reset()
    g.receive_batch(np.array([0, 1], np.uint32), 1, copy_out=False)
    g.digest_fold()                                                          # a bulk receive folds ...
    g.receive_where([0, 1], 10, 0, make_filter(prios=[0]))
    with pytest.raises(SdbError) as e:                                       # ... a filtered one leaves nothing to fold
        g.digest_fold()
    assert e.value.code == -1
    g.close(); c.close()


@pytest.mark.parametrize("shape", ["wrap", "full", "handle_wrap"])
def test_window_shapes(shape):
    from oracle.cpu_ref import CpuOracle
    from swarmdb_b200._native import RECV_PEEK, RECV_PRIORITY, Shard, make_filter
    rng = np.random.default_rng(["wrap", "full", "handle_wrap"].index(shape))
    A, R = 64, 64
    g = Shard(max_agents=A, ring_slots=R, arena_bytes=1 << 22, max_payload_bytes=256)
    c = WhereOracle(CpuOracle(A, 1), 1, watermark=A)
    g.register(np.arange(A, dtype=np.uint32)); c.register(np.arange(A))
    d0 = g.stats()["delivered"]
    if shape == "handle_wrap":
        g.debug_set_arena_pos((1 << 32) - 300)
    idx = np.arange(A, dtype=np.uint32)
    rounds = {"wrap": 5, "full": 1, "handle_wrap": 6}[shape]
    for k in range(rounds):
        n = R * A // 4 if shape != "full" else R * A             # ~16 per agent and round: the heads wrap, no ring fills
        s, r = rng.integers(0, A, n), (np.repeat(idx, R) if shape == "full" else rng.integers(0, A, n))
        prio, typ = rng.integers(0, 4, n), _types(rng, n)
        lens, off, buf = _payloads(rng, n, 200, typ)
        ts = rng.uniform(0, 10, n)
        c.send_batch(s, r, prio, typ, lens, off, buf, ts); g.send_batch(s, r, prio, typ, lens, off, buf, ts)
        for filt, flags, kk in ((make_filter(prios=[3]), RECV_PRIORITY, 3), (make_filter(keyword=b"ab"), 0, 5),
                                (make_filter(types=[2, 3], after=3.0), RECV_PEEK, 100)):
            cg, hg, pg = g.receive_where(idx, kk, flags, filt)
            cc, hc, pc = c.receive_where(idx, kk, flags, filt)
            assert np.array_equal(cg, cc) and hg.tobytes() == hc.tobytes() and pg.tobytes() == pc.tobytes(), (shape, k)
            _loads_same(g, c, idx, (shape, k))
            assert g.stats()["delivered"] - d0 == c.delivered, (shape, k)
        if shape == "full":
            assert g.agent_loads(idx)["pending"].max() > 0
        cg, hg, pg = g.receive_batch(idx, R // 3, RECV_PRIORITY if k % 2 else 0)
        cc, hc, pc = c.receive_batch(idx, R // 3, RECV_PRIORITY if k % 2 else 0)
        assert hg.tobytes() == hc.tobytes() and pg.tobytes() == pc.tobytes()
    assert g.stats()["ring_overflow"] == 0
    if shape == "handle_wrap":
        assert g.stats()["arena_tail_bytes"] > (1 << 32) * 32
    assert g.stats()["delivered"] - d0 == c.delivered
    cg, hg, pg = g.receive_batch(idx, 1000)
    cc, hc, pc = c.receive_batch(idx, 1000)
    assert hg.tobytes() == hc.tobytes() and pg.tobytes() == pc.tobytes()
    g.close(); c.close()


def test_owned_agents_of_a_sharded_handle():
    """SDB_RECV_OWNED on sharded handles (two shards on one GPU, group traffic imported from both ranks' wire batches):
    each shard's PEEK, take and drop over its own agents equal the oracle's over the same agents; counts come back one
    per owned agent."""
    from oracle.cpu_ref import CpuOracle
    from swarmdb_b200._native import RECV_OWNED, RECV_PEEK, RECV_PRIORITY, WHERE_DROP, make_filter
    from tests.test_gpu_xshard import _async_cluster
    rng = np.random.default_rng(23)
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
    o = WhereOracle(o, G, dict(enumerate(groups)), A)
    for r in range(world):
        sender, grp, prio, typ = rng.integers(0, A, S), rng.integers(0, G, S), rng.integers(0, 4, S), _types(rng, S)
        lens, off, buf = _payloads(rng, S, 256, typ)
        ts = rng.uniform(0, 10, S)
        shards[r].export_group_batch(sender, grp, prio, typ, lens, off, buf, bufs[1][r], wb, ts)
        shards[r].wire_publish(bufs[1][r], wb, 1)
        o.send_group_batch(sender, grp, prio, typ, lens, off, buf, ts)
    for s in shards:
        s.import_wire_ptrs_async(bufs[1], wb, 1)
    for r, s in enumerate(shards):
        local = np.nonzero(smap == r)[0].astype(np.uint32)
        d0, taken = s.stats()["delivered"], 0
        for filt, flags, k in ((make_filter(prios=[2, 3]), RECV_PEEK | RECV_PRIORITY, 3),
                               (make_filter(keyword=b"ab", icase=True), RECV_PEEK, 1000),
                               (make_filter(types=[1, 2]), RECV_PRIORITY, 2)):
            cg, hg, pg = s.receive_where(None, k, RECV_OWNED | flags, filt)
            cc, hc, pc = o.receive_where(local, k, flags, filt)
            assert len(cg) == len(local) and np.array_equal(cg, cc), (r, k)
            assert hg.tobytes() == hc.tobytes() and pg.tobytes() == pc.tobytes(), (r, k)
            _loads_same(s, o, local, (r, k))
            taken += 0 if flags & RECV_PEEK else len(hg)
        cnt, total = s.receive_where(None, 1, RECV_OWNED, make_filter(after=5.0), drop=True)
        cc, tc = o.receive_where(local, 1, 0, make_filter(after=5.0), drop=True)
        assert len(cnt) == len(local) and np.array_equal(cnt, cc) and total == tc > 0
        _loads_same(s, o, local, (r, "drop"))
        assert s.stats()["delivered"] - d0 == taken > 0                  # the take counts, PEEKs and the drop do not
        cg, hg, pg = s.receive_batch(None, 1000, RECV_OWNED)
        cc, hc, pc = o.receive_batch(local, 1000)
        assert np.array_equal(cg, cc) and hg.tobytes() == hc.tobytes() and pg.tobytes() == pc.tobytes(), r
    for s in shards:
        s.close()
    o.close()


def test_c2_backlog_peek_queries_match_oracle():
    """The 1M-agent c2 backlog (4,194,304 pending records): PEEK group-clause and keyword queries over every agent
    against the oracle's PEEK of the whole queue, filtered in numpy."""
    from bench import Workload
    from oracle.cpu_ref import CpuOracle
    from swarmdb_b200._native import RECV_PEEK, Shard, make_filter, payload_offsets
    wl = Workload()
    g = Shard(max_agents=wl.A, ring_slots=64, arena_bytes=1 << 31, max_payload_bytes=wl.L, max_groups=wl.G,
              member_pool_entries=wl.A + 1024, max_batch_sends=wl.S, max_batch_payload=wl.S * wl.L,
              max_recv_records=1 << 23, max_recv_payload=(1 << 23) * wl.L)
    o = CpuOracle(wl.A, wl.G)
    g.register(np.arange(wl.A, dtype=np.uint32)); o.register(np.arange(wl.A))
    for k in range(wl.G):
        g.create_group(k, wl.members(k)); o.create_group(k, wl.members(k))
    b = wl.batch()
    g.send_group_batch(*b); o.send_group_batch(*b)
    idx = np.arange(wl.A, dtype=np.uint32)
    cc, hc, pc = o.receive_batch(idx, 100, RECV_PEEK, rec_cap=wl.S * wl.F, pay_cap=wl.S * wl.F * ((wl.L + 31) & ~31))
    assert len(hc) == wl.S * wl.F
    owner = np.repeat(idx, cc.astype(np.int64))
    poff = payload_offsets(hc)
    grp = int(b[1][0])
    keep = hc["group"] == grp
    cg, hg, pg = g.receive_where(None, 100, RECV_PEEK, make_filter(group=grp))
    assert np.array_equal(cg, np.bincount(owner[keep], minlength=wl.A)[: len(cg)])
    assert hg.tobytes() == hc[keep].tobytes()
    want_pay = b"".join(pc[int(poff[i]):int(poff[i]) + ((int(hc["len"][i]) + 31) & ~31)].tobytes() for i in np.nonzero(keep)[0])
    assert pg.tobytes() == want_pay
    # keyword: 8 bytes taken from one send's payload, ASCII-folded; decided per distinct payload in Python
    sender, group, prio, typ, lens, off, pay = b
    p0 = pay[int(off[0]):int(off[0]) + int(lens[0])].tobytes()
    kw = p0[10:18] if len(p0) >= 18 else p0
    per_send = np.array([fold_ascii(kw) in fold_ascii(pay[int(off[i]):int(off[i]) + int(lens[i])].tobytes())
                         for i in range(wl.S)])
    seq_send = (hc["seq"].astype(np.int64) - int(hc["seq"].min())) // wl.F
    keep = per_send[seq_send]
    cg, hg, pg = g.receive_where(None, 100, RECV_PEEK, make_filter(keyword=kw, icase=True))
    assert keep.sum() > 0 and np.array_equal(cg, np.bincount(owner[keep], minlength=wl.A)[: len(cg)])
    assert hg.tobytes() == hc[keep].tobytes()
    g.close(); o.close()
