"""Receive by token budget (sdb_receive_tokens, sdb_receive_compact_tokens, sdb_pending_tokens) against the model of
tests/tokens_ref.py.

Three twin handles take the same traffic: point-to-point sends (private payload images), shared-layout group sends
and broadcast-list sends, payloads from 0 to max_payload_bytes bytes, all four priorities, three quarters of the
records tagged with TYPEF_TOKENS and a random u32 count (some near 2^32, so sums pass 32 bits; some tagged records
shorter than 4 bytes, which weigh 0), over more agents than one plan tile holds, with holey windows after priority
and filtered receives.  Each step the first twin takes a full-format token call, the second a compact token call,
and the third replays each agent's model take through receive_budget (the equivalence the header promises): counts,
headers, payload bytes, rings, counters and digests must be identical.
"""
import numpy as np
import pytest

from tests.budget_ref import pad32
from tests.tokens_ref import call_counts, weight

pytestmark = pytest.mark.gpu

P = 1024
A = 700                  # plan tiles hold 256 request slots: agents on both sides of two tile boundaries
G, F = 6, 40
RING = 256
TOK = 0x40


def _twins(n=3, **kw):
    from swarmdb_b200._native import Shard
    kw.setdefault("max_recv_records", 1 << 15)
    kw.setdefault("max_recv_payload", 32 << 20)
    return [Shard(max_agents=A, ring_slots=RING, max_payload_bytes=P, max_groups=G, max_batch_sends=4096, **kw)
            for _ in range(n)]


def _pad16(x):
    return (x.astype(np.uint64) + 15) & ~np.uint64(15)


def _tagged(rng, lens, tag_frac=0.75):
    """Payload bytes (16-byte aligned images), offsets and type bytes: tagged records carry a random u32 count."""
    n = len(lens)
    off = np.zeros(n, np.uint64)
    np.cumsum(_pad16(lens[:-1]), out=off[1:])
    pay = rng.integers(0, 256, int(_pad16(lens).sum()) + 16, dtype=np.uint8)
    typ = np.where(rng.random(n) < tag_frac, TOK, 0).astype(np.uint8) | rng.integers(0, 7, n).astype(np.uint8)
    counts = np.where(rng.random(n) < 0.05, rng.integers(1 << 31, 1 << 32, n), rng.integers(0, 513, n)).astype(np.uint32)
    for i in np.flatnonzero((typ & TOK) != 0):
        pay[int(off[i]):int(off[i]) + 4] = np.frombuffer(int(counts[i]).to_bytes(4, "little"), np.uint8)
    return off, pay, typ


def _traffic(shards, rng, rounds=3):
    members = [rng.choice(A, F, replace=False).astype(np.uint32) for _ in range(G)]
    for s in shards:
        s.register(np.arange(A, dtype=np.uint32))
        for g, m in enumerate(members):
            s.create_group(g, m)
    for _ in range(rounds):
        n = 1500
        recv = np.where(rng.random(n) < 0.3, rng.integers(0, 16, n), rng.integers(0, A, n)).astype(np.uint32)
        lens = rng.choice([0, 1, 3, 4, 5, 31, 32, 33, 200, 512, P - 1, P], n).astype(np.uint16)
        prio = rng.integers(0, 4, n).astype(np.uint8)
        off, pay, typ = _tagged(rng, lens)
        send = rng.integers(0, A, n).astype(np.uint32)
        k = 24
        glens = rng.choice([4, 64, 300, P], k).astype(np.uint16)
        goff, gpay, gtyp = _tagged(rng, glens)
        gsend = rng.integers(0, A, k).astype(np.uint32)
        grp = rng.integers(0, G, k).astype(np.uint32)
        gprio = rng.integers(0, 4, k).astype(np.uint8)
        m = 40                                                            # broadcast lists of 0 to 30 recipients
        lsz = rng.integers(0, 31, m)
        lo = np.zeros(m + 1, np.uint64); lo[1:] = np.cumsum(lsz)
        lidx = np.concatenate([rng.choice(A, int(z), replace=False) for z in lsz]).astype(np.uint32)
        llens = rng.choice([2, 8, 100, P], m).astype(np.uint16)
        loff, lpay, ltyp = _tagged(rng, llens)
        lsend = rng.integers(0, A, m).astype(np.uint32)
        lprio = rng.integers(0, 4, m).astype(np.uint8)
        for s in shards:
            s.send_batch(send, recv, prio, typ, lens, off, pay, np.arange(n, dtype=np.float64))
            s.send_group_batch(gsend, grp, gprio, gtyp, glens, goff, gpay, np.arange(k, dtype=np.float64))
            s.send_list_batch(lsend, lo, lidx, lprio, ltyp, llens, loff, lpay, np.arange(m, dtype=np.float64))


def _holes(shards, rng):
    """Holey windows: a priority receive of two records from some agents, a filtered receive of priority-1 records
    from others; the same calls on every twin."""
    from swarmdb_b200._native import RECV_PRIORITY, make_filter
    a1 = np.sort(rng.choice(A, 120, replace=False)).astype(np.uint32)
    a2 = np.sort(rng.choice(A, 120, replace=False)).astype(np.uint32)
    for s in shards:
        s.receive_batch(a1, 2, RECV_PRIORITY)
        s.receive_where(a2, 3, 0, make_filter(prios=[1]))


def _orders(shard, agents, flags):
    """(payload length, token weight) of each listed agent's pending records in delivery order (a PEEK)."""
    from swarmdb_b200._native import RECV_PEEK, payload_offsets
    cnt, hdr, pay = shard.receive_batch(agents, RING, flags | RECV_PEEK)
    offs, raw = payload_offsets(hdr), pay.tobytes()
    out, pos = [], 0
    for c in cnt.astype(int):
        out.append([(int(hdr["len"][i]), weight(int(hdr["type"][i]), raw[int(offs[i]):int(offs[i]) + int(hdr["len"][i])]))
                    for i in range(pos, pos + c)])
        pos += c
    return out


def _replay(shard, agents, counts, nbytes, flags):
    """Each agent's take through receive_budget with max_messages set to it: bytes from a PEEK, then the same call with
    the digests folded."""
    from swarmdb_b200._native import RECV_PEEK
    hs, ps = [], []
    for a, k in zip(agents, counts):
        if k == 0:
            continue
        _, h, p = shard.receive_budget([int(a)], int(k), nbytes, flags | RECV_PEEK)
        assert len(h) == k
        hs.append(h.copy()); ps.append(p.copy())
        if not flags & 2:
            shard.receive_budget([int(a)], int(k), nbytes, flags)
            shard.digest_fold()
    if not hs:
        return None, b""
    return np.concatenate(hs), b"".join(p.tobytes() for p in ps)


def _same_state(a, b):
    assert a.stats()["delivered"] == b.stats()["delivered"]
    la, lb = a.agent_loads(), b.agent_loads()
    for f in la.dtype.names:
        assert np.array_equal(la[f], lb[f]), f
    assert np.array_equal(a.pending_tokens(), b.pending_tokens())


def _step(tw, agents, max_messages, tokens, nbytes, flags, rec_cap=None, byte_cap=None):
    from swarmdb_b200._native import ENTRY_DTYPE, HDR_DTYPE, SEND_DTYPE, expand_compact
    full, cmp_, ref = tw
    orders = _orders(ref, agents, flags & 1)
    rc = rec_cap or full.max_recv_records
    bc = byte_cap or (32 << 20)
    want = call_counts(orders, max_messages, nbytes, tokens, rc, bc)
    cnt, hdr, pay = full.receive_tokens(agents, max_messages, tokens, nbytes, flags,
                                        out_hdr=np.zeros(rc, HDR_DTYPE), out_payload=np.zeros(bc, np.uint8))
    assert list(cnt.astype(int)) == want
    if not flags & 2:
        full.digest_fold()
    ccnt, ent, snd, cpay = cmp_.receive_compact_tokens(agents, max_messages, tokens, nbytes, flags,
                                                       out_entries=np.zeros(rc, ENTRY_DTYPE),
                                                       out_sends=np.zeros(rc, SEND_DTYPE), out_payload=np.zeros(bc, np.uint8))
    assert np.array_equal(ccnt, cnt)
    chdr, cfull = expand_compact(ent, snd, cpay)
    phdr, ppay = _replay(ref, agents, want, nbytes, flags)
    assert len(hdr) == sum(want) == len(chdr)
    if sum(want):
        for f in hdr.dtype.names:
            assert np.array_equal(hdr[f], phdr[f]), f
            assert np.array_equal(chdr[f], phdr[f]), f
    assert pay.tobytes() == ppay == cfull.tobytes()
    assert len(pay) == sum(pad32(x) for x in hdr["len"])
    _same_state(full, ref)
    _same_state(cmp_, ref)
    return want, orders


def _limits(orders, rng):
    """Token limits at, just below and just above prefix sums of a few agents' windows."""
    sums = sorted({int(s) for recs in orders if recs for s in np.cumsum([w for _, w in recs]) if s > 1})
    pick = [sums[int(i)] for i in rng.integers(0, len(sums), 3)] if sums else [5]
    return [x + d for x in pick for d in (-1, 0, 1)]


@pytest.mark.parametrize("priority", [False, True])
@pytest.mark.parametrize("nbytes", [0, 700])
def test_token_calls_match_the_model_and_the_budget_replay(priority, nbytes):
    from swarmdb_b200._native import RECV_PRIORITY
    rng = np.random.default_rng(11 + priority + nbytes)
    tw = _twins()
    try:
        _traffic(tw, rng)
        _holes(tw, rng)
        flags = RECV_PRIORITY if priority else 0
        agents = np.arange(A, dtype=np.uint32)
        orders = _orders(tw[2], agents, flags)
        assert sum(len(o) for o in orders) > 4000 and any(len(o) > 8 for o in orders)
        assert any(w >= (1 << 31) for o in orders for _, w in o)
        for lim in _limits(orders, rng):
            sub = np.sort(rng.choice(A, 400, replace=False)).astype(np.uint32)
            _step(tw, sub, int(rng.choice([3, 50, RING])), lim, nbytes, flags)
        while sum(_step(tw, agents, RING, 700, nbytes, flags)[0]):
            pass
        assert tw[0].agent_loads()["pending"].sum() == 0
        d = [t.digest_read() for t in (tw[0], tw[2])]
        assert np.array_equal(d[0], d[1])
    finally:
        for t in tw:
            t.close()


@pytest.mark.parametrize("priority", [False, True])
def test_capacity_truncation_peek_and_zero_limit(priority):
    from swarmdb_b200._native import RECV_PEEK, RECV_PRIORITY
    rng = np.random.default_rng(5 + priority)
    tw = _twins()
    try:
        _traffic(tw, rng, rounds=2)
        _holes(tw, rng)
        flags = RECV_PRIORITY if priority else 0
        agents = np.arange(A, dtype=np.uint32)
        # PEEK: the same result, nothing retired
        before = [t.agent_loads() for t in tw], tw[0].stats()["delivered"], tw[0].pending_tokens()
        want, _ = _step(tw, agents, RING, 900, 0, flags | RECV_PEEK)
        assert tw[0].stats()["delivered"] == before[1] and np.array_equal(tw[0].pending_tokens(), before[2])
        for t, la in zip(tw, before[0]):
            assert np.array_equal(t.agent_loads(), la)
        got, _ = _step(tw, agents, RING, 900, 0, flags)
        assert got == want
        # the call's record and byte capacity cut the output: an agent first in the output takes a prefix
        _step(tw, agents, RING, 5000, 0, flags, rec_cap=37)
        _step(tw, agents, RING, 1 << 40, 0, flags, rec_cap=1 << 12, byte_cap=P)
        _step(tw, agents[100:], RING, 3000, 4096, flags, rec_cap=300, byte_cap=9000)
        # max_agent_tokens = 0 is the budget call
        for nbytes in (0, 2000):
            c1, h1, p1 = tw[0].receive_tokens(agents, 7, 0, nbytes, flags | RECV_PEEK)
            c1, h1, p1 = c1.copy(), h1.copy(), p1.copy()
            c2, h2, p2 = tw[0].receive_budget(agents, 7, nbytes, flags | RECV_PEEK)
            assert np.array_equal(c1, c2) and h1.tobytes() == h2.tobytes() and p1.tobytes() == p2.tobytes()
        # refused calls leave every queue untouched
        from swarmdb_b200._native import SdbError
        loads = tw[0].agent_loads()
        with pytest.raises(SdbError):
            tw[0].receive_tokens(agents, 7, 100, 0, flags, out_payload=np.zeros(P - 32, np.uint8))
        with pytest.raises(SdbError):
            tw[0].receive_tokens(np.array([3, 3], np.uint32), 7, 100, 0, flags)
        assert np.array_equal(tw[0].agent_loads(), loads)
    finally:
        for t in tw:
            t.close()


def _model_pending(shard):
    return np.array([sum(w for _, w in recs) for recs in _orders(shard, np.arange(A, dtype=np.uint32), 0)], np.uint64)


def test_pending_tokens_survive_restore_relocation_and_redelivery():
    from swarmdb_b200._native import ENTRY_DTYPE, RECV_PEEK, SEND_DTYPE, Shard
    rng = np.random.default_rng(21)
    (a,) = _twins(1, arena_bytes=1 << 26)
    b = None
    try:
        _traffic([a], rng, rounds=2)
        _holes([a], rng)
        want = _model_pending(a)
        assert want.sum() > (1 << 32) and np.array_equal(a.pending_tokens(), want)
        sub = np.array([5, 9, 400], np.uint32)
        assert np.array_equal(a.pending_tokens(sub), want[sub])
        # restore from a snapshot (a PEEK compact receive) on a fresh handle
        cnt, ent, snd, pay = a.receive_compact(None, RING, RECV_PEEK, out_entries=np.zeros(1 << 15, ENTRY_DTYPE),
                                               out_sends=np.zeros(1 << 15, SEND_DTYPE), out_payload=np.zeros(32 << 20, np.uint8))
        (b,) = _twins(1)
        b.register(np.arange(A, dtype=np.uint32))
        b.restore_compact(np.arange(A, dtype=np.uint32), cnt, ent, snd, pay)
        assert np.array_equal(b.pending_tokens(), want)
        # relocation moves every pending record to the arena tail
        s = a.relocate(a.stats()["arena_tail_bytes"])
        assert s["records"] > 0
        assert np.array_equal(a.pending_tokens(), want) and np.array_equal(_model_pending(a), want)
        # a leased receive takes records out of the queues; a sweep redelivers them
        a.lease_reserve(1 << 15, 32 << 20)
        lc, le, ls, lp, _ = a.receive_leased(np.arange(0, A, 3, dtype=np.uint32), 4, 1.0)
        assert len(le) > 0
        assert a.pending_tokens().sum() < want.sum()
        red, _, left = a.lease_sweep(2.0)
        assert red == len(le) and left == 0
        assert np.array_equal(a.pending_tokens(), want) and np.array_equal(_model_pending(a), want)
    finally:
        a.close()
        if b is not None:
            b.close()


def test_keyword_search_skips_the_token_count():
    """The same records with and without TYPEF_TOKENS: a keyword search finds the same ones.  Every count spells the
    keyword's first four bytes, so a kernel that searched the count would find more in the tagged handle."""
    from swarmdb_b200._native import RECV_PEEK, make_filter
    rng = np.random.default_rng(8)
    n = 3000
    kw = b"ab\x00z"
    tagged, plain = _twins(2)
    try:
        for s in (tagged, plain):
            s.register(np.arange(A, dtype=np.uint32))
        bodies, typ_p = [], []
        for i in range(n):
            c = bytes(rng.choice(list(b"abz\x00xy"), int(rng.integers(0, 40))).astype(np.uint8))
            if rng.random() < 0.5:                                         # u32 content length | content | extras
                body = len(c).to_bytes(4, "little") + c + bytes(rng.choice(list(b"ab\x00z"), int(rng.integers(0, 9))).astype(np.uint8))
                typ_p.append(0x10)
            else:
                body = c
                typ_p.append(0)
            bodies.append(body)
        typ_p = np.array(typ_p, np.uint8)
        recv = rng.integers(0, A, n).astype(np.uint32)
        send = rng.integers(0, A, n).astype(np.uint32)
        prio = rng.integers(0, 4, n).astype(np.uint8)
        for s, pre, typ in ((plain, b"", typ_p), (tagged, kw, typ_p | TOK)):
            imgs = [pre + b for b in bodies]
            lens = np.array([len(x) for x in imgs], np.uint16)
            off = np.zeros(n, np.uint64)
            np.cumsum(_pad16(lens[:-1]), out=off[1:])
            buf = np.zeros(int(_pad16(lens).sum()) + 16, np.uint8)
            for o, x in zip(off, imgs):
                buf[int(o):int(o) + len(x)] = np.frombuffer(x, np.uint8)
            s.send_batch(send, recv, prio, typ, lens, off, buf)
        for k in (kw, kw[:2], kw[1:], b"z", b"abz"):
            for icase in (False, True):
                f = make_filter(keyword=k, icase=icase)
                c1, h1, _ = tagged.receive_where(None, RING, RECV_PEEK, f)
                c2, h2, _ = plain.receive_where(None, RING, RECV_PEEK, f)
                assert np.array_equal(c1, c2) and np.array_equal(h1["seq"], h2["seq"]), (k, icase)
        assert c1.sum() > 0
    finally:
        tagged.close(); plain.close()


# ---- the surface -------------------------------------------------------------------------------------------------
def _db(tmp_path, **kw):
    import swarmdb_b200 as sdb
    g = dict(max_agents=64, max_groups=4, ring_slots=256, arena_bytes=1 << 22, deterministic_ids=True)
    g.update(kw)
    return sdb.SwarmsDB(save_dir=str(tmp_path), auto_save=False, gpu_config=sdb.GpuConfig(**g),
                        token_counter=lambda text: len(text.split()))


def _fill(db):
    db.register_agent("b"); db.register_agent("c")
    db.add_agent_group("team", ["a", "b", "c"])
    texts = ["one two three", "four", "five six", "seven eight nine ten", "x", "y z"]
    for i, t in enumerate(texts):
        if i % 3 == 2:
            db.send_to_group("a", "team", t, metadata={"i": i})
        else:
            db.send_message("a", t, "b", metadata={"i": i} if i % 2 else None)
    db.flush()
    return texts


def _check_surface(db, texts):
    assert db.pending_tokens(["b"]) == {"b": sum(len(t.split()) for t in texts)}
    got = db.peek_messages("b", max_tokens=6)
    assert [m.content for m in got] == texts[:3]
    got = db.receive_messages("b", max_tokens=6)
    assert [m.content for m in got] == texts[:3] and [m.token_count for m in got] == [3, 1, 2]
    got = db.receive_messages("b", max_tokens=2)
    assert [m.content for m in got] == texts[3:4]                      # heavier first message alone
    got = db.receive_messages("b", max_tokens=100, max_bytes=32)
    assert [m.content for m in got] == texts[4:5]
    assert [m.content for m in db.receive_messages("b")] == texts[5:]


def test_receive_messages_by_tokens(tmp_path):
    db = _db(tmp_path)
    try:
        texts = _fill(db)
        _check_surface(db, texts)
        assert [m.token_count for m in db.receive_messages("c")] == [2, 2]
    finally:
        db.close()


def test_sharded_front_end_by_tokens(tmp_path):
    import swarmdb_b200 as sdb
    from swarmdb_b200.sharded import ShardedSwarmsDB
    db = ShardedSwarmsDB(0, 1, save_dir=str(tmp_path), auto_save=False, token_counter=lambda text: len(text.split()),
                         gpu_config=sdb.GpuConfig(max_agents=64, max_groups=4, ring_slots=256, arena_bytes=1 << 22))
    try:
        texts = _fill(db)
        _check_surface(db, texts)
    finally:
        db.close()


def test_rest_receive_by_tokens(tmp_path):
    pytest.importorskip("fastapi"); pytest.importorskip("jwt"); pytest.importorskip("httpx")
    from fastapi.testclient import TestClient
    from swarmdb_b200.server import Settings, create_app
    db = _db(tmp_path)
    try:
        c = TestClient(create_app(db, Settings(history_dir=str(tmp_path))))

        def token(user):
            r = c.post("/auth/token", json={"username": user, "password": "pw"})
            return {"Authorization": f"Bearer {r.json()['access_token']}"}
        ha, hb = token("a"), token("b")
        for who, h in (("a", ha), ("b", hb)):
            assert c.post("/agents/register", json={"agent_id": who}, headers=h).status_code == 201
        for t in ("one two", "three four five", "six"):
            assert c.post("/messages", json={"content": t, "receiver_id": "b"}, headers=ha).status_code == 200
        r = c.post("/agents/receive", params={"max_tokens": 4}, headers=hb)
        assert r.status_code == 200 and [m["content"] for m in r.json()] == ["one two"]
        assert c.post("/agents/receive", params={"max_tokens": 0}, headers=hb).status_code == 422
        r = c.post("/agents/receive", params={"max_tokens": 4}, headers=hb)
        assert [m["content"] for m in r.json()] == ["three four five", "six"]
        assert c.post("/agents/receive", headers=hb).json() == []
    finally:
        db.close()


# ---- the c2 scale ------------------------------------------------------------------------------------------------
def _group_take(w, lim):
    """token_take of every group's send list at once: w[g, i] the weight of group g's i-th send in delivery order
    (-1: none)."""
    cum = np.cumsum(np.where(w < 0, 0, w), axis=1)
    fits = (cum <= lim) & (w >= 0)
    take = fits.sum(axis=1)
    return np.where((take == 0) & (w[:, 0] >= 0), 1, take)


@pytest.mark.parametrize("priority", [False, True])
def test_c2_backlog_of_tagged_group_sends(priority):
    """1 M agents, 65,536 group sends of 64 members, every send tagged with a count in 1..512: each agent's take and
    pending sum is its group's, computed from the batch alone; the output's record seqs follow from the take."""
    from bench import Workload
    from swarmdb_b200._native import ENTRY_DTYPE, RECV_PEEK, RECV_PRIORITY, SEND_DTYPE, Shard
    wl = Workload()
    rng = np.random.default_rng(4)
    snd, grp, prio, typ, lens, off, pay = wl.batch(var_len=True)
    lens = np.maximum(lens, 4).astype(np.uint16)
    counts = rng.integers(1, 513, wl.S).astype(np.uint32)
    pay = pay.copy()
    pay.reshape(wl.S, wl.L)[:, :4] = counts.view(np.uint8).reshape(wl.S, 4)
    typ = np.full(wl.S, TOK, np.uint8)
    rec_cap = wl.S * wl.F + (1 << 16)
    s = Shard(max_agents=wl.A, ring_slots=64, arena_bytes=1 << 31, max_payload_bytes=wl.L, max_groups=1 << 14,
              member_pool_entries=wl.A + 1024, max_batch_sends=wl.S, max_batch_payload=wl.S * wl.L,
              max_recv_records=rec_cap, max_recv_payload=rec_cap * wl.L)
    try:
        s.register(np.arange(wl.A, dtype=np.uint32))
        for g in range(wl.G):
            s.create_group(g, wl.members(g))
        base = s.send_group_batch(snd, grp, prio, typ, lens, off, pay)
        flags = RECV_PRIORITY if priority else 0
        # each group's sends in delivery order
        order = np.lexsort((np.arange(wl.S), (-prio.astype(np.int64)) if priority else np.zeros(wl.S), grp))
        per = np.bincount(grp, minlength=wl.G)
        start = np.r_[0, np.cumsum(per)[:-1]]
        width = int(per.max())
        slot = np.arange(wl.S) - np.repeat(start, per)
        idx = np.full((wl.G, width), -1, np.int64)
        idx[grp[order], slot] = order
        w = np.where(idx >= 0, counts[np.maximum(idx, 0)].astype(np.int64), -1)
        gsum = np.where(w < 0, 0, w).sum(axis=1)
        g_of = wl.group_of.astype(np.int64)
        assert np.array_equal(s.pending_tokens(), gsum[g_of].astype(np.uint64))
        rank = np.empty(wl.A, np.int64)                           # member position j: seq = base + F * send + j
        for g in range(wl.G):
            rank[wl.members(g)] = np.arange(wl.F)
        out = dict(out_entries=np.zeros(rec_cap, ENTRY_DTYPE), out_sends=np.zeros(rec_cap, SEND_DTYPE),
                   out_payload=np.zeros(rec_cap * wl.L, np.uint8))            # bytes are counted per record
        for lim in (300, 777, 1500):
            take = _group_take(w, lim)
            cnt, ent, _, _ = s.receive_compact_tokens(None, 64, lim, 0, flags | RECV_PEEK, **out)
            assert np.array_equal(cnt.astype(np.int64), take[g_of])
            k = take[g_of]
            ag = np.repeat(np.arange(wl.A), k)
            pos = np.arange(len(ag)) - np.repeat(np.r_[0, np.cumsum(k)[:-1]], k)
            want = base + wl.F * idx[g_of[ag], pos].astype(np.uint64) + rank[ag].astype(np.uint64)
            assert np.array_equal(ent["seq"], want)
        cnt, ent, _, _ = s.receive_compact_tokens(None, 64, 777, 0, flags, **out)
        left = gsum - np.array([w[g][:t].sum() for g, t in enumerate(_group_take(w, 777))])
        assert np.array_equal(s.pending_tokens(), left[g_of].astype(np.uint64))
    finally:
        s.close()
