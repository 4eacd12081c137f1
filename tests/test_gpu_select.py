"""Filtered and leased receives by byte and token budget (sdb_receive_where_budget, sdb_receive_leased_select).

The header promises that each call is the existing call (sdb_receive_where, sdb_receive_leased) with every agent's
max_messages lowered to its take over the matching records.  Twin handles take the same traffic: point-to-point sends,
shared-payload group sends and broadcast lists, tagged (TYPEF_TOKENS) and untagged records, lengths 0 to
max_payload_bytes, all four priorities.  One twin runs the new call; the other replays each agent's take, computed by
tests/select_ref.py from a PEEK of its matches, through the existing call.  Results must be byte-identical, and so must
what is left queued.
"""
import numpy as np
import pytest

from tests.budget_ref import pad32
from tests.select_ref import take
from tests.tokens_ref import weight

pytestmark = pytest.mark.gpu

P = 512
A = 600                  # request slots on both sides of two 256-slot plan tile boundaries
G, F = 5, 32
RING = 256
TOK = 0x40


def _shards(n=2, a=A, ring=RING, **kw):
    from swarmdb_b200._native import Shard
    kw.setdefault("max_recv_records", 1 << 15)
    kw.setdefault("max_recv_payload", 16 << 20)
    return [Shard(max_agents=a, ring_slots=ring, max_payload_bytes=P, max_groups=G, max_batch_sends=4096, **kw)
            for _ in range(n)]


def _pad16(x):
    return (x.astype(np.uint64) + 15) & ~np.uint64(15)


def _payloads(rng, lens, tag_frac=0.7):
    """16-byte aligned images, offsets and type bytes; tagged records start with a random u32 count, a few near 2^32."""
    n = len(lens)
    off = np.zeros(n, np.uint64)
    np.cumsum(_pad16(lens[:-1]), out=off[1:])
    pay = rng.integers(97, 123, int(_pad16(lens).sum()) + 16, dtype=np.uint8)
    typ = np.where(rng.random(n) < tag_frac, TOK, 0).astype(np.uint8) | rng.integers(0, 7, n).astype(np.uint8)
    cnt = np.where(rng.random(n) < 0.03, rng.integers(1 << 31, 1 << 32, n), rng.integers(0, 300, n)).astype(np.uint32)
    for i in np.flatnonzero((typ & TOK) != 0):
        pay[int(off[i]):int(off[i]) + 4] = np.frombuffer(int(cnt[i]).to_bytes(4, "little"), np.uint8)
    return off, pay, typ


def _traffic(shards, rng, a=A, rounds=2, n=1200):
    members = [rng.choice(a, F, replace=False).astype(np.uint32) for _ in range(G)]
    for s in shards:
        s.register(np.arange(a, dtype=np.uint32))
        for g, m in enumerate(members):
            s.create_group(g, m)
    for _ in range(rounds):
        recv = np.where(rng.random(n) < 0.3, rng.integers(0, 12, n), rng.integers(0, a, n)).astype(np.uint32)
        lens = rng.choice([0, 1, 4, 5, 31, 32, 33, 100, 200, P - 1, P], n).astype(np.uint16)
        prio = rng.integers(0, 4, n).astype(np.uint8)
        off, pay, typ = _payloads(rng, lens)
        send = rng.integers(0, 8, n).astype(np.uint32)
        k = 20
        glens = rng.choice([4, 64, 300, P], k).astype(np.uint16)
        goff, gpay, gtyp = _payloads(rng, glens)
        gsend, grp = rng.integers(0, 8, k).astype(np.uint32), rng.integers(0, G, k).astype(np.uint32)
        gprio = rng.integers(0, 4, k).astype(np.uint8)
        m = 30
        lsz = rng.integers(0, 25, m)
        lo = np.zeros(m + 1, np.uint64); lo[1:] = np.cumsum(lsz)
        lidx = np.concatenate([rng.choice(a, int(z), replace=False) for z in lsz]).astype(np.uint32)
        llens = rng.choice([2, 8, 100, P], m).astype(np.uint16)
        loff, lpay, ltyp = _payloads(rng, llens)
        lsend, lprio = rng.integers(0, 8, m).astype(np.uint32), rng.integers(0, 4, m).astype(np.uint8)
        for s in shards:
            s.send_batch(send, recv, prio, typ, lens, off, pay, np.arange(n, dtype=np.float64))
            s.send_group_batch(gsend, grp, gprio, gtyp, glens, goff, gpay, np.arange(k, dtype=np.float64))
            s.send_list_batch(lsend, lo, lidx, lprio, ltyp, llens, loff, lpay, np.arange(m, dtype=np.float64))


def _filters(kind):
    from swarmdb_b200._native import make_filter
    if kind == "header":
        return make_filter(types=[0, 2, 3], prios=[1, 2, 3])
    if kind == "sender":
        return make_filter(sender=3)
    if kind == "keyword":
        return make_filter(keyword=b"q", icase=True)
    return None


def _costs(shard, agents, flags, filt):
    """(length, weight) of each listed agent's matches in delivery order: a PEEK of the existing filtered call."""
    from swarmdb_b200._native import RECV_PEEK, make_filter, payload_offsets
    cnt, hdr, pay = shard.receive_where(agents, 1 << 14, (flags & 1) | RECV_PEEK, filt or make_filter())
    offs, raw, out, pos = payload_offsets(hdr), pay.tobytes(), [], 0
    for c in cnt.astype(int):
        out.append([(int(hdr["len"][i]), weight(int(hdr["type"][i]), raw[int(offs[i]):int(offs[i]) + int(hdr["len"][i])]))
                    for i in range(pos, pos + c)])
        pos += c
    return out


def _queues(shard, agents):
    """Everything left queued, in both orders (PEEKs), and the counters."""
    from swarmdb_b200._native import RECV_PEEK, RECV_PRIORITY
    out = []
    for fl in (0, RECV_PRIORITY):
        c, h, p = shard.receive_batch(agents, RING, fl | RECV_PEEK)
        out.append((c.tobytes(), h.tobytes(), p.tobytes()))
    loads = shard.agent_loads()
    return out, shard.stats()["delivered"], [loads[f].tobytes() for f in loads.dtype.names]


def _replay_where(shard, agents, counts, flags, filt, drop=False):
    """Each agent's take through the existing filtered call with max_messages set to it."""
    from swarmdb_b200._native import make_filter
    hs, ps = [], []
    for a, k in zip(agents, counts):
        if k == 0:
            continue
        if drop:
            c, t = shard.receive_where([int(a)], int(k), flags, filt or make_filter(), drop=True)
            assert t == k
            continue
        c, h, p = shard.receive_where([int(a)], int(k), flags, filt or make_filter())
        assert len(h) == k
        hs.append(h.copy()); ps.append(p.tobytes())
    return (np.concatenate(hs).tobytes() if hs else b""), b"".join(ps)


LIMITS = {"bytes": (700, 0), "tokens": (0, 500), "both": (1500, 350)}


@pytest.mark.parametrize("prio", [0, 1], ids=["stream", "priority"])
@pytest.mark.parametrize("limits", list(LIMITS))
@pytest.mark.parametrize("mode", ["peek", "take", "drop"])
def test_filtered_budget_equals_replay(prio, limits, mode):
    from swarmdb_b200._native import RECV_PEEK
    rng = np.random.default_rng(100 + 7 * prio + 3 * list(LIMITS).index(limits))
    tw = _shards()
    _traffic(tw, rng)
    nb, nt = LIMITS[limits]
    flags = prio | (RECV_PEEK if mode == "peek" else 0)
    agents = np.sort(rng.choice(A, 400, replace=False)).astype(np.uint32)
    for step, kind in enumerate(["header", "sender", "keyword", None]):
        filt = _filters(kind)
        costs = _costs(tw[1], agents, prio, filt)
        want = [take(c, 6, nb, nt) for c in costs]
        if mode == "drop":
            got, total = tw[0].receive_where(agents, 6, flags, filt, drop=True, max_agent_bytes=nb, max_agent_tokens=nt)
            assert total == sum(want)
        else:
            got, hdr, pay = tw[0].receive_where(agents, 6, flags, filt, max_agent_bytes=nb, max_agent_tokens=nt)
        assert got.tolist() == want, (kind, step)
        h2, p2 = _replay_where(tw[1], agents, want, flags, filt, drop=mode == "drop")
        if mode != "drop":
            assert hdr.tobytes() == h2 and pay.tobytes() == p2
        assert _queues(tw[0], agents) == _queues(tw[1], agents)
    for s in tw:
        s.close()


def test_ids_and_limits_zero():
    """id_hits / id_agent count the matches before the cut; both limits 0 is the existing call byte for byte."""
    from swarmdb_b200._native import RECV_PEEK, RECV_PRIORITY, make_filter
    rng = np.random.default_rng(5)
    tw = _shards()
    _traffic(tw, rng)
    agents = np.arange(A, dtype=np.uint32)
    _, hdr, _ = tw[1].receive_batch(agents, RING, RECV_PEEK)
    ids = rng.choice(np.unique(hdr["seq"]), 300, replace=False).astype(np.uint64)
    filt = make_filter(ids=ids)
    hits = [np.zeros(len(ids), np.uint32) for _ in range(2)]
    first = [np.zeros(len(ids), np.uint32) for _ in range(2)]
    c0, h0, p0 = tw[0].receive_where(agents, 4, RECV_PRIORITY, filt, id_hits=hits[0], id_agent=first[0],
                                     max_agent_tokens=1)
    costs = _costs(tw[1], agents, RECV_PRIORITY, filt)
    assert c0.tolist() == [take(c, 4, 0, 1) for c in costs]
    c1, h1, p1 = tw[1].receive_where(agents, 4, RECV_PRIORITY | RECV_PEEK, filt, id_hits=hits[1], id_agent=first[1])
    assert np.array_equal(hits[0], hits[1]) and np.array_equal(first[0], first[1])
    _replay_where(tw[1], agents, c0.tolist(), RECV_PRIORITY, filt)
    assert _queues(tw[0], agents) == _queues(tw[1], agents)
    # limits 0: sdb_receive_where itself
    filt = make_filter(prios=[0, 3])
    a0 = tw[0].receive_where(agents, 3, 0, filt, max_agent_bytes=0, max_agent_tokens=0)
    a1 = tw[1].receive_where(agents, 3, 0, filt)
    assert all(x.tobytes() == y.tobytes() for x, y in zip(a0, a1))
    for s in tw:
        s.close()


def _one_agent(ring=4096, n_agents=4):
    return _shards(2, a=n_agents, ring=ring, max_recv_records=1 << 14)


def _send(shards, recv, lens, prio, typ, counts, sender=None):
    n = len(lens)
    lens = np.asarray(lens, np.uint16)
    off = np.zeros(n, np.uint64)
    np.cumsum(_pad16(lens[:-1]), out=off[1:])
    pay = np.full(int(_pad16(lens).sum()) + 16, 120, np.uint8)
    typ = np.asarray(typ, np.uint8)
    for i in range(n):
        if typ[i] & TOK:
            pay[int(off[i]):int(off[i]) + 4] = np.frombuffer(int(counts[i]).to_bytes(4, "little"), np.uint8)
    snd = np.zeros(n, np.uint32) if sender is None else np.asarray(sender, np.uint32)
    for s in shards:
        s.send_batch(snd, np.asarray(recv, np.uint32), np.asarray(prio, np.uint8), typ, lens, off, pay,
                     np.arange(n, dtype=np.float64))


@pytest.mark.parametrize("prio", [0, 1], ids=["stream", "priority"])
def test_edges_of_the_take(prio):
    """A first match heavier than the limit, limits met exactly, a cut inside a priority level, matches sparse after
    more than 1,000 non-matches in a window that wraps the ring and spans many warp steps."""
    from swarmdb_b200._native import RECV_PEEK, make_filter
    tw = _one_agent()
    for s in tw:
        s.register(np.arange(4, dtype=np.uint32))
    # move the ring's head near its end so the window wraps
    _send(tw, [0] * 3000, [8] * 3000, [0] * 3000, [0] * 3000, [0] * 3000)
    for s in tw:
        s.receive_batch([0], 3000, 0)
    rng = np.random.default_rng(prio)
    n = 3500
    sender = np.where(np.arange(n) < 1200, 1, np.where(rng.random(n) < 0.1, 2, 1))     # matches: sender 2, sparse
    lens = rng.choice([0, 4, 32, 33, 256, P], n)
    pr = rng.integers(0, 4, n)
    cnt = rng.integers(0, 50, n)
    cnt[1200:1260] = 10
    typ = np.full(n, TOK)
    _send(tw, [0] * n, lens, pr, typ, cnt, sender)
    filt = make_filter(sender=2)
    costs = _costs(tw[1], [0], prio, filt)[0]
    assert len(costs) > 100
    b0, t0 = pad32(costs[0][0]), costs[0][1]
    cases = [(1, 0), (0, t0 - 1), (b0, 0), (0, t0), (0, sum(w for _, w in costs[:37])),    # heavier first, met exactly
             (sum(pad32(ln) for ln, _ in costs[:29]), 0), (1 << 40, 1 << 40), (0, 1 << 33), (64 * 32, 200)]
    for nb, nt in cases:
        if nb == 0 and nt == 0:
            continue
        for mm in (RING * 16, 5):
            got, hdr, pay = tw[0].receive_where([0], mm, prio | RECV_PEEK, filt, max_agent_bytes=nb, max_agent_tokens=nt)
            assert got.tolist() == [take(costs, mm, nb, nt)], (nb, nt, mm)
            _, h2, p2 = tw[1].receive_where([0], int(got[0]), prio | RECV_PEEK, filt)
            assert hdr.tobytes() == h2.tobytes() and pay.tobytes() == p2.tobytes()
    # take for real, then the rest must agree
    got, _, _ = tw[0].receive_where([0], 4096, prio, filt, max_agent_tokens=sum(w for _, w in costs[:50]))
    _replay_where(tw[1], [0], got.tolist(), prio, filt)
    assert _queues(tw[0], [0]) == _queues(tw[1], [0])
    for s in tw:
        s.close()


def _leased_shards(n=2, **kw):
    tw = _shards(n, **kw)
    for s in tw:
        s.lease_reserve(1 << 15, 16 << 20)
    return tw


def _expand(res):
    from swarmdb_b200._native import expand_compact
    cnt, ent, snd, pay, base = res
    hdr, full = expand_compact(ent, snd, pay)
    return cnt, hdr, full, base


@pytest.mark.parametrize("prio", [0, 1], ids=["stream", "priority"])
@pytest.mark.parametrize("case", ["filter", "bytes", "tokens", "filter_tokens"])
def test_leased_select_equals_where_budget(prio, case):
    from swarmdb_b200._native import RECV_PEEK, make_filter
    rng = np.random.default_rng(40 + prio)
    tw = _leased_shards()
    _traffic(tw, rng)
    agents = np.sort(rng.choice(A, 300, replace=False)).astype(np.uint32)
    filt = make_filter(prios=[1, 2, 3], types=[0, 1, 2, 4]) if "filter" in case else None
    nb = 900 if case == "bytes" else 0
    nt = 400 if "tokens" in case else 0
    base_next = None
    for _ in range(2):
        cnt, hdr, full, base = _expand(tw[0].receive_leased(agents, 5, 1e18, prio, max_agent_bytes=nb,
                                                            max_agent_tokens=nt, filt=filt))
        if base_next is not None:
            assert base == base_next                                     # lease ids are consecutive
        base_next = base + len(hdr)
        c1, h1, p1 = tw[1].receive_where(agents, 5, prio, filt or make_filter(), max_agent_bytes=nb,
                                         max_agent_tokens=nt)
        assert cnt.tolist() == c1.tolist()
        assert hdr.tobytes() == h1.tobytes() and full.tobytes() == p1.tobytes()
    a, b = _queues(tw[0], agents), _queues(tw[1], agents)
    assert a[0] == b[0]                                                  # what is left queued
    for s in tw:
        s.close()


def test_leased_select_without_limits_is_receive_leased():
    rng = np.random.default_rng(9)
    tw = _leased_shards()
    _traffic(tw, rng)
    agents = np.arange(A, dtype=np.uint32)
    for prio in (1, 0):
        a = tw[0].receive_leased(agents, 4, 123.0, prio, max_agent_bytes=0, max_agent_tokens=0)
        # the binding routes limits 0 and no filter to sdb_receive_leased; call the new entry directly
        b = _leased_select_raw(tw[1], agents, 4, 123.0, prio)
        assert all(x.tobytes() == y.tobytes() for x, y in zip(a[:4], b[:4])) and a[4] == b[4]
    assert _queues(tw[0], agents) == _queues(tw[1], agents)
    for s in tw:
        s.close()


def _leased_select_raw(shard, agents, max_messages, deadline, flags):
    import ctypes as C
    from swarmdb_b200._native import _p
    a, n, counts = shard._agents_arg(agents)
    ent, snd, pay = shard._compact_outputs(None, None, None)
    total, n_sends, pbytes, base = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
    shard._check(shard._L.sdb_receive_leased_select(
        shard._h, n, _p(a), max_messages, 0, 0, None, flags, float(deadline), _p(counts), _p(ent), len(ent), _p(snd),
        len(snd), _p(pay), pay.nbytes, C.cast(C.byref(total), C.c_void_p), C.cast(C.byref(n_sends), C.c_void_p),
        C.cast(C.byref(pbytes), C.c_void_p), C.cast(C.byref(base), C.c_void_p)))
    return counts, ent[: total.value].copy(), snd[: n_sends.value].copy(), pay[: pbytes.value].copy(), int(base.value)


def test_leased_round_trip_and_dead_letter_counts():
    """Ack, nack and sweep: redelivered records keep ids and weights and come back behind pending records; with a
    redelivery limit a record taken again by a filtered leased receive reads delivery count k + 1, and a non-matching
    record's count survives for a later leased receive."""
    from swarmdb_b200._native import LEASE_ACK, LEASE_RENEW, RECV_PEEK, make_filter
    tw = _one_agent(ring=256)
    s = tw[0]
    s.register(np.arange(4, dtype=np.uint32))
    s.lease_reserve(1024, 1 << 20)
    s.lease_set_policy(3, 1024)
    _send([s], [0] * 6, [8, 40, 8, 40, 8, 8], [1] * 6, [TOK] * 6, [5, 6, 7, 8, 9, 10], sender=[1, 2, 1, 2, 1, 1])
    f1, f2 = make_filter(sender=1), make_filter(sender=2)
    # every record delivered once, all nacked and swept back
    _, hdr, _, base = _expand(s.receive_leased([0], 10, 1e18, 0, max_agent_tokens=1000))
    assert len(hdr) == 6
    seqs = hdr["seq"].tolist()
    s.lease_settle(np.arange(base, base + 6, dtype=np.uint64), LEASE_RENEW, float("-inf"))
    assert s.lease_sweep(0.0)[0] == 6
    tokens = s.pending_tokens([0]).tolist()
    assert tokens == [45]
    # a filtered leased receive takes sender 1's first two (tokens 5 + 7 <= 12): delivery count 2
    cnt, hdr, full, base = _expand(s.receive_leased([0], 10, 1e18, 0, max_agent_tokens=12, filt=f1))
    assert hdr["seq"].tolist() == [seqs[0], seqs[2]]
    assert s.lease_deliveries(np.arange(base, base + 2, dtype=np.uint64)).tolist() == [2, 2]
    s.lease_settle(np.arange(base, base + 2, dtype=np.uint64), LEASE_ACK)
    # sender 2's records were not taken: their counts survive for a later leased receive
    cnt, hdr, full, base = _expand(s.receive_leased([0], 10, 1e18, 0, filt=f2))
    assert hdr["seq"].tolist() == [seqs[1], seqs[3]]
    assert s.lease_deliveries(np.arange(base, base + 2, dtype=np.uint64)).tolist() == [2, 2]
    # nack them: they come back behind what is pending, with their ids and weights
    s.lease_settle(np.arange(base, base + 2, dtype=np.uint64), LEASE_RENEW, float("-inf"))
    s.lease_sweep(0.0)
    _, h, _ = s.receive_batch([0], 10, RECV_PEEK)
    assert h["seq"].tolist() == [seqs[4], seqs[5], seqs[1], seqs[3]]
    assert s.pending_tokens([0]).tolist() == [9 + 10 + 6 + 8]
    s.close()
    tw[1].close()


def test_full_store_refuses_and_changes_nothing():
    from swarmdb_b200._native import SdbError, make_filter
    tw = _one_agent(ring=256)
    s = tw[0]
    s.register(np.arange(4, dtype=np.uint32))
    s.lease_reserve(2, 1 << 20)
    _send([s], [0] * 5, [8] * 5, [0] * 5, [TOK] * 5, [1] * 5)
    cnt, hdr, _, _ = _expand(s.receive_leased([0], 10, 1e18, 0, max_agent_tokens=100, filt=make_filter(sender=0)))
    assert len(hdr) == 2
    before = _queues(s, [0])
    led = s.lease_stats()
    for kw in ({"max_agent_tokens": 100}, {"filt": make_filter(sender=0)}, {"max_agent_bytes": 64}):
        with pytest.raises(SdbError) as e:
            s.receive_leased([0], 10, 1e18, 0, **kw)
        assert e.value.code == -6
        assert _queues(s, [0]) == before and s.lease_stats() == led
    s.close()
    tw[1].close()


def test_c2_backlog_tagged():
    """At the c2 scale (131,072 agents, 64-member groups, a million queued records, every send tagged): a filtered
    token-budget PEEK and a leased token-budget take give per-agent counts and records equal to the model computed
    from a full PEEK."""
    from swarmdb_b200._native import RECV_PEEK, Shard, expand_compact, make_filter, payload_offsets
    n_agents, groups, fan = 1 << 17, 2048, 64
    s = Shard(max_agents=n_agents, max_groups=groups, ring_slots=64, max_payload_bytes=256, arena_bytes=1 << 30,
              max_batch_sends=1 << 16, max_recv_records=1 << 22, max_recv_payload=1 << 30)
    s.lease_reserve(1 << 22, 1 << 30)
    rng = np.random.default_rng(2)
    s.register(np.arange(n_agents, dtype=np.uint32))
    perm = rng.permutation(n_agents).astype(np.uint32)
    for g in range(groups):
        s.create_group(g, perm[g * fan:(g + 1) * fan])
    k = 1 << 14
    lens = rng.integers(4, 257, k).astype(np.uint16)
    off = np.arange(k, dtype=np.uint64) * 256
    pay = rng.integers(97, 123, k * 256 + 64).astype(np.uint8)
    cnts = rng.integers(1, 200, k).astype(np.uint32)
    for i in range(k):
        pay[i * 256:i * 256 + 4] = np.frombuffer(int(cnts[i]).to_bytes(4, "little"), np.uint8)
    typ = (TOK | rng.integers(0, 4, k)).astype(np.uint8)
    s.send_group_batch(rng.integers(0, n_agents, k).astype(np.uint32), rng.integers(0, groups, k).astype(np.uint32),
                       rng.integers(0, 4, k).astype(np.uint8), typ, lens, off, pay)
    agents = np.arange(n_agents, dtype=np.uint32)
    filt = make_filter(types=[0, 2])
    cnt, hdr, full = (x.copy() for x in s.receive_where(agents, 64, RECV_PEEK, filt))   # views of reused buffers
    offs, raw, pos, want = payload_offsets(hdr), full.tobytes(), 0, []
    for c in cnt.astype(int):
        recs = [(int(hdr["len"][i]), weight(int(hdr["type"][i]), raw[int(offs[i]):int(offs[i]) + int(hdr["len"][i])]))
                for i in range(pos, pos + c)]
        want.append(take(recs, 64, 0, 300))
        pos += c
    got, h2, p2 = (x.copy() for x in s.receive_where(agents, 64, RECV_PEEK, filt, max_agent_tokens=300))
    assert got.tolist() == want and len(h2) == sum(want)
    first = np.concatenate([[0], np.cumsum(cnt)[:-1]]).astype(np.int64)
    sel = np.concatenate([np.arange(f, f + w) for f, w in zip(first, want)]).astype(np.int64)
    assert h2.tobytes() == hdr[sel].tobytes()
    res = s.receive_leased(agents, 64, 1e18, 0, max_agent_tokens=300, filt=filt)
    h3, p3 = expand_compact(res[1], res[2], res[3])
    assert res[0].tolist() == want and h3.tobytes() == h2.tobytes() and p3.tobytes() == p2.tobytes()
    assert s.lease_stats()["live"] == sum(want)
    s.close()
