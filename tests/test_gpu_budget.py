"""Receive by byte budget (sdb_receive_budget, sdb_receive_compact_budget) against the plain receive.

Three twin handles take the same traffic: point-to-point sends (private payload images) and group sends (one shared
payload per send), payloads from 0 to max_payload_bytes bytes and all four priorities, over more agents than one plan
tile holds, some with more pending records than the plan keeps in registers and some with holey windows (after a
priority receive and a filtered receive).  Each step the first twin takes a full-format budget call, the second a
compact budget call, and the third the plain receive of each listed agent with max_messages set to the take
tests/budget_ref.py computes from a PEEK of the third twin.  Counts, headers and padded payload bytes must be identical,
and so must the rings, counters, digests and the drains that follow.
"""
import numpy as np
import pytest

from tests.budget_ref import call_counts, pad32

pytestmark = pytest.mark.gpu

P = 1024
A = 700                  # plan tiles hold 256 request slots: agents on both sides of two tile boundaries
G, F = 6, 40
RING = 256


def _twins(n=3, **kw):
    from swarmdb_b200._native import Shard
    kw.setdefault("max_recv_records", 1 << 15)
    kw.setdefault("max_recv_payload", 32 << 20)
    return [Shard(max_agents=A, ring_slots=RING, max_payload_bytes=P, max_groups=G, max_batch_sends=4096, **kw)
            for _ in range(n)]


def _traffic(shards, rng, rounds=3):
    members = [rng.choice(A, F, replace=False).astype(np.uint32) for _ in range(G)]
    for s in shards:
        s.register(np.arange(A, dtype=np.uint32))
        for g, m in enumerate(members):
            s.create_group(g, m)
    _rounds(shards, rng, rounds)


def _rounds(shards, rng, rounds):
    for _ in range(rounds):
        n = 2000
        recv = np.where(rng.random(n) < 0.3, rng.integers(0, 16, n), rng.integers(0, A, n)).astype(np.uint32)
        lens = rng.choice([0, 1, 31, 32, 33, 200, 512, P - 1, P], n).astype(np.uint16)
        prio = rng.integers(0, 4, n).astype(np.uint8)
        off = np.zeros(n, np.uint64)
        np.cumsum(_pad16(lens[:-1]), out=off[1:])                  # payload offsets are 16-byte aligned
        pay = rng.integers(0, 256, int(_pad16(lens).sum()), dtype=np.uint8)
        send = rng.integers(0, A, n).astype(np.uint32)
        ts = np.arange(n, dtype=np.float64)
        typ = np.zeros(n, np.uint8)
        k = 24
        glens = rng.choice([0, 64, 300, P], k).astype(np.uint16)
        goff = np.zeros(k, np.uint64)
        np.cumsum(_pad16(glens[:-1]), out=goff[1:])
        gpay = rng.integers(0, 256, int(_pad16(glens).sum()), dtype=np.uint8)
        gsend = rng.integers(0, A, k).astype(np.uint32)
        grp = rng.integers(0, G, k).astype(np.uint32)
        gprio = rng.integers(0, 4, k).astype(np.uint8)
        for s in shards:
            s.send_batch(send, recv, prio, typ, lens, off, pay, ts)
            s.send_group_batch(gsend, grp, gprio, np.zeros(k, np.uint8), glens, goff, gpay, np.arange(k, dtype=np.float64))


def _pad16(x):
    return (x.astype(np.uint64) + 15) & ~np.uint64(15)


def _orders(shard, agents, flags):
    """Payload lengths of each listed agent's pending records in delivery order (a PEEK of the plain receive)."""
    from swarmdb_b200._native import RECV_PEEK
    cnt, hdr, _ = shard.receive_batch(agents, RING, flags | RECV_PEEK)
    ends = np.cumsum(cnt.astype(np.int64))
    return [list(hdr["len"][e - c:e].astype(int)) for c, e in zip(cnt.astype(np.int64), ends)], cnt


def _plain(shard, agents, counts, flags):
    """The plain receive with each agent's max_messages set to its take: bytes from a PEEK, then the same call through
    the bulk path with the digests folded."""
    from swarmdb_b200._native import RECV_PEEK
    hs, ps = [], []
    for a, k in zip(agents, counts):
        if k == 0:
            continue
        _, h, p = shard.receive_batch([int(a)], int(k), flags | RECV_PEEK)
        assert len(h) == k
        hs.append(h.copy()); ps.append(p.copy())
        shard.receive_batch([int(a)], int(k), flags, copy_out=False)      # bulk path: leaves results to fold
        shard.digest_fold()
    if not hs:
        return None, b""
    return np.concatenate(hs), b"".join(p.tobytes() for p in ps)


def _same_state(a, b):
    assert a.stats()["delivered"] == b.stats()["delivered"]
    la, lb = a.agent_loads(), b.agent_loads()
    for f in la.dtype.names:
        assert np.array_equal(la[f], lb[f]), f


def _step(tw, agents, max_messages, budget, flags, rec_cap=None, byte_cap=None, owned=False):
    from swarmdb_b200._native import HDR_DTYPE, RECV_OWNED, expand_compact
    full, cmp_, ref = tw
    listed = agents
    if owned:
        listed = np.flatnonzero(np.asarray(ref._owner) == 0).astype(np.uint32)
    orders, _ = _orders(ref, listed, flags & ~RECV_OWNED)
    rc = rec_cap or full.max_recv_records
    bc = byte_cap or (32 << 20)
    want = call_counts(orders, max_messages, budget, rc, bc)
    hdr_buf = np.zeros(rc, HDR_DTYPE)
    pay_buf = np.zeros(bc, np.uint8)
    cnt, hdr, pay = full.receive_budget(None if owned else agents, max_messages, budget, flags,
                                        out_hdr=hdr_buf, out_payload=pay_buf)
    assert list(cnt.astype(int)) == want
    full.digest_fold()
    ccnt, ent, snd, cpay = cmp_.receive_compact(None if owned else agents, max_messages, flags, max_agent_bytes=budget,
                                                out_entries=np.zeros(rc, _entry_dtype()), out_sends=np.zeros(rc, _send_dtype()),
                                                out_payload=np.zeros(bc, np.uint8))
    assert np.array_equal(ccnt, cnt)
    chdr, cfull = expand_compact(ent, snd, cpay)
    assert len(cpay) <= len(pay)
    phdr, ppay = _plain(ref, listed, want, flags & ~RECV_OWNED)
    assert len(hdr) == sum(want) == len(chdr)
    if sum(want):
        for f in hdr.dtype.names:
            assert np.array_equal(hdr[f], phdr[f]), f
            assert np.array_equal(chdr[f], phdr[f]), f
    assert pay.tobytes() == ppay == cfull.tobytes()
    assert len(pay) == sum(pad32(x) for x in hdr["len"])
    _same_state(full, ref)
    _same_state(cmp_, ref)
    return sum(want)


def _entry_dtype():
    from swarmdb_b200._native import ENTRY_DTYPE
    return ENTRY_DTYPE


def _send_dtype():
    from swarmdb_b200._native import SEND_DTYPE
    return SEND_DTYPE


def _drain_same(tw, flags=0):
    full, cmp_, ref = tw
    outs = []
    for s in tw:
        cnt, hdr, pay = s.receive_batch(None, RING, flags)
        outs.append((cnt.copy(), hdr.copy(), pay.tobytes()))
    for o in outs[:2]:
        assert np.array_equal(o[0], outs[2][0])
        assert o[1].tobytes() == outs[2][1].tobytes()
        assert o[2] == outs[2][2]
    full.digest_fold(); ref.digest_fold()
    assert np.array_equal(full.digest_read(), ref.digest_read())


def _holes(tw, rng):
    """Holey windows on every twin: a priority receive and a filtered receive of a few agents."""
    from swarmdb_b200._native import RECV_PRIORITY, make_filter
    ag = rng.choice(A, 60, replace=False).astype(np.uint32)
    for s in tw:
        s.receive_batch(ag[:30], 3, RECV_PRIORITY, copy_out=False)
        s.receive_where(ag[30:], 2, 0, make_filter(prios=(2, 3)))


@pytest.mark.parametrize("priority", [False, True])
@pytest.mark.parametrize("peek", [False, True])
def test_budget_equals_plain_receive_with_the_take_as_max_messages(priority, peek):
    from swarmdb_b200._native import RECV_PEEK, RECV_PRIORITY
    rng = np.random.default_rng(11 + 2 * priority + peek)
    tw = _twins()
    try:
        _traffic(tw, rng)
        for s in tw:
            s.digest_reset()
        _holes(tw, rng)
        flags = (RECV_PRIORITY if priority else 0) | (RECV_PEEK if peek else 0)
        agents = rng.permutation(A).astype(np.uint32)
        # small takes first, so that a take-all step does not leave the later ones an empty queue
        for mm, budget in ((3, 33), (9, 1), (9, 700), (64, 32), (3, 0), (RING, 4096), (RING, 20000), (RING, 0)):
            _step(tw, agents, mm, budget, flags)
        _rounds(tw, rng, 2)
        # call caps that truncate mid-list: by records, by bytes, by both
        _step(tw, agents, RING, 2000, flags, rec_cap=500)
        _step(tw, agents, RING, 2000, flags, byte_cap=64 * 1024)
        _step(tw, agents, RING, 0, flags, rec_cap=300, byte_cap=40 * 1024)
        _step(tw, agents[:5], RING, 0, flags, rec_cap=7, byte_cap=P)        # the first agent takes what fits
        _drain_same(tw)
    finally:
        for s in tw:
            s.close()


def test_repeated_budget_calls_drain_every_queue():
    from swarmdb_b200._native import HDR_DTYPE
    rng = np.random.default_rng(5)
    tw = _twins()
    try:
        _traffic(tw, rng, rounds=2)
        full, cmp_, ref = tw
        got = []
        for _ in range(10000):
            cnt, hdr, pay = full.receive_budget(None, 5, 700, 0, out_hdr=np.zeros(64, HDR_DTYPE),
                                                out_payload=np.zeros(4 * P, np.uint8))
            if len(hdr) == 0:
                break
            got.append(hdr["seq"].copy())
        assert full.stats()["delivered"] == full.stats()["enqueued"]
        loads = full.agent_loads()
        assert int(loads["pending"].sum()) == 0
        seqs = np.concatenate(got)
        assert len(np.unique(seqs)) == len(seqs)
    finally:
        for s in tw:
            s.close()


def test_refused_calls_leave_the_queue_untouched():
    from swarmdb_b200._native import RECV_ASYNC, SdbError
    rng = np.random.default_rng(3)
    tw = _twins(2)
    try:
        _traffic(tw, rng, rounds=1)
        a, b = tw
        with pytest.raises(SdbError):
            a.receive_budget(None, 10, 0, 0, out_payload=np.zeros(P - 1, np.uint8))
        with pytest.raises(SdbError):
            a.receive_compact(None, 10, 0, out_payload=np.zeros(P - 32, np.uint8), max_agent_bytes=64)
        with pytest.raises(SdbError):
            a._check(a._L.sdb_receive_budget(a._h, 0, None, 10, 0, RECV_ASYNC, None, None, 0, None, 0, None, None))
        _same_state(a, b)
        ca, ha, pa = a.receive_batch(None, RING, 0)
        cb, hb, pb = b.receive_batch(None, RING, 0)
        assert ha.tobytes() == hb.tobytes() and pa.tobytes() == pb.tobytes()
    finally:
        for s in tw:
            s.close()


def test_exact_capacity_takes_more_small_records_per_call():
    from swarmdb_b200._native import recv_capacity
    tw = _twins(2, max_recv_records=1 << 15, max_recv_payload=1 << 20)
    try:
        a, b = tw
        for s in tw:
            s.register(np.arange(A, dtype=np.uint32))
        n = 3000
        recv = (np.arange(n) % A).astype(np.uint32)
        lens = np.full(n, 64, np.uint16)
        off = (np.arange(n) * 64).astype(np.uint64)
        for s in tw:
            s.send_batch(np.zeros(n, np.uint32), recv, np.zeros(n, np.uint8), np.zeros(n, np.uint8), lens, off,
                         np.zeros(n * 64, np.uint8), np.zeros(n))
        _, h_plain, _ = b.receive_batch(None, 100, 0)
        _, h_budget, _ = a.receive_budget(None, 100, 0, 0)
        assert len(h_plain) <= recv_capacity(b.cfg) == (1 << 20) // P
        assert len(h_budget) == n                  # 3000 x 64 bytes fit 1 MiB exactly by bytes
    finally:
        for s in tw:
            s.close()


def test_owned_agents_of_a_sharded_handle():
    from swarmdb_b200._native import RECV_OWNED, RECV_PRIORITY
    rng = np.random.default_rng(21)
    tw = _twins(num_shards=2, shard_id=0)
    try:
        owner = (np.arange(A) % 3 == 0).astype(np.uint8)
        _traffic(tw, rng, rounds=1)                   # sent before the handles become sharded (then sends are exports)
        for s in tw:
            s.set_agent_shards(owner)
            s._owner = owner
        for s in tw:
            s.digest_reset()
        for flags in (RECV_OWNED, RECV_OWNED | RECV_PRIORITY):
            _step(tw, None, 4, 500, flags, owned=True)
    finally:
        for s in tw:
            s.close()


def test_surface_max_bytes(tmp_path):
    from swarmdb_b200.core import GpuConfig, SwarmsDB
    dbs = [SwarmsDB(save_dir=str(tmp_path / str(i)), auto_save=False,
                    gpu_config=GpuConfig(max_agents=64, max_payload_bytes=4096)) for i in range(2)]
    try:
        rng = np.random.default_rng(9)
        texts = ["x" * int(k) for k in rng.choice([0, 5, 40, 300, 2000], 120)]
        for db in dbs:
            db.register_agent("a"); db.register_agent("b")
            for t in texts:
                db.send_message("a", t, receiver_id="b")
        plain = [m.content for m in dbs[1].receive_messages("b", max_messages=1000)]
        got = []
        for _ in range(1000):
            peek = dbs[0].peek_messages("b", max_messages=7, max_bytes=600)
            ms = dbs[0].receive_messages("b", max_messages=7, max_bytes=600)
            assert [m.id for m in peek] == [m.id for m in ms]
            if not ms:
                break
            assert len(ms) <= 7
            enc = sum(len(str(m.content).encode()) for m in ms)
            assert len(ms) == 1 or enc <= 600
            got.extend(m.content for m in ms)
        assert got == plain
    finally:
        for db in dbs:
            db.close()
