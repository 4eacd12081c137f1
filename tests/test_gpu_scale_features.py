"""Relocation, leases, dead letters, lease snapshots, restore and byte-budget receives at the c2 scale (bench.Workload:
1M agents, 15,625 groups of 64, 65,536 group sends per batch = 4,194,304 records).

Every device feature sizes its grid with sdb_grid(items, per_block, 32 x SMs) (csrc/sdb_common.cuh): above that cap a
kernel gets no more blocks and its grid-stride loop runs another pass.  One pass covers 32 x SMs x per_block items:
  32  (8 lanes per agent)    k_reloc_mark, k_reloc_ring, k_restore_plan, k_restore_ring
  8   (one warp per item)    k_reloc_copy (bitmap words), k_lease_append_agents, k_lease_stage_rows, k_lease_copy_rows,
                             k_ledger_insert (runs), k_ledger_import, k_restore_payloads (rows)
  256 (one thread per item)  k_lease_append_copy, k_ledger_take, k_lease_import_check, k_restore_headers
Each test first asserts that its sizes are at least twice the one-pass coverage of the kernels it targets on the card it
runs on, so a card with more SMs cannot turn it into a one-pass test.  sdb_scan_u32 sweeps its tile totals in chunks of
1,024 tiles of 4,096 elements; the relocation scans one bitmap word per 32 granules (1 KiB of arena), so only a relocated
span above 4 GiB carries across a chunk.

Relocation checks run after enough traffic to overwrite the region a relocation freed: a ring entry that was not
rewritten still reads the right bytes until then.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ALNUM = np.frombuffer(b"ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789", np.uint8)
SCAN_CHUNK = 1024 * 4096                   # elements one k_scan_tops chunk covers


def _one_pass(per_block):
    """Items one pass of a grid-stride loop covers under sdb_grid(items, per_block, 32 x SMs)."""
    import torch
    return per_block * 32 * torch.cuda.get_device_properties(0).multi_processor_count


def _c2(wl, arena, rec_cap, ring=64):
    from swarmdb_b200._native import Shard
    s = Shard(max_agents=wl.A, ring_slots=ring, arena_bytes=arena, max_payload_bytes=wl.L, max_groups=1 << 14,
              member_pool_entries=wl.A + 1024, max_batch_sends=wl.S, max_batch_payload=wl.S * wl.L,
              max_recv_records=rec_cap, max_recv_payload=rec_cap * wl.L)
    s.register(np.arange(wl.A, dtype=np.uint32))
    for g in range(wl.G):
        s.create_group(g, wl.members(g))
    return s


def _group_batch(wl, rng, lo=1):
    """One c2 batch of group sends, payload lengths uniform in [lo, 256], four priorities."""
    snd, grp, prio, typ, lens, off, payload = wl.batch()
    lens = rng.integers(lo, wl.L + 1, wl.S).astype(np.uint16)
    return snd, grp, prio, typ, lens, off, payload


def _p2p_batch(wl, rng, receivers=None, lo=0):
    """wl.S point-to-point sends (one private payload image each) to random agents (or random `receivers`)."""
    n = wl.S
    snd = rng.integers(0, wl.A, n).astype(np.uint32)
    rcv = (rng.integers(0, wl.A, n) if receivers is None else rng.choice(receivers, n)).astype(np.uint32)
    prio = rng.integers(0, 4, n).astype(np.uint8)
    typ = rng.integers(0, 7, n).astype(np.uint8)
    lens = rng.integers(lo, wl.L + 1, n).astype(np.uint16)
    off = np.arange(n, dtype=np.uint64) * wl.L
    return snd, rcv, prio, typ, lens, off, ALNUM[rng.integers(0, 62, n * wl.L)]


def _backlog(wl, handles, rng):
    """A c2 group batch and a batch of point-to-point records on every handle: 4,194,304 + 65,536 records, 131,072
    payload rows in a compact receive of all of them."""
    gb, pb = _group_batch(wl, rng), _p2p_batch(wl, rng)
    n = wl.S * wl.F + wl.S
    for s in handles:
        s.send_group_batch(*gb)
        s.send_batch(*pb)
        assert s.queue_stats()["pending"] == n
    return n


def _copy(res):
    return tuple(x.copy() if isinstance(x, np.ndarray) else x for x in res)


def _records_equal(cnt, ent, snd, pay, want_cnt, want_hdr, want_pay, what):
    """A compact-format result, expanded, equals the expected counts, headers and padded payload bytes."""
    from swarmdb_b200._native import expand_compact
    assert np.array_equal(cnt, want_cnt), what
    hdr, full = expand_compact(ent, snd, pay)
    assert len(hdr) == len(want_hdr), what
    for f in hdr.dtype.names:
        assert np.array_equal(hdr[f], want_hdr[f]), (what, f)
    assert full.tobytes() == want_pay.tobytes(), what


def _drain_digests(s):
    """Every agent's digest over a full drain (reset first)."""
    s.digest_reset()
    while True:
        _, total, _ = s.receive_batch(None, 1 << 10, 0, copy_out=False)
        s.digest_fold()
        if not total:
            break
    assert s.queue_stats()["pending"] == 0
    return s.digest_read()


def _pending_equal(x, y, what):
    lx, ly = x.agent_loads(), y.agent_loads()
    for f in ("pending", "pending_by_prio", "pending_granules"):
        assert np.array_equal(lx[f], ly[f]), (what, f)


def _mismatch(da, db):
    bad = np.nonzero(da != db)[0]
    return f"{len(bad)} agents differ, first {bad[:8].tolist()}" if len(bad) else ""


def _relocate(x, cut):
    """One relocation held to the contract: the dry run equals the real call, no counter moves, the floor moves, and a
    second call at the same cut moves nothing."""
    st0 = x.stats()
    keep = lambda st: {k: v for k, v in st.items() if k != "kernel_launches"}          # noqa: E731
    dry = x.relocate(cut, peek=True)
    assert keep(x.stats()) == keep(st0)
    s = x.relocate(cut)
    assert s == dry
    st1 = x.stats()
    moved = {k: st1[k] - st0[k] for k in st0 if k not in ("arena_tail_bytes", "arena_floor_bytes", "kernel_launches")}
    assert all(v == 0 for v in moved.values()), moved
    assert s["records"] > 0
    assert st1["arena_tail_bytes"] == st0["arena_tail_bytes"] + s["skipped_bytes"] + s["moved_bytes"] == s["tail_after"]
    assert st1["arena_floor_bytes"] == s["floor_after"] > st0["arena_floor_bytes"]
    again = x.relocate(cut)
    assert again["records"] == 0 and again["moved_bytes"] == 0
    assert x.stats()["arena_tail_bytes"] == st1["arena_tail_bytes"]
    return s


def test_relocation_twins_at_c2():
    """A (1 GiB arena) relocates every pending record twice while every third agent never receives; B (8 GiB) never
    relocates.  Busy agents take partial receives between c2 batches, so their leftovers are moved too.  After the
    second relocation, point-to-point traffic to the busy agents overwrites the freed regions; then loads, queue stats
    and the digests of everything delivered and of full drains must agree."""
    from bench import Workload
    wl = Workload()
    rec_cap = wl.S * wl.F + (1 << 16)
    idle = np.arange(0, wl.A, 3, dtype=np.uint32)                   # never received until the final drain
    busy = np.setdiff1d(np.arange(wl.A, dtype=np.uint32), idle)
    assert wl.A > 2 * _one_pass(32) and len(idle) > 2 * _one_pass(32)   # k_reloc_mark / k_reloc_ring
    rng = np.random.default_rng(41)
    a, b = _c2(wl, 1 << 30, rec_cap), _c2(wl, 1 << 33, rec_cap)
    try:
        for x in (a, b):
            x.digest_reset()

        def receive(agents, k):
            ta = a.receive_batch(agents, k, 0, copy_out=False)[1:]
            a.digest_fold()
            tb = b.receive_batch(agents, k, 0, copy_out=False)[1:]
            b.digest_fold()
            assert ta == tb

        def send_p2p(batch):
            assert a.send_batch(*batch) == b.send_batch(*batch)            # the same first seq

        relocations = []
        for _ in range(2):
            for _ in range(2):
                batch = _group_batch(wl, rng)
                assert a.send_group_batch(*batch) == b.send_group_batch(*batch)
                receive(busy, 3)                                      # leaves most busy agents a remainder
            st = a.stats()
            words = (st["arena_tail_bytes"] - st["arena_floor_bytes"]) // 1024
            assert words > 2 * _one_pass(8)                            # k_reloc_copy
            s = _relocate(a, st["arena_tail_bytes"])                   # every pending record moves
            assert s["agents"] > 2 * _one_pass(32), s
            relocations.append(s)
            assert a.agent_loads().tobytes() == b.agent_loads().tobytes()
            receive(busy, 1 << 10)                                    # the busy agents catch up
        assert len(relocations) == 2
        # overwrite what the relocations freed: A's live records now sit in [floor, tail); the arena is 1 GiB, so writing
        # up to floor + 1 GiB reuses every physical position below the floor
        arena = 1 << 30
        batch_bytes = wl.S * (32 + wl.L)
        floor = a.stats()["arena_floor_bytes"]
        assert floor >= relocations[-1]["floor_after"]
        while a.stats()["arena_tail_bytes"] + batch_bytes <= floor + arena - batch_bytes:
            send_p2p(_p2p_batch(wl, rng, busy, lo=wl.L))
            receive(busy, 1 << 10)
        assert a.stats()["arena_tail_bytes"] > floor + arena - 3 * batch_bytes
        la, lb = a.agent_loads(), b.agent_loads()
        assert la.tobytes() == lb.tobytes() and a.queue_stats() == b.queue_stats()
        delivered = a.digest_read()                                   # everything delivered so far
        assert np.array_equal(delivered, b.digest_read()) and int((delivered[busy] != 0).sum()) > 0.99 * len(busy)
        da, db = _drain_digests(a), _drain_digests(b)
        assert not _mismatch(da, db), _mismatch(da, db)
        assert int((da[idle] != 0).sum()) > 0.99 * len(idle)
        for x in (a, b):
            st = x.stats()
            assert st["ring_overflow"] == 0 and st["enqueued"] == st["delivered"]
    finally:
        a.close(); b.close()


def test_relocation_across_scan_chunks():
    """300 pinned agents keep four records each, spread over 4.6 GB of point-to-point traffic that the other agents
    drain, so the relocated span holds more bitmap words than one k_scan_tops chunk.  The summary must count exactly what
    the host sent, and after an arena's worth of overwrite traffic the pinned queues must read back byte for byte."""
    from swarmdb_b200._native import NO_GROUP, RECV_PEEK, Shard, pad32
    A, P, N = 4096, 4096, 1 << 14
    pinned = np.arange(300, dtype=np.uint32)
    filler = np.arange(300, A, dtype=np.uint32)
    arena = 1 << 33
    s = Shard(max_agents=A, ring_slots=64, arena_bytes=arena, max_payload_bytes=P, max_batch_sends=N,
              max_batch_payload=N * P, max_recv_records=1 << 15, max_recv_payload=(1 << 15) * P)
    try:
        s.register(np.arange(A, dtype=np.uint32))
        rng = np.random.default_rng(43)
        buf = rng.integers(0, 256, N * P, dtype=np.uint8)
        per_batch = N * (32 + P)
        nb = -(-int(4.6e9) // per_batch)
        # pinned records go out in the first nb - 2 batches, so each lies at least two batches below the final tail
        pin_rcv = rng.permutation(np.repeat(pinned, 4))
        chunks = np.array_split(pin_rcv, nb - 2)
        kept = []                                                    # (receiver, sender, prio, type, len, ts, bytes)
        ts = 0.0

        def send(k_pin):
            nonlocal ts
            rcv = rng.choice(filler, N).astype(np.uint32)
            snd = rng.integers(0, A, N).astype(np.uint32)
            prio = rng.integers(0, 4, N).astype(np.uint8)
            typ = rng.integers(0, 7, N).astype(np.uint8)
            lens = np.full(N, P, np.uint16)
            off = np.arange(N, dtype=np.uint64) * P
            t = ts + np.arange(N, dtype=np.float64) / N
            m = len(k_pin)
            if m:
                rcv[:m] = k_pin
                lens[:m] = rng.integers(0, P + 1, m)
                off[:m] = rng.integers(0, (N * P - P) // 16, m).astype(np.uint64) * 16
                for i in range(m):
                    o, ln = int(off[i]), int(lens[i])
                    kept.append((int(rcv[i]), int(snd[i]), int(prio[i]), int(typ[i]), ln, float(t[i]), buf[o:o + ln].tobytes()))
            ts += 1.0
            s.send_batch(snd, rcv, prio, typ, lens, off, buf, t)
            _, total, _ = s.receive_batch(filler, 64, 0, copy_out=False)
            assert total == N - m

        for b in range(nb):
            send(chunks[b] if b < len(chunks) else pin_rcv[:0])
        st = s.stats()
        tail, floor = st["arena_tail_bytes"], st["arena_floor_bytes"]
        assert (tail - floor) // 1024 > SCAN_CHUNK                     # k_scan_tops carries across a chunk
        assert s.queue_stats()["pending"] == len(kept) == 1200
        # the pinned queues as the host sent them, in send order
        order = sorted(range(len(kept)), key=lambda i: (kept[i][0], i))
        want = [kept[i] for i in order]
        cnt, hdr, pay = _copy(s.receive_batch(pinned, 64, RECV_PEEK))
        assert np.array_equal(cnt, np.bincount([k[0] for k in kept], minlength=A)[pinned])
        assert list(hdr["receiver"]) == [w[0] for w in want] and list(hdr["sender"]) == [w[1] for w in want]
        assert list(hdr["prio"]) == [w[2] for w in want] and list(hdr["type"]) == [w[3] for w in want]
        assert list(hdr["len"]) == [w[4] for w in want] and list(hdr["timestamp"]) == [w[5] for w in want]
        assert np.all(hdr["group"] == NO_GROUP)
        ends = np.cumsum(cnt.astype(np.int64))
        for e, c in zip(ends, cnt.astype(np.int64)):
            assert np.all(np.diff(hdr["seq"][e - c:e].astype(np.int64)) > 0)
        offs = np.concatenate([[0], np.cumsum(pad32(hdr["len"].astype(np.int64)))])
        for r, w in enumerate(want):
            assert pay[offs[r]:offs[r] + w[4]].tobytes() == w[6]

        sm = _relocate(s, tail)
        assert sm["agents"] == len(pinned) and sm["records"] == len(kept)
        assert sm["moved_bytes"] == sum(32 + pad32(w[4]) for w in kept)
        assert sm["skipped_bytes"] == 0 and sm["floor_after"] == tail
        # overwrite every physical position below the moved region
        while s.stats()["arena_tail_bytes"] + per_batch <= sm["floor_after"] + arena - per_batch:
            send(pin_rcv[:0])
        assert s.stats()["arena_tail_bytes"] > arena + tail - 2 * per_batch
        cnt2, hdr2, pay2 = s.receive_batch(pinned, 64, 0)
        assert np.array_equal(cnt2, cnt) and hdr2.tobytes() == hdr.tobytes() and pay2.tobytes() == pay.tobytes()
        assert s.stats()["ring_overflow"] == 0 and s.queue_stats()["pending"] == 0
    finally:
        s.close()


def _lease_handle(wl, rec_cap, max_deliveries):
    from swarmdb_b200._native import pad32
    s = _c2(wl, 1 << 32, rec_cap)
    s.lease_reserve(rec_cap, rec_cap * pad32(wl.L))
    s.lease_set_policy(max_deliveries, rec_cap)
    return s


def test_leases_at_c2():
    """A leased receive of the whole backlog, acks of a seeded random half of the lease ids, a sweep of the rest: every
    agent's queue is then its unacknowledged records in their original order, read back by a full compact drain.  A
    second leased receive of a sample of agents gives their redelivered records a delivery count of 2."""
    from bench import Workload
    from swarmdb_b200._native import LEASE_ACK, LEASE_ALL, expand_compact
    wl = Workload()
    rec_cap = wl.S * wl.F + (1 << 17)
    rng = np.random.default_rng(47)
    s = _lease_handle(wl, rec_cap, 0xFFFFFFFF)                     # delivery counts without a limit
    try:
        n = _backlog(wl, [s], rng)
        c, e, sn, p, base = _copy(s.receive_leased(None, 1 << 10, 1.0))
        assert len(e) == n and base >= 0
        assert wl.A > 2 * _one_pass(8)                                 # k_lease_append_agents
        assert n > 2 * _one_pass(256)                                  # k_lease_append_copy
        assert len(sn) > 2 * _one_pass(8)                              # k_lease_stage_rows, k_lease_copy_rows
        acked = rng.permutation(n)[: n // 2]
        _, m = s.lease_settle(base + acked.astype(np.uint64), LEASE_ACK)
        assert m == len(acked)
        assert s.lease_sweep(2.0) == (n - len(acked), 0, 0)
        keep = np.ones(n, bool); keep[acked] = False
        who = np.repeat(np.arange(len(c)), c.astype(np.int64))
        want_cnt = np.bincount(who[keep], minlength=len(c)).astype(np.uint32)
        want_hdr, want_pay = expand_compact(e[keep], sn, p)
        # a second leased receive of a sample of agents: counts of 2, then swept back unchanged in order
        sample = np.sort(rng.choice(wl.A, 50_000, replace=False)).astype(np.uint32)
        c2, e2, _, _, base2 = _copy(s.receive_leased(sample, 1 << 10, 1.0))
        in_sample = np.isin(who[keep], sample)
        assert np.array_equal(c2, want_cnt[sample]) and np.array_equal(e2["seq"], want_hdr["seq"][in_sample])
        assert np.all(s.lease_deliveries(base2 + np.arange(len(e2), dtype=np.uint64)) == 2)
        assert s.lease_sweep(3.0, LEASE_ALL) == (len(e2), 0, 0)
        res = _copy(s.receive_compact(None, 1 << 10, 0))
        _records_equal(*res, want_cnt, want_hdr, want_pay, "full compact drain after settle and sweep")
        assert s.queue_stats()["pending"] == 0
        ls = s.lease_stats()
        assert ls["live"] == ls["acked_unreclaimed"] == ls["entries_used"] == ls["payload_used"] == 0, ls
        assert ls["acked_total"] == len(acked) and ls["redelivered_total"] == n - len(acked) + len(e2)
    finally:
        s.close()


def test_dead_letters_at_c2():
    """Policy M = 2: the whole backlog leased and swept back (its counts enter the ledger through k_ledger_insert), leased
    again with counts of 2 and swept into the dead letters; taking them returns the original backlog per agent, in order."""
    from bench import Workload
    from swarmdb_b200._native import LEASE_ALL, RECV_PEEK, expand_compact
    wl = Workload()
    rec_cap = wl.S * wl.F + (1 << 17)
    rng = np.random.default_rng(53)
    s = _lease_handle(wl, rec_cap, 2)
    try:
        n = _backlog(wl, [s], rng)
        c0, e0, sn0, p0 = _copy(s.receive_compact(None, 1 << 10, RECV_PEEK))
        h0, pl0 = expand_compact(e0, sn0, p0)
        assert len(e0) == n
        assert int((c0 > 0).sum()) > 2 * _one_pass(8)                  # k_ledger_insert: at least one run per agent
        assert n > 2 * _one_pass(256)                                  # k_ledger_take
        assert len(s.receive_leased(None, 1 << 10, 1.0)[1]) == n
        assert s.lease_sweep(0.0, LEASE_ALL) == (n, 0, 0)
        assert s.lease_policy_stats()["dead"] == 0
        _, e1, _, _, base = s.receive_leased(None, 1 << 10, 1.0)
        assert len(e1) == n
        assert np.all(s.lease_deliveries(base + np.arange(n, dtype=np.uint64)) == 2)
        assert s.lease_sweep(0.0, LEASE_ALL) == (0, 0, 0)
        assert s.lease_policy_stats()["dead"] == n and s.queue_stats()["pending"] == 0
        c, e, sn, p, d = _copy(s.lease_dead_letters(None))
        assert np.all(d == 2) and len(d) == n
        _records_equal(c, e, sn, p, c0, h0, pl0, "dead letters against the original backlog")
        assert s.lease_policy_stats()["dead"] == 0 and s.lease_stats()["live"] == 0
        assert s.queue_stats()["pending"] == 0
    finally:
        s.close()


def test_lease_snapshot_at_c2():
    """Policy M = 3: the backlog leased, a third of it nacked and swept back, a seeded quarter of the rest renewed to an
    earlier deadline.  The store and the ledger are exported; a fresh handle is given the pending records, the ledger and
    the store.  Both are swept at the same `now`: stats, ledgers and the drains that follow must agree."""
    from bench import Workload
    from swarmdb_b200._native import LEASE_ALL, LEASE_RENEW, RECV_PEEK
    wl = Workload()
    rec_cap = wl.S * wl.F + (1 << 17)
    rng = np.random.default_rng(59)
    s = _lease_handle(wl, rec_cap, 3)
    d = None
    try:
        n = _backlog(wl, [s], rng)
        base = s.receive_leased(None, 1 << 10, 1e300)[4]
        nacked = n // 3
        s.lease_settle(base + rng.permutation(n)[:nacked].astype(np.uint64), LEASE_RENEW, -np.inf)
        assert s.lease_sweep(0.0) == (nacked, 0, 0)
        live = n - nacked
        early = rng.permutation(live)[: live // 4]
        cnt, ent, snd, pay = _copy(s.receive_compact(None, 1 << 10, RECV_PEEK))
        assert len(ent) == nacked
        e, sn, p, m, nxt = _copy(s.lease_export(0))
        assert len(e) == live and len(s.lease_export(nxt)[0]) == 0
        ids = m["id"][early]
        assert s.lease_settle(ids, LEASE_RENEW, 4.0)[1] == len(ids)
        m["deadline"][early] = 4.0                                    # the same renewal, carried in the snapshot
        la, lseq, lc = _copy(s.ledger_export())
        assert len(la) == nacked
        assert live > 2 * _one_pass(256)                               # k_lease_import_check, k_lease_append_copy
        assert len(sn) > 2 * _one_pass(8) and nacked > 2 * _one_pass(8)  # k_lease_stage_rows / copy_rows, k_ledger_import
        d = _lease_handle(wl, rec_cap, 3)
        assert d.restore_compact(np.arange(len(cnt), dtype=np.uint32), cnt, ent, snd, pay)[0] == nacked
        assert d.ledger_import(la, lseq, lc) == nacked
        d.lease_import(e, sn, p, m)
        assert d.lease_stats()["live"] == live

        def ledger(x):
            a, q, k = x.ledger_export()
            o = np.lexsort((q, a))
            return a[o], q[o], k[o]

        def same(what):
            for x, y in zip(ledger(s), ledger(d)):
                assert np.array_equal(x, y), what
            hist = ("redelivered_total", "acked_total")
            ls, ld = s.lease_stats(), d.lease_stats()
            assert {k: v for k, v in ls.items() if k not in hist} == {k: v for k, v in ld.items() if k not in hist}, what
            assert s.lease_policy_stats() == d.lease_policy_stats(), what
            _pending_equal(s, d, what)

        same("after the import")
        for x in (s, d):
            assert x.lease_sweep(5.0) == (len(early), 0, 0)
        same("after a sweep of the renewed quarter")
        ds, dd = _drain_digests(s), _drain_digests(d)
        assert not _mismatch(ds, dd), _mismatch(ds, dd)
        for x in (s, d):
            assert x.lease_sweep(5.0, LEASE_ALL) == (live - len(early), 0, 0)
        same("after a sweep of every lease")
        ds, dd = _drain_digests(s), _drain_digests(d)
        assert not _mismatch(ds, dd), _mismatch(ds, dd)
        assert s.lease_stats()["live"] == d.lease_stats()["live"] == 0
    finally:
        s.close()
        if d is not None:
            d.close()


def _shared_entries(cnt, rows):
    """Entries sdb_restore_compact lays out as shared rows: each agent's entries up to its first row descent."""
    c = cnt.astype(np.int64)
    start = np.zeros(len(c) + 1, np.int64); np.cumsum(c, out=start[1:])
    rows = rows.astype(np.int64)
    desc = np.zeros(len(rows), bool)
    desc[1:] = rows[1:] < rows[:-1]
    desc[start[:-1][c > 0]] = False                                   # an agent's first entry starts its own run
    agent = np.repeat(np.arange(len(c)), c)
    at = np.flatnonzero(desc)
    shared = c.copy()
    np.minimum.at(shared, agent[at], at - start[agent[at]])
    return int(shared.sum())


def test_restore_many_rows_at_c2():
    """A PEEK compact snapshot of a c2 backlog that also holds point-to-point records (rows renumbered by smallest seq, as
    a snapshot restore does), restored into a fresh handle: the drains' digests must be equal, and the restore must take
    exactly the arena bytes the sends took."""
    from bench import Workload
    from swarmdb_b200._native import RECV_PEEK
    from swarmdb_b200.core import _renumber_rows
    wl = Workload()
    rec_cap = wl.S * wl.F + (1 << 17)
    rng = np.random.default_rng(61)
    src = _c2(wl, 1 << 31, rec_cap)
    dst = None
    try:
        t0 = src.stats()["arena_tail_bytes"]
        n = _backlog(wl, [src], rng)
        sent = src.stats()["arena_tail_bytes"] - t0
        cnt, ent, snd, pay = _copy(src.receive_compact(None, 1 << 10, RECV_PEEK))
        assert len(ent) == n
        ent2, snd2 = _renumber_rows(ent, snd)
        used = np.bincount(ent2["send"].astype(np.int64), minlength=len(snd2))
        assert int((used > 0).sum()) > 2 * _one_pass(8)                # k_restore_payloads
        assert _shared_entries(cnt, ent2["send"]) > 2 * _one_pass(256)  # k_restore_headers
        assert wl.A > 2 * _one_pass(32)                                # k_restore_plan, k_restore_ring
        dst = _c2(wl, 1 << 31, rec_cap)
        t1 = dst.stats()["arena_tail_bytes"]
        assert dst.restore_compact(np.arange(len(cnt), dtype=np.uint32), cnt, ent2, snd2, pay)[0] == n
        assert dst.stats()["arena_tail_bytes"] - t1 == sent
        _pending_equal(src, dst, "after the restore")
        ds, dd = _drain_digests(src), _drain_digests(dst)
        assert not _mismatch(ds, dd), _mismatch(ds, dd)
        assert int((ds != 0).sum()) > 0.98 * wl.A
    finally:
        src.close()
        if dst is not None:
            dst.close()


def _budget_counts(cnt, lens, max_messages, max_agent_bytes, rec_cap, byte_cap):
    """tests/budget_ref.call_counts, vectorised: agent i's candidates are the first cnt[i] entries of `lens` after the
    earlier agents' (its delivery order, at least max_messages of it or all of its queue)."""
    from tests.budget_ref import prefix
    c = cnt.astype(np.int64)
    start = np.zeros(len(c) + 1, np.int64); np.cumsum(c, out=start[1:])
    agent = np.repeat(np.arange(len(c)), c)
    j = np.arange(len(agent)) - start[agent]
    p = (lens.astype(np.int64) + 31) & ~31
    before = np.concatenate([[0], np.cumsum(p)])
    inside = before[1:] - before[start[:-1]][agent]                   # inclusive running bytes within the agent
    ok = (j < max_messages) & ((max_agent_bytes == 0) | (inside <= max_agent_bytes) | (j == 0))
    k = np.bincount(agent[ok], minlength=len(c))
    b = np.bincount(agent[ok], weights=p[ok], minlength=len(c)).astype(np.int64)
    K, B = np.cumsum(k), np.cumsum(b)
    out = k.copy()
    bad = np.flatnonzero((K > rec_cap) | (B > byte_cap))
    if len(bad):
        i = int(bad[0])
        out[i:] = 0
        if K[i] - k[i] == 0:                                           # first in the output: the prefix that fits
            out[i] = prefix(list(lens[start[i]:start[i] + k[i]]), rec_cap, byte_cap)
    return out


def test_budget_receive_at_c2():
    """Full-format and compact budget calls in stream and priority order on two c2 backlogs (lengths 0..256, four
    priorities) with a per-agent limit that cuts inside most queues, then calls whose record cap or byte cap truncates
    mid-list.  Expected records: one PEEK of the plain receive per call, cut by tests/budget_ref.py's rule.  A third
    twin takes the same records through the id-set filter; the final drains of all three must agree."""
    from bench import Workload
    from swarmdb_b200._native import ENTRY_DTYPE, HDR_DTYPE, RECV_PEEK, RECV_PRIORITY, SEND_DTYPE, expand_compact, make_filter
    from tests.budget_ref import call_counts
    wl = Workload()
    rec_cap = 2 * wl.S * wl.F + (1 << 16)
    rng = np.random.default_rng(67)
    # the vectorised count against budget_ref on a small case with every edge: caps, first-agent prefix, empty queues
    for _ in range(20):
        cnt = rng.integers(0, 6, 300)
        lens = rng.choice([0, 1, 32, 33, 200, 256, 700], int(cnt.sum()))
        s0 = np.concatenate([[0], np.cumsum(cnt)])
        orders = [list(lens[s0[i]:s0[i + 1]]) for i in range(len(cnt))]
        for mm, lim, rc, bc in ((3, 600, 10 ** 9, 10 ** 12), (5, 0, 200, 10 ** 12), (4, 300, 10 ** 9, 20000), (9, 0, 2, 100)):
            assert list(_budget_counts(cnt, lens, mm, lim, rc, bc)) == call_counts(orders, mm, lim, rc, bc)
    tw = [_c2(wl, 1 << 31, rec_cap) for _ in range(3)]
    full, cmp_, ref = tw
    try:
        def send():
            batch = _group_batch(wl, rng, lo=0)
            assert len({x.send_group_batch(*batch) for x in tw}) == 1

        send(); send()
        assert wl.A > 2 * _one_pass(32)
        bcap = rec_cap * wl.L
        steps = [(0, 3, 600, rec_cap, bcap), (RECV_PRIORITY, 3, 600, rec_cap, bcap), None,
                 (0, 5, 1000, 2_500_003, bcap), (RECV_PRIORITY, 5, 1000, rec_cap, 300 << 20)]
        for step in steps:
            if step is None:
                send()                                                # deeper queues for the truncating calls
                continue
            flags, mm, limit, rc, bc = what = step
            pc, ph, pp = _copy(ref.receive_batch(None, mm, flags | RECV_PEEK))
            want = _budget_counts(pc, ph["len"], mm, limit, rc, bc)
            if rc < rec_cap or bc < bcap:                             # cut mid-list, after thousands of plan tiles
                last = int(np.flatnonzero(want)[-1])
                assert last > 256 * 1000 and int((pc[last + 1:] > 0).sum()) > 1000, (what, last)
            start = np.concatenate([[0], np.cumsum(pc.astype(np.int64))])
            j = np.arange(len(ph)) - np.repeat(start[:-1], pc.astype(np.int64))
            sel = j < np.repeat(want, pc.astype(np.int64))
            plen = (ph["len"].astype(np.int64) + 31) & ~31
            want_hdr, want_pay = ph[sel], pp[np.repeat(sel, plen)]
            cnt, hdr, pay = full.receive_budget(None, mm, limit, flags, out_hdr=np.zeros(rc, HDR_DTYPE),
                                                out_payload=np.zeros(bc, np.uint8))
            assert np.array_equal(cnt, want), what
            assert hdr.tobytes() == want_hdr.tobytes() and pay.tobytes() == want_pay.tobytes(), what
            cc, ce, cs, cp = cmp_.receive_compact(None, mm, flags, out_entries=np.zeros(rc, ENTRY_DTYPE),
                                                  out_sends=np.zeros(rc, SEND_DTYPE), out_payload=np.zeros(bc, np.uint8),
                                                  max_agent_bytes=limit)
            assert np.array_equal(cc, want), what
            ch, cf = expand_compact(ce, cs, cp)
            assert ch.tobytes() == want_hdr.tobytes() and cf.tobytes() == want_pay.tobytes(), what
            rcnt, total = ref.receive_where(None, mm, 0, make_filter(ids=want_hdr["seq"]), drop=True)
            assert total == len(want_hdr) and np.array_equal(rcnt, want), what
            _pending_equal(full, ref, what)
            _pending_equal(cmp_, ref, what)
        dg = [_drain_digests(x) for x in tw]
        assert not _mismatch(dg[0], dg[2]), _mismatch(dg[0], dg[2])
        assert not _mismatch(dg[1], dg[2]), _mismatch(dg[1], dg[2])
        assert int((dg[2] != 0).sum()) > wl.A // 4
    finally:
        for x in tw:
            x.close()
