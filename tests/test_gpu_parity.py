"""GPU parity: the CUDA path (through the C ABI) against the CPU oracle, bit-exact.

Every test drives `swarmdb_b200._native.Shard` (ctypes -> libswarmdb_b200.so -> sm_90a kernels)
and `oracle.cpu_ref.CpuOracle` (gcc-built restatement, pinned to the reference's goldens by
tests/test_oracle_c.py) with the same seeded batches and compares headers and payload bytes
of every delivered record, per agent, in delivery order.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _mk_payloads(rng, n, max_len, fixed=False):
    lens = np.full(n, max_len, np.uint16) if fixed else rng.integers(0, max_len + 1, n).astype(np.uint16)
    stride = (max_len + 31) & ~31
    buf = np.zeros(n * stride + 64, np.uint8)
    off = (np.arange(n, dtype=np.uint64) * stride)
    alnum = np.frombuffer(b"ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789", np.uint8)
    for i in range(n):
        buf[int(off[i]): int(off[i]) + int(lens[i])] = alnum[rng.integers(0, 62, int(lens[i]))]
    return lens, off, buf


def _same(res_gpu, res_cpu):
    cg, hg, pg = res_gpu
    cc, hc, pc = res_cpu
    assert np.array_equal(cg, cc), (cg[:16], cc[:16])
    assert len(hg) == len(hc)
    for f in hg.dtype.names:
        assert np.array_equal(hg[f], hc[f]), f
    assert pg.tobytes() == pc.tobytes()


def _pair(max_agents, max_groups=8, **kw):
    from oracle.cpu_ref import CpuOracle
    from swarmdb_b200._native import Shard
    g = Shard(max_agents=max_agents, max_groups=max_groups, **kw)
    c = CpuOracle(max_agents, max_groups)
    return g, c


@pytest.mark.parametrize("variant", [0, 1, 2, 3])
def test_p2p_then_drain(variant):
    rng = np.random.default_rng(11)
    A = 200
    g, c = _pair(A, fanout_variant=variant)
    idx = np.arange(A, dtype=np.uint32)
    g.register(idx); c.register(idx)
    for rnd in range(3):
        n = 3000
        s = rng.integers(0, A, n); r = rng.integers(0, A, n)
        prio = rng.integers(0, 4, n); typ = rng.integers(0, 7, n)
        lens, off, buf = _mk_payloads(rng, n, 256)
        ts = rng.random(n)
        assert g.send_batch(s, r, prio, typ, lens, off, buf, ts) == c.send_batch(s, r, prio, typ, lens, off, buf, ts)
        _same(g.receive_batch(idx, 7), c.receive_batch(idx, 7))
    _same(g.receive_batch(idx, 1000), c.receive_batch(idx, 1000))
    _same(g.receive_batch(idx, 1000), c.receive_batch(idx, 1000))      # empty drain
    st = g.stats()
    assert st["enqueued"] == 9000 and st["delivered"] == 9000 and st["ring_overflow"] == 0


@pytest.mark.parametrize("variant", [0, 1, 2, 3])
@pytest.mark.parametrize("fixed", [True, False])
def test_group_fanout_parity(variant, fixed):
    rng = np.random.default_rng(5 + variant)
    A, G, F = 4096, 64, 64
    g, c = _pair(A, max_groups=G + 2, fanout_variant=variant, ring_slots=256)
    perm = rng.permutation(A)
    for k in range(G):
        m = perm[k * F:(k + 1) * F]
        g.create_group(k, m); c.create_group(k, m)
    # a group with duplicate members and one of size 1, one empty
    dup = np.array([3, 9, 3, 3, 17], np.uint32)
    g.create_group(G, dup); c.create_group(G, dup)
    g.create_group(G + 1, np.array([5], np.uint32)); c.create_group(G + 1, np.array([5], np.uint32))
    allidx = np.arange(A, dtype=np.uint32)
    for rnd in range(3):
        n = 700
        grp = rng.integers(0, G + 2, n)
        s = rng.integers(0, A, n)                      # sometimes a member: skip-sender exercised
        s[:20] = 3; grp[:20] = G                       # sender inside the duplicate group
        s[20:30] = 5; grp[20:30] = G + 1               # group of one whose only member is the sender
        prio = rng.integers(0, 4, n); typ = rng.integers(0, 7, n)
        lens, off, buf = _mk_payloads(rng, n, 256, fixed=fixed)
        bg = g.send_group_batch(s, grp, prio, typ, lens, off, buf)
        bc, routed = c.send_group_batch(s, grp, prio, typ, lens, off, buf)
        assert bg == bc
        if rnd == 1:
            _same(g.receive_batch(allidx, 3), c.receive_batch(allidx, 3))
    _same(g.receive_batch(None, 1000), c.receive_batch(None, 1000))
    st = g.stats()
    assert st["enqueued"] == st["delivered"] and st["skipped_sender"] > 0 and st["ring_overflow"] == 0


def test_group_overwrite_and_large_group():
    rng = np.random.default_rng(3)
    A = 3000
    g, c = _pair(A, max_groups=4, ring_slots=64)
    big = rng.permutation(A)[:1500]                    # > 256 members: several tiles per send
    g.create_group(0, big); c.create_group(0, big)
    lens, off, buf = _mk_payloads(rng, 4, 96)
    g.send_group_batch([1, 2, 3, 4], [0, 0, 0, 0], [0, 1, 2, 3], [0, 0, 0, 0], lens, off, buf)
    c.send_group_batch([1, 2, 3, 4], [0, 0, 0, 0], [0, 1, 2, 3], [0, 0, 0, 0], lens, off, buf)
    small = np.array([7, 8], np.uint32)                # overwrite (M:1223)
    g.create_group(0, small); c.create_group(0, small)
    g.send_group_batch([1], [0], [1], [0], lens[:1], off[:1], buf)
    c.send_group_batch([1], [0], [1], [0], lens[:1], off[:1], buf)
    _same(g.receive_batch(None, 100), c.receive_batch(None, 100))
    with pytest.raises(Exception):
        g.send_group_batch([1], [3], [1], [0], lens[:1], off[:1], buf)   # undefined group


def test_broadcast_lists_share_one_seq():
    rng = np.random.default_rng(9)
    A = 500
    g, c = _pair(A, list_pool_entries=8192)
    idx = np.arange(A, dtype=np.uint32)
    g.register(idx); c.register(idx)
    n = 12
    lists = [rng.choice(A, size=int(rng.integers(0, 300)), replace=False) for _ in range(n)]
    lo = np.zeros(n + 1, np.uint64); lo[1:] = np.cumsum([len(x) for x in lists])
    li = np.concatenate(lists).astype(np.uint32)
    s = rng.integers(0, A, n); prio = rng.integers(0, 4, n); typ = rng.integers(0, 7, n)
    lens, off, buf = _mk_payloads(rng, n, 200)
    # interleave with p2p traffic so stream order across kinds is checked
    l2, o2, b2 = _mk_payloads(rng, 50, 64)
    s2 = rng.integers(0, A, 50); r2 = rng.integers(0, A, 50)
    for sys in (g, c):
        sys.send_batch(s2, r2, None, None, l2, o2, b2)
        sys.send_list_batch(s, lo, li, prio, typ, lens, off, buf)
        sys.send_batch(r2, s2, None, None, l2, o2, b2)
    _same(g.receive_batch(idx, 1000), c.receive_batch(idx, 1000))


def test_priority_receive_matches_oracle_and_equal_priority_is_fifo():
    rng = np.random.default_rng(21)
    from swarmdb_b200._native import RECV_PEEK, RECV_PRIORITY
    A = 64
    g, c = _pair(A, ring_slots=4096)
    idx = np.arange(A, dtype=np.uint32)
    g.register(idx); c.register(idx)
    for rnd in range(4):
        n = 20000
        s = rng.integers(0, A, n); r = rng.integers(0, A, n)
        prio = rng.integers(0, 4, n)
        lens, off, buf = _mk_payloads(rng, n, 64)
        g.send_batch(s, r, prio, None, lens, off, buf); c.send_batch(s, r, prio, None, lens, off, buf)
        for k in (1, 5, 33, 100):
            _same(g.receive_batch(idx, k, RECV_PRIORITY | RECV_PEEK), c.receive_batch(idx, k, RECV_PRIORITY | RECV_PEEK))
            _same(g.receive_batch(idx, k, RECV_PRIORITY), c.receive_batch(idx, k, RECV_PRIORITY))
        # stream-order receive while holes exist (peek first: same selection, nothing retired)
        _same(g.receive_batch(idx, 17, RECV_PEEK), c.receive_batch(idx, 17, RECV_PEEK))
        _same(g.receive_batch(idx, 17, 0), c.receive_batch(idx, 17, 0))
    while True:
        rg, rc = g.receive_batch(idx, 100, RECV_PRIORITY), c.receive_batch(idx, 100, RECV_PRIORITY)
        _same(rg, rc)
        if len(rg[1]) == 0:
            break
    # equal priorities: priority mode must equal stream order (the tie-break obligation)
    n = 5000
    s = rng.integers(0, A, n); r = rng.integers(0, A, n)
    lens, off, buf = _mk_payloads(rng, n, 32)
    g.send_batch(s, r, np.full(n, 2), None, lens, off, buf); c.send_batch(s, r, np.full(n, 2), None, lens, off, buf)
    _same(g.receive_batch(idx, 40, RECV_PRIORITY), c.receive_batch(idx, 40, 0))
    _same(g.receive_batch(idx, 1000, 0), c.receive_batch(idx, 1000, RECV_PRIORITY))


def test_ring_overflow_is_reported_not_silent():
    rng = np.random.default_rng(2)
    g, c = _pair(8, ring_slots=4)
    lens, off, buf = _mk_payloads(rng, 10, 16)
    base0 = g.stats()["next_seq"]
    g.send_batch(np.zeros(10), np.ones(10), None, None, lens, off, buf)
    st = g.stats()
    assert st["enqueued"] == 4 and st["ring_overflow"] == 6
    cnt, hdr, pay = g.receive_batch([1], 100)
    assert cnt[0] == 4
    assert hdr["seq"].tolist() == [base0 + k for k in range(4)]     # ranked enqueue: the FIRST sends of the batch are the ones kept
    ag, sq, dropped = g.overflow_log()                      # which records were lost, not only how many
    assert dropped == 6 and ag.tolist() == [1] * 6 and sorted(sq.tolist()) == [base0 + k for k in range(4, 10)]
    assert g.overflow_log()[2] == 0                         # reading clears the log
    # ring usable again afterwards
    g.send_batch(np.zeros(3), np.ones(3), None, None, lens[:3], off[:3], buf)
    assert g.receive_batch([1], 100)[0][0] == 3
    # a partly filled ring: 3 pending + 5 more -> one slot left, four overflow; other receivers are not affected
    g.send_batch(np.zeros(3), np.ones(3), None, None, lens[:3], off[:3], buf)
    base = g.stats()["next_seq"]
    g.send_batch(np.zeros(7), np.array([1, 2, 1, 1, 2, 1, 1]), None, None, lens[:7], off[:7], buf)
    st2 = g.stats()
    assert st2["ring_overflow"] == 6 + 4
    cnt, hdr, _ = g.receive_batch([1, 2], 100)
    assert cnt.tolist() == [4, 2]
    assert hdr["seq"][3] == base and hdr["seq"][4:].tolist() == [base + 1, base + 4]
    ag, sq, dropped = g.overflow_log()
    assert dropped == 4 and sorted(sq.tolist()) == [base + 2, base + 3, base + 5, base + 6]
    # group fan-out through the owner-computes index build (batch above the pull threshold) and a broadcast list
    g2, _ = _pair(20000, max_groups=2, ring_slots=4, max_batch_sends=64)
    members = np.arange(17000, dtype=np.uint32)
    g2.create_group(0, members)
    lens2, off2, buf2 = _mk_payloads(rng, 6, 16)
    b2 = g2.stats()["next_seq"]
    g2.send_group_batch(np.full(6, 19999), np.zeros(6), None, None, lens2, off2, buf2)       # 6 sends x 17000 members, 4 slots each
    ag, sq, dropped = g2.overflow_log()
    assert dropped == 2 * 17000 and len(sq) == 4096
    rel = sq - b2                                             # seq = base + send * 17000 + member position
    assert set((rel // 17000).tolist()) <= {4, 5} and np.array_equal(rel % 17000, ag)
    assert g2.receive_batch(members, 100)[0].tolist() == [4] * 17000
    lo = np.array([0, 17000, 34000, 51000, 68000, 85000, 102000], np.uint64)
    g2.send_list_batch(np.full(6, 19999), lo, np.tile(members, 6), None, None, lens2, off2, buf2)
    ag, sq, dropped = g2.overflow_log()
    b3 = g2.stats()["next_seq"] - 6
    assert dropped == 2 * 17000 and set((sq - b3).tolist()) <= {4, 5}                         # a broadcast is ONE sequence number
    g2.close()


def test_ranked_p2p_enqueue_many_per_receiver_and_staged_resubmit():
    """Pure point-to-point batches are ranked per receiver at staging time (slot = ctail + rank, no atomics, no
    commit sort): heavy fan-in on a few receivers, empty payloads, a staged batch submitted twice, receives in
    between - every stream must equal the oracle's."""
    from swarmdb_b200._native import RECV_PRIORITY
    rng = np.random.default_rng(61)
    A = 64
    g, c = _pair(A, ring_slots=16384)
    idx = np.arange(A, dtype=np.uint32)
    for rnd in range(6):
        n = 3000
        s = rng.integers(0, A, n)
        r = np.where(rng.random(n) < 0.7, rng.integers(0, 3, n), rng.integers(0, A, n))      # 70 % to three receivers
        prio = rng.integers(0, 4, n)
        lens, off, buf = _mk_payloads(rng, n, 256)
        lens[rng.random(n) < 0.1] = 0
        g.send_batch(s, r, prio, None, lens, off, buf); c.send_batch(s, r, prio, None, lens, off, buf)
        if rnd % 2:
            _same(g.receive_batch(idx, 500, RECV_PRIORITY if rnd == 3 else 0), c.receive_batch(idx, 500, RECV_PRIORITY if rnd == 3 else 0))
    st = g.stage(0, s, r, prio, None, lens, off, buf)
    for _ in range(2):
        g.submit(st); c.send_batch(s, r, prio, None, lens, off, buf)
    _same(g.receive_batch(idx, 100000), c.receive_batch(idx, 100000))
    assert g.stats()["ring_overflow"] == 0


def test_arena_wraps_and_reclaims():
    rng = np.random.default_rng(4)
    A = 32
    g, c = _pair(A, arena_bytes=1 << 16, ring_slots=64)      # 64 KiB arena: wraps every few batches
    idx = np.arange(A, dtype=np.uint32)
    for rnd in range(40):
        n = 100
        s = rng.integers(0, A, n); r = rng.integers(0, A, n)
        lens, off, buf = _mk_payloads(rng, n, 200)
        g.send_batch(s, r, None, None, lens, off, buf); c.send_batch(s, r, None, None, lens, off, buf)
        _same(g.receive_batch(idx, 1000), c.receive_batch(idx, 1000))
    st = g.stats()
    assert st["arena_tail_bytes"] > 4 * (1 << 16)
    # an undrained backlog larger than the arena must be refused, not overwritten
    from swarmdb_b200._native import SdbError
    with pytest.raises(SdbError):
        for _ in range(40):
            lens, off, buf = _mk_payloads(rng, 100, 200, fixed=True)
            g.send_batch(rng.integers(0, A, 100), rng.integers(0, A, 100), None, None, lens, off, buf)


def test_receive_capacity_truncates_by_whole_agents_without_loss():
    rng = np.random.default_rng(8)
    A = 50
    g, c = _pair(A, max_recv_records=64, ring_slots=256)
    idx = np.arange(A, dtype=np.uint32)
    n = 2000
    s = rng.integers(0, A, n); r = rng.integers(0, A, n)
    lens, off, buf = _mk_payloads(rng, n, 64)
    g.send_batch(s, r, None, None, lens, off, buf); c.send_batch(s, r, None, None, lens, off, buf)
    got = {a: [] for a in range(A)}
    for _ in range(1000):
        cnt, hdr, pay = g.receive_batch(idx, 30)             # at most 2 agents x 30 fit in 64 records
        if len(hdr) == 0:
            break
        assert len(hdr) <= 64
        pos = 0
        for a in range(A):
            got[a].extend(hdr["seq"][pos:pos + cnt[a]].tolist()); pos += cnt[a]
    cc, hc, pc = c.receive_batch(np.arange(A, dtype=np.uint32), 100000)
    pos = 0
    for a in range(A):
        assert got[a] == hc["seq"][pos:pos + cc[a]].tolist(); pos += cc[a]


@pytest.mark.parametrize("mode", [0, 1])
def test_backend_select_matches_oracle(mode):
    rng = np.random.default_rng(5)
    g, c = _pair(4)
    w = rng.integers(1, 9, 256); l0 = rng.integers(0, 50, 256)
    g.set_backends(w, l0); c.set_backends(w, l0)
    for n in (1, 1000, 100000):
        pg, pc = g.select_backends(n, None, mode, seed=6), c.select_backends(n, None, mode, seed=6)
        assert np.array_equal(pg, pc)
        assert np.array_equal(g.backend_loads(), c.backend_loads())
    cost = rng.integers(1, 20, 5000)
    assert np.array_equal(g.select_backends(5000, cost, mode, seed=7), c.select_backends(5000, cost, mode, seed=7))
    assert np.array_equal(g.backend_loads(), c.backend_loads())
    g.release_backends([0, 1, 1], [1, 2, 3])


@pytest.mark.parametrize("max_len", [4096, 8192, 60000])
def test_large_payloads_all_kernel_variants(max_len):
    """Payloads above 4 KiB leave the warp-per-send kernel for the CTA-per-send variants."""
    rng = np.random.default_rng(max_len)
    A, G = 300, 6
    for variant in (0, 1, 2, 3):
        g, c = _pair(A, max_groups=G, fanout_variant=variant, max_payload_bytes=max_len, arena_bytes=1 << 28,
                     max_batch_sends=64, max_batch_payload=64 * ((max_len + 31) & ~31) + 64, ring_slots=256,
                     max_recv_records=4096, max_recv_payload=1 << 28)
        groups = [rng.choice(A, size=int(rng.integers(1, 70)), replace=False) for _ in range(G)]
        for k, m in enumerate(groups):
            g.create_group(k, m); c.create_group(k, m)
        n = 40
        lens, off, buf = _mk_payloads(rng, n, max_len)
        lens[0] = max_len; lens[1] = 0
        s = rng.integers(0, A, n); grp = rng.integers(0, G, n); prio = rng.integers(0, 4, n)
        assert g.send_group_batch(s, grp, prio, None, lens, off, buf) == c.send_group_batch(s, grp, prio, None, lens, off, buf)[0]
        r = rng.integers(0, A, n)
        g.send_batch(s, r, prio, None, lens, off, buf); c.send_batch(s, r, prio, None, lens, off, buf)
        idx = np.arange(A, dtype=np.uint32)
        _same(g.receive_batch(idx, 3), c.receive_batch(idx, 3, pay_cap=1 << 29))
        _same(g.receive_batch(idx, 1000), c.receive_batch(idx, 1000, pay_cap=1 << 29))
        g.close(); c.close()


def test_ring_handles_wrap_at_2_pow_32_granules():
    """Ring handles are the low 32 bits of the arena position: run batches across the 2^32 boundary."""
    rng = np.random.default_rng(77)
    A, G = 500, 8
    g, c = _pair(A, max_groups=G, arena_bytes=1 << 24, ring_slots=512)
    groups = [rng.choice(A, size=40, replace=False) for _ in range(G)]
    for k, m in enumerate(groups):
        g.create_group(k, m); c.create_group(k, m)
    g.debug_set_arena_pos((1 << 32) - 20000)             # ~20k granules before the handles wrap
    idx = np.arange(A, dtype=np.uint32)
    from swarmdb_b200._native import RECV_PRIORITY
    for step in range(6):
        n = 60
        lens, off, buf = _mk_payloads(rng, n, 200)
        s = rng.integers(0, A, n); grp = rng.integers(0, G, n); prio = rng.integers(0, 4, n)
        g.send_group_batch(s, grp, prio, None, lens, off, buf); c.send_group_batch(s, grp, prio, None, lens, off, buf)
        r = rng.integers(0, A, 200); l2, o2, b2 = _mk_payloads(rng, 200, 64); s2 = rng.integers(0, A, 200)
        g.send_batch(s2, r, None, None, l2, o2, b2); c.send_batch(s2, r, None, None, l2, o2, b2)
        flags = RECV_PRIORITY if step % 2 else 0
        _same(g.receive_batch(idx, 4, flags), c.receive_batch(idx, 4, flags))       # leaves a backlog that straddles the wrap
    _same(g.receive_batch(idx, 10000), c.receive_batch(idx, 10000))
    assert g.stats()["arena_tail_bytes"] > (1 << 32) * 32


@pytest.mark.parametrize("per_agent", [40, 1500, 5000])
def test_many_records_for_one_agent_in_one_batch(per_agent):
    """commit must order a hot receiver's entries: register network (<=16), shared-memory bitonic sort
    (<=4096) and the in-ring odd-even sort beyond that."""
    rng = np.random.default_rng(per_agent)
    A = 64
    g, c = _pair(A, ring_slots=16384, arena_bytes=1 << 26, max_batch_sends=3 * per_agent, max_batch_payload=3 * per_agent * 32 + 64,
                 max_recv_records=1 << 16)
    n = 3 * per_agent
    recv = np.concatenate([np.full(per_agent, 5), np.full(per_agent, 9), rng.integers(0, A, per_agent)])
    rng.shuffle(recv)
    lens, off, buf = _mk_payloads(rng, n, 32)
    s = rng.integers(0, A, n); prio = rng.integers(0, 4, n)
    for _ in range(2):
        g.send_batch(s, recv, prio, None, lens, off, buf); c.send_batch(s, recv, prio, None, lens, off, buf)
    idx = np.arange(A, dtype=np.uint32)
    _same(g.receive_batch(idx, 100000), c.receive_batch(idx, 100000))
    assert g.stats()["ring_overflow"] == 0


def test_long_broadcast_lists_are_chunked_without_changing_results():
    """Lists longer than the descriptor chunk (1024 recipients) are split into several descriptors on the host:
    same sequence number on every copy, same per-recipient order against p2p traffic before and after."""
    rng = np.random.default_rng(31)
    A = 6000
    g, c = _pair(A, list_pool_entries=1 << 16, ring_slots=64, arena_bytes=1 << 27, max_recv_records=1 << 17)
    idx = np.arange(A, dtype=np.uint32)
    g.register(idx); c.register(idx)
    sizes = [0, 1, 1023, 1024, 1025, 2048, 5000, 6000]
    lists = [rng.choice(A, size=k, replace=False) for k in sizes]
    n = len(lists)
    lo = np.zeros(n + 1, np.uint64); lo[1:] = np.cumsum(sizes)
    li = np.concatenate(lists).astype(np.uint32)
    s = rng.integers(0, A, n); prio = rng.integers(0, 4, n); typ = rng.integers(0, 7, n)
    lens, off, buf = _mk_payloads(rng, n, 200)
    lens[3] = 0                                              # one long list without payload bytes
    l2, o2, b2 = _mk_payloads(rng, 300, 64)
    s2 = rng.integers(0, A, 300); r2 = rng.integers(0, A, 300)
    for sys in (g, c):
        sys.send_batch(s2, r2, None, None, l2, o2, b2)
        assert sys.send_list_batch(s, lo, li, prio, typ, lens, off, buf) == 301      # one sequence number per broadcast
        sys.send_batch(r2, s2, None, None, l2, o2, b2)
    assert g.stats()["next_seq"] == c.next_seq == 301 + n + 300
    _same(g.receive_batch(idx, 3), c.receive_batch(idx, 3))
    _same(g.receive_batch(idx, 1000, 1), c.receive_batch(idx, 1000, 1))
    # the same through a mixed batch (kind 2 = list number)
    kind = np.array([2, 0, 2, 2], np.uint8); target = np.array([6, 17, 7, 0], np.uint32)
    lens4, off4, buf4 = _mk_payloads(rng, 4, 96)
    g.send_mixed_batch([1, 2, 3, 4], kind, target, lo, li, None, None, lens4, off4, buf4)
    for i in range(4):                                       # the oracle takes the same sends one by one
        one = slice(i, i + 1)
        if kind[i] == 0:
            c.send_batch([i + 1], target[one], None, None, lens4[one], off4[one], buf4)
        else:
            t = int(target[i])
            c.send_list_batch([i + 1], [0, sizes[t]], lists[t], None, None, lens4[one], off4[one], buf4)
    _same(g.receive_batch(idx, 1000), c.receive_batch(idx, 1000))


def test_async_receive_enqueues_and_reports_totals_later():
    """SDB_RECV_ASYNC: the receive is only enqueued; totals and device-resident results are read afterwards."""
    from swarmdb_b200._native import HDR_DTYPE, RECV_ASYNC, SdbError
    rng = np.random.default_rng(41)
    A, n = 300, 4000
    g, c = _pair(A, ring_slots=256)
    idx = np.arange(A, dtype=np.uint32)
    g.register(idx); c.register(idx)
    s = rng.integers(0, A, n); r = rng.integers(0, A, n)
    lens, off, buf = _mk_payloads(rng, n, 96)
    g.send_batch(s, r, None, None, lens, off, buf); c.send_batch(s, r, None, None, lens, off, buf)
    assert g.receive_batch(None, 5, 0, copy_out=False, wait=False) == (None, None, None)
    cc, hc, pc = c.receive_batch(idx, 5)
    total, pbytes = g.last_receive_totals()
    assert total == len(hc) and pbytes == len(pc)
    cnt_dev, hdr_dev, pay_dev = g.last_receive_dev()
    from cuda.bindings import runtime as cudart                              # cuda-python: plain D2H of the device-resident results
    hdr = np.zeros(total, HDR_DTYPE); pay = np.zeros(pbytes, np.uint8)
    d2h = cudart.cudaMemcpyKind.cudaMemcpyDeviceToHost
    assert cudart.cudaMemcpy(hdr.ctypes.data, hdr_dev, hdr.nbytes, d2h)[0] == cudart.cudaError_t.cudaSuccess
    assert cudart.cudaMemcpy(pay.ctypes.data, pay_dev, pay.nbytes, d2h)[0] == cudart.cudaError_t.cudaSuccess
    assert hdr.tobytes() == hc.tobytes() and pay.tobytes() == pc.tobytes()
    _same(g.receive_batch(idx, 1000), c.receive_batch(idx, 1000))            # the rest, synchronously
    assert g.stats()["delivered"] == n
    with pytest.raises(SdbError):                                            # host outputs and ASYNC exclude each other
        g.receive_batch(idx, 5, RECV_ASYNC)


def test_latency_server_answers_like_the_ordinary_path():
    """sdb_latency_server: single-agent receives served by the persistent kernel (mailbox + answer in pinned host memory)
    return exactly what the launched path returns - stream and priority order, peeks, empty queues, traffic arriving
    between requests, and a stop/restart around a call that frees device memory."""
    rng = np.random.default_rng(77)
    A = 300
    g, c = _pair(A, ring_slots=512)
    idx = np.arange(A, dtype=np.uint32)
    g.register(idx); c.register(idx)
    g.latency_server(True)
    from swarmdb_b200._native import RECV_PEEK, RECV_PRIORITY
    for rnd in range(4):
        n = 2000
        s = rng.integers(0, A, n); r = rng.integers(0, A, n)
        prio = rng.integers(0, 4, n); typ = rng.integers(0, 7, n)
        lens, off, buf = _mk_payloads(rng, n, 256)
        ts = rng.random(n)
        assert g.send_batch(s, r, prio, typ, lens, off, buf, ts) == c.send_batch(s, r, prio, typ, lens, off, buf, ts)
        for a in rng.integers(0, A, 60):
            flags = [0, RECV_PRIORITY, RECV_PEEK, RECV_PEEK | RECV_PRIORITY][int(rng.integers(0, 4))]
            k = int(rng.integers(1, 9))
            hg, pg, _ = g.receive_one(int(a), k, flags)
            cc, hc, pc = c.receive_batch([int(a)], k, flags)
            assert hg.tobytes() == hc.tobytes() and pg.tobytes() == pc.tobytes(), (rnd, a, flags)
        if rnd == 1:
            st = g.stage(0, s[:10], r[:10], prio[:10], typ[:10], lens[:10], off[:10], buf)
            g.free_staged(st)                                   # cudaFree inside: the server is stopped and restarted
    _same(g.receive_batch(idx, 10000), c.receive_batch(idx, 10000))       # the bulk path sees the same queue state
    hg, pg, _ = g.receive_one(5, 10, 0)
    assert len(hg) == 0
    g.latency_server(False)
    st = g.stats()
    assert st["enqueued"] == st["delivered"] == 8000
    g.close(); c.close()


@pytest.mark.parametrize("shape", ["one_shared_list", "disjoint_lists_mixed_api", "overlapping_lists"])
def test_broadcast_batches_owner_computes_index_equals_oracle(shape):
    """Pure broadcast batches whose recipient lists are pairwise disjoint (typically ONE list shared by every
    broadcast of the batch) build their ring entries with k_list_index - no atomics, no commit sort; overlapping
    lists keep the atomic path.  Either way every stream must equal the oracle's (M:449-463, M:810-850)."""
    from swarmdb_b200._native import RECV_PRIORITY
    rng = np.random.default_rng({"one_shared_list": 5, "disjoint_lists_mixed_api": 6, "overlapping_lists": 7}[shape])
    A = 6000
    g, c = _pair(A, ring_slots=256, list_pool_entries=1 << 18, max_recv_records=1 << 19)
    idx = np.arange(A, dtype=np.uint32)
    # something pending beforehand, so that the entries are appended behind existing ones
    lens, off, buf = _mk_payloads(rng, 500, 64)
    s0, r0 = rng.integers(0, A, 500), rng.integers(0, A, 500)
    g.send_batch(s0, r0, None, None, lens, off, buf); c.send_batch(s0, r0, None, None, lens, off, buf)
    g.profile(True)
    for rnd in range(3):
        n = 40
        lens, off, buf = _mk_payloads(rng, n, 200)
        sender = rng.integers(0, A, n); prio = rng.integers(0, 4, n); typ = rng.integers(0, 7, n)
        if shape == "one_shared_list":
            everybody = rng.permutation(A)[:3000].astype(np.uint32)
            lo = np.arange(n + 1, dtype=np.uint64) * len(everybody)
            li = np.tile(everybody, n)
            g.send_list_batch(sender, lo, li, prio, typ, lens, off, buf); c.send_list_batch(sender, lo, li, prio, typ, lens, off, buf)
        else:
            perm = rng.permutation(A).astype(np.uint32)
            if shape == "disjoint_lists_mixed_api":
                lists = [perm[:2500], perm[2500:2501], perm[2600:4000], perm[5000:5000]]          # one single, one empty
            else:
                lists = [perm[:2500], perm[2400:4000], perm[3000:3100]]
            lo = np.zeros(len(lists) + 1, np.uint64); lo[1:] = np.cumsum([len(x) for x in lists])
            li = np.concatenate(lists)
            which = rng.integers(0, 3 if shape != "disjoint_lists_mixed_api" else 4, n)
            g.send_mixed_batch(sender, np.full(n, 2, np.uint8), which, lo, li, prio, typ, lens, off, buf)
            lo2 = np.zeros(n + 1, np.uint64); lo2[1:] = np.cumsum([len(lists[w]) for w in which])
            c.send_list_batch(sender, lo2, np.concatenate([lists[w] for w in which]) if lo2[-1] else np.zeros(0, np.uint32),
                              prio, typ, lens, off, buf)
        k = [5, 1000, 7][rnd]
        _same(g.receive_batch(idx, k, RECV_PRIORITY if rnd == 2 else 0), c.receive_batch(idx, k, RECV_PRIORITY if rnd == 2 else 0, rec_cap=1 << 19))
    _same(g.receive_batch(idx, 100000), c.receive_batch(idx, 100000, rec_cap=1 << 19))
    prof = g.profile_read()
    st = g.stats()
    assert st["ring_overflow"] == 0 and st["enqueued"] == st["delivered"]
    if shape == "overlapping_lists":
        assert prof.get("index", (0, 0))[1] == 0 and prof["commit"][1] == 3          # atomic path + commit sort
    else:
        assert prof["index"][1] == 3 and prof.get("commit", (0, 0))[1] == 0          # owner-computes, nothing to sort


def test_receive_list_naming_an_agent_twice_is_refused():
    """Every slot of a listed agent would read the same ring header and return the same records twice: a receive list
    with a repeated index is refused with SDB_EINVAL on the small path and on the bulk path, and consumes nothing."""
    from swarmdb_b200._native import RECV_PEEK, RECV_PRIORITY, SdbError
    rng = np.random.default_rng(88)
    A = 300
    g, c = _pair(A, ring_slots=256)
    idx = np.arange(A, dtype=np.uint32)
    g.register(idx); c.register(idx)
    n = 3000
    s, r, prio = rng.integers(0, A, n), rng.integers(0, A, n), rng.integers(0, 4, n)
    lens, off, buf = _mk_payloads(rng, n, 64)
    g.send_batch(s, r, prio, None, lens, off, buf); c.send_batch(s, r, prio, None, lens, off, buf)
    bulk = np.concatenate([idx[:200], [17]]).astype(np.uint32)
    for agents, k in (([5, 9, 5], 4), ([7, 7], 1), (bulk, 50), (np.concatenate([idx[1:], idx[-1:]]), 1000)):
        for flags in (0, RECV_PRIORITY, RECV_PEEK):
            with pytest.raises(SdbError) as ei:
                g.receive_batch(np.asarray(agents, np.uint32), k, flags)
            assert ei.value.code == -1 and "twice" in str(ei.value)
    assert g.stats()["delivered"] == 0
    _same(g.receive_batch([5, 9, 7], 4), c.receive_batch([5, 9, 7], 4))               # the table is clean afterwards
    _same(g.receive_batch(idx, 1000), c.receive_batch(idx, 1000))
    g.close(); c.close()
