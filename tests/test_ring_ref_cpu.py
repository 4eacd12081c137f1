"""The bounded-ring model (tests/ring_ref.py) on its own and over the CPU oracle.  No GPU:
tests/test_gpu_ring_capacity.py holds the device to the same model."""
import numpy as np
import pytest

from tests.ring_ref import BoundedOracle, RingModel

A, G = 16, 2


def _bounded(R, groups=None):
    from oracle.cpu_ref import CpuOracle
    o = BoundedOracle(CpuOracle(A, G), G, R)
    o.register(np.arange(A, dtype=np.uint32))
    for g, m in (groups or {}).items():
        o.create_group(g, m)
    return o


def _p2p(o, receivers, prio=None, sender=0):
    n = len(receivers)
    lens = np.full(n, 8, np.uint16)
    off = np.arange(n, dtype=np.uint64) * 32
    buf = np.arange(n * 32 + 64, dtype=np.uint64).astype(np.uint8)
    return o.send_batch(np.full(n, sender), receivers, prio, None, lens, off, buf)


def _worked_example(retire):
    """R = 64, one agent sent 41 records: priority 0, 39 at priority 3, priority 0.  A priority receive of 39 leaves
    tombstones 1-39 with head at record 0; `retire` then takes record 0, and a ranked batch of 64 records follows."""
    from tests.where_ref import RECV_PRIORITY
    o = _bounded(64)
    base = _p2p(o, [5] * 41, [0] + [3] * 39 + [0])
    _, hdr, _ = o.receive_batch([5], 39, RECV_PRIORITY)
    assert hdr["seq"].tolist() == list(range(base + 1, base + 40))
    assert o.ring.span(5) == 41 and o.ring.ntomb(5) == 39 and o.ring.head[5] == 0
    retire(o)
    assert o.ring.live_seqs(5) == [base + 40]
    assert o.ring.span(5) == 1 and o.ring.ntomb(5) == 0 and o.ring.head[5] == 40
    b2 = _p2p(o, [5] * 64)
    assert o.take_dropped() == [(5, b2 + 63)]                       # 63 records kept, not 55
    cnt, hdr, _ = o.receive_batch([5], 100)
    assert hdr["seq"].tolist() == [base + 40] + list(range(b2, b2 + 63))
    o.close()


def test_worked_example_stream_receive():
    _worked_example(lambda o: o.receive_batch([5], 1))


def test_worked_example_where_take():
    from swarmdb_b200._native import make_filter
    _worked_example(lambda o: o.receive_where([5], 1, 0, make_filter()))


def test_worked_example_expiry():
    from tests.expire_ref import EXPIRE_ALL
    _worked_example(lambda o: o.expire([5], 0.0, EXPIRE_ALL, rec_cap=1))


def test_hand_built_windows_cursor_arithmetic():
    """The model's head, tail and capacity on hand-built windows: long runs of tombstones, leading tombstones, a window
    exactly R long.  The model has no physical slots; chunk and wrap positions are exercised on the device
    (tests/test_gpu_ring_capacity.py)."""
    R, head = 1024, 1000
    m = RingModel(R)
    # live at 0, tombstones over [1, 160), live at 160 and 161, tombstone, live at 163
    slots = [(0, True)] + [(k, False) for k in range(1, 160)] + [(160, True), (161, True), (162, False), (163, True)]
    m.set_window(1, head, slots)
    assert m.span(1) == 164 and m.capacity(1) == R - 164 and m.ntomb(1) == 160
    m.retire(1, [0])
    assert m.head[1] == head + 160 and m.span(1) == 4 and m.ntomb(1) == 1
    m.retire(1, [161, 160])
    assert m.head[1] == head + 163 and m.span(1) == 1 and m.ntomb(1) == 0
    # leading tombstones never form a window start
    m.set_window(2, head, [(k, False) for k in range(40)] + [(40, True)])
    assert m.head[2] == head + 40 and m.span(2) == 1
    # exactly R long: nothing fits, a restore of one record is refused, one retire at the start frees one slot
    m.set_window(3, head, [(k, k % 3 != 1) for k in range(R)])
    assert m.capacity(3) == 0 and not m.fits([3], [1]) and m.fits([3], [0])
    assert m.offer(3, [5000, 5001]) == ([], [5000, 5001])
    m.retire(3, [0])
    assert m.head[3] == head + 2 and m.capacity(3) == 2 and m.fits([3], [2]) and not m.fits([3], [3])
    assert m.offer(3, [5000, 5001, 5002]) == ([5000, 5001], [5002])
    assert m.tail(3) == head + R + 2
    # a tombstone in the middle of a window still counts against capacity
    m.set_window(4, head, [(0, True), (1, False), (2, True)])
    assert m.capacity(4) == R - 3


def test_duplicate_seq_in_one_window_consumes_the_earlier_slot():
    m = RingModel(8)
    m.set_window(0, 0, [(7, True), (8, True), (7, True)])
    m.retire_to(0, [8, 7])                                           # one copy of 7 left: the later one
    assert m.window(0) == [[8, True], [7, True]] and m.head[0] == 1
    m.set_window(1, 0, [(7, True), (8, True), (7, True)])
    m.retire(1, [7])
    assert m.window(1) == [[8, True], [7, True]]


def test_agrees_with_the_unbounded_oracle_when_rings_are_large():
    """R larger than all traffic: the bounded oracle drops nothing and answers every call as the plain oracle does."""
    from oracle.cpu_ref import CpuOracle
    from swarmdb_b200._native import make_filter
    from tests.where_ref import RECV_PRIORITY
    rng = np.random.default_rng(3)
    groups = {0: np.arange(0, 6, dtype=np.uint32), 1: np.arange(4, 12, dtype=np.uint32)}
    o, c = _bounded(1 << 12, groups), CpuOracle(A, G)
    c.register(np.arange(A, dtype=np.uint32))
    for g, mm in groups.items():
        c.create_group(g, mm)
    for rnd in range(6):
        n = 60
        s, r, p = rng.integers(0, A, n), rng.integers(0, A, n), rng.integers(0, 4, n)
        lens = rng.integers(0, 64, n).astype(np.uint16)
        off = np.arange(n, dtype=np.uint64) * 64
        buf = rng.integers(0, 256, n * 64 + 64).astype(np.uint8)
        assert o.send_batch(s, r, p, None, lens, off, buf) == c.send_batch(s, r, p, None, lens, off, buf)
        assert o.send_group_batch(s[:4], [0, 1, 0, 1], p[:4], None, lens[:4], off[:4], buf) == \
            c.send_group_batch(s[:4], [0, 1, 0, 1], p[:4], None, lens[:4], off[:4], buf)
        lo = np.array([0, 3, 5], np.uint64)
        li = np.array([1, 2, 1, 9, 9], np.uint32)                      # agent 1 and 9 listed twice
        assert o.send_list_batch(s[:2], lo, li, p[:2], None, lens[:2], off[:2], buf) == \
            c.send_list_batch(s[:2], lo, li, p[:2], None, lens[:2], off[:2], buf)
        ag = rng.permutation(A)[:10].astype(np.uint32)
        k, flags = int(rng.integers(1, 6)), int(rng.integers(0, 2)) * RECV_PRIORITY
        a1, a2 = o.receive_batch(ag, k, flags), c.receive_batch(ag, k, flags)
        assert all(x.tobytes() == y.tobytes() for x, y in zip(a1, a2)), rnd
        if rnd % 2:                                                   # a where take equals a receive on the oracle
            w1 = o.receive_where(ag[:3], 2, 0, make_filter())
            w2 = c.receive_batch(ag[:3], 2)
            assert all(x.tobytes() == y.tobytes() for x, y in zip(w1, w2)), rnd
    assert o.take_dropped() == [] and o.overflow == 0
    for a in range(A):
        assert o.ring.span(a) - o.ring.ntomb(a) == int(c.pending(a))
    ld_o, ld_c = o.agent_loads(np.arange(A)), c.agent_loads(np.arange(A))
    assert ld_o.tobytes() == ld_c.tobytes()
    o.close(); c.close()


def test_overflow_drops_the_last_records_of_a_ranked_batch():
    """Agent 3 is sent ten records into an empty 8-slot ring: the last two are dropped, leave the oracle (replay) and
    are not counted as received."""
    o = _bounded(8)
    b = _p2p(o, [3, 4, 3, 3, 4, 3, 3, 3, 3, 3, 3, 3])
    assert o.take_dropped() == [(3, b + 10), (3, b + 11)] and o.overflow == 2
    assert [int(x) for x in o.agent_loads([3, 4])["received"]] == [8, 2]
    assert o.receive_batch([3], 100)[1]["seq"].tolist() == [b, b + 2, b + 3, b + 5, b + 6, b + 7, b + 8, b + 9]
    assert o.ring.capacity(3) == 8
    o.close()


def test_atomic_claim_survivors_reconcile_the_model():
    o = _bounded(4)
    _p2p(o, [2, 2])
    b = o.next_seq
    o.enqueue(lambda: _p2p(o, [2] * 5), keep={2: [b + 1, b + 4]})
    assert sorted(o.take_dropped()) == [(2, b), (2, b + 2), (2, b + 3)]
    assert o.receive_batch([2], 10)[1]["seq"].tolist()[2:] == [b + 1, b + 4]
    with pytest.raises(AssertionError):                               # more survivors than the ring takes
        o.enqueue(lambda: _p2p(o, [2] * 6), keep={2: [o.next_seq + k for k in range(5)]})
    o.close()


def test_group_and_list_drops_need_the_path_declared():
    """A group or list send that overflows a ring may take an atomic-claim path on the device: the model refuses to
    guess which records survive unless the caller declares the path."""
    z = np.zeros(64, np.uint8)
    o = _bounded(2, {0: np.array([2, 3], np.uint32)})
    o.send_group_batch([0, 0], [0, 0], None, None, [8, 8], np.zeros(2, np.uint64), z)         # fits: no declaration
    with pytest.raises(AssertionError, match="atomic-claim"):
        o.send_group_batch([0], [0], None, None, [8], np.zeros(1, np.uint64), z)
    o.close()
    o = _bounded(2, {0: np.array([2, 3], np.uint32)})
    o.send_list_batch([0], [0, 2], [2, 3], None, None, [8], np.zeros(1, np.uint64), z)
    b = o.next_seq
    o.enqueue(lambda: o.send_group_batch([0, 0], [0, 0], None, None, [8, 8], np.zeros(2, np.uint64), z), ordered=True)
    assert o.take_dropped() == [(2, b + 2), (3, b + 3)]              # seq = base + send * F + member position
    assert o.ring.live_seqs(2) == [b - 1, b] and o.ring.capacity(2) == 0
    o.close()


def test_offer_order_for_an_agent_in_several_groups_and_listed_twice():
    """The index build merges an agent's records by (send, member position): group 0 lists agent 2 twice, group 1 holds
    it once, so a batch g0, g1, g0 delivers it positions 0 and 2 of send 0, position 1 of send 1, then send 2; a sender
    inside a group skips its own records.  A 4-slot ring keeps the first four."""
    z = np.zeros(64, np.uint8)
    o = _bounded(4, {0: np.array([2, 3, 2], np.uint32), 1: np.array([4, 2], np.uint32)})
    b = o.next_seq
    o.enqueue(lambda: o.send_group_batch([0, 0, 0, 2], [0, 1, 0, 1], None, None, [8] * 4, np.zeros(4, np.uint64), z),
              ordered=True)
    # records: send 0 -> b .. b+2 (2, 3, 2), send 1 -> b+3, b+4 (4, 2), send 2 -> b+5 .. b+7, send 3 (sender 2) -> b+8, b+9
    assert o.ring.live_seqs(2) == [b, b + 2, b + 4, b + 5]
    assert o.take_dropped() == [(2, b + 7)]
    assert o.ring.live_seqs(3) == [b + 1, b + 6] and o.ring.live_seqs(4) == [b + 3, b + 8]
    assert o.receive_batch([2], 10)[1]["seq"].tolist() == [b, b + 2, b + 4, b + 5]
    o.close()


def test_import_replayed_through_the_oracle_shard_with_composite_seqs():
    """A cross-shard import bounded as one call: OracleShard replays the wire into a BoundedOracle, keeps the members
    this rank owns, and numbers records from the wire's explicit (composite) sequence base, which the drops carry."""
    from tests.fake_shard import OracleShard
    z = np.zeros(64, np.uint8)
    members = np.array([2, 3, 4, 5], np.uint32)
    src, dst = OracleShard(A, G, 1, 2), OracleShard(A, G, 0, 2)
    dst.o = BoundedOracle(dst.o, G, 2)
    dst.o.register(np.arange(A, dtype=np.uint32))
    owner = np.arange(A) % 2                                          # even agents live on rank 0
    for sh in (src, dst):
        sh.set_agent_shards(owner)
        sh.create_group(0, members)
    sb = (5 << 40) + 1000
    cap = 1 << 14
    wire = np.zeros(cap, np.uint8)
    src.export_group_batch(np.zeros(3, np.uint32), np.zeros(3, np.uint32), np.zeros(3, np.uint8), np.zeros(3, np.uint8),
                           np.full(3, 8, np.uint16), np.zeros(3, np.uint64), z, wire, cap)
    hdr = wire[:56].view(np.int64).copy()
    hdr[4] = sb                                                       # the wire's explicit sequence base
    wire[:56] = hdr.view(np.uint8)
    with dst.o.appending(ordered=True):
        dst.import_wire_batches(1, wire, cap)
    # member position j of send i is record sb + 4 i + j; rank 0 owns agents 2 (position 0) and 4 (position 2)
    assert dst.o.ring.live_seqs(2) == [sb, sb + 4] and dst.o.ring.live_seqs(4) == [sb + 2, sb + 6]
    assert dst.o.take_dropped() == [(2, sb + 8), (4, sb + 10)]
    assert dst.o.ring.live_seqs(3) == [] and dst.o.overflow == 2
    src.close(); dst.close()


def test_keep_for_pull_and_atomic_entries_to_one_agent():
    """A mixed batch with group traffic above the pull threshold: the fan-out's atomic claims land before the index
    build appends, so the survivors need not be the first records of the call.  keep= takes any subsequence of the
    new records in seq order, of exactly as many records as the ring has free slots."""
    z = np.zeros(64, np.uint8)
    o = _bounded(4, {0: np.array([2, 3], np.uint32)})
    _p2p(o, [2])
    b = o.next_seq

    def mixed():
        o.send_group_batch([0, 0], [0, 0], None, None, [8, 8], np.zeros(2, np.uint64), z)     # b .. b+3
        _p2p(o, [2, 2, 3])                                                                      # b+4 .. b+6
    o.enqueue(mixed, keep={2: [b, b + 4, b + 5], 3: [b + 1, b + 3, b + 6]})
    assert sorted(o.take_dropped()) == [(2, b + 2)]
    assert o.ring.live_seqs(2)[1:] == [b, b + 4, b + 5] and o.ring.capacity(2) == 0
    assert o.ring.capacity(3) == 1
    with pytest.raises(AssertionError, match="survivors must fill the free slots"):     # agent 3 keeps none of three
        o.enqueue(mixed, keep={2: [], 3: []})
    o.close()


def test_lease_sweep_blocks_on_tombstones_not_on_pending():
    """Priority leases that leave record 0 behind fill the window: with R = 8 and the window 8 slots long, two records
    pending and six leased, a sweep of those six is blocked (pending + six would have fit)."""
    from tests.lease_ref import LeaseModel
    from tests.where_ref import RECV_PRIORITY
    o = _bounded(8)
    _p2p(o, [6] * 8, [0] + [3] * 6 + [0])
    m = LeaseModel(o, {}, rec_cap=64, cap=64)
    _, hdr, _, _ = m.lease([6], 6, 1.0, RECV_PRIORITY)
    assert len(hdr) == 6 and int(o.pending(6)) == 2 and o.ring.span(6) == 8
    assert m.sweep(1.0) == (0, 1, 0)
    o.receive_batch([6], 1)                                          # record 0 leaves: head jumps over the six tombstones
    assert o.ring.span(6) == 1
    assert m.sweep(1.0) == (6, 0, 0)
    assert o.ring.span(6) == 7 and o.ring.ntomb(6) == 0
    o.close()
