"""Ring capacity once a window holds tombstones, against the bounded-ring model (tests/ring_ref.py).

A send to a full ring is dropped, sdb_restore_compact refuses and sdb_lease_sweep blocks an agent, all by the rule
tail - head + count > ring_slots, where the window [head, tail) also holds tombstones (records consumed out of order by
priority receives, filtered takes and expiry).  So where head lands after a retiring call decides how many records the
ring takes next, and agent_loads cannot show it: pending = tail - head - ntomb is the same wherever head lands.  The
rule (include/swarmdb_b200.h) is that head is the oldest pending record after every retiring call.

Each test builds holey windows, retires records through one path (asserting from the profiler which kernel served the
call), then probes every agent with a ranked p2p batch of R records: the ring_overflow delta, the overflow log, the
survivors and agent_loads must equal the model's.
"""
import numpy as np
import pytest

from tests.ring_ref import BoundedOracle
from tests.test_gpu_receive_paths import EMPTY, Rig, _payloads, _same

pytestmark = pytest.mark.gpu

R = 256


@pytest.fixture(params=["1", "0"])
def shared(request, monkeypatch):
    monkeypatch.setenv("SDB_SHARED_PAYLOAD", request.param)
    return request.param == "1"


def _rig(seed, A, ring_slots=R, **kw):
    rig = Rig(np.random.default_rng(seed), A, ring_slots=ring_slots, **kw)
    rig.c = BoundedOracle(rig.c, 1, ring_slots, None, A)
    return rig


def _send_ts(rig, receivers, prio, ts):
    receivers = np.asarray(receivers, np.uint32)
    m = len(receivers)
    s = rig.rng.integers(0, rig.A, m)
    lens, off, buf = _payloads(rig.rng, m, rig.max_len)
    typ = rig.rng.integers(0, 7, m)
    assert rig.g.send_batch(s, receivers, prio, typ, lens, off, buf, ts) == \
        rig.c.send_batch(s, receivers, prio, typ, lens, off, buf, ts)


def _expand(res):
    from swarmdb_b200._native import expand_compact
    return (res[0],) + tuple(expand_compact(res[1], res[2], res[3]))


def _served(rig, kind):
    prof = rig.g.profile_read()
    assert prof[kind][1] >= 1, (kind, {k: c for k, (_, c) in prof.items() if c})
    rig.delivered = rig.g.stats()["delivered"]          # calls outside rig.recv: its running count follows


def _drain(rig):
    idx = np.arange(rig.A, dtype=np.uint32)
    while len(rig.recv(idx, 1 << 12, 0, "stream", what="drain")[1]):
        pass
    rig.check_loads(None, "drained")
    assert rig.g.queue_stats()["pending"] == 0


def _probe(rig, agents, what):
    """A ranked p2p batch of R records to each agent (interleaved): overflow count, log, survivors and loads."""
    agents = np.asarray(agents, np.uint32)
    R_ = rig.c.ring.R
    assert rig.g.overflow_log()[2] == 0
    rig.c.take_dropped()
    st0 = rig.g.stats()
    recv = rig.rng.permutation(np.repeat(agents, R_)).astype(np.uint32)
    rig.send(recv, rig.rng.integers(0, 4, len(recv)))
    want = rig.c.take_dropped()
    st1 = rig.g.stats()
    assert st1["ring_overflow"] - st0["ring_overflow"] == len(want), (what, st1["ring_overflow"] - st0["ring_overflow"], len(want))
    ag, sq, dropped = rig.g.overflow_log(1 << 16)
    assert dropped == len(want), what
    assert sorted(zip(ag.tolist(), sq.tolist())) == sorted(want), what
    rig.check_loads(None, what + " probe")
    for a in agents.tolist():
        assert rig.c.ring.span(a) == R_, (what, a)       # every probed ring is full: the model's windows are exact
    got = rig.g.receive_batch(agents, 2 * R_)
    _same(got, rig.c.receive_batch(agents, 2 * R_), what + " survivors")
    rig.delivered = rig.g.stats()["delivered"]


# window layouts: (priorities in arrival order, k of the priority receive that punches the holes)
LAYOUTS = {
    "ex41": ([0] + [3] * 39 + [0], 39),          # tombstones 1-39: head 0, the next live entry at 40
    "ex152": ([0] + [3] * 150 + [0], 150),       # tombstones across the 32- and 128-entry chunks
    "b201": ([2] * 160 + [3] * 40 + [0], 40),    # 40 tombstones right after the 160 records a C > 128 receive takes
}


def _retire_steps():
    """(layout, name, call): each retires the oldest record(s) of one agent through one path."""
    from swarmdb_b200._native import RECV_PRIORITY
    from tests.expire_ref import EXPIRE_ALL

    def recv(path, k=1, flags=0, pad=None):
        def f(rig, a):
            n = {"stream": 9, "priority": 9, "small": 2, "server": 1}[path] if pad is None else pad
            rig.recv(np.concatenate([[a], rig.empties[: n - 1]]).astype(np.uint32), k, flags, path, what=path)
            rig._set_server(False)
        return f

    def compact(rig, a):
        agents = np.concatenate([[a], rig.empties]).astype(np.uint32)
        _same(_expand(rig.g.receive_compact(agents, 1)), rig.c.receive_batch(agents, 1), "compact")
        _served(rig, "recv_compact")

    def leased(rig, a):
        _same(_expand(rig.g.receive_leased([a], 1, 1.0)[:4]), rig.c.receive_batch([a], 1), "leased")
        _served(rig, "lease")

    def where(drop):
        def f(rig, a):
            from swarmdb_b200._native import make_filter
            got = rig.g.receive_where([a], 1, 0, make_filter(), drop=drop)
            want = rig.c.receive_where([a], 1, 0, make_filter(), drop=drop)
            if drop:
                assert np.array_equal(got[0], want[0]) and got[1] == want[1]
            else:
                _same(got, want, "where")
            _served(rig, "where")
        return f

    def expire(archive, flags=0):
        def f(rig, a):
            got = rig.g.expire([a], 1.0, flags, archive=archive)
            if archive:
                _same(_expand(got), rig.c.expire([a], 1.0, flags), "expire archive")
            else:
                want = rig.c.expire([a], 1.0, flags, materialise=False)
                assert np.array_equal(got[0], want[0]) and got[1] == want[1]
            _served(rig, "expire")
        return f

    return [
        ("ex41", "stream plan", recv("stream")),
        ("ex41", "<= 8 agents", recv("small")),
        ("ex41", "latency server", recv("server")),
        ("ex41", "priority, C <= 128", recv("priority", flags=RECV_PRIORITY)),
        ("ex41", "compact", compact),
        ("ex41", "leased", leased),
        ("ex41", "where take", where(False)),
        ("ex41", "where drop", where(True)),
        ("ex41", "expire drop", expire(False)),
        ("ex41", "expire archive", expire(True)),
        ("ex41", "expire all", expire(False, EXPIRE_ALL)),
        ("ex152", "stream plan", recv("stream")),
        ("ex152", "<= 8 agents", recv("small")),
        ("ex152", "latency server", recv("server")),
        ("ex152", "priority, C <= 128", recv("priority", 2, RECV_PRIORITY)),
        ("b201", "priority, C > 128", recv("priority", 160, RECV_PRIORITY)),
        ("b201", "<= 8 agents, priority", recv("small", 160, RECV_PRIORITY)),
        ("b201", "latency server, priority", recv("server", 160, RECV_PRIORITY)),
    ]


@pytest.mark.parametrize("wrapped", [False, True])
def test_head_lands_on_the_oldest_pending_record_on_every_path(shared, wrapped):
    """Holey windows (tombstones left by a priority receive), then one retiring call per agent and path, then the
    probe.  wrapped: every window starts at slot 200 of 256, so the holes cross the ring's physical wrap."""
    from swarmdb_b200._native import RECV_PRIORITY
    steps = _retire_steps()
    A = EMPTY + len(steps)
    rig = _rig(11 + wrapped, A, max_recv_records=1 << 14)
    try:
        rig.g.lease_reserve(1 << 12, 1 << 20)
        targets = np.arange(EMPTY, A, dtype=np.uint32)
        if wrapped:
            rig.send(np.repeat(targets, 200), np.zeros(200 * len(targets)))
            rig.recv(targets, 200, 0, "stream", what="wrap")
        for name, (prios, k) in LAYOUTS.items():
            mine = targets[[i for i, s in enumerate(steps) if s[0] == name]]
            n = len(prios)
            recv = np.tile(mine, n)
            ts = np.where(np.arange(n) == 0, 0.5, 5.0).repeat(len(mine))         # record 0 of each agent is old
            _send_ts(rig, recv, np.repeat(prios, len(mine)), ts)
            pad = np.concatenate([mine, rig.empties[: max(0, 9 - len(mine))]]).astype(np.uint32)
            rig.recv(pad, k, RECV_PRIORITY, "priority", what=f"holes {name}")
        for a, (name, path, call) in zip(targets.tolist(), steps):
            span0 = rig.c.ring.span(a)
            rig.g.profile_read()
            call(rig, a)
            assert rig.c.ring.span(a) < span0, (name, path)
        rig.check_loads(None, "after the retiring calls")
        _probe(rig, targets, "head placement")
        _drain(rig)
    finally:
        rig.close()


@pytest.mark.parametrize("ring_slots", [4, 8, 64, 128])
def test_ranked_p2p_fills_holey_rings_to_the_slot(shared, ring_slots):
    """Holey windows filled to within 0-3 slots of full (tails aligned and unaligned to the 32-byte sector of four
    entries), then a ranked batch: exact survivors and an exact log."""
    from swarmdb_b200._native import RECV_PRIORITY
    rng = np.random.default_rng(ring_slots)
    n_t = 16
    A = EMPTY + n_t
    rig = _rig(ring_slots, A, ring_slots=ring_slots)
    try:
        targets = np.arange(EMPTY, A, dtype=np.uint32)
        for rnd in range(3):
            # fill each ring to within `gap` of full with random priorities, punch holes with a priority receive, then
            # take one stream record: the window keeps its tombstones or sheds them, as the model says
            gap = (np.arange(n_t) + rnd) % 4
            want = np.array([rig.c.ring.capacity(a) for a in targets.tolist()]) - gap
            recv = np.concatenate([np.full(max(0, w), a) for a, w in zip(targets.tolist(), want.tolist())])
            rig.send(rng.permutation(recv).astype(np.uint32), rng.integers(0, 4, len(recv)))
            assert rig.c.take_dropped() == []
            k = max(1, ring_slots // 4)
            rig.recv(targets, k, RECV_PRIORITY, "priority", what="holes")
            rig.recv(targets[::2], 1, 0, "stream" if len(targets[::2]) > 8 else "small", what="oldest")
            _probe(rig, targets, f"R={ring_slots} round {rnd}")
        _drain(rig)
    finally:
        rig.close()


def test_restore_and_lease_sweep_at_the_boundary(shared):
    """On holey rings a restore of exactly the free slots is accepted and one more is refused with the state unchanged;
    a sweep blocks exactly the agents the model blocks."""
    from swarmdb_b200._native import RECV_PEEK, RECV_PRIORITY, SdbError
    from tests.lease_ref import LeaseModel
    from tests.restore_ref import restore_append
    n_t = 9
    A = EMPTY + n_t
    rig = _rig(5, A, ring_slots=64)
    try:
        targets = np.arange(EMPTY, A, dtype=np.uint32)
        prios, k = [0] + [3] * 39 + [0], 39
        _send_ts(rig, np.tile(targets, len(prios)), np.repeat(prios, n_t), np.full(len(prios) * n_t, 5.0))
        rig.recv(targets, k, RECV_PRIORITY, "priority", what="holes")
        rig.recv(targets[:8], 1, 0, "small", what="oldest")          # head jumps to the last record on 8 agents
        # records to restore: a snapshot of other agents' traffic
        src = _rig(6, A, ring_slots=256)
        src.g.advance_seq(1 << 20)                                     # seqs apart from the handle's own
        src.c.next_seq = 1 << 20
        src.send(np.repeat(targets, 70), np.zeros(70 * n_t))
        cnt, ent, snd, pay = src.g.receive_compact(None, 1 << 20, RECV_PEEK)
        ent, snd, pay = ent.copy(), snd.copy(), pay.copy()
        from swarmdb_b200.core import _renumber_rows
        first = np.concatenate([[0], np.cumsum(cnt.astype(np.int64))])

        def state():
            st = rig.g.stats()
            return ({k_: st[k_] for k_ in ("next_seq", "enqueued", "delivered", "arena_tail_bytes", "n_agents")},
                    rig.g.agent_loads(np.arange(A)).tobytes(), rig.g.receive_compact(None, 1 << 13, RECV_PEEK)[1].tobytes())

        for extra in (1, 0):
            free = np.array([rig.c.capacity(a) for a in targets.tolist()])
            # eight windows of one live record (63 free) and the holey one: 2 pending, 39 tombstones, 23 free.  Only
            # the holey agent goes one past its free slots: a check by pending + count <= R would accept it
            assert free[:8].tolist() == [63] * 8 and free[8] == 23 and int(rig.c.pending(targets[8])) == 2
            take = free.copy()
            take[8] += extra
            sub = np.concatenate([ent[first[a]:first[a] + t] for a, t in zip(targets.tolist(), take.tolist())])
            e2, s2 = _renumber_rows(sub, snd)
            if extra:
                s0 = state()
                with pytest.raises(SdbError) as ei:
                    rig.g.restore_compact(targets, take, e2, s2, pay)
                assert ei.value.code == -4 and state() == s0
                assert not rig.c.ring.fits(targets, take)
            else:
                assert rig.c.ring.fits(targets, take)
                assert rig.g.restore_compact(targets, take, e2, s2, pay)[0] == int(take.sum())
                with rig.c.appending():
                    restore_append(rig.c, {}, targets, take, e2, s2, pay)
                assert rig.c.take_dropped() == []
        rig.check_loads(None, "restored")
        src.close()
        # every ring is full now.  Priority leases leave record 0 behind on agents whose head did not move: their sweep
        # is blocked although pending + leased would fit
        rig.recv(targets, 64, 0, "stream", what="empty the rings")
        _send_ts(rig, np.tile(targets, 41), np.repeat([0] + [3] * 39 + [0], n_t), np.full(41 * n_t, 5.0))
        rig.g.lease_reserve(1 << 12, 1 << 20)
        from swarmdb_b200._native import recv_capacity
        m = LeaseModel(rig.c, {}, recv_capacity(rig.g.cfg), 1 << 12, shared)
        got = _expand(rig.g.receive_leased(targets, 39, 1.0, RECV_PRIORITY)[:4])
        _same(got, m.lease(targets, 39, 1.0, RECV_PRIORITY)[:3], "priority lease")
        rig.delivered = rig.g.stats()["delivered"]
        rig.recv(targets[:4], 1, 0, "small", what="oldest")
        fill = [rig.c.capacity(a) for a in targets.tolist()]
        rig.send(np.repeat(targets, fill), np.zeros(int(sum(fill))))
        # the first four make room for their 39 leases; the other five hold 25 pending records in a full window
        rig.recv(targets[:4], 40, 0, "small", what="room")
        assert [int(rig.c.pending(a)) for a in targets[4:].tolist()] == [25] * 5
        got = rig.g.lease_sweep(1.0)
        assert got == m.sweep(1.0) == (4 * 39, n_t - 4, 0), got
        rig.check_loads(None, "swept")
        _drain(rig)
    finally:
        rig.close()


def _bounded_send(rig, members, dev_send, orc_send, ordered, index, what, launches=None, commit=None, lossy=True):
    """One send on the device and in the model, into holey, nearly full rings.  ordered: an index build, which keeps the
    first records of the call in send order, so survivors and log are exact.  Otherwise an atomic-claim path: the
    survivors are read from the device (they must come out in seq order), and the model checks that each ring took
    exactly as many as it had free slots and that survivors and logged records split the call's records.
    launches / commit, when given: the kernel_launches delta of the call and whether the commit class ran (the profiler's
    index class times both pull kernels as one, so the launch count tells which of them ran).  lossy: whether some record
    is dropped (None: either)."""
    from swarmdb_b200._native import RECV_PEEK
    R_ = rig.c.ring.R
    assert rig.g.overflow_log()[2] == 0
    rig.c.take_dropped()
    st0 = rig.g.stats()
    base = st0["next_seq"]
    rig.g.profile_read()
    dev_send()
    prof = rig.g.profile_read()
    assert (prof["index"][1] > 0) == index, what
    if commit is not None:
        assert (prof["commit"][1] > 0) == commit, what
    if launches is not None:
        assert rig.g.stats()["kernel_launches"] - st0["kernel_launches"] == launches, \
            (what, rig.g.stats()["kernel_launches"] - st0["kernel_launches"], launches)
    if ordered:
        rig.c.enqueue(orc_send, ordered=True)
    else:
        cnt, hdr, _ = rig.g.receive_batch(members, 4 * R_, RECV_PEEK)
        who = np.repeat(members, cnt.astype(np.int64))
        keep = {int(a): [] for a in members.tolist()}
        new = hdr["seq"] >= base
        for a, s in zip(who[new].tolist(), hdr["seq"][new].tolist()):
            keep[a].append(int(s))
        for a, ss in keep.items():
            assert ss == sorted(ss), (what, a, ss)
        rig.c.enqueue(orc_send, keep=keep)
    want = rig.c.take_dropped()
    st1 = rig.g.stats()
    assert st1["ring_overflow"] - st0["ring_overflow"] == len(want), (what, st1["ring_overflow"] - st0["ring_overflow"], len(want))
    assert lossy is None or (len(want) > 0) == lossy, (what, len(want))
    ag, sq, dropped = rig.g.overflow_log(1 << 16)
    assert dropped == len(want), what
    got = sorted(zip(ag.tolist(), sq.tolist()))
    if len(want) <= 4096:
        assert got == sorted(want), what
    else:                                                # the device logs the first 4096 of an interval
        assert len(got) == 4096 and set(got) <= set(want), what
    rig.check_loads(None, what)
    _same(rig.g.receive_batch(members, 4 * R_, RECV_PEEK), rig.c.receive_batch(members, 4 * R_, RECV_PEEK),
          what + " survivors")
    return len(want)


def test_index_builds_and_atomic_claims_at_the_boundary(shared):
    """One group of 4096 members with 8-slot rings, made holey and nearly full (0-3 free slots before the holes) before
    each send: a group batch above the pull threshold (k_pull_index_group) and a broadcast of disjoint lists
    (k_list_index), both order-deterministic, one of them dropping more than 4096 records; then the atomic-claim paths:
    a group batch below the threshold and a mixed batch of p2p sends and overlapping lists."""
    from swarmdb_b200._native import RECV_PRIORITY
    from tests.test_gpu_shared_layout import THRESHOLD
    Rr, M = 8, 4096
    A = EMPTY + M
    rig = _rig(21, A, ring_slots=Rr, list_pool_entries=1 << 16)
    try:
        rng = rig.rng
        members = np.arange(EMPTY, A, dtype=np.uint32)
        rig.g.create_group(0, members)
        rig.c.create_group(0, members)

        def holey():
            rig.recv(members, Rr, 0, "stream", what="empty")
            fill = Rr - rng.integers(0, 4, M)
            rig.send(rng.permutation(np.repeat(members, fill)).astype(np.uint32), rng.integers(0, 4, int(fill.sum())))
            rig.recv(members, 2, RECV_PRIORITY, "priority", what="holes")
            rig.recv(rng.permutation(members)[: M // 2], 1, 0, "stream", what="oldest")

        def payloads(n):
            lens, off, buf = _payloads(rng, n, rig.max_len)
            return rng.integers(0, EMPTY, n), rng.integers(0, 4, n), rng.integers(0, 7, n), lens, off, buf

        def group(n):
            s, p, t, lens, off, buf = payloads(n)
            g = np.zeros(n, np.uint32)
            return (lambda: rig.g.send_group_batch(s, g, p, t, lens, off, buf),
                    lambda: rig.c.send_group_batch(s, g, p, t, lens, off, buf))

        holey()
        assert 4 * M >= THRESHOLD
        lost = _bounded_send(rig, members, *group(4), True, True, "group batch, pull index")
        assert lost > 4096
        holey()
        nb = 4
        s, p, t, lens, off, buf = payloads(nb)
        lo = np.arange(nb + 1, dtype=np.uint64) * M
        li = np.tile(rng.permutation(members), nb).astype(np.uint32)         # one list named by every broadcast
        _bounded_send(rig, members, lambda: rig.g.send_list_batch(s, lo, li, p, t, lens, off, buf),
                      lambda: rig.c.send_list_batch(s, lo, li, p, t, lens, off, buf), True, True, "lists, list index")
        holey()
        assert 2 * M < THRESHOLD
        _bounded_send(rig, members, *group(2), False, False, "group batch below the pull threshold")
        holey()
        n_p, n_l = 3000, 40
        lists = [rng.choice(members, 300, replace=False) for _ in range(n_l)]     # lists overlap one another
        lo = np.zeros(n_l + 1, np.uint64); lo[1:] = np.cumsum([len(x) for x in lists])
        li = np.concatenate(lists).astype(np.uint32)
        s, p, t, lens, off, buf = payloads(n_p + n_l)
        kind = np.r_[np.zeros(n_p, np.uint8), np.full(n_l, 2, np.uint8)]
        target = np.r_[rng.choice(members, n_p), np.arange(n_l)].astype(np.uint32)
        pe, le = slice(0, n_p), slice(n_p, n_p + n_l)

        def orc_mixed():                                 # the oracle takes the p2p sends, then the lists, in order
            rig.c.send_batch(s[pe], target[pe], p[pe], t[pe], lens[pe], off[pe], buf)
            rig.c.send_list_batch(s[le], lo, li, p[le], t[le], lens[le], off[le], buf)

        _bounded_send(rig, members, lambda: rig.g.send_mixed_batch(s, kind, target, lo, li, p, t, lens, off, buf),
                      orc_mixed, False, False, "mixed batch, overlapping lists")
        _drain(rig)
    finally:
        rig.close()
