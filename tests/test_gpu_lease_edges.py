"""Leases, restore and dead letters at the edges of their device sorts and of the ledger's index, against
tests/lease_ref.py and tests/deadletter_ref.py, byte for byte, in both arena layouts.

- Sequence numbers around 2^8, 2^16, 2^24, 2^32 and above: the sweep numbers a redelivered row by its smallest seq
  (a radix sort on the low word, then on the high word from 2^32 on), so a sort with a digit too few renumbers rows;
  every case checks that its traffic would show that in the arena bytes.
- Ledger keys that differ only above bit 32, and probe chains that wrap from the index's last slot to slot 0.
- More than 2^16 agents: three-digit agent keys in the sweep, list positions in the dead-letter readout, and a restore
  of more than 65,536 rows.
"""
import numpy as np
import pytest

from tests.deadletter_ref import lg_slot, seqs_at_slot
from tests.restore_ref import restore_granules
from tests.test_gpu_compact_receive import Rig, _same
from tests.test_gpu_dead_letter import _dead, _lease as _lease_counted, _model, _nack_all, _sweep, _to_the_limit
from tests.test_gpu_lease import _lease as _lease_plain
from tests.test_gpu_restore import _every_path, _expand, _fresh, _renumber, _restore_both

pytestmark = pytest.mark.gpu


@pytest.fixture(params=["1", "0"])
def shared(request, monkeypatch):
    monkeypatch.setenv("SDB_SHARED_PAYLOAD", request.param)
    return request.param == "1"


def _rig(seed, **kw):
    rig = Rig(np.random.default_rng(seed), G=8, F=64, extra=64, **kw)
    rig.check_advance = False
    return rig


def _advance(rig, seq):
    """The handles' and the oracle's sequence counters, moved together."""
    for g in rig.gs:
        g.advance_seq(seq)
    rig.c.next_seq = seq
    assert rig.g.stats()["next_seq"] == seq


def _p2p_to(rig, receivers, max_len=120):
    """Ranked p2p records to the listed receivers, in list order; returns the first seq."""
    from tests.test_gpu_shared_layout import _payloads
    r = np.asarray(receivers, np.uint32)
    s, prio = rig.rng.integers(0, rig.A, len(r)), rig.rng.integers(0, 4, len(r))
    lens, off, buf = _payloads(rig.rng, len(r), max_len)
    lens[lens == 0] = 1
    base = rig.c.send_batch(s, r, prio, None, lens, off, buf)
    for g in rig.gs:
        assert g.send_batch(s, r, prio, None, lens, off, buf) == base
    return base


def _lease(rig, m, agents, k, flags=0):
    """A leased receive checked against the model; with a policy also every delivery count.  Returns the lease ids."""
    if m.policy:
        return _lease_counted(rig, m, agents, k, 10.0, flags)
    ent, base = _lease_plain(rig, m, agents, k, 10.0, flags)
    return np.arange(base, base + len(ent), dtype=np.uint64)


def _set_policy(rig, m, M, ledger):
    rig.g.lease_set_policy(M, ledger)
    m.set_policy(M, ledger)


def _redrive_all(rig, m, agents=None):
    """Take every dead letter (listed agents first), redrive it through restore_compact."""
    while True:
        cnt, ent, snd, pay, _ = _dead(rig, m, agents)
        if len(ent) == 0:
            if agents is None:
                break
            agents = None
            continue
        idx = np.arange(len(cnt), dtype=np.uint32) if agents is None else np.asarray(agents, np.uint32)
        assert rig.g.restore_compact(idx, cnt, ent, snd, pay)[0] == len(ent)
        m.redrive(idx, cnt, ent, snd, pay)
    assert rig.g.lease_policy_stats()["dead"] == 0


# ---- 1. seq-sort digit counts ---------------------------------------------------------------------------------------
# (boundary the traffic straddles, the modulus a sort with a digit too few would keep)
BASES = [(1 << 8, 1 << 8), (1 << 16, 1 << 16), (1 << 24, 1 << 24), (1 << 32, 1 << 32),
         ((3 << 40) | (5 << 32), 1 << 32), (1 << 48, 1 << 48), (1 << 56, 1 << 56)]


def _truncation_shows(m, base, mod):
    """The self-check: the last sweep staged seqs on both sides of `base`, and numbering its rows by seq % mod would
    have changed the arena bytes (some agent's rows ascend in seq and descend in seq % mod)."""
    seqs = [int(r["hdr"]["seq"]) for _, rs in m.last_staged for r in rs]
    assert min(seqs) < base <= max(seqs)
    agents, counts, ent, snd, _ = m.staged_input(m.last_staged)
    true = restore_granules(counts, ent, snd, True, agents)
    assert true == m.last_granules or not m.shared
    _, c2, e2, s2, _ = m.staged_input(m.last_staged, lambda s: s % mod)
    assert restore_granules(c2, e2, s2, True, agents) != true


@pytest.mark.parametrize("base,mod", BASES, ids=["2^8", "2^16", "2^24", "2^32", "composite", "2^48", "2^56"])
def test_seq_sort_digit_counts(shared, base, mod):
    from swarmdb_b200._native import RECV_PEEK, WHERE_DROP, make_filter
    rig = _rig(base % 997 + 31)
    _advance(rig, base - 200)
    rig.p2p(150)                                                     # base - 200 .. base - 51
    rig.shared_batch(300)                                            # base - 50 .. base + 249: one batch across the boundary
    rig.broadcast(4)                                                 # one seq for many agents
    rig.p2p(100)
    assert rig.c.next_seq == rig.g.stats()["next_seq"] > base
    sub = np.concatenate([rig.members[0], rig.idx[rig.G * rig.F:]])  # one group's members and every non-member
    # no policy: lease everything they have, nack, sweep
    m = _model(rig, shared, 0, 0)
    ids = _lease(rig, m, sub, 1000)
    _nack_all(rig, m, ids)
    assert _sweep(rig, m, 0.0) == (len(ids), 0, 0)
    if shared:
        _truncation_shows(m, base, mod)
    # a limit of 2: count 1 into the ledger, count 2, then dead letters
    _set_policy(rig, m, 2, 1 << 13)
    ids = _lease(rig, m, sub, 1000)
    _nack_all(rig, m, ids)
    assert _sweep(rig, m, 0.0) == (len(ids), 0, 0)
    if shared:
        _truncation_shows(m, base, mod)
    ids = _lease(rig, m, sub, 1000)
    assert set(rig.g.lease_deliveries(ids).tolist()) == {2}
    _nack_all(rig, m, ids)
    assert _sweep(rig, m, 0.0) == (0, 0, 0) and rig.g.lease_policy_stats()["dead"] == len(ids)
    a = _dead(rig, m, None, peek=True)
    assert set(a[4].tolist()) == {2}
    _redrive_all(rig, m, rig.rng.permutation(sub)[:100].astype(np.uint32))
    # a filter whose seq clause straddles the boundary: PEEK, then a drop
    f = make_filter(seq=(base - 5, base + 5))
    got = rig.g.receive_where(rig.idx, 1000, RECV_PEEK, f)
    want = rig.c.receive_where(rig.idx, 1000, RECV_PEEK, f)
    _same(got, want, "where peek")
    assert int(want[1]["seq"].min()) < base <= int(want[1]["seq"].max())
    f = make_filter(seq=(base - 3, base + 3))
    got = rig.g.receive_where(rig.idx, 1000, WHERE_DROP, f, drop=True)
    want = rig.c.receive_where(rig.idx, 1000, 0, f, drop=True)
    assert np.array_equal(got[0], want[0]) and got[1] == want[1] > 0
    # a snapshot restored into a fresh handle: next_seq is the largest seq + 1 and the next send takes it
    snap = rig.g.receive_compact(None, 1 << 20, RECV_PEEK)
    _same(_expand(snap), rig.c.receive_batch(rig.idx, 1 << 20, RECV_PEEK, rec_cap=1 << 21), "snapshot")
    cnt, (ent, snd), pay = snap[0].copy(), _renumber(snap[1], snap[2]), snap[3].copy()
    g, c = _fresh(rig)
    _restore_both(rig, g, c, rig.idx, cnt, ent, snd, pay, shared)
    seq_end = int(ent["seq"].max()) + 1
    assert seq_end == g.stats()["next_seq"] == c.next_seq and seq_end > base
    assert g.send_batch([0], [1], [1], None, [4], [0], np.zeros(64, np.uint8)) == seq_end
    assert c.send_batch([0], [1], [1], None, [4], [0], np.zeros(64, np.uint8)) == seq_end
    _every_path(rig, g, c, shared, rig.rng)
    g.close(); c.close(); rig.close()


# ---- 2. ledger keys that differ only above bit 32 -------------------------------------------------------------------
def test_ledger_keys_that_differ_only_above_bit_32(shared):
    rig = _rig(41)
    a = rig.G * rig.F + 5
    slots = 2 * 2                                                    # a ledger of 2 entries
    s = (1 << 33) + 1
    while lg_slot(a, s, slots) != lg_slot(a, s + (1 << 32), slots):  # both keys probe from the same slot
        s += 1
    _advance(rig, s)
    _p2p_to(rig, [a])
    _advance(rig, s + (1 << 32))
    _p2p_to(rig, [a])
    _p2p_to(rig, rig.rng.integers(0, a, 50))                         # other agents' traffic
    m = _model(rig, shared, 3, 2)

    def lease_a(k):
        ids = _lease(rig, m, [a], k)
        return ids, [int(x) for x in rig.g.lease_deliveries(ids)]

    ids, d = lease_a(1)                                              # seq s
    assert d == [1]
    _nack_all(rig, m, ids)
    assert _sweep(rig, m, 0.0) == (1, 0, 0)
    ids, d = lease_a(1)                                              # seq s + 2^32: the ledger holds only (a, s)
    assert d == [1]
    _nack_all(rig, m, ids)
    assert _sweep(rig, m, 0.0) == (1, 0, 0)
    ids, d = lease_a(1)                                              # seq s again
    assert d == [2]
    _nack_all(rig, m, ids)
    assert _sweep(rig, m, 0.0) == (1, 0, 0)
    ids, d = lease_a(2)                                              # s + 2^32 at 2, s at 3
    assert d == [2, 3]
    _nack_all(rig, m, ids)
    assert _sweep(rig, m, 0.0) == (1, 0, 0) and rig.g.lease_policy_stats()["dead"] == 1
    _to_the_limit(rig, m, [a])
    cnt, ent, snd, pay, dl = _dead(rig, m, [a], peek=True)
    assert sorted(int(x) for x in ent["seq"]) == [s, s + (1 << 32)] and dl.tolist() == [3, 3]
    _redrive_all(rig, m, [a])
    ids, d = lease_a(2)
    assert d == [1, 1]
    _every_path(rig, rig.g, rig.c, shared, rig.rng)
    rig.close()


# ---- 4. ledger probes across the end of the index -------------------------------------------------------------------
@pytest.mark.parametrize("N", [2, 4])
def test_ledger_probe_chains_wrap_to_slot_0(shared, N):
    rig = _rig(50 + N)
    a, b = rig.G * rig.F + 7, rig.G * rig.F + 9
    slots = 2 * N
    seqs = seqs_at_slot(a, slots, slots - 1, 1000, N + 1)
    # self-check: every record probes from the last slot, so N entries fill it and then slots 0 .. N - 2
    assert N >= 2 and all(lg_slot(a, q, slots) == slots - 1 for q in seqs)
    for q in seqs:
        _advance(rig, q)
        _p2p_to(rig, [a])
    _p2p_to(rig, [b] * 3)                                            # another agent's records behind them
    m = _model(rig, shared, 3, N)
    ids = _lease(rig, m, [a], N)                                     # the first N: their entries fill the chain
    _nack_all(rig, m, ids)
    assert _sweep(rig, m, 0.0) == (N, 0, 0)
    assert rig.g.lease_policy_stats()["ledger_used"] == N
    ids = _lease(rig, m, [a, b], N + 1)                              # the N + 1st has no entry: its probe ends at slot N - 1
    d = rig.g.lease_deliveries(ids).tolist()
    assert d[:N + 1] == [1] + [2] * N and d[N + 1:] == [1] * 3
    _nack_all(rig, m, ids)
    red, _, left = _sweep(rig, m, 0.0)
    assert red == N and left == 4                                    # the ledger's room: N of the N + 4 due records
    _to_the_limit(rig, m, [a, b])
    _dead(rig, m, None, peek=True)
    _redrive_all(rig, m)
    _every_path(rig, rig.g, rig.c, shared, rig.rng)
    rig.close()


# ---- 3. sort keys of three digits: more than 2^16 agents ------------------------------------------------------------
A3 = 70_000


def _rig3(seed, **kw):
    rig = Rig(np.random.default_rng(seed), G=2, F=64, extra=A3 - 128, **kw)
    rig.check_advance = False
    return rig


def test_agent_keys_and_list_positions_of_three_digits(shared):
    rig = _rig3(61, ring_slots=64)
    P = 300
    lo = rig.rng.choice(np.arange(128, A3 - 65536), P, replace=False).astype(np.uint32)
    order = np.stack([lo, lo + 65536], 1).ravel()                   # pairs (a, a + 65536), interleaved
    _p2p_to(rig, np.tile(order, 3))
    m = _model(rig, shared, 0, 0)

    def lease_alternating():                                         # lease ids alternate between a and a + 65536
        ids = [_lease(rig, m, order, 1) for _ in range(3)]
        assert all(len(x) == len(order) for x in ids)
        return np.concatenate(ids)

    ids = lease_alternating()
    _nack_all(rig, m, ids)
    assert _sweep(rig, m, 0.0) == (len(ids), 0, 0)
    _set_policy(rig, m, 2, 1 << 12)
    for _ in range(2):
        ids = lease_alternating()
        _nack_all(rig, m, ids)
        _sweep(rig, m, 0.0)
    assert rig.g.lease_policy_stats()["dead"] == len(ids) == 6 * P
    _dead(rig, m, None, peek=True)                                   # 70,000 list positions
    _dead(rig, m, rig.rng.permutation(order), peek=True)             # 600 listed agents
    full = rig.rng.permutation(A3).astype(np.uint32)                 # positions that are not agent ids
    _dead(rig, m, full, peek=True)
    cnt, ent, snd, pay, _ = _dead(rig, m, full)
    assert len(ent) == 6 * P
    assert rig.g.restore_compact(full, cnt, ent, snd, pay)[0] == len(ent)
    m.redrive(full, cnt, ent, snd, pay)
    _every_path(rig, rig.g, rig.c, shared, rig.rng)
    rig.close()


def test_restore_of_more_than_65536_rows(shared):
    from swarmdb_b200._native import RECV_PEEK
    rig = _rig3(62, ring_slots=256, max_batch_sends=A3, max_recv_records=1 << 18)   # a member gets ~150 group sends
    rig.shared_batch(300)
    _p2p_to(rig, rig.rng.permutation(A3), max_len=64)               # one p2p record per agent: a row each
    snap = rig.g.receive_compact(None, 1 << 20, RECV_PEEK)
    _same(_expand(snap), rig.c.receive_batch(rig.idx, 1 << 20, RECV_PEEK, rec_cap=1 << 21), "snapshot")
    cnt, (ent, snd), pay = snap[0].copy(), _renumber(snap[1], snap[2]), snap[3].copy()
    assert len(snd) > 65536                                          # row keys of three digits
    g, c = _fresh(rig, ring_slots=256, max_batch_sends=A3, max_recv_records=1 << 18)
    _restore_both(rig, g, c, rig.idx, cnt, ent, snd, pay, shared)
    _every_path(rig, g, c, shared, rig.rng)
    g.close(); c.close(); rig.close()
