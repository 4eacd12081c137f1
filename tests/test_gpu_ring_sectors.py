"""Whole-sector ring appends of the index build (k_pull_index_group, k_list_index) against the CPU oracle, bit-exact.

The index build writes a member's new ring entries as whole 32-byte sectors (four 8-byte slots) when no live entry
shares them: the tail is sector-aligned, or the ring is drained (head == tail), and the rounded-up end stays within
ring_slots of head.  Slots of such a sector that get no entry hold a consumed filler.  Otherwise (live entries in the
tail's sector after a partial drain, tombstoned windows after priority receives, filtered receives or expiry, a ring
within 1-3 slots of full, rings of 2 slots) every entry is stored where it belongs.  The traffic here drives both sides
of that choice round after round, and every receive path (stream plan, priority pipeline, the <= 8-agent kernel, the
latency server, compact, filtered, expire, restore and the digests) must return what the oracle returns.

The oracle's rings are unbounded, so sends never overflow a ring here except in the overflow test: the test keeps an
upper bound of tail - head per agent.  Three kinds of groups:
  tight   received only in stream order, so the window holds no consumed entries and the bound is exact: partial drains,
          and rings filled to exactly full or to within 1-3 slots of it;
  holey   the receives that leave consumed entries in the window (priority, filtered, expire); the bound only grows;
  fresh   drained completely before every batch (head == tail at any alignment, the usual case), which also gives each
          group batch the 256 sends of 64 members it needs to take the pull index build.
"""
import numpy as np
import pytest

from tests.test_gpu_compact_receive import THRESHOLD, _check_format, _same
from tests.test_gpu_expire import _expire_all_calls
from tests.test_gpu_shared_layout import _payloads
from tests.test_gpu_where import _check, _rig

pytestmark = pytest.mark.gpu

G, F = 512, 64
TIGHT, HOLEY = 0, 1                              # group g is of kind min(g % 4, 2): 2 = fresh


class Rings:
    """The rig plus, per agent, an upper bound of the ring window tail - head."""

    def __init__(self, rng, R):
        self.R = R
        self.rig = _rig(rng, G=G, F=F, extra=64, ring_slots=R, max_batch_sends=16384, list_pool_entries=1 << 17)
        self.rng = rng
        self.occ = np.zeros(self.rig.A, np.int64)
        self.kind = np.minimum(np.arange(G) % 4, 2)
        self.of = [np.concatenate([self.rig.members[g] for g in range(G) if self.kind[g] == k]).astype(np.uint32)
                   for k in range(3)]
        self.rig.g.profile(True)

    def index_launches(self):
        return self.rig.g.profile_read().get("index", (0, 0))[1]

    def p2p(self, n):
        rig, rng = self.rig, self.rng
        free = np.flatnonzero(self.occ < self.R)
        r = rng.choice(free, size=min(n, len(free)), replace=False).astype(np.uint32)
        s = rng.integers(0, rig.A, len(r))
        lens, off, buf = _payloads(rng, len(r), 200)
        ts = rng.uniform(0, 10, len(r))
        prio = rng.integers(0, 4, len(r))
        base = rig.c.send_batch(s, r, prio, None, lens, off, buf, ts)
        assert rig.g.send_batch(s, r, prio, None, lens, off, buf, ts) == base
        self.occ[r] += 1

    def group_batch(self, want, own=0.5):
        """One pure group batch (the pull index build): group g gets min(want_g, room_g) sends, room_g being what its
        fullest member can take; a fraction `own` of the sends come from a member of the group, who skips its own."""
        rig, rng = self.rig, self.rng
        room = np.array([self.R - self.occ[m].max() for m in rig.members])
        cnt = np.clip(np.minimum(want, room), 0, None)
        grp = rng.permutation(np.repeat(np.arange(G), cnt))
        n = len(grp)
        assert n * F >= THRESHOLD, n
        mine = rng.random(n) < own
        s = np.where(mine, [rig.members[g][rng.integers(0, F)] for g in grp], rng.integers(G * F, rig.A, n)).astype(np.uint32)
        prio, typ = rng.integers(0, 4, n), rng.integers(0, 7, n)
        lens, off, buf = _payloads(rng, n, 256)
        ts = rng.uniform(0, 10, n)
        l0 = self.index_launches()
        base = rig.c.send_group_batch(s, grp, prio, typ, lens, off, buf, ts)[0]
        assert rig.g.send_group_batch(s, grp, prio, typ, lens, off, buf, ts) == base
        assert self.index_launches() > l0
        for g, k in enumerate(cnt):
            self.occ[rig.members[g]] += k
        np.subtract.at(self.occ, s[mine], 1)

    def broadcast(self, nb):
        """nb broadcasts to ONE list of every member with room for them (the owner-computes index build)."""
        rig, rng = self.rig, self.rng
        lst = rng.permutation(np.flatnonzero(self.occ[: G * F] <= self.R - nb)).astype(np.uint32)
        assert nb * len(lst) >= THRESHOLD
        lo = np.arange(nb + 1, dtype=np.uint64) * len(lst)
        li = np.tile(lst, nb)
        s, prio, typ = rng.integers(0, rig.A, nb), rng.integers(0, 4, nb), rng.integers(0, 7, nb)
        lens, off, buf = _payloads(rng, nb, 200)
        ts = rng.uniform(0, 10, nb)
        l0 = self.index_launches()
        base = rig.c.send_list_batch(s, lo, li, prio, typ, lens, off, buf, ts)
        assert rig.g.send_list_batch(s, lo, li, prio, typ, lens, off, buf, ts) == base
        assert self.index_launches() == l0 + 1
        self.occ[lst] += nb

    def stream(self, agents, k, what, compact=False):
        """A stream-order receive: the bound of these (tight or fresh) agents becomes their pending count."""
        rig = self.rig
        agents = np.asarray(agents, np.uint32)
        want = rig.c.receive_batch(agents, k, rec_cap=1 << 21)
        got = _check_format(rig.g.receive_compact(agents, k)) if compact else rig.g.receive_batch(agents, k)
        _same(got, want, what)
        self.occ[agents] = rig.c.agent_loads(agents)["pending"]


def _receives(w, rnd):
    """Partial drains of tight agents through the stream paths; priority, filtered and expiring receives of holey
    agents.  Every call against the oracle."""
    from swarmdb_b200._native import RECV_PEEK, RECV_PRIORITY, make_filter
    rig, rng = w.rig, w.rng
    tight, holey = rng.permutation(w.of[TIGHT]), rng.permutation(w.of[HOLEY])
    n = len(tight)
    w.stream(tight[: n // 3], int(rng.integers(1, 4)), f"stream plan {rnd}")                     # live entries stay in the sector
    w.stream(tight[n // 3: n // 3 + 6], 2, f"small {rnd}")
    w.stream(tight[n // 3 + 6: n // 2], int(rng.integers(1, 3)), f"compact {rnd}", compact=True)
    w.stream(tight[n // 2: 2 * n // 3], 1000, f"full drain {rnd}")
    rig.g.latency_server(True)
    for a in tight[2 * n // 3: 2 * n // 3 + 6]:
        h, p, _ = rig.g.receive_one(int(a), 1)
        _, hc, pc = rig.c.receive_batch([a], 1)
        assert h.tobytes() == hc.tobytes() and p.tobytes() == pc.tobytes(), ("latency server", rnd, a)
        w.occ[a] = rig.c.agent_loads([a])["pending"][0]
    rig.g.latency_server(False)
    q = len(holey) // 4
    _same(rig.g.receive_batch(holey[:q], 1, RECV_PRIORITY), rig.c.receive_batch(holey[:q], 1, RECV_PRIORITY),
          f"priority {rnd}")
    _same(rig.g.receive_batch(holey[q: q + 5], 1, RECV_PRIORITY), rig.c.receive_batch(holey[q: q + 5], 1, RECV_PRIORITY),
          f"priority small {rnd}")
    filt = make_filter(prios=[int(rng.integers(0, 4))])
    _same(rig.g.receive_where(holey[q: 2 * q], 1, 0, filt), rig.c.receive_where(holey[q: 2 * q], 1, 0, filt), f"where {rnd}")
    cut = float(rng.uniform(2, 5))
    got = _expire_all_calls(rig.g, holey[2 * q: 3 * q], cut)
    _same(got[:3], rig.c.expire(holey[2 * q: 3 * q], cut), f"expire {rnd}")
    some = rng.choice(rig.A, 3000, replace=False).astype(np.uint32)
    _same(rig.g.receive_batch(some, 1 << 10, RECV_PEEK), rig.c.receive_batch(some, 1 << 10, RECV_PEEK, rec_cap=1 << 21),
          f"peek {rnd}")
    _check(rig, f"round {rnd}")


@pytest.mark.parametrize("R", [2, 4, 8, 64])
def test_sector_appends_through_every_receive_path(R):
    from swarmdb_b200._native import RECV_PRIORITY
    from swarmdb_b200.core import _renumber_rows
    from tests.restore_ref import restore_append
    rng = np.random.default_rng(900 + R)
    w = Rings(rng, R)
    rig = w.rig
    try:
        for rnd in range(4):
            w.stream(w.of[2], 1000, f"fresh {rnd}")
            if R == 2:
                w.stream(w.of[TIGHT], 1000, f"tight {rnd}")
            w.p2p(0 if R == 2 else 60)
            want = np.where(w.kind == 2, rng.integers(1, 6, G), 0)
            full = R <= 8 or rnd == 3                     # 64-slot rings: filled once (the oracle's cost grows with them)
            want = np.where(w.kind == TIGHT, w.R - rng.integers(0, 4, G) if full else rng.integers(1, 6, G), want)
            want = np.where(w.kind == HOLEY, 1, want)
            w.group_batch(want)
            if rnd % 2:
                w.stream(w.of[2], 1000, f"fresh before broadcast {rnd}")
                w.broadcast(min(2, R))
            _receives(w, rnd)
        # requeue: records taken from tight agents go back behind what they still hold, then one more batch
        sel = rng.choice(w.of[TIGHT], 300, replace=False).astype(np.uint32)
        cnt, ent, snd, pay = (x.copy() for x in rig.g.receive_compact(sel, 2))
        rig.c.receive_batch(sel, 2)
        ent, snd = _renumber_rows(ent, snd)
        n = rig.g.restore_compact(sel, cnt, ent, snd, pay)[0]
        assert n == restore_append(rig.c, dict(enumerate(rig.members)), sel, cnt, ent, snd, pay) == int(cnt.sum())
        _check(rig, "after requeue")
        w.stream(w.of[2], 1000, "fresh after requeue")
        w.group_batch(np.where(w.kind == 2, 3, w.R))
        _same(rig.g.receive_batch(w.of[HOLEY], 2, RECV_PRIORITY), rig.c.receive_batch(w.of[HOLEY], 2, RECV_PRIORITY),
              "priority after requeue")
        rig.g.digest_reset(); rig.c.digest_enable()
        while True:
            _, total, _ = rig.g.receive_batch(None, 3, copy_out=False)
            rig.g.digest_fold()
            rig.c.receive_counts(None, 3)
            if total == 0:
                break
        assert np.array_equal(rig.g.digest_read(), rig.c.digest_read())
        assert rig.g.stats()["ring_overflow"] == 0 and rig.g.queue_stats()["pending"] == 0
    finally:
        rig.close()


@pytest.mark.parametrize("R", [4, 8])
def test_exact_overflow_keeps_the_first_entries_and_logs_the_rest(R):
    """Rings filled to R - d (d = 0..3), then d + e more sends per group from non-members: each member keeps the first R
    entries (the filler of a whole-sector append must not land on them), the e more are dropped and logged."""
    rng = np.random.default_rng(950 + R)
    w = Rings(rng, R)
    rig = w.rig
    try:
        d = rng.integers(0, 4, G)
        w.group_batch(R - d, own=0.0)                  # tail = R - d: aligned, or within 1-3 slots of full
        e = rng.integers(0, 3, G)
        grp = rng.permutation(np.repeat(np.arange(G), d + e))
        n = len(grp)
        assert n * F >= THRESHOLD
        s = rng.integers(G * F, rig.A, n)
        prio, typ = rng.integers(0, 4, n), rng.integers(0, 7, n)
        lens, off, buf = _payloads(rng, n, 256)
        base = rig.c.send_group_batch(s, grp, prio, typ, lens, off, buf)[0]
        assert rig.g.send_group_batch(s, grp, prio, typ, lens, off, buf) == base
        lost_n = int((e * F).sum())
        assert rig.g.stats()["ring_overflow"] == lost_n
        ag, sq, dropped = rig.g.overflow_log()
        assert dropped == lost_n and len(sq) == min(lost_n, 4096)
        members = np.concatenate(rig.members).astype(np.uint32)
        _same(rig.g.receive_batch(members, 100), rig.c.receive_batch(members, R, rec_cap=1 << 21), "survivors")
        cc, hc, _ = rig.c.receive_batch(members, 100, rec_cap=1 << 21)
        lost = set(zip(np.repeat(members, cc.astype(np.int64)).tolist(), hc["seq"].tolist()))
        assert len(lost) == lost_n and set(zip(ag.tolist(), sq.tolist())) <= lost
        assert rig.g.queue_stats()["pending"] == 0
    finally:
        rig.close()
