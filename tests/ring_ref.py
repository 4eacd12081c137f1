"""Bounded-ring model of the per-agent rings (TESTS ONLY).

The CPU oracle's inboxes have no bound, so on its own it cannot say how many records a ring takes.  The capacity rule
of include/swarmdb_b200.h is stated here literally.  Each agent's window [head, tail) is a list of slots in stream
order, each a live record or a tombstone (a record already consumed but still inside the window):

  - a retiring call (receive, leased receive, filtered take or drop, expiry) tombstones the records it returned;
  - head then moves to the first live slot, or to tail when none is left;
  - the ring takes R - (tail - head) more records.

A slot is identified by its position in the agent's stream, not by its seq alone: a broadcast list that names an agent
twice delivers one seq to it twice.  Of two equal records the earlier one is consumed first.

Appends follow the send path.  Order-deterministic paths (ranked p2p, the pull index, disjoint lists, the async
import's group traffic) keep the first records of the batch in send order and drop the rest.  Atomic-claim paths only
fix how many survive; for those the caller reads the survivors from the device and passes them as `keep`.
sdb_restore_compact is all or nothing (`fits`), and sdb_lease_sweep blocks an agent whose ring cannot take all of its
records (tests/lease_ref.py).

`BoundedOracle` keeps a RingModel in step with a WhereOracle (tests/where_ref.py): after each send it bounds the
appended records and removes the dropped ones from the oracle with the replay of tests/expire_ref.py; after each
retiring call it tombstones the records that left the oracle's queues.
"""
from __future__ import annotations

import contextlib

import numpy as np

from tests.expire_ref import RECV_PEEK
from tests.where_ref import RECV_PRIORITY, WhereOracle


class RingModel:
    """Windows of slots [seq, live] per agent, with absolute head and tail cursors."""

    def __init__(self, ring_slots: int):
        assert ring_slots >= 1 and ring_slots & (ring_slots - 1) == 0
        self.R = ring_slots
        self.win = {}
        self.head = {}

    def window(self, a):
        self.head.setdefault(int(a), 0)
        return self.win.setdefault(int(a), [])

    def tail(self, a):
        return self.head.get(int(a), 0) + len(self.window(a))

    def span(self, a):
        """tail - head."""
        return len(self.window(a))

    def capacity(self, a):
        return self.R - self.span(a)

    def ntomb(self, a):
        return sum(1 for _, live in self.window(a) if not live)

    def live_seqs(self, a):
        return [s for s, live in self.window(a) if live]

    def _advance(self, a):
        w = self.window(a)
        k = 0
        while k < len(w) and not w[k][1]:
            k += 1
        if k:
            del w[:k]
            self.head[int(a)] = self.head.get(int(a), 0) + k

    def append(self, a, seqs):
        seqs = [int(s) for s in seqs]
        assert len(seqs) <= self.capacity(a), (a, len(seqs), self.capacity(a))
        self.window(a).extend([s, True] for s in seqs)

    def offer(self, a, seqs):
        """An order-deterministic append: the first records that fit are kept.  Returns (kept, dropped)."""
        seqs = [int(s) for s in seqs]
        n = max(0, min(len(seqs), self.capacity(a)))
        self.append(a, seqs[:n])
        return seqs[:n], seqs[n:]

    def fits(self, agents, counts):
        """sdb_restore_compact's test: every listed agent's ring takes all of its records."""
        return all(int(c) <= self.capacity(a) for a, c in zip(np.asarray(agents).tolist(), np.asarray(counts).tolist()))

    def retire(self, a, seqs):
        """Tombstone the earliest live slot of each seq (the records one call returned), then move head."""
        w = self.window(a)
        for s in (int(x) for x in seqs):
            slot = next((e for e in w if e[1] and e[0] == s), None)
            assert slot is not None, (a, s)
            slot[1] = False
        self._advance(a)

    def retire_to(self, a, pending):
        """Tombstone every live slot that is not in `pending` (the agent's pending seqs in stream order, a subsequence
        of its live slots).  Matched from the end, so that of two equal records the earlier one is the one consumed."""
        pending = [int(s) for s in pending]
        j = len(pending) - 1
        for e in reversed(self.window(a)):
            if not e[1]:
                continue
            if j >= 0 and e[0] == pending[j]:
                j -= 1
            else:
                e[1] = False
        assert j == -1, (a, "pending records the window does not hold", pending[: j + 1])
        self._advance(a)

    def set_window(self, a, head, slots):
        """A hand-built window: head cursor and [(seq, live), ...] from head on (tests of the model itself)."""
        self.head[int(a)] = int(head)
        self.win[int(a)] = [[int(s), bool(v)] for s, v in slots]
        self._advance(a)


class BoundedOracle(WhereOracle):
    """A WhereOracle whose queues are bounded by a RingModel of `ring_slots` slots per agent.

    send_batch (ranked p2p), restores and sweeps are bounded as order-deterministic paths: the first records of the
    call are kept.  Group and list sends take either path on the device (the pull / list index build keeps send order,
    smaller batches and overlapping lists claim slots atomically), so a direct group or list send that would drop a
    record fails: the caller says which path the device took, `enqueue(send, ordered=True)` for an index build or
    `enqueue(send, keep=...)` with the survivors read from the device.  Records pending at construction start as
    contiguous windows.  `dropped` collects the (agent, seq) pairs the model drops;
    `take_dropped()` reads and clears it, as sdb_overflow_log does."""

    def __init__(self, inner, max_groups, ring_slots, groups=None, watermark=0):
        super().__init__(inner, max_groups, groups, watermark)
        self.ring = RingModel(ring_slots)
        self.dropped = []
        self.overflow = 0
        self._hold = 0
        for a, seqs in self._pending().items():
            self.ring.append(a, seqs)

    # ---- model upkeep
    def _pending(self):
        return {a: [int(h["seq"]) for h, _ in lst] for a, lst in self.snapshot().items()}

    def _retired(self):
        pend = self._pending()
        for a in list(self.ring.win):
            self.ring.retire_to(a, pend.get(a, []))

    def _appended(self, keep=None, ordered=True):
        state = self.snapshot()
        gone, lost = set(), {}
        for a in sorted(set(state) | set(self.ring.win)):
            seqs = [int(h["seq"]) for h, _ in state.get(a, [])]
            live = self.ring.live_seqs(a)
            assert seqs[: len(live)] == live, (a, "an append changed the records already queued")
            new = seqs[len(live):]
            if keep is not None and a in keep:
                want = [int(s) for s in keep[a]]
                kept_pos, k = [], 0
                for i, s in enumerate(new):
                    if k < len(want) and s == want[k]:
                        kept_pos.append(i)
                        k += 1
                assert k == len(want), (a, "survivors that were not sent", want[k:])
                assert len(want) == min(len(new), self.ring.capacity(a)), \
                    (a, "survivors must fill the free slots", len(want), len(new), self.ring.capacity(a))
                kept = set(kept_pos)
            else:
                kept = set(range(min(len(new), self.ring.capacity(a))))
                assert ordered or len(kept) == len(new), (a, "a drop on an atomic-claim path: pass the device's survivors")
            self.ring.append(a, [new[i] for i in sorted(kept)])
            for i in range(len(new)):
                if i not in kept:
                    gone.add((a, len(live) + i))
                    self.dropped.append((a, new[i]))
                    lost[a] = lost.get(a, 0) + 1
        if gone:
            self._replay({a: [r for i, r in enumerate(lst) if (a, i) not in gone] for a, lst in state.items()})
            for a, n in lost.items():                # a dropped record never reached the ring: not `received`
                self._recv_extra[a] -= n
            self.overflow += len(gone)

    @contextlib.contextmanager
    def appending(self, keep=None, ordered=True):
        """Several oracle sends bounded as one call (a restore, a sweep, a multi-part batch)."""
        self._hold += 1
        try:
            yield
        finally:
            self._hold -= 1
        if not self._hold:
            self._appended(keep, ordered)

    def enqueue(self, send, keep=None, ordered=False):
        """Run `send()` on this oracle and bound it as one call: keep={agent: survivor seqs} for an atomic-claim path
        (every receiver of the call listed), ordered=True for an order-deterministic one."""
        with self.appending(keep, ordered or keep is not None):
            return send()

    def take_dropped(self):
        out, self.dropped = self.dropped, []
        return out

    def capacity(self, a):
        return self.ring.capacity(a)

    # ---- sends: bounded after the call (unless inside `appending`)
    def _send(self, ordered, fn, *a, **k):
        if self._hold:
            return fn(*a, **k)
        with self.appending(None, ordered):
            return fn(*a, **k)

    def send_batch(self, *a, **k):
        return self._send(True, super().send_batch, *a, **k)

    def send_list_batch(self, *a, **k):
        return self._send(False, super().send_list_batch, *a, **k)

    def send_group_batch(self, *a, **k):
        return self._send(False, self.inner.send_group_batch, *a, **k)

    def send_group_seq(self, *a, **k):
        return self._send(False, self.inner.send_group_seq, *a, **k)

    # ---- retiring calls: tombstones after the call
    def receive_batch(self, agents, max_messages, flags=0, **kw):
        out = super().receive_batch(agents, max_messages, flags, **kw)
        if not flags & RECV_PEEK:
            self._retired()
        return out

    def receive_counts(self, agents, max_messages, flags=0):
        """Stream order only, and followed without a snapshot: its PEEK would fold into the oracle's stream digests,
        which digest drains (the only callers) have enabled."""
        assert not flags & RECV_PRIORITY
        cnt, total = self.inner.receive_counts(agents, max_messages, flags)
        if not flags & RECV_PEEK:
            idx = range(len(cnt)) if agents is None else np.asarray(agents).tolist()
            for a, k in zip(idx, cnt.tolist()):
                if k:
                    self.ring.retire(a, self.ring.live_seqs(a)[:k])
        return cnt, total

    def receive_where(self, *a, **k):
        out = super().receive_where(*a, **k)
        self._retired()
        return out

    def expire(self, *a, **k):
        out = super().expire(*a, **k)
        self._retired()
        return out
