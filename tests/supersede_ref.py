"""Reference for superseding sends (sdb_supersede) on top of the trim model (TESTS ONLY).

`supersede_select` states the key, the newest-record rule, the scope and the capacity rule of include/swarmdb_b200.h
literally, on the model queue of `expire_ref` ({agent: [(header record, padded payload bytes), ...]} in ring order, so
records put back by a sweep, a restore or a requeue sit at the end).  `SupersedingOracle` is a `TrimmingOracle` whose
`supersede` removes the chosen records and replays the survivors, so every later receive is the unmodified oracle's
over a queue in which the superseded records were never sent.
"""
from __future__ import annotations

import numpy as np

from oracle.cpu_ref import HDR_DTYPE
from tests.expire_ref import RECV_PEEK
from tests.trim_ref import TrimmingOracle

TYPEF_SUPERSEDE = 0x20
TYPE_MASK = 0x07


def supersede_key(h):
    """The key of a flagged record (sender, group, type & TYPE_MASK); None for a record without the flag."""
    t = int(h["type"])
    if not t & TYPEF_SUPERSEDE:
        return None
    return int(h["sender"]), int(h["group"]), t & TYPE_MASK


def supersede_drops(recs):
    """Positions (ring order) of the superseded records of one agent: every flagged record but its key's newest, the
    largest seq, and on a tie in seq the one later in the ring."""
    newest = {}
    for i, (h, _) in enumerate(recs):
        k = supersede_key(h)
        if k is not None and (k not in newest or int(h["seq"]) >= newest[k][0]):
            newest[k] = (int(h["seq"]), i)
    return [i for i, (h, _) in enumerate(recs) if supersede_key(h) is not None and newest[supersede_key(h)][1] != i]


def supersede_select(state, agents, flags, rec_cap):
    """sdb_supersede's selection: per listed agent its superseded records, agents laid out in list order; an agent
    whose records do not all fit stays whole with every later agent, except the first agent in the output, which gives
    its first rec_cap in ring order.  Returns (counts, [(agent, position in its list)])."""
    counts, chosen, total, cut = [], [], 0, False
    for a in agents:
        drops = supersede_drops(state.get(int(a), []))
        take = 0 if cut else len(drops)
        if not cut and drops and total + len(drops) > rec_cap:
            take, cut = (rec_cap if total == 0 else 0), True
        counts.append(take)
        chosen += [(int(a), i) for i in drops[:take]]
        total += take
    return counts, chosen


class SupersedingOracle(TrimmingOracle):
    """A TrimmingOracle with `supersede`."""

    def supersede(self, agents, flags: int = 0, rec_cap: int = (1 << 64) - 1, materialise: bool = True):
        """sdb_supersede's result: (counts, headers, padded payloads) in the full receive format (the device's compact
        output expands to it), or (counts, total) with materialise=False; PEEK retires nothing."""
        state = self.snapshot()
        listed = np.arange(self._wm) if agents is None else np.asarray(agents, np.int64)
        counts, chosen = supersede_select(state, listed, flags, rec_cap)
        out_counts = np.zeros(self.max_agents if agents is None else len(listed), np.uint32)
        out_counts[: len(counts)] = counts
        hdr = np.array([state[a][i][0] for a, i in chosen], HDR_DTYPE) if chosen else np.zeros(0, HDR_DTYPE)
        pay = np.frombuffer(b"".join(state[a][i][1] for a, i in chosen), np.uint8).copy()
        if chosen and not flags & RECV_PEEK:
            gone = set(chosen)
            self._replay({a: [rec for i, rec in enumerate(lst) if (a, i) not in gone] for a, lst in state.items()})
        if not materialise:
            return out_counts, len(chosen)
        return out_counts, hdr, pay
