"""Reference for bounded queues (sdb_trim) on top of the expiry model (TESTS ONLY).

`trim_select` states the selection, eviction order and capacity rule of include/swarmdb_b200.h literally, on the model
queue of `expire_ref` ({agent: [(header record, padded payload bytes), ...]} in stream order).  `TrimmingOracle` is an
`ExpiringOracle` (by way of `WhereOracle`, so filtered takes are modelled too) whose `trim` removes the chosen records
and replays the survivors, so every later receive is the unmodified oracle's over a queue in which the trimmed records
were never sent.
"""
from __future__ import annotations

import numpy as np

from oracle.cpu_ref import HDR_DTYPE
from tests.expire_ref import RECV_PEEK, _pad32
from tests.where_ref import WhereOracle

RECV_PRIORITY = 1


def eviction_order(recs, flags):
    """Positions of an agent's records in eviction order: stream order, or with RECV_PRIORITY level 0 first, then 1, 2,
    3, stream order within a level."""
    idx = list(range(len(recs)))
    if flags & RECV_PRIORITY:
        idx.sort(key=lambda i: (int(recs[i][0]["prio"]), i))
    return idx


def trim_drops(recs, max_records, max_bytes, flags):
    """The shortest prefix of the eviction order whose removal leaves at most max_records records and at most
    max_bytes (rounded down to 32-byte granules) of pad32(len) payload; 0 is no limit.  In eviction order."""
    n_cap = max_records if max_records else float("inf")
    b_cap = max_bytes // 32 * 32 if max_bytes else float("inf")
    left_n, left_b = len(recs), sum(_pad32(int(h["len"])) for h, _ in recs)
    drops = []
    for i in eviction_order(recs, flags):
        if left_n <= n_cap and left_b <= b_cap:
            break
        drops.append(i)
        left_n -= 1
        left_b -= _pad32(int(recs[i][0]["len"]))
    return drops


def trim_select(state, agents, max_records, max_bytes, flags, rec_cap):
    """sdb_trim's selection: per listed agent its drops (trim_drops), agents laid out in list order; an agent whose drops
    do not all fit stays whole with every later agent, except the first agent in the output, which gives the first
    rec_cap of its eviction order.  Returns (counts, [(agent, position in its list)]), stream order within an agent."""
    counts, chosen, total, cut = [], [], 0, False
    for a in agents:
        drops = trim_drops(state.get(int(a), []), max_records, max_bytes, flags)
        take = 0 if cut else len(drops)
        if not cut and drops and total + len(drops) > rec_cap:
            take, cut = (rec_cap if total == 0 else 0), True
        counts.append(take)
        chosen += [(int(a), i) for i in sorted(drops[:take])]
        total += take
    return counts, chosen


class TrimmingOracle(WhereOracle):
    """A WhereOracle (an ExpiringOracle with filtered receives) with `trim`."""

    def trim(self, agents, max_records: int = 0, max_bytes: int = 0, flags: int = 0, rec_cap: int = (1 << 64) - 1,
             materialise: bool = True):
        """sdb_trim's result: (counts, headers, padded payloads) in the full receive format (the device's compact output
        expands to it), or (counts, total) with materialise=False; PEEK retires nothing."""
        state = self.snapshot()
        listed = np.arange(self._wm) if agents is None else np.asarray(agents, np.int64)
        counts, chosen = trim_select(state, listed, max_records, max_bytes, flags, rec_cap)
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
