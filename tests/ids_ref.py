"""Reference for the id clause of the filtered receive (SDB_FILTER_IDS) on top of tests/where_ref.py (TESTS ONLY).

A record matches the clause when its seq is one of the filter's ids; every other clause is decided by `where_match`.
`ids_outputs` restates the per-id outputs: id_hits[i] counts the pending records of the listed agents with seq ==
ids[i] that pass every clause (before max_messages and the capacity cut), id_agent[i] is the smallest agent holding one
(NO_RECEIVER: none).  `IdsOracle.receive_where` is WhereOracle's, with that predicate and those outputs.
"""
from __future__ import annotations

import ctypes

import numpy as np

from oracle.cpu_ref import HDR_DTYPE
from tests.expire_ref import RECV_PEEK
from tests.where_ref import RECV_PRIORITY, WhereOracle, where_match

F_IDS = 512
NO_RECEIVER = 0xFFFFFFFF


def ids_of(filt) -> np.ndarray:
    """The filter's id list as u64 (empty without the clause)."""
    if not filt.fields & F_IDS or not filt.n_ids:
        return np.zeros(0, np.uint64)
    return np.ctypeslib.as_array(ctypes.cast(filt.ids, ctypes.POINTER(ctypes.c_uint64)), (int(filt.n_ids),)).copy()


def ids_match(h, padded: bytes, filt, idset) -> bool:
    if filt.fields & F_IDS and int(h["seq"]) not in idset:
        return False
    return where_match(h, padded, filt)


def ids_select(state, agents, max_messages, flags, filt, rec_cap):
    """where_ref.where_select with the id clause."""
    idset = set(ids_of(filt).tolist())
    counts, chosen, total, cut = [], [], 0, False
    for a in agents:
        recs = state.get(int(a), [])
        match = [i for i, (h, p) in enumerate(recs) if ids_match(h, p, filt, idset)]
        if flags & RECV_PRIORITY:
            match.sort(key=lambda i: -int(recs[i][0]["prio"]))
        match = match[:max_messages]
        take = 0 if cut else len(match)
        if not cut and match and total + len(match) > rec_cap:
            take, cut = (rec_cap if total == 0 else 0), True
        counts.append(take)
        chosen += [(int(a), i) for i in match[:take]]
        total += take
    return counts, chosen


def ids_outputs(state, agents, filt):
    """(id_hits, id_agent) in input order."""
    ids = ids_of(filt)
    idset = set(ids.tolist())
    hits, first = {}, {}
    for a in agents:
        for h, p in state.get(int(a), []):
            if ids_match(h, p, filt, idset):
                s = int(h["seq"])
                hits[s] = hits.get(s, 0) + 1
                first[s] = min(first.get(s, NO_RECEIVER), int(a))
    return (np.array([hits.get(int(s), 0) for s in ids], np.uint32),
            np.array([first.get(int(s), NO_RECEIVER) for s in ids], np.uint32))


class IdsOracle(WhereOracle):
    """WhereOracle whose receive_where also knows SDB_FILTER_IDS and fills id_hits / id_agent."""

    def receive_where(self, agents, max_messages, flags=0, filt=None, rec_cap=(1 << 64) - 1, drop=False,
                      id_hits=None, id_agent=None):
        state = self.snapshot()
        listed = np.arange(self._wm) if agents is None else np.asarray(agents, np.int64)
        if id_hits is not None or id_agent is not None:
            hits, first = ids_outputs(state, listed if max_messages else [], filt)
            if id_hits is not None:
                id_hits[:] = hits
            if id_agent is not None:
                id_agent[:] = first
        counts, chosen = ids_select(state, listed, max_messages, flags, filt, (1 << 64) - 1 if drop else rec_cap)
        out_counts = np.zeros(len(listed), np.uint32)
        out_counts[: len(counts)] = counts
        if chosen and not flags & RECV_PEEK:
            gone = set(chosen)
            self._replay({a: [rec for i, rec in enumerate(lst) if (a, i) not in gone] for a, lst in state.items()})
            if not drop:
                self.delivered += len(chosen)
        if drop:
            return out_counts, len(chosen)
        hdr = np.array([state[a][i][0] for a, i in chosen], HDR_DTYPE) if chosen else np.zeros(0, HDR_DTYPE)
        pay = np.frombuffer(b"".join(state[a][i][1] for a, i in chosen), np.uint8).copy()
        return out_counts, hdr, pay
