"""Reference for the filtered receive (sdb_receive_where) on top of tests/expire_ref.py (TESTS ONLY).

The contract of sdb_receive_where is that its result equals what sdb_receive_batch returns on a queue holding only the
matching records, and that every later receive delivers what it would have delivered had the taken records been
received.  `WhereOracle` restates it literally: it reads the pending records of the wrapped CpuOracle (a PEEK receive),
decides every record with `where_match` (plain Python), selects the first max_messages matches per agent in delivery
order with the capacity rule, and replays the survivors into a fresh oracle (ExpiringOracle._replay).  `delivered`
counts what sdb_stats.delivered counts: records returned by receives that are not PEEKs, filtered or not.
"""
from __future__ import annotations

import ctypes

import numpy as np

from oracle.cpu_ref import HDR_DTYPE
from tests.expire_ref import RECV_PEEK, ExpiringOracle

RECV_PRIORITY = 1
WHERE_DROP = 32
TYPEF_EXTRAS = 0x10
F_SENDER, F_RECEIVER, F_GROUP, F_TYPE, F_PRIO, F_TIME, F_SEQ, F_KEYWORD, F_ICASE = 1, 2, 4, 8, 16, 32, 64, 128, 256


def content_bytes(h, padded: bytes) -> bytes:
    """The bytes a keyword is matched against: payload [0, len), or with TYPEF_EXTRAS [4, 4 + clen), clen = the
    little-endian u32 at the payload's start clamped to len - 4 (empty when len < 4)."""
    n = int(h["len"])
    if int(h["type"]) & TYPEF_EXTRAS:
        if n < 4:
            return b""
        clen = int.from_bytes(padded[:4], "little")
        return padded[4:4 + min(clen, n - 4)]
    return padded[:n]


def fold_ascii(b: bytes) -> bytes:
    return bytes(c + 32 if 65 <= c <= 90 else c for c in b)


def keyword_of(filt) -> bytes:
    return ctypes.string_at(filt.keyword, filt.keyword_len) if filt.keyword_len else b""


def where_match(h, padded: bytes, filt) -> bool:
    """One record against an SdbFilter, clause by clause as include/swarmdb_b200.h states them."""
    f = int(filt.fields)
    if f & F_SENDER and int(h["sender"]) != filt.sender:
        return False
    if f & F_RECEIVER and int(h["receiver"]) != filt.receiver:
        return False
    if f & F_GROUP and int(h["group"]) != filt.group:
        return False
    if f & F_TYPE and not (filt.type_mask >> (int(h["type"]) & 7)) & 1:
        return False
    if f & F_PRIO and not (int(h["prio"]) < 8 and (filt.prio_mask >> int(h["prio"])) & 1):
        return False
    if f & F_TIME and not (filt.after < float(h["timestamp"]) < filt.before):
        return False
    if f & F_SEQ and not (filt.seq_lo <= int(h["seq"]) < filt.seq_hi):
        return False
    if f & F_KEYWORD and filt.keyword_len:
        kw, text = keyword_of(filt), content_bytes(h, padded)
        if f & F_ICASE:
            kw, text = fold_ascii(kw), fold_ascii(text)
        if kw not in text:
            return False
    return True


def where_select(state, agents, max_messages, flags, filt, rec_cap):
    """The selection on a model queue {agent: [(header, padded payload), ...]} in stream order: per listed agent the
    first max_messages matches in delivery order (priority order: priority descending, stream order within a level),
    agents laid out in list order; an agent whose matches do not all fit stays whole with every later agent, except
    the first agent in the output, which gives its first rec_cap.  Returns (counts, [(agent, position)]) in output order."""
    counts, chosen, total, cut = [], [], 0, False
    for a in agents:
        recs = state.get(int(a), [])
        match = [i for i, (h, p) in enumerate(recs) if where_match(h, p, filt)]
        if flags & RECV_PRIORITY:
            match.sort(key=lambda i: -int(recs[i][0]["prio"]))          # stable: stream order within a level
        match = match[:max_messages]
        take = 0 if cut else len(match)
        if not cut and match and total + len(match) > rec_cap:
            take, cut = (rec_cap if total == 0 else 0), True
        counts.append(take)
        chosen += [(int(a), i) for i in match[:take]]
        total += take
    return counts, chosen


class WhereOracle(ExpiringOracle):
    """ExpiringOracle + receive_where, and the `delivered` counter of sdb_stats."""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.delivered = 0

    def receive_batch(self, agents, max_messages, flags=0, **kw):
        out = self.inner.receive_batch(agents, max_messages, flags, **kw)
        if not flags & RECV_PEEK:
            self.delivered += len(out[1])
        return out

    def receive_where(self, agents, max_messages, flags=0, filt=None, rec_cap=(1 << 64) - 1, drop=False):
        """sdb_receive_where's result: (counts, headers, padded payloads), or (counts, total) with drop=True."""
        state = self.snapshot()
        listed = np.arange(self._wm) if agents is None else np.asarray(agents, np.int64)
        counts, chosen = where_select(state, listed, max_messages, flags, filt, (1 << 64) - 1 if drop else rec_cap)
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
