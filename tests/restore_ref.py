"""Reference for restore (sdb_restore_compact) on top of the CPU oracle (TESTS ONLY).

The contract of sdb_restore_compact is that each listed agent gets its records appended behind whatever it has pending,
with their own sequence numbers and header fields, and that every later receive delivers what it would deliver had
those records been sent in that position.  `restore_append` restates it literally: it sends every record to the
unmodified CpuOracle, one at a time and in entry order, with its original seq (the per-record replay of
tests/expire_ref.py::_replay), then puts the group table and the sequence counter back.

`restore_granules` is a pure-Python model of the arena placement rule, so tests can predict arena_tail_bytes.
"""
from __future__ import annotations

import numpy as np

NO_GROUP = 0xFFFFFFFF
NO_RECEIVER = 0xFFFFFFFF
HDRS_PER_PAYLOAD = 65535


def _pad32(n):
    return (n + 31) & ~31


def _records(counts, entries, agents):
    """(agent, entry index) of every record, in entry order."""
    e = 0
    for a, c in zip(np.asarray(agents).tolist(), np.asarray(counts).tolist()):
        for _ in range(int(c)):
            yield int(a), e
            e += 1


def restore_append(oracle, groups, agents, counts, entries, sends, payload, skip=None):
    """Append the records to `oracle` as sdb_restore_compact does.  groups: {g: members} of the oracle, restored
    afterwards (the replay of a group record re-points its group at the one receiver).  skip(a) -> True leaves an
    agent's entries out (SDB_RECV_OWNED).  Returns the records appended."""
    zero = np.zeros(1, np.uint64)
    pay = np.asarray(payload, np.uint8)
    next_seq, top, n = oracle.next_seq, 0, 0
    for a, e in _records(counts, entries, agents):
        if skip is not None and skip(a):
            continue
        en, row = entries[e], sends[int(entries[e]["send"])]
        off, ln = int(row["payload_off"]), int(row["len"])
        buf = np.concatenate([pay[off:off + _pad32(ln)], np.zeros(32, np.uint8)])
        s, pr, ty, ts = [int(row["sender"])], [int(row["prio"])], [int(row["type"])], [float(row["timestamp"])]
        seq = int(en["seq"])
        if int(en["receiver"]) == NO_RECEIVER:
            oracle.next_seq = seq
            oracle.send_list_batch(s, [0, 1], [a], pr, ty, [ln], zero, buf, ts)
        elif int(row["group"]) == NO_GROUP:
            oracle.next_seq = seq
            oracle.send_batch(s, [a], pr, ty, [ln], zero, buf, ts)
        else:
            g = int(row["group"])
            oracle.create_group_pos(g, [a], [0])
            oracle.send_group_seq(s, [g], pr, ty, [ln], zero, buf, [seq], ts)
        top, n = max(top, seq), n + 1
    for g, m in groups.items():
        oracle.create_group_pos(g, m, np.arange(len(m), dtype=np.uint32))
    oracle.next_seq = max(next_seq, top + 1) if n else next_seq
    return n


def restore_granules(counts, entries, sends, shared=True, agents=None, skip=None):
    """Arena granules one sdb_restore_compact call takes: rows (in the shared layout) hold their shared headers and one
    payload per block of at most 65535 headers; every private record (each entry from its agent's first row descent on,
    or all of them with shared=False) takes 1 + pad32(len) / 32."""
    sends = np.asarray(sends)
    row_n = {}
    private = 0
    e = 0
    agents = np.arange(len(counts)) if agents is None else np.asarray(agents)
    for a, c in zip(agents.tolist(), np.asarray(counts).tolist()):
        rows = [int(x) for x in entries["send"][e:e + int(c)]]
        e += int(c)
        if skip is not None and skip(a):
            continue
        d = len(rows) if shared else 0
        for j in range(1, len(rows)):
            if rows[j] < rows[j - 1]:
                d = min(d, j)
                break
        for j, r in enumerate(rows):
            if j < d:
                row_n[r] = row_n.get(r, 0) + 1
            else:
                private += 1 + _pad32(int(sends[r]["len"])) // 32
    rows_total = sum(n + -(-n // HDRS_PER_PAYLOAD) * (_pad32(int(sends[r]["len"])) // 32) for r, n in row_n.items())
    return rows_total + private
