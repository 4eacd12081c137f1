"""CPU model of deduplicated sends (include/swarmdb_b200.h "deduplicated sends"): the content key in numpy, bit for bit
as sdb_dedup.cu computes it, the table with its window, capacity and rebuild rule, and the verdicts of a batch.  The
accepted sends are replayed into the queue oracle one by one at the sequence numbers the whole batch gives them, so
the oracle's queues are what the device must hold (as tests/ids_ref.py layers the id clause on the same oracle)."""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

M64 = (1 << 64) - 1
PHI = 0x9E3779B97F4A7C15
SEED_A = 0x243F6A8885A308D3
SEED_B = 0x13198A2E03707344


def _mix64(z: np.ndarray) -> np.ndarray:
    z = np.asarray(z, np.uint64)
    with np.errstate(over="ignore"):
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def content_words(sender: int, kind: int, target: int, recipients: Optional[Sequence[int]], length: int, prio: int,
                  typ: int, payload: bytes) -> np.ndarray:
    """The identity of a send as 64-bit words: sender | kind << 32, target (or the list's length), the list's
    recipients, len | prio << 16 | type << 24, then the payload little-endian with bytes past len zero."""
    rec = np.asarray(recipients if kind == 2 else [], np.uint64)
    head = [sender | (kind << 32), len(rec) if kind == 2 else target]
    pb = bytes(payload[:length]) + b"\0" * ((-length) % 8)
    pw = np.frombuffer(pb, "<u8").astype(np.uint64) if pb else np.zeros(0, np.uint64)
    return np.concatenate([np.asarray(head, np.uint64), rec, np.asarray([length | prio << 16 | typ << 24], np.uint64), pw])


def content_key(sender: int, kind: int, target: int, recipients, length: int, prio: int, typ: int,
                payload: bytes) -> Tuple[int, int]:
    """(lo, hi): S_x = sum_j mix64(w_j + SEED_x + (j + 1) PHI), key = (mix64(S_a ^ m), mix64(S_b ^ (m << 32)))."""
    w = content_words(sender, kind, target, recipients, length, prio, typ, payload)
    m = len(w)
    with np.errstate(over="ignore"):
        pos = (np.arange(1, m + 1, dtype=np.uint64) * np.uint64(PHI))
        sa = int(_mix64(w + np.uint64(SEED_A) + pos).sum(dtype=np.uint64))
        sb = int(_mix64(w + np.uint64(SEED_B) + pos).sum(dtype=np.uint64))
    lo = int(_mix64(np.uint64(sa ^ m)))
    hi = int(_mix64(np.uint64(sb ^ ((m << 32) & M64))))
    if lo == 0 and hi == 0:
        lo = 1
    return lo, hi


def content_keys(sender, kind, target, list_off, list_idx, lens, prio, typ, payload_off, payload):
    """content_key of every send of a mixed batch as (lo, hi) uint64 arrays.  Sends with the same word layout (the same
    len, and for a list send the same list length) share one matrix of words, so a batch of tens of thousands of sends
    costs one numpy pass per layout instead of one call per send."""
    sender, kind, target = (np.asarray(x, np.uint64) for x in (sender, kind, target))
    lens, off = np.asarray(lens, np.int64), np.asarray(payload_off, np.int64)
    lpt = lens.astype(np.uint64) | np.asarray(prio, np.uint64) << np.uint64(16) | np.asarray(typ, np.uint64) << np.uint64(24)
    lo_, hi_ = np.zeros(len(lens), np.uint64), np.zeros(len(lens), np.uint64)
    lb = np.zeros(len(lens), np.int64)
    cnt = np.full(len(lens), -1, np.int64)                       # -1: not a list send
    lst = np.flatnonzero(kind == 2)
    if len(lst):
        lo_off = np.asarray(list_off, np.int64)
        lb[lst] = lo_off[target[lst].astype(np.int64)]
        cnt[lst] = lo_off[target[lst].astype(np.int64) + 1] - lb[lst]
    layouts, which = np.unique(np.stack([cnt, lens], 1), axis=0, return_inverse=True)
    pay = np.asarray(payload, np.uint8)
    for u, (c, ln) in enumerate(layouts.tolist()):
        idx = np.flatnonzero(which.ravel() == u)
        nr, nw = max(c, 0), (ln + 7) // 8
        m = 3 + nr + nw
        w = np.zeros((len(idx), m), np.uint64)
        w[:, 0] = sender[idx] | kind[idx] << np.uint64(32)
        w[:, 1] = np.uint64(c) if c >= 0 else target[idx]
        if nr:
            w[:, 2:2 + nr] = np.asarray(list_idx, np.uint64)[lb[idx][:, None] + np.arange(nr)]
        w[:, 2 + nr] = lpt[idx]
        if ln:
            b = np.zeros((len(idx), nw * 8), np.uint8)
            b[:, :ln] = pay[off[idx][:, None] + np.arange(ln)]
            w[:, 3 + nr:] = b.view("<u8").astype(np.uint64)
        with np.errstate(over="ignore"):
            pos = np.arange(1, m + 1, dtype=np.uint64) * np.uint64(PHI)
            sa = _mix64(w + np.uint64(SEED_A) + pos).sum(axis=1, dtype=np.uint64)
            sb = _mix64(w + np.uint64(SEED_B) + pos).sum(axis=1, dtype=np.uint64)
        lo_[idx] = _mix64(sa ^ np.uint64(m))
        hi_[idx] = _mix64(sb ^ np.uint64((m << 32) & M64))
    lo_[(lo_ == 0) & (hi_ == 0)] = 1
    return lo_, hi_


def edge_lengths(max_len: int) -> list:
    """Payload lengths at the edges of a content key's 16-byte loads and 512-byte warp steps: 0, 1-17, every residue
    mod 16 around the first four 512-byte boundaries, 1023-1025, 8191 and max_len."""
    out = set(range(0, 18)) | {1023, 1024, 1025, 8191, max_len}
    for k in range(1, 5):
        out |= set(range(512 * k - 16, 512 * k + 17))
    return sorted(x for x in out if x <= max_len)


def table_mask(entries: int) -> int:
    """Slot mask of a table reserved for `entries` keys: pow2_at_least(2 entries) - 1, at least 64 slots."""
    p = 64
    while p < 2 * entries:
        p <<= 1
    return p - 1


def slot_hash(lo, hi) -> np.ndarray:
    """The home slot hash of sdb_dedup.cu: mix64(lo ^ rotl(hi, 32)), before the mask."""
    lo, hi = np.asarray(lo, np.uint64), np.asarray(hi, np.uint64)
    return _mix64(lo ^ ((hi << np.uint64(32)) | (hi >> np.uint64(32))))


class DedupModel:
    """The table as the host and the kernels keep it: key -> [seq, inserted_at] for every occupied slot (live,
    expired or forgotten until a rebuild drops it)."""

    def __init__(self, entries: int, window: float):
        self.entries, self.window = entries, float(window)
        self.tab: Dict[Tuple[int, int], List[float]] = {}
        self.last_now = -np.inf
        self.accepted = self.dups = self.expired = self.forgotten = self.rebuilds = 0

    def live(self, k, now) -> bool:
        e = self.tab.get(k)
        return e is not None and now < e[1] + self.window

    def verdicts(self, keys: Sequence[Tuple[int, int]], seq_of: Sequence[int], now: float):
        """dup_of per send (0: accepted) and the number of new keys, for a batch whose send i starts at seq_of[i]."""
        first: Dict[Tuple[int, int], int] = {}
        dup_of, n_new = [], 0
        for i, k in enumerate(keys):
            if k == (0, 0):
                dup_of.append(0)
                continue
            if self.live(k, now):
                dup_of.append(int(self.tab[k][0]))
            elif k in first:
                dup_of.append(int(seq_of[first[k]]))
            else:
                first[k] = i
                dup_of.append(0)
                n_new += 1
        return dup_of, n_new

    def send(self, keys, seq_of, now: float):
        """The verdicts and the capacity rule of one call.  Raises OverflowError (SDB_ECAPACITY) and changes nothing when
        the new keys do not fit beside the entries live at `now`."""
        dup_of, n_new = self.verdicts(keys, seq_of, now)
        if len(self.tab) + n_new > self.entries:
            if sum(1 for k in self.tab if self.live(k, now)) + n_new > self.entries:
                raise OverflowError("table full of live entries")
        return dup_of, n_new

    def commit(self, keys, seq_of, dup_of, n_new, now: float) -> None:
        """The rebuild (when the new keys overflow the occupied slots) and the inserts after an accepted enqueue."""
        if len(self.tab) + n_new > self.entries:
            self.rebuild(now)
        for k, s, d in zip(keys, seq_of, dup_of):
            if k != (0, 0) and d == 0:
                self.tab[k] = [int(s), float(now)]
        self.accepted += n_new
        self.dups += sum(1 for d in dup_of if d)
        self.last_now = now

    def rebuild(self, now: float) -> None:
        keep = {k: e for k, e in self.tab.items() if now < e[1] + self.window}
        self.expired += len(self.tab) - len(keep)
        self.tab = keep
        self.rebuilds += 1

    def forget(self, keys) -> List[int]:
        out = []
        for k in keys:
            k = tuple(int(x) for x in k)
            r = 1 if self.live(k, self.last_now) else 0
            if k in self.tab:
                self.tab[k][1] = -np.inf
            out.append(r)
            self.forgotten += r
        return out

    def stats(self) -> dict:
        return {"capacity": self.entries, "live": sum(1 for k in self.tab if self.live(k, self.last_now)),
                "used": len(self.tab), "window": self.window, "accepted_total": self.accepted,
                "duplicate_total": self.dups, "expired_total": self.expired, "forgotten_total": self.forgotten,
                "rebuilds": self.rebuilds}


def batch_seqs(next_seq: int, kind, target, group_sizes: Dict[int, int]) -> List[int]:
    """First seq of each send of a mixed batch: a group send takes one per member (the sender's own included)."""
    out, s = [], next_seq
    for k, t in zip(kind, target):
        out.append(s)
        s += group_sizes[int(t)] if int(k) == 1 else 1
    return out


def replay(oracle, kind, sender, target, list_off, list_idx, prio, typ, lens, payload_off, payload, ts, seq_of, keep,
           end_seq: int) -> None:
    """Write the accepted sends into the queue oracle, each at its own seq, and leave its counter at end_seq."""
    for i in np.flatnonzero(keep):
        oracle.next_seq = int(seq_of[i])
        one = dict(prio=np.asarray(prio)[i:i + 1], typ=np.asarray(typ)[i:i + 1], lens=np.asarray(lens)[i:i + 1],
                   payload_off=np.zeros(1, np.uint64), ts=np.asarray(ts, np.float64)[i:i + 1])
        o, ln = int(payload_off[i]), int(lens[i])
        pl = np.zeros(max(16, ln), np.uint8)
        pl[:ln] = payload[o:o + ln]
        k, t = int(kind[i]), int(target[i])
        if k == 0:
            oracle.send_batch(np.asarray([sender[i]], np.uint32), np.asarray([t], np.uint32), one["prio"], one["typ"],
                              one["lens"], one["payload_off"], pl, one["ts"])
        elif k == 1:
            oracle.send_group_batch(np.asarray([sender[i]], np.uint32), np.asarray([t], np.uint32), one["prio"],
                                    one["typ"], one["lens"], one["payload_off"], pl, one["ts"])
        else:
            rec = np.asarray(list_idx[int(list_off[t]):int(list_off[t + 1])], np.uint32)
            oracle.send_list_batch(np.asarray([sender[i]], np.uint32), np.asarray([0, len(rec)], np.uint64), rec,
                                   one["prio"], one["typ"], one["lens"], one["payload_off"], pl, one["ts"])
    oracle.next_seq = end_seq
