"""Reference for dead letters of leased receives (sdb_lease_set_policy / sdb_lease_deliveries / sdb_lease_dead_letters)
on top of tests/lease_ref.py (TESTS ONLY).

Every lease carries a delivery count.  A sweep puts each redelivered record's count into a ledger keyed by (agent, seq)
together with the record's ring slot in the tests/ring_ref.py model: its absolute position p and the slot object itself,
which plays the arena handle (a slot object is unique while the record is pending, as a handle is).  Each leased receive
and sweep first drops the entries whose slot has left the window, is a tombstone or is no longer that object; the
leased receive then looks every returned record up and gives it count + 1 (1 when absent).  A sweep redelivers at most
the ledger's free room.  With a limit M, due leases at M become dead letters after a sweep's redelivery; they stay in
the store until dead_letters takes them, in the compact format (rows numbered by first appearance).
"""
from __future__ import annotations

import numpy as np

from tests.lease_ref import ACKED, LIVE, REDELIVERED, LeaseModel
from tests.restore_ref import restore_append

DEAD = 3


class DeadLetterModel(LeaseModel):
    def __init__(self, oracle, groups, rec_cap, cap, shared=True, max_deliveries=0, ledger_entries=0):
        super().__init__(oracle, groups, rec_cap, cap, shared)
        self.set_policy(max_deliveries, ledger_entries)
        self.dead_total = self.held_total = 0

    def set_policy(self, max_deliveries, ledger_entries):
        assert not any(r["state"] in (LIVE, DEAD) for r in self.recs)
        self.M, self.lcap = int(max_deliveries), int(ledger_entries) if max_deliveries else 0
        self.ledger = []              # {"agent", "seq", "count", "p", "slot", "taken"}; taken ones leave at a collection
        self._by_key = {}             # (agent, seq) -> its entries in ledger order
        self.taken = 0

    @property
    def policy(self):
        return self.M > 0

    # ---- the ledger
    def _add(self, en):
        en["taken"] = False
        self.ledger.append(en)
        self._by_key.setdefault((en["agent"], en["seq"]), []).append(en)

    def collect(self):
        ring = self.o.ring
        old, self.ledger, self._by_key, self.taken = self.ledger, [], {}, 0
        for en in old:
            if en["taken"]:
                continue
            w, h = ring.window(en["agent"]), ring.head[en["agent"]]
            i = en["p"] - h
            if 0 <= i < len(w) and w[i] is en["slot"] and w[i][1]:
                self._add(en)

    def _take(self, a, seq):
        """The first untaken entry of (agent, seq) in ledger order: its count, and the entry is taken."""
        for en in self._by_key.get((a, seq), []):
            if not en["taken"]:
                en["taken"] = True
                self.taken += 1
                return en["count"]
        return 0

    # ---- sdb_receive_leased
    def lease(self, agents, max_messages, deadline, flags=0, rows=None):
        if self.policy and self.ledger:
            self.collect()
        n0 = len(self.recs)
        out = super().lease(agents, max_messages, deadline, flags, rows)
        for r in self.recs[n0:]:
            r["deliveries"] = self._take(r["agent"], int(r["hdr"]["seq"])) + 1 if self.policy else 1
        return out

    # ---- sdb_lease_sweep
    def sweep(self, now, all_=False):
        if not self.policy:
            return super().sweep(now, all_)
        if self.ledger:
            self.collect()

        def due(r):
            return r["state"] == LIVE and (all_ or r["deadline"] <= now)

        at_limit = [r for r in self.recs if due(r) and r["deliveries"] >= self.M]
        aside = [r for r in self.recs if r["state"] == DEAD or (due(r) and r["deliveries"] >= self.M)]
        n_due = sum(1 for r in self.recs if due(r) and r["deliveries"] < self.M)
        n = min(n_due, self.rec_cap)
        held = n - min(n, self.lcap - len(self.ledger))
        ids = {id(r) for r in aside}
        chunk_due = [r for r in self.recs if due(r) and r["deliveries"] < self.M][: n - held]
        self.recs = [r for r in self.recs if id(r) not in ids]
        rec_cap, self.rec_cap = self.rec_cap, n - held
        try:
            red, blocked, _ = super().sweep(now, all_)
        finally:
            self.rec_cap = rec_cap
        # the redelivered records' counts go to the ledger: an agent's run of c sits at the end of its window
        by_agent = {}
        for r in chunk_due:
            if r["state"] == REDELIVERED:
                by_agent.setdefault(r["agent"], []).append(r)
        ring = self.o.ring
        for a, rs in by_agent.items():
            w, h = ring.window(a), ring.head[a]
            for j, r in enumerate(rs):
                i = len(w) - len(rs) + j
                self._add({"agent": a, "seq": int(r["hdr"]["seq"]), "count": r["deliveries"], "p": h + i, "slot": w[i]})
        for r in at_limit:
            r["state"] = DEAD
        self.live -= len(at_limit)
        self.dead_total += len(at_limit)
        self.held_total += held
        self.recs = sorted(self.recs + aside, key=lambda r: r["id"])
        return red, blocked, n_due - (n - held)

    # ---- sdb_lease_settle: dead letters are not live (LeaseModel's rule)

    # ---- sdb_lease_deliveries
    def deliveries(self, ids):
        by_id = {r["id"]: r for r in self.recs if r["state"] in (LIVE, DEAD)}
        return np.array([by_id[int(i)]["deliveries"] if int(i) in by_id else 0 for i in ids], np.uint32)

    # ---- sdb_lease_dead_letters
    def dead_letters(self, agents, rec_cap, peek=False):
        """(counts, entries, sends, payload, deliveries) of one call: agents in list order (None: every index below
        max_agents), lease-id order within an agent, the receive capacity rule with its lead-agent exception."""
        from swarmdb_b200._native import ENTRY_DTYPE, SEND_DTYPE
        listed = list(range(self.o.max_agents)) if agents is None else [int(a) for a in agents]
        per = {a: [] for a in listed}
        for r in self.recs:
            if r["state"] == DEAD and r["agent"] in per:
                per[r["agent"]].append(r)
        cnt = np.zeros(len(listed), np.uint32)
        took, m = [], 0
        for q, a in enumerate(listed):
            c = len(per[a])
            if m + c <= rec_cap:
                cnt[q] = c; took += per[a]; m += c
                continue
            if m == 0:
                cnt[q] = rec_cap; took += per[a][:rec_cap]
            break
        rows = {}
        for r in took:
            rows.setdefault(r["row"], len(rows))
        ent = np.zeros(len(took), ENTRY_DTYPE)
        snd = np.zeros(len(rows), SEND_DTYPE)
        pays = [None] * len(rows)
        for k, r in enumerate(took):
            j = rows[r["row"]]
            h = r["hdr"]
            ent[k] = (h["seq"], j, h["receiver"])
            snd[j] = (h["timestamp"], 0, h["sender"], h["group"], h["len"], h["prio"], h["type"], 0)
            pays[j] = r["pay"]
        lens = np.array([len(p) for p in pays], np.int64)
        if len(rows) > 1:
            snd["payload_off"][1:] = np.cumsum(lens)[:-1].astype(np.uint64)
        payload = np.concatenate(pays) if pays else np.zeros(0, np.uint8)
        deliv = np.array([r["deliveries"] for r in took], np.uint32)
        if not peek:
            gone = {id(r) for r in took}
            self.recs = [r for r in self.recs if id(r) not in gone and r["state"] != ACKED]
            self.acked = 0
        return cnt, ent, snd, payload, deliv

    def redrive(self, agents, counts, ent, snd, payload):
        """restore_compact of a dead-letter take, as it stands."""
        with self.o.appending():
            restore_append(self.o, self.groups, np.asarray(agents, np.uint32), np.asarray(counts, np.uint32), ent, snd, payload)

    def stats(self):
        out = super().stats()
        if self.policy:
            out["entries_used"] = len(self.recs)
        return out

    def policy_stats(self):
        return {"max_deliveries": self.M, "dead": sum(1 for r in self.recs if r["state"] == DEAD),
                "dead_total": self.dead_total, "ledger_used": len(self.ledger) - self.taken, "ledger_cap": self.lcap,
                "held_by_ledger_total": self.held_total}


# ---- the ledger's index (sdb_lease.cu: lg_slot): open addressing over slots = 2 x ledger_entries, probes run forward
# and wrap from the last slot to slot 0
_M64 = (1 << 64) - 1


def lg_slot(agent, seq, slots):
    """The first probe slot of (agent, seq), restated from sdb_lease.cu."""
    x = (int(seq) ^ (int(agent) * 0x9E3779B97F4A7C15)) & _M64
    x ^= x >> 33
    x = (x * 0xFF51AFD7ED558CCD) & _M64
    x ^= x >> 33
    x = (x * 0xC4CEB9FE1A85EC53) & _M64
    x ^= x >> 33
    return (x * int(slots)) >> 64


def seqs_at_slot(agent, slots, slot, start, n):
    """The first n seqs >= start whose probe for `agent` starts at `slot`."""
    out, s = [], int(start)
    while len(out) < n:
        if lg_slot(agent, s, slots) == slot:
            out.append(s)
        s += 1
    return out
