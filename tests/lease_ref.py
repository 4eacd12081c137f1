"""Reference for leased receives (sdb_receive_leased / sdb_lease_settle / sdb_lease_sweep) on the CPU oracle (TESTS ONLY).

A lease is the unchanged oracle's receive plus a Python store that keeps every returned record (header and padded
payload) with its lease id, agent, deadline and state.  A sweep takes the live due records in lease-id order, at most
`rec_cap` of them, groups them by agent (ascending agent index, lease-id order within an agent), drops every agent whose
ring cannot take all of its records, and appends the rest with tests/restore_ref.py::restore_append, agent by agent.
Acked and redelivered records then leave the store.

Row identity is not visible in the full format, so a caller that wants the arena advance of a sweep predicted
(`last_granules`) passes each lease's row numbers (the compact result's entry.send); rows are then numbered by their
smallest redelivered seq, as the device does, and restore_ref.restore_granules gives the region.
"""
from __future__ import annotations

import numpy as np

from tests.restore_ref import restore_append, restore_granules

LIVE, ACKED, REDELIVERED = 0, 1, 2


def _pad32(n):
    return (n + 31) & ~31


class LeaseModel:
    """`oracle` is a tests/ring_ref.py::BoundedOracle: its ring model decides which agents a sweep blocks."""

    def __init__(self, oracle, groups, rec_cap, cap, shared=True):
        self.o, self.groups, self.rec_cap, self.cap, self.shared = oracle, groups, rec_cap, cap, shared
        self.recs = []            # dicts in lease-id order
        self.next_id = 0
        self.n_leases = 0         # leased calls so far (row keys are (call, row))
        self.live = self.acked = self.redelivered_total = self.acked_total = 0
        self.last_granules = 0
        self.last_staged = []     # [(agent, [records])] the last sweep redelivered

    # ---- sdb_receive_leased
    def lease(self, agents, max_messages, deadline, flags=0, rows=None):
        """The oracle's receive of what one leased call takes (capacity: rec_cap and free store entries); returns the
        oracle's (counts, headers, payload) and the lease base."""
        cap = min(self.rec_cap, self.cap - len(self.recs))
        cnt, hdr, pay = self._receive(agents, max_messages, flags, cap)
        idx = np.arange(len(cnt)) if agents is None else np.asarray(agents)
        who = np.repeat(idx, cnt.astype(np.int64))
        off = 0
        base = self.next_id
        for r in range(len(hdr)):
            pl = _pad32(int(hdr[r]["len"]))
            self.recs.append({"id": base + r, "agent": int(who[r]), "hdr": hdr[r].copy(), "pay": pay[off:off + pl].copy(),
                              "deadline": float(deadline), "state": LIVE,
                              "row": (self.n_leases, int(rows[r]) if rows is not None else r)})
            off += pl
        self.next_id += len(hdr)
        self.n_leases += 1
        self.live += len(hdr)
        return cnt, hdr, pay, base

    def _receive(self, agents, k, flags, cap):
        """The oracle's receive under the capacity rule of include/swarmdb_b200.h (the oracle has none): agents in list
        order while their records fit, or the lead agent alone with its first `cap` records."""
        from oracle.cpu_ref import HDR_DTYPE
        big = 1 << 21
        agents = np.arange(self.o.max_agents, dtype=np.uint32) if agents is None else np.asarray(agents, np.uint32)
        want = self.o.receive_batch(agents, k, (flags & 1) | 2, rec_cap=big)[0]          # PRIORITY bit kept, PEEK
        acc, cut, lead = 0, len(agents), False
        for q in range(len(agents)):
            if acc + int(want[q]) > cap:
                cut, lead = q, acc == 0
                break
            acc += int(want[q])
        cnt = np.zeros(len(agents), np.uint32)
        sub, kk = (agents[cut:cut + 1], cap) if lead else (agents[:cut], k)
        if len(sub) == 0 or kk == 0:
            return cnt, np.zeros(0, HDR_DTYPE), np.zeros(0, np.uint8)
        cc, hc, pc = self.o.receive_batch(sub, kk, flags, rec_cap=big)
        if lead:
            cnt[cut] = cc[0]
        else:
            cnt[:cut] = cc
        return cnt, hc, pc

    # ---- sdb_lease_settle
    def settle(self, ids, op, deadline=0.0):
        by_id = {r["id"]: r for r in self.recs}
        out = np.zeros(len(ids), np.uint8)
        live_before = {i for i in (int(x) for x in ids) if i in by_id and by_id[i]["state"] == LIVE}
        for k, i in enumerate(int(x) for x in ids):
            if i in live_before:
                out[k] = 1
                if op == 0:
                    if by_id[i]["state"] == LIVE:
                        by_id[i]["state"] = ACKED
                        self.live -= 1; self.acked += 1; self.acked_total += 1
                else:
                    by_id[i]["deadline"] = float(deadline)
        return out, int(out.sum())

    # ---- sdb_lease_sweep
    def sweep(self, now, all_=False):
        due = [r for r in self.recs if r["state"] == LIVE and (all_ or r["deadline"] <= now)]
        chunk = due[: self.rec_cap]
        by_agent = {}
        for r in chunk:
            by_agent.setdefault(r["agent"], []).append(r)
        staged, blocked = [], 0
        for a in sorted(by_agent):
            rs = by_agent[a]
            if len(rs) > self.o.capacity(a):         # tail - head counts tombstones: pending records alone do not
                blocked += 1
            else:
                staged.append((a, rs))
        flat = [r for _, rs in staged for r in rs]
        self.last_granules = 0
        self.last_staged = staged
        if flat:
            agents, counts, ent, snd, payload = self.staged_input(staged)
            with self.o.appending():
                restore_append(self.o, self.groups, agents, counts, ent, snd, payload)
            self.last_granules = restore_granules(counts, ent, snd, self.shared, agents)
            for r in flat:
                r["state"] = REDELIVERED
        self.live -= len(flat); self.redelivered_total += len(flat)
        self.recs = [r for r in self.recs if r["state"] == LIVE]
        self.acked = 0
        return len(flat), blocked, len(due) - len(chunk)

    @staticmethod
    def staged_input(staged, seq_key=int):
        """The restore input of a sweep's staged records [(agent, [records])]: (agents, counts, entries, sends,
        payload), rows numbered by smallest seq_key(seq) (ties: first in agent order), one payload each.  A seq_key
        other than the identity shows what a sort on part of the seq would have numbered."""
        from swarmdb_b200._native import ENTRY_DTYPE, SEND_DTYPE
        flat = [r for _, rs in staged for r in rs]
        first = {}
        for p, r in sorted(enumerate(flat), key=lambda t: (seq_key(int(t[1]["hdr"]["seq"])), t[0])):
            first.setdefault(r["row"], len(first))
        ent = np.zeros(len(flat), ENTRY_DTYPE)
        snd = np.zeros(len(first), SEND_DTYPE)
        pays = [None] * len(first)
        for k, r in enumerate(flat):
            j = first[r["row"]]
            ent[k] = (r["hdr"]["seq"], j, r["hdr"]["receiver"])
            h = r["hdr"]
            snd[j] = (h["timestamp"], 0, h["sender"], h["group"], h["len"], h["prio"], h["type"], 0)
            pays[j] = r["pay"]
        off = np.zeros(len(first), np.int64)
        lens = np.array([len(p) for p in pays], np.int64)
        if len(first) > 1:
            off[1:] = np.cumsum(lens)[:-1]
        snd["payload_off"] = off.astype(np.uint64)
        payload = np.concatenate(pays) if pays else np.zeros(0, np.uint8)
        agents = np.array([a for a, _ in staged], np.uint32)
        counts = np.array([len(rs) for _, rs in staged], np.uint32)
        return agents, counts, ent, snd, payload

    def stats(self):
        return {"live": self.live, "acked_unreclaimed": self.acked, "redelivered_total": self.redelivered_total,
                "acked_total": self.acked_total, "entries_used": len(self.recs)}
