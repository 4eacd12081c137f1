"""Reference for snapshots of the lease store and the redelivery ledger (sdb_lease_export / sdb_lease_import /
sdb_lease_ledger_export / sdb_lease_ledger_import) on top of tests/deadletter_ref.py (TESTS ONLY).

Export is the model's live and dead records with id >= start in id order, at most rec_cap of them, rows numbered by first
appearance of their store row.  Import appends records with new ids behind what the store holds, each its own store row
key per (import call, row).  A ledger import gives each (agent, seq, count) triple an entry on the agent's oldest live
slot with that seq, if there is one.
"""
from __future__ import annotations

import numpy as np

from tests.deadletter_ref import DEAD, DeadLetterModel
from tests.lease_ref import LIVE


class SnapshotModel(DeadLetterModel):
    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.n_imports = 0

    def export(self, start_id, rec_cap):
        """(entries, sends, payload, meta, next_id) of one sdb_lease_export call."""
        from swarmdb_b200._native import ENTRY_DTYPE, META_DTYPE, SEND_DTYPE
        recs = [r for r in self.recs if r["state"] in (LIVE, DEAD) and r["id"] >= start_id][:rec_cap]
        rows = {}
        for r in recs:
            rows.setdefault(r["row"], len(rows))
        ent = np.zeros(len(recs), ENTRY_DTYPE)
        snd = np.zeros(len(rows), SEND_DTYPE)
        meta = np.zeros(len(recs), META_DTYPE)
        pays = [None] * len(rows)
        for k, r in enumerate(recs):
            j, h = rows[r["row"]], r["hdr"]
            ent[k] = (h["seq"], j, h["receiver"])
            snd[j] = (h["timestamp"], 0, h["sender"], h["group"], h["len"], h["prio"], h["type"], 0)
            pays[j] = r["pay"]
            meta[k] = (r["id"], r["deadline"], r["agent"], r["deliveries"] if self.policy else 0, r["state"], 0)
        lens = np.array([len(p) for p in pays], np.int64)
        if len(rows) > 1:
            snd["payload_off"][1:] = np.cumsum(lens)[:-1].astype(np.uint64)
        payload = np.concatenate(pays) if pays else np.zeros(0, np.uint8)
        return ent, snd, payload, meta, (recs[-1]["id"] + 1 if recs else start_id)

    def import_(self, entries, sends, payload, meta):
        """sdb_lease_import: the records behind the store's tail with ids next_id.. ; returns the first id."""
        from swarmdb_b200._native import expand_compact
        hdr, full = expand_compact(entries, sends, payload)
        base, off = self.next_id, 0
        for k in range(len(entries)):
            pl = (int(hdr[k]["len"]) + 31) & ~31
            m = meta[k]
            d = int(m["deliveries"])
            self.recs.append({"id": base + k, "agent": int(m["agent"]), "hdr": hdr[k].copy(), "pay": full[off:off + pl].copy(),
                              "deadline": float(m["deadline"]), "state": int(m["state"]),
                              "deliveries": max(d, 1) if self.policy else 1,
                              "row": ("import", self.n_imports, int(entries[k]["send"]))})
            off += pl
            if int(m["state"]) == LIVE:
                self.live += 1
        self.next_id += len(entries)
        self.n_imports += 1
        return base

    def ledger_triples(self):
        """sdb_lease_ledger_export after a collection, as a set of (agent, seq, count)."""
        if self.ledger:
            self.collect()
        return {(en["agent"], en["seq"], en["count"]) for en in self.ledger}

    def ledger_import(self, agent, seq, count):
        """sdb_lease_ledger_import: returns the triples matched."""
        if self.ledger:
            self.collect()
        ring, matched = self.o.ring, 0
        for a, s, c in zip(np.asarray(agent).tolist(), np.asarray(seq).tolist(), np.asarray(count).tolist()):
            w, h = ring.window(a), ring.head[a]
            i = next((i for i, e in enumerate(w) if e[1] and e[0] == s), None)
            if i is not None:
                self._add({"agent": a, "seq": s, "count": c, "p": h + i, "slot": w[i]})
                matched += 1
        return matched
