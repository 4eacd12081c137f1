"""Reference for retention (sdb_expire) on top of the CPU oracle (TESTS ONLY).

The contract of sdb_expire is that every later receive delivers what it would have delivered had the expired records
never been enqueued.  `ExpiringOracle` restates it literally: it reads the wrapped CpuOracle's pending records (a PEEK
receive), removes the expired ones in a pure-Python model of the selection and capacity rule (include/swarmdb_b200.h),
and then REPLAYS the survivors, one record at a time with their original sequence numbers and header fields, into a
fresh CpuOracle.  Every receive after that is the unmodified oracle's receive over a queue in which the expired
records were never sent.  Digests are not carried across an expiry: enable them afterwards.
"""
from __future__ import annotations

import numpy as np

from oracle.cpu_ref import HDR_DTYPE, CpuOracle

NO_GROUP = 0xFFFFFFFF
NO_RECEIVER = 0xFFFFFFFF
RECV_PEEK = 2
EXPIRE_ALL = 16


def _pad32(n):
    return (n + 31) & ~31


def expire_select(state, agents, older_than, flags, rec_cap):
    """The selection of sdb_expire on a model queue {agent: [(header record, padded payload bytes), ...]} in stream
    order: per listed agent every record with timestamp < older_than (all with EXPIRE_ALL), agents laid out in list
    order; an agent whose matches do not all fit stays whole with every later agent, except the first agent in the
    output, which gives its first rec_cap.  Returns (counts, [(agent, position in its list)]) of the chosen records."""
    counts, chosen, total, cut = [], [], 0, False
    for a in agents:
        recs = state.get(int(a), [])
        match = [i for i, (h, _) in enumerate(recs) if flags & EXPIRE_ALL or h["timestamp"] < older_than]
        take = 0 if cut else len(match)
        if not cut and match and total + len(match) > rec_cap:
            take, cut = (rec_cap if total == 0 else 0), True
        counts.append(take)
        chosen += [(int(a), i) for i in match[:take]]
        total += take
    return counts, chosen


class ExpiringOracle:
    """A CpuOracle (the `inner` one, replaced at every retiring expiry) plus `expire`; every other call is the
    oracle's.  `received` in agent_loads keeps counting the expired records, as sdb_agent_loads does."""

    def __init__(self, inner: CpuOracle, max_groups: int, groups=None, watermark: int = 0):
        self.inner = inner
        self.max_agents = inner.max_agents
        self.max_groups = max_groups
        self._groups = {}                   # g -> (members, positions or None): restored after a replay
        for g, m in (groups or {}).items():
            self._groups[g] = (np.asarray(m, np.uint32), None)
        self._recv_extra = np.zeros(self.max_agents, np.int64)
        self._wm = watermark                # registered-index watermark (agents=None lists every agent below it)
        self._backends = None

    # ---- bookkeeping of what a replay has to restore
    def _see(self, *idx):
        for x in idx:
            x = np.asarray(x).ravel()
            if len(x):
                self._wm = max(self._wm, int(x.max()) + 1)

    def register(self, idx):
        self._see(idx); self.inner.register(idx)

    def create_group(self, g, members):
        self._groups[g] = (np.asarray(members, np.uint32), None); self._see(members); self.inner.create_group(g, members)

    def create_group_pos(self, g, members, pos):
        self._groups[g] = (np.asarray(members, np.uint32), np.asarray(pos, np.uint32)); self._see(members)
        self.inner.create_group_pos(g, members, pos)

    def set_backends(self, weight, load0=None):
        self._backends = np.asarray(weight, np.uint32); self.inner.set_backends(weight, load0)

    def send_batch(self, sender, receiver, *a, **k):
        self._see(sender, receiver); return self.inner.send_batch(sender, receiver, *a, **k)

    def send_list_batch(self, sender, list_off, list_idx, *a, **k):
        self._see(sender, list_idx); return self.inner.send_list_batch(sender, list_off, list_idx, *a, **k)

    @property
    def next_seq(self):
        return self.inner.next_seq

    @next_seq.setter
    def next_seq(self, v):
        self.inner.next_seq = v

    def __getattr__(self, name):            # everything else: the current oracle
        return getattr(self.inner, name)

    def agent_loads(self, agents=None, n=None):
        out = self.inner.agent_loads(agents, n)
        idx = np.arange(len(out)) if agents is None else np.asarray(agents, np.int64)
        out["received"] = (out["received"].astype(np.int64) + self._recv_extra[idx]).astype(np.uint32)
        return out

    def queue_stats(self, n=None):
        return CpuOracle.queue_stats(self, n)

    # ---- the model queue and the replay
    def snapshot(self):
        """{agent: [(header record, padded payload bytes), ...]} of every pending record, stream order; consumes nothing."""
        ld = self.inner.agent_loads(None, self.max_agents)
        n_rec = int(ld["pending"].astype(np.int64).sum())
        n_pay = int(ld["pending_granules"].astype(np.int64).sum()) * 32
        cnt, hdr, pay = self.inner.receive_batch(np.arange(self.max_agents), 1 << 31, RECV_PEEK, rec_cap=max(n_rec, 1),
                                                 pay_cap=max(n_pay, 32))
        state, r, off = {}, 0, 0
        for a in np.nonzero(cnt)[0]:
            lst = []
            for k in range(int(cnt[a])):
                h = hdr[r + k]
                pl = _pad32(int(h["len"]))
                lst.append((h, pay[off:off + pl].tobytes()))
                off += pl
            r += int(cnt[a])
            state[int(a)] = lst
        return state

    def _replay(self, state):
        old = self.inner
        new = CpuOracle(self.max_agents, self.max_groups)
        if self._wm:
            new.register([self._wm - 1])
        zero = np.zeros(1, np.uint64)
        for a in sorted(state):
            for h, p in state[a]:
                buf = np.frombuffer(p + bytes(32), np.uint8)
                s, pr, ty, ln, ts = [int(h["sender"])], [int(h["prio"])], [int(h["type"])], [int(h["len"])], [float(h["timestamp"])]
                seq = int(h["seq"])
                if int(h["receiver"]) == NO_RECEIVER:
                    new.next_seq = seq
                    new.send_list_batch(s, [0, 1], [a], pr, ty, ln, zero, buf, ts)
                elif int(h["group"]) == NO_GROUP:
                    new.next_seq = seq
                    new.send_batch(s, [a], pr, ty, ln, zero, buf, ts)
                else:
                    g = int(h["group"])
                    new.create_group_pos(g, [a], [0])
                    new.send_group_seq(s, [g], pr, ty, ln, zero, buf, [seq], ts)
        for g, (m, pos) in self._groups.items():      # identity positions: what create_group means for every send path
            new.create_group_pos(g, m, np.arange(len(m), dtype=np.uint32) if pos is None else pos)
        if self._backends is not None:
            new.set_backends(self._backends, old.backend_loads())
        new.next_seq = old.next_seq
        self._recv_extra += (old.agent_loads(None, self.max_agents)["received"].astype(np.int64)
                             - new.agent_loads(None, self.max_agents)["received"].astype(np.int64))
        self.inner = new
        old.close()

    def expire(self, agents, older_than: float, flags: int = 0, rec_cap: int = (1 << 64) - 1, materialise: bool = True):
        """sdb_expire's result: (counts, headers, padded payloads) in the full receive format (the device's compact
        output expands to it), or (counts, total) with materialise=False; PEEK retires nothing."""
        state = self.snapshot()
        listed = np.arange(self._wm) if agents is None else np.asarray(agents, np.int64)
        counts, chosen = expire_select(state, listed, older_than, flags, rec_cap)
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
