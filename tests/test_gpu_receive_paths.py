"""Every receive selection path at its thresholds, against the CPU oracle, bit-exact.

The code that picks the records decides which ring entries an agent gets, in which order, where each lands in the
output, and where head and ntomb (the count of consumed entries still inside the window) end up.  Each test here
drives a chosen path and asserts, from the profiler's launch counts, that this path served the call, so that a later
change of a threshold cannot quietly move a case elsewhere:

  k_recv_small        2-8 agents (or 1 with the server off), n k <= 1024, host outputs   recv_gather only
  latency server      one agent, host outputs, the server running                        no launch
  bulk, stream order  k_recv_plan + gather                                               recv_select, no recv_count
  bulk, priority      k_recv_count, scans, k_recv_select(_big), gather                   recv_count

After every call the counts, every header field and the padded payload bytes, stats()["delivered"] and agent_loads()
(pending, pending_by_prio) must equal the oracle's: an ntomb that disagrees with head shows in the loads even when the
returned records happen to be right.  Where head lands does not (pending = tail - head - ntomb is the same either way);
it decides the ring's free slots, which tests/test_gpu_ring_capacity.py checks against a bounded-ring model.

Capacity (include/swarmdb_b200.h): records are laid out agent by agent in list order; an agent whose records do not
all fit is truncated together with every later agent (they stay queued), except an agent first in the output, which
gets its first rec_cap records.  The oracle has no capacity, so the expectation is built from it: the oracle's receive
on the prefix of the list that fits, or on the lead agent alone with k = rec_cap.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

EMPTY = 8                       # agents that never receive anything: padding for the request lists
LAUNCHES = {                    # profiler launch counts of the receive kernel classes, per path
    "small": {"recv_gather": 1},
    "server": {},
    "stream": {"recv_select": 1, "recv_gather": 1},
    "priority": {"recv_count": 1, "recv_scan": 2, "recv_select": 1, "recv_gather": 1},
}


def _pad32(n):
    return (int(n) + 31) & ~31


def _payloads(rng, n, max_len):
    lens = rng.integers(0, max_len + 1, n).astype(np.uint16)
    stride = _pad32(max_len)
    off = np.arange(n, dtype=np.uint64) * stride
    buf = rng.integers(0, 256, n * stride + 64).astype(np.uint8)
    return lens, off, buf


def _same(res_gpu, res_cpu, what=""):
    cg, hg, pg = res_gpu
    cc, hc, pc = res_cpu
    assert np.array_equal(cg, cc), (what, cg[:16], cc[:16])
    assert len(hg) == len(hc), (what, len(hg), len(hc))
    for f in hg.dtype.names:
        assert np.array_equal(hg[f], hc[f]), (what, f)
    assert pg.tobytes() == pc.tobytes(), what


class Rig:
    """A Shard and the oracle in lockstep; agents 0 .. EMPTY - 1 stay empty."""

    def __init__(self, rng, A, max_len=64, G=1, **kw):
        from oracle.cpu_ref import CpuOracle
        from swarmdb_b200._native import Shard
        self.rng, self.A, self.max_len = rng, A, max_len
        self.g = Shard(max_agents=A, max_groups=G, **kw)
        self.c = CpuOracle(A, G)
        idx = np.arange(A, dtype=np.uint32)
        self.g.register(idx); self.c.register(idx)
        self.empties = idx[:EMPTY]
        self.P = _pad32(self.g.cfg.max_payload_bytes)
        mrp = int(self.g.cfg.max_recv_payload) or self.g.max_recv_records * 256
        self.dev_cap = min(self.g.max_recv_records, _pad32(mrp) // self.P)
        self.delivered = 0
        self.seqs = []                                   # seq of every record delivered (not peeked)
        self.server = False
        self.g.profile(True)

    def close(self):
        if self.server:
            self.g.latency_server(False)
        self.g.close(); self.c.close()

    def send(self, receivers, prio):
        receivers = np.asarray(receivers, np.uint32)
        n = len(receivers)
        for s0 in range(0, n, 65536):
            r = receivers[s0:s0 + 65536]
            m = len(r)
            s = self.rng.integers(0, self.A, m)
            p = np.asarray(prio[s0:s0 + 65536], np.uint8)
            typ = self.rng.integers(0, 7, m)
            lens, off, buf = _payloads(self.rng, m, self.max_len)
            assert self.g.send_batch(s, r, p, typ, lens, off, buf) == self.c.send_batch(s, r, p, typ, lens, off, buf)

    def _set_server(self, on):
        if on != self.server:
            self.g.latency_server(on)
            self.server = on

    def expect(self, agents, k, flags, cap):
        """The oracle's answer under the capacity rule."""
        from oracle.cpu_ref import HDR_DTYPE
        from swarmdb_b200._native import RECV_PEEK, RECV_PRIORITY
        n = len(agents)
        tot = max(1, min(n * k, int(self.pending(agents).sum())))          # output arrays of the oracle calls
        want = self.c.receive_batch(agents, k, (flags & RECV_PRIORITY) | RECV_PEEK, rec_cap=tot,
                                    pay_cap=tot * _pad32(self.max_len))[0]
        acc, cut, lead = 0, n, False
        for q in range(n):
            if acc + int(want[q]) > cap:
                cut, lead = q, acc == 0
                break
            acc += int(want[q])
        cnt = np.zeros(n, np.uint32)
        sub, kk = (agents[cut:cut + 1], cap) if lead else (agents[:cut], k)
        if len(sub) == 0:
            return cnt, np.zeros(0, HDR_DTYPE), np.zeros(0, np.uint8)
        cc, hc, pc = self.c.receive_batch(sub, kk, flags, rec_cap=tot, pay_cap=tot * _pad32(self.max_len))
        if lead:
            cnt[cut] = cc[0]
        else:
            cnt[:cut] = cc
        return cnt, hc, pc

    def recv(self, agents, k, flags, path, out_cap=None, what=""):
        """One receive through `path` (after checking that it is the one taken), compared with the oracle."""
        from swarmdb_b200._native import HDR_DTYPE, RECV_PEEK, RECV_PRIORITY
        agents = np.asarray(agents, np.uint32)
        n = len(agents)
        if path == "server":
            assert n == 1 and n * k <= 1024
            self._set_server(True)
        elif path == "small":
            assert n <= 8 and n * k <= 1024
            if n == 1:
                self._set_server(False)
        else:
            assert n > 8 or n * k > 1024
            assert path == ("priority" if flags & RECV_PRIORITY else "stream")
        if out_cap is None:
            out_hdr, out_pay = None, None
            cap = min(self.dev_cap, self.g.max_recv_records, len(self.g._grow_pay()) // self.P)
        else:
            out_hdr, out_pay = np.zeros(out_cap, HDR_DTYPE), np.zeros(out_cap * self.P, np.uint8)
            cap = min(self.dev_cap, out_cap)
        if path in ("small", "server"):
            cap = min(cap, 1024)
        self.g.profile_read()
        got = self.g.receive_batch(agents, k, flags, out_hdr=out_hdr, out_payload=out_pay)
        prof = {kind: c for kind, (_, c) in self.g.profile_read().items() if kind.startswith("recv_") and c}
        assert prof == LAUNCHES[path], (what, path, prof)
        want = self.expect(agents, k, flags, cap)
        _same(got, want, f"{what} path={path} n={n} k={k} flags={flags} cap={cap}")
        if not flags & RECV_PEEK:
            self.delivered += len(want[1])
            self.seqs.append(want[1]["seq"].copy())
        assert self.g.stats()["delivered"] == self.delivered, what
        self.check_loads(agents, what)
        return want

    def check_loads(self, agents=None, what=""):
        ag = np.arange(self.A, dtype=np.uint32) if agents is None else np.asarray(agents, np.uint32)
        lg, lc = self.g.agent_loads(ag), self.c.agent_loads(ag)
        assert np.array_equal(lg["pending"], lc["pending"]), (what, lg["pending"][:16], lc["pending"][:16])
        assert np.array_equal(lg["pending_by_prio"], lc["pending_by_prio"]), what

    def pending(self, agents):
        return self.c.agent_loads(np.asarray(agents, np.uint32))["pending"].astype(np.int64)

    def drain(self, k=100000):
        idx = np.arange(self.A, dtype=np.uint32)
        while len(self.recv(idx, k, 0, "stream", what="drain")[1]):       # ends: every call makes progress
            pass
        self.check_loads(None, "drained")
        st = self.g.stats()
        assert st["ring_overflow"] == 0 and st["enqueued"] == st["delivered"] == self.delivered
        seqs = np.concatenate(self.seqs) if self.seqs else np.zeros(0, np.uint64)
        assert len(np.unique(seqs)) == len(seqs) == st["enqueued"]         # nothing lost, nothing twice


# ---------------------------------------------------------------------------------------------------------------------
# a. + b.  ring window states x k x flags x path
R = 512
KS = [1, 8, 9, 31, 32, 33, 64, 65, 127, 128, 129, 255, 256, 257, R - 1, R, 2 * R]


def _bulk(rig, agents, k, flags, what):
    from swarmdb_b200._native import RECV_PRIORITY
    rig.recv(agents, k, flags, "priority" if flags & RECV_PRIORITY else "stream", what=what)


def _state(rig, name, targets):
    """Bring every target agent into the window state `name` (the same pattern of priorities for all of them)."""
    from swarmdb_b200._native import RECV_PEEK, RECV_PRIORITY
    rng, nt = rig.rng, len(targets)

    def fill(prios):                                     # one record per target per entry of prios, in arrival order
        prios = np.asarray(prios)
        rig.send(np.tile(targets, len(prios)), np.repeat(prios, nt))

    def rand(m):
        return rng.integers(0, 4, m)

    if name == "contiguous":
        fill(rand(450))
    elif name in ("holey", "after_peek"):
        fill(rand(500))
        _bulk(rig, targets, 37, RECV_PRIORITY, "prep")
        _bulk(rig, targets, 5, RECV_PRIORITY, "prep")
        if name == "after_peek":                         # peeks in both orders: nothing may change (checked by recv)
            _bulk(rig, targets, R, RECV_PRIORITY | RECV_PEEK, "prep peek")
            _bulk(rig, targets, 2 * R, RECV_PEEK, "prep peek")
            _bulk(rig, targets, 100, RECV_PRIORITY | RECV_PEEK, "prep peek")
    elif name == "full":                                 # T - H = R, head not at 0
        fill(rand(100))
        _bulk(rig, targets, 100, 0, "prep")
        fill(rand(R))
    elif name == "wrapped_odd_head":                     # window [301, 701) straddles the ring wrap
        fill(rand(301))
        _bulk(rig, targets, 301, 0, "prep")
        fill(rand(400))
    elif name == "tombstones_then_last":
        # 300 entries: 0, 3 x 298, 0.  The priority receive takes the 298, the stream receive the first entry: head
        # then jumps over the 298 tombstones to the one live entry left
        fill([0] + [3] * 298 + [0])
        _bulk(rig, targets, 298, RECV_PRIORITY, "prep")
        _bulk(rig, targets, 1, 0, "prep")
        assert (rig.pending(targets) == 1).all()
    elif name == "single_level":
        fill(np.full(400, 2))
    elif name == "ascending":
        fill(np.arange(480) * 4 // 480)
    elif name == "descending":
        fill(3 - np.arange(480) * 4 // 480)
    else:
        raise AssertionError(name)


STATES = ["contiguous", "holey", "full", "wrapped_odd_head", "tombstones_then_last", "single_level", "ascending",
          "descending", "after_peek"]


@pytest.mark.parametrize("state", STATES)
def test_window_states_k_flags_paths_match_oracle(state):
    """Each (k, flags, path) combination on a fresh agent in the window state.  Paths:
      bulk    the agent among empty ones: 9 agents for k <= 128, 8 agents (n k > 1024) above;
      small   the agent among empty ones, n = min(8, 1024 // k) >= 2 agents.  k = 2R = 1024 cannot reach it: two
              agents would ask for 2048 records, more than the single-launch path takes;
      server  the agent alone.  Its fast path serves stream-order answers of <= 32 records from a window without
              tombstones (contiguous, full, wrapped, single level, ascending, descending, k <= 32); everything
              else takes its slow path (select_agent_warp)."""
    from swarmdb_b200._native import RECV_PEEK, RECV_PRIORITY
    rng = np.random.default_rng(STATES.index(state) + 100)
    combos = [(f, k, p) for f in (0, RECV_PRIORITY, RECV_PEEK, RECV_PEEK | RECV_PRIORITY) for k in KS
              for p in ("bulk", "small", "server") if not (p == "small" and 2 * k > 1024)]
    A = EMPTY + len(combos)
    rig = Rig(rng, A, ring_slots=R, max_recv_records=1 << 17)
    try:
        targets = np.arange(EMPTY, A, dtype=np.uint32)
        _state(rig, state, targets)
        rig.check_loads(None, state)
        order = rng.permutation(len(combos))
        for i in order:
            flags, k, path = combos[i]
            a = targets[i]
            what = f"{state} agent={a}"
            if path == "server":
                rig.recv([a], k, flags, "server", what=what)
                continue
            n = (9 if k <= 128 else 8) if path == "bulk" else max(2, min(8, 1024 // k))
            agents = np.concatenate([[a], rng.choice(rig.empties, n - 1, replace=False)]).astype(np.uint32)
            rng.shuffle(agents)
            if path == "bulk":
                _bulk(rig, agents, k, flags, what)
            else:
                rig.recv(agents, k, flags, "small", what=what)
        rig.drain()
    finally:
        rig.close()


# ---------------------------------------------------------------------------------------------------------------------
# c.  warp and tile mixing in k_recv_plan
def test_plan_warps_mix_empty_simple_holey_and_truncated_agents():
    """Scrambled request lists in which a 32-agent warp holds empty agents, simple agents with <= 8 and > 8 records,
    agents with holes and C > 32 or C > 256, and (when the capacity cuts inside it) truncated agents.  List lengths
    just below and above one plan tile (256 agents) and 32 tiles (8192, one look-back super-tile)."""
    from swarmdb_b200._native import RECV_PRIORITY
    rng = np.random.default_rng(7)
    A = 8400
    cap = 300_000
    rig = Rig(rng, A, max_len=32, ring_slots=1024, max_recv_records=cap, arena_bytes=1 << 28)
    try:
        agents = np.arange(EMPTY, A, dtype=np.uint32)
        kind = rng.choice(5, len(agents), p=[0.2, 0.25, 0.25, 0.18, 0.12])
        per = np.select([kind == 1, kind == 2, kind == 3, kind == 4],
                        [rng.integers(1, 9, len(agents)), rng.integers(9, 151, len(agents)),
                         np.full(len(agents), 120), np.full(len(agents), 700)], 0)
        recv = np.repeat(agents, per)
        rng.shuffle(recv)                                 # arrival order interleaved over agents
        rig.send(recv, rng.integers(0, 4, len(recv)))
        _bulk(rig, agents[kind == 3], 20, RECV_PRIORITY, "holes C > 32")
        _bulk(rig, agents[kind == 4], 40, RECV_PRIORITY, "holes C > 256")
        is_simple = np.zeros(A, bool); is_simple[agents[(kind == 1) | (kind == 2)]] = True
        is_holey = np.zeros(A, bool); is_holey[agents[kind >= 3]] = True
        for n_list in (255, 257, 8193, 8191):
            lst = rng.permutation(np.arange(A, dtype=np.uint32))[:n_list]
            pend = rig.pending(lst)
            cum = np.cumsum(pend)
            cut = int(np.searchsorted(cum, cap, side="right"))       # first agent that does not fit
            # what the list holds, per 32-slot warp of the plan kernel
            w = len(lst) // 32
            simple_recs = (np.where(is_simple[lst], pend, 0)[: w * 32]).reshape(w, 32).sum(axis=1)
            holey = (is_holey[lst] & (pend > 0))[: w * 32].reshape(w, 32).any(axis=1)
            assert simple_recs.max() > 512 and ((simple_recs > 256) & holey).any(), n_list
            assert (pend[is_holey[lst]] > 256).any() and (pend[is_holey[lst] & (pend > 32)] <= 256).any()
            if n_list > 8000:
                assert cut < n_list and pend[cut] > 0 and 0 < cut          # the capacity cuts inside the list
            rig.recv(lst, 1000, 0, "stream", what=f"list of {n_list}")
        rig.drain()
    finally:
        rig.close()


# ---------------------------------------------------------------------------------------------------------------------
# d.  capacity truncation on every path, both orders
def _cap_rig(rng, source, cap):
    """A rig whose record capacity is `cap` through `source`; returns (rig, out_cap for recv)."""
    A = EMPTY + 40
    if source == "max_recv_records":       # the caller's buffers are larger: the device capacity binds
        return Rig(rng, A, ring_slots=256, max_recv_records=cap), 4 * cap
    if source == "max_recv_payload":       # 4 KiB maximum payloads: cap of them fill the payload buffer
        return Rig(rng, A, ring_slots=256, max_payload_bytes=4096, max_recv_payload=cap * 4096), 4 * cap
    return Rig(rng, A, ring_slots=256), cap


@pytest.mark.parametrize("cap", [5, 20, 45])
@pytest.mark.parametrize("source", ["max_recv_records", "max_recv_payload", "out_buffers"])
def test_capacity_truncation_on_every_path(source, cap):
    """A single agent with more than rec_cap pending, a list whose first (or first non-empty) agent alone exceeds
    rec_cap, a list that fills rec_cap exactly, and one that overflows inside it, through the small path, the latency
    server (fast path for stream order without holes when cap <= 32, slow path otherwise) and both bulk paths, in
    stream and priority order, with and without PEEK.  Then single agents are drained one call at a time - every call
    must make progress - and the rest in bulk; every record is delivered exactly once."""
    from swarmdb_b200._native import RECV_PEEK, RECV_PRIORITY
    rng = np.random.default_rng(1000 * cap + len(source))
    rig, out_cap = _cap_rig(rng, source, cap)
    if source != "out_buffers":
        assert rig.dev_cap == cap
    try:
        agents = np.arange(EMPTY, rig.A, dtype=np.uint32)
        # more than 3 cap records each: after the two consuming passes below every agent still holds more than cap
        per = rng.integers(3 * cap + 1, 4 * cap + 1, len(agents))
        recv = np.repeat(agents, per)
        rng.shuffle(recv)
        rig.send(recv, rng.integers(0, 4, len(recv)))
        m = next(d for d in (2, 3, 4, 5) if cap % d == 0)   # m agents of cap / m records fill the output exactly
        for flags in (RECV_PEEK, RECV_PEEK | RECV_PRIORITY, 0, RECV_PRIORITY):
            bulk = "priority" if flags & RECV_PRIORITY else "stream"
            a = rng.permutation(agents).astype(np.uint32)
            assert (rig.pending(a) > cap).all()
            e = rng.permutation(rig.empties).astype(np.uint32)
            what = f"{source} cap={cap}"
            # one agent, k > cap
            rig.recv(a[0:1], 100, flags, "server", out_cap, what + " one agent")
            rig.recv(a[1:2], 100, flags, "small", out_cap, what + " one agent")
            rig.recv(a[2:3], 1500, flags, bulk, out_cap, what + " one agent")
            # the first agent alone exceeds the capacity, alone or after empty agents
            rig.recv(a[3:6], 100, flags, "small", out_cap, what + " first too big")
            rig.recv(np.concatenate([e[:2], a[6:8]]), 100, flags, "small", out_cap, what + " lead after empties")
            rig.recv(np.concatenate([e[:3], a[8:10], e[3:]]), 100, flags, bulk, out_cap, what + " lead after empties")
            # m agents fill the output exactly, the next one is truncated
            rig.recv(a[10:11 + m], cap // m, flags, "small", out_cap, what + " exact fill")
            rig.recv(np.concatenate([a[16:17 + m], e]), cap // m, flags, bulk, out_cap, what + " exact fill")
            # the second agent overflows: only the first is delivered
            k2 = cap // 2 + 1
            rig.recv(a[22:24], k2, flags, "small", out_cap, what + " second overflows")
            rig.recv(np.concatenate([a[24:26], e]), k2, flags, bulk, out_cap, what + " second overflows")
        # a caller looping "until empty" on one agent finishes, on every path
        for path in ("server", "small", "stream", "priority"):
            a = agents[np.argmax(rig.pending(agents))]
            left = int(rig.pending([a])[0])
            assert left > cap
            flags = RECV_PRIORITY if path == "priority" else 0
            k = 1500 if path in ("stream", "priority") else 1000
            for _ in range(left // cap + 1):
                rig.recv([a], k, flags, path, out_cap, f"{source} cap={cap} drain one agent via {path}")
            assert rig.pending([a])[0] == 0, path
        rig.drain()
    finally:
        rig.close()
