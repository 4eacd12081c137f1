"""Ring capacity on the enqueue paths that keep their own drop decision, against the bounded-ring model (tests/ring_ref.py).

The rule is one: a ring takes ring_slots - (tail - head) more records, tombstones included.  Each path below applies it
in its own code, so each is compared with the model on rings made holey and nearly full first (a random-priority fill
to within 0-3 slots of full, a priority receive that punches tombstones, a stream take of the oldest record on half the
agents), with windows that cross the ring's physical wrap:

  k_pull_index            agents in several groups (serial merge by (send, member position)) and agents with one
                          membership in a non-exclusive group (quad path), beside k_pull_index_group in one batch
  pull + atomic claims    a mixed batch with group sends above the pull threshold: the index build leaves ctail to the
                          commit sort, which then orders both kinds of entry
  commit sort             commit_agent's clamp, then the register network (<= 16 new records for an agent), the
                          shared-memory bitonic sort (<= 4096) and the in-ring odd-even sort beyond that
  cross-shard imports     sync (import_wire_batches, import_wire_ptrs with composite seqs) and asynchronous imports of
                          exclusive-group, shared-group and mixed traffic, each shard against its own model
  SwarmsDB.flush          the overflow report: FAILED marks, undelivered_to, unread counts, resends

After each send: the ring_overflow delta, the overflow log, the survivors byte for byte (a PEEK receive) and
agent_loads must equal the model's, and the launch counts say which kernels served the call.
"""
import numpy as np
import pytest

from tests.ring_ref import BoundedOracle
from tests.test_gpu_receive_paths import EMPTY, Rig, _payloads, _same
from tests.test_gpu_ring_capacity import _bounded_send, _drain, _probe

pytestmark = pytest.mark.gpu


@pytest.fixture(params=["1", "0"])
def shared(request, monkeypatch):
    monkeypatch.setenv("SDB_SHARED_PAYLOAD", request.param)
    return request.param == "1"


def _grig(seed, A, G, ring_slots, **kw):
    """_rig of tests/test_gpu_ring_capacity.py with G groups."""
    rig = Rig(np.random.default_rng(seed), A, G=G, ring_slots=ring_slots, **kw)
    rig.c = BoundedOracle(rig.c, G, ring_slots, None, A)
    return rig


def _path(n, k, flags=0):
    from swarmdb_b200._native import RECV_PRIORITY
    if n <= 8 and n * k <= 1024:
        return "small"
    return "priority" if flags & RECV_PRIORITY else "stream"


def _holey(rig, targets, fill_to):
    """Fill each target's ring with random priorities up to `fill_to` free slots (per target), punch tombstones with a
    priority receive, then take the oldest record of half the targets.  Returns whether some window crosses the ring's
    physical wrap."""
    from swarmdb_b200._native import RECV_PRIORITY
    rng, R_ = rig.rng, rig.c.ring.R
    fill = np.array([rig.c.capacity(a) for a in targets.tolist()]) - np.asarray(fill_to)
    fill = np.maximum(fill, 0)
    rig.send(rng.permutation(np.repeat(targets, fill)).astype(np.uint32), rng.integers(0, 4, int(fill.sum())))
    assert rig.c.take_dropped() == []
    k = max(1, R_ // 4)
    rig.recv(targets, k, RECV_PRIORITY, _path(len(targets), k, RECV_PRIORITY), what="holes")
    half = rng.permutation(targets)[: max(1, len(targets) // 2)]
    rig.recv(half, 1, 0, _path(len(half), 1), what="oldest")
    return any(rig.c.ring.head[a] % R_ + rig.c.ring.span(a) > R_ for a in targets.tolist())


# ---------------------------------------------------------------------------------------------------------------------
# A. agent-parallel index build
@pytest.mark.parametrize("ring_slots", [4, 8, 64])
def test_agent_parallel_index_build_at_capacity(shared, ring_slots):
    """Groups where agents sit in two or three groups, one group lists an agent twice, a non-exclusive group whose other
    members have one membership (quad path) and an exclusive group (k_pull_index_group): a group batch above the pull
    threshold keeps exactly the model's first records (send order, then member position); a mixed batch with the same
    group traffic plus p2p and list sends to the same agents (pull plus atomic claims, one commit sort) keeps exactly as
    many records as each ring has free slots, in seq order."""
    from tests.test_gpu_shared_layout import THRESHOLD
    Rr, G = ring_slots, 8
    n_x, n_q, n_m = 64, 64, 48
    A = EMPTY + n_x + n_q + n_m
    rig = _grig(100 + Rr, A, G, Rr, list_pool_entries=1 << 16)
    try:
        rng = rig.rng
        ag = np.arange(EMPTY, A, dtype=np.uint32)
        X, Q, M = ag[:n_x], ag[n_x:n_x + n_q], ag[n_x + n_q:]
        groups = [X,                                              # exclusive: k_pull_index_group
                  np.r_[Q, M[:1]],                                # non-exclusive: Q have one membership (quad path)
                  M[:32], M[16:48], np.r_[M[8:24], M[40:48]],     # M[16:24] in three groups, most of M in two
                  np.r_[M[0:6], M[3:4], M[30:34]]]                # M[3] listed twice
        for k, m in enumerate(groups):
            rig.g.create_group(k, m)
            rig.c.create_group(k, m)
        sizes = np.array([len(m) for m in groups])

        def group_sends(n):
            grp = rng.integers(0, len(groups), n).astype(np.uint32)
            # half the senders are members of the group they send to: their own record is skipped (M:1268)
            snd = np.array([rng.choice(groups[g]) if rng.random() < 0.5 else rng.integers(0, EMPTY) for g in grp.tolist()])
            assert sizes[grp].sum() >= THRESHOLD
            return snd.astype(np.uint32), grp

        crossed = False
        for rnd in range(2):
            crossed |= _holey(rig, ag, rng.integers(0, 4, len(ag)))
            s, grp = group_sends(480)
            p, t = rng.integers(0, 4, len(s)), rng.integers(0, 7, len(s))
            lens, off, buf = _payloads(rng, len(s), rig.max_len)
            _bounded_send(rig, ag, lambda: rig.g.send_group_batch(s, grp, p, t, lens, off, buf),
                          lambda: rig.c.send_group_batch(s, grp, p, t, lens, off, buf), True, True,
                          f"R={Rr} round {rnd}: group batch, both index kernels", launches=3, commit=False)

            # mixed: the group sends first, then p2p sends, then lists (the oracle takes the three blocks in order)
            crossed |= _holey(rig, ag, rng.integers(0, 4, len(ag)))
            n_g, n_p, n_l = 480, 600, 30
            sg, gg = group_sends(n_g)
            lists = [rng.choice(ag, 40, replace=False) for _ in range(n_l)]
            lo = np.zeros(n_l + 1, np.uint64); lo[1:] = np.cumsum([len(x) for x in lists])
            li = np.concatenate(lists).astype(np.uint32)
            n = n_g + n_p + n_l
            s = np.r_[sg, rng.integers(0, A, n_p + n_l)].astype(np.uint32)
            p, t = rng.integers(0, 4, n), rng.integers(0, 7, n)
            lens, off, buf = _payloads(rng, n, rig.max_len)
            kind = np.r_[np.ones(n_g, np.uint8), np.zeros(n_p, np.uint8), np.full(n_l, 2, np.uint8)]
            target = np.r_[gg, rng.choice(ag, n_p), np.arange(n_l)].astype(np.uint32)
            ge, pe, le = slice(0, n_g), slice(n_g, n_g + n_p), slice(n_g + n_p, n)

            def orc_mixed():
                rig.c.send_group_batch(s[ge], target[ge], p[ge], t[ge], lens[ge], off[ge], buf)
                rig.c.send_batch(s[pe], target[pe], p[pe], t[pe], lens[pe], off[pe], buf)
                rig.c.send_list_batch(s[le], lo, li, p[le], t[le], lens[le], off[le], buf)

            _bounded_send(rig, ag, lambda: rig.g.send_mixed_batch(s, kind, target, lo, li, p, t, lens, off, buf),
                          orc_mixed, False, True, f"R={Rr} round {rnd}: mixed batch, pull and atomic claims",
                          launches=5, commit=True)
        assert crossed
        _probe(rig, ag[:: len(ag) * Rr // 4096 + 1], f"R={Rr} after the index builds")     # an exact log: <= 4096 drops
        _drain(rig)
    finally:
        rig.close()


# ---------------------------------------------------------------------------------------------------------------------
# B. the commit sort above 16 records per agent
# (new records for the hot agent, ring slots, free slots before the batch, batch kind, at the 2^32 handle wrap).  A batch
# never straddles the arena's wrap (arena_reserve moves it to the next multiple of the arena size, which divides 2^32),
# so in the wrap32 cases the batch starts exactly at 2^32: batch_base32 is 0 and every sorted key equals its raw handle.
# They check only that such a batch lands correctly behind older pending records whose handles sit just below 2^32;
# the subtraction handle - batch_base32 itself cannot be told apart from a raw comparison by any reachable batch
SORT_CASES = [
    (16, 64, 16, "group", True),          # register network, fits exactly
    (16, 64, 15, "lists", False),         # register network, one over
    (17, 64, 17, "mixed", False),         # shared-memory sort, fits exactly
    (17, 64, 16, "group", False),         # 17 claimed, 16 kept: the clamp brings it back to the register network
    (4096, 8192, 4096, "group", True),    # shared memory, fits exactly
    (4096, 8192, 4095, "mixed", False),
    (4097, 8192, 4097, "lists", False),   # in-ring sort, fits exactly
    (4097, 8192, 4096, "group", False),   # clamped to the shared-memory sort
    (5000, 8192, 5000, "group", True),    # in-ring sort
    (5000, 8192, 4999, "lists", False),
    (5000, 8192, 2000, "mixed", False),   # thousands over: shared-memory sort of the 2000 kept
    (7000, 8192, 4500, "group", False),   # thousands over, in-ring sort of head + R - ctail = 4500 entries
]


@pytest.mark.parametrize("n_new,ring_slots,free,kind,wrap32", SORT_CASES,
                         ids=[f"{c[0]}-R{c[1]}-free{c[2]}-{c[3]}{'-wrap32' if c[4] else ''}" for c in SORT_CASES])
def test_commit_sort_at_capacity(shared, n_new, ring_slots, free, kind, wrap32):
    """One hot agent gets n_new records from an atomic-claim batch (a two-member group sent n_new times below the pull
    threshold, overlapping lists, or p2p sends plus lists) into a ring that holds older pending records before ctail,
    tombstones, and a window across the wrap, with exactly `free` slots left: the older records stay first and
    unchanged, exactly min(n_new, free) new ones survive in seq order, and survivors plus the log are the batch."""
    from tests.test_gpu_shared_layout import THRESHOLD
    Rr = ring_slots
    A = EMPTY + 4
    rig = _grig(n_new + free, A, 2, Rr, list_pool_entries=1 << 16)
    try:
        rng = rig.rng
        hot, o1, o2, filler = (EMPTY + i for i in range(4))
        targets = np.array([hot, o1, o2], np.uint32)
        # the window starts three quarters into the ring, so a window of more than R / 4 slots crosses the wrap
        w = Rr - Rr // 4
        rig.send(np.repeat(targets, w), np.zeros(w * 3))
        rig.recv(targets, w, 0, _path(3, w), what="wrap")
        if wrap32:                                       # nothing pending: the arena may move close to 2^32 granules
            rig.g.debug_set_arena_pos((1 << 32) - 16 * (Rr + n_new))
        # holey: older pending records, tombstones, the oldest taken on the hot agent; then a ranked top-up to `free`
        _holey(rig, targets, [free + 4, Rr // 2, Rr // 2])
        top = rig.c.capacity(hot) - free
        assert top >= 0
        rig.send(np.full(top, hot, np.uint32), rng.integers(0, 4, top))
        assert rig.c.capacity(hot) == free and rig.c.ring.ntomb(hot) > 0 and rig.c.take_dropped() == []
        assert rig.c.ring.head[hot] % Rr + rig.c.ring.span(hot) > Rr, "the hot agent's window crosses the ring's wrap"
        if wrap32:
            # records through a bystander until the batch's records (2 n_new of them, at least a granule each) no
            # longer fit below 2^32 granules: the batch starts at the wrap of the 32-bit ring handles
            def gap():
                return (1 << 32) - rig.g.stats()["arena_tail_bytes"] // 32
            assert gap() > n_new
            while gap() > n_new:
                m = int(min(Rr, max(1, (gap() - n_new) // 8)))     # a record takes at most 8 granules here
                rig.send(np.full(m, filler, np.uint32), np.zeros(m))
                rig.recv([filler], m, 0, _path(1, m), what="filler")
            assert gap() > 0

        def block(n):
            lens, off, buf = _payloads(rng, n, rig.max_len)
            return rng.integers(0, EMPTY, n).astype(np.uint32), rng.integers(0, 4, n), rng.integers(0, 7, n), lens, off, buf

        if kind == "group":
            rig.g.create_group(0, [hot, o1]); rig.c.create_group(0, [hot, o1])
            s, p, t, lens, off, buf = block(n_new)
            s[::7] = o1                                  # o1's own sends skip o1, never the hot agent
            grp = np.zeros(n_new, np.uint32)
            assert 2 * n_new < THRESHOLD
            dev = lambda: rig.g.send_group_batch(s, grp, p, t, lens, off, buf)
            orc = lambda: rig.c.send_group_batch(s, grp, p, t, lens, off, buf)
        else:
            n_l = n_new if kind == "lists" else n_new // 3
            n_p = n_new - n_l
            lists = [[hot, (o1, o2)[i % 2]] if i % 3 else [o2, hot] for i in range(n_l)]      # overlapping lists
            lo = np.zeros(n_l + 1, np.uint64); lo[1:] = np.cumsum([len(x) for x in lists])
            li = np.concatenate(lists).astype(np.uint32)
            s, p, t, lens, off, buf = block(n_p + n_l)
            if kind == "lists":
                dev = lambda: rig.g.send_list_batch(s, lo, li, p, t, lens, off, buf)
                orc = lambda: rig.c.send_list_batch(s, lo, li, p, t, lens, off, buf)
            else:
                k_ = np.r_[np.zeros(n_p, np.uint8), np.full(n_l, 2, np.uint8)]
                target = np.r_[np.full(n_p, hot), np.arange(n_l)].astype(np.uint32)
                pe, le = slice(0, n_p), slice(n_p, n_p + n_l)
                dev = lambda: rig.g.send_mixed_batch(s, k_, target, lo, li, p, t, lens, off, buf)

                def orc():
                    rig.c.send_batch(s[pe], target[pe], p[pe], t[pe], lens[pe], off[pe], buf)
                    rig.c.send_list_batch(s[le], lo, li, p[le], t[le], lens[le], off[le], buf)
        old = list(rig.c.ring.window(hot))
        lost = _bounded_send(rig, targets, dev, orc, False, False, f"{n_new} into {free} free ({kind})",
                             launches=3, commit=True, lossy=None)
        assert lost >= max(0, n_new - free)
        win = rig.c.ring.window(hot)
        assert win[: len(old)] == old and len(win) == Rr             # the older slots are unchanged and come first
        if wrap32:
            assert rig.g.stats()["arena_tail_bytes"] > (1 << 32) * 32
        rig.check_loads(None, "after the batch")
        _drain(rig)
    finally:
        rig.close()


# ---------------------------------------------------------------------------------------------------------------------
# E. a snapshot that does not fit is refused before anything is restored
def test_snapshot_larger_than_the_rings_is_refused_whole(shared, tmp_path):
    """Saved from 64-slot rings, loaded into 16-slot rings with the over-full agent in the last of several chunks: the
    load raises the full-ring error before any chunk is restored, the instance stays fresh, and an instance with
    64-slot rings loads the same file."""
    import swarmdb_b200 as sdb
    from swarmdb_b200._native import SdbError
    # a receive call holds 32 records: the nine small agents (27 records) make one chunk, the big one the next
    cfg = dict(max_agents=64, ring_slots=64, arena_bytes=1 << 22, max_groups=4, id_nonce=0x99, max_recv_records=32)
    db = sdb.SwarmsDB(save_dir=tmp_path, auto_save=False, gpu_config=sdb.GpuConfig(**cfg))
    names = [f"agent_{i}" for i in range(10)]
    db.register_agents(names)
    for i in range(9):
        for k in range(3):
            db.send_message(names[9], f"m{i}.{k}", names[i])
    for k in range(20):                                   # the last agent: 20 records, more than 16 slots
        db.send_message(names[0], f"big{k}", names[9])
    db.flush()
    want = {a: [m.content for m in db.peek_messages(a, 100)] for a in names}
    path = db.save_queue_snapshot(tmp_path / "q.npz")
    db.close()
    with np.load(path) as z:
        chunks = len(z["chunk_off"]) - 1
        assert chunks > 1 and int(z["agents"][-1]) == 9 and int(z["counts"][-1]) == 20
    small = sdb.SwarmsDB(save_dir=tmp_path, auto_save=False, gpu_config=sdb.GpuConfig(**{**cfg, "ring_slots": 16}))
    with pytest.raises(SdbError) as ei:
        small.load_queue_snapshot(path)
    assert ei.value.code == -4
    st = small.shard.stats()
    assert st["enqueued"] == 0 and st["next_seq"] == 1
    small._check_fresh()
    small.close()
    db2 = sdb.SwarmsDB(save_dir=tmp_path, auto_save=False, gpu_config=sdb.GpuConfig(**cfg))
    db2.load_queue_snapshot(path)
    assert {a: [m.content for m in db2.receive_messages(a, 100)] for a in names} == want
    db2.close()


# ---------------------------------------------------------------------------------------------------------------------
# C. cross-shard imports into holey rings (two shards on one GPU, one handle each)
class _Cluster:
    """Two shards of `world` = 2 and, per shard, an OracleShard replaying the same wire batches into a BoundedOracle.
    how: "batches" (import_wire_batches), "ptrs" (import_wire_ptrs, composite sequence bases) or "async"
    (import_wire_ptrs_async between the ready / done flags)."""

    def __init__(self, how, groups, A, G, R, S=4096):
        import torch
        from swarmdb_b200._native import Shard
        from swarmdb_b200.sharded import shard_map_numbered
        from tests.fake_shard import OracleShard
        self.how, self.A, self.R, self.k = how, A, R, 0
        self.smap = shard_map_numbered("agent_", 7, A, 2)
        cap_pay = S * 128 + 64 + 4 * 4096
        self.g, self.m = [], []
        for r in range(2):
            s = Shard(max_agents=A, max_groups=G, ring_slots=R, arena_bytes=1 << 26, max_batch_sends=S,
                      max_batch_payload=cap_pay, shard_id=r, num_shards=2, max_recv_records=1 << 18,
                      max_payload_bytes=128, list_pool_entries=1 << 16)
            s.set_agent_shards(self.smap)
            m = OracleShard(A, G, r, 2)
            m.o = BoundedOracle(m.o, G, R, None, A)
            m.o.register(np.arange(A, dtype=np.uint32))
            m.set_agent_shards(self.smap)
            for g, mem in enumerate(groups):
                s.create_group(g, mem); m.create_group(g, mem)
            s.profile(True)
            self.g.append(s); self.m.append(m)
        self.local = [np.nonzero(self.smap == r)[0].astype(np.uint32) for r in range(2)]
        self.wb = self.g[0].wire_bytes(S, cap_pay)
        if how == "async":
            self.bufs = [[self.g[r].wire_alloc(self.wb)[0] for r in range(2)] for _ in range(2)]
        else:
            self.wire = torch.zeros(2 * self.wb, dtype=torch.uint8, device="cuda")
        self.rb = self.m[0].wire_bytes(S, cap_pay)
        self.ref = np.zeros(2 * self.rb, np.uint8)

    def close(self):
        for s in self.g + self.m:
            s.close()

    def owner_capacity(self, a):
        return self.m[int(self.smap[a])].o.capacity(a)

    def import_(self, batches, keep_mode, what, index=None, commit=None):
        """batches[r] = export_mixed_batch columns of rank r.  keep_mode: the device's survivors bound the model
        (atomic claims); otherwise the call is order-deterministic.  Returns the records dropped on each shard."""
        from swarmdb_b200._native import RECV_PEEK
        from swarmdb_b200.sharded import composite_seq
        self.k += 1
        step, par = self.k, self.k & 1
        bases = [composite_seq(step, r) if self.how == "ptrs" else 0 for r in range(2)]
        for s in self.g:
            assert s.overflow_log()[2] == 0
            s.profile_read()
        st0 = [s.stats() for s in self.g]
        for r, b in enumerate(batches):
            if self.how == "async":
                if step > 2:
                    self.g[r].wire_wait_done(self.bufs[par], self.wb, step - 2)
                self.g[r].export_mixed_batch(*b, self.bufs[par][r], self.wb)
                self.g[r].wire_publish(self.bufs[par][r], self.wb, step)
            else:
                self.g[r].export_mixed_batch(*b, self.wire.data_ptr() + r * self.wb, self.wb, None, bases[r])
            self.g[r].sync()
            self.m[0].export_mixed_batch(*b, self.ref[r * self.rb:(r + 1) * self.rb], self.rb, None, bases[r])
        for s in self.g:
            if self.how == "async":
                s.import_wire_ptrs_async(self.bufs[par], self.wb, step)
            elif self.how == "ptrs":
                s.import_wire_ptrs([self.wire.data_ptr() + r * self.wb for r in range(2)])
            else:
                s.import_wire_batches(2, self.wire.data_ptr(), self.wb)
        lost = []
        for r, (s, m) in enumerate(zip(self.g, self.m)):
            s.sync()
            prof = s.profile_read()
            if index is not None:
                assert (prof["index"][1] > 0) == index, (what, r)
            if commit is not None:
                assert (prof["commit"][1] > 0) == commit, (what, r)
            loc = self.local[r]
            m.o.take_dropped()
            keep = None
            if keep_mode:
                old = {int(a): set(m.o.ring.live_seqs(a)) for a in loc.tolist()}
                cnt, hdr, _ = s.receive_batch(loc, 4 * self.R, RECV_PEEK)
                keep = {a: [] for a in old}
                for a, sq in zip(np.repeat(loc, cnt.astype(np.int64)).tolist(), hdr["seq"].tolist()):
                    if int(sq) not in old[a]:
                        keep[a].append(int(sq))
                for a, ss in keep.items():
                    assert ss == sorted(ss), (what, r, a, ss)
            with m.o.appending(keep=keep, ordered=True):
                m.import_wire_batches(2, self.ref, self.rb)
            want = m.o.take_dropped()
            st1 = s.stats()
            assert st1["ring_overflow"] - st0[r]["ring_overflow"] == len(want), (what, r, st1["ring_overflow"] - st0[r]["ring_overflow"], len(want))
            assert st1["next_seq"] == m.o.next_seq, (what, r)
            ag, sq, dropped = s.overflow_log(1 << 16)
            assert dropped == len(want) <= 4096, (what, r)
            assert sorted(zip(ag.tolist(), sq.tolist())) == sorted(want), (what, r)
            if self.how == "ptrs" and want:
                assert min(sq.tolist()) >= composite_seq(step, 0), (what, r)        # the log names composite seqs
            lg, lc = s.agent_loads(loc), m.o.agent_loads(loc)
            assert np.array_equal(lg["pending"], lc["pending"]) and np.array_equal(lg["pending_by_prio"], lc["pending_by_prio"]), (what, r)
            _same(s.receive_batch(loc, 4 * self.R, RECV_PEEK), m.o.receive_batch(loc, 4 * self.R, RECV_PEEK, rec_cap=1 << 18),
                  f"{what} survivors on shard {r}")
            lost.append(len(want))
        return lost

    def recv(self, r, agents, k, flags, what):
        agents = np.asarray(agents, np.uint32)
        _same(self.g[r].receive_batch(agents, k, flags), self.m[r].o.receive_batch(agents, k, flags, rec_cap=1 << 18), what)

    def holey(self, rng):
        """Every ring within 0-3 slots of full (p2p traffic exported by rank 0), tombstones from a priority receive, the
        oldest record taken on half the agents.  Returns whether some window crosses the ring's physical wrap."""
        from swarmdb_b200._native import RECV_PRIORITY
        ag = np.arange(EMPTY, self.A)
        fill = np.array([self.owner_capacity(a) for a in ag.tolist()]) - rng.integers(0, 4, len(ag))
        recv = rng.permutation(np.repeat(ag, np.maximum(fill, 0))).astype(np.uint32)
        self.import_([_mixed_cols(rng, np.zeros(len(recv), np.uint8), recv), _mixed_cols(rng, [], [])], False, "fill")
        crossed = False
        for r in range(2):
            loc = self.local[r][self.local[r] >= EMPTY]
            self.recv(r, loc, max(1, self.R // 4), RECV_PRIORITY, "holes")
            self.recv(r, rng.permutation(loc)[: len(loc) // 2], 1, 0, "oldest")
            ring = self.m[r].o.ring
            crossed |= any(ring.head[a] % self.R + ring.span(a) > self.R for a in loc.tolist())
        return crossed


def _mixed_cols(rng, kind, target, lists=()):
    kind, target = np.asarray(kind, np.uint8), np.asarray(target, np.uint32)
    n = len(kind)
    lo = np.zeros(len(lists) + 1, np.uint64); lo[1:] = np.cumsum([len(x) for x in lists])
    li = np.concatenate(lists).astype(np.uint32) if lists else np.zeros(0, np.uint32)
    lens = rng.integers(0, 129, n).astype(np.uint16)
    buf = rng.integers(48, 123, max(n, 1) * 128 + 64).astype(np.uint8)
    return (rng.integers(0, EMPTY, n).astype(np.uint32), kind, target, lo, li, rng.integers(0, 4, n), rng.integers(0, 7, n),
            lens, np.arange(n, dtype=np.uint64) * 128, buf)


@pytest.mark.parametrize("traffic", ["exclusive groups", "shared groups", "mixed"])
@pytest.mark.parametrize("how", ["batches", "ptrs", "async"])
def test_cross_shard_import_at_capacity(shared, how, traffic):
    """world = 2 on one GPU.  Group-only imports are order-deterministic (k_pull_index_group with sources for exclusive
    groups, k_pull_index for shared ones); mixed p2p / list / group imports claim fan-out slots atomically and the
    commit sort orders them (driven by the device-side batch record in the asynchronous import).  Shared groups make
    the asynchronous import fall back to the synchronous body between the same flags.  Each shard is checked on its
    own against the model: overflow count, exact log, survivors, loads."""
    A, G, R = 264, 8, 8
    rng = np.random.default_rng(700 + 10 * ["batches", "ptrs", "async"].index(how) +
                                ["exclusive groups", "shared groups", "mixed"].index(traffic))
    ag = np.arange(EMPTY, A)
    if traffic == "shared groups":
        groups = [rng.choice(ag, 40, replace=False) for _ in range(G - 1)] + [np.array([EMPTY, EMPTY, EMPTY + 1], np.uint32)]
    else:
        perm = rng.permutation(ag)
        groups = [perm[g * 32:(g + 1) * 32] for g in range(G)]
    cl = _Cluster(how, groups, A, G, R)
    try:
        crossed = False
        for rnd in range(2):
            crossed |= cl.holey(rng)
            batches = []
            for r in range(2):
                if traffic == "mixed":
                    n = 96
                    kind = rng.integers(0, 3, n).astype(np.uint8)
                    lists = [rng.choice(ag, 20, replace=False) for _ in range(4)]
                    target = np.where(kind == 0, rng.choice(ag, n), np.where(kind == 1, rng.integers(0, G, n), rng.integers(0, 4, n)))
                    cols = _mixed_cols(rng, kind, target, lists)
                else:
                    n = 48
                    cols = _mixed_cols(rng, np.ones(n, np.uint8), rng.integers(0, G, n))
                cols[0][: n // 4] = [rng.choice(groups[t]) if k == 1 else rng.integers(0, EMPTY)
                                     for k, t in zip(cols[1][: n // 4].tolist(), cols[2][: n // 4].tolist())]   # senders inside their group
                batches.append(cols)
            lost = cl.import_(batches, traffic == "mixed", f"{how}, {traffic}, round {rnd}", index=True,
                              commit=True if traffic == "mixed" else None)
            assert sum(lost) > 0
        assert crossed
    finally:
        cl.close()


# ---------------------------------------------------------------------------------------------------------------------
# D. the front end's overflow report
def test_front_end_overflow_report_on_holey_rings(shared, tmp_path):
    """SwarmsDB with priority dequeue and 8-slot rings: holes from priority receives, a filtered take and expiry, then
    one flush of p2p, group and broadcast messages.  The device decides which atomically claimed records survive; the
    model (a RingModel over message ids) says how many: FAILED lands on exactly the lost p2p / group messages, each
    broadcast names exactly the receivers that missed it, unread counts follow, and a resend into drained rings
    delivers every failed message once.  A flush that loses more than the log holds fails its whole batch."""
    import time

    import swarmdb_b200 as sdb
    from tests.ring_ref import RingModel
    R = 8
    cfg = sdb.GpuConfig(max_agents=4096, max_groups=4, ring_slots=R, deterministic_ids=True, flush_threshold=100000,
                        priority_dequeue=True)
    db = sdb.SwarmsDB(save_dir=str(tmp_path), auto_save=False, gpu_config=cfg)
    rng = np.random.default_rng(8)
    rcv = [f"r{i}" for i in range(6)]
    everyone = ["s"] + rcv
    db.register_agents(everyone)
    db.add_agent_group("team", rcv[:4])
    ring, num, rev = RingModel(R), {}, {}
    ix = {a: i for i, a in enumerate(everyone)}            # the model's agent keys
    inbox = {a: [] for a in everyone}
    prio, read, failed, missed = {}, set(), set(), set()          # missed: (agent, broadcast id) never queued

    def key(mid):
        if mid not in num:
            num[mid] = len(num) + 1; rev[num[mid]] = mid
        return num[mid]

    def live(a):
        return [rev[x] for x in ring.live_seqs(ix[a])]

    def pending(a):
        return {m.id for m in db.peek_messages(a, 100)}

    def retired(a, gone):
        p = pending(a)
        assert p == set(live(a)) - set(gone), a
        ring.retire_to(ix[a], [key(x) for x in live(a) if x in p])

    def p2p(a, k):
        out = []
        for _ in range(k):
            pr = sdb.MessagePriority(int(rng.integers(0, 4)))
            mid = db.send_message("s", f"to {a} #{len(num)}", a, priority=pr)
            prio[mid] = int(pr); key(mid); inbox[a].append(mid); out.append(mid)
        return out

    # fill: six messages per receiver, the first three older than the expiry cutoff
    for a in rcv:
        ring.append(ix[a], [key(m) for m in p2p(a, 3)])
    db.flush()
    time.sleep(0.02)
    cut = time.time()
    time.sleep(0.02)
    for a in rcv:
        ring.append(ix[a], [key(m) for m in p2p(a, 3)])
    db.flush()
    # holes
    for a in rcv[:4]:
        got = [m.id for m in db.receive_messages(a, 2)]
        top = sorted(live(a), key=lambda x: -prio[x])                 # stable: stream order within a priority
        assert got == top[:2], a
        read.update(got); retired(a, got)
    got = [m.id for m in db.receive_matching(rcv[5], 8, min_priority=sdb.MessagePriority.HIGH)]
    assert sorted(got) == sorted(x for x in live(rcv[5]) if prio[x] >= 2)
    read.update(got); retired(rcv[5], got)
    old = live(rcv[4])[:3]
    assert db.expire_pending(older_than=cut, agent_ids=[rcv[4]]) == 3
    retired(rcv[4], old)
    assert any(ring.ntomb(ix[a]) for a in rcv)

    def unread(a):
        return sum(1 for m in inbox[a] if m not in failed and m not in read and (a, m) not in missed)

    # the flush under test: p2p, group and broadcast messages in one buffer
    cap = {a: ring.capacity(ix[a]) for a in rcv}
    new = {a: p2p(a, 3) for a in rcv}
    groups, bcast = [], []
    for k in range(2):
        ids = db.send_to_group("s", "team", f"team #{k}", priority=sdb.MessagePriority.NORMAL)
        for a, mid in zip(rcv[:4], ids):
            new[a].append(mid); inbox[a].append(mid); groups.append(mid)
        mid = db.broadcast_message("s", f"all #{k}")
        bcast.append(mid)
        for a in everyone:
            inbox[a].append(mid)
        for a in rcv:
            new[a].append(mid)
    lost = sum(max(0, len(new[a]) - cap[a]) for a in rcv)
    assert lost > 0
    with pytest.raises(sdb.RingOverflow) as ei:
        db.flush()
    assert ei.value.exact and f"{lost} message(s)" in str(ei.value)
    dropped = {}
    for a in rcv:
        p = pending(a)
        surv = [m for m in new[a] if m in p]
        assert len(surv) == min(len(new[a]), cap[a]), (a, len(surv), len(new[a]), cap[a])
        assert p == set(live(a)) | set(surv), a
        dropped[a] = set(new[a]) - p
        ring.append(ix[a], [key(m) for m in surv])
    for a in rcv:
        for m in new[a]:
            msg = db.get_message(m)
            if m in bcast:
                continue
            assert (msg.status == sdb.MessageStatus.FAILED) == (m in dropped[a]), (a, m)
            if m in dropped[a]:
                failed.add(m)
    for m in bcast:
        msg = db.get_message(m)
        assert msg.status == sdb.MessageStatus.DELIVERED
        want = sorted(a for a in rcv if m in dropped[a])
        assert sorted(msg.metadata.get("undelivered_to", [])) == want, m
        missed.update((a, m) for a in want)
    for a in everyone:
        assert db.get_unread_message_count(a) == unread(a), a
    # drain, then resend: every failed message arrives once, nothing else
    for a in rcv:
        read.update(m.id for m in db.receive_messages(a, 100))
        assert pending(a) == set()
    contents = sorted(db.get_message(m).content for m in failed)
    resent = db.resend_failed_messages()
    db.flush()
    got = [m for a in rcv for m in db.receive_messages(a, 100)]
    assert sorted(m.id for m in got) == sorted(resent) and len(set(resent)) == len(resent) == len(failed)
    assert sorted(m.content for m in got) == contents
    # more drops than the log holds: the whole batch is FAILED
    many = [db.send_message("s", f"flood {k}", rcv[0]) for k in range(4200)]
    with pytest.raises(sdb.RingOverflow) as ei:
        db.flush()
    assert not ei.value.exact
    assert all(db.get_message(m).status == sdb.MessageStatus.FAILED for m in many)
    db.close()
