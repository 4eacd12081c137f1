"""Shared-payload records (DESIGN 4.5) through every receive path, against the CPU oracle, bit-exact.

A pure group batch above the pull threshold (16,384 records) to exclusive groups with payloads <= 512 bytes keeps, per
send, one header per member and ONE payload in the arena log; the ring entry of member j then carries the distance
from its header to the payload (dm1 != 0 except for the last member).  Every consumer must find the payload there:
the <= 8-agent single-launch receive (k_recv_small), the latency server's fast and slow paths, the bulk gathers (LSU
below 4096 records, TMA from 4096), PEEK, the arena wrap, the 2^32-granule handle wrap, the overflow log and the
Python surface.  Point-to-point and broadcast records (dm1 = 0) are interleaved so both kinds sit side by side in a
ring.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

THRESHOLD = 16384


def _payloads(rng, n, max_len):
    lens = rng.integers(0, max_len + 1, n).astype(np.uint16)
    stride = (max_len + 31) & ~31
    off = np.arange(n, dtype=np.uint64) * stride
    buf = rng.integers(33, 127, n * stride + 64).astype(np.uint8)      # printable: the surface decodes it as text
    return lens, off, buf


def _same(res_gpu, res_cpu, what=""):
    cg, hg, pg = res_gpu
    cc, hc, pc = res_cpu
    assert np.array_equal(cg, cc), (what, cg[:16], cc[:16])
    assert len(hg) == len(hc), (what, len(hg), len(hc))
    for f in hg.dtype.names:
        assert np.array_equal(hg[f], hc[f]), (what, f)
    assert pg.tobytes() == pc.tobytes(), what


class World:
    """G exclusive groups of F members (agents 0 .. G F - 1) and `extra` non-member agents that send."""

    def __init__(self, rng, G, F, extra=64, **kw):
        from oracle.cpu_ref import CpuOracle
        from swarmdb_b200._native import Shard
        self.rng, self.G, self.F = rng, G, F
        self.A = G * F + extra
        kw.setdefault("ring_slots", 512)
        kw.setdefault("max_batch_sends", 4096)
        kw.setdefault("list_pool_entries", 1 << 16)
        self.g = Shard(max_agents=self.A, max_groups=G, **kw)
        self.c = CpuOracle(self.A, G)
        perm = rng.permutation(G * F).astype(np.uint32)
        self.members = [perm[k * F:(k + 1) * F] for k in range(G)]
        for k, m in enumerate(self.members):
            self.g.create_group(k, m); self.c.create_group(k, m)
        self.idx = np.arange(self.A, dtype=np.uint32)
        self.g.register(self.idx); self.c.register(self.idx)

    def close(self):
        self.g.close(); self.c.close()

    def shared_batch(self, n, max_len=256):
        """n group sends from non-members: n F records; returns the arena advance of the device."""
        rng = self.rng
        assert n * self.F >= THRESHOLD
        s = rng.integers(self.G * self.F, self.A, n)
        grp = rng.integers(0, self.G, n)
        prio, typ = rng.integers(0, 4, n), rng.integers(0, 7, n)
        lens, off, buf = _payloads(rng, n, max_len)
        ts = rng.random(n)
        t0 = self.g.stats()["arena_tail_bytes"]
        assert self.g.send_group_batch(s, grp, prio, typ, lens, off, buf, ts) == \
            self.c.send_group_batch(s, grp, prio, typ, lens, off, buf, ts)[0]
        return self.g.stats()["arena_tail_bytes"] - t0, lens

    def p2p(self, n, max_len=200):
        rng = self.rng
        s, r = rng.integers(0, self.A, n), rng.integers(0, self.A, n)
        prio = rng.integers(0, 4, n)
        lens, off, buf = _payloads(rng, n, max_len)
        assert self.g.send_batch(s, r, prio, None, lens, off, buf) == self.c.send_batch(s, r, prio, None, lens, off, buf)

    def broadcast(self, n, max_len=200):
        rng = self.rng
        lists = [rng.choice(self.A, size=int(rng.integers(1, 200)), replace=False) for _ in range(n)]
        lo = np.zeros(n + 1, np.uint64); lo[1:] = np.cumsum([len(x) for x in lists])
        li = np.concatenate(lists).astype(np.uint32)
        s, prio = rng.integers(0, self.A, n), rng.integers(0, 4, n)
        lens, off, buf = _payloads(rng, n, max_len)
        assert self.g.send_list_batch(s, lo, li, prio, None, lens, off, buf) == \
            self.c.send_list_batch(s, lo, li, prio, None, lens, off, buf)

    def recv(self, agents, k, flags=0, what=""):
        _same(self.g.receive_batch(agents, k, flags),
              self.c.receive_batch(self.idx if agents is None else agents, k, flags, rec_cap=1 << 21), what)

    def drain(self):
        self.recv(self.idx, 100000, 0, "drain")
        st = self.g.stats()
        assert st["enqueued"] == st["delivered"] and st["ring_overflow"] == 0


def _arena_advance(F, lens):
    """Arena bytes of a group batch to groups of F members: with shared payloads F headers + ONE payload per send
    (sum (F + rgran - 1) granules), otherwise F full records (sum F rgran); SDB_SHARED_PAYLOAD=0 selects the latter."""
    from swarmdb_b200._native import shared_payload_enabled
    rgran = 1 + ((lens.astype(np.int64) + 31) // 32)
    return int(((F + rgran - 1) if shared_payload_enabled() else F * rgran).sum()) * 32


def _mixed_traffic(w, rounds=2):
    for _ in range(rounds):
        w.p2p(400)
        adv, lens = w.shared_batch(300)
        assert adv == _arena_advance(w.F, lens)
        w.broadcast(6)


def test_shared_records_through_the_small_receive_path():
    """k_recv_small (1, 2 and 8 agents, n k <= 1024) under flags 0, PRIORITY, PEEK and PEEK | PRIORITY."""
    from swarmdb_b200._native import RECV_PEEK, RECV_PRIORITY
    rng = np.random.default_rng(401)
    w = World(rng, G=40, F=64)
    try:
        _mixed_traffic(w)
        for rnd in range(30):
            n = [1, 2, 8][rnd % 3]
            agents = rng.choice(w.G * w.F, size=n, replace=False).astype(np.uint32)
            k = int(rng.integers(1, 1024 // n + 1))
            k = min(k, [7, 40, 1024 // n][rnd % 3])
            for flags in (RECV_PEEK, RECV_PEEK | RECV_PRIORITY):
                w.recv(agents, k, flags, f"small peek n={n} k={k} flags={flags}")
            flags = [0, RECV_PRIORITY][(rnd // 3) % 2]
            w.recv(agents, k, flags, f"small n={n} k={k} flags={flags}")
            if rnd == 15:
                _mixed_traffic(w, 1)
        w.drain()
    finally:
        w.close()


def test_shared_records_through_the_latency_server():
    """receive_one with the server on: the fast path (<= 32 records, stream order, no tombstones) and the slow path
    (after a priority receive left tombstones, and with more than 32 records), peeks included."""
    from swarmdb_b200._native import RECV_PEEK, RECV_PRIORITY
    rng = np.random.default_rng(402)
    w = World(rng, G=16, F=64)                           # about 19 records per member and batch
    try:
        w.g.latency_server(True)
        _mixed_traffic(w, 3)
        agents = rng.choice(w.G * w.F, size=120, replace=False)
        for i, a in enumerate(agents):
            a = int(a)
            if i < 40:                                   # fast path: fresh ring, stream order, short answers
                plan = [(RECV_PEEK, 5), (0, 3), (0, 32), (RECV_PEEK, 32)]
            elif i < 80:                                 # tombstones first: the stream receive takes the slow path
                plan = [(RECV_PRIORITY, 3), (RECV_PEEK, 8), (0, 8), (RECV_PRIORITY | RECV_PEEK, 6), (0, 32)]
            else:                                        # more than 32 records: slow path
                plan = [(RECV_PEEK, 100), (0, 40), (RECV_PRIORITY, 50), (0, 1000)]
            for flags, k in plan:
                hg, pg, _ = w.g.receive_one(a, k, flags)
                _, hc, pc = w.c.receive_batch([a], k, flags)
                assert hg.tobytes() == hc.tobytes() and pg.tobytes() == pc.tobytes(), (i, a, flags, k, len(hg), len(hc))
        w.g.latency_server(False)
        w.drain()
    finally:
        w.close()


def test_shared_records_through_the_bulk_gathers():
    """Bulk receives below 4096 records (LSU gather) and from 4096 (TMA gather), stream and priority order."""
    from swarmdb_b200._native import RECV_PEEK, RECV_PRIORITY
    rng = np.random.default_rng(403)
    w = World(rng, G=40, F=64)
    try:
        _mixed_traffic(w, 3)
        some = rng.choice(w.A, size=300, replace=False).astype(np.uint32)
        w.recv(some, 3, 0, "lsu stream")                          # bound 900
        w.recv(some, 4, RECV_PRIORITY, "lsu priority")            # bound 1200
        w.recv(some, 13, RECV_PEEK, "lsu peek")
        w.recv(w.idx, 2, RECV_PRIORITY | RECV_PEEK, "tma priority peek")
        w.recv(w.idx, 2, RECV_PRIORITY, "tma priority")           # bound 2 A >= 4096
        w.recv(None, 3, 0, "tma stream")
        _mixed_traffic(w, 1)
        w.recv(w.idx, 5, 0, "tma stream 2")
        w.drain()
    finally:
        w.close()


def test_shared_batches_wrap_a_small_arena():
    """A 4 MiB arena: shared batches wrap it many times; partial drains leave backlogs that straddle the wrap."""
    from swarmdb_b200._native import RECV_PRIORITY
    rng = np.random.default_rng(404)
    arena = 1 << 22
    w = World(rng, G=40, F=64, arena_bytes=arena, ring_slots=256)
    try:
        for rnd in range(24):
            w.p2p(200)
            w.shared_batch(260)
            if rnd % 3 == 0:
                w.broadcast(4)
            flags = RECV_PRIORITY if rnd % 4 == 1 else 0
            if rnd % 2:
                w.recv(w.idx, 9, flags, f"round {rnd}")
            else:
                w.recv(w.idx[:6], 12, flags, f"round {rnd} small")          # most agents keep their backlog
                w.recv(w.idx, 7, flags, f"round {rnd} bulk")
        assert w.g.stats()["arena_tail_bytes"] > 3 * arena
        w.drain()
    finally:
        w.close()


def test_shared_batches_across_the_2_pow_32_handle_wrap():
    """Ring handles are the low 32 bits of the arena position: shared batches run across that boundary."""
    from swarmdb_b200._native import RECV_PRIORITY
    rng = np.random.default_rng(405)
    w = World(rng, G=40, F=64, arena_bytes=1 << 24)
    try:
        w.g.debug_set_arena_pos((1 << 32) - 30000)                 # a shared batch of 300 sends is ~20k granules
        for step in range(6):
            w.shared_batch(300)
            w.p2p(300)
            flags = RECV_PRIORITY if step % 2 else 0
            w.recv(w.idx, 4, flags, f"step {step}")                 # leaves a backlog that straddles the wrap
            w.recv(w.idx[:5], 3, flags, f"step {step} small")
        assert w.g.stats()["arena_tail_bytes"] > (1 << 32) * 32
        w.drain()
    finally:
        w.close()


def test_shared_layout_ring_overflow_keeps_the_first_and_logs_the_rest():
    """Full rings in the shared layout: the survivors are the first sends of the batch, with their content, and the
    overflow log names dropped (agent, sequence number) pairs of exactly the other ones."""
    rng = np.random.default_rng(406)
    F, slots = 16400, 4
    w = World(rng, G=1, F=F, extra=4, ring_slots=slots, max_batch_sends=64)
    try:
        w.shared_batch(7, max_len=96)                              # 7 sends x 16,400 members, 4 slots each
        st = w.g.stats()
        assert st["ring_overflow"] == 3 * F
        ag, sq, dropped = w.g.overflow_log()
        assert dropped == 3 * F and len(sq) == 4096
        members = w.members[0]
        _same(w.g.receive_batch(members, 100), w.c.receive_batch(members, slots), "survivors")
        cc, hc, _ = w.c.receive_batch(members, 100)                # the oracle (unbounded rings) still has the rest
        lost = set(zip(np.repeat(members, cc.astype(np.int64)).tolist(), hc["seq"].tolist()))
        assert len(lost) == 3 * F and set(zip(ag.tolist(), sq.tolist())) <= lost
    finally:
        w.close()


@pytest.mark.parametrize("server", [False, True])
def test_surface_reads_shared_records(tmp_path, server):
    """SwarmsDB.send_to_group_batch above the threshold, then receive_messages, peek_messages and pending_snapshot
    (the single-agent path and the bulk path of the surface), with the latency server off and on."""
    import swarmdb_b200 as sdb
    from oracle.cpu_ref import CpuOracle
    rng = np.random.default_rng(407 + server)
    G, F, extra = 20, 1000, 10
    cfg = sdb.GpuConfig(max_agents=G * F + extra + 16, max_groups=G, ring_slots=256, arena_bytes=1 << 26,
                        max_payload_bytes=256, deterministic_ids=True)
    db = sdb.SwarmsDB(save_dir=str(tmp_path), auto_save=False, gpu_config=cfg)
    try:
        names = [f"agent{i}" for i in range(G * F + extra)]
        for a in names:
            db.register_agent(a)
        idx = {a: db.agent_index(a) for a in names}
        perm = rng.permutation(G * F)
        gidx = []
        c = CpuOracle(cfg.max_agents, G)
        for k in range(G):
            mem = [names[int(i)] for i in perm[k * F:(k + 1) * F]]
            db.add_agent_group(f"g{k}", mem)
            gidx.append(db._group_idx[f"g{k}"])
            c.create_group(gidx[-1], [idx[m] for m in mem])
        c.register(np.arange(cfg.max_agents))
        if server:
            db.shard.latency_server(True)
        n = 40                                                     # 40 sends x 1000 members >= 16,384 records
        s = np.array([idx[names[G * F + int(x)]] for x in rng.integers(0, extra, n)], np.uint32)
        grp = np.array([gidx[int(x)] for x in rng.integers(0, G, n)], np.uint32)
        prio = rng.integers(0, 4, n)
        lens, off, buf = _payloads(rng, n, 200)
        t0 = db.shard.stats()["arena_tail_bytes"]
        db.send_to_group_batch(s, grp, prio, np.zeros(n), lens, off, buf)
        c.send_group_batch(s, grp, prio, np.zeros(n), lens, off, buf)
        assert db.shard.stats()["arena_tail_bytes"] - t0 == _arena_advance(F, lens)
        r2 = np.array([idx[names[int(x)]] for x in rng.integers(0, G * F, 300)], np.uint32)
        l2, o2, b2 = _payloads(rng, 300, 100)
        db.send_batch(s[:1].repeat(300), r2, None, np.zeros(300), l2, o2, b2)
        c.send_batch(s[:1].repeat(300), r2, None, np.zeros(300), l2, o2, b2)

        def want(a, k, flags):
            _, h, p = c.receive_batch([idx[a]], k, flags)
            offs = np.concatenate([[0], np.cumsum(((h["len"].astype(np.int64) + 31) // 32) * 32)])
            return [(names[int(h["sender"][i])], bytes(p[offs[i]:offs[i] + int(h["len"][i])]).decode(), int(h["prio"][i]),
                     db._group_name[int(h["group"][i])] if int(h["group"][i]) != 0xFFFFFFFF else None) for i in range(len(h))]

        def got(msgs):
            return [(m.sender_id, m.content, int(m.priority), m.metadata.get("group")) for m in msgs]

        picked = [names[int(i)] for i in rng.choice(G * F, size=40, replace=False)]
        for a in picked[:20]:
            assert got(db.peek_messages(a, 5)) == want(a, 5, 2), a
            assert got(db.receive_messages(a, 3)) == want(a, 3, 0), a
        snap = db.pending_snapshot()
        for a in picked:
            assert got(snap.get(a, [])) == want(a, 1024, 2), a
        for a in picked:
            assert got(db.receive_messages(a, 1000)) == want(a, 1000, 0), a
        c.close()
    finally:
        db.close()
