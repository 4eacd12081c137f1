"""Compact receive (sdb_receive_compact) against the CPU oracle and against sdb_receive_batch, bit-exact.

A compact receive returns the records a full receive would return as one 16-byte entry per record plus one row and one
padded payload per distinct payload image.  After expand_compact every call must equal the oracle's receive: counts,
every header field and the padded payload bytes; stats()["delivered"] and agent_loads() must follow.  The format's own
rules are checked on every result: rows in order of first appearance, payload offsets the running sum of pad32(len),
reserved = 0, and exactly one row per shared-layout group send that has records in the call plus one per other record.
"""
import numpy as np
import pytest

from tests.test_gpu_shared_layout import THRESHOLD, _arena_advance, _payloads

pytestmark = pytest.mark.gpu

NO_GROUP = 0xFFFFFFFF


def _check_format(res, shared=True):
    """Invariants of a compact result; returns the expanded (counts, headers, payload)."""
    from swarmdb_b200._native import expand_compact, pad32
    cnt, ent, snd, pay = res
    assert int(cnt.sum()) == len(ent)
    assert np.all(snd["reserved"] == 0)
    plen = pad32(snd["len"].astype(np.int64))
    off = np.zeros(len(snd), np.int64)
    if len(snd) > 1:
        np.cumsum(plen[:-1], out=off[1:])
    assert np.array_equal(snd["payload_off"].astype(np.int64), off)
    assert len(pay) == int(plen.sum())
    s = ent["send"].astype(np.int64)
    assert len(ent) == 0 or s.max() < len(snd)
    _, first = np.unique(s, return_index=True)
    assert np.array_equal(s[np.sort(first)], np.arange(len(snd)))          # first appearance order: 0, 1, 2, ..
    hdr, full = expand_compact(ent, snd, pay)
    # expected rows: group records (all from shared-layout batches here) share a row per send - identified by their
    # per-send random timestamp - and every other record has its own
    grp = hdr["group"] != NO_GROUP
    sends = np.stack([hdr["timestamp"][grp].view(np.uint64), hdr["sender"][grp].astype(np.uint64)])
    want = int((~grp).sum()) + (np.unique(sends, axis=1).shape[1] if shared else int(grp.sum()))
    assert len(snd) == want, (len(snd), want)
    return cnt, hdr, full


def _same(got, want, what=""):
    cg, hg, pg = got
    cc, hc, pc = want
    assert np.array_equal(cg, cc), (what, cg[:16], cc[:16])
    assert len(hg) == len(hc), (what, len(hg), len(hc))
    for f in hg.dtype.names:
        assert np.array_equal(hg[f], hc[f]), (what, f)
    assert pg.tobytes() == pc.tobytes(), what


class Rig:
    """One or more GPU handles fed the same traffic as the CPU oracle: G exclusive groups of F members (agents
    0 .. G F - 1) and `extra` non-member agents that send."""

    def __init__(self, rng, G=40, F=64, extra=64, twins=1, **kw):
        from oracle.cpu_ref import CpuOracle
        from swarmdb_b200._native import Shard
        self.rng, self.G, self.F = rng, G, F
        self.A = G * F + extra
        kw.setdefault("ring_slots", 512)
        kw.setdefault("max_batch_sends", 4096)
        kw.setdefault("list_pool_entries", 1 << 16)
        self.gs = [Shard(max_agents=self.A, max_groups=G, **kw) for _ in range(twins)]
        self.g = self.gs[0]
        self.c = CpuOracle(self.A, G)
        perm = rng.permutation(G * F).astype(np.uint32)
        self.members = [perm[k * F:(k + 1) * F] for k in range(G)]
        self.idx = np.arange(self.A, dtype=np.uint32)
        for x in self.gs + [self.c]:
            for k, m in enumerate(self.members):
                x.create_group(k, m)
            x.register(self.idx)
        self.delivered = 0
        self.check_advance = True

    def close(self):
        for g in self.gs:
            g.close()
        self.c.close()

    def shared_batch(self, n, max_len=256):
        rng = self.rng
        assert n * self.F >= THRESHOLD
        s = rng.integers(self.G * self.F, self.A, n)
        grp = rng.integers(0, self.G, n)
        prio, typ = rng.integers(0, 4, n), rng.integers(0, 7, n)
        lens, off, buf = _payloads(rng, n, max_len)
        ts = rng.random(n) + 1.0
        t0 = self.g.stats()["arena_tail_bytes"]
        base = self.c.send_group_batch(s, grp, prio, typ, lens, off, buf, ts)[0]
        for g in self.gs:
            assert g.send_group_batch(s, grp, prio, typ, lens, off, buf, ts) == base
        if self.check_advance:                 # proves the shared layout (a batch that meets the wrap point skips to it)
            assert self.g.stats()["arena_tail_bytes"] - t0 == _arena_advance(self.F, lens)

    def p2p(self, n, max_len=200):
        rng = self.rng
        s, r = rng.integers(0, self.A, n), rng.integers(0, self.A, n)
        prio = rng.integers(0, 4, n)
        lens, off, buf = _payloads(rng, n, max_len)
        base = self.c.send_batch(s, r, prio, None, lens, off, buf)
        for g in self.gs:
            assert g.send_batch(s, r, prio, None, lens, off, buf) == base

    def broadcast(self, n, max_len=200):
        rng = self.rng
        lists = [rng.choice(self.A, size=int(rng.integers(1, 200)), replace=False) for _ in range(n)]
        lo = np.zeros(n + 1, np.uint64); lo[1:] = np.cumsum([len(x) for x in lists])
        li = np.concatenate(lists).astype(np.uint32)
        s, prio = rng.integers(0, self.A, n), rng.integers(0, 4, n)
        lens, off, buf = _payloads(rng, n, max_len)
        base = self.c.send_list_batch(s, lo, li, prio, None, lens, off, buf)
        for g in self.gs:
            assert g.send_list_batch(s, lo, li, prio, None, lens, off, buf) == base

    def mixed(self, rounds=2):
        for _ in range(rounds):
            self.p2p(400)
            self.shared_batch(300)
            self.broadcast(6)

    def compact(self, agents, k, flags=0, what="", shared=True):
        """Compact receive on the first handle against the oracle's full receive, then delivered + loads."""
        from swarmdb_b200._native import RECV_PEEK
        got = _check_format(self.g.receive_compact(agents, k, flags), shared)
        want = self.c.receive_batch(self.idx if agents is None else agents, k, flags, rec_cap=1 << 21)
        _same(got, want, what)
        if not flags & RECV_PEEK:
            self.delivered += len(want[1])
        assert self.g.stats()["delivered"] == self.delivered, what
        ag = self.idx if agents is None else np.asarray(agents, np.uint32)
        lg, lc = self.g.agent_loads(ag), self.c.agent_loads(ag)
        assert np.array_equal(lg["pending"], lc["pending"]), what
        assert np.array_equal(lg["pending_by_prio"], lc["pending_by_prio"]), what
        return got

    def drain(self, shared=True):
        self.compact(self.idx, 100000, 0, "drain", shared)
        st = self.g.stats()
        assert st["enqueued"] == st["delivered"] and st["ring_overflow"] == 0


FLAG_SETS = [0, 1, 2, 3]          # 0, PRIORITY, PEEK, PEEK | PRIORITY


def test_compact_matches_the_oracle_on_shared_p2p_and_broadcast_records():
    """Bulk compact receives over all agents, a subset and single agents, with every flag combination."""
    rng = np.random.default_rng(501)
    r = Rig(rng)
    try:
        r.mixed(3)
        for flags in FLAG_SETS:
            r.compact(None, 3, flags, f"all flags={flags}")
        some = rng.choice(r.A, size=300, replace=False).astype(np.uint32)
        for flags in FLAG_SETS:
            r.compact(some, 5, flags, f"subset flags={flags}")
        for a in rng.choice(r.G * r.F, size=6, replace=False):
            for flags in FLAG_SETS:
                r.compact([int(a)], 4, flags, f"one agent {a} flags={flags}")
        r.mixed(1)
        r.compact(r.idx, 7, 1, "priority after more traffic")
        r.drain()
    finally:
        r.close()


def test_rows_follow_first_appearance_and_each_shared_payload_is_returned_once():
    """One shared batch alone: every row is one send, referenced by the members in the call; the payload bytes are
    the sends' padded payloads, each once."""
    from swarmdb_b200._native import pad32
    rng = np.random.default_rng(502)
    r = Rig(rng)
    try:
        r.shared_batch(300)
        cnt, ent, snd, pay = r.g.receive_compact(r.idx, 1000, 2)
        _check_format((cnt, ent, snd, pay))
        assert len(snd) == 300 and len(ent) == 300 * r.F
        assert len(pay) == int(pad32(snd["len"].astype(np.int64)).sum())
        assert np.array_equal(np.bincount(ent["send"].astype(np.int64), minlength=300), np.full(300, r.F))
        r.compact(r.idx, 1000, 0, "all")
        r.drain()
    finally:
        r.close()


def test_compact_peek_then_full_receive_returns_the_same_records():
    from swarmdb_b200._native import RECV_PEEK, RECV_PRIORITY, expand_compact
    rng = np.random.default_rng(503)
    r = Rig(rng)
    try:
        r.mixed(2)
        for flags, agents, k in ((0, None, 4), (RECV_PRIORITY, r.idx[::3], 6), (0, r.idx[5:9], 50)):
            cnt, ent, snd, pay = r.g.receive_compact(agents, k, flags | RECV_PEEK)
            hdr, full = expand_compact(ent, snd, pay)
            cnt, ent = cnt.copy(), ent.copy()
            cg, hg, pg = r.g.receive_batch(agents, k, flags)
            assert np.array_equal(cnt, cg) and hdr.tobytes() == hg.tobytes() and full.tobytes() == pg.tobytes()
            cc, hc, pc = r.c.receive_batch(r.idx if agents is None else agents, k, flags, rec_cap=1 << 21)
            assert hg.tobytes() == hc.tobytes() and pg.tobytes() == pc.tobytes()
    finally:
        r.close()


def test_partial_sends_keep_one_row_each():
    """Agent subsets and small k take only some members of a send: that send still gets exactly one row."""
    rng = np.random.default_rng(504)
    r = Rig(rng)
    try:
        r.shared_batch(300)
        r.p2p(200)
        r.shared_batch(300)
        half = np.sort(rng.choice(r.G * r.F, size=r.G * r.F // 2, replace=False)).astype(np.uint32)
        r.compact(half, 3, 0, "half of the members, k=3")
        r.compact(rng.permutation(r.idx)[:700], 1, 1, "scrambled subset, k=1, priority")
        r.compact(r.members[3], 2, 0, "one group's members")
        r.drain()
    finally:
        r.close()


def _twin_step(r, agents, k, flags, cap_kw, what):
    """Compact on handle 0 and full receive on handle 1 under the same capacity: the same records."""
    from swarmdb_b200._native import ENTRY_DTYPE, HDR_DTYPE, SEND_DTYPE, RECV_PEEK
    ent = snd = pay = hdr = fpay = None
    if cap_kw.get("entries"):
        ent = np.zeros(cap_kw["entries"], ENTRY_DTYPE); hdr = np.zeros(cap_kw["entries"], HDR_DTYPE)
    if cap_kw.get("sends"):
        snd = np.zeros(cap_kw["sends"], SEND_DTYPE); hdr = np.zeros(cap_kw["sends"], HDR_DTYPE)
    if cap_kw.get("payload"):
        pay = np.zeros(cap_kw["payload"], np.uint8); fpay = np.zeros(cap_kw["payload"], np.uint8)
    got = _check_format(r.gs[0].receive_compact(agents, k, flags, out_entries=ent, out_sends=snd, out_payload=pay))
    want = r.gs[1].receive_batch(agents, k, flags, out_hdr=hdr, out_payload=fpay)
    _same(got, want, what)
    if not flags & RECV_PEEK:
        r.delivered += len(want[1])
    assert r.gs[0].stats()["delivered"] == r.gs[1].stats()["delivered"] == r.delivered, what
    return len(want[1])


@pytest.mark.parametrize("source", ["max_recv_records", "entry_cap", "send_cap", "payload_cap"])
def test_capacity_truncates_like_the_full_receive(source):
    """The record capacity binds through the handle's max_recv_records or one of the caller's buffers: the records a
    compact call takes equal sdb_receive_batch's under the same capacity, the lead-agent exception included, and a
    drain loop delivers every record exactly once."""
    rng = np.random.default_rng(505 + len(source))
    cap = 700
    kw = {"max_recv_records": cap} if source == "max_recv_records" else {}
    r = Rig(rng, twins=2, **kw)
    ck = {"entry_cap": {"entries": cap}, "send_cap": {"sends": cap}, "payload_cap": {"payload": cap * 256}}.get(source, {})
    try:
        r.mixed(2)
        heavy = r.idx[np.argsort(-r.c.agent_loads(r.idx)["pending"].astype(np.int64), kind="stable")]
        for flags in FLAG_SETS:
            _twin_step(r, None, 3, flags, ck, f"{source} all flags={flags}")
            _twin_step(r, heavy[:40], 100, flags, ck, f"{source} heavy agents flags={flags}")
        _twin_step(r, heavy[:1], 100000, 2, ck, f"{source} lead agent peek")
        rounds = 0
        while _twin_step(r, r.idx, 100000, rounds % 2, ck, f"{source} drain round {rounds}"):
            rounds += 1
        assert rounds >= 2
        for g in r.gs:
            st = g.stats()
            assert st["enqueued"] == st["delivered"] == r.delivered and st["ring_overflow"] == 0
    finally:
        r.close()


def test_zero_length_payloads_of_adjacent_sends_do_not_merge():
    rng = np.random.default_rng(506)
    r = Rig(rng)
    try:
        r.shared_batch(300, max_len=0)
        r.p2p(300, max_len=0)
        r.shared_batch(300, max_len=0)
        cnt, ent, snd, pay = r.g.receive_compact(r.idx, 1000, 2)
        assert len(pay) == 0 and np.all(snd["len"] == 0)
        assert len(snd) == 600 + 300
        r.compact(r.idx, 2, 1, "zero-length priority")
        r.drain()
    finally:
        r.close()


def test_per_recipient_layout_gives_every_record_its_own_row(monkeypatch):
    monkeypatch.setenv("SDB_SHARED_PAYLOAD", "0")
    rng = np.random.default_rng(507)
    r = Rig(rng)
    try:
        r.mixed(2)
        cnt, ent, snd, pay = r.g.receive_compact(r.idx, 5, 2)
        assert len(snd) == len(ent) > 0
        r.compact(r.idx, 5, 0, "per-recipient", shared=False)
        r.drain(shared=False)
    finally:
        r.close()


def test_compact_across_a_wrapping_arena_and_the_2_pow_32_handle_wrap():
    rng = np.random.default_rng(508)
    r = Rig(rng, arena_bytes=1 << 22, ring_slots=256)
    r.check_advance = False
    try:
        for rnd in range(16):
            r.p2p(200)
            r.shared_batch(260)
            flags = 1 if rnd % 4 == 1 else 0
            r.compact(r.idx if rnd % 2 else r.idx[:6], 9 if rnd % 2 else 12, flags, f"small arena round {rnd}")
            if rnd % 2 == 0:
                r.compact(r.idx, 7, flags, f"small arena round {rnd} bulk")
        assert r.g.stats()["arena_tail_bytes"] > 2 * (1 << 22)
        r.drain()
    finally:
        r.close()
    r = Rig(rng, arena_bytes=1 << 24)
    r.check_advance = False
    try:
        r.g.debug_set_arena_pos((1 << 32) - 30000)
        for step in range(6):
            r.shared_batch(300)
            r.p2p(300)
            r.compact(r.idx, 4, step % 2, f"handle wrap step {step}")
        assert r.g.stats()["arena_tail_bytes"] > (1 << 32) * 32
        r.drain()
    finally:
        r.close()


def test_refusals_and_the_digest_after_a_compact_receive():
    from swarmdb_b200._native import RECV_ASYNC, SdbError
    rng = np.random.default_rng(509)
    r = Rig(rng)
    try:
        r.mixed(1)
        with pytest.raises(SdbError, match="SDB_EINVAL"):
            r.g.receive_compact(None, 3, RECV_ASYNC)
        r.compact(None, 3, 0, "after the refusal")
        r.g.digest_reset()
        with pytest.raises(SdbError, match="compact"):
            r.g.digest_fold()
        want = r.c.receive_batch(r.idx, 2, 0, rec_cap=1 << 21)
        _same(r.g.receive_batch(r.idx, 2, 0), want, "full receive after a compact one")
        r.delivered += len(want[1])
        assert r.g.stats()["delivered"] == r.delivered
        r.g.digest_fold()                                  # a full receive restores the digest
        r.drain()
    finally:
        r.close()


def test_one_agent_compact_with_the_latency_server_running():
    """A one-agent compact call takes the bulk plan, not the server, and the server still answers afterwards."""
    rng = np.random.default_rng(510)
    r = Rig(rng, G=16, F=64)
    try:
        r.g.latency_server(True)
        r.mixed(3)
        r.g.profile(True)
        agents = rng.choice(r.G * r.F, size=8, replace=False)
        for i, a in enumerate(agents):
            r.compact([int(a)], [3, 40][i % 2], [0, 2, 1, 3][i % 4], f"server running, agent {a}")
            hg, pg, _ = r.g.receive_one(int(agents[-1 - i]), 2, 0)
            _, hc, pc = r.c.receive_batch([int(agents[-1 - i])], 2, 0)
            assert hg.tobytes() == hc.tobytes() and pg.tobytes() == pc.tobytes()
            r.delivered += len(hc)
        prof = r.g.profile_read()
        assert prof["recv_compact"][1] == len(agents)
        r.g.latency_server(False)
        r.drain()
    finally:
        r.close()


def test_surface_receive_batch_compact_matches_receive_batch(tmp_path):
    import swarmdb_b200 as sdb
    from swarmdb_b200._native import expand_compact
    rng = np.random.default_rng(511)
    G, F, extra = 20, 1000, 10
    cfg = dict(max_agents=G * F + extra + 16, max_groups=G, ring_slots=256, arena_bytes=1 << 26, max_payload_bytes=256,
               deterministic_ids=True)
    dbs = [sdb.SwarmsDB(save_dir=str(tmp_path / f"d{i}"), auto_save=False, gpu_config=sdb.GpuConfig(**cfg)) for i in range(2)]
    try:
        names = [f"agent{i}" for i in range(G * F + extra)]
        perm = rng.permutation(G * F)
        for db in dbs:
            for a in names:
                db.register_agent(a)
            for k in range(G):
                db.add_agent_group(f"g{k}", [names[int(i)] for i in perm[k * F:(k + 1) * F]])
        idx = np.array([dbs[0].agent_index(a) for a in names], np.uint32)
        n = 40
        s = idx[G * F + rng.integers(0, extra, n)]
        grp = np.array([dbs[0]._group_idx[f"g{int(x)}"] for x in rng.integers(0, G, n)], np.uint32)
        prio = rng.integers(0, 4, n)
        lens, off, buf = _payloads(rng, n, 200)
        l2, o2, b2 = _payloads(rng, 300, 100)
        r2 = idx[rng.integers(0, G * F, 300)]
        for db in dbs:
            db.send_to_group_batch(s, grp, prio, np.zeros(n), lens, off, buf)
            db.send_batch(s[:1].repeat(300), r2, None, np.zeros(300), l2, o2, b2)
        for k, pr in ((3, False), (5, True), (1000, None)):
            cg, hg, pg = dbs[0].receive_batch(None, k, pr)
            cc, ent, snd, pay = dbs[1].receive_batch_compact(None, k, pr)
            hc, pc = expand_compact(ent, snd, pay)
            assert np.array_equal(cg, cc) and hg.tobytes() == hc.tobytes() and pg.tobytes() == pc.tobytes()
            assert len(snd) <= len(ent)
        assert dbs[0].shard.stats()["delivered"] == dbs[1].shard.stats()["delivered"] == n * F + 300
    finally:
        for db in dbs:
            db.close()


def _record_hashes(payload, lens):
    """A 64-bit hash per padded payload (the granules of each record, position-keyed), vectorised."""
    w = np.ascontiguousarray(payload).view(np.uint64)
    nw = ((lens.astype(np.int64) + 31) // 32) * 4
    start = np.zeros(len(nw), np.int64)
    if len(nw) > 1:
        np.cumsum(nw[:-1], out=start[1:])
    pos = np.arange(len(w), dtype=np.int64) - np.repeat(start, nw)
    x = (w ^ (pos.astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15))) * np.uint64(0xFF51AFD7ED558CCD)
    x ^= x >> np.uint64(29)
    h = np.zeros(len(nw), np.uint64)
    nz = nw > 0
    h[nz] = np.add.reduceat(x, start[nz])
    return h


def test_c2_compact_peek_matches_the_full_receive():
    """The bench's c2 construction: 1M agents, 65,536 group sends to 64-member groups (fixed 256-byte payloads, then
    U[1,256]).  A compact PEEK of the whole step has 65,536 rows and expands to the full receive that follows; payloads
    are compared through per-record hashes."""
    from bench import Workload
    from swarmdb_b200._native import RECV_PEEK, Shard
    wl = Workload()
    rec_cap = wl.S * wl.F + (1 << 16)
    shard = Shard(max_agents=wl.A, ring_slots=64, arena_bytes=1 << 33, max_payload_bytes=wl.L, max_groups=1 << 14,
                  member_pool_entries=wl.A + 1024, max_batch_sends=wl.S, max_batch_payload=wl.S * wl.L,
                  max_recv_records=rec_cap, max_recv_payload=rec_cap * wl.L)
    try:
        shard.register(np.arange(wl.A, dtype=np.uint32))
        for g in range(wl.G):
            shard.create_group(g, wl.members(g))
        for step in range(2):
            shard.send_group_batch(*wl.parity_batch(step, 0))
            cnt, ent, snd, pay = shard.receive_compact(None, 100, RECV_PEEK)
            assert len(ent) == wl.S * wl.F and len(snd) == wl.S
            s = ent["send"].astype(np.int64)
            _, first = np.unique(s, return_index=True)
            assert np.array_equal(s[np.sort(first)], np.arange(wl.S))
            cnt, ent, snd = cnt.copy(), ent.copy(), snd.copy()
            row_hash = _record_hashes(pay, snd["len"])
            cg, hg, pg = shard.receive_batch(None, 100, 0)
            assert np.array_equal(cnt, cg) and len(hg) == len(ent)
            assert np.array_equal(hg["seq"], ent["seq"]) and np.array_equal(hg["receiver"], ent["receiver"])
            row = snd[s]
            for f in ("timestamp", "sender", "group", "len", "prio", "type"):
                assert np.array_equal(hg[f], row[f]), f
            assert np.array_equal(_record_hashes(pg, hg["len"]), row_hash[s])
        st = shard.stats()
        assert st["delivered"] == st["enqueued"] == 2 * wl.S * wl.F
    finally:
        shard.close()
