"""Restore on the device (sdb_restore_compact) against the CPU oracle, byte for byte.

The oracle side of a restore is tests/restore_ref.py: every record is sent to the oracle with its original seq and
header fields, behind what the agent has pending.  After each call the handle's stats, agent_loads and arena tail are
checked (the tail against the placement model), then every receive path must deliver what the oracle delivers.
"""
import numpy as np
import pytest

from tests.restore_ref import restore_append, restore_granules
from tests.test_gpu_compact_receive import Rig, _same

pytestmark = pytest.mark.gpu

NO_GROUP = 0xFFFFFFFF


def _expand(res):
    """(counts, headers, payload) of a compact result (rows here are not one per send: duplicate-member groups are
    unshared)."""
    from swarmdb_b200._native import expand_compact
    cnt, ent, snd, pay = res
    return (cnt,) + tuple(expand_compact(ent, snd, pay))


def _renumber(ent, snd):
    from swarmdb_b200.core import _renumber_rows
    return _renumber_rows(ent, snd)


def _fresh(rig, **kw):
    """A new handle + oracle with the rig's groups and registrations and no traffic."""
    from oracle.cpu_ref import CpuOracle
    from swarmdb_b200._native import Shard
    kw.setdefault("ring_slots", 512)
    kw.setdefault("max_batch_sends", 4096)
    kw.setdefault("list_pool_entries", 1 << 16)
    g = Shard(max_agents=rig.A, max_groups=rig.G, **kw)
    c = CpuOracle(rig.A, rig.G)
    for x in (g, c):
        for k, m in enumerate(rig.members):
            x.create_group(k, m)
        x.register(rig.idx)
    return g, c


def _groups(rig):
    return {k: m for k, m in enumerate(rig.members)}


def _loads_equal(g, c, idx, what):
    lg, lc = g.agent_loads(idx), c.agent_loads(idx)
    for f in ("received", "pending", "pending_by_prio", "pending_granules"):
        assert np.array_equal(lg[f], lc[f]), (what, f)


def _restore_both(rig, g, c, agents, cnt, ent, snd, pay, shared, flags=0):
    """Restore on the device and in the oracle; checks the counters and the arena tail after the call."""
    st0 = g.stats()
    n, seq_end = g.restore_compact(agents, cnt, ent, snd, pay, flags)
    assert n == restore_append(c, _groups(rig), agents, cnt, ent, snd, pay)
    st1 = g.stats()
    assert st1["enqueued"] - st0["enqueued"] == n and st1["delivered"] == st0["delivered"]
    top = int(ent["seq"].max()) + 1 if len(ent) else 0
    assert seq_end == st1["next_seq"] == max(st0["next_seq"], top)
    assert st1["next_seq"] == c.next_seq
    grans = restore_granules(cnt, ent, snd, shared)
    assert st1["arena_tail_bytes"] - st0["arena_tail_bytes"] == 32 * grans, (st1["arena_tail_bytes"] - st0["arena_tail_bytes"], 32 * grans)
    _loads_equal(g, c, rig.idx, "after restore")
    return n


def _every_path(rig, g, c, shared, rng):
    from swarmdb_b200._native import RECV_PEEK, RECV_PRIORITY
    _same(_expand(g.receive_compact(None, 1 << 20, RECV_PEEK)), c.receive_batch(rig.idx, 1 << 20, RECV_PEEK, rec_cap=1 << 21),
          "peek compact")
    sel = rng.choice(rig.A, 300, replace=False).astype(np.uint32)
    _same(g.receive_batch(sel, 2, RECV_PRIORITY), c.receive_batch(sel, 2, RECV_PRIORITY), "priority pipeline")
    _same(g.receive_batch(sel, 2), c.receive_batch(sel, 2), "stream plan")
    eight = sel[:8]
    for flags in (0, RECV_PRIORITY):
        _same(g.receive_batch(eight, 3, flags), c.receive_batch(eight, 3, flags), "<= 8 agents")
    g.latency_server(True)
    for a in sel[8:16]:
        for flags in (0, RECV_PRIORITY):
            h, p, _ = g.receive_one(int(a), 2, flags)
            _, hc, pc = c.receive_batch([a], 2, flags)
            assert h.tobytes() == hc.tobytes() and p.tobytes() == pc.tobytes(), ("latency server", a)
    g.latency_server(False)
    _same(_expand(g.receive_compact(sel[16:], 2)), c.receive_batch(sel[16:], 2, 0, rec_cap=1 << 21), "compact")
    g.digest_reset(); c.digest_enable()
    while True:
        _, total, _ = g.receive_batch(None, 64, copy_out=False)
        g.digest_fold()
        c.receive_counts(None, 64)
        if total == 0:
            break
    assert np.array_equal(g.digest_read(), c.digest_read())
    assert g.queue_stats()["pending"] == 0 == c.queue_stats()["pending"]


def _traffic(rig):
    rig.mixed(2)
    # duplicate group members: a small (non-shared) group send where one agent is listed twice
    dup = np.array([rig.A - 1, rig.A - 2, rig.A - 1], np.uint32)
    for x in rig.gs + [rig.c]:
        x.create_group(rig.G - 1, dup)
    rig.members[rig.G - 1] = dup
    from tests.test_gpu_shared_layout import _payloads
    lens, off, buf = _payloads(rig.rng, 3, 256)
    lens[0] = 0
    lens[1] = 256
    base = rig.c.send_group_batch([0, 1, 2], [rig.G - 1] * 3, [1, 2, 3], None, lens, off, buf)[0]
    assert rig.g.send_group_batch([0, 1, 2], [rig.G - 1] * 3, [1, 2, 3], None, lens, off, buf) == base
    # partial sends: some records already received
    some = rig.rng.choice(rig.A, 200, replace=False).astype(np.uint32)
    _same(rig.g.receive_batch(some, 1), rig.c.receive_batch(some, 1), "partial")


@pytest.mark.parametrize("shared", ["1", "0"])
def test_snapshot_restore_into_fresh_handle_then_every_path(shared, monkeypatch):
    from swarmdb_b200._native import RECV_PEEK
    monkeypatch.setenv("SDB_SHARED_PAYLOAD", shared)
    rng = np.random.default_rng(7)
    rig = Rig(rng, G=8, F=64, extra=64)
    rig.check_advance = False
    _traffic(rig)
    cnt, ent, snd, pay = rig.g.receive_compact(None, 1 << 20, RECV_PEEK)
    ent, snd = _renumber(ent, snd)
    pay = pay.copy()
    g, c = _fresh(rig)
    g.profile(True)
    n = _restore_both(rig, g, c, rig.idx, cnt, ent, snd, pay, shared == "1")
    assert g.profile_read()["restore"][1] == 2          # plan phase + write phase
    assert n == len(ent) == int(rig.g.queue_stats()["pending"])
    assert np.array_equal(g.agent_loads(rig.idx)["pending_granules"], rig.g.agent_loads(rig.idx)["pending_granules"])
    # a send after the restore takes a fresh seq
    seq_end = g.stats()["next_seq"]
    assert g.send_batch([0], [1], [1], None, [4], [0], np.zeros(64, np.uint8)) == seq_end
    assert c.send_batch([0], [1], [1], None, [4], [0], np.zeros(64, np.uint8)) == seq_end
    _every_path(rig, g, c, shared == "1", rng)
    g.close(); c.close(); rig.close()


@pytest.mark.parametrize("shared", ["1", "0"])
def test_requeue_behind_newer_records_then_snapshot_of_that_queue(shared, monkeypatch):
    from swarmdb_b200._native import RECV_PEEK, RECV_PRIORITY
    monkeypatch.setenv("SDB_SHARED_PAYLOAD", shared)
    rng = np.random.default_rng(11)
    rig = Rig(rng, G=8, F=64, extra=64)
    rig.check_advance = False
    rig.mixed(1)
    sel = rng.choice(rig.A, 400, replace=False).astype(np.uint32)
    taken = rig.g.receive_compact(sel, 3, RECV_PRIORITY)
    cnt, ent, snd, pay = taken[0].copy(), taken[1].copy(), taken[2].copy(), taken[3].copy()
    rig.c.receive_batch(sel, 3, RECV_PRIORITY)
    rig.mixed(1)                                        # newer records now pending ahead of the requeue
    ent2, snd2 = _renumber(ent, snd)
    _restore_both(rig, rig.g, rig.c, sel, cnt, ent2, snd2, pay, shared == "1")
    # the queue now has old seqs behind newer ones: its stream-order snapshot descends (private tail)
    cnt, ent, snd, pay = rig.g.receive_compact(None, 1 << 20, RECV_PEEK)
    ent, snd = _renumber(ent, snd)
    pay = pay.copy()
    if shared == "1":
        assert restore_granules(cnt, ent, snd, True) < restore_granules(cnt, ent, snd, False)
    g, c = _fresh(rig)
    _restore_both(rig, g, c, rig.idx, cnt, ent, snd, pay, shared == "1")
    _every_path(rig, g, c, shared == "1", rng)
    g.close(); c.close(); rig.close()


def _one_row(n_agents, length, rng, group=0):
    from swarmdb_b200._native import ENTRY_DTYPE, SEND_DTYPE
    ent = np.zeros(n_agents, ENTRY_DTYPE)
    ent["seq"] = np.arange(n_agents) + 5
    ent["receiver"] = np.arange(n_agents)
    snd = np.zeros(1, SEND_DTYPE)
    snd["timestamp"], snd["sender"], snd["group"], snd["len"], snd["prio"], snd["type"] = 1.5, 0, group, length, 2, 3
    pay = rng.integers(0, 256, ((length + 31) & ~31) + 32).astype(np.uint8)
    return np.ones(n_agents, np.uint32), ent, snd, pay


def test_row_split_past_65535_records():
    from swarmdb_b200._native import HDR_DTYPE, Shard, expand_compact
    rng = np.random.default_rng(3)
    A = 70000
    g = Shard(max_agents=A, ring_slots=4, arena_bytes=1 << 26, max_recv_records=1 << 17)
    cnt, ent, snd, pay = _one_row(A, 100, rng)
    agents = np.arange(A, dtype=np.uint32)
    n, seq_end = g.restore_compact(agents, cnt, ent, snd, pay)
    assert n == A and seq_end == A + 5
    st = g.stats()
    assert st["arena_tail_bytes"] == 32 * restore_granules(cnt, ent, snd) == 32 * (A + 2 * 4)
    c2, e2, s2, p2 = g.receive_compact(agents, 1)
    assert np.array_equal(c2, cnt)
    hdr, full = expand_compact(e2, s2, p2)
    assert np.array_equal(hdr["seq"], ent["seq"]) and np.array_equal(hdr["receiver"], agents)
    assert np.all(hdr["len"] == 100) and np.all(hdr["group"] == 0) and np.all(hdr["prio"] == 2)
    assert np.array_equal(full.reshape(A, 128), np.tile(pay[:128], (A, 1)))
    assert len(s2) == 2                                 # two payload copies: one per block of headers
    assert HDR_DTYPE.itemsize == 32
    g.close()


@pytest.mark.parametrize("pos", ["arena_wrap", "handle_wrap"])
def test_restore_across_wraps(pos):
    """Records pending just below the wrap point; the restored region does not straddle it and starts there, so the
    agents' rings hold handles from both sides of the arena wrap, or of the 2^32 handle wrap."""
    from swarmdb_b200._native import RECV_PEEK
    rng = np.random.default_rng(5)
    rig = Rig(rng, G=4, F=64, extra=64)
    rig.check_advance = False
    rig.mixed(1)
    cnt, ent, snd, pay = rig.g.receive_compact(None, 1 << 20, RECV_PEEK)
    ent, snd = _renumber(ent, snd)
    pay = pay.copy()
    g, c = _fresh(rig, arena_bytes=1 << 22)
    grans = restore_granules(cnt, ent, snd)
    edge = 1 << 32 if pos == "handle_wrap" else 5 * ((1 << 22) // 32)
    g.debug_set_arena_pos(edge - 40)
    busy = np.nonzero(cnt)[0][:4].astype(np.uint32)
    buf = rng.integers(0, 256, 256).astype(np.uint8)
    for x in (g, c):                                   # 4 records of 2 granules below the edge, on restored agents
        x.send_batch([1, 2, 3, 4], busy, [0, 1, 2, 3], None, [20, 32, 0, 7], [0, 64, 128, 192], buf)
    assert grans > 40
    n, _ = g.restore_compact(rig.idx, cnt, ent, snd, pay)
    assert n == restore_append(c, _groups(rig), rig.idx, cnt, ent, snd, pay)
    assert g.stats()["arena_tail_bytes"] // 32 == edge + grans
    _loads_equal(g, c, rig.idx, "wrap")
    _every_path(rig, g, c, True, rng)
    g.close(); c.close(); rig.close()


def test_refusals_leave_state_unchanged():
    from swarmdb_b200._native import RECV_PEEK, SdbError, Shard
    rng = np.random.default_rng(9)
    rig = Rig(rng, G=4, F=64, extra=64)
    rig.check_advance = False
    rig.mixed(1)
    cnt, ent, snd, pay = rig.g.receive_compact(None, 1 << 20, RECV_PEEK)
    ent, snd = _renumber(ent, snd)
    pay = pay.copy()
    g, c = _fresh(rig, arena_bytes=1 << 20, max_recv_records=1 << 14)
    busy = np.nonzero(cnt)[0][:40].astype(np.uint32)
    first = np.concatenate([[0], np.cumsum(cnt.astype(np.int64))])
    sub_ent = np.concatenate([ent[first[a]:first[a + 1]] for a in busy])
    sub_cnt = cnt[busy]
    base = (busy, sub_cnt, sub_ent, snd, pay)

    def state():
        st = g.stats()
        return ({k: st[k] for k in ("next_seq", "enqueued", "delivered", "arena_tail_bytes", "n_agents")},
                g.agent_loads(rig.idx).tobytes(), g.receive_compact(None, 1 << 13, RECV_PEEK)[1].tobytes())

    s0 = state()

    def refused(code, args, flags=0):
        with pytest.raises(SdbError) as ei:
            g.restore_compact(*args, flags=flags)
        assert ei.value.code == code, (ei.value, code)
        assert state() == s0

    EINVAL, ERING, EARENA, ECAP = -1, -4, -5, -6
    bad = sub_ent.copy(); bad["send"][3] = len(snd)
    refused(EINVAL, (busy, sub_cnt, bad, snd, pay))
    bad = sub_ent.copy(); bad["receiver"][0] = (int(busy[0]) + 1) % rig.A
    refused(EINVAL, (busy, sub_cnt, bad, snd, pay))
    for field, v in (("len", 257), ("prio", 4), ("payload_off", 8), ("payload_off", len(pay))):
        s2 = snd.copy(); s2[field][len(s2) - 1] = v
        if field == "payload_off":
            s2["len"][len(s2) - 1] = 64                # a row that reads 64 bytes: at len(pay) it overruns
        refused(EINVAL, (busy, sub_cnt, sub_ent, s2, pay))
    refused(EINVAL, (np.concatenate([busy, busy[:1]]), np.concatenate([sub_cnt, [0]]), sub_ent, snd, pay))
    refused(EINVAL, (np.concatenate([busy[:-1], [rig.A + 5]]), sub_cnt, sub_ent, snd, pay))
    c2 = sub_cnt.copy(); c2[0] += 1
    refused(EINVAL, (busy, c2, sub_ent, snd, pay))
    refused(EINVAL, base, flags=RECV_PEEK)
    # ring overflow: one agent given more records than its ring holds
    big = 513
    one = np.repeat(sub_ent[:1], big); one["seq"] = np.arange(big) + 1
    refused(ERING, (busy[:1], [big], one, snd, pay))
    # capacity: more rows than one compact receive holds
    many = np.repeat(snd[:1], (1 << 14) + 1)
    refused(ECAP, (busy, sub_cnt, sub_ent, many, pay))
    g.restore_compact(*base)                           # the state is usable: the same input restores
    restore_append(c, _groups(rig), *base)
    _loads_equal(g, c, rig.idx, "after refusals")
    # arena full: a small arena that the restore cannot fit
    small = Shard(max_agents=rig.A, max_groups=rig.G, ring_slots=512, arena_bytes=1 << 16)
    with pytest.raises(SdbError) as ei:
        small.restore_compact(rig.idx, cnt, ent, snd, pay)
    assert ei.value.code == EARENA
    st = small.stats()
    assert st["enqueued"] == 0 and st["arena_tail_bytes"] == 0 and st["next_seq"] == 1
    small.close()
    g.close(); c.close(); rig.close()


def test_owned_on_sharded_handles():
    from oracle.cpu_ref import CpuOracle
    from swarmdb_b200._native import RECV_OWNED, RECV_PEEK, Shard
    rng = np.random.default_rng(13)
    rig = Rig(rng, G=4, F=64, extra=64)
    rig.check_advance = False
    rig.mixed(1)
    cnt, ent, snd, pay = rig.g.receive_compact(None, 1 << 20, RECV_PEEK)
    ent, snd = _renumber(ent, snd)
    pay = pay.copy()
    shard_of = (np.arange(rig.A) % 2).astype(np.uint8)
    for r in (0, 1):
        g = Shard(max_agents=rig.A, max_groups=rig.G, ring_slots=512, shard_id=r, num_shards=2)
        g.set_agent_shards(shard_of)
        n, _ = g.restore_compact(rig.idx, cnt, ent, snd, pay, RECV_OWNED)
        mine = shard_of == r
        assert n == int(cnt[mine].sum())
        ld = g.agent_loads(rig.idx)
        assert np.array_equal(ld["pending"][mine], cnt[mine]) and np.all(ld["pending"][~mine] == 0)
        o = CpuOracle(rig.A, rig.G)
        for k, m in enumerate(rig.members):
            o.create_group(k, m)
        o.register(rig.idx)
        assert restore_append(o, _groups(rig), rig.idx, cnt, ent, snd, pay, skip=lambda a: shard_of[a] != r) == n
        mine_idx = rig.idx[mine]
        _same(_expand(g.receive_compact(mine_idx, 1 << 20)), o.receive_batch(mine_idx, 1 << 20, 0, rec_cap=1 << 21), "owned")
        g.close(); o.close()
    rig.close()


@pytest.mark.parametrize("recv_cap", [1 << 16, 8])
def test_swarmsdb_snapshot_round_trip_and_requeue(tmp_path, recv_cap):
    """recv_cap = 8: the snapshot has several chunks, and every restored message must keep its own contents."""
    import swarmdb_b200 as sdb
    cfg = dict(max_agents=256, ring_slots=64, arena_bytes=1 << 22, max_payload_bytes=512, max_groups=8, id_nonce=0x1234,
               max_recv_records=recv_cap)
    db = sdb.SwarmsDB(save_dir=tmp_path, auto_save=False, gpu_config=sdb.GpuConfig(**cfg))
    names = [f"agent_{i}" for i in range(12)]
    for a in names:
        db.register_agent(a)
    db.add_agent_group("team", names[4:10])
    ids = [db.send_message(names[i % 3], {"k": i}, names[3 + i % 5]) for i in range(20)]
    ids += db.send_to_group(names[0], "team", "hello team")
    ids.append(db.broadcast_message(names[1], "to all", exclude_agents=names[9:]))
    db.flush()
    want = {a: [(m.id, m.content, m.sender_id, m.receiver_id, m.metadata.get("group"), m.visible_to)
                for m in db.peek_messages(a, 100)] for a in names}
    path = db.save_queue_snapshot(tmp_path / "q.npz")
    with np.load(path) as z:
        assert (len(z["chunk_off"]) - 1 > 2) == (recv_cap == 8)
    with pytest.raises(RuntimeError):                   # only a fresh instance takes a snapshot
        db.load_queue_snapshot(path)
    db.close()
    with pytest.raises(ValueError):                     # another id nonce
        sdb.SwarmsDB(save_dir=tmp_path, auto_save=False, gpu_config=sdb.GpuConfig(**{**cfg, "id_nonce": 7})).load_queue_snapshot(path)
    db2 = sdb.SwarmsDB(save_dir=tmp_path, auto_save=False, gpu_config=sdb.GpuConfig(**{**cfg, "id_nonce": None}))
    db2.load_queue_snapshot(path)
    assert db2.agent_index(names[5]) == 5
    got = {a: [(m.id, m.content, m.sender_id, m.receiver_id, m.metadata.get("group"), m.visible_to)
               for m in db2.receive_messages(a, 100)] for a in names}
    assert got == want
    new_id = db2.send_message(names[0], "after", names[1])
    assert int(new_id.replace("-", ""), 16) & ((1 << 64) - 1) > max(int(i.replace("-", ""), 16) & ((1 << 64) - 1) for i in ids)
    # requeue: what a compact receive took goes back behind the newer message, ids unchanged
    db2.send_message(names[2], "first", names[1])
    cnt, ent, snd, pay = db2.receive_batch_compact(np.array([1], np.uint32), 100)
    cnt, ent, snd, pay = cnt.copy(), ent.copy(), snd.copy(), pay.copy()
    db2.send_message(names[2], "newer", names[1])
    assert db2.requeue_batch_compact(cnt, ent, snd, pay, np.array([1], np.uint32)) == len(ent)
    order = [m.content for m in db2.receive_messages(names[1], 100)]
    assert order == ["newer", "after", "first"]
    db2.close()


def test_one_row_of_400k_records_is_linear():
    """A pending broadcast is one row; its restore must not cost more per record as the row grows (the rank of an entry
    in its row comes from a stable sort, not from pairwise compares)."""
    from swarmdb_b200._native import NO_RECEIVER, Shard, expand_compact
    rng = np.random.default_rng(6)
    times = {}
    for A in (50_000, 400_000):
        g = Shard(max_agents=A, ring_slots=4, arena_bytes=1 << 26, max_recv_records=1 << 19)
        cnt, ent, snd, pay = _one_row(A, 64, rng, group=NO_GROUP)
        ent["receiver"] = NO_RECEIVER
        agents = np.arange(A, dtype=np.uint32)
        g.restore_compact(agents[:1], cnt[:1], ent[:1], snd, pay)            # loads the kernels
        g.receive_batch(agents[:1], 1)
        g.profile(True)
        n, _ = g.restore_compact(agents, cnt, ent, snd, pay)
        times[A] = g.profile_read()["restore"][0]
        assert n == A and g.stats()["arena_tail_bytes"] - 32 * 3 == 32 * (A + -(-A // 65535) * 2)
        c2, e2, s2, p2 = g.receive_compact(agents, 1)
        hdr, full = expand_compact(e2, s2, p2)
        assert np.array_equal(hdr["seq"], ent["seq"]) and np.all(hdr["receiver"] == NO_RECEIVER)
        assert np.array_equal(full.reshape(A, 64), np.tile(pay[:64], (A, 1)))
        g.close()
    print(f"restore kernel ms for one row: {times}")
    assert times[400_000] < 16 * max(times[50_000], 0.05), times
