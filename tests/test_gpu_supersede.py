"""Superseding sends on the device (sdb_supersede) against tests/supersede_ref.py, byte for byte.

Superseded records are returned (archive mode) in the compact receive format; expanded they must equal the model's:
counts, every header field and the padded payload bytes.  Afterwards every receive path must deliver what the oracle
delivers after the same pass, i.e. what it would have delivered had the superseded records never been enqueued.
"""
import math

import numpy as np
import pytest

from tests.supersede_ref import TYPEF_SUPERSEDE, SupersedingOracle
from tests.test_gpu_compact_receive import Rig, _check_format, _same
from tests.test_gpu_expire import _loads_equal
from tests.test_gpu_shared_layout import _payloads
from tests.test_gpu_trim import _every_path

pytestmark = pytest.mark.gpu

F = TYPEF_SUPERSEDE


def _rig(rng, **kw):
    rig = Rig(rng, **kw)
    rig.check_advance = False
    rig.c = SupersedingOracle(rig.c, rig.G, dict(enumerate(rig.members)), rig.A)
    return rig


def _types(rng, n, p=0.7):
    """Types 0-2 (few, so keys collide), the flag on a share p, the JSON or extras bit on some."""
    t = rng.integers(0, 3, n) | np.where(rng.random(n) < 0.2, 0x08, 0)
    return (t | np.where(rng.random(n) < p, F, 0)).astype(np.uint8)


def _flagged_sends(rig, rounds=2, senders=None):
    """p2p, group and list sends from few senders with flagged and unflagged types, distinct timestamps."""
    rng = rig.rng
    senders = np.arange(rig.G * rig.F, rig.G * rig.F + 6) if senders is None else senders
    for _ in range(rounds):
        n = 600
        s, r, prio = rng.choice(senders, n), rng.integers(0, rig.A, n), rng.integers(0, 4, n)
        lens, off, buf = _payloads(rng, n, 200)
        ts, typ = rng.uniform(0, 10, n), _types(rng, n)
        base = rig.c.send_batch(s, r, prio, typ, lens, off, buf, ts)
        assert rig.g.send_batch(s, r, prio, typ, lens, off, buf, ts) == base
        n = 300
        s, grp, prio = rng.choice(senders, n), rng.integers(0, rig.G, n), rng.integers(0, 4, n)
        lens, off, buf = _payloads(rng, n, 256)
        ts, typ = rng.uniform(0, 10, n), _types(rng, n)
        base = rig.c.send_group_batch(s, grp, prio, typ, lens, off, buf, ts)[0]
        assert rig.g.send_group_batch(s, grp, prio, typ, lens, off, buf, ts) == base
        n = 6
        lists = [rng.choice(rig.A, size=int(rng.integers(1, 200)), replace=False) for _ in range(n)]
        lo = np.zeros(n + 1, np.uint64); lo[1:] = np.cumsum([len(x) for x in lists])
        li = np.concatenate(lists).astype(np.uint32)
        s, prio = rng.choice(senders, n), rng.integers(0, 4, n)
        lens, off, buf = _payloads(rng, n, 200)
        ts, typ = rng.uniform(0, 10, n), _types(rng, n)
        base = rig.c.send_list_batch(s, lo, li, prio, typ, lens, off, buf, ts)
        assert rig.g.send_list_batch(s, lo, li, prio, typ, lens, off, buf, ts) == base


def _all_calls(g, agents, flags=0, shared=True, **kw):
    """Archive-mode calls until nothing comes back; (summed counts, expanded headers, payload, calls)."""
    from swarmdb_b200._native import HDR_DTYPE
    total_cnt, hdrs, pays, calls = None, [], [], 0
    while True:
        cnt, hdr, pay = _check_format(g.supersede(agents, flags, **kw), shared)
        calls += 1
        total_cnt = cnt.astype(np.int64) if total_cnt is None else total_cnt + cnt
        if len(hdr) == 0:
            break
        hdrs.append(hdr); pays.append(pay)
    hdr = np.concatenate(hdrs) if hdrs else np.zeros(0, HDR_DTYPE)
    pay = np.concatenate(pays) if pays else np.zeros(0, np.uint8)
    return total_cnt.astype(np.uint32), hdr, pay, calls


@pytest.mark.parametrize("shared", ["1", "0"])
def test_supersede_matches_the_model_then_every_receive_path(shared, monkeypatch):
    from swarmdb_b200._native import RECV_PEEK, RECV_PRIORITY, make_filter
    monkeypatch.setenv("SDB_SHARED_PAYLOAD", shared)
    rng = np.random.default_rng(71)
    rig = _rig(rng, G=8, F=64, extra=64)
    _flagged_sends(rig)
    # holes in the windows: a priority receive and a filtered take
    some = rng.choice(rig.A, 120, replace=False).astype(np.uint32)
    _same(rig.g.receive_batch(some[:60], 2, RECV_PRIORITY), rig.c.receive_batch(some[:60], 2, RECV_PRIORITY), "holes")
    f = make_filter(prios=[1])
    _same(rig.g.receive_where(some[60:], 1, 0, f), rig.c.receive_where(some[60:], 1, 0, f), "filtered holes")
    st0 = rig.g.stats()
    perm = rng.permutation(rig.A).astype(np.uint32)
    parts = np.array_split(perm, 3)
    p1 = _check_format(rig.g.supersede(parts[0], RECV_PEEK), shared == "1")
    p2 = _check_format(rig.g.supersede(parts[0], RECV_PEEK), shared == "1")
    _same(p1, p2, "peek twice")
    _loads_equal(rig, "after peek")
    want = rig.c.supersede(parts[0])
    assert len(want[1]) > 100
    _same(p1, want, "peek vs model")
    got = _all_calls(rig.g, parts[0], shared=shared == "1")
    _same(got[:3], want, "superseded set")
    _loads_equal(rig, "after archive")
    assert rig.g.supersede(parts[0], archive=False)[1] == 0                 # the newest of every key stays
    cnt, total = rig.g.supersede(parts[1], archive=False)
    cc, tc = rig.c.supersede(parts[1], materialise=False)
    assert total == tc > 0 and np.array_equal(cnt, cc)
    st1 = rig.g.stats()
    assert {k: st1[k] for k in ("enqueued", "delivered")} == {k: st0[k] for k in ("enqueued", "delivered")}
    _every_path(rig, shared == "1", "after supersede")
    rig.close()


def test_capacity_partial_first_agent_and_argument_checks():
    from swarmdb_b200._native import ENTRY_DTYPE, RECV_PEEK, SEND_DTYPE, SdbError
    rng = np.random.default_rng(8)
    rig = _rig(rng, G=4, F=64, extra=64, max_recv_records=64)
    _flagged_sends(rig, 1)
    n = 300                                          # agent 7: 3 senders x 100 versions of one type
    s = rng.integers(0, 3, n) + rig.G * rig.F
    lens, off, buf = _payloads(rng, n, 100)
    r, typ = np.full(n, 7), np.full(n, F | 1, np.uint8)
    rig.c.send_batch(s, r, None, typ, lens, off, buf); rig.g.send_batch(s, r, None, typ, lens, off, buf)
    agents = np.concatenate([[7], rng.permutation(np.setdiff1d(rig.idx, [7]))]).astype(np.uint32)
    c1 = _check_format(rig.g.supersede(agents, RECV_PEEK))
    assert c1[0][0] == 64 and int(c1[0][1:].sum()) == 0
    _same(c1, rig.c.supersede(agents, RECV_PEEK, rec_cap=64), "partial first agent")
    ent, snd = np.zeros(10, ENTRY_DTYPE), np.zeros(10, SEND_DTYPE)
    want = rig.c.supersede(agents, materialise=False)
    got = _all_calls(rig.g, agents, out_entries=ent, out_sends=snd)
    assert got[3] > 30 and np.array_equal(got[0], want[0])
    _loads_equal(rig, "after capped calls")
    with pytest.raises(SdbError) as e:
        rig.g.supersede(agents, out_entries=np.zeros(0, ENTRY_DTYPE), out_sends=np.zeros(0, SEND_DTYPE))
    assert e.value.code == -8
    for bad_flags in (1, 4, 16, 32):
        with pytest.raises(SdbError) as e:
            rig.g.supersede(agents, bad_flags)
        assert e.value.code == -1
    for bad in ([1, 2, 1], [rig.A]):
        with pytest.raises(SdbError) as e:
            rig.g.supersede(np.array(bad, np.uint32), archive=False)
        assert e.value.code == -1
    rig.close()


def _one_agent(ring_slots=64, A=8):
    from swarmdb_b200._native import Shard
    g = Shard(max_agents=A, ring_slots=ring_slots, arena_bytes=1 << 24, max_payload_bytes=64)
    g.register(np.arange(A, dtype=np.uint32))
    return g


def _send(g, sender, receiver, typ, n=None, tag=0):
    n = len(np.atleast_1d(sender)) if n is None else n
    lens, off = np.full(n, 8, np.uint16), np.arange(n, dtype=np.uint64) * 64
    buf = np.full(n * 64 + 64, 65 + tag, np.uint8)
    return g.send_batch(np.broadcast_to(sender, n), np.broadcast_to(receiver, n), None, np.broadcast_to(typ, n), lens, off, buf)


def test_stale_versions_put_back_by_a_sweep_and_a_requeue_go_leases_stay():
    from swarmdb_b200._native import LEASE_RENEW, RECV_PEEK
    g = _one_agent()
    g.lease_reserve(256, 256 * 64)
    g.lease_set_policy(10, 256)
    s1 = _send(g, 1, 0, F | 1)                                        # v1 of sender 1
    _, ent, _, _, lb = g.receive_leased([0], 1, 10.0)                 # v1 in flight
    s2 = _send(g, 1, 0, F | 1)                                        # v2 pending
    assert g.supersede([0], archive=False)[1] == 0                    # a lease is not compared
    assert g.lease_stats()["live"] == 1
    g.lease_settle(np.array([lb], np.uint64), LEASE_RENEW, -math.inf)
    assert g.lease_sweep(0.0)[0] == 1                                 # v1 back behind v2
    cnt, ent, snd, pay = g.supersede([0])
    assert cnt[0] == 1 and ent["seq"].tolist() == [s1]                # by seq: the redelivered stale version goes
    assert g.receive_batch([0], 10, RECV_PEEK)[1]["seq"].tolist() == [s2]
    # a requeue of a taken older version behind the newer one
    c3, e3, n3, p3 = (x.copy() for x in g.receive_compact([0], 10))
    s4 = _send(g, 1, 0, F | 1)
    assert g.restore_compact([0], c3, e3, n3, p3)[0] == 1
    assert g.supersede([0], archive=False)[1] == 1
    assert g.receive_batch([0], 10)[1]["seq"].tolist() == [s4]
    g.close()


def test_a_seq_tie_from_restoring_a_peek_goes_to_the_later_record():
    from swarmdb_b200._native import RECV_PEEK
    g = _one_agent()
    a = _send(g, 1, 0, F | 2, tag=1)
    b = _send(g, 2, 0, F | 2, tag=2)
    cnt, ent, snd, pay = (x.copy() for x in g.receive_compact([0], 10, RECV_PEEK))
    assert g.restore_compact([0], cnt, ent, snd, pay)[0] == 2          # ring: a b a' b'
    hdr0 = g.receive_batch([0], 10, RECV_PEEK)[1]
    assert hdr0["seq"].tolist() == [a, b, a, b]
    cnt, ent, snd, pay = g.supersede([0])
    assert cnt[0] == 2 and ent["seq"].tolist() == [a, b]               # the first two positions: the earlier copies
    loads = g.agent_loads([0])
    assert loads["pending"][0] == 2
    g.close()


@pytest.mark.parametrize("senders", [7, 3000])
def test_deep_rings(senders):
    from oracle.cpu_ref import CpuOracle
    from swarmdb_b200._native import Shard
    rng = np.random.default_rng(senders)
    A, R = 32, 4096
    g = Shard(max_agents=4096, ring_slots=R, arena_bytes=1 << 28, max_payload_bytes=64, max_batch_sends=1 << 16,
              max_recv_records=1 << 18)
    c = CpuOracle(4096, 1)
    g.register(np.arange(4096, dtype=np.uint32)); c.register(np.arange(4096))
    c = SupersedingOracle(c, 1, watermark=4096)
    for _ in range(3):
        n = 1 << 14
        s, r = rng.integers(0, senders, n), rng.integers(0, A, n)
        typ = (rng.integers(0, 2, n) | np.where(rng.random(n) < 0.9, F, 0)).astype(np.uint8)
        lens, off, buf = _payloads(rng, n, 48)
        ts = rng.uniform(0, 1, n)
        assert c.send_batch(s, r, None, typ, lens, off, buf, ts) == g.send_batch(s, r, None, typ, lens, off, buf, ts)
    agents = np.arange(A, dtype=np.uint32)
    want = c.supersede(agents)
    _same(_all_calls(g, agents)[:3], want, "deep rings")
    _same(g.receive_batch(None, R), c.receive_batch(None, R), "drain")
    g.close(); c.close()


def test_seq_past_2_32_and_the_arena_handle_wrap():
    from oracle.cpu_ref import CpuOracle
    from swarmdb_b200._native import Shard
    A = 256
    rng = np.random.default_rng(4)
    g, c = Shard(max_agents=A, ring_slots=256, arena_bytes=1 << 22, max_payload_bytes=256), CpuOracle(A, 1)
    g.register(np.arange(A, dtype=np.uint32)); c.register(np.arange(A))
    c = SupersedingOracle(c, 1, watermark=A)
    g.debug_set_arena_pos((1 << 32) - 300)
    g.advance_seq((1 << 32) - 500)
    c.next_seq = (1 << 32) - 500
    for _ in range(6):
        n = 200
        s, r = rng.integers(0, 4, n), rng.integers(0, A, n)
        typ = (rng.integers(0, 2, n) | F).astype(np.uint8)
        lens, off, buf = _payloads(rng, n, 200)
        assert c.send_batch(s, r, None, typ, lens, off, buf) == g.send_batch(s, r, None, typ, lens, off, buf)
    assert g.stats()["arena_tail_bytes"] > (1 << 32) * 32 and g.stats()["next_seq"] > (1 << 32)
    _same(_all_calls(g, None)[:3], c.supersede(None), "wrap")
    _same(g.receive_batch(None, 1000), c.receive_batch(None, 1000), "drain")
    g.close(); c.close()


def test_sharded_handle_owned_agents():
    from oracle.cpu_ref import CpuOracle
    from swarmdb_b200._native import RECV_OWNED
    from tests.test_gpu_xshard import _async_cluster
    rng = np.random.default_rng(23)
    A, G, Fm, S = 2048, 32, 64, 300
    perm = rng.permutation(A)
    groups = [perm[k * Fm:(k + 1) * Fm] for k in range(G)]
    smap, shards, wb, bufs = _async_cluster(1, A, G, S, groups)
    s = shards[0]
    s.register(np.arange(A, dtype=np.uint32))
    o = CpuOracle(A, G)
    for k, m in enumerate(groups):
        o.create_group(k, m)
    o.register(np.arange(A))
    o = SupersedingOracle(o, G, dict(enumerate(groups)), A)
    for step in (1, 2):
        sender, grp, prio = rng.integers(0, 3, S), rng.integers(0, G, S), rng.integers(0, 4, S)
        typ = (rng.integers(0, 2, S) | F).astype(np.uint8)
        lens, off, buf = _payloads(rng, S, 256)
        ts = rng.uniform(0, 10, S)
        s.export_group_batch(sender, grp, prio, typ, lens, off, buf, bufs[step & 1][0], wb, ts)
        s.wire_publish(bufs[step & 1][0], wb, step)
        s.import_wire_ptrs_async(bufs[step & 1], wb, step)
        o.send_group_batch(sender, grp, prio, typ, lens, off, buf, ts)
    got = _all_calls(s, None, RECV_OWNED)
    want = o.supersede(None)
    assert len(want[1]) > 0
    _same(got[:3], (want[0][:A],) + want[1:], "owned archive")
    _same(s.receive_batch(np.arange(A, dtype=np.uint32), 1000), o.receive_batch(np.arange(A), 1000), "drain")
    s.close(); o.close()


def test_c2_backlog_drop_mode_matches_oracle_digests():
    """The 1M-agent c2 backlog with every send flagged, one drop-mode pass, then the full drain's digests and the queue
    statistics against an oracle that was only ever sent the surviving sends: per (group, sender, type) the last."""
    from bench import Workload
    from oracle.cpu_ref import CpuOracle
    from swarmdb_b200._native import Shard
    wl = Workload()
    g = Shard(max_agents=wl.A, ring_slots=64, arena_bytes=1 << 31, max_payload_bytes=wl.L, max_groups=wl.G,
              member_pool_entries=wl.A + 1024, max_batch_sends=wl.S, max_batch_payload=wl.S * wl.L,
              max_recv_records=1 << 23, max_recv_payload=(1 << 23) * wl.L)
    surv = CpuOracle(wl.A, wl.G)
    g.register(np.arange(wl.A, dtype=np.uint32))
    surv.register(np.arange(wl.A))
    for k in range(wl.G):
        g.create_group(k, wl.members(k)); surv.create_group(k, wl.members(k))
    sender, grp, prio, typ, lens, off, pay = wl.batch()
    typ = (np.asarray(typ, np.uint8) & 0x07) | F
    sender = sender % 64                                   # few senders: every group sees repeated keys ...
    while True:                                            # ... and, as in the workload, none is a member of its group
        bad = wl.group_of[sender] == grp
        if not bad.any():
            break
        sender[bad] = (sender[bad] + 1) % 64
    base = g.send_group_batch(sender, grp, prio, typ, lens, off, pay)
    key = (grp.astype(np.int64) << 16) | (sender.astype(np.int64) << 3) | (typ & 7)
    last = np.zeros(len(key), bool)
    _, first_rev = np.unique(key[::-1], return_index=True)
    last[len(key) - 1 - first_rev] = True
    assert 0 < last.sum() < wl.S
    surv.send_group_seq(sender[last], grp[last], prio[last], typ[last], lens[last], off[last], pay,
                        base + wl.F * np.nonzero(last)[0].astype(np.uint64))
    cnt, total = g.supersede(None, archive=False)
    assert total == wl.F * int((~last).sum())
    qg, qs = g.queue_stats(), surv.queue_stats(wl.A)
    assert {k: qg[k] for k in ("pending", "pending_by_prio", "pending_granules", "agents_with_pending")} == \
        {k: qs[k] for k in ("pending", "pending_by_prio", "pending_granules", "agents_with_pending")}
    g.digest_reset(); surv.digest_enable()
    _, tot, _ = g.receive_batch(None, 100, copy_out=False)
    g.digest_fold()
    surv.receive_counts(None, 100)
    assert tot == wl.S * wl.F - total
    assert np.array_equal(g.digest_read(), surv.digest_read())
    g.close(); surv.close()


def test_swarmsdb_coordinator_gets_each_workers_newest_status_and_every_command(tmp_path):
    import swarmdb_b200 as sdb
    from swarmdb_b200 import MessageType
    db = sdb.SwarmsDB(save_dir=str(tmp_path), auto_save=False,
                      gpu_config=sdb.GpuConfig(max_agents=128, ring_slots=512, arena_bytes=1 << 24, max_payload_bytes=1024,
                                               deterministic_ids=True))
    db.register_agent("coord")
    workers = [f"w{i}" for i in range(64)]
    for w in workers:
        db.register_agent(w)
    ids = {}
    for v in range(4):
        for i, w in enumerate(workers):
            ids[w, v] = db.send_message(w, {"worker": w, "v": v}, "coord", message_type=MessageType.STATUS, supersede=True)
            if i % 16 == 0:
                db.send_message(w, f"cmd {w} {v}", "coord", message_type=MessageType.COMMAND)
        db.flush()
    assert db.get_stats()["superseded"] == 64 * 3
    assert db.get_unread_message_count("coord") == 64 + 16
    assert all(db.get_message(ids[w, v]).metadata["superseded_for"] == ["coord"] for w in workers for v in range(3))
    got = db.receive_messages("coord", max_messages=1000)
    status = sorted((m.content["worker"], m.content["v"]) for m in got if m.type == MessageType.STATUS)
    assert status == sorted((w, 3) for w in workers)
    assert sorted(m.content for m in got if m.type == MessageType.COMMAND) == \
        sorted(f"cmd {w} {v}" for v in range(4) for i, w in enumerate(workers) if i % 16 == 0)
    assert db.supersede_pending() == 0
    db.close()
