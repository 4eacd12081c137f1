"""CPU checks of retention (sdb_expire): the reference (tests/expire_ref.py) against oracles that never saw the expired
records, and the Python surface (SwarmsDB.expire_pending / flush_old_messages(include_device=True) /
deregister_agent(purge=True), the sharded front-end under gloo, the REST route) on the oracle-backed stand-in shard.
tests/test_gpu_expire.py runs the device."""
import json
import os
import socket
import time

import numpy as np
import pytest

from oracle.cpu_ref import CpuOracle
from swarmdb_b200 import _native
from swarmdb_b200._native import ENTRY_DTYPE, EXPIRE_ALL, RECV_OWNED, RECV_PEEK, RECV_PRIORITY, SEND_DTYPE
from tests.fake_shard import OracleShard


# ---- the reference: expiry equals a queue in which the expired records were never sent ---------------------------------
def _traffic(o, rng, A=24, G=4, k=40, keep=None):
    """p2p, group and broadcast sends with non-monotonic timestamps (some NaN), one send per call with the sequence
    number taken from a shared counter, so a second oracle can be fed a subset with the same numbers.  keep(ts) -> bool
    selects the sends the oracle receives (None: all).  Returns nothing; the same rng stream gives the same traffic."""
    seq = 1
    for _ in range(3):
        for kind in ("p2p", "group", "list"):
            for _ in range(k):
                ln = int(rng.integers(0, 97)); buf = rng.integers(0, 256, 160).astype(np.uint8)
                ts = float(rng.uniform(0.0, 100.0)) if rng.random() > 0.05 else float("nan")
                s, pr, ty = [int(rng.integers(0, A))], [int(rng.integers(0, 4))], [int(rng.integers(0, 7))]
                r, g = int(rng.integers(0, A)), int(rng.integers(0, G))
                lst = rng.choice(A, 3, replace=False)
                take = keep is None or keep(ts)
                o.next_seq = seq
                if kind == "p2p":
                    if take:
                        o.send_batch(s, [r], pr, ty, [ln], [0], buf, [ts])
                    seq += 1
                elif kind == "group":
                    if take:
                        o.send_group_batch(s, [g], pr, ty, [ln], [0], buf, [ts])
                    seq += 6
                else:
                    if take:
                        o.send_list_batch(s, [0, 3], lst, pr, ty, [ln], [0], buf, [ts])
                    seq += 1
    o.next_seq = seq


def _pair(A=24, G=4, keep=None, seed=5):
    from tests.expire_ref import ExpiringOracle
    out = []
    for kp in (None, keep):
        rng = np.random.default_rng(seed)
        o = CpuOracle(A, G)
        for g in range(G):
            o.create_group(g, np.random.default_rng(g).choice(A, 6, replace=False))
        o.register(np.arange(A))
        _traffic(o, rng, A, G, keep=kp)
        out.append(ExpiringOracle(o, G, {g: np.random.default_rng(g).choice(A, 6, replace=False) for g in range(G)}, A))
    return out


def _drain_equal(x, y, A):
    x.digest_enable(); y.digest_enable()
    for flags in (RECV_PRIORITY, 0, RECV_PRIORITY, 0):
        cx, hx, px = x.receive_batch(np.arange(A), 3, flags)
        cy, hy, py = y.receive_batch(np.arange(A), 3, flags)
        assert np.array_equal(cx, cy) and hx.tobytes() == hy.tobytes() and px.tobytes() == py.tobytes()
    assert np.array_equal(x.digest_read(), y.digest_read())


@pytest.mark.parametrize("cutoff", [50.0, 80.0, float("nan"), 1e9])
def test_expiry_equals_never_sent(cutoff):
    """Expire by timestamp over every agent: later receives, in both orders, equal those of an oracle that was only
    ever sent the survivors (NaN timestamps never expire); PEEK retires nothing; loads keep `received`."""
    A = 24
    full, survivors = _pair(A, keep=lambda ts: not ts < cutoff)
    loads0 = full.agent_loads(np.arange(A))
    pc, ph, pp = full.expire(None, cutoff, RECV_PEEK)
    cnt, hdr, pay = full.expire(None, cutoff)
    assert np.array_equal(pc, cnt) and ph.tobytes() == hdr.tobytes() and pp.tobytes() == pay.tobytes()
    assert not np.isnan(hdr["timestamp"]).any() and (hdr["timestamp"] < cutoff).all()
    ld, ls = full.agent_loads(np.arange(A)), survivors.agent_loads(np.arange(A))
    assert np.array_equal(ld["pending"], ls["pending"]) and np.array_equal(ld["received"], loads0["received"])
    assert np.array_equal(cnt[:A].astype(np.int64), loads0["pending"].astype(np.int64) - ls["pending"])
    _drain_equal(full, survivors, A)


def test_expire_all_capacity_and_agent_lists():
    """Purge of listed agents; a record capacity: repeated calls return, concatenated, exactly the uncapped result in
    order (a partial first agent included), and what did not fit stays queued."""
    A = 24
    a, b = _pair(A)
    agents = np.random.default_rng(1).permutation(A)[:17]
    want = b.expire(agents, 60.0)
    got_c, got_h, got_p = np.zeros(len(agents), np.int64), [], []
    while True:
        c, h, p = a.expire(agents, 60.0, 0, rec_cap=4)
        assert len(h) <= 4 and (len(h) == 0 or c[np.nonzero(c)[0][0]] > 0)
        got_c += c
        if len(h) == 0:
            break
        got_h.append(h.tobytes()); got_p.append(p.tobytes())
    assert np.array_equal(got_c, want[0]) and b"".join(got_h) == want[1].tobytes() and b"".join(got_p) == want[2].tobytes()
    first = a.expire(agents, 1e9, RECV_PEEK, rec_cap=2)[0]            # first agent with matches gives its first 2
    assert first.sum() == 2 and first[np.nonzero(first)[0][0]] == 2
    c, t = a.expire(agents[:5], 0.0, EXPIRE_ALL, materialise=False)
    b.expire(agents[:5], 0.0, EXPIRE_ALL)
    assert t == int(c.sum()) and a.agent_loads(agents[:5])["pending"].sum() == 0
    _drain_equal(a, b, A)


# ---- the surface, on an oracle-backed shard that also expires ----------------------------------------------------------
class ExpiringShard(OracleShard):
    """OracleShard + Shard.expire's surface: every call is logged; archive results come back in the compact format
    (one row per record, which expand_compact turns back into the full format)."""

    def __init__(self, max_agents, max_groups, rank, world):
        from tests.expire_ref import ExpiringOracle
        super().__init__(max_agents, max_groups, rank, world)
        self.o = ExpiringOracle(self.o, max_groups)
        self.expire_calls = []

    def send_batch(self, sender, receiver, prio, typ, lens, payload_off, payload, ts=None):
        return self.o.send_batch(sender, receiver, prio, typ, lens, payload_off, payload, ts)    # device-only traffic

    def expire(self, agents, older_than, flags=0, archive=True, **kw):
        self.expire_calls.append((None if agents is None else list(map(int, agents)), older_than, flags, archive))
        if agents is None and flags & RECV_OWNED:
            agents = np.nonzero(self.smap == self.rank)[0].astype(np.uint32)
        if not archive:
            return self.o.expire(agents, older_than, flags & ~RECV_OWNED, materialise=False)
        counts, hdr, pay = self.o.expire(agents, older_than, flags & ~RECV_OWNED, rec_cap=5)    # small calls: callers loop
        ent = np.zeros(len(hdr), ENTRY_DTYPE)
        snd = np.zeros(len(hdr), SEND_DTYPE)
        ent["seq"], ent["receiver"], ent["send"] = hdr["seq"], hdr["receiver"], np.arange(len(hdr))
        for f in ("timestamp", "sender", "group", "len", "prio", "type"):
            snd[f] = hdr[f]
        snd["payload_off"] = _native.payload_offsets(hdr)
        return counts, ent, snd, pay


def _db(tmp_path, **kw):
    import swarmdb_b200 as sdb
    shard = ExpiringShard(64, 8, 0, 1)
    db = sdb.SwarmsDB(save_dir=str(tmp_path), auto_save=False, _shard=shard,
                      gpu_config=sdb.GpuConfig(max_agents=64, max_groups=8, deterministic_ids=True), **kw)
    return db, shard


def _archives(tmp_path):
    d = tmp_path / "archives"
    return {} if not d.exists() else {k: v for p in sorted(d.glob("*.json")) for k, v in json.loads(p.read_text()).items()}


def test_default_flush_old_messages_makes_no_device_call(tmp_path):
    db, shard = _db(tmp_path)
    db.register_agents(["a", "b"])
    old = db.send_message("a", "old", "b"); db.messages[old].timestamp = 10.0
    new = db.send_message("a", "new", "b")
    assert db.flush_old_messages(100.0) == 1
    assert shard.expire_calls == []
    assert set(_archives(tmp_path)) == {old} and _archives(tmp_path)[old]["content"] == "old"
    assert old not in db.messages and new in db.messages
    assert [m.content for m in db.receive_messages("b")] == ["old", "new"]      # the device queue is untouched
    db.close()


def test_flush_old_messages_include_device_archives_device_only_messages(tmp_path):
    db, shard = _db(tmp_path)
    names = [f"a{i}" for i in range(6)]
    db.register_agents(names)
    db.add_agent_group("g", names[:4])
    idx = {n: db.agent_index(n) for n in names}
    # device-only traffic: bulk index-level sends, timestamps around the cutoff (0.0 when none is given)
    lens = np.array([3, 3, 3], np.uint16)
    off = np.array([0, 32, 64], np.uint64)
    buf = np.frombuffer(b"old" + bytes(29) + b"new" + bytes(29) + b"zer" + bytes(61), np.uint8)
    base = db.send_batch([idx["a0"]] * 3, [idx["a1"], idx["a2"], idx["a3"]], None, None, lens, off, buf, np.array([5.0, 500.0, 7.0]))
    db.send_batch([idx["a0"]], [idx["a4"]], None, None, lens[:1], off[:1], buf)           # timestamp 0.0
    host = db.send_message("a5", "host copy", "a1")
    db.messages[host].timestamp = 1.0
    grp = db.send_to_group("a0", "g", "group hello")
    for mid in grp:
        db.messages[mid].timestamp = 2.0
    bc = db.broadcast_message("a0", "to all", exclude_agents=["a5"])
    db.messages[bc].timestamp = 3.0
    db.flush()
    # a cutoff after every send: the device copies of the host messages (stamped at send time) go too
    n = db.flush_old_messages(time.time() + 3600, include_device=True)
    arch = _archives(tmp_path)
    want_ids = {db._make_id(base), db._make_id(base + 1), db._make_id(base + 2), db._make_id(base + 3), host, bc, *grp}
    assert set(arch) == want_ids and n == len(want_ids)                    # broadcast: one entry, not one per copy
    assert arch[host]["content"] == "host copy" and arch[host]["timestamp"] == 1.0         # host record wins
    assert arch[db._make_id(base)]["content"] == "old" and arch[db._make_id(base + 3)]["timestamp"] == 0.0
    assert bc not in db.messages and host not in db.messages                              # deleted as before
    assert set(arch[host]) == {"id", "sender_id", "receiver_id", "content", "type", "priority", "timestamp", "status",
                               "metadata", "token_count", "visible_to"}
    assert set(arch[db._make_id(base)]) == set(arch[host])
    assert all(shard.expire_calls[i][3] for i in range(len(shard.expire_calls)))          # archive mode, looped
    assert len(shard.expire_calls) >= 3 and db.shard.queue_stats()["pending"] == 0
    assert not any(db.receive_messages(a) for a in names)
    db.close()


def test_flush_include_device_keeps_newer_device_messages(tmp_path):
    db, shard = _db(tmp_path)
    db.register_agents(["a", "b"])
    ia, ib = db.agent_index("a"), db.agent_index("b")
    buf = np.frombuffer(b"x" * 64, np.uint8)
    db.send_batch([ia, ia], [ib, ib], None, None, np.array([1, 1], np.uint16), np.array([0, 32], np.uint64), buf,
                  np.array([10.0, 1000.0]))
    assert db.flush_old_messages(100.0, include_device=True) == 1
    assert [m.timestamp for m in db.receive_messages("b")] == [1000.0]
    db.close()


def test_expire_pending_defaults_to_retention_ms(tmp_path):
    import swarmdb_b200 as sdb
    db, shard = _db(tmp_path, config=sdb.KafkaConfig(retention_ms=60_000))
    db.register_agents(["a", "b", "c"])
    t0 = time.time()
    db.expire_pending()
    assert len(shard.expire_calls) == 1
    agents, cutoff, flags, archive = shard.expire_calls[0]
    assert agents is None and flags == 0 and archive is False
    assert t0 - 60.0 - 1.0 <= cutoff <= time.time() - 60.0
    ia, ib, ic = (db.agent_index(x) for x in "abc")
    buf = np.zeros(64, np.uint8)
    db.send_batch([ia] * 3, [ib, ib, ic], None, None, np.ones(3, np.uint16), np.array([0, 0, 0], np.uint64), buf,
                  np.array([t0 - 120.0, t0, t0 - 120.0]))
    assert db.expire_pending(agent_ids=["b", "b", "nobody"]) == 1                # repeats and unknown agents are dropped
    assert shard.expire_calls[-1][0] == [ib]
    assert db.expire_pending() == 1                                                # c's old record
    assert [m.timestamp for m in db.receive_messages("b")] == [t0]
    assert db.receive_messages("c") == []
    db.close()


def test_deregister_agent_purge(tmp_path):
    db, shard = _db(tmp_path)
    db.register_agents(["a", "b", "c"])
    for i in range(4):
        db.send_message("a", f"m{i}", "b")
        db.send_message("a", f"n{i}", "c")
    db.flush()
    db.deregister_agent("b")                                                       # default: queue kept
    assert shard.expire_calls == [] and db.shard.agent_loads([db.agent_index("b")])["pending"][0] == 4
    db.register_agent("b")
    db.deregister_agent("b", purge=True)
    assert shard.expire_calls[-1] == ([db.agent_index("b")], 0.0, EXPIRE_ALL, False)
    assert db.shard.agent_loads([db.agent_index("b")])["pending"][0] == 0
    assert [m.content for m in db.receive_messages("c")] == ["n0", "n1", "n2", "n3"]
    db.close()


def test_flush_route_takes_include_device(tmp_path):
    pytest.importorskip("fastapi"); pytest.importorskip("jwt"); pytest.importorskip("httpx")
    from fastapi.testclient import TestClient
    from swarmdb_b200.server import Settings, create_app
    db, shard = _db(tmp_path)
    c = TestClient(create_app(db, Settings(history_dir=str(tmp_path))))
    adm = {"Authorization": "Bearer " + c.post("/auth/token", json={"username": "admin", "password": "pw"}).json()["access_token"]}
    db.register_agents(["a", "b"])
    ia, ib = db.agent_index("a"), db.agent_index("b")
    db.send_batch([ia], [ib], None, None, np.ones(1, np.uint16), np.zeros(1, np.uint64), np.zeros(64, np.uint8), np.array([1.0]))
    r = c.post("/admin/flush", params={"older_than": 100.0}, headers=adm)
    assert r.json() == {"status": "success", "flushed_count": 0} and shard.expire_calls == []
    r = c.post("/admin/flush", params={"older_than": 100.0, "include_device": True}, headers=adm)
    assert r.json() == {"status": "success", "flushed_count": 1} and shard.expire_calls
    assert db.receive_messages("b") == []
    db.close()


# ---- sharded front-end: each rank expires what it owns, no collective -------------------------------------------------
AGENTS = [f"agent{i}" for i in range(16)]


def _sharded_worker(rank, world, port, q, tmp):
    import torch.distributed as dist
    from swarmdb_b200 import sharded
    from swarmdb_b200.core import GpuConfig
    from tests.test_sharded_cpu import CpuBackend
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        cfg = GpuConfig(max_agents=64, max_groups=8, flush_threshold=64, max_payload_bytes=256, deterministic_ids=True)
        shard = ExpiringShard(64, 8, rank, world)
        db = sharded.make_sharded_swarmsdb(
            rank, world, shard=shard,
            exchange_factory=lambda sh, r, w, ms, mp: sharded.ShardExchange(sh, r, w, ms, mp, CpuBackend()),
            save_dir=f"{tmp}/r{rank}", auto_save=False, gpu_config=cfg)
        db.register_agents(AGENTS)
        db.add_agent_group("all", AGENTS)
        mine = [a for a in AGENTS if db.owner(a) == rank]
        for i in range(3):
            db.send_to_group(AGENTS[rank], "all", f"r{rank}-{i}")
        db.flush()                                                    # collective
        res = {"owned_scope": shard.expire_calls == []}
        # LOCAL from here on: ranks make different numbers of calls, which would hang a collective
        if rank == 0:
            n_exp = db.expire_pending(older_than=time.time() + 60, agent_ids=AGENTS[:4])
            res["n_exp"] = n_exp
            res["listed"] = sorted(shard.expire_calls[-1][0]) == sorted(db.agent_index(a) for a in AGENTS[:4] if db.owner(a) == 0)
        n_arch = db.flush_old_messages(time.time() + 60, include_device=True)
        res["flags_owned"] = all(c[2] & RECV_OWNED for c in shard.expire_calls if c[0] is None)
        res["pending_left"] = int(shard.o.queue_stats()["pending"])
        res["n_arch"] = n_arch
        res["arch_ids"] = sorted(_archives(__import__("pathlib").Path(f"{tmp}/r{rank}")))
        res["mine"] = mine
        # purge on the owner only: deregistration is replicated
        victim = AGENTS[5]
        before = len(shard.expire_calls)
        db.deregister_agent(victim, purge=True)
        res["purge_calls"] = len(shard.expire_calls) - before
        res["owner_of_victim"] = db.owner(victim)
        dist.barrier()
        q.put((rank, res))
        db.close()
    finally:
        dist.destroy_process_group()


def test_sharded_frontend_expires_owned_agents_only(tmp_path):
    import torch.multiprocessing as mp
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_sharded_worker, args=(r, 2, port, q, str(tmp_path))) for r in range(2)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=240) for _ in procs)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for r in (0, 1):
        assert res[r]["owned_scope"] and res[r]["flags_owned"] and res[r]["pending_left"] == 0, res[r]
        assert res[r]["purge_calls"] == (1 if res[r]["owner_of_victim"] == r else 0)
    assert res[0]["listed"]
    # every group send reaches 15 members; each rank archives the ids of the records its own agents held
    assert res[0]["n_arch"] + res[0]["n_exp"] > 0 and res[1]["n_arch"] > 0
    assert set(res[0]["arch_ids"]) | set(res[1]["arch_ids"]) and len(res[0]["arch_ids"]) == res[0]["n_arch"]
