"""Superseding sends (sdb_supersede) without a GPU: the model of tests/supersede_ref.py on hand-written queues, then
SwarmsDB's automatic pass, host records, requeue, argument checks, the sharded refusals and the REST fields, against an
oracle-backed shard that can supersede and restore."""
import numpy as np
import pytest

from oracle.cpu_ref import HDR_DTYPE
from tests.fake_shard import OracleShard
from tests.restore_ref import restore_append
from tests.supersede_ref import TYPEF_SUPERSEDE, SupersedingOracle, supersede_drops, supersede_select

F = TYPEF_SUPERSEDE
NG = 0xFFFFFFFF


def _queue(*recs):
    """[(header, payload)] in ring order from (seq, sender, group, type) tuples."""
    out = []
    for seq, snd, grp, typ in recs:
        h = np.zeros(1, HDR_DTYPE)[0]
        h["seq"], h["sender"], h["group"], h["type"], h["len"] = seq, snd, grp, typ, 8
        out.append((h, bytes(32)))
    return out


def test_key_fields():
    q = _queue((1, 5, NG, F | 2), (2, 6, NG, F | 2), (3, 5, 7, F | 2), (4, 5, NG, F | 3), (5, 5, NG, F | 2 | 0x08),
               (6, 5, 7, F | 2 | 0x10), (7, 6, NG, F | 2))
    # (5, NG, 2): seqs 1 and 5 (the JSON bit is not part of the key); (6, NG, 2): 2 and 7; (5, 7, 2): 3 and 6
    assert supersede_drops(q) == [0, 1, 2]


def test_unflagged_records_are_untouched():
    q = _queue((1, 5, NG, 2), (2, 5, NG, F | 2), (3, 5, NG, 2), (4, 5, NG, F | 2), (5, 5, NG, 2))
    assert supersede_drops(q) == [1]
    assert supersede_drops(_queue((1, 5, NG, 2), (2, 5, NG, 2))) == []
    assert supersede_drops([]) == []


def test_seq_order_not_ring_order():
    # a stale version put back behind newer ones (a sweep, redrive or requeue) is the one that goes
    q = _queue((10, 5, NG, F | 1), (12, 5, NG, F | 1), (4, 5, NG, F | 1), (11, 5, NG, F | 1))
    assert supersede_drops(q) == [0, 2, 3]


def test_seq_tie_goes_to_the_later_record():
    q = _queue((7, 5, NG, F | 1), (3, 5, NG, F | 1), (7, 5, NG, F | 1))
    assert supersede_drops(q) == [0, 1]


def test_capacity_rule_and_ring_order_output():
    state = {0: _queue(*[(s, 1, NG, F | 1) for s in range(8)]),          # 7 superseded
             1: _queue(*[(s, 2, NG, F | 1) for s in range(3)]),          # 2
             2: _queue((1, 3, NG, F | 1), (2, 3, NG, F | 1))}            # 1
    counts, chosen = supersede_select(state, [0, 1, 2], 0, 5)
    assert counts == [5, 0, 0] and chosen == [(0, i) for i in range(5)]
    counts, chosen = supersede_select(state, [1, 0, 2], 0, 4)
    assert counts == [2, 0, 0] and chosen == [(1, 0), (1, 1)]           # agent 0's 7 do not fit behind agent 1's 2
    counts, chosen = supersede_select(state, [2, 1, 0, 9], 0, 100)
    assert counts == [1, 2, 7, 0]


@pytest.mark.parametrize("seed", range(6))
def test_archive_calls_until_empty_equal_one_drop_call(seed):
    rng = np.random.default_rng(seed)
    state = {a: _queue(*[(int(rng.integers(0, 40)), int(rng.integers(0, 4)), int(rng.choice([NG, 1, 2])),
                          int(rng.integers(0, 8)) | (F if rng.random() < 0.7 else 0))
                         for _ in range(int(rng.integers(0, 30)))]) for a in range(12)}
    agents = rng.permutation(12)
    _, once = supersede_select(state, agents, 0, 1 << 60)
    left = {a: list(enumerate(q)) for a, q in state.items()}          # (original position, record)
    taken = set()
    for _ in range(1000):
        cur = {a: [r for _, r in lst] for a, lst in left.items()}
        _, chosen = supersede_select(cur, agents, 0, int(rng.integers(1, 8)))
        if not chosen:
            break
        gone = set(chosen)
        for a, i in chosen:
            taken.add((a, left[a][i][0]))
        left = {a: [x for i, x in enumerate(lst) if (a, i) not in gone] for a, lst in left.items()}
    assert taken == set(once)


def _compact(hdr, pay):
    """The compact format of full-format records, one row per record."""
    from swarmdb_b200._native import ENTRY_DTYPE, SEND_DTYPE
    ent, snd = np.zeros(len(hdr), ENTRY_DTYPE), np.zeros(len(hdr), SEND_DTYPE)
    ent["seq"], ent["send"], ent["receiver"] = hdr["seq"], np.arange(len(hdr)), hdr["receiver"]
    for f in ("timestamp", "sender", "group", "len", "prio", "type"):
        snd[f] = hdr[f]
    pad = (hdr["len"].astype(np.int64) + 31) & ~31
    snd["payload_off"] = np.concatenate([[0], np.cumsum(pad)])[:-1]
    return ent, snd, np.asarray(pay, np.uint8)


class SupersedeShard(OracleShard):
    """The oracle-backed stand-in shard with superseding (tests/supersede_ref.py) and restore (tests/restore_ref.py);
    it counts its supersede calls."""

    def __init__(self, max_agents, max_groups, rank, world, rec_cap=1 << 40):
        super().__init__(max_agents, max_groups, rank, world)
        self.o = SupersedingOracle(self.o, max_groups, watermark=max_agents)
        self.rec_cap, self.calls = rec_cap, []

    def supersede(self, agents, flags=0, archive=True, **kw):
        self.calls.append(None if agents is None else sorted(np.asarray(agents).tolist()))
        if not archive:
            return self.o.supersede(agents, flags, materialise=False)
        cnt, hdr, pay = self.o.supersede(agents, flags, rec_cap=self.rec_cap)
        return (cnt,) + _compact(hdr, pay)

    def trim(self, agents, max_records=0, max_bytes=0, flags=0, archive=True, **kw):
        assert not archive
        return self.o.trim(agents, max_records, max_bytes, flags, materialise=False)

    def restore_compact(self, agents, counts, entries, sends, payload, flags=0):
        n = restore_append(self.o, self.groups, agents, counts, entries, sends, payload)
        return n, self.o.next_seq

    def send_batch(self, sender, receiver, prio, typ, lens, payload_off, payload, ts=None):
        return self.o.send_batch(sender, receiver, prio, typ, lens, payload_off, payload, ts)

    def peek_all(self, agent):
        return self.o.receive_batch([agent], 1000, 2)[1]


def _db(tmp_path, **kw):
    import swarmdb_b200 as sdb
    shard = SupersedeShard(64, 4, 0, 1, rec_cap=kw.pop("rec_cap", 1 << 40))
    db = sdb.SwarmsDB(save_dir=str(tmp_path), auto_save=False, _shard=shard,
                      gpu_config=sdb.GpuConfig(max_agents=64, max_groups=4, deterministic_ids=True, **kw))
    return db, shard


def test_flush_keeps_each_workers_newest_status_and_every_command(tmp_path):
    from swarmdb_b200 import MessageType
    db, shard = _db(tmp_path, rec_cap=3)                              # several archive calls per pass
    db.register_agent("coord")
    workers = [f"w{i}" for i in range(4)]
    ids = {}
    for v in range(3):
        for w in workers:
            ids[w, v] = db.send_message(w, f"{w} v{v}", "coord", message_type=MessageType.STATUS, supersede=True)
        db.send_message("w0", f"cmd{v}", "coord", message_type=MessageType.COMMAND)
        db.flush()
    assert shard.calls[-1] == [db.agent_index("coord")]             # only the receivers of the batch
    assert db.get_stats()["superseded"] == 8
    assert db.get_unread_message_count("coord") == 4 + 3
    for w in workers:
        for v in range(2):
            m = db.get_message(ids[w, v])
            assert m.metadata["superseded_for"] == ["coord"] and m.id not in db.agent_inbox["coord"]
        assert "superseded_for" not in db.get_message(ids[w, 2]).metadata
    got = [m.content for m in db.receive_messages("coord")]
    assert sorted(got) == sorted([f"{w} v2" for w in workers] + ["cmd0", "cmd1", "cmd2"])
    n = len(shard.calls)
    db.send_message("w0", "plain", "coord")
    db.flush()
    assert len(shard.calls) == n                                      # a flush without a superseding send: no pass
    db.close()


def test_the_pass_runs_before_the_queue_caps(tmp_path):
    db, shard = _db(tmp_path, queue_max_messages=2)
    db.register_agent("b")
    for i in range(3):
        db.send_message("a", f"s{i}", "b", supersede=True)
    db.send_message("a", "c0", "b")
    db.flush()
    # the pass leaves s2 and c0: within the cap, so the caps trim nothing
    st = db.get_stats()
    assert st["superseded"] == 2 and st["trimmed"] == 0
    assert [m.content for m in db.receive_messages("b")] == ["s2", "c0"]
    db.close()


def test_group_and_broadcast_copies(tmp_path):
    db, shard = _db(tmp_path)
    for a in ("a", "b", "c", "d"):
        db.register_agent(a)
    db.add_agent_group("g", ["a", "b", "c"])
    old = db.send_to_group("a", "g", "v0", supersede=True)
    new = db.send_to_group("a", "g", "v1", supersede=True)
    db.flush()
    assert sorted(shard.calls[-1]) == sorted(db.agent_index(x) for x in ("b", "c"))   # members minus the sender
    for mid in old:
        m = db.get_message(mid)
        assert m.metadata["superseded_for"] == [m.receiver_id]
    assert all("superseded_for" not in db.get_message(mid).metadata for mid in new)
    b0 = db.broadcast_message("a", "p0", supersede=True)
    b1 = db.broadcast_message("a", "p1", supersede=True)
    db.flush()
    assert sorted(db.get_message(b0).metadata["superseded_for"]) == ["b", "c", "d"]
    assert "superseded_for" not in db.get_message(b1).metadata
    assert db.get_stats()["superseded"] == 2 + 3
    for x in ("b", "c", "d"):
        assert b0 not in db.agent_inbox[x] and b1 in db.agent_inbox[x]
    db.close()


def test_requeue_puts_a_stale_version_back_and_the_pass_retires_it(tmp_path):
    db, shard = _db(tmp_path)
    db.register_agent("b")
    v0 = db.send_message("a", "v0", "b", supersede=True)
    db.flush()
    hdr = shard.peek_all(db.agent_index("b"))
    cnt = np.array([len(hdr)], np.uint32)
    assert [m.content for m in db.receive_messages("b")] == ["v0"]
    db.send_message("a", "v1", "b", supersede=True)
    db.flush()
    before = db.get_stats()["superseded"]
    assert db.requeue_batch_compact(cnt, *_compact(hdr, np.zeros(64, np.uint8)), np.array([db.agent_index("b")], np.uint32)) == 1
    assert db.get_stats()["superseded"] == before + 1                # v0 went back behind v1, and is the one that goes
    assert db.get_message(v0).metadata["superseded_for"] == ["b"]
    assert [m.content for m in db.receive_messages("b")] == ["v1"]
    db.close()


def test_supersede_pending_and_index_level_sends(tmp_path):
    from swarmdb_b200._native import TYPEF_SUPERSEDE as T
    db, shard = _db(tmp_path)
    for a in ("a", "b", "c"):
        db.register_agent(a)
    lens, off = np.full(3, 4, np.uint16), np.arange(3, dtype=np.uint64) * 32
    buf = np.frombuffer(b"abcd".ljust(32, b"\0") * 3 + bytes(32), np.uint8)
    b, c = db.agent_index("b"), db.agent_index("c")
    db.send_batch([0, 0, 0], [b, b, c], None, [T | 1, T | 1, 1], lens, off, buf)
    assert shard.calls[-1] == [b]                                    # receivers of the flagged sends only
    assert db.get_stats()["superseded"] == 1
    assert db.supersede_pending() == 0 and db.supersede_pending(["nobody"]) == 0
    db.close()


def test_argument_checks_come_before_any_device_call(tmp_path):
    db, shard = _db(tmp_path)

    class NoDevice:
        def __getattr__(self, name):
            raise AssertionError(f"device call {name} before the arguments were checked")
    db.shard = NoDevice()
    for bad in (1, "yes", None):
        with pytest.raises(TypeError):
            db.send_message("a", "x", "b", supersede=bad)
        with pytest.raises(TypeError):
            db.broadcast_message("a", "x", supersede=bad)
        with pytest.raises(TypeError):
            db.send_to_group("a", "g", "x", supersede=bad)


def test_sharded_front_end_refuses():
    from swarmdb_b200.sharded import ShardedSwarmsDB
    db = ShardedSwarmsDB.__new__(ShardedSwarmsDB)              # the per-call refusals come before any state is read
    with pytest.raises(NotImplementedError, match="supersede"):
        db.send_message("a", "x", "b", supersede=True)
    with pytest.raises(NotImplementedError, match="supersede"):
        db.send_to_group("a", "g", "x", supersede=True)
    with pytest.raises(NotImplementedError, match="supersede"):
        db.broadcast_message("a", "x", supersede=True)
    with pytest.raises(NotImplementedError, match="supersede"):
        db.supersede_pending()


def test_rest_send_routes_take_supersede(tmp_path):
    pytest.importorskip("fastapi"); pytest.importorskip("jwt"); pytest.importorskip("httpx")
    from fastapi.testclient import TestClient
    from swarmdb_b200.server import Settings, create_app
    db, shard = _db(tmp_path)
    c = TestClient(create_app(db, Settings(history_dir=str(tmp_path))))
    r = c.post("/auth/token", json={"username": "a1", "password": "pw"})
    hd = {"Authorization": f"Bearer {r.json()['access_token']}"}
    for who in ("a1", "a2", "a3"):
        db.register_agent(who)
    db.add_agent_group("g", ["a1", "a2"])
    for i in range(3):
        assert c.post("/messages", json={"content": f"s{i}", "receiver_id": "a2", "supersede": True}, headers=hd).status_code == 200
    assert c.post("/messages", json={"content": "plain", "receiver_id": "a2"}, headers=hd).status_code == 200
    assert c.post("/messages/broadcast", json={"content": "b0", "supersede": True}, headers=hd).status_code == 200
    assert c.post("/messages/broadcast", json={"content": "b1", "supersede": True}, headers=hd).status_code == 200
    assert c.post("/groups/message", json={"group_name": "g", "content": "g0", "supersede": True}, headers=hd).status_code == 200
    assert c.post("/groups/message", json={"group_name": "g", "content": "g1", "supersede": True}, headers=hd).status_code == 200
    db.flush()
    # point-to-point sends and broadcast copies of one sender and type share a key: b1 supersedes s2 too
    assert sorted(m.content for m in db.receive_messages("a2")) == ["b1", "g1", "plain"]
    assert [m.content for m in db.receive_messages("a3")] == ["b1"]
    assert db.get_stats()["superseded"] == 3 + 2 + 1
    db.close()
