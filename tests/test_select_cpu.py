"""Filtered and leased receives by budget without a GPU: the composed take model of tests/select_ref.py, and the
front ends (SwarmsDB.receive_matching, receive_messages_leased, receive_batch_leased, ShardedSwarmsDB) on an
oracle-backed stand-in shard that answers the new calls as the header says the device does."""
import numpy as np
import pytest

from oracle.cpu_ref import HDR_DTYPE
from tests.fake_shard import OracleShard
from tests.select_ref import select, take
from tests.where_ref import RECV_PRIORITY

TOK = 0x40


# ---- the model ------------------------------------------------------------------------------------------------------
def test_take_is_the_shortest_of_the_three():
    recs = [(100, 5), (0, 0), (64, 9), (32, 1), (500, 2)]           # pad32: 128, 0, 64, 32, 512
    assert take(recs, 10, 0, 0) == 5
    assert take(recs, 2, 0, 0) == 2
    assert take(recs, 10, 192, 0) == 3                               # 128 + 0 + 64 met exactly
    assert take(recs, 10, 191, 0) == 2
    assert take(recs, 10, 0, 14) == 3                                # 5 + 0 + 9 met exactly
    assert take(recs, 10, 0, 13) == 2
    assert take(recs, 10, 224, 14) == 3 and take(recs, 10, 224, 100) == 4
    assert take(recs, 10, 1, 0) == 1 and take(recs, 10, 0, 1) == 1   # a heavier first alone
    assert take([], 10, 1, 1) == 0


def _rec(seq, prio, ln, typ=0, tokens=None, sender=0):
    h = np.zeros(1, HDR_DTYPE)[0]
    h["seq"], h["prio"], h["len"], h["type"], h["sender"] = seq, prio, ln, typ, sender
    body = (tokens.to_bytes(4, "little") if tokens is not None else b"") + bytes(ln)
    body = body[:ln] if tokens is None else body[:max(ln, 4)]
    return h, body + bytes((-len(body)) % 32)


def test_select_filters_orders_and_truncates():
    from swarmdb_b200._native import make_filter
    state = {0: [_rec(1, 0, 8, TOK, 3, sender=1), _rec(2, 3, 8, TOK, 4, sender=2), _rec(3, 2, 8, TOK, 5, sender=1),
                 _rec(4, 3, 8, TOK, 6, sender=1)],
             1: [_rec(5, 1, 40, TOK, 1, sender=1), _rec(6, 1, 40, TOK, 1, sender=1)]}
    f = make_filter(sender=1)
    assert select(state, [0, 1], 10, 0, 0, 0, f, 100) == ([3, 2], [(0, 0), (0, 2), (0, 3), (1, 0), (1, 1)])
    counts, chosen = select(state, [0, 1], 10, 0, 9, RECV_PRIORITY, f, 100)
    assert counts == [1, 2] and chosen[0] == (0, 3)                  # priority order: seq 4 (6 tokens) then 5 > 9
    assert select(state, [0, 1], 10, 0, 9, 0, f, 100)[0] == [2, 2]   # stream order: 3 + 5
    assert select(state, [0, 1], 10, 0, 0, 0, f, 4)[0] == [3, 0]     # a later agent that does not fit stays queued
    assert select(state, [0, 1], 10, 0, 0, 0, f, 2)[0] == [2, 0]     # the first agent gives its first rec_cap
    assert select(state, [1, 0], 10, 64, 0, 0, f, 100)[0] == [1, 2]  # bytes: 64 + 64 > 64 at agent 1; 32 + 32 fits at 0


# ---- the front ends on a stand-in shard ---------------------------------------------------------------------------
class SelectShard(OracleShard):
    """OracleShard with receive_where (limits included) answered by select_ref over the oracle's queues, and
    receive_leased answered from the same take with consecutive lease ids; every call is logged."""
    max_recv_records = 1 << 10

    def __init__(self, max_agents, max_groups, rank, world):
        from tests.where_ref import WhereOracle
        super().__init__(max_agents, max_groups, rank, world)
        self.o = WhereOracle(self.o, max_groups)
        self.calls = []
        self.next_lease = 100

    def send_batch(self, sender, receiver, prio, typ, lens, payload_off, payload, ts=None):
        return self.o.send_batch(sender, receiver, prio, typ, lens, payload_off, payload, ts)

    def receive_where(self, agents, max_messages, flags=0, filt=None, drop=False, max_agent_bytes=0,
                      max_agent_tokens=0, **kw):
        self.calls.append(("where", list(map(int, agents)), max_messages, flags, max_agent_bytes, max_agent_tokens))
        counts, _ = select(self.o.snapshot(), agents, max_messages, max_agent_bytes, max_agent_tokens, flags, filt,
                           1 << 20)
        hs, ps = [], []
        for a, k in zip(agents, counts):
            if k:
                _, h, p = self.o.receive_where([a], k, flags, filt)
                hs.append(h); ps.append(p)
        hdr = np.concatenate(hs) if hs else np.zeros(0, HDR_DTYPE)
        pay = np.concatenate(ps) if ps else np.zeros(0, np.uint8)
        return np.array(counts, np.uint32), hdr, pay

    def receive_leased(self, agents, max_messages, deadline, flags=0, max_agent_bytes=0, max_agent_tokens=0,
                       filt=None):
        from swarmdb_b200._native import ENTRY_DTYPE, SEND_DTYPE, make_filter
        self.calls.append(("leased", list(map(int, agents)), max_messages, flags, max_agent_bytes, max_agent_tokens,
                           filt is not None, deadline))
        cnt, hdr, pay = self.receive_where(agents, max_messages, flags, filt or make_filter(), False, max_agent_bytes,
                                           max_agent_tokens)
        self.calls.pop()
        ent, snd = np.zeros(len(hdr), ENTRY_DTYPE), np.zeros(len(hdr), SEND_DTYPE)
        ent["seq"], ent["send"], ent["receiver"] = hdr["seq"], np.arange(len(hdr)), hdr["receiver"]
        for f in ("timestamp", "sender", "group", "len", "prio", "type"):
            snd[f] = hdr[f]
        pl = (hdr["len"].astype(np.int64) + 31) & ~31
        if len(pl) > 1:
            snd["payload_off"][1:] = np.cumsum(pl)[:-1]
        base = self.next_lease
        self.next_lease += len(hdr)
        return cnt, ent, snd, pay, base

    def lease_deliveries(self, ids):
        return np.full(len(ids), 1, np.uint32)

    def lease_sweep(self, now, flags=0):
        return 0, 0, 0

    def lease_reserve(self, *a):
        pass

    def lease_set_policy(self, *a):
        pass


def _db(tmp_path, **kw):
    import swarmdb_b200 as sdb
    shard = SelectShard(64, 4, 0, 1)
    db = sdb.SwarmsDB(save_dir=str(tmp_path), auto_save=False, _shard=shard, token_counter=lambda t: int(t.split()[0]),
                      gpu_config=sdb.GpuConfig(max_agents=64, max_groups=4, deterministic_ids=True, **kw))
    for a in ("a", "b", "c"):
        db.register_agent(a)
    return db, shard


def _fill(db):
    from swarmdb_b200.core import MessageType
    ids = []
    for i, (snd, c) in enumerate([("a", "3 x"), ("c", "4 x"), ("a", "5 x"), ("a", "1 x"), ("c", "2 x"), ("a", "9 x")]):
        ids.append(db.send_message(snd, c, "b", message_type=MessageType.CHAT))
    db.flush()
    return ids


def test_receive_matching_with_limits_is_one_call(tmp_path):
    db, shard = _db(tmp_path)
    _fill(db)
    got = db.receive_matching("b", sender_id="a", max_tokens=8)
    assert [m.content for m in got] == ["3 x", "5 x"]
    assert shard.calls[-1][0] == "where" and shard.calls[-1][4:] == (0, 8)
    n = len(shard.calls)
    assert [m.content for m in db.receive_matching("b", sender_id="a", max_tokens=1)] == ["1 x"]   # heavier first alone
    assert len(shard.calls) == n + 1
    assert [m.content for m in db.receive_matching("b", sender_id="c", max_bytes=1)] == ["4 x"]
    assert shard.calls[-1][4:] == (1, 0)
    assert [m.content for m in db.receive_matching("b", max_messages=10)] == ["2 x", "9 x"]
    db.close()


def test_leased_matching_and_leased_limits_keep_the_bookkeeping(tmp_path):
    db, shard = _db(tmp_path, lease_records=64)
    ids = _fill(db)
    got = db.receive_matching("b", sender_id="a", max_tokens=8, leased=True, visibility_timeout=60.0)
    assert [m.id for m in got] == [ids[0], ids[2]]
    call = shard.calls[-1]
    assert call[0] == "leased" and call[4:7] == (0, 8, True)
    assert db._leases[ids[0]] == [(db.agent_index("b"), 100)] and db._leases[ids[2]] == [(db.agent_index("b"), 101)]
    assert db._lease_deadlines and all(m.metadata.get("delivery_count") is None for m in got)
    got = db.receive_messages_leased("b", max_bytes=64)
    assert [m.id for m in got] == [ids[1], ids[3]] and shard.calls[-1][4:7] == (64, 0, False)
    got = db.receive_matching("b", sender_id="c", leased=True)                                       # no limit: a loop
    assert [m.id for m in got] == [ids[4]] and shard.calls[-1][4:7] == (0, 0, True)
    db.close()


def test_delivery_counts_on_limited_leases(tmp_path):
    db, shard = _db(tmp_path, lease_records=64, lease_max_deliveries=3)
    _fill(db)
    got = db.receive_messages_leased("b", max_tokens=7)
    assert [m.content for m in got] == ["3 x", "4 x"] and [m.metadata["delivery_count"] for m in got] == [1, 1]
    db.close()


def test_receive_batch_leased_passes_limits_and_filter(tmp_path):
    from swarmdb_b200._native import make_filter
    db, shard = _db(tmp_path, lease_records=64)
    _fill(db)
    b = db.agent_index("b")
    cnt, ent, snd, pay, base = db.receive_batch_leased([b], 10, max_tokens=9, filt=make_filter(sender=db.agent_index("a")))
    assert cnt.tolist() == [3] and base == 100 and shard.calls[-1][4:7] == (0, 9, True)
    db.receive_batch_leased([b], 1)
    assert shard.calls[-1][4:7] == (0, 0, False)
    db.close()


@pytest.mark.parametrize("kw", [{"max_bytes": -1}, {"max_tokens": 0}, {"max_tokens": 1 << 64}, {"max_tokens": -3}])
def test_argument_checks(tmp_path, kw):
    db, shard = _db(tmp_path, lease_records=64)
    _fill(db)
    n = len(shard.calls)
    for call in (lambda: db.receive_matching("b", sender_id="a", **kw),
                 lambda: db.receive_matching("b", sender_id="a", leased=True, **kw),
                 lambda: db.receive_messages_leased("b", **kw),
                 lambda: db.receive_batch_leased(None, 4, **kw)):
        with pytest.raises(ValueError):
            call()
    assert len(shard.calls) == n
    db.close()


def test_sharded_front_end(tmp_path):
    import swarmdb_b200 as sdb
    from swarmdb_b200 import sharded

    class Ex:
        def __init__(self, *a): pass
        def close(self): pass
    shard = SelectShard(64, 4, 0, 1)
    db = sharded.ShardedSwarmsDB(0, 1, exchange_factory=Ex, shard=shard, save_dir=str(tmp_path), auto_save=False,
                                 gpu_config=sdb.GpuConfig(max_agents=64, max_groups=4, deterministic_ids=True),
                                 token_counter=lambda t: int(t.split()[0]))
    for a in ("a", "b"):
        db.register_agent(a)
    with pytest.raises(NotImplementedError):
        db.receive_matching("b", sender_id="a", leased=True)
    with pytest.raises(NotImplementedError):
        db.receive_matching("b", sender_id="a", max_tokens=5, leased=True)
    db.close()
