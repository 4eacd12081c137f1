"""CPU checks of the id clause of the filtered receive (SDB_FILTER_IDS): the ctypes struct against the C header, the
reference (tests/ids_ref.py) on hand-made queues, and the Python surface (get_message / get_messages with
include_device, delete_messages, receive_matching(message_ids=)) on an oracle-backed stand-in shard.
tests/test_gpu_ids.py runs the device."""
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

from oracle.cpu_ref import CpuOracle
from swarmdb_b200._native import NO_RECEIVER, RECV_OWNED, RECV_PEEK, RECV_PRIORITY, SdbFilter, make_filter
from tests.fake_shard import OracleShard
from tests.ids_ref import F_IDS, IdsOracle, ids_of
from tests.test_where_cpu import _bulk

ROOT = Path(__file__).resolve().parents[1]

LAYOUT_C = r"""
#include <stddef.h>
#include <stdio.h>
#include "swarmdb_b200.h"
#define F(m) printf(#m " %zu %zu\n", offsetof(sdb_filter, m), sizeof(((sdb_filter*)0)->m))
int main(void) {
  printf("size %zu\n", sizeof(sdb_filter));
  F(keyword); F(n_ids); F(ids); F(id_hits); F(id_agent);
  printf("consts %u %u\n", SDB_FILTER_IDS, SDB_FILTER_MAX_IDS);
  return 0;
}
"""


def test_id_block_matches_the_c_header(tmp_path):
    from swarmdb_b200 import _native as n
    import ctypes
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text(LAYOUT_C)
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", f"-I{ROOT / 'include'}",
                           str(src), "-o", str(exe)])
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split("\n")
    assert out[0] == f"size {ctypes.sizeof(SdbFilter)}"
    for line in out[1:6]:
        name, off, size = line.split()
        f = getattr(SdbFilter, name)
        assert (f.offset, f.size) == (int(off), int(size)), name
    assert [int(x) for x in out[6].split()[1:]] == [n.FILTER_IDS, n.FILTER_MAX_IDS]
    assert SdbFilter.n_ids.offset == 64                          # the struct_bytes older callers pass


def test_make_filter_ids():
    f = make_filter(ids=[7, 3, 7, 0])
    assert f.fields == F_IDS and f.n_ids == 4 and ids_of(f).tolist() == [7, 3, 7, 0]
    a = np.array([1 << 40, 5], np.uint64)
    f = make_filter(ids=a, sender=2)
    assert f.fields == F_IDS | 1 and ids_of(f).tolist() == [1 << 40, 5]
    f = make_filter(ids=[])
    assert f.fields == F_IDS and f.n_ids == 0 and f.ids                 # an empty set still points somewhere
    with pytest.raises(ValueError):
        make_filter(ids=np.zeros((2, 2), np.uint64))


def _queue():
    """8 agents; p2p (seqs 1..12), a group send to 4 members (13..16 in one send: one seq per copy), a broadcast list
    to every agent (one seq shared by its 8 copies)."""
    A, G = 8, 2
    o = CpuOracle(A, G)
    o.create_group(0, [1, 3, 5, 6])
    o.register(np.arange(A))
    rng = np.random.default_rng(3)
    n = 12
    lens = rng.integers(1, 40, n).astype(np.uint16)
    buf = rng.choice(np.frombuffer(b"abcXYZ ", np.uint8), n * 64 + 64).astype(np.uint8)
    o.send_batch(rng.integers(0, A, n), rng.integers(0, A, n), rng.integers(0, 4, n), rng.integers(0, 7, n), lens,
                 np.arange(n, dtype=np.uint64) * 64, buf, rng.uniform(0, 10, n))
    o.send_group_batch([2], [0], [3], [1], [20], [0], buf, [4.0])
    o.send_list_batch([4], [0, A], np.arange(A, dtype=np.uint32), [2], [0], [30], [64], buf, [6.0])
    return IdsOracle(o, G, {0: np.array([1, 3, 5, 6])}, A), A


def test_one_id_equals_the_seq_range():
    """The id clause with one id selects exactly what SDB_FILTER_SEQ [s, s + 1) selects, in both orders and modes."""
    for s in range(0, 20):
        for flags in (RECV_PEEK, RECV_PEEK | RECV_PRIORITY):
            x, A = _queue()
            a = x.receive_where(None, 100, flags, make_filter(ids=[s]))
            b = x.receive_where(None, 100, flags, make_filter(seq=(s, s + 1)))
            assert np.array_equal(a[0], b[0]) and a[1].tobytes() == b[1].tobytes() and a[2].tobytes() == b[2].tobytes()
        x, A = _queue()
        y, _ = _queue()
        assert x.receive_where(None, 100, 0, make_filter(ids=[s]), drop=True)[1] == \
            y.receive_where(None, 100, 0, make_filter(seq=(s, s + 1)), drop=True)[1]
        assert x.snapshot().keys() == y.snapshot().keys()
        for a in x.snapshot():
            assert [h.tobytes() for h, _ in x.snapshot()[a]] == [h.tobytes() for h, _ in y.snapshot()[a]]


def test_id_outputs_duplicates_absent_and_zero():
    x, A = _queue()
    st = x.snapshot()
    where = {}
    for a, recs in st.items():
        for h, _ in recs:
            where.setdefault(int(h["seq"]), []).append(a)
    bc = max(where, key=lambda s: len(where[s]))                    # the broadcast: one seq at every agent
    assert len(where[bc]) == A
    p2p = min(where)
    ids = [bc, p2p, 999, 0, p2p, bc]
    hits, first = np.zeros(len(ids), np.uint32), np.zeros(len(ids), np.uint32)
    c, total = x.receive_where(None, 100, RECV_PEEK, make_filter(ids=ids), drop=True, id_hits=hits, id_agent=first)
    assert hits.tolist() == [A, len(where[p2p]), 0, 0, len(where[p2p]), A]
    assert first.tolist() == [0, min(where[p2p]), NO_RECEIVER, NO_RECEIVER, min(where[p2p]), 0]
    assert total == A + len(where[p2p])
    # counted before max_messages, over the listed agents only, with every other clause applied
    sub = np.array([5, 2], np.uint32)
    x.receive_where(sub, 1, RECV_PEEK, make_filter(ids=ids, prios=[2]), drop=True, id_hits=hits, id_agent=first)
    assert hits.tolist()[0] == 2 and first.tolist()[0] == 2
    x.receive_where(sub, 1, RECV_PEEK, make_filter(ids=ids, prios=[1]), drop=True, id_hits=hits, id_agent=first)
    assert hits.tolist()[0] == 0 and first.tolist()[0] == NO_RECEIVER
    # keyword: the broadcast's content decides for every copy at once
    pay = st[0][[int(h["seq"]) for h, _ in st[0]].index(bc)][1]
    for kw, want in ((pay[:3], A), (b"\x01\x02\x03", 0)):
        x.receive_where(None, 100, RECV_PEEK, make_filter(ids=ids, keyword=kw), drop=True, id_hits=hits)
        assert hits.tolist()[0] == want
    # an empty set matches nothing; then a drop of the broadcast leaves everything else
    assert x.receive_where(None, 100, RECV_PEEK, make_filter(ids=[]), drop=True)[1] == 0
    before = sum(len(v) for v in x.snapshot().values())
    assert x.receive_where(None, 100, 0, make_filter(ids=[bc, bc]), drop=True)[1] == A
    assert sum(len(v) for v in x.snapshot().values()) == before - A


# ---- the surface, on an oracle-backed shard that also takes the id clause ----------------------------------------------
class IdsShard(OracleShard):
    """OracleShard + Shard.receive_where with the id clause and its outputs; every call is logged."""

    def __init__(self, max_agents, max_groups, rank=0, world=1):
        super().__init__(max_agents, max_groups, rank, world)
        self.o = IdsOracle(self.o, max_groups)
        self.where_calls = []

    def send_batch(self, sender, receiver, prio, typ, lens, payload_off, payload, ts=None):
        return self.o.send_batch(sender, receiver, prio, typ, lens, payload_off, payload, ts)

    def receive_where(self, agents, max_messages, flags=0, filt=None, drop=False, id_hits=None, id_agent=None, **kw):
        self.where_calls.append((None if agents is None else list(map(int, agents)), max_messages, flags, drop,
                                 int(filt.fields) if filt is not None else 0))
        if agents is None and flags & RECV_OWNED:
            agents = np.nonzero(self.smap == self.rank)[0].astype(np.uint32)
        return self.o.receive_where(agents, max_messages, flags & ~RECV_OWNED, filt or make_filter(), drop=drop,
                                    id_hits=id_hits, id_agent=id_agent)


def _db(tmp_path):
    import swarmdb_b200 as sdb
    shard = IdsShard(64, 8)
    db = sdb.SwarmsDB(save_dir=str(tmp_path), auto_save=False, _shard=shard,
                      gpu_config=sdb.GpuConfig(max_agents=64, max_groups=8, deterministic_ids=True, max_recv_records=8,
                                               max_payload_bytes=256, max_recv_payload=8 * 256))
    return db, shard


def test_get_message_and_get_messages_include_device(tmp_path):
    db, shard = _db(tmp_path)
    db.register_agents(["a", "b", "c"])
    base = _bulk(db, "a", ["b", "c", "b"], [b"one", b"two", b"three"])
    bc = db.broadcast_message("a", "everyone")
    host = db.send_message("c", "host", receiver_id="b")
    db.flush()
    ids = [db._make_id(base + k) for k in range(3)]
    assert db.get_message(ids[1]) is None and shard.where_calls == []                 # default: host records only
    m = db.get_message(ids[1], include_device=True)
    assert m.content == "two" and m.receiver_id == "c" and m.status.value == "delivered"
    # one counting call over every agent (PEEK | DROP with the id clause), then a PEEK of the holder only
    assert shard.where_calls[0][0] is None and shard.where_calls[0][2] & RECV_PEEK and shard.where_calls[0][3]
    assert shard.where_calls[1][0] == [db.agent_index("c")] and not shard.where_calls[1][3]
    assert all(c[4] & F_IDS for c in shard.where_calls)
    got = db.get_messages([ids[2], "nope", host, ids[0], ids[2], db._make_id(999)], include_device=True)
    assert [None if x is None else x.content for x in got] == ["three", None, "host", "one", "three", None]
    assert got[2] is db.messages[host]                                                 # a host record wins
    assert db.get_messages([ids[0]]) == [None]
    assert db.get_message(bc, include_device=True) is db.messages[bc]
    db.messages.pop(bc)
    b = db.get_message(bc, include_device=True)
    assert b.content == "everyone" and b.receiver_id is None
    assert db.shard.agent_loads([0, 1, 2])["pending"].tolist() == [0, 4, 2]            # nothing consumed
    db.close()


def test_delete_messages_and_receive_matching_ids(tmp_path, monkeypatch):
    from swarmdb_b200 import core
    db, shard = _db(tmp_path)
    db.register_agents(["a", "b", "c"])
    base = _bulk(db, "a", ["b", "c", "b", "b"], [b"one", b"two", b"three", b"four"])
    bc = db.broadcast_message("a", "everyone")
    db.flush()
    ids = [db._make_id(base + k) for k in range(4)]
    n0 = len(shard.where_calls)
    assert db.delete_messages([ids[0], "x", bc, ids[1], ids[0]], include_device=True) == [True, False, True, True, True]
    assert len(shard.where_calls) == n0 + 1 and shard.where_calls[-1][3]                # one drop for every id
    assert db.messages.get(bc) is None
    assert db.delete_messages([ids[0], bc]) == [False, False]
    got = db.receive_matching("b", message_ids=[ids[3], ids[1], "junk"])
    assert [m.content for m in got] == ["four"] and ids[3] in db.messages
    assert db.receive_matching("b", message_ids=["junk"]) == []
    assert [m.content for m in db.receive_messages("b")] == ["three"]
    monkeypatch.setattr(core, "FILTER_MAX_IDS", 2)
    with pytest.raises(ValueError):
        db.receive_matching("b", message_ids=ids[:3])
    with pytest.raises(ValueError):
        db.delete_messages(ids[:3], include_device=True)
    with pytest.raises(ValueError):
        db.get_messages(ids[:3], include_device=True)
    db.close()


def test_messages_route_takes_include_device(tmp_path):
    pytest.importorskip("fastapi"); pytest.importorskip("jwt"); pytest.importorskip("httpx")
    from fastapi.testclient import TestClient
    from swarmdb_b200.server import Settings, create_app
    db, shard = _db(tmp_path)
    c = TestClient(create_app(db, Settings(history_dir=str(tmp_path))))
    tok = lambda u: {"Authorization": "Bearer " + c.post("/auth/token", json={"username": u, "password": "pw"}).json()["access_token"]}
    db.register_agents(["a", "b", "c"])
    mid = db._make_id(_bulk(db, "a", ["b"], [b"device only"]))
    assert c.get(f"/messages/{mid}", headers=tok("b")).status_code == 404
    r = c.get(f"/messages/{mid}", params={"include_device": True}, headers=tok("b"))
    assert r.status_code == 200 and r.json()["content"] == "device only"
    assert c.get(f"/messages/{mid}", params={"include_device": True}, headers=tok("admin")).status_code == 200
    db.close()
