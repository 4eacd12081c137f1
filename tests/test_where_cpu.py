"""CPU checks of the filtered receive (sdb_receive_where): the ctypes struct against the C header, the record predicate
against brute force, the reference (tests/where_ref.py) against oracles that were only ever sent the surviving records,
and the Python surface (receive_matching, the include_device queries, delete_message, the REST parameter) on an
oracle-backed stand-in shard.  tests/test_gpu_where.py runs the device."""
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

from oracle.cpu_ref import HDR_DTYPE, CpuOracle
from swarmdb_b200._native import NO_GROUP, NO_RECEIVER, RECV_OWNED, RECV_PEEK, RECV_PRIORITY, SdbFilter, make_filter
from tests.fake_shard import OracleShard
from tests.where_ref import content_bytes, fold_ascii, where_match

ROOT = Path(__file__).resolve().parents[1]

LAYOUT_C = r"""
#include <stddef.h>
#include <stdio.h>
#include "swarmdb_b200.h"
#define F(m) printf(#m " %zu %zu\n", offsetof(sdb_filter, m), sizeof(((sdb_filter*)0)->m))
int main(void) {
  printf("size %zu\n", sizeof(sdb_filter));
  F(struct_bytes); F(fields); F(sender); F(receiver); F(group); F(type_mask); F(prio_mask); F(keyword_len);
  F(after); F(before); F(seq_lo); F(seq_hi); F(keyword);
  printf("consts %u %u %u %u %u %u %u %u %u %u %u %d\n", SDB_FILTER_SENDER, SDB_FILTER_RECEIVER, SDB_FILTER_GROUP,
         SDB_FILTER_TYPE, SDB_FILTER_PRIO, SDB_FILTER_TIME, SDB_FILTER_SEQ, SDB_FILTER_KEYWORD, SDB_FILTER_ICASE,
         SDB_FILTER_MAX_KEYWORD, SDB_WHERE_DROP, (int)SDB_PK_WHERE);
  return 0;
}
"""


def test_filter_struct_matches_the_c_header(tmp_path):
    import ctypes
    from swarmdb_b200 import _native as n
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text(LAYOUT_C)
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", f"-I{ROOT / 'include'}",
                           str(src), "-o", str(exe)])
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split("\n")
    assert out[0] == f"size {ctypes.sizeof(SdbFilter)}"
    for line in out[1:14]:
        name, off, size = line.split()
        f = getattr(SdbFilter, name)
        assert (f.offset, f.size) == (int(off), int(size)), name
    consts = [int(x) for x in out[14].split()[1:]]
    assert consts == [n.FILTER_SENDER, n.FILTER_RECEIVER, n.FILTER_GROUP, n.FILTER_TYPE, n.FILTER_PRIO, n.FILTER_TIME,
                      n.FILTER_SEQ, n.FILTER_KEYWORD, n.FILTER_ICASE, n.FILTER_MAX_KEYWORD, n.WHERE_DROP,
                      n.Shard.PROFILE_KINDS.index("where")]


def _hdr(**kw):
    h = np.zeros(1, HDR_DTYPE)[0]
    base = dict(seq=10, timestamp=5.0, sender=1, receiver=2, group=NO_GROUP, len=0, prio=1, type=0)
    base.update(kw)
    for k, v in base.items():
        h[k] = v
    return h


def _rec(body: bytes, extras: bool = False, clen=None, **kw):
    if extras:
        body = np.uint32(len(body) if clen is None else clen).tobytes() + body
    h = _hdr(len=len(body), type=0x10 if extras else 0, **kw)
    return h, body + bytes((-len(body)) % 32)


def test_where_match_against_brute_force():
    rng = np.random.default_rng(0)
    alpha = b"abAB\xc3\xa9\xc3\x89 "
    for _ in range(3000):
        n = int(rng.integers(0, 40))
        body = bytes(rng.choice(list(alpha), n).astype(np.uint8))
        extras = bool(rng.random() < 0.4)
        clen = None if rng.random() < 0.5 else int(rng.integers(0, 60))
        h, p = _rec(body, extras, clen)
        k = int(rng.integers(0, 4))
        kw = bytes(rng.choice(list(alpha), k).astype(np.uint8))
        icase = bool(rng.random() < 0.5)
        # brute force: every start position of the content slice, byte by byte
        ln = int(h["len"])
        if extras:
            cont = b"" if ln < 4 else p[4:4 + min(int.from_bytes(p[:4], "little"), ln - 4)]
        else:
            cont = p[:ln]
        f = (lambda c: c + 32 if 65 <= c <= 90 else c) if icase else (lambda c: c)
        want = any(all(f(cont[s + i]) == f(kw[i]) for i in range(k)) for s in range(len(cont) - k + 1))
        assert where_match(h, p, make_filter(keyword=kw, icase=icase)) == want, (body, kw, icase, extras, clen)
    # EXTRAS: a keyword in the extras, one across the boundary, a bogus clen, len < 4
    assert not where_match(*_rec(b"abc" + b"{\"m\": 1}", True, 3), make_filter(keyword=b"m"))
    assert not where_match(*_rec(b"abcNee" + b"dle", True, 6), make_filter(keyword=b"Needle"))
    assert where_match(*_rec(b"xNeedle", True, 1 << 31), make_filter(keyword=b"Needle"))
    h, p = _hdr(len=3, type=0x10), b"Nee" + bytes(29)
    assert not where_match(h, p, make_filter(keyword=b"N")) and where_match(h, p, make_filter(keyword=b""))
    assert content_bytes(*_rec(b"hello", True, 2)) == b"he"
    assert fold_ascii("ÉA".encode()) == "Éa".encode()


def test_header_clauses():
    h = _hdr(seq=100, timestamp=5.0, sender=3, receiver=NO_RECEIVER, group=7, prio=2, type=0x08 | 4)
    p = bytes(32)
    assert where_match(h, p, make_filter())
    assert where_match(h, p, make_filter(sender=3, receiver=NO_RECEIVER, group=7, types=[4], prios=[2, 3],
                                         after=4.0, before=6.0, seq=(100, 101)))
    for f in (make_filter(sender=4), make_filter(receiver=3), make_filter(group=NO_GROUP), make_filter(types=[0]),
              make_filter(prios=[0, 1, 3]), make_filter(after=5.0), make_filter(before=5.0), make_filter(seq=(101, 200)),
              make_filter(seq=(0, 100))):
        assert not where_match(h, p, f)
    assert not where_match(_hdr(timestamp=float("nan")), p, make_filter(after=float("-inf")))


# ---- the reference against oracles that were only ever sent the surviving records ----------------------------------
def _traffic(o, rng, A=24, G=4, keep=None):
    """p2p, group and broadcast sends, one per call with the sequence number from a shared counter, so a second oracle
    can be fed a subset with the same numbers.  keep(header fields) -> bool selects the sends the oracle receives."""
    seq = 1
    for _ in range(2):
        for kind in ("p2p", "group", "list"):
            for _ in range(30):
                ln = int(rng.integers(0, 60))
                buf = rng.choice(list(b"abcAB"), 96).astype(np.uint8)
                ts = float(rng.uniform(0.0, 10.0))
                s, pr, ty = int(rng.integers(0, A)), int(rng.integers(0, 4)), int(rng.integers(0, 7))
                r, g = int(rng.integers(0, A)), int(rng.integers(0, G))
                lst = rng.choice(A, 3, replace=False)
                take = keep is None or keep(dict(sender=s, prio=pr, type=ty, ts=ts, body=buf[:ln].tobytes(),
                                                 group=g if kind == "group" else NO_GROUP))
                o.next_seq = seq
                if kind == "p2p":
                    if take:
                        o.send_batch([s], [r], [pr], [ty], [ln], [0], buf, [ts])
                    seq += 1
                elif kind == "group":
                    if take:
                        o.send_group_batch([s], [g], [pr], [ty], [ln], [0], buf, [ts])
                    seq += 6
                else:
                    if take:
                        o.send_list_batch([s], [0, 3], lst, [pr], [ty], [ln], [0], buf, [ts])
                    seq += 1
    o.next_seq = seq


def _pair(keep, A=24, G=4, seed=5):
    from tests.where_ref import WhereOracle
    out = []
    for kp in (None, keep):
        rng = np.random.default_rng(seed)
        o = CpuOracle(A, G)
        for g in range(G):
            o.create_group(g, np.random.default_rng(g).choice(A, 6, replace=False))
        o.register(np.arange(A))
        _traffic(o, rng, A, G, keep=kp)
        out.append(WhereOracle(o, G, {g: np.random.default_rng(g).choice(A, 6, replace=False) for g in range(G)}, A))
    return out


def _drain_equal(x, y, A):
    for flags in (RECV_PRIORITY, 0, RECV_PRIORITY, 0):
        cx, hx, px = x.receive_batch(np.arange(A), 3, flags)
        cy, hy, py = y.receive_batch(np.arange(A), 3, flags)
        assert np.array_equal(cx, cy) and hx.tobytes() == hy.tobytes() and px.tobytes() == py.tobytes()


@pytest.mark.parametrize("case", ["sender", "group_prio", "keyword", "time_types"])
@pytest.mark.parametrize("flags", [0, RECV_PRIORITY])
def test_taking_every_match_equals_never_sent(case, flags):
    """Taking (and dropping) every match leaves the queue of an oracle that never saw them; PEEK retires nothing;
    `delivered` counts taken records, not dropped ones."""
    filt, keep = {
        "sender": (make_filter(sender=3), lambda d: d["sender"] != 3),
        "group_prio": (make_filter(group=2, prios=[1, 3]), lambda d: not (d["group"] == 2 and d["prio"] in (1, 3))),
        "keyword": (make_filter(keyword=b"aB", icase=True), lambda d: b"ab" not in fold_ascii(d["body"])),
        "time_types": (make_filter(after=2.0, before=6.0, types=[1, 2, 6]),
                       lambda d: not (2.0 < d["ts"] < 6.0 and d["type"] in (1, 2, 6))),
    }[case]
    A = 24
    for drop in (False, True):
        full, surv = _pair(keep)
        loads0 = full.agent_loads(np.arange(A))
        peek = full.receive_where(np.arange(A), 1 << 20, RECV_PEEK | flags, filt)
        got = full.receive_where(np.arange(A), 1 << 20, flags, filt, drop=drop)
        assert np.array_equal(peek[0], got[0])
        if not drop:
            assert peek[1].tobytes() == got[1].tobytes() and peek[2].tobytes() == got[2].tobytes()
            assert full.delivered == len(got[1]) > 0
        else:
            assert full.delivered == 0 and got[1] == int(peek[0].sum()) > 0
        ld, ls = full.agent_loads(np.arange(A)), surv.agent_loads(np.arange(A))
        assert np.array_equal(ld["pending"], ls["pending"]) and np.array_equal(ld["received"], loads0["received"])
        _drain_equal(full, surv, A)


def test_max_messages_order_and_capacity():
    """Priority order is priority-descending, stream order within a level; max_messages per agent; the capacity cut
    leaves whole agents queued except a lead agent; repeated calls return the uncapped result in order."""
    full, _ = _pair(lambda d: True)
    agents = np.random.default_rng(1).permutation(24)
    filt = make_filter(prios=[0, 2, 3])
    c, h, _ = full.receive_where(agents, 4, RECV_PEEK | RECV_PRIORITY, filt)
    pos = 0
    for k in c:
        seg = h[pos:pos + int(k)]
        assert len(seg) <= 4 and list(seg["prio"]) == sorted(seg["prio"], reverse=True)
        pos += int(k)
    want = full.receive_where(agents, 1 << 20, RECV_PEEK, filt)
    got_c, hs = np.zeros(len(agents), np.int64), []
    while True:
        c, h, _ = full.receive_where(agents, 1 << 20, 0, filt, rec_cap=5)
        assert len(h) <= 5
        if len(h) == 0:
            break
        assert c[np.nonzero(c)[0][0]] > 0
        got_c += c; hs.append(h.tobytes())
    assert np.array_equal(got_c, want[0]) and b"".join(hs) == want[1].tobytes()


# ---- the surface, on an oracle-backed shard that also takes filtered receives ------------------------------------------
class WhereShard(OracleShard):
    """OracleShard + Shard.receive_where with a small record capacity per call (callers loop; the front end is given
    the same capacity through GpuConfig.max_recv_records); every call is logged."""

    def __init__(self, max_agents, max_groups, rank, world, rec_cap=8):
        from tests.where_ref import WhereOracle
        super().__init__(max_agents, max_groups, rank, world)
        self.o = WhereOracle(self.o, max_groups)
        self.where_calls = []
        self.rec_cap = rec_cap

    def send_batch(self, sender, receiver, prio, typ, lens, payload_off, payload, ts=None):
        return self.o.send_batch(sender, receiver, prio, typ, lens, payload_off, payload, ts)    # device-only traffic

    def receive_where(self, agents, max_messages, flags=0, filt=None, drop=False, **kw):
        self.where_calls.append((None if agents is None else list(map(int, agents)), max_messages, flags, drop))
        if agents is None and flags & RECV_OWNED:
            agents = np.nonzero(self.smap == self.rank)[0].astype(np.uint32)
        return self.o.receive_where(agents, max_messages, flags & ~RECV_OWNED, filt or make_filter(), rec_cap=self.rec_cap, drop=drop)


def _db(tmp_path, rec_cap=8, **kw):
    import swarmdb_b200 as sdb
    shard = WhereShard(64, 8, 0, 1, rec_cap)
    db = sdb.SwarmsDB(save_dir=str(tmp_path), auto_save=False, _shard=shard,
                      gpu_config=sdb.GpuConfig(max_agents=64, max_groups=8, deterministic_ids=True, max_recv_records=rec_cap,
                                               max_payload_bytes=256, max_recv_payload=rec_cap * 256), **kw)
    return db, shard


def _bulk(db, sender, receivers, bodies, ts=None, prio=None, typ=None):
    n = len(bodies)
    buf = b"".join(b + bytes((-len(b)) % 32) for b in bodies) + bytes(32)
    off = np.cumsum([0] + [len(b) + (-len(b)) % 32 for b in bodies[:-1]]).astype(np.uint64)
    return db.send_batch([db.agent_index(sender)] * n, [db.agent_index(r) for r in receivers], prio, typ,
                         np.array([len(b) for b in bodies], np.uint16), off, np.frombuffer(buf, np.uint8), ts)


def test_receive_matching_takes_only_the_matches(tmp_path):
    from swarmdb_b200.core import MessagePriority, MessageType
    db, shard = _db(tmp_path)
    db.register_agents(["a", "b", "coord"])
    db.add_agent_group("g", ["a", "b", "coord"])
    db.send_message("a", "chat one", "b")
    db.send_message("coord", "do it", "b", message_type=MessageType.COMMAND, priority=MessagePriority.HIGH)
    db.send_message("a", "chat two", "b", priority=MessagePriority.CRITICAL)
    db.send_message("coord", {"op": "Stop"}, "b", message_type=MessageType.COMMAND)
    db.send_to_group("a", "g", "group note")
    got = db.receive_matching("b", message_type=MessageType.COMMAND)
    assert [m.content for m in got] == ["do it", {"op": "Stop"}] and all(db.messages[m.id].status.value == "read" for m in got)
    assert [m.content for m in db.receive_matching("b", min_priority=MessagePriority.CRITICAL)] == ["chat two"]
    assert db.receive_matching("b", sender_id="nobody") == [] and db.receive_matching("b", group_name="nope") == []
    assert [m.content for m in db.receive_matching("b", keyword="GROUP")] == ["group note"]
    assert [m.content for m in db.receive_messages("b")] == ["chat one"]          # the rest stayed queued, in order
    with pytest.raises(ValueError):
        db.receive_matching("b", keyword="x" * 257)
    db.close()


def test_include_device_queries(tmp_path):
    db, shard = _db(tmp_path)
    db.register_agents(["a", "b", "c"])
    base = _bulk(db, "a", ["b", "c", "b"], [b"alpha Kw", b"beta", b"gamma kw"], ts=np.array([1.0, 2.0, 3.0]))
    host = db.send_message("a", "host kw", "b")
    bc = db.broadcast_message("c", "to all KW")
    db.messages.pop(bc)                                                         # device-only broadcast: one message
    db.flush()
    ids = [db._make_id(base + i) for i in range(3)]
    assert db.query_messages(sender_id="a") == [db.messages[host]]               # default: host records only
    q = db.query_messages(sender_id="a", include_device=True)
    assert [m.id for m in q] == [host, ids[2], ids[1], ids[0]]                  # host first, then newest device-only
    assert [m.id for m in db.query_messages(sender_id="a", include_device=True, limit=2)] == [host, ids[2]]
    assert [m.id for m in db.query_messages(receiver_id="b", include_device=True)] == [host, ids[2], ids[0]]
    assert db.query_messages(status="read", include_device=True) == []
    assert [m.id for m in db.query_messages(after_timestamp=1.5, before_timestamp=2.5, include_device=True)] == [ids[1]]
    s = db.search_messages("kw", include_device=True)
    assert [m.id for m in s] == [host, bc, ids[2], ids[0]]                      # the broadcast once, not per copy
    assert [m.id for m in db.search_messages("Kw", case_sensitive=True, include_device=True)] == [ids[0]]
    long_kw = "alpha Kw" + "z" * 300
    assert db.search_messages(long_kw, include_device=True) == []               # truncated on the device, then checked
    conv = db.get_conversation("a", "b", include_device=True)
    assert [m.id for m in conv] == [host, ids[2], ids[0]]
    assert not any(c[3] for c in shard.where_calls) and all(c[2] & RECV_PEEK for c in shard.where_calls)
    db.close()


def test_delete_message_include_device(tmp_path):
    db, shard = _db(tmp_path)
    db.register_agents(["a", "b", "c"])
    base = _bulk(db, "a", ["b", "b"], [b"one", b"two"])
    bc = db.broadcast_message("a", "everyone")
    db.flush()
    assert db.delete_message(db._make_id(base)) is False                        # default: host records only
    assert db.delete_message(db._make_id(base), include_device=True) is True
    assert db.delete_message(bc, include_device=True) is True                  # host record and every device copy
    assert db.delete_message("not-an-id", include_device=True) is False
    assert db.delete_message("00000000-0000-0001-0000-000000000005", include_device=True) is False   # not our id
    assert [m.content for m in db.receive_messages("b")] == ["two"]
    assert db.receive_messages("c") == []
    db.close()


def test_messages_route_takes_include_device(tmp_path):
    pytest.importorskip("fastapi"); pytest.importorskip("jwt"); pytest.importorskip("httpx")
    from fastapi.testclient import TestClient
    from swarmdb_b200.server import Settings, create_app
    db, shard = _db(tmp_path)
    c = TestClient(create_app(db, Settings(history_dir=str(tmp_path))))
    adm = {"Authorization": "Bearer " + c.post("/auth/token", json={"username": "admin", "password": "pw"}).json()["access_token"]}
    db.register_agents(["a", "b"])
    _bulk(db, "a", ["b"], [b"device only"])
    assert c.get("/messages", headers=adm).json() == [] and shard.where_calls == []
    r = c.get("/messages", params={"include_device": True}, headers=adm).json()
    assert [m["content"] for m in r] == ["device only"]
    # a caller that is not admin reads its own device queue only
    tok = lambda u: {"Authorization": "Bearer " + c.post("/auth/token", json={"username": u, "password": "pw"}).json()["access_token"]}
    assert c.get("/messages", params={"include_device": True}, headers=tok("a")).status_code == 403
    assert c.get("/messages", params={"include_device": True, "receiver_id": "a"}, headers=tok("b")).status_code == 403
    r = c.get("/messages", params={"include_device": True, "receiver_id": "b"}, headers=tok("b")).json()
    assert [m["content"] for m in r] == ["device only"]
    db.close()


def test_device_queries_decode_only_what_they_return(tmp_path, monkeypatch):
    """include_device queries decode each call's records newest first and stop at `limit` taken ones; the result is
    the same as ranking every match."""
    import swarmdb_b200.core as core
    db, shard = _db(tmp_path, rec_cap=64)
    db.register_agents(["a", "b", "c"])
    base = _bulk(db, "a", ["b", "c"] * 40, [b"kw %d" % i for i in range(80)])
    decoded = []
    real = core.SwarmsDB._decode
    monkeypatch.setattr(core.SwarmsDB, "_decode", lambda self, hdr, *a, **k: decoded.append(len(hdr)) or real(self, hdr, *a, **k))
    got = db.search_messages("KW", limit=5, include_device=True)
    assert [m.id for m in got] == [db._make_id(base + i) for i in range(79, 74, -1)]
    assert sum(decoded) <= 2 * 5 * max(1, len(shard.where_calls))
    got = db.query_messages(receiver_id="b", limit=3, include_device=True)
    assert [m.content for m in got] == ["kw 78", "kw 76", "kw 74"]
    db.close()


# ---- sharded front-end: each rank reads and takes from what it owns, no collective ---------------------------------------
AGENTS = [f"agent{i}" for i in range(16)]


def _sharded_worker(rank, world, port, q, tmp):
    import os
    import torch.distributed as dist
    from swarmdb_b200 import sharded
    from swarmdb_b200.core import GpuConfig, MessageType
    from tests.test_sharded_cpu import CpuBackend
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        cfg = GpuConfig(max_agents=64, max_groups=8, flush_threshold=64, max_payload_bytes=256, deterministic_ids=True,
                        max_recv_records=8, max_recv_payload=8 * 256)
        shard = WhereShard(64, 8, rank, world, 8)
        db = sharded.make_sharded_swarmsdb(
            rank, world, shard=shard,
            exchange_factory=lambda sh, r, w, ms, mp: sharded.ShardExchange(sh, r, w, ms, mp, CpuBackend()),
            save_dir=f"{tmp}/r{rank}", auto_save=False, gpu_config=cfg)
        db.register_agents(AGENTS)
        db.add_agent_group("all", AGENTS)
        sent = {}
        for i in range(3):
            sent[i] = db.send_to_group(AGENTS[rank], "all", f"r{rank}-{i}")
        db.send_message(AGENTS[rank], f"cmd from r{rank}", AGENTS[8 + rank], message_type=MessageType.COMMAND)
        db.flush()                                                    # collective
        res = {"no_calls_yet": shard.where_calls == []}
        mine = [a for a in AGENTS if db.owner(a) == rank]
        theirs = [a for a in AGENTS if db.owner(a) != rank]
        owned_idx = {db.agent_index(a) for a in mine}
        other = 1 - rank
        # LOCAL from here on: the ranks make different numbers of calls, which would hang a collective
        for _ in range(1 + 2 * rank):
            hits = db.search_messages(f"r{other}-", include_device=True, limit=1000)
        res["search_other"] = sorted({m.content for m in hits})
        res["search_ids_unique"] = len({m.id for m in hits}) == len(hits)
        q_theirs = db.query_messages(receiver_id=theirs[0], include_device=True)
        res["theirs_no_device_call"] = all(c[0] is None or set(c[0]) <= owned_idx for c in shard.where_calls)
        res["theirs_host_only"] = all(m.id in db.messages for m in q_theirs)
        a = next(x for x in mine if x not in (AGENTS[0], AGENTS[1], AGENTS[8], AGENTS[9]))    # receives group sends only
        conv = db.get_conversation(AGENTS[other], a, include_device=True)
        res["conv"] = sorted(m.content for m in conv)                 # device-only: the other rank's sends to `a`
        res["conv_want"] = [f"r{other}-{i}" for i in range(3)]
        try:
            db.receive_matching(a, sender=AGENTS[other])              # a misspelled clause is refused, nothing taken
            res["typo_refused"] = False
        except TypeError:
            res["typo_refused"] = True
        got = db.receive_matching(a, sender_id=AGENTS[other], keyword="-1")
        res["took"] = [m.content for m in got]
        try:
            db.receive_matching(theirs[0])
            res["non_owner_refused"] = False
        except ValueError:
            res["non_owner_refused"] = True
        n_before = len(shard.where_calls)
        mid = next(m for m in sent[2] if db.messages[m].receiver_id == a)          # a group send: one id per member
        res["deleted"] = db.delete_message(mid, include_device=True)
        res["delete_call"] = shard.where_calls[n_before:] == [(None, 1, RECV_OWNED, True)]
        left = [m.content for m in db.receive_messages(a, 100)]
        res["left"] = left
        res["where_owned_only"] = all(c[0] is None or set(c[0]) <= owned_idx for c in shard.where_calls)
        res["calls"] = len(shard.where_calls)
        dist.barrier()
        q.put((rank, res))
        db.close()
    finally:
        dist.destroy_process_group()


def test_sharded_frontend_reads_and_takes_owned_agents_only(tmp_path):
    import socket
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
        x = res[r]
        assert x["no_calls_yet"] and x["search_ids_unique"] and x["theirs_no_device_call"] and x["theirs_host_only"], x
        assert x["search_other"] == [f"r{1 - r}-{i}" for i in range(3)], x
        assert x["conv"] == x["conv_want"], x
        assert x["typo_refused"] and x["non_owner_refused"] and x["took"] == [f"r{1 - r}-1"], x
        assert x["deleted"] and x["delete_call"] and x["where_owned_only"], x
        # what stayed queued, in order: the other rank's group sends except the one taken, and this rank's own
        # sends except the deleted one
        assert sorted(x["left"]) == sorted([f"r{1 - r}-0", f"r{1 - r}-2", f"r{r}-0", f"r{r}-1"]), x
    assert res[0]["calls"] != res[1]["calls"]                         # different numbers of calls: no collective
