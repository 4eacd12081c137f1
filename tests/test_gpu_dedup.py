"""Deduplicated sends on the device against tests/dedup_ref.py: verdicts, keys, sequence numbers and the queues the
accepted sends leave, byte for byte against the queue oracle, on mixed batches of point-to-point, group, list and
empty-list sends."""
import numpy as np
import pytest

from tests.dedup_ref import DedupModel, batch_seqs, content_key, replay

A, G, F = 256, 8, 16


def send_keys(b) -> list:
    """Content key of every send of a batch dict (the fields send_mixed_batch_dedup takes)."""
    out = []
    for i in range(len(b["sender"])):
        k, t, o, ln = int(b["kind"][i]), int(b["target"][i]), int(b["payload_off"][i]), int(b["lens"][i])
        rec = b["list_idx"][int(b["list_off"][t]):int(b["list_off"][t + 1])] if k == 2 else None
        out.append(content_key(int(b["sender"][i]), k, t, None if rec is None else [int(x) for x in rec], ln,
                               int(b["prio"][i]), int(b["typ"][i]), bytes(b["payload"][o:o + ln])))
    return out


class Rig:
    def __init__(self, seed, entries=4096, window=100.0, ring_slots=256, arena_bytes=1 << 24, **kw):
        from oracle.cpu_ref import CpuOracle
        from swarmdb_b200._native import Shard
        self.rng = np.random.default_rng(seed)
        self.g = Shard(max_agents=A, max_groups=G, ring_slots=ring_slots, arena_bytes=arena_bytes, **kw)
        self.o = CpuOracle(A, G)
        self.g.register(np.arange(A)); self.o.register(np.arange(A))    # sends name agents beyond their recipients
        self.sizes = {}
        for g in range(G):
            m = np.arange(g * F, (g + 1) * F, dtype=np.uint32)
            self.g.create_group(g, m); self.o.create_group(g, m)
            self.sizes[g] = F
        self.g.dedup_reserve(entries, window)
        self.m = DedupModel(entries, window)

    def close(self):
        self.g.close(); self.o.close()

    def batch(self, n, kinds=(0, 1, 2), max_len=120):
        rng = self.rng
        kind = rng.choice(kinds, n).astype(np.uint8)
        n_lists = max(1, n // 4)
        lists = [rng.choice(A, size=int(rng.integers(0, 12)), replace=False) for _ in range(n_lists)]
        list_off = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.uint64)
        list_idx = np.concatenate(lists).astype(np.uint32) if list_off[-1] else np.zeros(0, np.uint32)
        target = np.where(kind == 0, rng.integers(0, A, n), np.where(kind == 1, rng.integers(0, G, n),
                                                                      rng.integers(0, n_lists, n))).astype(np.uint32)
        lens = rng.integers(0, max_len + 1, n).astype(np.uint16)
        off = (np.arange(n, dtype=np.uint64) * 128)
        payload = rng.integers(0, 256, n * 128 + 64).astype(np.uint8)
        return dict(sender=rng.integers(0, A, n).astype(np.uint32), kind=kind, target=target, list_off=list_off,
                    list_idx=list_idx, prio=rng.integers(0, 4, n).astype(np.uint8), typ=rng.integers(0, 7, n).astype(np.uint8),
                    lens=lens, payload_off=off, payload=payload, ts=rng.random(n) * 100)

    def send(self, b, keys=None, content=False, now=0.0):
        """One deduplicated call on the device and the model; the accepted sends go into the oracle."""
        n = len(b["sender"])
        kin = [(0, 0)] * n if keys is None else [tuple(int(x) for x in k) for k in keys]
        want_keys = send_keys(b) if content else None
        used = [wk if k == (0, 0) else k for k, wk in zip(kin, want_keys)] if content else kin
        seq = batch_seqs(self.o.next_seq, b["kind"], b["target"], self.sizes)
        dup, n_new = self.m.send(used, seq, now)
        base, got_dup, got_keys = self.g.send_mixed_batch_dedup(
            b["sender"], b["kind"], b["target"], b["list_off"], b["list_idx"], b["prio"], b["typ"], b["lens"],
            b["payload_off"], b["payload"], b["ts"], keys=None if keys is None else np.asarray(kin, np.uint64),
            content=content, now=now)
        assert base == seq[0]
        assert got_dup.tolist() == dup
        assert list(zip(got_keys["lo"].tolist(), got_keys["hi"].tolist())) == used
        self.m.commit(used, seq, dup, n_new, now)
        end = seq[-1] + (self.sizes[int(b["target"][-1])] if int(b["kind"][-1]) == 1 else 1)
        replay(self.o, b["kind"], b["sender"], b["target"], b["list_off"], b["list_idx"], b["prio"], b["typ"],
               b["lens"], b["payload_off"], b["payload"], b["ts"], seq, [d == 0 for d in dup], end)
        return dup

    def check(self, drain=False, leased=False):
        """Every receive path against the oracle: PEEKs of the full, compact and byte-budget receives in both orders,
        or a drain (plain, or leased and acked)."""
        from swarmdb_b200._native import RECV_PEEK, RECV_PRIORITY, expand_compact

        def same(cg, hg, pg, flags):
            cc, hc, pc = self.o.receive_batch(None, 1 << 16, flags)
            assert np.array_equal(cg, cc[:len(cg)]) and not cc[len(cg):].any()
            assert hg.tobytes() == hc.tobytes() and pg.tobytes() == pc.tobytes()
        if drain and leased:
            cg, ent, snd, pay, base = self.g.receive_leased(None, 1 << 16, 1e18)
            same(cg, *expand_compact(ent, snd, pay), 0)
            self.g.lease_settle(np.arange(base, base + len(ent), dtype=np.uint64), 0)
        elif drain:
            same(*self.g.receive_batch(None, 1 << 16, 0), 0)
        else:
            for order in (0, RECV_PRIORITY):
                flags = RECV_PEEK | order
                cg, ent, snd, pay = self.g.receive_compact(None, 1 << 16, flags)
                same(cg, *expand_compact(ent, snd, pay), flags)
                same(*self.g.receive_budget(None, 1 << 16, 0, flags), flags)
                same(*self.g.receive_batch(None, 1 << 16, flags), flags)
        lg, lc = self.g.agent_loads(None, A), self.o.agent_loads(None, A)
        assert lg.tobytes() == lc.tobytes()
        st = self.g.stats()
        assert st["next_seq"] == self.o.next_seq
        ds = self.g.dedup_stats()
        ms = self.m.stats()
        for k in ("live", "used", "accepted_total", "duplicate_total", "expired_total", "forgotten_total", "rebuilds"):
            assert ds[k] == ms[k], k


def _queue_stats(g) -> dict:
    """sdb_stats without the launch counter (a refused call still launched its probe)."""
    return {k: v for k, v in g.stats().items() if k != "kernel_launches"}


def _keys(rng, n, pool):
    k = rng.integers(1, pool + 1, n).astype(np.uint64)
    k[rng.random(n) < 0.2] = 0                                   # some sends bypass the table
    return np.stack([k, k * np.uint64(3)], 1)


@pytest.mark.gpu
def test_mixed_batches_with_explicit_keys_match_the_model():
    # a mixed batch writes its group sends with a private payload per record (the shared-payload layout is taken by
    # pure group batches only), so the deduplicated call has one layout to match
    r = Rig(11)
    r.g.lease_reserve(1 << 16, (1 << 16) * 128)
    try:
        for step in range(6):
            b = r.batch(300)
            dup = r.send(b, _keys(r.rng, 300, 200), now=float(step))
            assert any(dup) and not all(dup)
            r.check()
        r.check(drain=True, leased=True)
    finally:
        r.close()


@pytest.mark.gpu
def test_content_keys_match_numpy_and_a_repeated_batch_is_all_duplicates():
    r = Rig(12)
    try:
        b = r.batch(400)
        r.send(b, content=True, now=1.0)
        r.check()
        dup = r.send(b, content=True, now=2.0)                   # the same sends again: every one is a duplicate
        assert all(dup)
        r.check()
        b2 = r.batch(200)
        ks = _keys(r.rng, 200, 50)
        r.send(b2, ks, content=True, now=3.0)                    # explicit keys where given, content keys elsewhere
        r.check(drain=True)
    finally:
        r.close()


@pytest.mark.gpu
def test_sequence_numbers_past_2_32():
    r = Rig(13)
    try:
        r.g.advance_seq((1 << 32) - 7)
        r.o.next_seq = (1 << 32) - 7
        for step in range(3):
            r.send(r.batch(100), _keys(r.rng, 100, 60), now=float(step))
            r.check()
        assert r.g.stats()["next_seq"] > (1 << 32)
        r.check(drain=True)
    finally:
        r.close()


@pytest.mark.gpu
def test_rebuild_under_expiry_and_the_capacity_refusal():
    from swarmdb_b200._native import SdbError
    r = Rig(14, entries=64, window=10.0)
    try:
        b = r.batch(64, kinds=(0,))
        r.send(b, np.stack([np.arange(1, 65), np.zeros(64)], 1).astype(np.uint64), now=0.0)
        r.check()
        before = _queue_stats(r.g)
        with pytest.raises(SdbError) as e:                       # 64 live entries: one more key does not fit
            r.g.send_mixed_batch_dedup(b["sender"][:1], b["kind"][:1], b["target"][:1], None, None, b["prio"][:1],
                                       b["typ"][:1], b["lens"][:1], b["payload_off"][:1], b["payload"], b["ts"][:1],
                                       keys=np.array([[999, 0]], np.uint64), now=5.0)
        assert e.value.code == -6 and _queue_stats(r.g) == before
        assert r.g.dedup_stats() == r.m.stats() | {"window": 10.0}         # the refusal left the table as it was
        b2 = r.batch(32, kinds=(0,))
        r.send(b2, np.stack([np.arange(100, 132), np.zeros(32)], 1).astype(np.uint64), now=10.0)    # all 64 expired
        r.check()
        assert r.g.dedup_stats()["expired_total"] == 64
        r.check(drain=True)
    finally:
        r.close()


@pytest.mark.gpu
def test_arena_full_refusal_leaves_the_table_and_a_retry_gets_the_same_ids():
    from swarmdb_b200._native import SdbError
    # 128-byte records in a 64 KiB arena: the second batch does not fit behind the first (a batch never straddles the
    # wrap), and fits below the first's end once it is consumed
    r = Rig(15, arena_bytes=1 << 16)
    try:
        b = r.batch(400, kinds=(0,))
        b["lens"][:] = 96
        ks = np.stack([np.arange(1, 401), np.zeros(400)], 1).astype(np.uint64)
        r.send(b, ks, now=0.0)
        before, dbefore = _queue_stats(r.g), r.g.dedup_stats()
        b2 = r.batch(150, kinds=(0,))
        b2["lens"][:] = 96
        k2 = np.stack([np.r_[np.arange(1, 11), np.arange(1000, 1140)], np.zeros(150)], 1).astype(np.uint64)
        with pytest.raises(SdbError) as e:
            r.g.send_mixed_batch_dedup(b2["sender"], b2["kind"], b2["target"], b2["list_off"], b2["list_idx"],
                                       b2["prio"], b2["typ"], b2["lens"], b2["payload_off"], b2["payload"], b2["ts"],
                                       keys=k2, now=1.0)
        assert e.value.code == -5
        assert _queue_stats(r.g) == before and r.g.dedup_stats() == dbefore
        r.check(drain=True)                                      # consumers free the arena ...
        r.send(b2, k2, now=1.0)                                  # ... and the retry gets the model's verdicts and ids
        r.check(drain=True)
    finally:
        r.close()


@pytest.mark.gpu
def test_ring_overflow_then_forget_lets_the_same_keys_in_again():
    r = Rig(16, ring_slots=16)
    try:
        n = 24
        b = r.batch(n, kinds=(0,))
        b["target"][:] = 5                                       # one receiver: its ring takes 16 of the 24
        ks = np.stack([np.arange(1, n + 1), np.full(n, 7)], 1).astype(np.uint64)
        base, dup, keys = r.g.send_mixed_batch_dedup(b["sender"], b["kind"], b["target"], b["list_off"], b["list_idx"],
                                                     b["prio"], b["typ"], b["lens"], b["payload_off"], b["payload"],
                                                     b["ts"], keys=ks, now=0.0)
        assert not dup.any() and r.g.stats()["ring_overflow"] == n - 16
        agents, seqs, dropped = r.g.overflow_log()
        lost = sorted(int(s) - base for s in seqs)              # which sends lose the race for the ring is not fixed
        assert dropped == n - 16 and len(set(lost)) == n - 16 and set(agents.tolist()) == {5}
        removed = r.g.dedup_forget(keys[lost])
        assert removed.tolist() == [1] * len(lost)
        assert r.g.dedup_forget(keys[lost]).tolist() == [0] * len(lost)
        r.g.receive_batch(None, 1 << 10, 0)
        base2, dup2, _ = r.g.send_mixed_batch_dedup(b["sender"], b["kind"], b["target"], b["list_off"], b["list_idx"],
                                                    b["prio"], b["typ"], b["lens"], b["payload_off"], b["payload"],
                                                    b["ts"], keys=ks, now=1.0)
        assert dup2.tolist() == [0 if i in lost else base + i for i in range(n)]
        assert r.g.dedup_stats()["forgotten_total"] == n - 16
    finally:
        r.close()


@pytest.mark.gpu
def test_refusals():
    from swarmdb_b200._native import SdbError, Shard
    g = Shard(max_agents=16)
    try:
        one = (np.zeros(1, np.uint32), np.zeros(1, np.uint8), np.ones(1, np.uint32), None, None, np.ones(1, np.uint8),
               np.zeros(1, np.uint8), np.ones(1, np.uint16), np.zeros(1, np.uint64), np.zeros(64, np.uint8))
        with pytest.raises(SdbError):                            # no table
            g.send_mixed_batch_dedup(*one, keys=np.array([[1, 0]], np.uint64))
        g.dedup_reserve(16, 1.0)
        with pytest.raises(SdbError):
            g.send_mixed_batch_dedup(*one, now=float("nan"))
        with pytest.raises(SdbError):
            g._check(g._L.sdb_send_mixed_batch_dedup(g._h, 0, None, None, None, 0, None, None, None, None, None, None,
                                                     None, 0, None, None, 2, 0.0, None, None, None, None))
        g.profile(True)
        g.send_mixed_batch_dedup(*one, content=True, now=0.0)
        assert g.profile_read()["dedup"][1] >= 2
        g.profile(False)
        g.dedup_reserve(0)
        assert g.dedup_stats()["capacity"] == 0
    finally:
        g.close()


def _db(tmp_path, **kw):
    import swarmdb_b200 as sdb
    g = dict(max_agents=64, max_groups=4, ring_slots=256, arena_bytes=1 << 22, deterministic_ids=True, dedup_entries=1024)
    g.update(kw)
    return sdb.SwarmsDB(save_dir=str(tmp_path), auto_save=False, gpu_config=sdb.GpuConfig(**g))


@pytest.mark.gpu
def test_swarmsdb_dedup_id_original_id_and_unread_counts(tmp_path):
    db = _db(tmp_path)
    try:
        for a in ("a", "b", "c"):
            db.register_agent(a)
        m1 = db.send_message("a", "hi", "b", dedup_id="r1")
        m2 = db.send_message("a", "hi", "b", dedup_id="r1")         # inside the batch
        db.flush()
        m3 = db.send_message("a", "other text", "b", dedup_id="r1")  # across flushes: the key, not the content
        m4 = db.send_message("c", "hi", "b", dedup_id="r1")          # another sender's r1 is another key
        db.flush()
        assert db.original_id(m2) == m1 and db.original_id(m3) == m1 and db.original_id(m1) is None
        assert db.original_id(m4) is None
        assert db.get_message(m2).id == m1 and m2 not in db.messages and m3 not in db.messages
        assert db.agent_inbox["b"] == [m1, m4] and db.get_agent_load("b")["unread_count"] == 2
        assert [m.id for m in db.receive_messages("b", 10)] == [m1, m4]
        db.create_group("t", ["a", "b", "c"])
        g1 = db.send_to_group("a", "t", "x", dedup_id="g")
        g2 = db.send_to_group("a", "t", "y", dedup_id="g")
        b1 = db.broadcast_message("a", "z", dedup_id="bc")
        b2 = db.broadcast_message("a", "z", dedup_id="bc")
        db.flush()
        assert [db.original_id(i) for i in g2] == g1 and db.original_id(b2) == b1
        got = {a: [m.id for m in db.receive_messages(a, 10)] for a in ("b", "c")}
        assert got == {"b": [g1[0], b1], "c": [g1[1], b1]}
        st = db.get_stats()["dedup"]
        assert st["duplicate_total"] == 4 and st["accepted_total"] == 4          # sends: m2, m3, g2, b2 / m1, m4, g1, b1
    finally:
        db.close()
    off = _db(tmp_path, dedup_entries=0)
    try:
        with pytest.raises(ValueError):
            off.send_message("a", "hi", "b", dedup_id="r1")
        assert "dedup" not in off.get_stats()
    finally:
        off.close()


@pytest.mark.gpu
def test_swarmsdb_content_keys(tmp_path):
    db = _db(tmp_path, dedup_content=True)
    try:
        m1 = db.send_message("a", {"cmd": "deploy"}, "b")
        m2 = db.send_message("a", {"cmd": "deploy"}, "b")            # the same send re-emitted
        m3 = db.send_message("a", {"cmd": "deploy"}, "c")            # another receiver: another identity
        db.flush()
        assert db.original_id(m2) == m1 and db.original_id(m3) is None
        assert [m.id for m in db.receive_messages("b", 10)] == [m1]
    finally:
        db.close()


@pytest.mark.gpu
def test_swarmsdb_overflow_forgets_the_failed_keys_and_a_resend_is_accepted(tmp_path):
    from swarmdb_b200.core import MessageStatus
    db = _db(tmp_path, ring_slots=16)
    try:
        ids = [db.send_message("a", f"m{i}", "b", dedup_id=f"d{i}") for i in range(20)]
        with pytest.raises(Exception):
            db.flush()
        failed = [i for i in ids if db.messages[i].status == MessageStatus.FAILED]
        assert len(failed) == 4
        first = [m.id for m in db.receive_messages("b", 100)]
        assert sorted(first) == sorted(set(ids) - set(failed))
        new = db.resend_failed_messages()
        db.flush()
        assert len(new) == 4 and all(db.original_id(i) is None for i in new)
        assert sorted(m.id for m in db.receive_messages("b", 100)) == sorted(new)
        again = db.send_message("a", "x", "b", dedup_id="d0")        # an accepted key stays live
        db.flush()
        assert db.original_id(again) is not None
    finally:
        db.close()


@pytest.mark.gpu
def test_swarmsdb_relocate_and_retry_gets_the_same_verdicts(tmp_path):
    # 256-byte records in a 64 KiB arena: one message for "lag" pins the log while "x" consumes 200; the next flush
    # does not fit until relocation moves lag's record to the tail, and the retried call keeps the first's verdicts
    db = _db(tmp_path, arena_bytes=1 << 16, arena_relocate=True)
    try:
        body = lambda i: f"{i:03d}".ljust(200, ".")
        lag = db.send_message("a", body(999), "lag")
        first = [db.send_message("a", body(i), "x", dedup_id=f"k{i}") for i in range(200)]
        db.flush()
        assert len(db.receive_messages("x", 1000)) == 200
        more = [db.send_message("a", body(i), "x", dedup_id=f"k{i}") for i in range(195, 260)]
        db.flush()
        st = db.shard.stats()
        assert st["ring_overflow"] == 0
        assert [db.original_id(i) for i in more[:5]] == first[195:]
        assert all(db.original_id(i) is None for i in more[5:])
        assert [m.id for m in db.receive_messages("x", 1000)] == more[5:]
        assert [m.id for m in db.receive_messages("lag", 10)] == [lag]
    finally:
        db.close()


@pytest.mark.gpu
def test_rest_idempotency_key(tmp_path):
    pytest.importorskip("fastapi"); pytest.importorskip("jwt"); pytest.importorskip("httpx")
    from fastapi.testclient import TestClient
    from swarmdb_b200.server import Settings, create_app
    db = _db(tmp_path)
    try:
        c = TestClient(create_app(db, Settings(history_dir=str(tmp_path))))

        def token(user):
            r = c.post("/auth/token", json={"username": user, "password": "pw"})
            return {"Authorization": f"Bearer {r.json()['access_token']}"}
        h1, h2, h3 = token("a1"), token("a2"), token("a3")
        for who, h in (("a1", h1), ("a2", h2), ("a3", h3)):
            assert c.post("/agents/register", json={"agent_id": who}, headers=h).status_code == 201
        k = {**h1, "Idempotency-Key": "req-7"}
        r1 = c.post("/messages", json={"content": "once", "receiver_id": "a2"}, headers=k).json()
        r2 = c.post("/messages", json={"content": "once", "receiver_id": "a2"}, headers=k).json()
        assert r1["id"] == r2["id"] and r2["content"] == "once"
        got = c.post("/agents/receive", params={"max_messages": 10}, headers=h2).json()
        assert [m["id"] for m in got] == [r1["id"]]
        assert c.post("/groups", json={"group_name": "t", "agent_ids": ["a1", "a2", "a3"]}, headers=h1).status_code == 201
        kg = {**h1, "Idempotency-Key": "grp"}
        g1 = c.post("/groups/message", json={"group_name": "t", "content": "s"}, headers=kg).json()["message_ids"]
        g2 = c.post("/groups/message", json={"group_name": "t", "content": "s"}, headers=kg).json()["message_ids"]
        assert g1 == g2 and len(g1) == 2
        kb = {**h1, "Idempotency-Key": "bc"}
        b1 = c.post("/messages/broadcast", json={"content": "all"}, headers=kb).json()["message_id"]
        b2 = c.post("/messages/broadcast", json={"content": "all"}, headers=kb).json()["message_id"]
        assert b1 == b2
        plain = c.post("/messages", json={"content": "once", "receiver_id": "a2"}, headers=h1).json()
        assert plain["id"] != r1["id"]                               # no header: not deduplicated
        assert db.get_stats()["dedup"]["duplicate_total"] == 3
    finally:
        db.close()
