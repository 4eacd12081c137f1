"""Restore (sdb_restore_compact) without a GPU: the C struct and profiler slot, the reference against oracles that were
sent the records directly, the arena placement model, and the host-side row handling of the snapshot writer."""
import ctypes as C
import re
from pathlib import Path

import numpy as np

from tests.restore_ref import restore_append, restore_granules

ROOT = Path(__file__).resolve().parent.parent


def _compact_of(hdr, pay):
    """Compact format of a full receive, one row per record (what an unshared queue returns)."""
    from swarmdb_b200._native import ENTRY_DTYPE, SEND_DTYPE
    ent = np.zeros(len(hdr), ENTRY_DTYPE)
    snd = np.zeros(len(hdr), SEND_DTYPE)
    ent["seq"], ent["receiver"], ent["send"] = hdr["seq"], hdr["receiver"], np.arange(len(hdr))
    for f in ("timestamp", "sender", "group", "len", "prio", "type"):
        snd[f] = hdr[f]
    pl = ((hdr["len"].astype(np.int64) + 31) & ~31)
    snd["payload_off"][1:] = np.cumsum(pl)[:-1]
    return ent, snd, pay


def test_header_declares_restore_and_profiler_slot():
    h = (ROOT / "include" / "swarmdb_b200.h").read_text()
    assert re.search(r"int sdb_restore_compact\(sdb_handle h, uint32_t n_agents, const uint32_t\* agent_idx", h)
    assert "SDB_PK_RESTORE = 15" in h and "SDB_PK_N = 16" in h
    from swarmdb_b200._native import EXPORTS, Shard
    assert "sdb_restore_compact" in EXPORTS
    assert Shard.PROFILE_KINDS[15] == "restore" and len(Shard.PROFILE_KINDS) == 16
    assert C.sizeof(C.c_uint64) == 8


def _traffic(o, rng, A, G, members):
    for g, m in enumerate(members):
        o.create_group(g, m)
    o.register(np.arange(A, dtype=np.uint32))
    buf = rng.integers(33, 127, 64 * 288).astype(np.uint8)
    off = np.arange(64, dtype=np.uint64) * 288
    lens = rng.integers(0, 257, 64).astype(np.uint16)
    lens[0] = 0
    o.send_batch(rng.integers(0, A, 64), rng.integers(0, A, 64), rng.integers(0, 4, 64), None, lens, off, buf)
    o.send_group_batch(rng.integers(0, A, 8), rng.integers(0, G, 8), rng.integers(0, 4, 8), None, lens[:8], off[:8], buf)
    o.send_list_batch([1, 2], [0, 3, 6], [4, 5, 6, 7, 8, 9], [2, 3], None, lens[:2], off[:2], buf)


def test_reference_equals_oracle_sent_directly():
    """Appending a PEEK of one oracle to an empty one reproduces every agent's stream, loads and sequence counter."""
    from oracle.cpu_ref import CpuOracle
    rng = np.random.default_rng(2)
    A, G = 40, 3
    members = [rng.permutation(A)[:10].astype(np.uint32) for _ in range(G)]
    a, b = CpuOracle(A, G), CpuOracle(A, G)
    _traffic(a, rng, A, G, members)
    b.register(np.arange(A, dtype=np.uint32))
    for g, m in enumerate(members):
        b.create_group(g, m)
    agents = np.arange(A, dtype=np.uint32)
    cnt, hdr, pay = a.receive_batch(agents, 1 << 20, 2)
    ent, snd, pay = _compact_of(hdr, pay)
    n = restore_append(b, dict(enumerate(members)), agents, cnt, ent, snd, pay)
    assert n == len(hdr) and b.next_seq == int(hdr["seq"].max()) + 1
    for flags in (1, 0):
        ca, ha, pa = a.receive_batch(agents, 3, flags)
        cb, hb, pb = b.receive_batch(agents, 3, flags)
        assert np.array_equal(ca, cb) and ha.tobytes() == hb.tobytes() and pa.tobytes() == pb.tobytes()
    la, lb = a.agent_loads(agents), b.agent_loads(agents)
    assert np.array_equal(la["pending"], lb["pending"]) and np.array_equal(la["pending_granules"], lb["pending_granules"])
    # a send to both afterwards gets the same fresh seq
    buf = np.zeros(64, np.uint8)
    assert a.send_batch([0], [1], [1], None, [3], [0], buf) == b.send_batch([0], [1], [1], None, [3], [0], buf)
    a.close(); b.close()


def test_placement_model():
    from swarmdb_b200._native import ENTRY_DTYPE, SEND_DTYPE
    snd = np.zeros(3, SEND_DTYPE)
    snd["len"] = [64, 0, 100]                                # 2, 0 and 4 payload granules
    ent = np.zeros(6, ENTRY_DTYPE)
    ent["send"] = [0, 1, 2,  2, 0, 1]                        # agent 0: ascending; agent 1: descends at its 2nd entry
    cnt = [3, 3]
    # shared: rows 0 (1 header), 1 (1), 2 (2 headers) + payloads 2 + 0 + 4; private: row 0 (1 + 2) and row 1 (1 + 0)
    assert restore_granules(cnt, ent, snd, True) == (1 + 2) + (1 + 0) + (2 + 4) + (3 + 1)
    assert restore_granules(cnt, ent, snd, False) == 2 * (3 + 1 + 5)
    assert restore_granules(cnt, ent, snd, True, agents=[0, 1], skip=lambda a: a == 1) == 3 + 1 + 5
    big = np.zeros(70000, ENTRY_DTYPE)
    assert restore_granules(np.ones(70000, np.int64), big, snd[:1]) == 70000 + 2 * 2


def test_renumber_and_compact_rows():
    from swarmdb_b200._native import ENTRY_DTYPE, SEND_DTYPE, expand_compact
    from swarmdb_b200.core import _compact_rows, _renumber_rows
    rng = np.random.default_rng(4)
    snd = np.zeros(4, SEND_DTYPE)
    snd["len"] = [40, 0, 33, 10]
    snd["payload_off"] = [0, 64, 64, 128]
    snd["sender"] = [9, 8, 7, 6]
    pay = rng.integers(0, 256, 160).astype(np.uint8)
    ent = np.zeros(5, ENTRY_DTYPE)
    ent["send"], ent["seq"] = [2, 0, 2, 1, 0], [30, 10, 31, 5, 11]
    e2, s2 = _renumber_rows(ent, snd)
    assert s2["sender"].tolist() == [8, 9, 7, 6]             # smallest seq 5, 10, 30; the unreferenced row last
    h1, p1 = expand_compact(ent, snd, pay)
    h2, p2 = expand_compact(e2, s2, pay)
    assert h1.tobytes() == h2.tobytes() and p1.tobytes() == p2.tobytes()
    e3, s3, p3 = _compact_rows(e2[[0, 3]], s2, pay)          # rows 2 (seq 30) and 0 (len 0): packed, in row order
    assert s3["sender"].tolist() == [8, 7] and s3["payload_off"].tolist() == [0, 0] and len(p3) == 64
    h3, q3 = expand_compact(e3, s3, p3)
    h4, q4 = expand_compact(e2[[0, 3]], s2, pay)
    assert h3.tobytes() == h4.tobytes() and q3.tobytes() == q4.tobytes()


def test_snapshot_that_overfills_a_ring_is_refused_before_any_restore(tmp_path):
    """load_queue_snapshot restores chunk by chunk; an agent with more records than ring_slots in a later chunk used to
    be found only after the earlier chunks were restored, leaving the instance half-loaded and no longer fresh.  The
    whole snapshot is checked first: nothing reaches the device and the instance can still load another snapshot."""
    import pytest

    import swarmdb_b200 as sdb
    from swarmdb_b200._native import ENTRY_DTYPE, SEND_DTYPE, SdbError
    from tests.fake_shard import OracleShard

    class Recording(OracleShard):
        def __init__(self, *a):
            super().__init__(*a)
            self.calls = []

        def stats(self):
            return {**super().stats(), "enqueued": sum(int(np.sum(c)) for _, c in self.calls)}

        def restore_compact(self, agents, counts, entries, sends, payload, flags=0):
            self.calls.append((np.asarray(agents).tolist(), np.asarray(counts).tolist()))
            return int(np.sum(counts)), int(entries["seq"].max()) + 1

    def snapshot(path, counts):
        chunks = [[0, 1], [2]]                              # two chunks; agent 2 alone in the last one
        n = sum(counts)
        ent = np.zeros(n, ENTRY_DTYPE)
        ent["seq"] = np.arange(1, n + 1); ent["send"] = np.arange(n); ent["receiver"] = np.repeat([0, 1, 2], counts)
        snd = np.zeros(n, SEND_DTYPE)
        off = np.zeros((3, 4), np.uint64)
        for k, c in enumerate(chunks):
            m = sum(counts[a] for a in c)
            off[k + 1] = off[k] + [len(c), m, m, 0]
        np.savez(path, version=np.uint32(sdb.SwarmsDB.SNAPSHOT_VERSION), shard=np.array([0, 1], np.uint32),
                 id_nonce=np.uint64(0), next_seq=np.uint64(n + 1), agent_names=np.array(["a", "b", "c"], np.str_),
                 registered=np.ones(3, bool), group_names=np.zeros(0, np.str_), group_off=np.zeros(1, np.uint64),
                 group_members=np.zeros(0, np.uint32), chunk_off=off, agents=np.array([0, 1, 2], np.uint32),
                 counts=np.array(counts, np.uint32), entries=ent, sends=snd, payload=np.zeros(0, np.uint8))
        return path

    def fresh():
        shard = Recording(64, 4, 0, 1)
        cfg = sdb.GpuConfig(max_agents=64, max_groups=4, ring_slots=16, max_recv_records=64, deterministic_ids=True)
        return shard, sdb.SwarmsDB(save_dir=str(tmp_path), auto_save=False, gpu_config=cfg, _shard=shard)

    shard, db = fresh()
    with pytest.raises(SdbError) as ei:
        db.load_queue_snapshot(snapshot(tmp_path / "over.npz", [2, 3, 17]))
    assert ei.value.code == -4 and "ring_slots=16" in str(ei.value)
    assert shard.calls == []
    db._check_fresh()                                       # still fresh: a snapshot that fits loads into it
    db.load_queue_snapshot(snapshot(tmp_path / "fits.npz", [2, 3, 16]))
    assert shard.calls == [([0, 1], [2, 3]), ([2], [16])]
    db.close()


def test_sharded_front_end_refuses_snapshots_and_requeue(tmp_path):
    """A sharded deployment does not snapshot or requeue yet: the inherited single-shard versions would restore every
    agent's records on every rank, so the sharded class refuses them."""
    import pytest

    import swarmdb_b200 as sdb
    from swarmdb_b200 import sharded
    from tests.fake_shard import OracleShard

    class Ex:
        def __init__(self, *a): pass
        def close(self): pass
    db = sharded.ShardedSwarmsDB(0, 1, exchange_factory=Ex, shard=OracleShard(64, 4, 0, 1), save_dir=str(tmp_path),
                                 auto_save=False, gpu_config=sdb.GpuConfig(max_agents=64, max_groups=4))
    for call in (lambda: db.save_queue_snapshot(tmp_path / "q.npz"), lambda: db.load_queue_snapshot(tmp_path / "q.npz"),
                 lambda: db.requeue_batch_compact([], [], [], [], [])):
        with pytest.raises(NotImplementedError):
            call()
    assert not (tmp_path / "q.npz").exists()
    db.close()
