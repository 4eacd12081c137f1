"""Queue snapshots that keep in-flight work (save_queue_snapshot(in_flight=True), format 2) without a GPU: the header
and binding of the four export / import calls, and the host side of the snapshot writer and reader against a recording
stand-in shard (tests/fake_shard.py) that plays the lease store and the ledger."""
import re
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent

FORMAT_1_KEYS = {"version", "shard", "id_nonce", "next_seq", "agent_names", "registered", "group_names", "group_off",
                 "group_members", "chunk_off", "agents", "counts", "entries", "sends", "payload"}
LEASE_KEYS = {"lease_entries", "lease_sends", "lease_payload", "lease_meta", "lease_chunk_off", "ledger_agent", "ledger_seq",
              "ledger_count", "ledger_max_deliveries"}


def test_header_binding_and_meta_layout():
    import ctypes as C

    from swarmdb_b200._native import EXPORTS, META_DTYPE, Shard
    h = (ROOT / "include" / "swarmdb_b200.h").read_text()
    for name in ("sdb_lease_export", "sdb_lease_import", "sdb_lease_ledger_export", "sdb_lease_ledger_import"):
        assert re.search(rf"int {name}\(sdb_handle h,", h) and name in EXPORTS
    assert "SDB_LEASE_STATE_DEAD 3u" in h and "SDB_LS_DEAD 3u" in (ROOT / "swarmdb_b200/csrc/sdb_common.cuh").read_text()
    assert META_DTYPE.itemsize == 32 and [META_DTYPE.fields[f][1] for f in META_DTYPE.names] == [0, 8, 16, 20, 24, 28]
    for m in ("lease_export", "lease_import", "ledger_export", "ledger_import"):
        assert callable(getattr(Shard, m))
    assert C.sizeof(C.c_double) == 8


def _store(rng, n, lens, agents):
    """n leased records over len(lens) rows in the compact format, as an export returns them: rows numbered by first
    appearance, each record's meta."""
    from swarmdb_b200._native import ENTRY_DTYPE, META_DTYPE, SEND_DTYPE
    rows = np.sort(rng.integers(0, len(lens), n))
    rows[: len(lens)] = np.arange(len(lens))
    rows = np.sort(rows)
    ent = np.zeros(n, ENTRY_DTYPE)
    ent["seq"] = np.arange(100, 100 + n)
    ent["send"] = rows
    ent["receiver"] = agents
    snd = np.zeros(len(lens), SEND_DTYPE)
    snd["len"] = lens
    snd["sender"] = np.arange(len(lens)) + 7
    pl = (np.asarray(lens, np.int64) + 31) & ~31
    snd["payload_off"][1:] = np.cumsum(pl)[:-1]
    pay = rng.integers(0, 256, int(pl.sum())).astype(np.uint8)
    meta = np.zeros(n, META_DTYPE)
    meta["id"] = np.arange(n) + 40
    meta["deadline"] = 1000.0 + np.arange(n)
    meta["agent"] = agents
    meta["deliveries"] = 1 + np.arange(n) % 3
    meta["state"] = np.where(np.arange(n) % 4 == 3, 3, 0)
    return ent, snd, pay, meta


def _recording_shard(chunk=3, store=None, ledger=None, ledger_cap=64, lease_cap=64):
    from swarmdb_b200._native import expand_compact
    from swarmdb_b200.core import _compact_rows
    from tests.fake_shard import OracleShard

    class Recording(OracleShard):
        def __init__(self, *a):
            super().__init__(*a)
            self.calls, self.next_id = [], 500

        def stats(self):
            return {**super().stats(), "enqueued": sum(len(c[1]) for c in self.calls if c[0] == "restore")}

        def lease_reserve(self, n, p): self.reserved = (n, p)
        def lease_set_policy(self, m, n): self.policy = (m, n)
        def lease_stats(self): return {"live": 0, "entries_used": 0, "entries_reserved": lease_cap, "payload_used": 0,
                                       "payload_reserved": lease_cap * 256}
        def lease_policy_stats(self): return {"dead": 0, "ledger_cap": ledger_cap}

        def lease_export(self, start=0):
            """The stand-in store's records with meta id >= start, `chunk` at a time, rows renumbered per chunk."""
            ent, snd, pay, meta = store
            sel = np.nonzero(meta["id"] >= start)[0][:chunk]
            if len(sel) == 0:
                return ent[:0], snd[:0], pay[:0], meta[:0], start
            e, s, p = _compact_rows(ent[sel], snd, pay)
            return e, s, p, meta[sel].copy(), int(meta["id"][sel[-1]]) + 1

        def ledger_export(self):
            return ledger

        def restore_compact(self, agents, counts, entries, sends, payload, flags=0):
            self.calls.append(("restore", np.asarray(counts).tolist()))
            return int(np.sum(counts)), int(entries["seq"].max()) + 1

        def ledger_import(self, agent, seq, count):
            self.calls.append(("ledger", np.asarray(agent).tolist(), np.asarray(seq).tolist(), np.asarray(count).tolist()))
            return len(agent)

        def lease_import(self, entries, sends, payload, meta):
            h, p = expand_compact(entries, sends, payload)
            self.calls.append(("lease", h.copy(), p.copy(), meta.copy()))
            base = self.next_id
            self.next_id += len(entries)
            return base

    return Recording


def _db(tmp_path, shard_cls, **kw):
    import swarmdb_b200 as sdb
    shard = shard_cls(64, 4, 0, 1)
    cfg = dict(max_agents=64, max_groups=4, ring_slots=16, max_recv_records=64, deterministic_ids=True)
    cfg.update(kw)
    return shard, sdb.SwarmsDB(save_dir=str(tmp_path), auto_save=False, gpu_config=sdb.GpuConfig(**cfg), _shard=shard)


def test_writer_concatenates_export_chunks_with_rows_and_payload_rebased(tmp_path):
    from swarmdb_b200._native import expand_compact
    rng = np.random.default_rng(1)
    store = _store(rng, 8, [40, 0, 100, 7, 64], rng.integers(0, 3, 8))
    ledger = (np.array([1, 2], np.uint32), np.array([5, 9], np.uint64), np.array([2, 3], np.uint32))
    shard, db = _db(tmp_path, _recording_shard(3, store, ledger), lease_records=64, lease_max_deliveries=3)
    for a in "abc":
        db.register_agent(a)
    path = db.save_queue_snapshot(tmp_path / "q2.npz", in_flight=True)
    with np.load(path, allow_pickle=False) as z:
        snap = {k: z[k] for k in z.files}
    assert set(snap) == FORMAT_1_KEYS | LEASE_KEYS and int(snap["version"]) == 2
    off = snap["lease_chunk_off"].astype(np.int64)
    assert off[:, 0].tolist() == [0, 3, 6, 8]                          # three export calls of at most 3 records
    for k in range(3):                                                   # each chunk, rebased, expands to the store's records
        e0, e1 = off[k, 0], off[k + 1, 0]
        ent = snap["lease_entries"][e0:e1]
        assert ent["send"].min() >= off[k, 1] and ent["send"].max() < off[k + 1, 1]
        got = expand_compact(ent, snap["lease_sends"], snap["lease_payload"])
        want = expand_compact(store[0][e0:e1], store[1], store[2])
        assert all(x.tobytes() == y.tobytes() for x, y in zip(got, want))
    assert snap["lease_meta"].tobytes() == store[3].tobytes()
    assert snap["ledger_agent"].tolist() == [1, 2] and snap["ledger_seq"].tolist() == [5, 9]
    assert snap["ledger_count"].tolist() == [2, 3] and int(snap["ledger_max_deliveries"]) == 3
    db.close()


def test_in_flight_false_writes_exactly_the_format_1_keys(tmp_path, caplog):
    rng = np.random.default_rng(2)
    store = _store(rng, 4, [10, 20], np.zeros(4, np.uint32))
    shard, db = _db(tmp_path, _recording_shard(3, store), lease_records=64)
    db.register_agent("a")
    with np.load(db.save_queue_snapshot(tmp_path / "q1.npz"), allow_pickle=False) as z:
        assert set(z.files) == FORMAT_1_KEYS and int(z["version"]) == 1
    with pytest.raises(ValueError):
        _db(tmp_path, _recording_shard())[1].save_queue_snapshot(tmp_path / "x.npz", in_flight=True)   # no store
    assert not (tmp_path / "x.npz").exists()
    db.close()


def _format_2(path, counts, store, ledger, version=2):
    """A snapshot with pending records of agents a, b, c in one chunk (format 1), and the lease and ledger sections."""
    from swarmdb_b200._native import ENTRY_DTYPE, META_DTYPE, SEND_DTYPE
    n = sum(counts)
    ent = np.zeros(n, ENTRY_DTYPE)
    ent["seq"] = np.arange(1, n + 1); ent["send"] = np.arange(n); ent["receiver"] = np.repeat([0, 1, 2], counts)
    off = np.array([[0, 0, 0, 0], [3, n, n, 0]], np.uint64)
    arrays = dict(version=np.uint32(version), shard=np.array([0, 1], np.uint32), id_nonce=np.uint64(0),
                  next_seq=np.uint64(n + 1000), agent_names=np.array(["a", "b", "c"], np.str_), registered=np.ones(3, bool),
                  group_names=np.zeros(0, np.str_), group_off=np.zeros(1, np.uint64), group_members=np.zeros(0, np.uint32),
                  chunk_off=off, agents=np.array([0, 1, 2], np.uint32), counts=np.array(counts, np.uint32), entries=ent,
                  sends=np.zeros(n, SEND_DTYPE), payload=np.zeros(0, np.uint8))
    if version == 2:
        le, ls, lp, lm = store if store is not None else (np.zeros(0, ENTRY_DTYPE), np.zeros(0, SEND_DTYPE),
                                                          np.zeros(0, np.uint8), np.zeros(0, META_DTYPE))
        la, lq, lc = ledger if ledger is not None else (np.zeros(0, np.uint32), np.zeros(0, np.uint64), np.zeros(0, np.uint32))
        arrays.update(lease_entries=le, lease_sends=ls, lease_payload=lp, lease_meta=lm,
                      lease_chunk_off=np.array([[0, 0, 0], [len(le), len(ls), len(lp)]], np.uint64),
                      ledger_agent=la, ledger_seq=lq, ledger_count=lc, ledger_max_deliveries=np.uint32(3))
    np.savez(path, **arrays)
    return path


def test_load_order_split_and_host_lease_map(tmp_path):
    """Restore, then ledger import, then lease import; a chunk larger than this instance's receive capacity is split, each
    part with only its rows; the host's lease map and deadline heap point at the new lease ids."""
    from swarmdb_b200._native import expand_compact
    rng = np.random.default_rng(3)
    store = _store(rng, 7, [40, 0, 100, 64], rng.integers(0, 3, 7))
    ledger = (np.array([0], np.uint32), np.array([2], np.uint64), np.array([2], np.uint32))
    shard, db = _db(tmp_path, _recording_shard(), lease_records=64, lease_max_deliveries=3, max_recv_records=3)
    db.load_queue_snapshot(_format_2(tmp_path / "q.npz", [1, 1, 1], store, ledger))
    kinds = [c[0] for c in shard.calls]
    assert kinds == ["restore", "ledger", "lease", "lease", "lease"]
    assert shard.calls[1][1:] == ([0], [2], [2])
    leases = shard.calls[2:]
    assert [len(c[3]) for c in leases] == [3, 3, 1]
    want_h, want_p = expand_compact(*store[:3])
    assert np.concatenate([c[1] for c in leases]).tobytes() == want_h.tobytes()
    assert np.concatenate([c[2] for c in leases]).tobytes() == want_p.tobytes()
    assert np.concatenate([c[3] for c in leases]).tobytes() == store[3].tobytes()
    for k, (seq, a) in enumerate(zip(store[0]["seq"].tolist(), store[3]["agent"].tolist())):
        assert db._leases[db._make_id(seq)] == [(a, 500 + k)]
    live = store[3]["state"] == 0
    assert sorted(db._lease_deadlines) == sorted(set(store[3]["deadline"][live].tolist()))
    db.close()


@pytest.mark.parametrize("case", ["no store", "dead without policy", "counts without policy", "store too small",
                                  "ledger too small"])
def test_refusal_before_adoption_keeps_the_instance_fresh(tmp_path, case):
    rng = np.random.default_rng(4)
    store = _store(rng, 6, [40, 10], rng.integers(0, 3, 6))
    ledger = (np.array([0, 1], np.uint32), np.array([2, 3], np.uint64), np.array([2, 2], np.uint32))
    kw = {"no store": {}, "dead without policy": dict(lease_records=64),
          "counts without policy": dict(lease_records=64),
          "store too small": dict(lease_records=64, lease_max_deliveries=3),
          "ledger too small": dict(lease_records=64, lease_max_deliveries=3)}[case]
    if case == "counts without policy":
        store[3]["state"] = 0
    shard, db = _db(tmp_path, _recording_shard(lease_cap=4 if case == "store too small" else 64,
                                               ledger_cap=1 if case == "ledger too small" else 64), **kw)
    why = {"no store": "lease store", "dead without policy": "lease_max_deliveries",
           "counts without policy": "lease_max_deliveries", "store too small": "free room",
           "ledger too small": "ledger holds"}[case]
    with pytest.raises(RuntimeError, match=why):
        db.load_queue_snapshot(_format_2(tmp_path / "q.npz", [1, 1, 1], store,
                                         None if case == "dead without policy" else ledger))
    assert shard.calls == [] and db._leases == {}
    db._check_fresh()
    db.close()


def test_format_1_still_loads_into_an_instance_with_a_store(tmp_path):
    shard, db = _db(tmp_path, _recording_shard(), lease_records=64, lease_max_deliveries=3)
    db.load_queue_snapshot(_format_2(tmp_path / "q1.npz", [2, 3, 4], None, None, version=1))
    assert shard.calls == [("restore", [2, 3, 4])]
    db.close()
    shard, db = _db(tmp_path, _recording_shard())                       # and a format-2 file without leases needs a store
    with pytest.raises(RuntimeError):
        db.load_queue_snapshot(_format_2(tmp_path / "q2.npz", [2, 3, 4], None, None))
    assert shard.calls == []
    db.close()
