"""The deduplication model (tests/dedup_ref.py) and the content-key function, and the ABI the binding declares.  No GPU:
tests/test_gpu_dedup.py holds the device to the same model."""
import ctypes as C
import re
from pathlib import Path

import numpy as np
import pytest

from tests.dedup_ref import DedupModel, batch_seqs, content_key, content_words

ROOT = Path(__file__).resolve().parent.parent


def test_header_declares_the_dedup_calls_and_profiler_class():
    h = (ROOT / "include" / "swarmdb_b200.h").read_text()
    assert "SDB_PK_DEDUP = 17" in h and "SDB_PK_CLASSES = 18" in h and "#define SDB_DEDUP_CONTENT 1u" in h
    for name in ("sdb_dedup_reserve", "sdb_send_mixed_batch_dedup", "sdb_dedup_forget", "sdb_dedup_stats"):
        assert re.search(rf"int {name}\(sdb_handle h,", h)
    from swarmdb_b200._native import EXPORTS, KEY_DTYPE, SdbDedupSummary, Shard
    for name in ("sdb_dedup_reserve", "sdb_send_mixed_batch_dedup", "sdb_dedup_forget", "sdb_dedup_stats"):
        assert name in EXPORTS
    assert Shard.PROFILE_CLASSES[17] == "dedup" and Shard.PROFILE_CLASSES[:17] == Shard.PROFILE_KINDS_ALL
    assert KEY_DTYPE.itemsize == 16 and C.sizeof(SdbDedupSummary) == 72


def test_first_send_of_a_batch_wins_and_later_ones_name_its_seq():
    m = DedupModel(16, 10.0)
    keys = [(5, 0), (7, 0), (5, 0), (0, 0), (7, 0), (5, 0)]
    seq = batch_seqs(100, [0, 1, 0, 0, 2, 0], [0, 0, 0, 0, 0, 0], {0: 4})
    assert seq == [100, 101, 105, 106, 107, 108]
    dup, n_new = m.send(keys, seq, 0.0)
    assert dup == [0, 0, 100, 0, 101, 100] and n_new == 2
    m.commit(keys, seq, dup, n_new, 0.0)
    assert m.tab == {(5, 0): [100, 0.0], (7, 0): [101, 0.0]}
    dup, n_new = m.send([(7, 0), (9, 0)], [200, 201], 1.0)      # across calls: the table's seq
    assert dup == [101, 0] and n_new == 1


def test_an_entry_is_live_until_now_reaches_inserted_at_plus_window():
    m = DedupModel(16, 10.0)
    m.commit([(1, 2)], [5], [0], 1, 3.0)
    assert m.verdicts([(1, 2)], [9], np.nextafter(13.0, 0))[0] == [5]
    assert m.verdicts([(1, 2)], [9], 13.0)[0] == [0]            # now == inserted_at + window: expired
    dup, n_new = m.send([(1, 2)], [9], 13.0)
    m.commit([(1, 2)], [9], dup, n_new, 13.0)
    assert m.tab[(1, 2)] == [9, 13.0] and len(m.tab) == 1        # the key's slot is reused, not doubled


def test_capacity_counts_new_keys_after_a_rebuild_drops_the_expired():
    m = DedupModel(4, 10.0)
    keys = [(k, 0) for k in range(1, 5)]
    dup, n = m.send(keys, [1, 2, 3, 4], 0.0)
    m.commit(keys, [1, 2, 3, 4], dup, n, 0.0)
    with pytest.raises(OverflowError):
        m.send([(9, 0)], [5], 5.0)                              # four live entries, one new key
    assert len(m.tab) == 4 and m.rebuilds == 0 and m.expired == 0      # a refusal changes nothing
    dup, n = m.send([(9, 0), (1, 0)], [5, 6], 10.0)             # all four expired at now = 10
    assert dup == [0, 0] and n == 2 and m.rebuilds == 0 and len(m.tab) == 4    # nothing changes before commit
    m.commit([(9, 0), (1, 0)], [5, 6], dup, n, 10.0)            # the accepted call rebuilds, then inserts
    assert m.rebuilds == 1 and m.expired == 4 and m.tab == {(9, 0): [5, 10.0], (1, 0): [6, 10.0]}


def test_forget_kills_live_entries_only_and_the_key_is_accepted_again():
    m = DedupModel(8, 10.0)
    m.commit([(3, 3), (4, 4)], [10, 11], [0, 0], 2, 0.0)
    m.last_now = 5.0
    assert m.forget([(3, 3), (6, 6)]) == [1, 0]
    assert m.forget([(3, 3)]) == [0] and m.forgotten == 1
    assert m.verdicts([(3, 3), (4, 4)], [20, 21], 5.0)[0] == [0, 11]
    assert m.stats()["live"] == 1 and m.stats()["used"] == 2


def test_key_zero_bypasses_the_table():
    m = DedupModel(1, 10.0)
    keys = [(0, 0)] * 5
    dup, n_new = m.send(keys, list(range(5)), 0.0)
    assert dup == [0] * 5 and n_new == 0
    m.commit(keys, list(range(5)), dup, n_new, 0.0)
    assert m.tab == {}


def _key(**kw):
    base = dict(sender=3, kind=0, target=9, recipients=None, length=20, prio=1, typ=2,
                payload=bytes(range(40, 60)) + b"\xff" * 12)
    base.update(kw)
    return content_key(**base)


def test_content_key_changes_with_each_identity_field_and_word_order():
    k0 = _key()
    assert k0 != (0, 0)
    variants = [_key(sender=4), _key(kind=1), _key(target=10), _key(length=19), _key(prio=2), _key(typ=3),
                _key(payload=bytes(range(41, 61))), _key(kind=2, recipients=[1, 2]), _key(kind=2, recipients=[2, 1])]
    assert len({k0, *variants}) == len(variants) + 1
    p = bytes(range(40, 56))
    swapped = p[8:16] + p[0:8]
    assert _key(payload=p, length=16) != _key(payload=swapped, length=16)
    # bytes past len are not part of the identity; a list send hashes its recipients, not its list number
    assert _key(payload=bytes(range(40, 60)) + b"\0" * 12) == k0
    assert _key(kind=2, target=0, recipients=[1, 2]) == _key(kind=2, target=5, recipients=[1, 2])


def test_content_key_ignores_the_timestamp():
    from tests.test_gpu_dedup import send_keys
    b = dict(sender=np.array([1, 1]), kind=np.array([0, 0]), target=np.array([2, 2]), list_off=np.array([0], np.uint64),
             list_idx=np.zeros(0, np.uint32), prio=np.array([1, 1]), typ=np.array([0, 0]), lens=np.array([5, 5]),
             payload_off=np.array([0, 16], np.uint64), payload=np.frombuffer(b"hello\0\0\0\0\0\0\0\0\0\0\0hello" + b"\0" * 11, np.uint8),
             ts=np.array([1.0, 2.0]))
    k = send_keys(b)
    assert k[0] == k[1]


def test_content_words_layout():
    w = content_words(7, 2, 0, [4, 5], 9, 3, 1, b"abcdefghi")
    assert w.tolist() == [7 | 2 << 32, 2, 4, 5, 9 | 3 << 16 | 1 << 24, int.from_bytes(b"abcdefgh", "little"), ord("i")]


def test_sharded_front_end_refuses_deduplication():
    from swarmdb_b200.core import GpuConfig
    from swarmdb_b200.sharded import ShardedSwarmsDB
    with pytest.raises(NotImplementedError, match="deduplicate"):
        ShardedSwarmsDB(0, 2, gpu_config=GpuConfig(dedup_entries=16), auto_save=False)
    db = ShardedSwarmsDB.__new__(ShardedSwarmsDB)              # the per-call refusals come before any state is read
    with pytest.raises(NotImplementedError, match="deduplicate"):
        db.send_message("a", "x", "b", dedup_id="k")
    with pytest.raises(NotImplementedError, match="deduplicate"):
        db.send_to_group("a", "g", "x", dedup_id="k")
    with pytest.raises(NotImplementedError, match="deduplicate"):
        db.broadcast_message("a", "x", dedup_id="k")


def test_dedup_key_is_blake2b_of_sender_and_id_and_needs_a_table():
    import hashlib
    from swarmdb_b200.core import GpuConfig, SwarmsDB
    db = SwarmsDB.__new__(SwarmsDB)
    db.gpu_config = GpuConfig(dedup_entries=8)
    d = hashlib.blake2b(b"alice\0req-1", digest_size=16).digest()
    assert db._dedup_key("alice", "req-1") == (int.from_bytes(d[:8], "little"), int.from_bytes(d[8:], "little"))
    assert db._dedup_key("bob", "req-1") != db._dedup_key("alice", "req-1")     # scoped to the sender
    assert db._dedup_key("alice", None) == (0, 0)
    db.gpu_config = GpuConfig()
    with pytest.raises(ValueError, match="dedup_entries"):
        db._dedup_key("alice", "req-1")
