"""Relocation of pinned queues, host side: the ABI declaration and binding, relocate_pinned's cut search and flush's
retry, against stand-ins of the device (tests/fake_shard.py)."""
import ctypes as C
import re
from pathlib import Path

import numpy as np
import pytest

from tests.fake_shard import OracleShard

ROOT = Path(__file__).resolve().parents[1]


def test_header_declares_the_call_and_the_binding_matches():
    from swarmdb_b200 import _native
    h = (ROOT / "include" / "swarmdb_b200.h").read_text()
    assert re.search(r"int sdb_arena_relocate\(sdb_handle h, uint64_t floor_bytes, uint32_t flags, sdb_relocate_summary\* out\);", h)
    body = h[h.index("typedef struct sdb_relocate_summary"): h.index("} sdb_relocate_summary;")]
    assert re.findall(r"uint64_t\s+([a-z_, ]+);", body) == ["agents", "records", "moved_bytes", "skipped_bytes",
                                                           "floor_before, floor_after, tail_after"]
    assert "SDB_RECV_PEEK: a dry run" in h and "Any other bit: SDB_EINVAL" in h
    assert C.sizeof(_native.SdbRelocateSummary) == 56
    assert [n for n, _ in _native.SdbRelocateSummary._fields_] == ["agents", "records", "moved_bytes", "skipped_bytes",
                                                                   "floor_before", "floor_after", "tail_after"]
    assert "sdb_arena_relocate" in _native.EXPORTS and hasattr(_native.Shard, "relocate")
    assert "sdb_relocate.cu" in (ROOT / "swarmdb_b200" / "csrc" / "Makefile").read_text()


class _PinnedLog(OracleShard):
    """The arena as relocate_pinned sees it: `arena` bytes, a tail, and pinned agents (oldest record, bytes of live
    records).  relocate() follows the device's placement rule; send_mixed_batch refuses with -5 while the batch's bound
    does not fit, and counts its calls."""

    def __init__(self, arena, tail, pinned, refuse=0, **kw):
        super().__init__(64, 16, 0, 1)
        self.arena, self.tail, self.pinned = arena, tail, dict(pinned)
        self.calls, self.sends, self.refuse = [], 0, refuse

    def stats(self):
        st = super().stats()
        st["arena_tail_bytes"] = self.tail
        return st

    def _plan(self, cut):
        sel = {a: v for a, v in self.pinned.items() if v[0] < cut}
        moved = sum(v[1] for v in sel.values())
        base = self.tail
        if moved and base % self.arena + moved > self.arena:
            base += self.arena - base % self.arena
        unsel = [v[0] for a, v in self.pinned.items() if a not in sel]
        floor = min(unsel + ([base] if moved else []), default=base + moved)
        if moved and base + moved - min(unsel + [v[0] for v in sel.values()]) > self.arena:
            from swarmdb_b200._native import SdbError
            raise SdbError(-5, "does not fit")
        return sel, base, moved, floor

    def relocate(self, cut, peek=False):
        sel, base, moved, floor = self._plan(cut)
        self.calls.append((cut, peek))
        s = {"agents": len(sel), "records": len(sel), "moved_bytes": moved, "skipped_bytes": base - self.tail,
             "floor_before": 0, "floor_after": floor, "tail_after": base + moved}
        if not peek:
            for k, (p, b) in enumerate(sorted(sel.items(), key=lambda kv: kv[1][0])):
                self.pinned[p] = (base + sum(v[1] for _, v in sorted(sel.items(), key=lambda kv: kv[1][0])[:k]), b[1])
            self.tail = base + moved
        return s

    def send_mixed_batch(self, *a, **k):
        self.sends += 1
        if self.refuse:
            self.refuse -= 1
            from swarmdb_b200._native import SdbError
            raise SdbError(-5, "message arena full (test)")
        return super().send_mixed_batch(*a, **k)


def _db(tmp_path, shard, **kw):
    import swarmdb_b200 as sdb
    cfg = sdb.GpuConfig(max_agents=64, max_groups=16, deterministic_ids=True, arena_bytes=shard.arena, **kw)
    return sdb, sdb.SwarmsDB(save_dir=str(tmp_path), auto_save=False, gpu_config=cfg, _shard=shard)


def test_cut_search_converges(tmp_path):
    # 100 kB free in a 1 MiB arena, ten agents pinning at 200k, 240k, ... 560k: the first dry run leaves the fourth agent
    # pinning 10 kB short, so the next cut is the floor that would have sufficed, which passes that agent
    pinned = {a: (200_000 + a * 40_000, 10_000) for a in range(10)}
    shard = _PinnedLog(1 << 20, (1 << 20) + 100_000, pinned)
    sdb, db = _db(tmp_path, shard)
    s = db.relocate_pinned(200_000)
    peeks = [c for c, p in shard.calls if p]
    assert [p for _, p in shard.calls] == [True] * len(peeks) + [False] and len(peeks) >= 2
    assert peeks == sorted(peeks) and shard.calls[-1][0] == peeks[-1]
    assert s["tail_after"] + 200_000 - s["floor_after"] <= 1 << 20 and s["agents"] == 4
    assert peeks == [300_000, 330_000]
    db.close()


def test_cut_search_jumps_past_an_agent_just_above_the_cut(tmp_path):
    # the second agent's oldest record sits 280 bytes above the first cut and each dry run leaves the room only 8 bytes
    # short: raising the cut by the shortfall would creep for 35 steps, the floor the dry run needed passes it at once
    G = 1 << 20
    shard = _PinnedLog(G, G + 50_000, {0: (100_000, 288), 1: (200_280, 288)})
    sdb, db = _db(tmp_path, shard)
    s = db.relocate_pinned(150_000)
    assert shard.calls == [(200_000, True), (200_288, True), (200_288, False)]
    assert s["agents"] == 2 and s["tail_after"] + 150_000 - s["floor_after"] <= G
    db.close()


def test_cut_search_ends_at_the_tail(tmp_path):
    # ten agents 8 kB apart, each with 9 kB live above its oldest record: every dry run passes one more agent and leaves
    # the room short by what the last one moved, so seven steps pass seven agents and the eighth must be the tail
    G = 1 << 20
    pinned = {a: (549_999 + 8_000 * a, 9_000) for a in range(10)}
    shard = _PinnedLog(G, G + 50_000, pinned)
    sdb, db = _db(tmp_path, shard)
    s = db.relocate_pinned(500_000)
    cuts = [c for c, p in shard.calls if p]
    assert cuts[:2] == [550_000, 557_999 + 1 + 1_000]
    assert [len([a for a, v in pinned.items() if v[0] < c]) for c in cuts] == [1, 2, 3, 4, 5, 6, 7, 10]
    assert cuts[-1] == G + 50_000 and shard.calls[-1] == (G + 50_000, False) and s["agents"] == 10
    db.close()


def test_cut_search_gives_up_and_changes_nothing(tmp_path):
    pinned = {a: (a * 100_000, 90_000) for a in range(9)}     # 810 kB live in 1 MiB: no cut frees 500 kB
    shard = _PinnedLog(1 << 20, 900_000, pinned)
    sdb, db = _db(tmp_path, shard)
    before = dict(shard.pinned), shard.tail
    with pytest.raises(sdb._native.SdbError) as e:
        db.relocate_pinned(500_000)
    assert e.value.code == -5
    assert all(p for _, p in shard.calls) and (dict(shard.pinned), shard.tail) == before
    db.close()


def test_refused_flush_relocates_and_retries_once(tmp_path):
    shard = _PinnedLog(1 << 20, 960 << 10, {0: (10_000, 1000)}, refuse=1)
    sdb, db = _db(tmp_path, shard, arena_relocate=True)
    db.register_agents(["a", "b"])
    mid = db.send_message("a", "hello", "b")
    db.flush()
    assert shard.sends == 2 and shard.calls[-1][1] is False
    assert [m.id for m in db.receive_messages("b")] == [mid]
    # refused again after the relocation: the existing failure path, no third attempt
    shard.refuse = 2
    mid2 = db.send_message("a", "again", "b")
    with pytest.raises(sdb._native.SdbError):
        db.flush()
    assert shard.sends == 4 and db.get_message(mid2).status == sdb.MessageStatus.FAILED
    mid3 = db.send_message("a", "fresh id", "b")
    assert mid3 not in (mid, mid2)
    db.close()


def test_no_retry_with_the_option_off(tmp_path):
    shard = _PinnedLog(1 << 20, 960 << 10, {0: (10_000, 1000)}, refuse=1)
    sdb, db = _db(tmp_path, shard)
    db.register_agents(["a", "b"])
    mid = db.send_message("a", "hello", "b")
    with pytest.raises(sdb._native.SdbError):
        db.flush()
    assert shard.sends == 1 and shard.calls == [] and db.get_message(mid).status == sdb.MessageStatus.FAILED
    db.close()


def test_sharded_refuses_the_option(tmp_path):
    import swarmdb_b200 as sdb
    from swarmdb_b200 import sharded
    cfg = sdb.GpuConfig(max_agents=64, max_groups=4, deterministic_ids=True, arena_relocate=True)
    with pytest.raises(NotImplementedError):
        sharded.ShardedSwarmsDB(0, 1, exchange_factory=object, shard=OracleShard(64, 4, 0, 1), save_dir=str(tmp_path),
                                auto_save=False, gpu_config=cfg)


def test_batch_bound_counts_every_copy(tmp_path):
    shard = _PinnedLog(1 << 20, 0, {})
    sdb, db = _db(tmp_path, shard, flush_threshold=1000)
    db.register_agents(["a", "b", "c", "d"])
    db.add_agent_group("g", ["a", "b", "c"])
    db.send_message("a", "x" * 40, "b")                        # 1 x (32 + 64)
    db.send_to_group("a", "g", "y" * 10)                       # 3 x (32 + 32): the bound counts the sender too
    db.broadcast_message("a", "z")                             # one copy per listed receiver
    n_bcast = db._b_list_off[-1] - db._b_list_off[-2]
    assert db._batch_bound() == 96 + 3 * 64 + n_bcast * 64
    db.close()
