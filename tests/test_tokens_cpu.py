"""Receive by token budget without a device: the take rule of tests/tokens_ref.py on hand-computed cases, and the
SwarmsDB front end (the token-count wire form, its decoding and the max_tokens receive arguments) on an oracle-backed
shard whose token calls follow the model."""
import json
import re
from pathlib import Path

import numpy as np
import pytest

from tests.fake_shard import OracleShard
from tests.tokens_ref import call_counts, token_take, weight

ROOT = Path(__file__).resolve().parents[1]
PEEK, PRIORITY = 2, 1


# ---- the model ---------------------------------------------------------------------------------------------------
def test_first_record_alone_when_heavier():
    assert token_take([10, 1, 1], 5) == 1
    assert token_take([10], 1) == 1
    assert token_take([], 5) == 0


def test_zero_weight_records_are_free():
    assert token_take([0, 0, 3, 0, 5], 3) == 4
    assert token_take([0, 0, 0], 1) == 3
    assert token_take([7, 0, 0, 1], 7) == 3          # the run stops at the first record that does not fit
    assert token_take([4, 4, 4], 0) == 3             # 0: no token limit


def test_limits_at_and_around_prefix_sums():
    w = [3, 5, 2, 7]
    for lim, want in [(3, 1), (7, 1), (8, 2), (9, 2), (10, 3), (16, 3), (17, 4), (1 << 40, 4)]:
        assert token_take(w, lim) == want, lim


def _level_rule(recs, lim):
    """The priority-order take as the device computes it: whole levels from the top while they fit, then the
    arrival-order prefix of the level where the limit falls (recs: (prio, weight) in arrival order)."""
    take, used = 0, 0
    for level in (3, 2, 1, 0):
        ws = [w for p, w in recs if p == level]
        if used + sum(ws) <= lim:
            take += len(ws); used += sum(ws)
            continue
        for w in ws:
            if used + w > lim and take > 0:
                break
            take += 1; used += w
        break
    return take


def test_priority_level_cut():
    recs = [(0, 5), (3, 2), (1, 4), (3, 3), (1, 1)]
    order = [w for _, w in sorted(recs, key=lambda r: -r[0])]      # stable: arrival order within a level
    assert order == [2, 3, 4, 1, 5]
    assert token_take(order, 9) == _level_rule(recs, 9) == 3       # level 3 whole, the first record of level 1
    assert token_take(order, 10) == _level_rule(recs, 10) == 4     # levels 3 and 1 whole
    assert token_take(order, 4) == _level_rule(recs, 4) == 1       # cut inside level 3
    assert token_take(order, 1) == _level_rule(recs, 1) == 1       # heavier first record alone
    rng = np.random.default_rng(3)
    for _ in range(2000):
        n = int(rng.integers(0, 12))
        recs = [(int(rng.integers(0, 4)), int(rng.choice([0, 1, 2, 5, 9, 100]))) for _ in range(n)]
        order = [w for _, w in sorted(recs, key=lambda r: -r[0])]
        lim = int(rng.integers(1, 40))
        assert token_take(order, lim) == _level_rule(recs, lim)


def test_joint_byte_and_token_take_is_the_shorter():
    # (len, weight): bytes count pad32(len)
    recs = [(40, 1), (40, 1), (40, 1), (40, 100), (10, 0)]
    assert call_counts([recs], 100, 0, 2, 1 << 20, 1 << 30) == [2]          # tokens cut first
    assert call_counts([recs], 100, 64, 0, 1 << 20, 1 << 30) == [1]         # bytes cut first (64 B per record)
    assert call_counts([recs], 100, 128, 3, 1 << 20, 1 << 30) == [2]        # both: the shorter run
    assert call_counts([recs], 100, 192, 3, 1 << 20, 1 << 30) == [3]
    assert call_counts([recs], 2, 0, 1000, 1 << 20, 1 << 30) == [2]         # max_messages
    assert call_counts([recs], 100, 0, 0, 1 << 20, 1 << 30) == [5]          # no limits
    assert call_counts([[(40, 10)] + recs], 100, 32, 5, 1 << 20, 1 << 30) == [1]   # the first record alone


def test_lead_agent_truncation_under_record_and_byte_caps():
    a = [(32, 1)] * 6
    b = [(32, 1)] * 3
    # the first agent's take (5 tokens) does not fit 4 records: it takes 4, the next agent stays queued
    assert call_counts([a, b], 100, 0, 5, 4, 1 << 30) == [4, 0]
    # ... nor 96 bytes: 3 records
    assert call_counts([a, b], 100, 0, 5, 100, 96) == [3, 0]
    # an agent after the first that does not fit stays queued with every later one
    assert call_counts([b, a, b], 100, 0, 5, 8, 1 << 30) == [3, 5, 0]
    assert call_counts([b, a, b], 100, 0, 5, 7, 1 << 30) == [3, 0, 0]
    # an empty agent takes nothing and does not close the call
    assert call_counts([[], a], 100, 0, 2, 4, 1 << 30) == [0, 2]


def test_weight_reads_only_tagged_records_of_four_bytes_or_more():
    assert weight(0x40, (7).to_bytes(4, "little") + b"abc") == 7
    assert weight(0x40 | 0x10, (2 ** 32 - 1).to_bytes(4, "little")) == 2 ** 32 - 1
    assert weight(0x00, (7).to_bytes(4, "little")) == 0
    assert weight(0x40, b"\x07\x00\x00") == 0


def test_header_flag_matches_the_binding():
    from swarmdb_b200 import _native
    h = (ROOT / "include" / "swarmdb_b200.h").read_text()
    m = re.search(r"#define SDB_TYPEF_TOKENS (0x[0-9a-fA-F]+)u", h)
    assert m and int(m.group(1), 16) == _native.TYPEF_TOKENS == 0x40
    flags = [int(x, 16) for x in re.findall(r"#define SDB_TYPEF_\w+ (0x[0-9a-fA-F]+)u", h)]
    assert len(flags) == len(set(flags)) and all(f & 0x07 == 0 for f in flags)   # distinct, clear of the type code
    for name in ("sdb_receive_tokens", "sdb_receive_compact_tokens", "sdb_pending_tokens"):
        assert name in _native.EXPORTS and re.search(rf"\bint {name}\(", h)


# ---- the front end on an oracle-backed shard ----------------------------------------------------------------------
class TokenShard(OracleShard):
    """OracleShard with the token calls of _native.Shard, computed by tests/tokens_ref.py over a PEEK and served by the
    oracle's plain receive (the equivalence the device promises)."""
    max_recv_records = 1 << 20

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.calls = []

    def _orders(self, agents, flags):
        from swarmdb_b200._native import payload_offsets
        cnt, hdr, pay = self.o.receive_batch(agents, 1 << 20, (flags & PRIORITY) | PEEK)
        offs, raw, out, pos = payload_offsets(hdr), pay.tobytes(), [], 0
        for c in cnt.astype(int):
            out.append([(int(hdr["len"][i]), weight(int(hdr["type"][i]), raw[int(offs[i]):int(offs[i]) + int(hdr["len"][i])]))
                        for i in range(pos, pos + c)])
            pos += c
        return out

    def receive_tokens(self, agents, max_messages, max_agent_tokens, max_agent_bytes=0, flags=0):
        self.calls.append((list(agents), max_messages, max_agent_tokens, max_agent_bytes, flags))
        want = call_counts(self._orders(agents, flags), max_messages, max_agent_bytes, max_agent_tokens, 1 << 20, 1 << 40)
        hs, ps = [], []
        for a, k in zip(agents, want):
            if k:
                _, h, p = self.o.receive_batch([a], k, flags)
                hs.append(h.copy()); ps.append(p.copy())
        if not hs:
            _, h, p = self.o.receive_batch([agents[0]], 1, PEEK)
            return np.array(want, np.uint32), h[:0], p[:0]
        return np.array(want, np.uint32), np.concatenate(hs), np.concatenate(ps)

    def pending_tokens(self, agents=None, n=None):
        return np.array([sum(w for _, w in recs) for recs in self._orders(list(agents), 0)], np.uint64)

    def peek_raw(self, agent):
        from swarmdb_b200._native import payload_offsets
        _, hdr, pay = self.o.receive_batch([agent], 1 << 10, PEEK)
        offs, raw = payload_offsets(hdr), pay.tobytes()
        return [(int(h["type"]), raw[int(o):int(o) + int(h["len"])]) for h, o in zip(hdr, offs)]


def _db(tmp_path, token_counter=len, **kw):
    import swarmdb_b200 as sdb
    shard = TokenShard(64, 4, 0, 1)
    db = sdb.SwarmsDB(save_dir=str(tmp_path), auto_save=False, _shard=shard, token_counter=token_counter,
                      gpu_config=sdb.GpuConfig(max_agents=64, max_groups=4, deterministic_ids=True, **kw))
    return db, shard


def _legacy_payload(content, extras):
    """The wire form before token counts had their own place: content bytes, or u32 len | content | JSON extras."""
    body = json.dumps(content).encode() if isinstance(content, (dict, list)) else content.encode()
    if not extras:
        return body
    return len(body).to_bytes(4, "little") + body + json.dumps(extras).encode()


CONTENTS = ["hello world", "", "héllo ∑", {"task": "plan", "steps": [1, 2, 3]}, [1, "two", {"three": 3}], []]


@pytest.mark.parametrize("with_metadata", [False, True])
def test_wire_round_trip_with_token_counts(tmp_path, with_metadata):
    from swarmdb_b200._native import TYPEF_EXTRAS, TYPEF_TOKENS
    db, shard = _db(tmp_path)
    db.register_agent("b")
    md = {"k": "v"} if with_metadata else None
    for c in CONTENTS:
        db.send_message("a", c, "b", metadata=dict(md) if md else None)
    db.flush()
    raw = shard.peek_raw(db.agent_index("b"))
    for c, (typ, p) in zip(CONTENTS, raw):
        text = json.dumps(c) if isinstance(c, (dict, list)) else c
        assert typ & TYPEF_TOKENS and int.from_bytes(p[:4], "little") == len(text)
        assert bool(typ & TYPEF_EXTRAS) == with_metadata
        assert p[4:] == _legacy_payload(c, {"m": md} if md else {})          # the rest is the untagged form
        assert len(p) < len(_legacy_payload(c, dict({"m": md} if md else {}, t=len(text))))
    got = db.receive_messages("b")
    assert [m.content for m in got] == CONTENTS
    assert [m.token_count for m in got] == [len(json.dumps(c) if isinstance(c, (dict, list)) else c) for c in CONTENTS]
    if with_metadata:
        assert all(m.metadata == md for m in got)
    db.close()


def test_wire_round_trip_of_broadcasts_and_group_sends(tmp_path):
    from swarmdb_b200._native import TYPEF_EXTRAS, TYPEF_TOKENS
    db, shard = _db(tmp_path)
    for a in ("a", "b", "c"):
        db.register_agent(a)
    db.add_agent_group("g", ["a", "b", "c"])
    db.broadcast_message("a", {"x": 1})                                      # visibility travels in the extras
    db.send_to_group("a", "g", "to the group", metadata={"r": 2})
    db.flush()
    (t0, p0), (t1, p1) = shard.peek_raw(db.agent_index("b"))
    assert t0 & TYPEF_TOKENS and t0 & TYPEF_EXTRAS and int.from_bytes(p0[:4], "little") == len('{"x": 1}')
    assert t1 & TYPEF_TOKENS and int.from_bytes(p1[:4], "little") == len("to the group")
    m0, m1 = db.receive_messages("b")
    assert m0.content == {"x": 1} and m0.token_count == 8 and sorted(m0.visible_to) == ["b", "c"]
    assert m1.content == "to the group" and m1.token_count == 12 and m1.metadata == {"r": 2, "group": "g"}
    db.close()


def test_messages_without_a_token_count_encode_as_before(tmp_path):
    from swarmdb_b200._native import TYPEF_TOKENS
    db, shard = _db(tmp_path, token_counter=None)
    db.register_agent("b"); db.register_agent("c")
    db.send_message("a", "plain", "b")
    db.send_message("a", {"d": [1]}, "b", metadata={"m": 1})
    bid = db.broadcast_message("a", "all")
    db.flush()
    raw = shard.peek_raw(db.agent_index("b"))
    assert [p for _, p in raw] == [_legacy_payload("plain", {}), _legacy_payload({"d": [1]}, {"m": {"m": 1}}),
                                   _legacy_payload("all", {"v": db.get_message(bid).visible_to})]
    assert not any(t & TYPEF_TOKENS for t, _ in raw)
    assert [m.token_count for m in db.receive_messages("b")] == [None, None, None]
    db.close()


def test_decode_still_reads_counts_from_the_extras(tmp_path):
    """Snapshots and history written before counts moved to the prefix carry them as "t" in the extras."""
    from swarmdb_b200._native import TYPEF_EXTRAS
    db, shard = _db(tmp_path, token_counter=None)
    b = db.agent_index("b"); a = db.agent_index("a")
    payload = np.frombuffer(_legacy_payload("old", {"t": 17}), np.uint8)
    shard.o.send_batch(np.array([a], np.uint32), np.array([b], np.uint32), np.array([1], np.uint8),
                     np.array([TYPEF_EXTRAS], np.uint8), np.array([len(payload)], np.uint16), np.zeros(1, np.uint64), payload)
    db.register_agent("b")
    (m,) = db.receive_messages("b")
    assert m.content == "old" and m.token_count == 17
    db.close()


@pytest.mark.parametrize("bad", [-1, 2 ** 32, 2 ** 40, 1.5, "3"])
def test_a_count_outside_u32_is_refused_at_send(tmp_path, bad):
    db, shard = _db(tmp_path, token_counter=lambda text: bad)
    db.register_agent("b")
    db.add_agent_group("g", ["a", "b"])
    n = len(db.messages)
    with pytest.raises(ValueError, match="token_count"):
        db.send_message("a", "x", "b")
    with pytest.raises(ValueError, match="token_count"):
        db.send_to_group("a", "g", "x")
    db.flush()
    assert len(db.messages) == n and shard.peek_raw(db.agent_index("b")) == []
    db.close()


def test_receive_and_peek_by_tokens(tmp_path):
    db, shard = _db(tmp_path, token_counter=lambda text: int(text.split()[0]))
    db.register_agent("b")
    for c in ["3 x", "4 x", "0 x", "2 x", "9 x", "1 x"]:
        db.send_message("a", c, "b")
    db.send_message("a", "0 free", "b")
    peek = db.peek_messages("b", max_tokens=7)
    assert [m.content for m in peek] == ["3 x", "4 x", "0 x"]
    got = db.receive_messages("b", max_tokens=7)
    assert [m.content for m in got] == ["3 x", "4 x", "0 x"] and [m.token_count for m in got] == [3, 4, 0]
    assert shard.calls[-1][2:4] == (7, 0)                                    # no byte limit
    assert db.pending_tokens(["b", "nobody"]) == {"b": 12, "nobody": 0}
    assert [m.content for m in db.receive_messages("b", max_tokens=1)] == ["2 x"]          # heavier first alone
    assert [m.content for m in db.receive_messages("b", max_tokens=5, max_bytes=32)] == ["9 x"]
    assert shard.calls[-1][2:4] == (5, 32)
    assert [m.content for m in db.receive_messages("b", max_tokens=100, max_messages=1)] == ["1 x"]
    assert db.pending_tokens() == {"a": 0, "b": 0}
    with pytest.raises(ValueError, match="max_tokens"):
        db.receive_messages("b", max_tokens=0)
    n = len(shard.calls)
    assert [m.content for m in db.receive_messages("b")] == ["0 free"]      # None keeps the plain receive
    assert len(shard.calls) == n
    db.close()
