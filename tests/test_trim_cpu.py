"""Bounded queues (sdb_trim) without a GPU: the model of tests/trim_ref.py on hand-written queues, the argument checks of
GpuConfig and SwarmsDB.trim_queues, and POST /admin/trim over HTTP against an oracle-backed shard that can trim."""
import numpy as np
import pytest

from oracle.cpu_ref import HDR_DTYPE
from tests.fake_shard import OracleShard
from tests.trim_ref import RECV_PRIORITY, TrimmingOracle, trim_drops, trim_select


def _queue(*recs):
    """[(header, payload)] from (prio, len) pairs; seq = position."""
    out = []
    for i, (p, n) in enumerate(recs):
        h = np.zeros(1, HDR_DTYPE)[0]
        h["prio"], h["len"], h["seq"] = p, n, i
        out.append((h, bytes((n + 31) & ~31)))
    return out


def test_count_bytes_and_both():
    q = _queue((1, 10), (1, 40), (1, 100), (1, 0), (1, 64))         # pad32: 32, 64, 128, 0, 64 = 288
    assert trim_drops(q, 3, 0, 0) == [0, 1]
    assert trim_drops(q, 5, 0, 0) == []
    assert trim_drops(q, 0, 192, 0) == [0, 1]                         # 288 - 96 = 192: exact fit
    assert trim_drops(q, 0, 191, 0) == [0, 1, 2]                      # rounded down to 160
    assert trim_drops(q, 0, 288, 0) == []
    assert trim_drops(q, 4, 100, 0) == [0, 1, 2]                      # bytes bind after the count
    assert trim_drops(q, 1, 1000, 0) == [0, 1, 2, 3]                  # count binds after the bytes
    assert trim_drops(q, 0, 31, 0) == [0, 1, 2, 3, 4]                 # 0 granules: a prefix, so the 0-byte record goes too
    assert trim_drops(_queue((1, 1), (1, 0)), 0, 31, 0) == [0]        # ... unless it is all that is left


def test_priority_order_with_ties_across_levels():
    q = _queue((2, 32), (0, 32), (3, 32), (0, 32), (1, 32), (2, 32), (1, 32))
    assert trim_drops(q, 3, 0, RECV_PRIORITY) == [1, 3, 4, 6]         # level 0 oldest first, then level 1
    assert trim_drops(q, 2, 0, RECV_PRIORITY) == [1, 3, 4, 6, 0]      # then the oldest of level 2
    assert trim_drops(q, 0, 96, RECV_PRIORITY) == [1, 3, 4, 6]
    assert trim_drops(q, 3, 0, 0) == [0, 1, 2, 3]


def test_single_oversized_record_and_empty_agents():
    q = _queue((3, 500))
    assert trim_drops(q, 0, 256, 0) == [0]
    assert trim_drops(q, 0, 512, 0) == []
    assert trim_drops([], 1, 32, RECV_PRIORITY) == []
    counts, chosen = trim_select({5: q}, [1, 5, 9], 0, 256, 0, 100)
    assert counts == [0, 1, 0] and chosen == [(5, 0)]


def test_capacity_rule_and_stream_order_output():
    state = {0: _queue(*[(p % 4, 32) for p in range(10)]), 1: _queue(*[(0, 32)] * 4), 2: _queue(*[(1, 32)] * 6)}
    counts, chosen = trim_select(state, [0, 1, 2], 2, 0, RECV_PRIORITY, 5)
    # agent 0 evicts levels 0 (0, 4, 8) then 1 (1, 5, 9) then 2 (2, 6): 8 drops, 5 fit; the rest stays whole
    assert counts == [5, 0, 0] and chosen == [(0, 0), (0, 1), (0, 4), (0, 5), (0, 8)]
    counts, chosen = trim_select(state, [1, 0, 2], 2, 0, 0, 9)
    assert counts == [2, 0, 0] and chosen == [(1, 0), (1, 1)]        # agent 0's 8 do not fit behind agent 1's 2


@pytest.mark.parametrize("seed", range(6))
def test_archive_calls_until_empty_equal_one_drop_call(seed):
    rng = np.random.default_rng(seed)
    state = {a: _queue(*[(int(rng.integers(0, 4)), int(rng.integers(0, 300))) for _ in range(int(rng.integers(0, 30)))])
             for a in range(12)}
    agents = rng.permutation(12)
    n, b = int(rng.integers(0, 6)), int(rng.integers(0, 2000))
    if n == 0 and b == 0:
        n = 2
    flags = RECV_PRIORITY if seed % 2 else 0
    _, once = trim_select(state, agents, n, b, flags, 1 << 60)
    left = {a: list(enumerate(q)) for a, q in state.items()}          # (original position, record)
    taken = set()
    for _ in range(1000):
        cur = {a: [r for _, r in lst] for a, lst in left.items()}
        _, chosen = trim_select(cur, agents, n, b, flags, int(rng.integers(1, 8)))
        if not chosen:
            break
        gone = set(chosen)
        for a, i in chosen:
            taken.add((a, left[a][i][0]))
        left = {a: [x for i, x in enumerate(lst) if (a, i) not in gone] for a, lst in left.items()}
    assert taken == set(once)


def test_gpu_config_and_trim_queues_refuse_bad_values_before_any_device_call(tmp_path):
    import swarmdb_b200 as sdb
    from swarmdb_b200.core import _trim_limits

    class NoDevice:
        def __getattr__(self, name):
            raise AssertionError(f"device call {name} before the arguments were checked")
    for bad in (dict(queue_max_messages=-1), dict(queue_max_messages=1 << 32), dict(queue_max_bytes=-5),
                dict(queue_max_bytes=1 << 64), dict(queue_max_messages=2.5), dict(queue_trim_priority=1)):
        with pytest.raises(ValueError):
            sdb.SwarmsDB(save_dir=str(tmp_path), auto_save=False, _shard=NoDevice(), gpu_config=sdb.GpuConfig(**bad))
    for args in ((None, None), (0, None), (None, 0), (-1, 10), (True, None), (1 << 32, None), (3, 1 << 64), ("3", None)):
        with pytest.raises(ValueError):
            _trim_limits(*args)
    assert _trim_limits(3, None) == (3, 0) and _trim_limits(None, 512) == (0, 512)
    db = sdb.SwarmsDB(save_dir=str(tmp_path), auto_save=False, _shard=TrimShard(16, 2, 0, 1),
                      gpu_config=sdb.GpuConfig(max_agents=16, max_groups=2, deterministic_ids=True))
    db.shard = NoDevice()
    with pytest.raises(ValueError):
        db.trim_queues()
    with pytest.raises(ValueError):
        db.trim_queues(max_messages=0)


class TrimShard(OracleShard):
    """The oracle-backed stand-in shard with drop-mode trimming (tests/trim_ref.py)."""

    def __init__(self, max_agents, max_groups, rank, world):
        super().__init__(max_agents, max_groups, rank, world)
        self.o = TrimmingOracle(self.o, max_groups, watermark=max_agents)

    def trim(self, agents, max_records=0, max_bytes=0, flags=0, archive=True, **kw):
        assert not archive
        return self.o.trim(agents, max_records, max_bytes, flags & RECV_PRIORITY, materialise=False)


def test_automatic_caps_on_the_oracle_shard(tmp_path):
    import swarmdb_b200 as sdb
    db = sdb.SwarmsDB(save_dir=str(tmp_path), auto_save=False, _shard=TrimShard(16, 2, 0, 1),
                      gpu_config=sdb.GpuConfig(max_agents=16, max_groups=2, deterministic_ids=True, queue_max_messages=2))
    db.register_agent("a"); db.register_agent("b")
    for i in range(5):
        db.send_message("a", f"m{i}", receiver_id="b")
    db.flush()
    assert db.get_stats()["trimmed"] == 3
    assert [m.content for m in db.receive_messages("b")] == ["m3", "m4"]
    db.close()


def test_admin_trim_over_http(tmp_path):
    pytest.importorskip("fastapi"); pytest.importorskip("jwt"); pytest.importorskip("httpx")
    import swarmdb_b200 as sdb
    from fastapi.testclient import TestClient
    from swarmdb_b200.server import Settings, create_app
    db = sdb.SwarmsDB(save_dir=str(tmp_path), auto_save=False, _shard=TrimShard(64, 4, 0, 1),
                      gpu_config=sdb.GpuConfig(max_agents=64, max_groups=4, deterministic_ids=True))
    c = TestClient(create_app(db, Settings(history_dir=str(tmp_path))))

    def token(user):
        r = c.post("/auth/token", json={"username": user, "password": "pw"})
        return {"Authorization": f"Bearer {r.json()['access_token']}"}
    a1, adm = token("a1"), token("admin")
    for who in ("a1", "a2", "a3"):
        db.register_agent(who)
    for i in range(6):
        db.send_message("a1", f"x{i}", receiver_id="a2", priority=sdb.MessagePriority.HIGH if i == 0 else sdb.MessagePriority.LOW)
        db.send_message("a1", f"y{i}", receiver_id="a3")
    assert c.post("/admin/trim", json={"max_messages": 2}, headers=a1).status_code == 403
    assert c.post("/admin/trim", json={}, headers=adm).status_code == 422
    assert c.post("/admin/trim", json={"max_messages": -1}, headers=adm).status_code == 422
    r = c.post("/admin/trim", json={"max_messages": 2, "by_priority": True, "agent_ids": ["a2"]}, headers=adm)
    assert r.status_code == 200 and r.json() == {"trimmed": 4}
    assert [m.content for m in db.receive_messages("a2")] == ["x0", "x5"]
    r = c.post("/admin/trim", json={"max_bytes": 64}, headers=adm)   # every "yN" pads to 32 bytes
    assert r.status_code == 200 and r.json() == {"trimmed": 4}
    assert [m.content for m in db.receive_messages("a3")] == ["y4", "y5"]
    db.close()
