"""GPU parity of the backend balancer (csrc/sdb_balance.cu) at the edges of its input space, against the sequential
definition in oracle/cpu_ref.c (itself pinned to exact rationals by tests/test_oracle_c.py).

Every call compares the picks AND the loads the device ends with, and every call starts from the loads the previous
one produced on the device (with completions released in between), so an error anywhere carries forward.

Edges covered: backend counts around the warp width, the 256-thread grid edge and the shared-memory sizes of each
pick kernel (k_ll_plan / k_ll_scatter ask for 20 B bytes, k_wr_pick for 12 B + 1028 bytes); equal weights (exact
ties everywhere), weights up to 65535, one heavy backend among light ones, one backend at the load cap; request counts
around the CTA size; costs 0 and up to 2^32 - 1; loads driven beyond 2^48, where load x weight needs more than
64 bits.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

BACKENDS = [1, 2, 31, 32, 33, 255, 1000, 2457, 2458, 4010, 4011, 4096]
WEIGHTS = ["equal", "u8", "u65535", "heavy", "one_light"]
LOADS = ["zero", "small", "cap", "one_at_cap"]
CAP = (1 << 40) - 1


def _weights(rng, kind, B):
    if kind == "equal":
        return np.full(B, 3, np.uint32)
    if kind == "u8":
        return rng.integers(1, 9, B).astype(np.uint32)
    if kind == "u65535":
        return rng.integers(1, 65536, B).astype(np.uint32)
    if kind == "heavy":
        w = rng.integers(1, 9, B).astype(np.uint32)
        w[int(rng.integers(0, B))] = 65535
        return w
    w = np.full(B, 65535, np.uint32)                 # one_light: backend 0 has weight 1, every other one 65535
    w[0] = 1
    return w


def _loads(rng, kind, B):
    if kind == "zero":
        return np.zeros(B, np.uint64)
    if kind == "small":
        return rng.integers(0, 50, B).astype(np.uint64)
    if kind == "cap":
        return rng.integers(0, CAP + 1, B, dtype=np.uint64)
    l0 = np.zeros(B, np.uint64)                       # one_at_cap: backend 0 at the cap, the rest empty
    l0[0] = CAP
    return l0


def _costs(rng, n):
    """Costs 0, small and up to 2^32 - 1, mixed."""
    c = rng.integers(1, 20, n).astype(np.uint32)
    c[rng.random(n) < 0.1] = 0
    big = rng.random(n) < 0.05
    c[big] = rng.integers(1 << 31, 1 << 32, int(big.sum()), dtype=np.uint64).astype(np.uint32)
    return c


def _pair(B):
    from oracle.cpu_ref import CpuOracle
    from swarmdb_b200._native import Shard
    g = Shard(max_agents=4, max_backends=B, arena_bytes=1 << 16, max_batch_sends=64, max_recv_records=1024,
              ring_slots=4, max_payload_bytes=64)
    return g, CpuOracle(4, 1)


def _release(g, c, w, rng, picks, cost):
    """Completion reports for a random part of the picks: the device folds them on the host side of the ABI, the
    oracle (which has no release) gets the same loads back through set_backends.  After costed picks those loads can
    exceed 2^40: the oracle's set_backends accepts any 64-bit load on purpose (the device's refuses initial loads of
    2^40 and more), and this helper depends on it."""
    k = int(min(len(picks), rng.integers(0, 64)))
    if k == 0:
        return
    sel = rng.choice(len(picks), size=k, replace=False)
    b = picks[sel].astype(np.uint32)
    cst = None if cost is None else cost[sel].astype(np.uint32)
    g.release_backends(b, cst)
    loads = [int(x) for x in c.backend_loads()]
    for i in range(k):
        d = 1 if cst is None else int(cst[i])
        loads[int(b[i])] = max(0, loads[int(b[i])] - d)
    c.set_backends(w, np.array(loads, np.uint64))


def _check(g, c, n, cost, mode, seed, what):
    pg = g.select_backends(n, cost, mode, seed)
    pc = c.select_backends(n, cost, mode, seed)
    if not np.array_equal(pg, pc):
        bad = int(np.nonzero(pg != pc)[0][0])
        raise AssertionError(f"{what}: first differing pick {bad}: device {pg[bad]} oracle {pc[bad]}")
    lg, lc = g.backend_loads(), c.backend_loads()
    assert np.array_equal(lg, lc), f"{what}: loads differ at {np.nonzero(lg != lc)[0][:8]}"
    return pg


def _requests(B, first):
    """Request counts per call: around the 256-thread CTA, one larger batch on the first combination only (the
    oracle is O(n B)), and 2^20 for a few small B."""
    ns = [1, 255, 256, 257]
    if first or B <= 33:
        ns.append(65537)
    if first and B in (1, 33, 255):
        ns.append(1 << 20)
    return ns


@pytest.mark.parametrize("path", ["unit", "costed", "random", "random_costed"])
@pytest.mark.parametrize("B", BACKENDS)
def test_balancer_matches_oracle_at_the_edges(B, path):
    """mode 0 unit cost (k_ll_plan + k_ll_scatter), mode 0 with costs (k_ll_seq), mode 1 with and without costs
    (k_wr_pick over many CTAs), for every weight and initial-load shape, several calls in a row on one handle."""
    rng = np.random.default_rng(B * 7 + len(path))
    mode = 1 if path.startswith("random") else 0
    with_cost = path in ("costed", "random_costed")
    g, c = _pair(B)
    try:
        first = True
        for wk in WEIGHTS:
            for lk in LOADS:
                w, l0 = _weights(rng, wk, B), _loads(rng, lk, B)
                g.set_backends(w, l0); c.set_backends(w, l0)
                for n in _requests(B, first):
                    if with_cost and mode == 0 and n > 65537:
                        continue                           # one warp, sequential: 2^20 costed picks take seconds
                    cost = _costs(rng, n) if with_cost else None
                    seed = int(rng.integers(0, 1 << 63))
                    picks = _check(g, c, n, cost, mode, seed, f"B={B} {path} w={wk} l={lk} n={n}")
                    _release(g, c, w, rng, picks, cost)
                first = False
        assert g.stats()["backend_picks"] > 0
    finally:
        g.close(); c.close()


@pytest.mark.parametrize("B", [2, 3, 40])
def test_balancer_loads_beyond_2_pow_48(B):
    """Costed picks with costs near 2^32 and weights 65535 push loads past 2^48, where load x weight no longer fits
    64 bits; unit-cost, costed and weighted-random picks from there must still equal the oracle's 128-bit compare."""
    rng = np.random.default_rng(B)
    g, c = _pair(B)
    try:
        w = np.full(B, 65535, np.uint32)
        w[-1] = int(rng.integers(1, 65535))
        l0 = rng.integers(CAP - 1000, CAP + 1, B, dtype=np.uint64)
        g.set_backends(w, l0); c.set_backends(w, l0)
        n = max(1 << 17, B << 16)                          # every backend gains about 2^48 per step
        for step in range(3):
            cost = rng.integers((1 << 32) - 4096, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
            _check(g, c, n, cost, 0, 0, f"B={B} costed step {step}")
            loads = g.backend_loads()
            for n2, cst, mode in ((257, None, 0), (4000, None, 0), (300, _costs(rng, 300), 0), (1000, None, 1),
                                  (700, _costs(rng, 700), 1)):
                _check(g, c, n2, cst, mode, step, f"B={B} step {step} n={n2} mode={mode} cost={cst is not None}")
        assert int(loads.max()) >= 1 << 49, loads.max()
        if B <= 3:
            # equal weights, equal loads beyond 2^48: exact ties everywhere, lowest index first
            wq = np.full(B, 65535, np.uint32)
            g.set_backends(wq); c.set_backends(wq)
            nt = B << 17
            _check(g, c, nt, np.full(nt, (1 << 32) - 1, np.uint32), 0, 0, f"B={B} lockstep")
            assert len(set(g.backend_loads().tolist())) == 1 and int(g.backend_loads()[0]) > 1 << 48
            _check(g, c, 4 * B + 1, None, 0, 0, f"B={B} unit ties")
            _check(g, c, 4 * B + 1, np.full(4 * B + 1, 7, np.uint32), 0, 0, f"B={B} costed ties")
    finally:
        g.close(); c.close()


def test_balancer_refuses_more_backends_than_it_can_hold():
    """sdb_create rejects max_backends above SDB_MAX_BACKENDS (4096) instead of failing every pick later; at the bound
    the handle works and set_backends refuses more backends than the handle was made for."""
    from swarmdb_b200._native import SdbError, Shard
    with pytest.raises(SdbError) as ei:
        Shard(max_agents=4, max_backends=4097, arena_bytes=1 << 16, max_recv_records=1024)
    assert ei.value.code == -1
    g, c = _pair(4096)
    try:
        with pytest.raises(SdbError):
            g.set_backends(np.ones(4097, np.uint32))
        with pytest.raises(SdbError):
            g.set_backends(np.array([1, 0], np.uint32))            # weight 0
        with pytest.raises(SdbError):
            g.set_backends(np.array([1, 1], np.uint32), np.array([0, 1 << 40], np.uint64))
        w = np.ones(4096, np.uint32)
        g.set_backends(w); c.set_backends(w)
        _check(g, c, 5000, None, 0, 0, "B=4096 after refusals")
    finally:
        g.close(); c.close()
