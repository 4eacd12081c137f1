"""At-scale content parity (SURVEY section 4, tiers T3/T4): the CUDA path against oracle/cpu_ref.c at the sizes
BASELINE.json quotes, compared through per-agent STREAM DIGESTS (include/swarmdb_b200.h): an order-sensitive
hash chain over every delivered record's 32-byte header and padded payload.  Equal digests for every agent mean
equal per-agent delivery order, header fields and payload bytes (reference contract: drain loop M:553-601,
filter M:579-585, fan-out loop M:1267-1277).  The digest definition itself is pinned on the CPU by
tests/test_oracle_c.py::test_stream_digest_definition_and_mt_path and, here, by a direct comparison of the
device digest with a host-side recomputation from the records the GPU returned.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ALNUM = np.frombuffer(b"ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789", np.uint8)


def _mismatch(dg, dc):
    bad = np.nonzero(dg != dc)[0]
    return f"{len(bad)} agents differ, first {bad[:8].tolist()}" if len(bad) else ""


def test_device_digest_equals_host_recomputation_of_returned_records():
    """Small case where both sides keep the records: digest(device results) == digest(D2H copy) == oracle."""
    from oracle.cpu_ref import CpuOracle
    from swarmdb_b200._native import RECV_PRIORITY, Shard
    from tests.test_oracle_c import _np_digest
    rng = np.random.default_rng(3)
    A, G, F = 2048, 32, 64
    gpu, cpu = Shard(max_agents=A, max_groups=G, ring_slots=256, arena_bytes=1 << 26), CpuOracle(A, G)
    perm = rng.permutation(A)
    for g in range(G):
        gpu.create_group(g, perm[g * F:(g + 1) * F]); cpu.create_group(g, perm[g * F:(g + 1) * F])
    cpu.digest_enable(); gpu.digest_reset()
    M, K = (1 << 64) - 1, 0x9E3779B97F4A7C15
    want = np.zeros(A, np.uint64)
    for rnd, flags in enumerate((0, RECV_PRIORITY, 0)):
        n = 400
        lens = rng.integers(0, 257, n).astype(np.uint16)
        off = np.arange(n, dtype=np.uint64) * 256
        buf = rng.integers(0, 256, n * 256 + 64).astype(np.uint8)
        s, g = rng.integers(0, A, n), rng.integers(0, G, n)
        prio, typ = rng.integers(0, 4, n), rng.integers(0, 7, n)
        gpu.send_group_batch(s, g, prio, typ, lens, off, buf); cpu.send_group_batch(s, g, prio, typ, lens, off, buf)
        idx = rng.permutation(A)[: A // 2].astype(np.uint32)            # a listed subset, in scrambled order
        cnt, hdr, pay = gpu.receive_batch(idx, 9, flags)
        gpu.digest_fold()
        cc, hc, pc = cpu.receive_batch(idx, 9, flags)
        assert np.array_equal(cnt, cc) and hdr.tobytes() == hc.tobytes() and pay.tobytes() == pc.tobytes()
        rh, r = _np_digest(hdr, pay), 0
        for q, a in enumerate(idx):
            d = int(want[a])
            for _ in range(int(cnt[q])):
                d = ((((d << 5) | (d >> 59)) & M) ^ rh[r]) * K & M
                r += 1
            want[a] = d
    dg = gpu.digest_read()
    assert not _mismatch(dg, want), _mismatch(dg, want)
    assert np.array_equal(cpu.digest_read(), want)
    some = rng.integers(0, A, 50).astype(np.uint32)
    assert np.array_equal(gpu.digest_read(some), want[some])
    gpu.close(); cpu.close()


@pytest.mark.parametrize("variant,fixed", [(2, False), (2, True), (3, False)])
def test_c2_full_batch_matches_oracle(variant, fixed):
    """BASELINE config 2 at full size: 1M agents, 15,625 groups x 64, one batch of 65,536 group sends
    (4,194,304 routed records), payload lengths U[1,256] (SURVEY 8d 'correctness variant') or fixed 256 (the timed
    shape), full drain; a second batch is enqueued BEFORE the first drain completes its follow-up drain so rings
    hold entries of two batches."""
    from bench import Workload
    from oracle.cpu_ref import CpuOracle
    from swarmdb_b200._native import Shard
    wl = Workload()
    gpu = Shard(max_agents=wl.A, ring_slots=64, arena_bytes=1 << 32, max_payload_bytes=wl.L, max_groups=1 << 14,
                member_pool_entries=wl.A + 1024, max_batch_sends=wl.S, max_batch_payload=wl.S * wl.L,
                max_recv_records=wl.S * wl.F * 2 + (1 << 16), max_recv_payload=(wl.S * wl.F * 2 + (1 << 16)) * wl.L,
                fanout_variant=variant)
    cpu = CpuOracle(wl.A, wl.G)
    gpu.register(np.arange(wl.A, dtype=np.uint32))
    for g in range(wl.G):
        gpu.create_group(g, wl.members(g)); cpu.create_group(g, wl.members(g))
    cpu.digest_enable(); gpu.digest_reset()
    rng = np.random.default_rng(8)

    def batch():
        snd, grp, prio, typ, lens, off, payload = wl.batch()
        if not fixed:
            lens = rng.integers(1, wl.L + 1, wl.S).astype(np.uint16)
        return snd, grp, prio, typ, lens, off, payload

    b1, b2 = batch(), batch()
    assert gpu.send_group_batch(*b1) == cpu.send_group_batch(*b1)[0]
    assert gpu.send_group_batch(*b2) == cpu.send_group_batch(*b2)[0]
    # first call takes at most 5 per agent (leaves a remainder in most rings), second call drains
    for k in (5, 100):
        _, total, _ = gpu.receive_batch(None, k, 0, copy_out=False)
        gpu.digest_fold()
        _, ctotal = cpu.receive_counts(None, k, 0)
        assert total == ctotal
    st = gpu.stats()
    assert st["ring_overflow"] == 0 and st["delivered"] == 2 * wl.S * wl.F
    dg, dc = gpu.digest_read(), cpu.digest_read()
    assert int((dc != 0).sum()) > 0.99 * wl.A
    assert not _mismatch(dg, dc), _mismatch(dg, dc)
    gpu.close(); cpu.close()


def test_c2_full_batch_priority_receive_matches_oracle():
    """The c2 construction (1M agents, two batches of 65,536 group sends to groups of 64) drained in PRIORITY order
    with k = 5, then k = 100.  The record bound min(n k, capacity) is above 4 x 2^20, so the payload scan's k_scan_tops
    sweeps more than 1024 tiles of 4096 records, and k_recv_select_big selects for every one of the 1M agents."""
    from bench import Workload
    from oracle.cpu_ref import CpuOracle
    from swarmdb_b200._native import RECV_PRIORITY, Shard
    wl = Workload()
    cap = wl.S * wl.F * 2 + (1 << 16)
    assert min(wl.A * 5, cap) > 1024 * 4096                       # tiles of 4096 records, 1024 tiles per sweep
    gpu = Shard(max_agents=wl.A, ring_slots=64, arena_bytes=1 << 32, max_payload_bytes=wl.L, max_groups=1 << 14,
                member_pool_entries=wl.A + 1024, max_batch_sends=wl.S, max_batch_payload=wl.S * wl.L,
                max_recv_records=cap, max_recv_payload=cap * wl.L)
    cpu = CpuOracle(wl.A, wl.G)
    gpu.register(np.arange(wl.A, dtype=np.uint32))
    for g in range(wl.G):
        gpu.create_group(g, wl.members(g)); cpu.create_group(g, wl.members(g))
    cpu.digest_enable(); gpu.digest_reset()
    rng = np.random.default_rng(9)
    for _ in range(2):
        snd, grp, prio, typ, lens, off, payload = wl.batch()
        prio = rng.integers(0, 4, wl.S).astype(np.uint8)                  # four levels: the selection has work to do
        lens = rng.integers(1, wl.L + 1, wl.S).astype(np.uint16)
        assert gpu.send_group_batch(snd, grp, prio, typ, lens, off, payload) == \
            cpu.send_group_batch(snd, grp, prio, typ, lens, off, payload)[0]
    gpu.profile(True)
    for k in (5, 100):
        _, total, _ = gpu.receive_batch(None, k, RECV_PRIORITY, copy_out=False)
        assert gpu.profile_read()["recv_count"][1] == 1                    # the priority pipeline served it
        gpu.digest_fold()
        _, ctotal = cpu.receive_counts(None, k, RECV_PRIORITY)
        assert total == ctotal
    st = gpu.stats()
    assert st["ring_overflow"] == 0 and st["delivered"] == 2 * wl.S * wl.F
    dg, dc = gpu.digest_read(), cpu.digest_read()
    assert int((dc != 0).sum()) > 0.99 * wl.A
    assert not _mismatch(dg, dc), _mismatch(dg, dc)
    gpu.close(); cpu.close()


@pytest.mark.parametrize("priority", [True, False])
def test_c4_sweeps_until_empty_match_oracle(priority):
    """BASELINE config 4 shape: ~10k agents, 2,048 pending records each, 4 priority levels; receive 100 per agent
    per sweep until empty (PRIORITY: segmented radix-select + tombstones; FIFO: stream order), more traffic
    arriving between sweeps."""
    from oracle.cpu_ref import CpuOracle
    from swarmdb_b200._native import RECV_PRIORITY, Shard
    rng = np.random.default_rng(4)
    G, F, L = 156, 64, 256
    A = G * F                                              # 9,984 agents
    per_group = 2048
    gpu = Shard(max_agents=A, ring_slots=4096, arena_bytes=1 << 33, max_payload_bytes=L, max_groups=G,
                max_batch_sends=65536, max_batch_payload=65536 * L, max_recv_records=A * 100 + 4096,
                max_recv_payload=(A * 100 + 4096) * L)
    cpu = CpuOracle(A, G)
    perm = rng.permutation(A)
    for g in range(G):
        gpu.create_group(g, perm[g * F:(g + 1) * F]); cpu.create_group(g, perm[g * F:(g + 1) * F])
    cpu.digest_enable(); gpu.digest_reset()
    flags = RECV_PRIORITY if priority else 0

    def send(n_sends):
        grp = rng.integers(0, G, n_sends).astype(np.uint32)
        snd = rng.integers(0, A, n_sends).astype(np.uint32)           # sometimes a member: skip-sender at scale
        prio = rng.integers(0, 4, n_sends).astype(np.uint8)
        typ = rng.integers(0, 7, n_sends).astype(np.uint8)
        lens = rng.integers(1, L + 1, n_sends).astype(np.uint16)
        off = np.arange(n_sends, dtype=np.uint64) * L
        pay = ALNUM[rng.integers(0, 62, n_sends * L)]
        assert gpu.send_group_batch(snd, grp, prio, typ, lens, off, pay) == cpu.send_group_batch(snd, grp, prio, typ, lens, off, pay)[0]

    total_sends = G * per_group
    for s0 in range(0, total_sends, 65536):
        send(min(65536, total_sends - s0))
    sweeps = 0
    while True:
        _, total, _ = gpu.receive_batch(None, 100, flags, copy_out=False)
        gpu.digest_fold()
        _, ctotal = cpu.receive_counts(None, 100, flags)
        assert total == ctotal, (sweeps, total, ctotal)
        if total == 0:
            break
        sweeps += 1
        if sweeps == 3:
            send(20000)                                    # new arrivals while rings hold tombstones
        if sweeps % 6 == 0:                                # digests agree along the way, not only at the end
            assert not _mismatch(gpu.digest_read(), cpu.digest_read())
    assert sweeps >= 20
    st = gpu.stats()
    assert st["ring_overflow"] == 0 and st["enqueued"] == st["delivered"]
    dg, dc = gpu.digest_read(), cpu.digest_read()
    assert not _mismatch(dg, dc), _mismatch(dg, dc)
    gpu.close(); cpu.close()


def test_p2p_one_million_records_match_oracle():
    """K1 at scale: 1,048,576 point-to-point records into 100k agents (hot and cold receivers), partial + full drain."""
    from oracle.cpu_ref import CpuOracle
    from swarmdb_b200._native import Shard
    rng = np.random.default_rng(6)
    A, L = 100_000, 256
    gpu = Shard(max_agents=A, ring_slots=4096, arena_bytes=1 << 30, max_payload_bytes=L, max_batch_sends=65536,
                max_batch_payload=65536 * L, max_recv_records=(1 << 20) + 4096, max_recv_payload=((1 << 20) + 4096) * L)
    cpu = CpuOracle(A, 1)
    idx = np.arange(A, dtype=np.uint32)
    gpu.register(idx); cpu.register(idx)
    cpu.digest_enable(); gpu.digest_reset()
    hot = rng.integers(0, A, 64)
    for b in range(16):
        n = 65536
        s = rng.integers(0, A, n).astype(np.uint32)
        r = rng.integers(0, A, n).astype(np.uint32)
        r[rng.random(n) < 0.02] = hot[rng.integers(0, 64)]                  # ~1300 records for one hot receiver per batch
        prio = rng.integers(0, 4, n).astype(np.uint8); typ = rng.integers(0, 7, n).astype(np.uint8)
        lens = rng.integers(0, L + 1, n).astype(np.uint16)
        off = np.arange(n, dtype=np.uint64) * L
        pay = ALNUM[rng.integers(0, 62, n * L)]
        assert gpu.send_batch(s, r, prio, typ, lens, off, pay) == cpu.send_batch(s, r, prio, typ, lens, off, pay)
        if b % 4 == 3:
            _, total, _ = gpu.receive_batch(None, 3, 0, copy_out=False)
            gpu.digest_fold()
            assert total == cpu.receive_counts(None, 3, 0)[1]
    while True:
        _, total, _ = gpu.receive_batch(None, 100, 0, copy_out=False)
        gpu.digest_fold()
        assert total == cpu.receive_counts(None, 100, 0)[1]
        if total == 0:
            break
    st = gpu.stats()
    assert st["ring_overflow"] == 0 and st["delivered"] == 16 * 65536
    assert not _mismatch(gpu.digest_read(), cpu.digest_read())
    gpu.close(); cpu.close()
