"""Group-send headers and receive headers are stored as whole 32-byte sectors: the lanes of a group exchange header
halves so that two lanes write one header in one instruction (sdb_st_headers).  A header the fan-out must not write
(the sender itself, skipped) stays unwritten, and the last warp step of a receive gather holds fewer than 32 records.
These tests put skipped senders at every tile position of groups whose sizes are not multiples of the tile (the wide
fan-out, 32 lanes per send, and the narrow one, 8 lanes per send, that imports use at 4 shards and more) and drain
through the bulk-copy gather with totals that leave a partial last step, against the CPU oracle.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

# tails of 1..31 records after whole tiles of 8, 16, 32 and 64 headers
SIZES = [1, 2, 7, 9, 31, 32, 33, 63, 64, 65, 97, 131]
EXTRA = 64                       # agents in no group: they send too


def _groups(rng):
    perm = rng.permutation(sum(SIZES)).astype(np.uint32)
    out, k = [], 0
    for f in SIZES:
        out.append(perm[k:k + f]); k += f
    return out


def _sends(rng, groups, n, max_len=256):
    """n group sends; three in four come from a member of the group at a tile edge or at random (skipped)."""
    A = sum(SIZES) + EXTRA
    grp = rng.integers(0, len(groups), n)
    sender = rng.integers(sum(SIZES), A, n)
    for i in range(n):
        m = groups[grp[i]]
        pick = int(rng.integers(0, 12))
        if pick < 9:
            j = [0, 1, 7, 8, 15, 16, 31, 32, len(m) - 1][pick]
            sender[i] = m[min(j, len(m) - 1)]
        elif pick < 10:
            sender[i] = m[int(rng.integers(0, len(m)))]
    prio, typ = rng.integers(0, 4, n), rng.integers(0, 7, n)
    lens = rng.integers(0, max_len + 1, n).astype(np.uint16)
    stride = (max_len + 31) & ~31
    off = np.arange(n, dtype=np.uint64) * stride
    buf = rng.integers(33, 127, n * stride + 64).astype(np.uint8)
    return sender, grp, prio, typ, lens, off, buf, rng.random(n)


def _same(res_gpu, res_cpu, what):
    cg, hg, pg = res_gpu
    cc, hc, pc = res_cpu
    assert np.array_equal(cg, cc), what
    assert hg.tobytes() == hc.tobytes(), what
    assert pg.tobytes() == pc.tobytes(), what


def test_skipped_senders_and_partial_gather_steps_one_shard():
    from oracle.cpu_ref import CpuOracle
    from swarmdb_b200._native import RECV_PEEK, RECV_PRIORITY, Shard, shared_payload_enabled
    rng = np.random.default_rng(911)
    groups = _groups(rng)
    A = sum(SIZES) + EXTRA
    g = Shard(max_agents=A, max_groups=len(groups), ring_slots=2048, max_batch_sends=4096, arena_bytes=1 << 27)
    c = CpuOracle(A, len(groups))
    try:
        for k, m in enumerate(groups):
            g.create_group(k, m); c.create_group(k, m)
        idx = np.arange(A, dtype=np.uint32)
        partial = 0
        for rnd, (n, k, flags) in enumerate([(500, 7, 0), (480, 8, RECV_PEEK), (520, 9, RECV_PRIORITY), (460, 100000, 0)]):
            sender, grp, prio, typ, lens, off, buf, ts = _sends(rng, groups, n)
            t0 = g.stats()["arena_tail_bytes"]
            assert g.send_group_batch(sender, grp, prio, typ, lens, off, buf, ts) == \
                c.send_group_batch(sender, grp, prio, typ, lens, off, buf, ts)[0]
            if shared_payload_enabled():                  # every send: one header per member, skipped or not, + one payload
                f = np.array(SIZES)[grp]
                rgran = 1 + ((lens.astype(np.int64) + 31) // 32)
                assert g.stats()["arena_tail_bytes"] - t0 == int((f + rgran - 1).sum()) * 32, rnd
            want = c.receive_batch(idx, k, flags, rec_cap=1 << 21)
            assert A * k >= 4096                          # bulk-copy gather
            partial += len(want[1]) % 32 != 0
            _same(g.receive_batch(idx, k, flags), want, (rnd, k, flags))
        assert partial >= 2
        st = g.stats()
        assert st["enqueued"] == st["delivered"] and st["ring_overflow"] == 0 and st["skipped_sender"] > 0
    finally:
        g.close(); c.close()


def test_skipped_senders_narrow_fanout_four_shards():
    """Imports at 4 shards write each send's local headers with 8 lanes per send."""
    import torch
    from oracle.cpu_ref import CpuOracle
    from swarmdb_b200._native import Shard
    from swarmdb_b200.sharded import shard_map_numbered
    rng = np.random.default_rng(912)
    world, S = 4, 300
    groups = _groups(rng)
    A, G = sum(SIZES) + EXTRA, len(groups)
    smap = shard_map_numbered("agent_", 7, A, world)
    shards = []
    oracle = CpuOracle(A, G)
    try:
        for r in range(world):
            s = Shard(max_agents=A, max_groups=G, ring_slots=2048, arena_bytes=1 << 27, max_batch_sends=S,
                      max_batch_payload=S * 256 + 64, shard_id=r, num_shards=world, max_recv_records=1 << 20)
            s.set_agent_shards(smap)
            for k, m in enumerate(groups):
                s.create_group(k, m)
            shards.append(s)
        for k, m in enumerate(groups):
            oracle.create_group(k, m)
        wire_bytes = shards[0].wire_bytes(S, S * 256 + 64)
        wire = torch.zeros(world * wire_bytes, dtype=torch.uint8, device="cuda")
        idx = np.arange(A, dtype=np.uint32)
        for step, k in enumerate([7, 100000]):
            for r in range(world):
                sender, grp, prio, typ, lens, off, buf, ts = _sends(rng, groups, S)
                shards[r].export_group_batch(sender, grp, prio, typ, lens, off, buf,
                                             wire.data_ptr() + r * wire_bytes, wire_bytes, ts)
                shards[r].sync()
                oracle.send_group_batch(sender, grp, prio, typ, lens, off, buf, ts)
            bases = [s.import_wire_batches(world, wire.data_ptr(), wire_bytes) for s in shards]
            assert len(set(bases)) == 1
            cc, hc, pc = oracle.receive_batch(idx, k, rec_cap=1 << 21)
            want, pos = {}, 0
            for a, n in zip(idx, cc):
                want[int(a)] = (hc[pos:pos + int(n)].tobytes(), int(n)); pos += int(n)
            for r, s in enumerate(shards):
                local = np.nonzero(smap == r)[0].astype(np.uint32)
                cg, hg, pg = s.receive_batch(local, k)
                pos = 0
                for a, n in zip(local, cg):
                    assert (hg[pos:pos + int(n)].tobytes(), int(n)) == want[int(a)], (step, r, int(a))
                    pos += int(n)
        assert shards[0].stats()["next_seq"] == oracle.next_seq
        for s in shards:
            st = s.stats()
            assert st["ring_overflow"] == 0 and st["enqueued"] == st["delivered"]
    finally:
        for s in shards:
            s.close()
        oracle.close()

