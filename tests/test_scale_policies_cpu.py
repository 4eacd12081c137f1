"""The vectorised helpers of tests/dedup_ref.py against its per-send definitions (no GPU)."""
import numpy as np

from tests.dedup_ref import content_key, content_keys, edge_lengths, slot_hash, table_mask, _mix64

LIST_LENS = [0, 1, 31, 32, 33, 64, 65, 1000]


def test_content_keys_equal_content_key_at_the_edge_lengths():
    rng = np.random.default_rng(5)
    lens = np.array(edge_lengths(65504) * 2, np.int64)          # every layout twice: groups of more than one send
    n = len(lens) + len(LIST_LENS)
    lens = np.concatenate([lens, rng.choice([0, 7, 8, 9, 520], len(LIST_LENS))]).astype(np.uint16)
    kind = np.concatenate([rng.integers(0, 2, n - len(LIST_LENS)), np.full(len(LIST_LENS), 2)]).astype(np.uint8)
    list_off = np.concatenate([[0], np.cumsum(LIST_LENS)]).astype(np.uint64)
    list_idx = rng.integers(0, 1 << 20, int(list_off[-1])).astype(np.uint32)
    target = np.where(kind == 2, 0, rng.integers(0, 1 << 20, n)).astype(np.uint32)
    target[kind == 2] = np.arange(len(LIST_LENS))
    stride = (lens.astype(np.int64) + 15) // 16 * 16 + 16
    off = np.concatenate([[0], np.cumsum(stride)[:-1]]).astype(np.uint64)
    payload = rng.integers(0, 256, int(stride.sum()) + 64).astype(np.uint8)
    sender, prio, typ = rng.integers(0, 1 << 20, n), rng.integers(0, 4, n), rng.integers(0, 256, n)
    lo, hi = content_keys(sender, kind, target, list_off, list_idx, lens, prio, typ, off, payload)
    for i in range(n):
        t, o, ln = int(target[i]), int(off[i]), int(lens[i])
        rec = [int(x) for x in list_idx[int(list_off[t]):int(list_off[t + 1])]] if kind[i] == 2 else None
        want = content_key(int(sender[i]), int(kind[i]), t, rec, ln, int(prio[i]), int(typ[i]), bytes(payload[o:o + ln]))
        assert (int(lo[i]), int(hi[i])) == want, (i, ln, int(kind[i]))


def test_edge_lengths_and_the_slot_hash():
    e = edge_lengths(65504)
    assert {0, 1, 17, 504, 520, 1023, 1025, 8191, 65504} <= set(e)
    for k in range(1, 5):                                       # every residue mod 16 on both sides of 512 k
        assert {x % 16 for x in e if 512 * k - 16 <= x < 512 * k} == set(range(16))
        assert {x % 16 for x in e if 512 * k <= x < 512 * k + 16} == set(range(16))
    assert (table_mask(1), table_mask(32), table_mask(33), table_mask(12288)) == (63, 63, 127, 32767)
    lo, hi = np.array([1, 2, 0xFFFFFFFF00000000], np.uint64), np.array([0, 0x0123456789ABCDEF, 5], np.uint64)
    for a, b, h in zip(lo.tolist(), hi.tolist(), slot_hash(lo, hi).tolist()):
        rot = ((b << 32) | (b >> 32)) & ((1 << 64) - 1)
        assert h == int(_mix64(np.uint64(a ^ rot)))
