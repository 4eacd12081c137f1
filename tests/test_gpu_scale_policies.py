"""Deduplicated sends, bounded queues and superseding sends past one pass of their loops, at the c2 scale, and composed
in the order SwarmsDB.flush runs them.

The loops and what one pass of each covers on the card the test runs on (SM = its multiprocessor count):
  k_dedup_content, sends     min(ceil(n / 8), 8 x SM) blocks of 8 warps, one warp per send: 64 x SM sends
  k_dedup_content, payload   32 lanes x 16-byte loads: 512 bytes per warp step
  k_dedup_content, lists     one recipient per lane: 32 per warp step
  k_trim, k_supersede        sdb_grid(n, 32, 32 x SM), 8 lanes per agent: 1,024 x SM agents per grid pass
  k_trim walk 1 / walk 2     8 ring entries per step / 32 ring entries per step (8 lanes x 4 in flight)
Each test first asserts that its sizes are at least twice the one-pass coverage of the loops it targets, so a card with
more SMs fails the guard instead of turning the test into a one-pass test.  Probe chains of the dedup table that wrap
past its last slot are built on purpose: the keys are chosen in numpy by their home slot (tests/dedup_ref.slot_hash).
"""
from types import SimpleNamespace

import numpy as np
import pytest

from tests.dedup_ref import DedupModel, content_keys, edge_lengths, replay, slot_hash, table_mask
from tests.supersede_ref import TYPEF_SUPERSEDE
from tests.test_gpu_compact_receive import _check_format, _same
from tests.test_gpu_dedup import Rig as DedupRig, _queue_stats
from tests.test_gpu_expire import _loads_equal
from tests.test_gpu_scale_features import _c2, _drain_digests, _mismatch, _one_pass
from tests.test_gpu_shared_layout import _payloads
from tests.test_gpu_trim import _every_path, _survivors, _trim_all_calls
from tests.trim_ref import TrimmingOracle

pytestmark = pytest.mark.gpu

QFIELDS = ("pending", "pending_by_prio", "pending_granules", "agents_with_pending")
MAX_PAYLOAD = 65504                               # the configuration maximum of max_payload_bytes


def _content_pass():
    """Sends one grid pass of k_dedup_content covers: 8 warps x 8 blocks per SM (_one_pass(2) = 2 x 32 x SM)."""
    return _one_pass(2)


def _qstats(x, n=None):
    q = x.queue_stats() if n is None else x.queue_stats(n)
    return {k: q[k] for k in QFIELDS}


def _oracle_digests(o):
    o.digest_enable()
    o.receive_counts(None, 1 << 20)
    return o.digest_read()


# ------------------------------------------------------------------------------------------ 1. content keys
def _content_send(r, b, now):
    """DedupRig.send with the content keys computed by the vectorised reference: verdicts against DedupModel, keys
    against content_keys, the accepted sends into the oracle.  Returns (dup_of, keys as (lo, hi) arrays)."""
    from tests.dedup_ref import batch_seqs
    lo, hi = content_keys(b["sender"], b["kind"], b["target"], b["list_off"], b["list_idx"], b["lens"], b["prio"],
                          b["typ"], b["payload_off"], b["payload"])
    used = list(zip(lo.tolist(), hi.tolist()))
    seq = batch_seqs(r.o.next_seq, b["kind"], b["target"], r.sizes)
    dup, n_new = r.m.send(used, seq, now)
    base, got_dup, got_keys = r.g.send_mixed_batch_dedup(
        b["sender"], b["kind"], b["target"], b["list_off"], b["list_idx"], b["prio"], b["typ"], b["lens"],
        b["payload_off"], b["payload"], b["ts"], content=True, now=now)
    assert base == seq[0]
    bad = np.flatnonzero((got_keys["lo"] != lo) | (got_keys["hi"] != hi))
    assert len(bad) == 0, (len(bad), bad[:8].tolist(), b["lens"][bad[:8]].tolist(), b["kind"][bad[:8]].tolist())
    assert got_dup.tolist() == dup
    r.m.commit(used, seq, dup, n_new, now)
    end = seq[-1] + (r.sizes[int(b["target"][-1])] if int(b["kind"][-1]) == 1 else 1)
    replay(r.o, b["kind"], b["sender"], b["target"], b["list_off"], b["list_idx"], b["prio"], b["typ"], b["lens"],
           b["payload_off"], b["payload"], b["ts"], seq, [d == 0 for d in dup], end)
    return np.asarray(dup, np.uint64), lo, hi


def _drain_to(r, left):
    """Receive 16 records per agent on the device and the oracle, equal call by call, until at most `left` are pending:
    a receive holds max_recv_payload / pad32(max_payload_bytes) records, 8,192 at 64 KiB payloads."""
    from tests.test_gpu_dedup import A
    while r.o.queue_stats(A)["pending"] > left:
        cg, hg, pg = r.g.receive_batch(None, 16, 0)
        cc, hc, pc = r.o.receive_batch(None, 16, 0)
        assert np.array_equal(cg, cc[:len(cg)]) and not cc[len(cg):].any()
        assert hg.tobytes() == hc.tobytes() and pg.tobytes() == pc.tobytes()


def test_content_keys_at_every_loop_edge():
    """One deduplicated batch of twice the sends one k_dedup_content pass covers, at every payload length edge up to
    65,504 bytes and list lengths up to 1,000; then the batch again with a byte changed at len - 1 (a new key), bytes
    changed at len and past it inside the last 16-byte load (still a duplicate), and payloads moved to other 16-byte
    aligned offsets (still duplicates)."""
    from tests.test_gpu_dedup import A
    n = 2 * _content_pass() + 1000
    rng = np.random.default_rng(101)
    edges = edge_lengths(MAX_PAYLOAD)
    list_lens = [0, 1, 31, 32, 33, 64, 65, 1000]
    assert max(list_lens) >= 2 * 32 and max(edges) >= 2 * 512 and n >= 2 * _content_pass()
    # lengths: the edges at the front, at the back (the second grid pass) and in between random small ones
    lens = rng.integers(0, 600, n)
    lens[:len(edges)] = edges
    lens[-len(edges):] = edges
    kind = rng.choice(3, n, p=[0.8, 0.18, 0.02]).astype(np.uint8)
    kind[:len(edges)] = 0
    kind[-len(edges):] = rng.integers(0, 2, len(edges))
    lists = [rng.integers(0, A, k) for k in list_lens]                # recipients may repeat: one record each
    list_off = np.concatenate([[0], np.cumsum(list_lens)]).astype(np.uint64)
    list_idx = np.concatenate(lists).astype(np.uint32)
    is_list = np.flatnonzero(kind == 2)
    target = np.where(kind == 1, rng.integers(0, 8, n), rng.integers(0, A, n)).astype(np.uint32)
    target[is_list] = np.arange(len(is_list)) % len(list_lens)          # every list length at both ends of the batch
    target[is_list[-len(list_lens):]] = np.arange(len(list_lens))
    lens[is_list] = rng.integers(0, 40, len(is_list))                   # list sends fan out: keep their payloads small
    lens = lens.astype(np.uint16)
    stride = (lens.astype(np.int64) + 15) // 16 * 16 + 16               # 16 spare bytes behind every payload
    off = np.concatenate([[0], np.cumsum(stride)[:-1]]).astype(np.uint64)
    spare = int(stride.sum())
    payload = np.zeros(2 * spare + 64, np.uint8)
    payload[:spare] = rng.integers(0, 256, spare)
    b = dict(sender=rng.integers(0, A, n).astype(np.uint32), kind=kind, target=target, list_off=list_off,
             list_idx=list_idx, prio=rng.integers(0, 4, n).astype(np.uint8), typ=rng.integers(0, 7, n).astype(np.uint8),
             lens=lens, payload_off=off, payload=payload, ts=rng.random(n) * 100)
    r = DedupRig(102, entries=4 * n, window=100.0, ring_slots=1 << 13, arena_bytes=1 << 28, max_payload_bytes=MAX_PAYLOAD,
                 max_batch_sends=n, max_batch_payload=len(payload), list_pool_entries=1 << 14,
                 max_recv_records=1 << 20, max_recv_payload=1 << 29)
    try:
        dup, lo, hi = _content_send(r, b, now=1.0)
        assert r.m.stats()["accepted_total"] > n // 2
        # the resend: three kinds of change on disjoint sends with a payload
        b2 = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in b.items()}
        with_pay = np.flatnonzero((lens > 0) & (kind != 2) & (dup == 0))
        pick = rng.permutation(with_pay)
        last, tail, moved = pick[:600], pick[600:1200], pick[1200:1800]
        p2 = b2["payload"]
        o = off.astype(np.int64)
        p2[o[last] + lens[last] - 1] ^= 0x5A                                # byte len - 1: a new key
        for i in tail:                                                      # bytes len .. end of its 16-byte load, and
            e = int(o[i]) + int(lens[i])                                    # the next load: not part of the key
            p2[e:(e + 15) // 16 * 16 + 16] = rng.integers(1, 256, (e + 15) // 16 * 16 + 16 - e)
        dest = spare + np.concatenate([[0], np.cumsum(stride[moved])[:-1]])  # the same bytes at other aligned offsets
        for i, d in zip(moved, dest):
            p2[d:d + int(lens[i])] = p2[int(o[i]):int(o[i]) + int(lens[i])]
        b2["payload_off"] = off.copy()
        b2["payload_off"][moved] = dest.astype(np.uint64)
        assert np.all(b2["payload_off"] % 16 == 0)
        dup2, lo2, hi2 = _content_send(r, b2, now=2.0)
        changed = np.zeros(n, bool); changed[last] = True
        assert np.all(dup2[last] == 0) and not np.any((lo2[last] == lo[last]) & (hi2[last] == hi[last]))
        assert np.all(lo2[~changed] == lo[~changed]) and np.all(hi2[~changed] == hi[~changed])
        first = dup == 0                                                    # keyed sends accepted the first time
        assert np.all(dup2[first & ~changed] != 0)                          # tail bytes and moved payloads: duplicates
        _drain_to(r, 1 << 13)
        r.check(drain=True)
    finally:
        r.close()


# ------------------------------------------------------------------------------------------ 2. the dedup table
def _wrapping_keys(mask, k, rng, home_slots=8):
    """k explicit keys whose home slots are the last `home_slots` slots of a table with this mask."""
    out_lo, out_hi = [], []
    while sum(len(x) for x in out_lo) < k:
        lo = rng.integers(1, 1 << 63, 1 << 20, dtype=np.uint64)
        hi = rng.integers(1, 1 << 63, 1 << 20, dtype=np.uint64)
        h = slot_hash(lo, hi) & np.uint64(mask)
        sel = h > np.uint64(mask - home_slots)
        out_lo.append(lo[sel]); out_hi.append(hi[sel])
    lo, hi = np.concatenate(out_lo)[:k], np.concatenate(out_hi)[:k]
    home = slot_hash(lo, hi) & np.uint64(mask)
    assert np.all(home > np.uint64(mask - home_slots))
    # k keys in home_slots slots at the end of the table: at least k - home_slots of them sit past slot `mask`, in
    # slots 0, 1, ... (linear probing keeps a key at or after its home, modulo the table)
    assert k > 4 * home_slots
    return np.stack([lo, hi], 1)


def test_dedup_table_at_its_limits():
    """A table of E = 3 B entries (B = max_batch_sends) filled to exactly E live keys by four full batches with in-batch
    duplicates and repeats of earlier batches; 64 of the keys hash to the last 8 of its slots, so their chain wraps.
    Then: the capacity refusal (nothing changes), dedup_forget of half of the wrapped chain (the other half must still
    be found), a forced rebuild, an expiry rebuild that reinserts the wrapped chain, and a probe of it afterwards."""
    from swarmdb_b200._native import SdbError
    B = 4096
    E = 3 * B
    mask = table_mask(E)
    rng = np.random.default_rng(103)
    wrapped = _wrapping_keys(mask, 64, rng)
    fresh_lo = rng.integers(1, 1 << 62, E, dtype=np.uint64)
    pool = np.stack([fresh_lo, fresh_lo ^ np.uint64(0x5555)], 1)
    pool[B: B + 64] = wrapped                                   # batch 1 (now = 1) holds the wrapped chain
    assert len({(int(a), int(c)) for a, c in pool}) == E
    r = DedupRig(104, entries=E, window=10.0, ring_slots=1024, arena_bytes=1 << 25, max_batch_sends=B,
                 list_pool_entries=1 << 16)
    try:
        def step(keys, now, what):
            b = r.batch(len(keys), kinds=(0,))
            dup = r.send(b, keys, now=now)
            r.check()
            return np.asarray(dup)

        fresh_per = 3 * B // 4                                  # 3/4 fresh keys, 1/8 in-batch repeats, 1/8 older ones
        taken = 0
        for k in range(4):
            new = pool[taken:taken + fresh_per]
            older = pool[rng.integers(0, max(taken, 1), B // 8)] if taken else new[rng.integers(0, fresh_per, B // 8)]
            keys = np.concatenate([new, new[rng.integers(0, fresh_per, B - fresh_per - B // 8)], older])
            keys = keys[rng.permutation(B)]
            dup = step(keys, float(k), f"fill {k}")
            assert int((dup != 0).sum()) >= B - fresh_per
            taken += fresh_per
        st = r.g.dedup_stats()
        assert st["live"] == st["used"] == E == st["capacity"], st
        # the capacity refusal: one more key, table and queues as they were
        before, dbefore = _queue_stats(r.g), r.g.dedup_stats()
        b = r.batch(1, kinds=(0,))
        with pytest.raises(SdbError) as e:
            r.g.send_mixed_batch_dedup(b["sender"], b["kind"], b["target"], None, None, b["prio"], b["typ"], b["lens"],
                                       b["payload_off"], b["payload"], b["ts"], keys=np.array([[7, 7]], np.uint64), now=4.0)
        assert e.value.code == -6 and _queue_stats(r.g) == before and r.g.dedup_stats() == dbefore
        # forget every other key of the wrapped chain: the rest, inside and behind the forgotten slots, must be found
        gone = wrapped[::2]
        assert r.g.dedup_forget(gone).tolist() == r.m.forget(gone) == [1] * len(gone)
        r.check()
        dup = step(wrapped[rng.permutation(len(wrapped))], 5.0, "forgotten half back")     # rebuild: used + 32 > E
        assert r.g.dedup_stats()["rebuilds"] == 1 and int((dup == 0).sum()) == len(gone)
        # the expiry rebuild at now = 10.5: batch 0's keys are dead, the wrapped chain (now 1 and 5) is reinserted
        expired = sum(1 for v in r.m.tab.values() if not 10.5 < v[1] + 10.0)
        assert expired >= fresh_per - 64
        new = np.stack([np.arange(1, B + 1, dtype=np.uint64) << np.uint64(40), np.full(B, 9, np.uint64)], 1)[:min(B, expired)]
        step(new, 10.5, "expiry rebuild")
        assert r.g.dedup_stats()["rebuilds"] == 2 and r.g.dedup_stats()["expired_total"] == len(gone) + expired
        dup = step(np.concatenate([wrapped, new[:100]]), 10.6, "the wrapped chain after the rebuild")
        assert np.all(dup != 0)
        r.check(drain=True)
    finally:
        r.close()


# ------------------------------------------------------------------------------------------ 3. a deduplicated c2 batch
def test_dedup_c2_group_batches():
    """Three batches of 65,536 group sends of the c2 workload through send_mixed_batch_dedup (private payloads per
    record): a quarter of each batch repeats keys of the batch before, a quarter repeats other sends of the same batch;
    the third batch is past the window of the first.  Verdicts against DedupModel; queue statistics and the digests of a
    full drain against an oracle fed only the accepted sends, at their sequence numbers."""
    from bench import Workload
    from oracle.cpu_ref import CpuOracle
    wl = Workload()
    rec_cap = wl.S * wl.F + (1 << 16)
    assert wl.S >= 2 * _content_pass()
    rng = np.random.default_rng(107)
    g = _c2(wl, 1 << 32, rec_cap)
    surv = CpuOracle(wl.A, wl.G)
    try:
        surv.register(np.arange(wl.A))
        for k in range(wl.G):
            surv.create_group(k, wl.members(k))
        g.dedup_reserve(1 << 18, 10.0)
        m = DedupModel(1 << 18, 10.0)
        earlier = []
        for bi, now in enumerate((0.0, 5.0, 12.0)):
            snd, grp, prio, typ, lens, off, pay = wl.batch(rng, rng, var_len=True)
            n = wl.S
            keys = np.stack([rng.integers(1, 1 << 62, n, dtype=np.uint64), np.full(n, bi + 1, np.uint64)], 1)
            q = rng.permutation(n)
            same = q[: n // 4]
            keys[same] = keys[q[n // 4: n // 2]][rng.integers(0, n // 4, len(same))]   # repeats inside the batch
            if earlier:                                   # repeats of earlier batches: at now = 12 the first one's
                old = np.concatenate(earlier)             # keys are past the window, the second one's are live
                keys[q[n // 2: 3 * n // 4]] = old[rng.integers(0, len(old), n // 4)]
            next_seq = g.stats()["next_seq"]
            seq = next_seq + wl.F * np.arange(n, dtype=np.uint64)
            used = [tuple(k) for k in keys.tolist()]
            want, n_new = m.send(used, seq.tolist(), now)
            base, dup, _ = g.send_mixed_batch_dedup(snd, np.ones(n, np.uint8), grp, None, None, prio, typ, lens, off, pay,
                                                    keys=keys, now=now)
            assert base == next_seq and dup.tolist() == want
            m.commit(used, seq.tolist(), want, n_new, now)
            acc = dup == 0
            assert 0.2 * n < int((~acc).sum()) < 0.6 * n
            surv.send_group_seq(snd[acc], grp[acc], prio[acc], typ[acc], lens[acc], off[acc], pay, seq[acc])
            earlier.append(keys)
        st = g.dedup_stats()
        for k in ("live", "used", "accepted_total", "duplicate_total", "expired_total", "rebuilds"):
            assert st[k] == m.stats()[k], k
        assert _qstats(g) == _qstats(surv, wl.A)
        dg, do = _drain_digests(g), _oracle_digests(surv)
        assert not _mismatch(dg, do), _mismatch(dg, do)
    finally:
        g.close(); surv.close()


# ------------------------------------------------------------------------------------------ 4. archive mode at c2
def _flagged_c2_batch(wl, n_senders=64):
    """The c2 batch with every send flagged and few senders (none a member of its group): keys repeat in every group."""
    sender, grp, prio, typ, lens, off, pay = wl.batch(var_len=True)
    typ = (np.asarray(typ, np.uint8) & 0x07) | TYPEF_SUPERSEDE
    sender = sender % n_senders
    while True:
        bad = wl.group_of[sender] == grp
        if not bad.any():
            break
        sender[bad] = (sender[bad] + 1) % n_senders
    return sender, grp, prio, typ, lens, off, pay


def _last_per_key(grp, sender, typ, among):
    """Of the sends where `among` holds, the last per (group, sender, type & 7); a bool mask over all sends."""
    idx = np.flatnonzero(among)
    key = (grp[idx].astype(np.int64) << 16) | (sender[idx].astype(np.int64) << 3) | (typ[idx] & 7)
    _, first_rev = np.unique(key[::-1], return_index=True)
    out = np.zeros(len(grp), bool)
    out[idx[len(idx) - 1 - first_rev]] = True
    return out


def _last_k_per_group(grp, among, k):
    """Of the sends where `among` holds, the last k per group."""
    idx = np.flatnonzero(among)
    order = idx[np.lexsort((-idx, grp[idx]))]                 # by group, newest first
    g = grp[order]
    start = np.r_[0, np.flatnonzero(g[1:] != g[:-1]) + 1]
    rank = np.arange(len(order)) - np.repeat(start, np.diff(np.r_[start, len(order)]))
    out = np.zeros(len(grp), bool)
    out[order[rank < k]] = True
    return out


@pytest.mark.parametrize("case", ["trim_count2", "trim_bytes512_priority", "supersede"])
def test_archive_mode_at_c2(case):
    """The c2 backlog, one PEEK archive call, then archive calls whose caller output arrays hold a fifth of the set (the
    capacity cut runs on every call) until nothing comes back.  The union of the returned records must be the model's
    retired set: per-agent counts, sorted (agent, seq) pairs and every payload byte against the batch.  A twin given
    the same traffic retires in drop mode; queue statistics and full-drain digests must be equal."""
    from bench import Workload
    from swarmdb_b200._native import ENTRY_DTYPE, RECV_PEEK, RECV_PRIORITY, SEND_DTYPE, expand_compact, pad32
    wl = Workload()
    assert wl.A >= 2 * _one_pass(32)                            # k_trim / k_supersede: 1,024 x SM agents per pass
    rec_cap = wl.S * wl.F + (1 << 16)
    flags, n_cap, b_cap = {"trim_count2": (0, 2, 0), "trim_bytes512_priority": (RECV_PRIORITY, 0, 512),
                           "supersede": (0, 0, 0)}[case]
    if case == "supersede":
        batch = _flagged_c2_batch(wl, n_senders=8)
    else:
        batch = wl.batch(var_len=True)
    sender, grp, prio, typ, lens, off, pay = batch
    a, d = _c2(wl, 1 << 31, rec_cap), _c2(wl, 1 << 31, rec_cap)
    try:
        base = a.send_group_batch(*batch)
        assert d.send_group_batch(*batch) == base
        plen = pad32(lens.astype(np.int64))
        if case == "supersede":
            keep = _last_per_key(grp, sender, typ, np.ones(wl.S, bool))
        else:
            keep = _survivors(grp, plen, prio, wl.G, n_cap, b_cap, flags != 0)
        gone = np.flatnonzero(~keep)
        assert 0 < len(gone) < wl.S
        # the retired set: member j of send i holds seq base + F i + j
        members = np.stack([wl.members(k) for k in range(wl.G)])
        want_agent = members[grp[gone]].ravel().astype(np.int64)
        want_seq = (base + wl.F * gone[:, None].astype(np.uint64) + np.arange(wl.F, dtype=np.uint64)).ravel()
        o = np.lexsort((want_seq, want_agent))
        want_agent, want_seq = want_agent[o], want_seq[o]
        want_cnt = np.bincount(want_agent, minlength=wl.A)
        total = len(want_seq)
        assert want_cnt[2 * _one_pass(32):].sum() > total // 2       # most of the set lies past the second grid pass

        def call(**kw):
            if case == "supersede":
                return a.supersede(None, **kw)
            return a.trim(None, n_cap, b_cap, **kw)

        peek = call(flags=flags | RECV_PEEK)
        assert int(peek[0].sum()) == len(peek[1]) == total     # the default arrays hold the whole set
        cap = total // 5 + 1237
        ent_buf, snd_buf = np.zeros(cap, ENTRY_DTYPE), np.zeros(cap, SEND_DTYPE)
        cnt_sum = np.zeros(wl.A, np.int64)
        agents, seqs = [], []
        calls = 0
        while True:
            cnt, ent, snd, p = (x.copy() for x in call(flags=flags, out_entries=ent_buf, out_sends=snd_buf))
            calls += 1
            assert calls <= 8, "more calls than the capacity cut allows"
            if len(ent) == 0:
                break
            assert len(ent) <= cap
            hdr, _ = expand_compact(ent, snd, p)
            cnt_sum += cnt
            agents.append(np.repeat(np.arange(wl.A), cnt.astype(np.int64)))
            seqs.append(hdr["seq"])
            # payload bytes: every row against the batch's payload of its send
            row_send = np.zeros(len(snd), np.int64)
            row_send[ent["send"].astype(np.int64)] = ((hdr["seq"] - np.uint64(base)) // np.uint64(wl.F)).astype(np.int64)
            assert np.array_equal(snd["len"], lens[row_send])
            ln = snd["len"].astype(np.int64)
            src = np.repeat(off[row_send].astype(np.int64), ln) + (np.arange(ln.sum()) - np.repeat(np.cumsum(ln) - ln, ln))
            dst = np.repeat(snd["payload_off"].astype(np.int64), ln) + (np.arange(ln.sum()) - np.repeat(np.cumsum(ln) - ln, ln))
            assert np.array_equal(p[dst], pay[src])
        assert calls >= 6                                      # the cut ran on every call but the last two
        assert np.array_equal(cnt_sum, want_cnt)
        ga, gs = np.concatenate(agents), np.concatenate(seqs)
        o = np.lexsort((gs, ga))
        assert np.array_equal(ga[o], want_agent) and np.array_equal(gs[o], want_seq)
        if case == "supersede":
            _, dt = d.supersede(None, archive=False)
        else:
            _, dt = d.trim(None, n_cap, b_cap, flags, archive=False)
        assert dt == total
        assert _qstats(a) == _qstats(d)
        da, dd = _drain_digests(a), _drain_digests(d)
        assert not _mismatch(da, dd), _mismatch(da, dd)
    finally:
        a.close(); d.close()


# ------------------------------------------------------------------------------------------ 5. trimming on deep rings
DEEP_CASES = [("prio_level0", 1, None, 0), ("prio_level1", 1, None, 0), ("prio_level2", 1, None, 0),
              ("prio_level3", 1, None, 0), ("stream_count", 0, 700, 0), ("stream_bytes17", 0, 0, 17),
              ("prio_bytes_odd", 1, 0, 30_001), ("stream_both", 0, 1500, 40_003), ("prio_both", 1, 900, 25_019)]


@pytest.mark.parametrize("case,prio_order,n_cap,b_cap", DEEP_CASES, ids=[c[0] for c in DEEP_CASES])
def test_trim_deep_rings(case, prio_order, n_cap, b_cap):
    """32 receivers with about 2,500 pending records each in 4,096-slot rings (random priorities, lengths 0-48, a tenth
    of them empty), holes punched by a priority receive and a filtered take; then one trim, byte for byte against
    TrimmingOracle in archive mode and in drop mode on a twin, then every receive path.  The prio_level cases put the
    cut inside one priority level for every agent."""
    from oracle.cpu_ref import CpuOracle
    from swarmdb_b200._native import RECV_PEEK, RECV_PRIORITY, Shard, make_filter
    rng = np.random.default_rng(109 + [c[0] for c in DEEP_CASES].index(case))
    A, R, NR = 4096, 4096, 32
    kw = dict(max_agents=A, ring_slots=R, arena_bytes=1 << 28, max_payload_bytes=64, max_batch_sends=1 << 16,
              max_recv_records=1 << 18)
    g, d = Shard(**kw), Shard(**kw)
    c = CpuOracle(A, 1)
    for x in (g, d, c):
        x.register(np.arange(A, dtype=np.uint32))
    c = TrimmingOracle(c, 1, watermark=A)
    try:
        for _ in range(5):
            n = 1 << 14
            s, r, pr = rng.integers(0, A, n), rng.integers(0, NR, n), rng.integers(0, 4, n)
            lens, off, buf = _payloads(rng, n, 48)
            lens[rng.random(n) < 0.1] = 0
            ts = rng.uniform(0, 1, n)
            base = c.send_batch(s, r, pr, None, lens, off, buf, ts)
            assert g.send_batch(s, r, pr, None, lens, off, buf, ts) == base == d.send_batch(s, r, pr, None, lens, off, buf, ts)
        agents = np.arange(NR, dtype=np.uint32)
        # holes: a priority receive on half of the agents, a filtered take of level-1 records on the other half
        f = make_filter(prios=[1])
        want = c.receive_batch(agents[:16], 40, RECV_PRIORITY)
        for x in (g, d):
            _same(x.receive_batch(agents[:16], 40, RECV_PRIORITY), want, "priority holes")
        want = c.receive_where(agents[16:], 30, 0, f)
        for x in (g, d):
            _same(x.receive_where(agents[16:], 30, 0, f), want, "filtered holes")
        ld = g.agent_loads(agents)
        pend, by = ld["pending"].astype(np.int64), ld["pending_by_prio"].astype(np.int64)
        assert pend.min() > 2000 and g.stats()["ring_overflow"] == 0
        assert pend.min() >= 2 * 32 * 8                         # dozens of walk-1 (8) and walk-2 (32 entry) steps
        flags = RECV_PRIORITY if prio_order else 0
        if n_cap is None:                                      # the cut inside level p for every agent
            p = int(case[-1])
            below, upto = by[:, :p].sum(1), by[:, :p + 1].sum(1)
            lo_, hi_ = int((pend - upto).max()) + 1, int((pend - below).min()) - 1
            assert lo_ + 8 < hi_, (lo_, hi_)
            n_cap = (lo_ + hi_) // 2
            drops = pend - n_cap
            assert np.all((drops > below) & (drops < upto))
        want = c.trim(agents, n_cap, b_cap, flags | RECV_PEEK)
        _same(_check_format(g.trim(agents, n_cap, b_cap, flags | RECV_PEEK), False), want, "peek")
        assert int(want[0].min()) > 0
        if not b_cap or b_cap >= 32:                           # the cut lies at least two walk-2 steps into the window
            assert int(want[0].min()) >= 2 * 32 and int((pend - want[0]).min()) >= 2 * 32
        got = _trim_all_calls(g, agents, n_cap, b_cap, flags, shared=False)
        wc = c.trim(agents, n_cap, b_cap, flags)
        _same(got[:3], wc, "archive")
        cnt, total = d.trim(agents, n_cap, b_cap, flags, archive=False)
        assert total == len(wc[1]) and np.array_equal(cnt, wc[0])
        for x in (g, d):
            assert x.trim(agents, n_cap, b_cap, flags, archive=False)[1] == 0
            if b_cap and b_cap < 32:                           # zero granules: only empty records may stay
                assert x.agent_loads(agents)["pending_granules"].max() == 0
        rig = SimpleNamespace(g=g, c=c, rng=rng, A=A, idx=np.arange(A, dtype=np.uint32))
        _loads_equal(rig, "archive twin")
        _loads_equal(SimpleNamespace(g=d, c=c, idx=rig.idx), "drop twin")
        _same(d.receive_batch(agents, R, RECV_PEEK), g.receive_batch(agents, R, RECV_PEEK), "drop twin queues")
        _every_path(rig, False, case)
    finally:
        g.close(); d.close(); c.close()


# ------------------------------------------------------------------------------------------ 6. the flush order
def test_flush_order_on_the_shard_at_c2():
    """A deduplicated c2 batch of superseding group sends (a quarter repeat another send's key), then supersede(None),
    then trim(None, 2, 0) in drop mode, as SwarmsDB.flush runs them; a twin trims before it supersedes.  Each must end
    with the queue statistics and drain digests of an oracle fed only the survivors of its order, and the two orders
    must differ on this data."""
    from bench import Workload
    from oracle.cpu_ref import CpuOracle
    wl = Workload()
    rng = np.random.default_rng(113)
    rec_cap = wl.S * wl.F + (1 << 16)
    assert wl.A >= 2 * _one_pass(32) and wl.S >= 2 * _content_pass()
    sender, grp, prio, typ, lens, off, pay = _flagged_c2_batch(wl, n_senders=4)
    typ = (typ & ~np.uint8(7)) | rng.integers(0, 2, wl.S).astype(np.uint8)
    n = wl.S
    keys = np.stack([np.arange(1, n + 1, dtype=np.uint64), np.full(n, 3, np.uint64)], 1)
    q = rng.permutation(n)
    keys[q[: n // 4]] = keys[q[n // 4: n // 2]]                    # a quarter repeat another send's key
    m = DedupModel(1 << 18, 100.0)
    s0 = 1 << 40                                                   # model seqs: dup_of 0 means accepted
    dup, _ = m.send([tuple(k) for k in keys.tolist()], (s0 + wl.F * np.arange(n)).tolist(), 0.0)
    dup = np.asarray(dup, np.uint64)
    acc = dup == 0
    flush_keep = _last_k_per_group(grp, _last_per_key(grp, sender, typ, acc), 2)
    twin_keep = _last_per_key(grp, sender, typ, _last_k_per_group(grp, acc, 2))
    assert not np.array_equal(flush_keep, twin_keep)               # the order matters on this data
    handles, oracles = [], []
    try:
        for keep, trim_first in ((flush_keep, False), (twin_keep, True)):
            g = _c2(wl, 1 << 31, rec_cap)
            handles.append(g)
            g.dedup_reserve(1 << 18, 100.0)
            base, got, _ = g.send_mixed_batch_dedup(sender, np.ones(n, np.uint8), grp, None, None, prio, typ, lens, off,
                                                    pay, keys=keys, now=0.0)
            assert np.array_equal(got == 0, acc) and np.array_equal(got[~acc], base + (dup[~acc] - np.uint64(s0)))
            if trim_first:
                g.trim(None, 2, 0, archive=False)
            superseded = g.supersede(None, archive=False)[1]
            if not trim_first:
                g.trim(None, 2, 0, archive=False)
            assert superseded > 0
            o = CpuOracle(wl.A, wl.G)
            oracles.append(o)
            o.register(np.arange(wl.A))
            for k in range(wl.G):
                o.create_group(k, wl.members(k))
            o.send_group_seq(sender[keep], grp[keep], prio[keep], typ[keep], lens[keep], off[keep], pay,
                             base + wl.F * np.flatnonzero(keep).astype(np.uint64))
            assert _qstats(g) == _qstats(o, wl.A), ("trim first" if trim_first else "flush order")
            dg, do = _drain_digests(g), _oracle_digests(o)
            assert not _mismatch(dg, do), _mismatch(dg, do)
            g.close(); o.close()
            handles.clear(); oracles.clear()
    finally:
        for x in handles + oracles:
            x.close()


def test_swarmsdb_flush_dedup_supersede_then_caps(tmp_path):
    """One flush with a deduplicated duplicate of a superseding send, a newer version and a queue cap of 3: the
    duplicate enqueues nothing and so supersedes nothing, the cap counts only what superseding left."""
    import swarmdb_b200 as sdb
    from swarmdb_b200 import MessageType
    db = sdb.SwarmsDB(save_dir=str(tmp_path), auto_save=False,
                      gpu_config=sdb.GpuConfig(max_agents=64, ring_slots=64, arena_bytes=1 << 22, max_payload_bytes=1024,
                                               deterministic_ids=True, dedup_entries=1024, queue_max_messages=3))
    try:
        for a in ("a", "b", "c"):
            db.register_agent(a)
        st = MessageType.STATUS
        v0 = db.send_message("a", "a v0", "c", message_type=st, supersede=True, dedup_id="k0")
        x0 = db.send_message("a", "x0", "c")
        w0 = db.send_message("b", "b w0", "c", message_type=st, supersede=True)
        db.flush()                                     # c: v0 x0 w0
        assert db.get_stats()["superseded"] == 0 and db.get_stats()["trimmed"] == 0
        v1 = db.send_message("a", "a v1", "c", message_type=st, supersede=True, dedup_id="k1")
        again = db.send_message("a", "a v0 again", "c", message_type=st, supersede=True, dedup_id="k0")
        x1 = db.send_message("a", "x1", "c")
        db.flush()
        # model: the duplicate is dropped; c = v0 x0 w0 v1 x1; v1 supersedes v0 -> x0 w0 v1 x1; the cap of 3 trims x0
        queue = [v0, x0, w0]
        queue += [v1, x1]
        queue.remove(v0)
        queue = queue[-3:]
        assert db.original_id(again) == v0 and db.original_id(v1) is None
        stats = db.get_stats()
        assert stats["superseded"] == 1 and stats["trimmed"] == 1
        assert stats["dedup"]["duplicate_total"] == 1
        assert [m.id for m in db.receive_messages("c", 10)] == queue == [w0, v1, x1]
        assert [m.content for m in db.receive_messages("c", 10)] == []
    finally:
        db.close()
