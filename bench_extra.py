#!/usr/bin/env python
"""Secondary measurements for the other BASELINE configs (one JSON line each):

  c1  2 agents, 1k point-to-point 128-byte messages through the SwarmsDB Python surface
  c4  priority dequeue: 10k agents x 10k pending 256-byte messages, 4 levels, receive_batch(all, 100)
  c5  backend balancer: 1M requests over 256 backends (weighted least-load, weighted random)
  k1  point-to-point enqueue kernel roofline (1M records x 256 B)
  compact  the c2 step with host buffers out: full receive format against the compact format (sdb_receive_compact)
  expire   retention on the c2 backlog (sdb_expire): drop mode at the median cutoff, SDB_EXPIRE_ALL, archive mode
  supersede  superseding sends (sdb_supersede): the c2 backlog without and with flagged sends, deep queues, a flush;
  trim     bounded queues on the c2 backlog (sdb_trim): count cap 2, byte cap 512 B, byte cap with priority, archive mode;
           and a SwarmsDB flush of 4,096 sends with and without GpuConfig.queue_max_messages
  where    filtered receive on the c2 backlog (sdb_receive_where): header-clause and keyword PEEKs, a take of one group's
           records, and keyword counts over deep queues
  restore  restore on the c2 backlog (sdb_restore_compact): snapshot, restore into a fresh handle, requeue

bench.py remains the contract benchmark (c2/c3); this file only feeds DESIGN.md.
"""
from __future__ import annotations

import argparse
import json
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from bench import ALNUM, hbm_peak  # noqa: E402


def c1(tmp="/tmp/sdb_c1"):
    import swarmdb_b200 as sdb
    rng = np.random.default_rng(1)
    contents = [ALNUM[rng.integers(0, 62, 128)].tobytes().decode() for _ in range(1000)]
    db = sdb.SwarmsDB(save_dir=tmp, auto_save=False, gpu_config=sdb.GpuConfig(max_agents=1024, ring_slots=2048, arena_bytes=1 << 26))
    db.register_agent("agent_a"); db.register_agent("agent_b")
    for c in contents[:50]:
        db.send_message("agent_a", c, "agent_b")
    db.receive_messages("agent_b", 100)
    t0 = time.perf_counter()
    for c in contents:
        db.send_message("agent_a", c, "agent_b")
    t1 = time.perf_counter()
    got = db.receive_messages("agent_b", 2000)
    t2 = time.perf_counter()
    assert [m.content for m in got] == contents
    db.close()
    return {"config": "c1: 2 agents, 1k p2p 128-byte messages, SwarmsDB Python surface (buffered sends, one flush at receive)",
            "send_msgs_per_s": 1000 / (t1 - t0), "receive_msgs_per_s": 1000 / (t2 - t1),
            "send_to_receive_msgs_per_s": 1000 / (t2 - t0),
            "reference_python_probe": "send 9.2k/s, receive 46k/s, end-to-end 7.6k/s (BASELINE.md, in-process Kafka stub)"}


def c4(n_agents=10_000, depth=10_000, reps=4):
    from swarmdb_b200._native import RECV_PRIORITY, Shard
    peak, src = hbm_peak()
    per_batch = 100                                   # messages per agent per preload batch
    n = n_agents * per_batch
    shard = Shard(max_agents=n_agents, ring_slots=16384, arena_bytes=1 << 35, max_payload_bytes=256, max_batch_sends=n,
                  max_batch_payload=n * 256, max_recv_records=n_agents * 100, max_recv_payload=n_agents * 100 * 256)
    rng = np.random.default_rng(4)
    recv = np.tile(np.arange(n_agents, dtype=np.uint32), per_batch)
    send = rng.integers(0, n_agents, n).astype(np.uint32)
    lens = np.full(n, 256, np.uint16)
    off = np.arange(n, dtype=np.uint64) * 256
    payload = ALNUM[rng.integers(0, 62, n * 256)]
    staged = [shard.stage(0, send, recv, rng.integers(0, 4, n).astype(np.uint8), None, lens, off, payload) for _ in range(2)]
    t0 = time.perf_counter()
    for b in range(depth // per_batch):
        shard.submit(staged[b % 2])
    shard.sync()
    load_s = time.perf_counter() - t0
    st = shard.stats()
    assert st["enqueued"] == n_agents * depth and st["ring_overflow"] == 0, st
    shard.profile(True)
    sweeps = []
    for r in range(reps):
        t1 = time.perf_counter()
        _, total, _ = shard.receive_batch(None, 100, RECV_PRIORITY, copy_out=False)
        sweeps.append((time.perf_counter() - t1) * 1e3)
        assert total == n_agents * 100
    prof = shard.profile_read()
    shard.close()
    sel = prof["recv_select"][0] / prof["recv_select"][1]
    gat = prof["recv_gather"][0] / prof["recv_gather"][1]
    k5_ms = sum(v[0] for k, v in prof.items() if k.startswith("recv")) / reps
    alg = n_agents * (depth * 1 + 2 * 100 * (256 + 16))          # SURVEY 8d: 64,400 B per agent-call
    return {"config": f"c4: {n_agents} agents x {depth} pending 256-B messages, 4 priorities, receive_batch(all agents, 100, PRIORITY)",
            "preload_s": load_s, "preload_msgs_per_s": n_agents * depth / load_s,
            "sweep_wall_ms": sweeps, "p50_sweep_wall_ms": float(np.median(sweeps)),
            "k5_kernels_ms_per_sweep": k5_ms, "select_ms": sel, "gather_ms": gat,
            "roofline": {"bound": "hbm", "algorithmic_bytes_per_sweep": alg, "achieved": alg / (k5_ms * 1e-3) / 1e9,
                         "peak": peak, "unit": "GB/s", "frac": alg / (k5_ms * 1e-3) / 1e9 / peak, "peak_source": src},
            "per_agent_call_us": k5_ms * 1e3 / n_agents}


def c5(n_req=1_000_000, n_backends=256):
    from oracle.cpu_ref import CpuOracle
    from swarmdb_b200._native import Shard
    rng = np.random.default_rng(5)
    w = rng.integers(1, 9, n_backends)
    out = {"config": f"c5: {n_req} unit-cost requests over {n_backends} backends, weights U{{1..8}}, load0 = 0"}
    for mode, name in ((0, "weighted_least_load"), (1, "weighted_random")):
        g = Shard(max_agents=16)
        g.set_backends(w)
        g.select_backends(1000, None, mode, 6)                   # warm-up
        g.set_backends(w)
        g.profile(True)
        t0 = time.perf_counter()
        picks = g.select_backends(n_req, None, mode, 6)
        wall = time.perf_counter() - t0
        prof = g.profile_read()
        o = CpuOracle(16)
        o.set_backends(w)
        t1 = time.perf_counter()
        ref = o.select_backends(n_req, None, mode, 6)
        cpu = time.perf_counter() - t1
        assert np.array_equal(picks, ref) and np.array_equal(g.backend_loads(), o.backend_loads())
        out[name] = {"picks_per_s_end_to_end": n_req / wall, "wall_ms": wall * 1e3,
                     "cpu_oracle_picks_per_s_1_core": n_req / cpu, "bit_exact_vs_oracle": True}
        g.close(); o.close()
    out["note"] = "not HBM-bound: the 256-entry table lives in shared memory / L1 (SURVEY 8d says report picks/s)"
    return out


def k1(n=1_000_000):
    from swarmdb_b200._native import Shard
    peak, src = hbm_peak()
    A = 1_000_000
    shard = Shard(max_agents=A, ring_slots=16, arena_bytes=1 << 32, max_payload_bytes=256, max_batch_sends=n,
                  max_batch_payload=n * 256, max_recv_records=n + 4096, max_recv_payload=(n + 4096) * 256)
    rng = np.random.default_rng(8)
    lens = np.full(n, 256, np.uint16)
    off = np.arange(n, dtype=np.uint64) * 256
    payload = ALNUM[rng.integers(0, 62, n * 256)]
    st = shard.stage(0, rng.integers(0, A, n).astype(np.uint32), rng.permutation(A)[:n].astype(np.uint32), None, None, lens, off, payload)
    shard.register(np.arange(A, dtype=np.uint32))
    for _ in range(3):
        shard.submit(st); shard.receive_batch(None, 100, 0, copy_out=False)
    shard.profile(True)
    for _ in range(8):
        shard.submit(st); shard.receive_batch(None, 100, 0, copy_out=False)
    prof = shard.profile_read()
    shard.close()
    ms = prof["p2p"][0] / prof["p2p"][1]
    alg = 2 * (256 + 16) * n
    return {"config": f"k1: {n} point-to-point 256-B records to distinct agents per batch",
            "p2p_ms": ms, "commit_ms": prof["commit"][0] / prof["commit"][1],
            "roofline": {"bound": "hbm", "algorithmic_bytes": alg, "achieved": alg / (ms * 1e-3) / 1e9, "peak": peak,
                         "unit": "GB/s", "frac": alg / (ms * 1e-3) / 1e9 / peak, "peak_source": src}}


def bcast(n_agents=1_000_000, n_sends=16):
    """R11 at scale: broadcasts to every registered agent (one record image per recipient)."""
    from swarmdb_b200._native import Shard
    peak, src = hbm_peak()
    shard = Shard(max_agents=n_agents, ring_slots=64, arena_bytes=1 << 33, max_payload_bytes=256, max_batch_sends=n_sends,
                  max_batch_payload=n_sends * 256 + 64, list_pool_entries=n_sends * n_agents + 1024,
                  max_recv_records=n_sends * n_agents + 4096, max_recv_payload=(n_sends * n_agents + 4096) * 256)
    rng = np.random.default_rng(11)
    shard.register(np.arange(n_agents, dtype=np.uint32))
    lo = np.arange(n_sends + 1, dtype=np.uint64) * n_agents
    li = np.tile(np.arange(n_agents, dtype=np.uint32), n_sends)
    lens = np.full(n_sends, 256, np.uint16)
    off = np.arange(n_sends, dtype=np.uint64) * 256
    payload = ALNUM[rng.integers(0, 62, n_sends * 256 + 64)]
    sender = rng.integers(0, n_agents, n_sends).astype(np.uint32)
    out = []
    shard.profile(True)
    for rep in range(3):
        shard.sync()
        t0 = time.perf_counter()
        shard.send_list_batch(sender, lo, li, None, None, lens, off, payload)
        shard.sync()
        t1 = time.perf_counter()
        _, total, _ = shard.receive_batch(None, 100, 0, copy_out=False)
        shard.sync()
        t2 = time.perf_counter()
        assert total == n_sends * n_agents
        out.append(((t1 - t0) * 1e3, (t2 - t1) * 1e3))
    prof = shard.profile_read()
    shard.close()
    kern = {k: v[0] / v[1] for k, v in prof.items() if v[1]}
    send_ms = kern.get("fanout", min(o[0] for o in out))
    alg = n_sends * n_agents * (256 + 16 + 4)
    return {"config": f"bcast: {n_sends} broadcasts x {n_agents} recipients, 256-B payloads (send_list_batch incl. the H2D of the recipient lists), then full drain",
            "send_wall_ms": [o[0] for o in out], "drain_wall_ms": [o[1] for o in out], "kernel_ms_per_launch": kern,
            "roofline": {"bound": "hbm", "algorithmic_bytes": alg, "achieved": alg / (send_ms * 1e-3) / 1e9, "peak": peak, "unit": "GB/s",
                         "frac": alg / (send_ms * 1e-3) / 1e9 / peak, "peak_source": src,
                         "note": "fan-out kernel only; the call's wall time adds host validation and 64 MB of recipient indices over PCIe"}}


def _gpu_card(index=0):
    """Name and enforced power limit of the card (NVML reads only)."""
    import torch
    out = {"gpu": torch.cuda.get_device_name(index), "power_limit_w": None}
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(index)
        out["power_limit_w"] = pynvml.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0
    except Exception as e:  # pragma: no cover
        out["power_limit_error"] = repr(e)
    return out


def compact(rounds=3, block=8):
    """The c2 step with host buffers out (bench.py's e2e step: send_group_batch from pinned inputs, then a receive of
    every agent into pinned outputs), full format against the compact format (sdb_receive_compact), alternated in
    blocks in one process.  D2H bytes per step come from the returned totals."""
    import torch
    from bench import ClockSampler, Workload
    from swarmdb_b200._native import ENTRY_DTYPE, HDR_DTYPE, RECV_PEEK, SEND_DTYPE, Shard, expand_compact
    if not torch.cuda.is_available():
        raise SystemExit("bench_extra.py compact: no CUDA device - swarmdb_b200 has no CPU fallback")
    wl = Workload()
    per_step = wl.S * wl.F
    rec_cap = per_step + (1 << 16)
    stream = torch.cuda.Stream()
    shard = Shard(max_agents=wl.A, ring_slots=64, arena_bytes=1 << 33, max_payload_bytes=wl.L, max_groups=1 << 14,
                  member_pool_entries=wl.A + 1024, max_batch_sends=wl.S, max_batch_payload=wl.S * wl.L,
                  max_recv_records=rec_cap, max_recv_payload=rec_cap * wl.L)
    shard.set_stream(stream.cuda_stream)
    shard.register(np.arange(wl.A, dtype=np.uint32))
    for g in range(wl.G):
        shard.create_group(g, wl.members(g))
    shard.sync()

    def pinned(nbytes):
        return torch.empty(nbytes, dtype=torch.uint8, pin_memory=True).numpy()

    pinned_in = []
    for _ in range(4):
        b = wl.batch()
        t = pinned(b[6].nbytes); t[:] = b[6]
        pinned_in.append(b[:6] + (t,))
    pin_hdr, pin_pay = pinned(rec_cap * 32).view(HDR_DTYPE), pinned(rec_cap * wl.L)
    pin_ent, pin_snd, pin_cpay = pinned(rec_cap * 16).view(ENTRY_DTYPE), pinned(rec_cap * 32).view(SEND_DTYPE), pinned(rec_cap * wl.L)

    def full_step(i):
        shard.send_group_batch(*pinned_in[i % len(pinned_in)])
        cnt, hdr, pay = shard.receive_batch(None, 100, 0, copy_out=True, out_hdr=pin_hdr, out_payload=pin_pay)
        assert len(hdr) == per_step
        return len(cnt) * 4 + len(hdr) * 32 + len(pay) + 16                   # counts + headers + payloads + totals

    def compact_step(i):
        shard.send_group_batch(*pinned_in[i % len(pinned_in)])
        cnt, ent, snd, pay = shard.receive_compact(None, 100, 0, out_entries=pin_ent, out_sends=pin_snd, out_payload=pin_cpay)
        assert len(ent) == per_step
        return len(cnt) * 4 + len(ent) * 16 + len(snd) * 32 + len(pay) + 24     # counts + entries + rows + payloads + totals

    def timed(step, i0):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t = time.perf_counter()
        e0.record(stream)
        nbytes = [step(i0 + i) for i in range(block)]
        e1.record(stream)
        torch.cuda.synchronize()
        ms = max(e0.elapsed_time(e1), (time.perf_counter() - t) * 1e3)         # host work between calls counts too
        return ms / block, nbytes[-1]

    res = {"full": [], "compact": []}
    d2h = {}
    with torch.cuda.stream(stream):
        for i in range(2):
            full_step(i); compact_step(i)
        # outside the timed region: one compact step equals a full receive of the same records
        shard.send_group_batch(*pinned_in[0])
        cnt, ent, snd, pay = shard.receive_compact(None, 100, RECV_PEEK)
        hdr_c, pay_c = expand_compact(ent, snd, pay)
        cnt = cnt.copy()
        cg, hg, pg = shard.receive_batch(None, 100, 0)
        assert np.array_equal(cnt, cg) and hdr_c.tobytes() == hg.tobytes() and pay_c.tobytes() == pg.tobytes()
        assert len(snd) == wl.S
        del hdr_c, pay_c
        clocks = ClockSampler(0); clocks.start()
        for r in range(rounds):
            for name, step in (("full", full_step), ("compact", compact_step)):
                ms, d2h[name] = timed(step, r * block)
                res[name].append(ms)
        clk = clocks.stop()
        kern = {}
        for name, step in (("full", full_step), ("compact", compact_step)):
            shard.profile(True)
            for i in range(block):
                step(i)
            prof = shard.profile_read()
            shard.profile(False)
            kern[name] = {k: v[0] / block for k, v in prof.items() if v[1]}
    st = shard.stats()
    assert st["ring_overflow"] == 0 and st["delivered"] == st["enqueued"]
    shard.close()
    out = {"config": f"c2 e2e: {wl.A} agents, {wl.S} group sends x {wl.F} members, {wl.L}-B payloads; pinned host "
                     f"buffers in and out; {rounds} rounds of {block} full-format steps, then {block} compact steps"}
    for name in ("full", "compact"):
        ms = float(np.median(res[name]))
        recv_k = kern[name].get("recv_select", 0.0) + kern[name].get("recv_gather" if name == "full" else "recv_compact", 0.0)
        out[name] = {"ms_per_step_blocks": res[name], "ms_per_step": ms, "msgs_per_s": per_step / (ms * 1e-3),
                     "d2h_bytes_per_step": d2h[name], "receive_kernels_ms_per_step": recv_k,
                     "kernel_ms_per_step": kern[name]}
    out["speedup"] = out["full"]["ms_per_step"] / out["compact"]["ms_per_step"]
    out.update(_gpu_card(0))
    out["clocks"] = clk
    return out


def expire(rounds=3, block=4):
    """sdb_expire on the c2 backlog (1M agents, 65,536 group sends x 64 = 4,194,304 pending records, a seeded uniform
    timestamp per send): drop mode at the median cutoff, SDB_EXPIRE_ALL, and archive mode into pinned host buffers,
    alternated in blocks in one process.  Every timed call starts from a fresh backlog (drain + resend, untimed).
    Outside the timed region the drop-mode result is drained through the digests and checked against an oracle that was
    only ever sent the surviving sends."""
    import torch
    from bench import ClockSampler, Workload
    from oracle.cpu_ref import CpuOracle
    from swarmdb_b200._native import ENTRY_DTYPE, EXPIRE_ALL, SEND_DTYPE, Shard
    if not torch.cuda.is_available():
        raise SystemExit("bench_extra.py expire: no CUDA device - swarmdb_b200 has no CPU fallback")
    wl = Workload()
    per_step = wl.S * wl.F
    rec_cap = per_step + (1 << 16)
    stream = torch.cuda.Stream()
    shard = Shard(max_agents=wl.A, ring_slots=64, arena_bytes=1 << 33, max_payload_bytes=wl.L, max_groups=1 << 14,
                  member_pool_entries=wl.A + 1024, max_batch_sends=wl.S, max_batch_payload=wl.S * wl.L,
                  max_recv_records=rec_cap, max_recv_payload=rec_cap * wl.L)
    shard.set_stream(stream.cuda_stream)
    shard.register(np.arange(wl.A, dtype=np.uint32))
    for g in range(wl.G):
        shard.create_group(g, wl.members(g))
    batch = wl.batch()
    ts = np.random.default_rng(4242).uniform(0.0, 1.0, wl.S)
    cut = float(np.median(ts))

    def pinned(nbytes):
        return torch.empty(nbytes, dtype=torch.uint8, pin_memory=True).numpy()
    pin_ent, pin_snd, pin_pay = pinned(rec_cap * 16).view(ENTRY_DTYPE), pinned(rec_cap * 32).view(SEND_DTYPE), pinned(rec_cap * wl.L)

    seq_base = [0]

    def backlog():
        while shard.receive_batch(None, 1 << 10, copy_out=False)[1]:
            pass
        seq_base[0] = shard.send_group_batch(*batch, ts=ts)
        shard.sync()

    calls = {"drop_median": lambda: shard.expire(None, cut, archive=False)[1],
             "expire_all": lambda: shard.expire(None, 0.0, EXPIRE_ALL, archive=False)[1],
             "archive_median": lambda: len(shard.expire(None, cut, out_entries=pin_ent, out_sends=pin_snd, out_payload=pin_pay)[1])}

    def timed(fn):
        backlog()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        t = time.perf_counter()
        n = fn()                                         # synchronises: it returns totals
        wall = (time.perf_counter() - t) * 1e3
        e1.record(stream)
        torch.cuda.synchronize()
        return wall, e0.elapsed_time(e1), n

    res = {k: {"call_ms": [], "event_ms": []} for k in calls}
    expired = {}
    with torch.cuda.stream(stream):
        for fn in calls.values():                        # warm-up: every shape once
            timed(fn)
        # outside the timed region: drop at the median, drain through the digests, compare with the oracle's own expiry
        backlog()
        n_drop = calls["drop_median"]()
        shard.digest_reset()
        while True:
            _, t, _ = shard.receive_batch(None, 100, copy_out=False)
            if not t:
                break
            shard.digest_fold()
        o = CpuOracle(wl.A, wl.G)
        o.register(np.arange(wl.A))
        for g in range(wl.G):
            o.create_group(g, wl.members(g))
        # the oracle is sent only the surviving sends, with the device's sequence numbers (send i numbers its F members
        # from seq_base + F i: every group has F members and no sender is in its own group)
        keep = ~(ts < cut)
        snd, grp, prio, typ, lens, off, pay = batch
        o.send_group_seq(snd[keep], grp[keep], prio[keep], typ[keep], lens[keep], off[keep], pay,
                         seq_base[0] + wl.F * np.nonzero(keep)[0].astype(np.uint64), ts[keep])
        assert n_drop == wl.F * int((~keep).sum())
        o.digest_enable()
        o.receive_counts(None, 100)
        digests_ok = bool(np.array_equal(shard.digest_read(), o.digest_read()))
        o.close()
        assert digests_ok, "digests after expiry differ from the oracle's"
        clocks = ClockSampler(0); clocks.start()
        for _ in range(rounds):
            for name, fn in calls.items():
                for _ in range(block):
                    wall, ev, n = timed(fn)
                    res[name]["call_ms"].append(wall); res[name]["event_ms"].append(ev)
                    expired[name] = n
        clk = clocks.stop()
        kern = {}
        for name, fn in calls.items():
            backlog()
            shard.profile(True)
            fn()
            prof = shard.profile_read()
            shard.profile(False)
            kern[name] = {k: v[0] for k, v in prof.items() if v[1]}
    shard.close()
    out = {"config": f"c2 backlog: {wl.A} agents, {wl.S} group sends x {wl.F} members = {per_step} pending records, "
                     f"{wl.L}-B payloads, timestamps U[0,1) per send; {rounds} rounds of {block} calls per mode, each on a "
                     f"fresh backlog", "digests_match_oracle": digests_ok}
    for name in calls:
        ms = float(np.median(res[name]["call_ms"]))
        n = expired[name]
        # algorithmic bytes: 16-B ring header per agent, then per pending record its 8-B entry and one 32-B timestamp
        # sector, plus an 8-B tombstone per expired record; SDB_EXPIRE_ALL reads no entries (header read + write)
        nbytes = 16 * wl.A * 2 if name == "expire_all" else 16 * wl.A + 40 * per_step + 8 * n
        kms = sum(kern[name].values())
        out[name] = {"records_expired": n, "ms_per_call": ms, "event_ms_per_call": float(np.median(res[name]["event_ms"])),
                     "records_per_s": n / (ms * 1e-3), "kernel_ms": kern[name], "kernel_ms_total": kms,
                     "algorithmic_bytes": nbytes, "algorithmic_gb_per_s_kernel": nbytes / (kms * 1e-3) / 1e9 if kms else None,
                     "call_ms_blocks": res[name]["call_ms"]}
    out.update(_gpu_card(0))
    out["clocks"] = clk
    return out


def trim(rounds=3, block=4):
    """sdb_trim on the c2 backlog (1M agents, 65,536 group sends x 64 = 4,194,304 pending records): drop mode with a
    count cap of 2, a byte cap of 512 B, the byte cap with SDB_RECV_PRIORITY, and the count cap in archive mode into
    pinned host buffers, alternated in blocks in one process.  Every timed call starts from a fresh backlog (drain +
    resend, untimed).  Then a SwarmsDB flush of 4,096 point-to-point sends over 1,024 agents (max_agents = 4,096, so the
    host's recipient-list pool holds the batch), with and without
    GpuConfig.queue_max_messages = 2, alternated (the queues are drained after every flush, untimed)."""
    import torch
    import swarmdb_b200 as sdb
    from bench import ClockSampler, Workload
    from swarmdb_b200._native import ENTRY_DTYPE, RECV_PRIORITY, SEND_DTYPE, Shard
    if not torch.cuda.is_available():
        raise SystemExit("bench_extra.py trim: no CUDA device - swarmdb_b200 has no CPU fallback")
    wl = Workload()
    per_step = wl.S * wl.F
    rec_cap = per_step + (1 << 16)
    stream = torch.cuda.Stream()
    shard = Shard(max_agents=wl.A, ring_slots=64, arena_bytes=1 << 33, max_payload_bytes=wl.L, max_groups=1 << 14,
                  member_pool_entries=wl.A + 1024, max_batch_sends=wl.S, max_batch_payload=wl.S * wl.L,
                  max_recv_records=rec_cap, max_recv_payload=rec_cap * wl.L)
    shard.set_stream(stream.cuda_stream)
    shard.register(np.arange(wl.A, dtype=np.uint32))
    for g in range(wl.G):
        shard.create_group(g, wl.members(g))
    batch = wl.batch()

    def pinned(nbytes):
        return torch.empty(nbytes, dtype=torch.uint8, pin_memory=True).numpy()
    pin_ent, pin_snd, pin_pay = pinned(rec_cap * 16).view(ENTRY_DTYPE), pinned(rec_cap * 32).view(SEND_DTYPE), pinned(rec_cap * wl.L)

    def backlog():
        while shard.receive_batch(None, 1 << 10, copy_out=False)[1]:
            pass
        shard.send_group_batch(*batch)
        shard.sync()

    # name: (call, walks over the ring entries per kernel, kernels)
    calls = {"drop_count2": (lambda: shard.trim(None, 2, 0, archive=False)[1], 1, 1),
             "drop_bytes512": (lambda: shard.trim(None, 0, 512, archive=False)[1], 2, 1),
             "drop_bytes512_priority": (lambda: shard.trim(None, 0, 512, RECV_PRIORITY, archive=False)[1], 2, 1),
             "archive_count2": (lambda: len(shard.trim(None, 2, 0, out_entries=pin_ent, out_sends=pin_snd,
                                                       out_payload=pin_pay)[1]), 1, 2)}

    def timed(fn):
        backlog()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        t = time.perf_counter()
        n = fn()                                         # synchronises: it returns totals
        wall = (time.perf_counter() - t) * 1e3
        e1.record(stream)
        torch.cuda.synchronize()
        return wall, e0.elapsed_time(e1), n

    res = {k: {"call_ms": [], "event_ms": []} for k in calls}
    trimmed = {}
    with torch.cuda.stream(stream):
        for fn, _, _ in calls.values():                  # warm-up: every shape once
            timed(fn)
        clocks = ClockSampler(0); clocks.start()
        for _ in range(rounds):
            for name, (fn, _, _) in calls.items():
                for _ in range(block):
                    wall, ev, n = timed(fn)
                    res[name]["call_ms"].append(wall); res[name]["event_ms"].append(ev)
                    trimmed[name] = n
        clk = clocks.stop()
        kern = {}
        for name, (fn, _, _) in calls.items():
            backlog()
            shard.profile(True)
            fn()
            prof = shard.profile_read()
            shard.profile(False)
            kern[name] = {k: v[0] for k, v in prof.items() if v[1]}
    shard.close()
    out = {"config": f"c2 backlog: {wl.A} agents, {wl.S} group sends x {wl.F} members = {per_step} pending records, "
                     f"{wl.L}-B payloads; {rounds} rounds of {block} calls per mode, each on a fresh backlog"}
    for name, (_, walks, kernels) in calls.items():
        ms = float(np.median(res[name]["call_ms"]))
        n = trimmed[name]
        # algorithmic bytes: per kernel a 16-B ring header per agent and 8 B per ring entry per walk, plus an 8-B
        # tombstone per trimmed record (archive mode: the count and select kernels; the compact back end is not counted)
        nbytes = kernels * (16 * wl.A + 8 * per_step * walks) + 8 * n
        kms = kern[name].get("expire", sum(kern[name].values()))
        out[name] = {"records_trimmed": n, "ms_per_call": ms, "event_ms_per_call": float(np.median(res[name]["event_ms"])),
                     "kernel_ms": kern[name], "trim_kernel_ms": kms, "algorithmic_bytes": nbytes,
                     "algorithmic_gb_per_s_kernel": nbytes / (kms * 1e-3) / 1e9 if kms else None,
                     "share_of_3_35_TBps": nbytes / (kms * 1e-3) / 3.35e12 if kms else None,
                     "call_ms_blocks": res[name]["call_ms"]}
    # SwarmsDB flush of 4,096 sends, with and without the automatic cap
    import tempfile
    n_agents, n_sends = 1024, 4096
    rng = np.random.default_rng(5)
    recv = rng.integers(0, n_agents, n_sends).tolist()
    flush_ms = {}
    with tempfile.TemporaryDirectory() as tmp:
        dbs = {name: sdb.SwarmsDB(save_dir=tmp, auto_save=False,
                                  gpu_config=sdb.GpuConfig(max_agents=n_sends, flush_threshold=n_sends + 1,
                                                           deterministic_ids=True, queue_max_messages=cap))
               for name, cap in (("flush_no_cap", 0), ("flush_cap2", 2))}
        names = [f"a{i}" for i in range(n_agents)]
        for db in dbs.values():
            for a in names:
                db.register_agent(a)
        flush_ms = {name: [] for name in dbs}
        for r in range(2 + rounds * block):
            for name, db in (dbs.items() if r % 2 == 0 else reversed(list(dbs.items()))):
                for i, a in enumerate(recv):
                    db.send_message(names[i % n_agents], "x" * 100, receiver_id=names[a])
                torch.cuda.synchronize()
                t = time.perf_counter()
                db.flush()
                db.shard.sync()
                if r >= 2:
                    flush_ms[name].append((time.perf_counter() - t) * 1e3)
                db.shard.receive_batch(None, 1 << 10, copy_out=False)
                db.messages.clear(); db.agent_inbox.clear()
        trimmed_db = dbs["flush_cap2"].get_stats()["trimmed"]
        for db in dbs.values():
            db.close()
    for name, v in flush_ms.items():
        out[name] = {"ms_per_flush": float(np.median(v)), "ms_blocks": v, "sends": n_sends, "agents": n_agents}
    out["flush_cap2"]["records_trimmed_total"] = trimmed_db
    out.update(_gpu_card(0))
    out["clocks"] = clk
    return out


def supersede(rounds=3, block=4):
    """sdb_supersede in drop mode: (a) on the c2 backlog (1M agents, 65,536 group sends x 64 = 4,194,304 pending
    records) with no flagged record, the cost every caller of the pass pays; (b) the same backlog with every send
    flagged; (c) deep queues, 10,000 agents x 1,000 pending point-to-point records, from 100 senders x 10 versions and
    from 1,000 distinct senders (nothing to retire); each timed call on a fresh backlog (drain + resend, untimed),
    modes alternated in blocks.  (d) a SwarmsDB flush of 4,096 point-to-point sends over 1,024 agents with 10 % of them
    flagged against none, alternated (queues drained after every flush, untimed)."""
    import torch
    import swarmdb_b200 as sdb
    from bench import ClockSampler, Workload
    from swarmdb_b200._native import TYPEF_SUPERSEDE, Shard
    if not torch.cuda.is_available():
        raise SystemExit("bench_extra.py supersede: no CUDA device - swarmdb_b200 has no CPU fallback")
    wl = Workload()
    per_step = wl.S * wl.F
    stream = torch.cuda.Stream()
    c2 = Shard(max_agents=wl.A, ring_slots=64, arena_bytes=1 << 33, max_payload_bytes=wl.L, max_groups=1 << 14,
               member_pool_entries=wl.A + 1024, max_batch_sends=wl.S, max_batch_payload=wl.S * wl.L,
               max_recv_records=1 << 16, max_recv_payload=(1 << 16) * wl.L)
    c2.set_stream(stream.cuda_stream)
    c2.register(np.arange(wl.A, dtype=np.uint32))
    for g in range(wl.G):
        c2.create_group(g, wl.members(g))
    plain = wl.batch()
    flagged = plain[:3] + ((np.asarray(plain[3], np.uint8) | TYPEF_SUPERSEDE),) + plain[4:]
    # deep queues: 10 batches of 1M sends, batch k holds pending records k*100 .. k*100+99 of every agent
    DA, DD = 10_000, 1_000
    deep = Shard(max_agents=DA, ring_slots=1024, arena_bytes=1 << 31, max_payload_bytes=64, max_batch_sends=1 << 20,
                 max_batch_payload=(1 << 20) * 32, max_recv_records=1 << 16, max_recv_payload=(1 << 16) * 64)
    deep.set_stream(stream.cuda_stream)
    deep.register(np.arange(DA, dtype=np.uint32))
    per = DD // 10
    recv = np.repeat(np.arange(DA, dtype=np.uint32), per)
    lens, off = np.full(len(recv), 16, np.uint16), np.zeros(len(recv), np.uint64)     # one shared 16-B payload
    dpay = np.full(64, 65, np.uint8)
    typ = np.full(len(recv), TYPEF_SUPERSEDE | 6, np.uint8)

    def deep_batches(distinct):
        j = np.tile(np.arange(per, dtype=np.uint32), DA)
        return [((j + k * per) if distinct else j) for k in range(10)]     # senders; 100 x 10 versions or 1,000
    senders = {"deep_100x10": deep_batches(False), "deep_1000_distinct": deep_batches(True)}

    def drain(sh):
        while sh.receive_batch(None, 1 << 10, copy_out=False)[1]:
            pass

    def c2_backlog(b):
        drain(c2)
        c2.send_group_batch(*b)
        c2.sync()

    def deep_backlog(name):
        drain(deep)
        for s in senders[name]:
            deep.send_batch(s, recv, None, typ, lens, off, dpay)
        deep.sync()

    # name: (shard, backlog, records pending)
    cases = {"c2_unflagged": (c2, lambda: c2_backlog(plain), per_step),
             "c2_flagged": (c2, lambda: c2_backlog(flagged), per_step),
             "deep_100x10": (deep, lambda: deep_backlog("deep_100x10"), DA * DD),
             "deep_1000_distinct": (deep, lambda: deep_backlog("deep_1000_distinct"), DA * DD)}

    def timed(sh, make):
        make()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        t = time.perf_counter()
        n = sh.supersede(None, archive=False)[1]          # synchronises: it returns totals
        wall = (time.perf_counter() - t) * 1e3
        e1.record(stream)
        torch.cuda.synchronize()
        return wall, e0.elapsed_time(e1), n

    res = {k: {"call_ms": [], "event_ms": []} for k in cases}
    retired, kern = {}, {}
    with torch.cuda.stream(stream):
        for sh, make, _ in cases.values():              # warm-up: every shape once
            timed(sh, make)
        clocks = ClockSampler(0); clocks.start()
        for _ in range(rounds):
            for name, (sh, make, _) in cases.items():
                for _ in range(block):
                    wall, ev, n = timed(sh, make)
                    res[name]["call_ms"].append(wall); res[name]["event_ms"].append(ev)
                    retired[name] = n
        clk = clocks.stop()
        for name, (sh, make, _) in cases.items():
            make()
            sh.profile(True)
            sh.supersede(None, archive=False)
            prof = sh.profile_read()
            sh.profile(False)
            kern[name] = {k: v[0] for k, v in prof.items() if v[1]}
    c2.close(); deep.close()
    out = {"config": f"c2 backlog: {wl.A} agents, {per_step} pending records, {wl.L}-B payloads; deep: {DA} agents x "
                     f"{DD} pending; {rounds} rounds of {block} calls per case, each on a fresh backlog"}
    for name, (_, _, N) in cases.items():
        A = wl.A if name.startswith("c2") else DA
        n = retired[name]
        flag = name != "c2_unflagged"
        # algorithmic bytes: the count walk (16-B ring header per agent, 8 B per ring entry, the header's last word from
        # one 32-B sector per record); with flagged records also the insert walk (the same, a whole sector per record,
        # a 24-B candidate and a 32-B table slot written), the tie and verdict passes (candidate and slot read twice,
        # a 4-B verdict word), the retire walk (header, entries, verdict words) and an 8-B tombstone per retired record
        nbytes = 16 * A + 8 * N + 32 * N
        if flag:
            nbytes += (16 * A + 8 * N + 32 * N + 24 * N + 32 * N) + 2 * (24 * N + 32 * N) + 4 * N + \
                      (16 * A + 8 * N + N // 8) + 8 * n
        kms = kern[name].get("expire", sum(kern[name].values()))
        out[name] = {"records_pending": N, "records_retired": n, "ms_per_call": float(np.median(res[name]["call_ms"])),
                     "event_ms_per_call": float(np.median(res[name]["event_ms"])), "kernel_ms": kern[name],
                     "supersede_kernel_ms": kms, "algorithmic_bytes": nbytes,
                     "algorithmic_gb_per_s_kernel": nbytes / (kms * 1e-3) / 1e9 if kms else None,
                     "share_of_3_35_TBps": nbytes / (kms * 1e-3) / 3.35e12 if kms else None,
                     "call_ms_blocks": res[name]["call_ms"]}
    # SwarmsDB flush of 4,096 point-to-point sends, 10 % flagged against none
    import tempfile
    n_agents, n_sends = 1024, 4096
    rng = np.random.default_rng(5)
    to = rng.integers(0, n_agents, n_sends).tolist()
    flag_mask = (rng.random(n_sends) < 0.1).tolist()
    with tempfile.TemporaryDirectory() as tmp:
        dbs = {name: sdb.SwarmsDB(save_dir=tmp, auto_save=False,
                                  gpu_config=sdb.GpuConfig(max_agents=n_sends, flush_threshold=n_sends + 1,
                                                           deterministic_ids=True))
               for name in ("flush_none_flagged", "flush_10pct_flagged")}
        names = [f"a{i}" for i in range(n_agents)]
        for db in dbs.values():
            for a in names:
                db.register_agent(a)
        flush_ms = {name: [] for name in dbs}
        for r in range(2 + rounds * block):
            for name, db in (dbs.items() if r % 2 == 0 else reversed(list(dbs.items()))):
                on = name == "flush_10pct_flagged"
                for i, a in enumerate(to):
                    db.send_message(names[i % n_agents], "x" * 100, receiver_id=names[a], supersede=on and flag_mask[i])
                torch.cuda.synchronize()
                t = time.perf_counter()
                db.flush()
                db.shard.sync()
                if r >= 2:
                    flush_ms[name].append((time.perf_counter() - t) * 1e3)
                db.shard.receive_batch(None, 1 << 10, copy_out=False)
                db.messages.clear(); db.agent_inbox.clear()
        superseded_db = dbs["flush_10pct_flagged"].get_stats()["superseded"]
        for db in dbs.values():
            db.close()
    for name, v in flush_ms.items():
        out[name] = {"ms_per_flush": float(np.median(v)), "ms_blocks": v, "sends": n_sends, "agents": n_agents}
    out["flush_10pct_flagged"]["records_superseded_total"] = superseded_db
    out.update(_gpu_card(0))
    out["clocks"] = clk
    return out


def where(rounds=3, block=4):
    """sdb_receive_where on the c2 backlog (1M agents, 65,536 group sends x 64 = 4,194,304 pending records): a
    header-clause PEEK over every agent, an ASCII-folded 8-byte keyword PEEK, and a take-mode filtered receive of one
    group's records (each take on a fresh backlog, rebuilt untimed); then a deep queue (10,000 agents x 1,000 pending
    64-byte records) for the keyword kernel's work distribution (DROP | PEEK: counted, nothing copied out), and the
    latency of a one-agent call.  Outside the timed region the c2 PEEK results are checked against the oracle's PEEK of
    the whole queue, filtered in numpy."""
    import torch
    from bench import ALNUM, ClockSampler, Workload
    from oracle.cpu_ref import CpuOracle
    from swarmdb_b200._native import HDR_DTYPE, RECV_PEEK, WHERE_DROP, Shard, make_filter, payload_offsets
    if not torch.cuda.is_available():
        raise SystemExit("bench_extra.py where: no CUDA device - swarmdb_b200 has no CPU fallback")
    wl = Workload()
    per_step = wl.S * wl.F
    rec_cap = per_step + (1 << 16)
    stream = torch.cuda.Stream()
    shard = Shard(max_agents=wl.A, ring_slots=64, arena_bytes=1 << 33, max_payload_bytes=wl.L, max_groups=1 << 14,
                  member_pool_entries=wl.A + 1024, max_batch_sends=wl.S, max_batch_payload=wl.S * wl.L,
                  max_recv_records=rec_cap, max_recv_payload=rec_cap * wl.L)
    shard.set_stream(stream.cuda_stream)
    shard.register(np.arange(wl.A, dtype=np.uint32))
    for g in range(wl.G):
        shard.create_group(g, wl.members(g))
    batch = wl.batch()
    snd, grp, prio, typ, lens, off, pay = batch
    g0 = int(grp[0])
    k0 = int(np.nonzero(grp != g0)[0][0])                 # the keyword's send is not among the records the take consumes
    kw = pay[int(off[k0]) + 20:int(off[k0]) + 28].tobytes().swapcase()

    def pinned(nbytes):
        return torch.empty(nbytes, dtype=torch.uint8, pin_memory=True).numpy()
    pin_hdr, pin_pay = pinned(rec_cap * 32).view(HDR_DTYPE), pinned(rec_cap * wl.L)

    def backlog():
        while shard.receive_batch(None, 1 << 10, copy_out=False)[1]:
            pass
        shard.send_group_batch(*batch)
        shard.sync()

    f_hdr, f_kw, f_grp = make_filter(prios=[3]), make_filter(keyword=kw, icase=True), make_filter(group=g0)
    calls = {"header_peek": (False, lambda: shard.receive_where(None, 100, RECV_PEEK, f_hdr, out_hdr=pin_hdr, out_payload=pin_pay)),
             "keyword_peek": (False, lambda: shard.receive_where(None, 100, RECV_PEEK, f_kw, out_hdr=pin_hdr, out_payload=pin_pay)),
             "take_group": (True, lambda: shard.receive_where(None, 100, 0, f_grp, out_hdr=pin_hdr, out_payload=pin_pay))}

    def timed(fn, fresh):
        if fresh:
            backlog()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        t = time.perf_counter()
        n = len(fn()[1])                                 # synchronises: it returns totals
        wall = (time.perf_counter() - t) * 1e3
        e1.record(stream)
        torch.cuda.synchronize()
        return wall, e0.elapsed_time(e1), n

    res = {k: {"call_ms": [], "event_ms": []} for k in calls}
    got = {}
    with torch.cuda.stream(stream):
        backlog()
        # outside the timed region: the PEEK queries against the oracle's PEEK of the whole queue, filtered in numpy
        o = CpuOracle(wl.A, wl.G)
        o.register(np.arange(wl.A))
        for g in range(wl.G):
            o.create_group(g, wl.members(g))
        o.send_group_batch(*batch)
        cc, hc, pc = o.receive_batch(np.arange(wl.A), 100, RECV_PEEK, rec_cap=per_step, pay_cap=per_step * wl.L)
        o.close()
        owner = np.repeat(np.arange(wl.A), cc.astype(np.int64))
        per_send = np.array([kw.lower() in pay[int(off[i]):int(off[i]) + int(lens[i])].tobytes().lower() for i in range(wl.S)])
        sel_kw = per_send[(hc["seq"].astype(np.int64) - int(hc["seq"].min())) // wl.F]
        checks = {}
        for name, keep in (("header_peek", hc["prio"] == 3), ("keyword_peek", sel_kw), ("take_group", hc["group"] == g0)):
            c, h, _ = shard.receive_where(None, 100, RECV_PEEK, {"header_peek": f_hdr, "keyword_peek": f_kw, "take_group": f_grp}[name])
            checks[name] = bool(np.array_equal(c, np.bincount(owner[keep], minlength=wl.A)[: len(c)]) and
                                h.tobytes() == hc[keep].tobytes())
        assert all(checks.values()), checks
        del hc, pc
        for fresh, fn in calls.values():                  # warm-up: every shape once
            timed(fn, fresh)
        backlog()
        clocks = ClockSampler(0); clocks.start()
        for _ in range(rounds):
            for name, (fresh, fn) in calls.items():
                for _ in range(block):
                    wall, ev, n = timed(fn, fresh)
                    res[name]["call_ms"].append(wall); res[name]["event_ms"].append(ev)
                    got[name] = n
        clk = clocks.stop()
        kern = {}
        for name, (fresh, fn) in calls.items():
            backlog()
            shard.profile(True)
            fn()
            prof = shard.profile_read()
            shard.profile(False)
            kern[name] = {k: v[0] for k, v in prof.items() if v[1]}
        # one agent, header clause, PEEK: the small-call latency (several launches even for one agent)
        one = np.array([int(wl.members(g0)[0])], np.uint32)
        for _ in range(20):
            shard.receive_where(one, 100, RECV_PEEK, f_grp)
        t = time.perf_counter()
        for _ in range(500):
            shard.receive_where(one, 100, RECV_PEEK, f_grp)
        one_us = (time.perf_counter() - t) / 500 * 1e6
    shard.close()
    # deep queues: 10,000 agents x 1,000 pending 64-byte records, keyword DROP | PEEK
    A2, D, L2 = 10_000, 1_000, 64
    deep = Shard(max_agents=A2, ring_slots=1024, arena_bytes=1 << 31, max_payload_bytes=L2, max_batch_sends=1 << 20,
                 max_batch_payload=(1 << 20) * L2)
    deep.register(np.arange(A2, dtype=np.uint32))
    rng = np.random.default_rng(5)
    n_all = A2 * D
    for b0 in range(0, n_all, 1 << 20):
        n = min(1 << 20, n_all - b0)
        r = (np.arange(b0, b0 + n) % A2).astype(np.uint32)
        dpay = ALNUM[rng.integers(0, 62, n * L2)]
        deep.send_batch(r, r, None, None, np.full(n, L2, np.uint16), np.arange(n, dtype=np.uint64) * L2, dpay)
    assert deep.queue_stats()["pending"] == n_all and deep.stats()["ring_overflow"] == 0
    dkw = dpay[:8].tobytes().swapcase()
    f_deep = make_filter(keyword=dkw, icase=True)
    deep_ms = []
    deep.receive_where(None, D, RECV_PEEK, f_deep, drop=True)
    for _ in range(rounds * block):
        t = time.perf_counter()
        _, deep_hits = deep.receive_where(None, D, RECV_PEEK, f_deep, drop=True)
        deep_ms.append((time.perf_counter() - t) * 1e3)
    deep.profile(True)
    deep.receive_where(None, D, RECV_PEEK, f_deep, drop=True)
    deep_kern = {k: v[0] for k, v in deep.profile_read().items() if v[1]}
    deep.close()

    peak = 3.35e12                                        # H100 SXM data sheet, HBM3
    out = {"config": f"c2 backlog: {wl.A} agents, {wl.S} group sends x {wl.F} members = {per_step} pending records, "
                     f"{wl.L}-B payloads; {rounds} rounds of {block} calls per query, takes on a fresh backlog; pinned "
                     f"host outputs", "oracle_checks": checks,
           "verdict_bitmap_bytes_c2": wl.A * ((64 + 31) // 32) * 4, "one_agent_peek_us": one_us}
    for name in calls:
        ms = float(np.median(res[name]["call_ms"]))
        kms = kern[name].get("where", 0.0)
        # algorithmic bytes of the selection kernels: 16-B ring header per agent and, per pending record, its 8-B entry
        # and 32-B header sector (the keyword pass also reads the 256-B payload of every record it searches)
        nbytes = 16 * wl.A + per_step * (40 + (wl.L if name == "keyword_peek" else 0))
        out[name] = {"records": got[name], "ms_per_call": ms, "event_ms_per_call": float(np.median(res[name]["event_ms"])),
                     "records_per_s_scanned": per_step / (ms * 1e-3), "kernel_ms": kern[name], "where_kernel_ms": kms,
                     "algorithmic_bytes": nbytes, "where_gb_per_s": nbytes / (kms * 1e-3) / 1e9 if kms else None,
                     "frac_of_3.35TB_s": nbytes / (kms * 1e-3) / peak if kms else None, "call_ms_blocks": res[name]["call_ms"]}
    dk = deep_kern.get("where", 0.0)
    dbytes = 16 * A2 + n_all * (40 + L2)
    out["deep_keyword_count"] = {"agents": A2, "pending_per_agent": D, "hits": deep_hits, "ms_per_call": float(np.median(deep_ms)),
                                 "records_per_s_scanned": n_all / (float(np.median(deep_ms)) * 1e-3), "where_kernel_ms": dk,
                                 "algorithmic_bytes": dbytes, "where_gb_per_s": dbytes / (dk * 1e-3) / 1e9 if dk else None,
                                 "frac_of_3.35TB_s": dbytes / (dk * 1e-3) / peak if dk else None}
    out.update(_gpu_card(0))
    out["clocks"] = clk
    return out


def ids(rounds=3):
    """The id clause of sdb_receive_where (SDB_FILTER_IDS) on the c2 backlog (1M agents, 65,536 group sends x 64 =
    4,194,304 pending records, one seq per record): (a) one drop call for 65,536 random pending ids with id_hits (the
    device call of SwarmsDB.delete_messages), each on a fresh backlog; (b) the per-id path delete_message used before,
    one SDB_FILTER_SEQ [s, s + 1) drop over every agent per id, for 64 of those ids, every call timed; (c) the calls of
    get_messages for 1,024 ids and of get_message for one: a DROP | PEEK count with id_agent over every agent, then a
    PEEK of the agents that hold them; (d) id_hits of one broadcast queued at every agent, the contention worst case.
    Outside the timed region the outputs are checked: every listed id is hit once, the 64 per-id drops remove one
    record each, the lookups return the listed seqs and the broadcast counts every agent."""
    import torch
    from bench import ClockSampler, Workload
    from swarmdb_b200._native import NO_RECEIVER, RECV_PEEK, WHERE_DROP, Shard, make_filter
    if not torch.cuda.is_available():
        raise SystemExit("bench_extra.py ids: no CUDA device - swarmdb_b200 has no CPU fallback")
    wl = Workload()
    per_step = wl.S * wl.F
    rec_cap = per_step + (1 << 16)
    stream = torch.cuda.Stream()
    shard = Shard(max_agents=wl.A, ring_slots=64, arena_bytes=1 << 33, max_payload_bytes=wl.L, max_groups=1 << 14,
                  member_pool_entries=wl.A + 1024, max_batch_sends=wl.S, max_batch_payload=wl.S * wl.L,
                  max_recv_records=rec_cap, max_recv_payload=rec_cap * wl.L, list_pool_entries=wl.A + 1024)
    shard.set_stream(stream.cuda_stream)
    shard.register(np.arange(wl.A, dtype=np.uint32))
    for g in range(wl.G):
        shard.create_group(g, wl.members(g))
    batch = wl.batch()
    rng = np.random.default_rng(17)
    state = {}

    def backlog():
        while shard.receive_batch(None, 1 << 10, copy_out=False)[1]:
            pass
        state["base"] = shard.send_group_batch(*batch)
        shard.sync()

    def timed(fn):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        t = time.perf_counter()
        r = fn()
        wall = (time.perf_counter() - t) * 1e3
        e1.record(stream)
        torch.cuda.synchronize()
        return wall, e0.elapsed_time(e1), r

    def profiled(fn):
        shard.profile(True)
        fn()
        prof = shard.profile_read()
        shard.profile(False)
        return {k: v[0] for k, v in prof.items() if v[1]}

    out = {"config": f"c2 backlog: {wl.A} agents, {wl.S} group sends x {wl.F} members = {per_step} pending records, "
                     f"{wl.L}-B payloads, one seq per record"}
    checks = {}
    with torch.cuda.stream(stream):
        backlog()
        seqs = lambda n: (state["base"] + rng.choice(per_step, n, replace=False)).astype(np.uint64)
        # (a) one bulk drop of 65,536 ids
        n_a = 1 << 16
        hits = np.zeros(n_a, np.uint32)
        bulk = lambda ids: shard.receive_where(None, n_a, WHERE_DROP, make_filter(ids=ids), drop=True, id_hits=hits)
        timed(lambda: bulk(seqs(n_a)))                                      # warm-up: allocates the id table
        a_ms, a_ev, a_kern = [], [], []
        for _ in range(rounds):
            backlog()
            ids_a = seqs(n_a)
            wall, ev, (_, dropped) = timed(lambda: bulk(ids_a))
            a_ms.append(wall); a_ev.append(ev)
            checks["bulk_drop_hits_one_each"] = bool((hits == 1).all()) and dropped == n_a
            backlog()
            ids_a = seqs(n_a)
            a_kern.append(profiled(lambda: bulk(ids_a)))
        # (b) the per-id seq-range drop, 64 calls
        backlog()
        one = lambda s: shard.receive_where(None, 1, WHERE_DROP, make_filter(seq=(int(s), int(s) + 1)), drop=True)
        timed(lambda: one(seqs(1)[0]))
        b_ms, b_ev, b_drop = [], [], 0
        for s in seqs(64):
            wall, ev, (_, d) = timed(lambda: one(s))
            b_ms.append(wall); b_ev.append(ev); b_drop += d
        checks["per_id_drops_one_each"] = b_drop == 64
        b_kern = profiled(lambda: one(seqs(1)[0]))
        # (c) get_messages (1,024 ids) and get_message (1 id): count with id_agent, then PEEK the holders
        backlog()

        def lookup(ids):
            where = np.zeros(len(ids), np.uint32)
            f = make_filter(ids=ids)
            shard.receive_where(None, 1, WHERE_DROP | RECV_PEEK, f, drop=True, id_agent=where)
            holders = np.unique(where[where != NO_RECEIVER]).astype(np.uint32)
            return shard.receive_where(holders, 1 << 20, RECV_PEEK, f)[1]
        look = {}
        for name, n in (("get_messages_1024", 1024), ("get_message_1", 1)):
            lookup(seqs(n))
            ms, ev = [], []
            for _ in range(rounds * 4):
                ids_c = seqs(n)
                wall, e, hdr = timed(lambda: lookup(ids_c))
                ms.append(wall); ev.append(e)
                checks[name + "_found"] = sorted(hdr["seq"].tolist()) == sorted(ids_c.tolist())
            look[name] = {"ms_per_call": float(np.median(ms)), "event_ms_per_call": float(np.median(ev)),
                          "kernel_ms": profiled(lambda: lookup(seqs(n)))}
        # (d) one broadcast queued at every agent: every record of the backlog is checked, all hits go to one slot
        backlog()
        shard.send_list_batch([0], np.array([0, wl.A], np.uint64), np.arange(wl.A, dtype=np.uint32), [1], [0], [16], [0],
                              np.zeros(64, np.uint8))
        shard.sync()
        bc = shard.stats()["next_seq"] - 1
        bh = np.zeros(1, np.uint32)
        count = lambda: shard.receive_where(None, 1, WHERE_DROP | RECV_PEEK, make_filter(ids=[bc]), drop=True, id_hits=bh)
        count()
        d_ms = [timed(count)[0] for _ in range(rounds * 4)]
        checks["broadcast_hits_every_agent"] = int(bh[0]) == wl.A
        d_kern = profiled(count)
        clocks = ClockSampler(0); clocks.start()
        clk_probe = [timed(count)[0] for _ in range(8)]
        clk = clocks.stop()
    shard.close()
    assert all(checks.values()), checks

    peak = 3.35e12                                        # H100 SXM data sheet, HBM3
    # algorithmic bytes of the where kernels: 16-B ring header per agent and, per pending record, its 8-B ring entry and
    # 32-B header sector, plus one 8-B key read per probe of the id table (one probe per record)
    scan = 16 * wl.A + per_step * (40 + 8)

    def rate(kern, nbytes):
        k = kern.get("where", 0.0)
        return {"where_kernel_ms": k, "algorithmic_bytes": nbytes, "where_gb_per_s": nbytes / (k * 1e-3) / 1e9 if k else None,
                "frac_of_3.35TB_s": nbytes / (k * 1e-3) / peak if k else None}
    a_k = [k.get("where", 0.0) for k in a_kern]
    out["bulk_drop_65536"] = {"ids": n_a, "records_dropped": n_a, "ms_per_call": float(np.median(a_ms)),
                              "event_ms_per_call": float(np.median(a_ev)), "kernel_ms": a_kern[-1],
                              **rate({"where": float(np.median(a_k))}, scan), "call_ms": a_ms}
    b_med = float(np.median(b_ms))
    out["per_id_drop"] = {"calls": 64, "ms_per_call": b_med, "event_ms_per_call": float(np.median(b_ev)),
                          "ms_64_calls_measured": float(np.sum(b_ms)), "kernel_ms": b_kern,
                          **rate(b_kern, 16 * wl.A + per_step * 40), "call_ms": b_ms}
    out["bulk_vs_per_id_per_message"] = {"bulk_us_per_id": float(np.median(a_ms)) * 1e3 / n_a, "per_id_us": b_med * 1e3}
    out.update(look)
    out["broadcast_every_agent"] = {"agents": wl.A, "ms_per_call": float(np.median(d_ms)), "kernel_ms": d_kern,
                                    **rate(d_kern, scan + 16 * wl.A + 40 * wl.A)}
    out["oracle_checks"] = checks
    out.update(_gpu_card(0))
    out["clocks"] = clk
    out["clock_probe_ms"] = clk_probe
    return out


def restore(rounds=3):
    """sdb_restore_compact on the c2 backlog (1M agents, 65,536 group sends x 64 = 4,194,304 pending records): a
    snapshot (PEEK compact receive into pinned host buffers), its restore into a fresh handle from those buffers, and the
    requeue of one full compact receive (rows renumbered by smallest seq, then restored behind an empty queue), each
    timed per call (wall clock around a synchronising call) with the restore kernels' time from the profiler.  Outside
    the timed region the restored handle's full drain is checked, by digests, against the original handle's, and the
    arena granules the restore took against those the original send took."""
    import torch
    from bench import ClockSampler, Workload
    from swarmdb_b200._native import ENTRY_DTYPE, RECV_PEEK, SEND_DTYPE, Shard
    from swarmdb_b200.core import _renumber_rows
    if not torch.cuda.is_available():
        raise SystemExit("bench_extra.py restore: no CUDA device - swarmdb_b200 has no CPU fallback")
    wl = Workload()
    per_step = wl.S * wl.F
    rec_cap = per_step + (1 << 16)

    def handle():
        s = Shard(max_agents=wl.A, ring_slots=64, arena_bytes=1 << 33, max_payload_bytes=wl.L, max_groups=1 << 14,
                  member_pool_entries=wl.A + 1024, max_batch_sends=wl.S, max_batch_payload=wl.S * wl.L,
                  max_recv_records=rec_cap, max_recv_payload=rec_cap * wl.L)
        s.register(np.arange(wl.A, dtype=np.uint32))
        for g in range(wl.G):
            s.create_group(g, wl.members(g))
        return s

    def pinned(nbytes):
        return torch.empty(nbytes, dtype=torch.uint8, pin_memory=True).numpy()

    def drain(s, digest=False):
        if digest:
            s.digest_reset()
        while True:
            _, total, _ = s.receive_batch(None, 1 << 10, copy_out=False)
            if digest:
                s.digest_fold()
            if not total:
                break
        return s.digest_read() if digest else None

    src, dst = handle(), handle()
    agents = np.arange(wl.A, dtype=np.uint32)
    pin_ent, pin_snd, pin_pay = pinned(rec_cap * 16).view(ENTRY_DTYPE), pinned(rec_cap * 32).view(SEND_DTYPE), pinned(rec_cap * wl.L)
    t0 = src.stats()["arena_tail_bytes"]
    src.send_group_batch(*wl.batch())
    sent_bytes = src.stats()["arena_tail_bytes"] - t0

    def snapshot():
        return src.receive_compact(None, 1 << 10, RECV_PEEK, out_entries=pin_ent, out_sends=pin_snd, out_payload=pin_pay)

    cnt, ent, snd, pay = snapshot()
    ent2, snd2 = _renumber_rows(ent, snd)
    pin_ent2, pin_snd2 = pinned(len(ent2) * 16).view(ENTRY_DTYPE), pinned(len(snd2) * 32).view(SEND_DTYPE)
    pin_ent2[:], pin_snd2[:] = ent2, snd2
    cnt = cnt.copy()
    n_rec, n_rows = len(ent2), len(snd2)

    def timed(fn, before=None):
        res = {"wall_ms": [], "kernel_ms": []}
        for _ in range(rounds):
            if before:
                before()
            for s in (src, dst):
                s.sync(); s.profile(True)
            t = time.perf_counter()
            part = fn()
            res["wall_ms"].append((time.perf_counter() - t) * 1e3)
            if isinstance(part, float):                      # the part of the call the step times itself
                res.setdefault("part_ms", []).append(part)
            k = 0.0
            for s in (src, dst):
                prof = s.profile_read(); s.profile(False)
                k += prof["restore"][0] + prof["recv_compact"][0] + sum(prof[x][0] for x in ("recv_count", "recv_scan", "recv_select"))
            res["kernel_ms"].append(k)
        return {k: float(np.median(v)) for k, v in res.items()} | {"per_round": res}

    clocks = ClockSampler(0); clocks.start()
    out = {"snapshot": timed(snapshot)}
    out["restore"] = timed(lambda: dst.restore_compact(agents, cnt, pin_ent2, pin_snd2, pin_pay[: len(pay)]),
                           before=lambda: drain(dst))
    # outside the timed region: the restored queue drains to the original's digests, in the original's arena bytes
    drain(dst)
    t1 = dst.stats()["arena_tail_bytes"]
    dst.restore_compact(agents, cnt, pin_ent2, pin_snd2, pin_pay[: len(pay)])
    restored_bytes = dst.stats()["arena_tail_bytes"] - t1
    same = bool(np.array_equal(drain(dst, True), drain(src, True)))

    def requeue():
        c, e, s, p = src.receive_compact(None, 1 << 10, 0, out_entries=pin_ent, out_sends=pin_snd, out_payload=pin_pay)
        t = time.perf_counter()
        e, s = _renumber_rows(e, s)
        src.restore_compact(agents, c, e, s, p)
        return (time.perf_counter() - t) * 1e3

    def refill():
        drain(src)
        src.send_group_batch(*wl.batch())
    out["requeue_receive_plus_restore"] = timed(requeue, before=refill)
    clk = clocks.stop()
    src.close(); dst.close()
    rk = out["restore"]["kernel_ms"]
    alg = n_rec * (16 + 32 + 8) + n_rows * (32 + 2 * ((wl.L + 31) & ~31))
    out.update({"config": f"c2 backlog: {wl.A} agents, {wl.S} group sends x {wl.F} members = {per_step} pending records, "
                          f"{wl.L}-B payloads; pinned host buffers; {rounds} calls each",
                "records": n_rec, "rows": n_rows, "h2d_bytes": n_rec * 16 + n_rows * 32 + len(pay),
                "restore_alg_bytes": alg, "restore_kernel_gbps": alg / (rk * 1e-3) / 1e9,
                "restore_floor_us_at_3.35TBps": alg / 3.35e12 * 1e6,
                "drain_digests_equal": same, "arena_bytes_sent": sent_bytes, "arena_bytes_restored": restored_bytes,
                "clocks": clk})
    out.update(_gpu_card(0))
    return out


def lease(rounds=3):
    """Leased receives on the c2 backlog (1M agents, 65,536 group sends x 64 = 4,194,304 pending records): a leased
    receive of the whole backlog against a plain compact receive of it (alternated, each after a fresh send), the settle
    of the acks of every other record (2,097,152 ids), the sweep that redelivers the other half, and, for comparison, the
    host requeue of the same half (requeue_batch_compact: rows renumbered on the host, then restored from host memory).
    Per call: wall clock around the synchronising call, and the `lease` kernel time from the profiler (the sweep's
    restore phases are reported apart).  Outside the timed region the redelivered half is checked by digests against
    the same half requeued on a twin handle."""
    import torch
    from bench import ClockSampler, Workload
    from swarmdb_b200._native import ENTRY_DTYPE, LEASE_ACK, LEASE_ALL, SEND_DTYPE, Shard, pad32
    from swarmdb_b200.core import _renumber_rows
    if not torch.cuda.is_available():
        raise SystemExit("bench_extra.py lease: no CUDA device - swarmdb_b200 has no CPU fallback")
    wl = Workload()
    per_step = wl.S * wl.F
    rec_cap = per_step + (1 << 16)

    def handle():
        s = Shard(max_agents=wl.A, ring_slots=64, arena_bytes=1 << 33, max_payload_bytes=wl.L, max_groups=1 << 14,
                  member_pool_entries=wl.A + 1024, max_batch_sends=wl.S, max_batch_payload=wl.S * wl.L,
                  max_recv_records=rec_cap, max_recv_payload=rec_cap * wl.L)
        s.register(np.arange(wl.A, dtype=np.uint32))
        for g in range(wl.G):
            s.create_group(g, wl.members(g))
        return s

    def pinned(nbytes):
        return torch.empty(nbytes, dtype=torch.uint8, pin_memory=True).numpy()

    def drain(s, digest=False):
        if digest:
            s.digest_reset()
        while True:
            _, total, _ = s.receive_batch(None, 1 << 10, copy_out=False)
            if digest:
                s.digest_fold()
            if not total:
                break
        return s.digest_read() if digest else None

    src, twin = handle(), handle()
    src.lease_reserve(rec_cap, rec_cap * pad32(wl.L))
    agents = np.arange(wl.A, dtype=np.uint32)
    pin_ent, pin_snd, pin_pay = pinned(rec_cap * 16).view(ENTRY_DTYPE), pinned(rec_cap * 32).view(SEND_DTYPE), pinned(rec_cap * wl.L)
    batch = wl.batch()

    def call(fn):
        src.sync(); src.profile(True)
        t = time.perf_counter()
        r = fn()
        wall = (time.perf_counter() - t) * 1e3
        prof = src.profile_read(); src.profile(False)
        recv = prof["recv_compact"][0] + sum(prof[x][0] for x in ("recv_count", "recv_scan", "recv_select"))
        return r, {"wall_ms": wall, "lease_kernel_ms": prof["lease"][0], "restore_kernel_ms": prof["restore"][0],
                   "receive_kernel_ms": recv}

    def med(rows):
        return {k: float(np.median([r[k] for r in rows])) for k in rows[0]} | {"per_round": rows}

    clocks = ClockSampler(0); clocks.start()
    plain, leased, settle, sweep, requeue = [], [], [], [], []
    for _ in range(rounds):
        for kind in ("plain", "leased"):
            drain(src)
            if src.lease_stats()["live"]:
                src.lease_sweep(0.0, LEASE_ALL); drain(src)
            src.send_group_batch(*batch)
            if kind == "plain":
                res, t = call(lambda: src.receive_compact(None, 1 << 10, 0, out_entries=pin_ent, out_sends=pin_snd,
                                                          out_payload=pin_pay))
                assert len(res[1]) == per_step
                plain.append(t)
            else:
                res, t = call(lambda: src.receive_leased(None, 1 << 10, 1.0, 0, out_entries=pin_ent, out_sends=pin_snd,
                                                         out_payload=pin_pay))
                assert len(res[1]) == per_step
                leased.append(t)
                base = res[4]
                half = np.arange(base, base + per_step, 2, dtype=np.uint64)
                (_, n_acked), t = call(lambda: src.lease_settle(half, LEASE_ACK))
                assert n_acked == len(half)
                settle.append(t)
                (red, blocked, left), t = call(lambda: src.lease_sweep(2.0))
                assert red == per_step - len(half) and blocked == 0 and left == 0
                sweep.append(t)
    # the host requeue of the same half (rows renumbered by smallest seq, restored from host memory), and the digest check
    drain(src)
    src.send_group_batch(*batch)
    c, e, s, p, base = src.receive_leased(None, 1 << 10, 1.0, 0, out_entries=pin_ent, out_sends=pin_snd, out_payload=pin_pay)
    keep = np.zeros(len(e), bool); keep[1::2] = True                  # the unacked half, as the sweep redelivers it
    who = np.repeat(np.arange(len(c)), c.astype(np.int64))
    cnt_half = np.bincount(who[keep], minlength=len(c)).astype(np.uint32)
    e_half = e[keep].copy(); s_all = s.copy(); p_all = p.copy()
    src.lease_settle(np.arange(base, base + len(e), 2, dtype=np.uint64), LEASE_ACK)
    src.lease_sweep(2.0)
    want = drain(src, True)
    for _ in range(rounds):
        drain(twin)
        twin.send_group_batch(*batch)
        twin.receive_compact(None, 1 << 10, 0, out_entries=pin_ent, out_sends=pin_snd, out_payload=pin_pay)
        twin.sync()
        t0 = time.perf_counter()
        ent2, snd2 = _renumber_rows(e_half, s_all)
        twin.restore_compact(agents, cnt_half, ent2, snd2, p_all)
        requeue.append({"wall_ms": (time.perf_counter() - t0) * 1e3})
    same = bool(np.array_equal(drain(twin, True), want))
    clk = clocks.stop()
    src.close(); twin.close()
    out = {"receive_compact": med(plain), "receive_leased": med(leased), "settle_acks": med(settle),
           "sweep_redeliver_half": med(sweep), "requeue_batch_compact_same_half": med(requeue),
           "config": f"c2 backlog: {wl.A} agents, {wl.S} group sends x {wl.F} members = {per_step} records, {wl.L}-B "
                     f"payloads; pinned host buffers; leased and plain receives alternated, {rounds} rounds",
           "records": per_step, "acked": per_step // 2, "redelivered": per_step - per_step // 2,
           "redelivered_digests_equal_requeue": same, "clocks": clk}
    out.update(_gpu_card(0))
    return out


def deadletter(rounds=3):
    """Dead letters on the c2 backlog (1M agents, 65,536 group sends x 64 = 4,194,304 records), every leased record
    nacked before each sweep:
      - a leased receive of the whole backlog with the policy on and an empty ledger, alternated with the policy off;
      - with M = 1, the sweep that dead-letters every record, the take of all of them into pinned buffers, and the
        redrive of what was taken (sdb_restore_compact of it as it stands);
      - with M = 2, the sweep that fills the ledger and the leased receive that looks every record up, against the same
        sweep and receive with the policy off.
    Per call: wall clock around the synchronising call and the `lease` (and `restore`) kernel time from the profiler."""
    import torch
    from bench import ClockSampler, Workload
    from swarmdb_b200._native import ENTRY_DTYPE, LEASE_ACK, LEASE_RENEW, SEND_DTYPE, Shard, pad32
    if not torch.cuda.is_available():
        raise SystemExit("bench_extra.py deadletter: no CUDA device - swarmdb_b200 has no CPU fallback")
    wl = Workload()
    per_step = wl.S * wl.F
    rec_cap = per_step + (1 << 16)
    s = Shard(max_agents=wl.A, ring_slots=64, arena_bytes=1 << 33, max_payload_bytes=wl.L, max_groups=1 << 14,
              member_pool_entries=wl.A + 1024, max_batch_sends=wl.S, max_batch_payload=wl.S * wl.L,
              max_recv_records=rec_cap, max_recv_payload=rec_cap * wl.L)
    s.register(np.arange(wl.A, dtype=np.uint32))
    for g in range(wl.G):
        s.create_group(g, wl.members(g))
    s.lease_reserve(rec_cap, rec_cap * pad32(wl.L))
    pin = lambda n: torch.empty(n, dtype=torch.uint8, pin_memory=True).numpy()          # noqa: E731
    pin_ent, pin_snd, pin_pay = pin(rec_cap * 16).view(ENTRY_DTYPE), pin(rec_cap * 32).view(SEND_DTYPE), pin(rec_cap * wl.L)
    batch = wl.batch()

    def drain():
        while s.receive_batch(None, 1 << 10, copy_out=False)[1]:
            pass

    def clear():                              # every lease was acked or taken: compact the store, drain, fresh backlog
        s.lease_sweep(0.0)
        assert s.lease_stats()["entries_used"] == 0
        drain()
        s.send_group_batch(*batch)

    def call(fn):
        s.sync(); s.profile(True)
        t = time.perf_counter()
        r = fn()
        wall = (time.perf_counter() - t) * 1e3
        prof = s.profile_read(); s.profile(False)
        return r, {"wall_ms": wall, "lease_kernel_ms": prof["lease"][0], "restore_kernel_ms": prof["restore"][0]}

    def med(rows):
        return {k: float(np.median([r[k] for r in rows])) for k in rows[0]} | {"per_round": rows}

    def lease():
        return s.receive_leased(None, 1 << 10, 1.0, 0, out_entries=pin_ent, out_sends=pin_snd, out_payload=pin_pay)

    def nack(base):
        s.lease_settle(np.arange(base, base + per_step, dtype=np.uint64), LEASE_RENEW, -np.inf)

    clocks = ClockSampler(0); clocks.start()
    rows = {k: [] for k in ("lease_policy_off", "lease_policy_on_empty_ledger", "sweep_m1_dead_letters_all", "take_all",
                            "redrive_all", "sweep_m2_fills_ledger", "lease_m2_looks_up_all", "sweep_policy_off",
                            "lease_after_sweep_policy_off")}
    for _ in range(rounds):
        for on in (False, True):
            clear()
            s.lease_set_policy(0xFFFFFFFF if on else 0, rec_cap if on else 0)
            r, t = call(lease)
            assert len(r[1]) == per_step
            rows["lease_policy_on_empty_ledger" if on else "lease_policy_off"].append(t)
            s.lease_settle(np.arange(r[4], r[4] + per_step, dtype=np.uint64), LEASE_ACK)
        # M = 1: every record dies; take them all; redrive them
        clear(); s.lease_set_policy(0, 0); s.lease_set_policy(1, rec_cap)
        r = lease(); nack(r[4])
        (red, blocked, left), t = call(lambda: s.lease_sweep(0.0))
        assert red == 0 and s.lease_policy_stats()["dead"] == per_step
        rows["sweep_m1_dead_letters_all"].append(t)
        (c, e, sn, p, d), t = call(lambda: s.lease_dead_letters(None, 0, out_entries=pin_ent, out_sends=pin_snd, out_payload=pin_pay))
        assert len(e) == per_step
        rows["take_all"].append(t)
        (n, _), t = call(lambda: s.restore_compact(np.arange(len(c), dtype=np.uint32), c, e, sn, p))
        assert n == per_step
        rows["redrive_all"].append(t)
        # M = 2 against no policy: the sweep after a nack of everything, then the leased receive of the redelivered records
        for on in (True, False):
            clear(); s.lease_set_policy(0, 0)
            if on:
                s.lease_set_policy(2, rec_cap)
            r = lease(); nack(r[4])
            (red, _, _), t = call(lambda: s.lease_sweep(0.0))
            assert red == per_step
            rows["sweep_m2_fills_ledger" if on else "sweep_policy_off"].append(t)
            r, t = call(lease)
            assert len(r[1]) == per_step
            rows["lease_m2_looks_up_all" if on else "lease_after_sweep_policy_off"].append(t)
            if on:
                assert int(s.lease_deliveries(np.array([r[4]], np.uint64))[0]) == 2
            s.lease_settle(np.arange(r[4], r[4] + per_step, dtype=np.uint64), LEASE_ACK)
    clk = clocks.stop()
    s.close()
    out = {k: med(v) for k, v in rows.items()}
    out.update({"config": f"c2 backlog: {wl.A} agents, {wl.S} group sends x {wl.F} members = {per_step} records, {wl.L}-B "
                          f"payloads; pinned host buffers; {rounds} rounds", "records": per_step, "clocks": clk})
    out.update(_gpu_card(0))
    return out


def lease_snapshot(rounds=3):
    """Snapshots of in-flight work on the c2 backlog (1M agents, 65,536 group sends x 64 = 4,194,304 records), policy
    M = 3: the whole backlog leased, half of it nacked and swept back, so the store holds 2,097,152 live leases and the
    ledger 2,097,152 counts of redelivered records still pending.  Per round:
      - the export of the whole store into pinned buffers (one call) and the ledger export;
      - into a fresh handle that was given the pending records (restore, not timed): the ledger import, then the lease
        import of the exported chunk.
    Per call: wall clock around the synchronising call and the `lease` kernel time from the profiler; algorithmic bytes of
    the store calls (the compact output read from the store and written once, or read once and written to the store)
    over that kernel time, against the H100 SXM's 3.35 TB/s."""
    import torch
    from bench import ClockSampler, Workload
    from swarmdb_b200._native import ENTRY_DTYPE, LEASE_RENEW, META_DTYPE, RECV_PEEK, SEND_DTYPE, Shard, pad32
    if not torch.cuda.is_available():
        raise SystemExit("bench_extra.py lease_snapshot: no CUDA device - swarmdb_b200 has no CPU fallback")
    wl = Workload()
    per_step = wl.S * wl.F
    rec_cap = per_step + (1 << 16)
    M = 3

    def shard():
        x = Shard(max_agents=wl.A, ring_slots=64, arena_bytes=1 << 33, max_payload_bytes=wl.L, max_groups=1 << 14,
                  member_pool_entries=wl.A + 1024, max_batch_sends=wl.S, max_batch_payload=wl.S * wl.L,
                  max_recv_records=rec_cap, max_recv_payload=rec_cap * wl.L)
        x.register(np.arange(wl.A, dtype=np.uint32))
        for g in range(wl.G):
            x.create_group(g, wl.members(g))
        x.lease_reserve(rec_cap, rec_cap * pad32(wl.L))
        x.lease_set_policy(M, rec_cap)
        return x

    pin = lambda n: torch.empty(n, dtype=torch.uint8, pin_memory=True).numpy()          # noqa: E731
    pin_ent, pin_snd, pin_pay = pin(rec_cap * 16).view(ENTRY_DTYPE), pin(rec_cap * 32).view(SEND_DTYPE), pin(rec_cap * wl.L)
    pin_meta = pin(rec_cap * 32).view(META_DTYPE)
    s = shard()
    s.send_group_batch(*wl.batch())
    base = s.receive_leased(None, 1 << 10, 1e300, 0, out_entries=pin_ent, out_sends=pin_snd, out_payload=pin_pay)[4]
    s.lease_settle(np.arange(base, base + per_step // 2, dtype=np.uint64), LEASE_RENEW, -np.inf)
    assert s.lease_sweep(0.0)[0] == per_step // 2
    cnt, ent, snd, pay = (x.copy() for x in s.receive_compact(None, 1 << 10, RECV_PEEK, out_entries=pin_ent,
                                                              out_sends=pin_snd, out_payload=pin_pay))

    def call(x, fn):
        x.sync(); x.profile(True)
        t = time.perf_counter()
        r = fn()
        wall = (time.perf_counter() - t) * 1e3
        prof = x.profile_read(); x.profile(False)
        return r, {"wall_ms": wall, "lease_kernel_ms": prof["lease"][0]}

    def med(rows):
        return {k: float(np.median([r[k] for r in rows])) for k in rows[0]} | {"per_round": rows}

    clocks = ClockSampler(0); clocks.start()
    rows = {k: [] for k in ("export_store", "export_ledger", "import_ledger", "import_store")}
    for _ in range(rounds):
        (e, sn, p, m, nxt), t = call(s, lambda: s.lease_export(0, pin_ent, pin_snd, pin_pay, pin_meta))
        assert len(e) == per_step // 2 and len(s.lease_export(nxt, pin_ent, pin_snd, pin_pay, pin_meta)[0]) == 0
        moved = 2 * (len(e) * (16 + 32) + len(sn) * 32 + len(p))
        rows["export_store"].append(t | {"bytes": moved, "tb_per_s": moved / t["lease_kernel_ms"] / 1e9})
        (la, ls, lc), t = call(s, s.ledger_export)
        assert len(la) == per_step // 2
        rows["export_ledger"].append(t)
        d = shard()
        assert d.restore_compact(np.arange(len(cnt), dtype=np.uint32), cnt, ent, snd, pay)[0] == per_step // 2
        n, t = call(d, lambda: d.ledger_import(la, ls, lc))
        assert n == len(la)
        rows["import_ledger"].append(t)
        b, t = call(d, lambda: d.lease_import(e, sn, p, m))
        rows["import_store"].append(t | {"bytes": moved, "tb_per_s": moved / t["lease_kernel_ms"] / 1e9})
        assert d.lease_stats()["live"] == per_step // 2
        d.close()
    clk = clocks.stop()
    s.close()
    out = {k: med(v) for k, v in rows.items()}
    out.update({"config": f"c2 backlog: {wl.A} agents, {wl.S} group sends x {wl.F} members = {per_step} records, {wl.L}-B "
                          f"payloads, all leased, half nacked and swept back (M = {M}); pinned host buffers; {rounds} rounds",
                "leases": per_step // 2, "ledger_counts": per_step // 2, "peak_tb_per_s": 3.35, "clocks": clk})
    out.update(_gpu_card(0))
    return out


def budget(rounds=2, per_agent=2):
    """Receive by byte budget (sdb_receive_compact_budget).
    drain: GpuConfig's default caps (32 KB max_payload_bytes, 64 MB and 65536 records per call) and a backlog of
      256-byte messages, `per_agent` per agent over 1 M agents, drained into pinned buffers by receive_compact (sized
      for the worst case: 2048 records per call) and by the budget call without a per-agent limit (sized by the bytes
      selected), alternated; calls, wall time per record drained and D2H bytes.
    plan: the c2 backlog (bench.py's step, 4,194,304 records over 1 M agents) received with a per-agent limit of two
      padded payloads (half of each queue) against the plain receive; the plan kernel's time from the library profiler
      (PEEK calls: the backlog stays)."""
    import torch
    from bench import Workload
    from swarmdb_b200._native import ENTRY_DTYPE, RECV_PEEK, SEND_DTYPE, Shard, pad32
    if not torch.cuda.is_available():
        raise SystemExit("bench_extra.py budget: no CUDA device - swarmdb_b200 has no CPU fallback")

    def pinned(nbytes):
        return torch.empty(nbytes, dtype=torch.uint8, pin_memory=True).numpy()

    # ---- drain at the default caps
    A, L, P = 1 << 20, 256, 32768
    n = A * per_agent
    shard = Shard(max_agents=A, ring_slots=64, arena_bytes=1 << 31, max_payload_bytes=P, max_batch_sends=1 << 16,
                  max_batch_payload=(1 << 16) * L, max_recv_records=1 << 16, max_recv_payload=1 << 26)
    shard.register(np.arange(A, dtype=np.uint32))
    rng = np.random.default_rng(7)
    B = 1 << 16
    recv_all = np.tile(np.arange(A, dtype=np.uint32), per_agent)
    pay_in = rng.integers(0, 256, B * L, dtype=np.uint8)
    off = (np.arange(B, dtype=np.uint64) * L)
    lens, z8, ts = np.full(B, L, np.uint16), np.zeros(B, np.uint8), np.zeros(B)

    def fill():
        for i in range(0, n, B):
            shard.send_batch(recv_all[i:i + B] ^ 1, recv_all[i:i + B], z8, z8, lens, off, pay_in, ts)
        shard.sync()

    pin_ent = pinned((1 << 16) * 16).view(ENTRY_DTYPE)
    pin_snd = pinned((1 << 16) * 32).view(SEND_DTYPE)
    pin_pay = pinned(1 << 26)
    seqs = {}

    def drain(name):
        calls, recs, d2h = 0, 0, 0
        got = []
        t = time.perf_counter()
        while True:
            kw = {} if name == "compact" else {"max_agent_bytes": 0}
            cnt, ent, snd, pay = shard.receive_compact(None, 100, 0, out_entries=pin_ent, out_sends=pin_snd,
                                                       out_payload=pin_pay, **kw)
            calls += 1
            d2h += len(cnt) * 4 + len(ent) * 16 + len(snd) * 32 + len(pay) + 24
            if len(ent) == 0:
                break
            recs += len(ent)
            got.append(ent["seq"].copy())
        sec = time.perf_counter() - t
        seqs[name] = np.sort(np.concatenate(got))
        return {"calls": calls, "records": recs, "s": sec, "ns_per_record": sec * 1e9 / recs, "d2h_bytes": d2h}

    res = {"compact": [], "budget": []}
    for r in range(rounds):
        for name in (("compact", "budget") if r % 2 == 0 else ("budget", "compact")):
            fill()
            res[name].append(drain(name))
    assert all(np.array_equal(s - s[0], np.arange(n)) for s in seqs.values())     # both drains took every message once
    st = shard.stats()
    assert st["ring_overflow"] == 0 and st["delivered"] == st["enqueued"]
    shard.close()
    out = {"drain_config": f"{A} agents x {per_agent} messages of {L} B, max_payload_bytes {P}, 64 MB / 65536 records "
                           f"per call, pinned outputs; {rounds} rounds, order alternated",
           "drain": {k: {"runs": v, "ns_per_record": float(np.median([x["ns_per_record"] for x in v])),
                         "calls": v[-1]["calls"], "d2h_bytes": v[-1]["d2h_bytes"]} for k, v in res.items()}}

    # ---- plan kernel on the c2 backlog, per-agent limit of half of each queue
    wl = Workload()
    per_step = wl.S * wl.F
    rec_cap = per_step + (1 << 16)
    shard = Shard(max_agents=wl.A, ring_slots=64, arena_bytes=1 << 33, max_payload_bytes=wl.L, max_groups=1 << 14,
                  member_pool_entries=wl.A + 1024, max_batch_sends=wl.S, max_batch_payload=wl.S * wl.L,
                  max_recv_records=rec_cap, max_recv_payload=rec_cap * wl.L)
    shard.register(np.arange(wl.A, dtype=np.uint32))
    for g in range(wl.G):
        shard.create_group(g, wl.members(g))
    shard.send_group_batch(*wl.batch())
    shard.sync()
    limit = 2 * pad32(wl.L)
    reps = 20
    kern, recs = {}, {}
    for name, kw in (("plain", {}), ("budget", {"max_agent_bytes": limit})) * 2:
        shard.receive_compact(None, 100, RECV_PEEK, **kw)                     # warm-up
        shard.profile(True)
        for _ in range(reps):
            cnt, ent, _, _ = shard.receive_compact(None, 100, RECV_PEEK, **kw)
        prof = shard.profile_read()
        shard.profile(False)
        kern.setdefault(name, []).append(prof["recv_select"][0] / reps)
        recs[name] = len(ent)
    shard.close()
    out["plan_config"] = (f"c2 backlog: {per_step} records over {wl.A} agents, {wl.L}-B payloads; per-agent limit "
                          f"{limit} B; PEEK compact receives, {reps} per block, blocks alternated")
    out["plan"] = {k: {"plan_ms_blocks": v, "plan_ms": float(np.median(v)), "records": recs[k]} for k, v in kern.items()}
    out.update(_gpu_card(0))
    return out


def tokens(rounds=2, reps=10):
    """Receive by token budget (sdb_receive_compact_tokens, sdb_pending_tokens).
    c2: the c2 backlog (bench.py's step, 4,194,304 records over 1 M agents) with every send tagged (TYPEF_TOKENS,
      counts uniform in 1..512): a token-limited PEEK (512 tokens, about half of each queue) against a budget PEEK of
      two padded payloads (the same share by bytes); wall time per call, and the plan (recv_select) and token pre-pass
      (recv_count) kernel times from the library profiler.  pending_tokens over the 1 M agents.
    deep: 10,000 agents x 1,000 pending tagged records (16-byte payloads, private images), a limit near a quarter of
      each window's tokens, in stream and priority order.
    Algorithmic bytes of the pre-pass: a 16-B ring header per agent, 8 B per ring entry, one 32-B header sector per
    record and one payload sector per distinct tagged payload it reads, over its kernel time, against the 3.35 TB/s
    of NVIDIA's H100 SXM data sheet.  The c2 windows (4 records) fit one 32-entry step, which reads them all; a deep
    stream-order walk stops at the end of the step holding the first record that does not fit; a priority-order walk
    reads every record once for its level totals (the bytes given: the second walk over the cut level is left out,
    so the rate is a lower bound)."""
    import torch
    from bench import Workload
    from swarmdb_b200._native import RECV_PEEK, RECV_PRIORITY, Shard, pad32
    if not torch.cuda.is_available():
        raise SystemExit("bench_extra.py tokens: no CUDA device - swarmdb_b200 has no CPU fallback")
    TOK, HBM = 0x40, 3.35e12

    def timed(shard, fn):
        fn()                                                                  # warm-up
        shard.sync()
        shard.profile(True)
        t = time.perf_counter()
        for _ in range(reps):
            r = fn()
        shard.sync()
        wall = (time.perf_counter() - t) * 1e3 / reps
        prof = shard.profile_read()
        shard.profile(False)
        return r, {"call_ms": wall, "prepass_ms": prof["recv_count"][0] / reps, "plan_ms": prof["recv_select"][0] / reps}

    def share(ms, nbytes):
        return {"algorithmic_bytes": nbytes, "prepass_tb_s": nbytes / (ms * 1e-3) / 1e12 if ms else None,
                "share_of_3_35_tb_s": nbytes / (ms * 1e-3) / HBM if ms else None}

    out = {}
    # ---- c2
    wl = Workload()
    rng = np.random.default_rng(9)
    snd, grp, prio, typ, lens, off, pay = wl.batch()
    pay = pay.copy()
    pay.reshape(wl.S, wl.L)[:, :4] = rng.integers(1, 513, wl.S).astype(np.uint32).view(np.uint8).reshape(wl.S, 4)
    typ = np.full(wl.S, TOK, np.uint8)
    per_step = wl.S * wl.F
    rec_cap = per_step + (1 << 16)
    shard = Shard(max_agents=wl.A, ring_slots=64, arena_bytes=1 << 33, max_payload_bytes=wl.L, max_groups=1 << 14,
                  member_pool_entries=wl.A + 1024, max_batch_sends=wl.S, max_batch_payload=wl.S * wl.L,
                  max_recv_records=rec_cap, max_recv_payload=rec_cap * wl.L)
    shard.register(np.arange(wl.A, dtype=np.uint32))
    for g in range(wl.G):
        shard.create_group(g, wl.members(g))
    shard.send_group_batch(snd, grp, prio, typ, lens, off, pay)
    shard.sync()
    res = {"tokens": [], "budget": [], "pending_tokens": []}
    recs = {}
    for r in range(rounds):
        for name in (("tokens", "budget", "pending_tokens") if r % 2 == 0 else ("pending_tokens", "budget", "tokens")):
            if name == "tokens":
                got, t = timed(shard, lambda: shard.receive_compact_tokens(None, 100, 512, 0, RECV_PEEK))
            elif name == "budget":
                got, t = timed(shard, lambda: shard.receive_compact(None, 100, RECV_PEEK, max_agent_bytes=2 * pad32(wl.L)))
            else:
                got, t = timed(shard, lambda: shard.pending_tokens())
            recs[name] = len(got[1]) if name != "pending_tokens" else int(got.sum())
            res[name].append(t)
    shard.close()
    nbytes = 16 * wl.A + 8 * per_step + 32 * per_step + 32 * wl.S
    out["c2_config"] = (f"c2 backlog: {per_step} records over {wl.A} agents, {wl.L}-B payloads, every send tagged "
                        f"(counts 1..512); token limit 512 vs byte limit {2 * pad32(wl.L)} B; PEEK compact receives, "
                        f"{reps} per block, blocks alternated")
    out["c2"] = {k: {"blocks": v, **{f: float(np.median([x[f] for x in v])) for f in ("call_ms", "prepass_ms", "plan_ms")},
                     "result": recs[k]} for k, v in res.items()}
    for k in ("tokens", "pending_tokens"):
        out["c2"][k].update(share(out["c2"][k]["prepass_ms"], nbytes))

    # ---- 10,000 agents x 1,000 pending
    A, D, L = 10_000, 1_000, 16
    n = A * D
    shard = Shard(max_agents=A, ring_slots=1024, arena_bytes=1 << 30, max_payload_bytes=64, max_batch_sends=1 << 16,
                  max_batch_payload=(1 << 16) * L, max_recv_records=1 << 22, max_recv_payload=1 << 28)
    shard.register(np.arange(A, dtype=np.uint32))
    B = 1 << 16
    recv_all = np.tile(np.arange(A, dtype=np.uint32), D)
    lens, ts = np.full(B, L, np.uint16), np.zeros(B)
    t8 = np.full(B, TOK, np.uint8)
    poff = np.arange(B, dtype=np.uint64) * L
    for i in range(0, n, B):
        m = min(B, n - i)
        p = rng.integers(0, 256, B * L, dtype=np.uint8)
        p.reshape(B, L)[:, :4] = rng.integers(1, 513, B).astype(np.uint32).view(np.uint8).reshape(B, 4)
        shard.send_batch(recv_all[i:i + m] ^ 1, recv_all[i:i + m], rng.integers(0, 4, m).astype(np.uint8), t8[:m],
                         lens[:m], poff[:m], p[:m * L], ts[:m])
    shard.sync()
    total = shard.pending_tokens()
    lim = int(np.median(total)) // 4
    deep = {}
    for r in range(rounds):
        for fl in ((0, RECV_PRIORITY) if r % 2 == 0 else (RECV_PRIORITY, 0)):
            got, t = timed(shard, lambda: shard.receive_compact_tokens(None, D, lim, 0, fl | RECV_PEEK))
            t["records"] = len(got[1])
            # records the walk reads: the whole window (priority), or the steps up to the first one that does not fit
            k = got[0].astype(np.int64)
            read = n if fl else int(np.minimum(D, 32 * ((k + 32) // 32)).sum())
            t["bytes"] = 16 * A + (8 + 32 + 32) * read
            deep.setdefault("priority" if fl else "stream", []).append(t)
    shard.close()
    out["deep_config"] = (f"{A} agents x {D} pending tagged records ({L}-B payloads, counts 1..512), token limit {lim} "
                          f"(a quarter of the median window); PEEK compact receives, {reps} per block, orders alternated")
    out["deep"] = {k: {"blocks": v, **{f: float(np.median([x[f] for x in v])) for f in ("call_ms", "prepass_ms", "plan_ms")},
                       "records": v[-1]["records"]} for k, v in deep.items()}
    for k in out["deep"]:
        out["deep"][k].update(share(out["deep"][k]["prepass_ms"], out["deep"][k]["blocks"][-1]["bytes"]))
    out.update(_gpu_card(0))
    return out


def select(rounds=2, reps=10):
    """Filtered and leased receives by budget (sdb_receive_where_budget, sdb_receive_leased_select) on the c2 backlog
    (bench.py's step, 4,194,304 records over 1 M agents) with every send tagged (TYPEF_TOKENS, counts uniform in
    1..512) and a priority filter (levels 1-3):
      where / where_tokens   a filtered PEEK, without a limit and with 512 tokens per agent; wall time per call and the
                             take pass (recv_count) kernel time from the library profiler
      lease / lease_tokens   a leased take of every agent (2 messages each, and 512 tokens with the filter) plus the ack
                             of every lease it made; the backlog is sent again and drained between calls, untimed
    Legs alternate within each round.  Algorithmic bytes of the take pass: a 16-B ring header per agent, 8 B per ring
    entry and 4 B per 32 verdict bits, and per match one 32-B header sector and one 32-B payload sector per distinct
    send (the c2 windows fit one 32-entry step, which reads them all), over its kernel time, against the 3.35 TB/s of
    NVIDIA's H100 SXM data sheet."""
    import torch
    from bench import Workload
    from swarmdb_b200._native import LEASE_ACK, RECV_PEEK, Shard, make_filter
    if not torch.cuda.is_available():
        raise SystemExit("bench_extra.py select: no CUDA device - swarmdb_b200 has no CPU fallback")
    TOK, HBM = 0x40, 3.35e12
    wl = Workload()
    rng = np.random.default_rng(9)
    snd, grp, prio, typ, lens, off, pay = wl.batch()
    pay = pay.copy()
    pay.reshape(wl.S, wl.L)[:, :4] = rng.integers(1, 513, wl.S).astype(np.uint32).view(np.uint8).reshape(wl.S, 4)
    typ = np.full(wl.S, TOK, np.uint8)
    per_step = wl.S * wl.F
    rec_cap = per_step + (1 << 16)
    shard = Shard(max_agents=wl.A, ring_slots=64, arena_bytes=1 << 33, max_payload_bytes=wl.L, max_groups=1 << 14,
                  member_pool_entries=wl.A + 1024, max_batch_sends=wl.S, max_batch_payload=wl.S * wl.L,
                  max_recv_records=rec_cap, max_recv_payload=rec_cap * wl.L)
    shard.register(np.arange(wl.A, dtype=np.uint32))
    for g in range(wl.G):
        shard.create_group(g, wl.members(g))
    shard.lease_reserve(rec_cap, rec_cap * wl.L)
    filt = make_filter(prios=[1, 2, 3])

    def fill():
        shard.send_group_batch(snd, grp, prio, typ, lens, off, pay)
        shard.sync()

    def drain():
        while len(shard.receive_compact(None, 64)[1]):
            pass
        shard.lease_sweep(0.0)
        shard.sync()

    def peek(limit):
        fn = lambda: shard.receive_where(None, 100, RECV_PEEK, filt, max_agent_tokens=limit)   # noqa: E731
        fn()                                                                  # warm-up
        shard.sync()
        shard.profile(True)
        t = time.perf_counter()
        for _ in range(reps):
            r = fn()
        shard.sync()
        wall = (time.perf_counter() - t) * 1e3 / reps
        prof = shard.profile_read()
        shard.profile(False)
        return r, {"call_ms": wall, "take_ms": prof["recv_count"][0] / reps, "where_ms": prof["where"][0] / reps}

    def lease(tokens):
        kw = {"max_agent_tokens": 512, "filt": filt} if tokens else {}
        calls, recs = [], 0
        for i in range(reps + 1):                                             # the first is a warm-up
            drain()
            fill()
            t = time.perf_counter()
            cnt, ent, sends, p, base = shard.receive_leased(None, 2 if not tokens else 100, 1e18, 0, **kw)
            shard.lease_settle(np.arange(base, base + len(ent), dtype=np.uint64), LEASE_ACK)
            shard.sync()
            if i:
                calls.append((time.perf_counter() - t) * 1e3)
            recs = len(ent)
        drain()
        return recs, {"take_ack_ms": float(np.median(calls))}

    fill()
    res = {"where": [], "where_tokens": [], "lease": [], "lease_tokens": []}
    out_recs = {}
    for r in range(rounds):
        for name in (list(res) if r % 2 == 0 else list(res)[::-1]):
            if name.startswith("where"):
                got, t = peek(512 if name == "where_tokens" else 0)
                out_recs[name] = len(got[1])
                if name == "where_tokens":
                    k = got[0].astype(np.int64)
                    _, h, _ = shard.receive_where(None, 100, RECV_PEEK, filt)
                    matches = len(h)
                    t["bytes"] = 16 * wl.A + 8 * per_step + 4 * wl.A + 32 * matches + 32 * matches // wl.F
                    t["matches"], t["taken"] = matches, int(k.sum())
            else:
                out_recs[name], t = lease(name == "lease_tokens")
                fill()
            res[name].append(t)
    shard.close()
    out = {"config": (f"c2 backlog: {per_step} records over {wl.A} agents, {wl.L}-B payloads, every send tagged "
                      f"(counts 1..512), filter prios 1-3; token limit 512; {reps} calls per block, legs alternated")}
    for k, v in res.items():
        fields = [f for f in v[0] if f.endswith("_ms")]
        out[k] = {"blocks": v, **{f: float(np.median([x[f] for x in v])) for f in fields}, "records": out_recs[k]}
    tk = out["where_tokens"]
    nb = tk["blocks"][-1]["bytes"]
    tk.update({"algorithmic_bytes": nb, "take_tb_s": nb / (tk["take_ms"] * 1e-3) / 1e12 if tk["take_ms"] else None,
               "share_of_3_35_tb_s": nb / (tk["take_ms"] * 1e-3) / HBM if tk["take_ms"] else None})
    out.update(_gpu_card(0))
    return out


def dedup(rounds=2, batch=1 << 16, n=1 << 20, L=256):
    """Deduplicated sends (sdb_send_mixed_batch_dedup) against plain sdb_send_mixed_batch of the same batches.
    send: n point-to-point sends of L bytes (one per agent), in batches of `batch`, host clock to a synchronise, each
      mode alternated with a plain run: zero keys (the table is consulted by nobody: the probe and its one
      synchronisation alone), explicit keys without duplicates, content keys, and content keys where the second half
      of every batch repeats the first (half duplicates).
    kernels: from torch.profiler in a run of its own: the content-key kernel's payload bytes per second against the
      H100 SXM data sheet's 3.35 TB/s, and a rebuild of a table of n entries of which half have expired."""
    import torch
    from swarmdb_b200._native import Shard
    if not torch.cuda.is_available():
        raise SystemExit("bench_extra.py dedup: no CUDA device - swarmdb_b200 has no CPU fallback")
    A = n
    shard = Shard(max_agents=A, ring_slots=64, arena_bytes=1 << 33, max_payload_bytes=L, max_batch_sends=batch,
                  max_batch_payload=batch * L + 64)
    shard.register(np.arange(A, dtype=np.uint32))
    shard.dedup_reserve(4 * n, 1e9)
    rng = np.random.default_rng(9)
    pay = torch.empty(batch * L + 64, dtype=torch.uint8, pin_memory=True).numpy()
    pay[:] = rng.integers(0, 256, len(pay), dtype=np.uint8)
    half = pay.copy()
    half[batch // 2 * L: batch * L] = half[: batch // 2 * L]
    half_pin = torch.empty(len(half), dtype=torch.uint8, pin_memory=True).numpy()
    half_pin[:] = half
    off = np.arange(batch, dtype=np.uint64) * L
    lens, kind, z8, ts = np.full(batch, L, np.uint16), np.zeros(batch, np.uint8), np.zeros(batch, np.uint8), np.zeros(batch)
    lo = np.zeros(1, np.uint64)
    key_ctr = [1]

    def run(mode):
        shard.dedup_reserve(4 * n, 1e9)                               # a cleared table for every run
        ndup = 0
        shard.sync()
        t = time.perf_counter()
        for b in range(0, n, batch):
            recv = np.arange(b, b + batch, dtype=np.uint32)
            snd = recv ^ 1
            p = half_pin if mode == "content_half_dup" else pay
            if mode == "plain":
                shard.send_mixed_batch(snd, kind, recv, lo, None, z8, z8, lens, off, p, ts)
                continue
            keys = None
            if mode == "keys":
                k = np.arange(key_ctr[0], key_ctr[0] + batch, dtype=np.uint64)
                key_ctr[0] += batch
                keys = np.stack([k, k], 1)
            if mode == "content_half_dup":
                snd = snd.copy(); snd[batch // 2:] = snd[: batch // 2]
                recv = recv.copy(); recv[batch // 2:] = recv[: batch // 2]
            _, dup, _ = shard.send_mixed_batch_dedup(snd, kind, recv, lo, None, z8, z8, lens, off, p, ts, keys=keys,
                                                     content=mode.startswith("content"), now=1.0)
            ndup += int((dup != 0).sum())
        shard.sync()
        return time.perf_counter() - t, ndup

    modes = ("zero_keys", "keys", "content", "content_half_dup")
    res = {m: [] for m in modes}
    res["plain"] = []
    for r in range(rounds):
        for m in modes:
            for name in (("plain", m) if r % 2 == 0 else (m, "plain")):
                sec, ndup = run(name)
                res[name].append({"s": sec, "ns_per_send": sec * 1e9 / n, "duplicates": ndup})
        shard.receive_compact(None, 1 << 10, 0)          # keep the rings clear between rounds
    out = {"send_config": f"{n} point-to-point {L}-B sends in batches of {batch}, one per agent over {A} agents; "
                          f"{rounds} rounds, each mode alternated with plain",
           "send": {k: {"runs": v, "ns_per_send": float(np.median([x["ns_per_send"] for x in v]))} for k, v in res.items()}}
    shard.close()

    # ---- kernel times: the content-key kernel, and a rebuild with half of the entries expired
    from torch.profiler import ProfilerActivity, profile
    shard = Shard(max_agents=A, ring_slots=64, arena_bytes=1 << 33, max_payload_bytes=L, max_batch_sends=batch,
                  max_batch_payload=batch * L + 64)
    shard.register(np.arange(A, dtype=np.uint32))
    recv = np.arange(batch, dtype=np.uint32)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        shard.dedup_reserve(4 * n, 1e9)
        for _ in range(4):
            shard.send_mixed_batch_dedup(recv ^ 1, kind, recv, lo, None, z8, z8, lens, off, pay, ts, content=True, now=6.0)
            shard.receive_compact(None, 1 << 10, 0)
        shard.dedup_reserve(n, 10.0)
        for b in range(0, n, batch):                               # n keys: half at now = 0, half at now = 5
            k = np.arange(b + 1, b + batch + 1, dtype=np.uint64)
            shard.send_mixed_batch_dedup(recv ^ 1, kind, recv, lo, None, z8, z8, lens, off, pay, ts,
                                         keys=np.stack([k, k], 1), now=0.0 if b < n // 2 else 5.0)
            shard.receive_compact(None, 1 << 10, 0)
        # the table is full and half of it expired at now = 10: the next new keys rebuild it
        k = np.arange(n + 1, n + 1 + batch, dtype=np.uint64)
        shard.send_mixed_batch_dedup(recv ^ 1, kind, recv, lo, None, z8, z8, lens, off, pay, ts,
                                     keys=np.stack([k, k], 1), now=10.0)
        shard.sync()
    ds = shard.dedup_stats()
    shard.close()
    ev = {}
    for e in prof.key_averages():
        for name in ("k_dedup_content", "k_dedup_rebuild", "k_dedup_probe", "k_dedup_verdict", "k_dedup_insert"):
            if name in e.key:
                ev[name] = {"us_avg": e.device_time_total / max(e.count, 1), "count": e.count}
    hash_bytes = batch * L
    if "k_dedup_content" in ev:
        bps = hash_bytes / (ev["k_dedup_content"]["us_avg"] * 1e-6)
        ev["k_dedup_content"]["payload_bytes"] = hash_bytes
        ev["k_dedup_content"]["bytes_per_s"] = bps
        ev["k_dedup_content"]["share_of_3_35_TBps"] = bps / 3.35e12
    out["kernels"] = ev
    out["rebuild"] = {"table_entries": n, "expired_before": n // 2, "stats_after": ds}
    out.update(_gpu_card(0))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("which", nargs="*", default=["c1", "c4", "c5", "k1", "bcast"])
    args = ap.parse_args()
    for w in args.which:
        print(json.dumps({"bench": w, **globals()[w]()}), flush=True)


if __name__ == "__main__":
    main()
