"""Multi-GPU plumbing: one process per GPU, agents hash-partitioned across the shards.

Replaces the reference's partitioned Kafka topic (`_get_partition`, M:309-312: Python's salted
`hash(agent_id) % num_partitions`, different on every process start) with a deterministic
FNV-1a-64 hash, and the broker round trip with one NCCL all-gather of per-SEND wire batches over
NVLink (torch.distributed is only the transport; expansion into per-recipient records happens
in the sm_90a kernels of each shard - see csrc/sdb_xshard.cu).
"""
from __future__ import annotations

import dataclasses
from typing import Iterable, Optional

import numpy as np

from ._native import RECV_OWNED, SdbError
from .core import GpuConfig, MessagePriority, MessageStatus, MessageType, SwarmsDB

FNV_OFFSET = 0xCBF29CE484222325
FNV_PRIME = 0x100000001B3
_MASK = (1 << 64) - 1


def fnv1a64(data: bytes) -> int:
    h = FNV_OFFSET
    for b in data:
        h = ((h ^ b) * FNV_PRIME) & _MASK
    return h


def shard_of_agent(agent_id: str, num_shards: int) -> int:
    """Owner shard of an agent id (deterministic replacement of M:312)."""
    return fnv1a64(agent_id.encode("utf-8")) % num_shards


def shard_map_for_names(names: Iterable[str], num_shards: int) -> np.ndarray:
    return np.fromiter((shard_of_agent(n, num_shards) for n in names), dtype=np.uint8)


def shard_map_numbered(prefix: str, width: int, n: int, num_shards: int) -> np.ndarray:
    """Vectorised fnv1a64(f"{prefix}{i:0{width}d}") % num_shards for i in range(n) (bench workloads)."""
    h = np.full(n, FNV_OFFSET, dtype=np.uint64)
    prime = np.uint64(FNV_PRIME)
    with np.errstate(over="ignore"):
        for b in prefix.encode("utf-8"):
            h = (h ^ np.uint64(b)) * prime
        idx = np.arange(n, dtype=np.uint64)
        for k in range(width - 1, -1, -1):
            digit = (idx // np.uint64(10 ** k)) % np.uint64(10)
            h = (h ^ (digit + np.uint64(48))) * prime
    return (h % np.uint64(num_shards)).astype(np.uint8)


class ShardExchange:
    """Owns the wire buffers of one rank and moves them between ranks.

    `backend` abstracts where the bytes live: the CUDA implementation keeps them in torch CUDA
    tensors and all-gathers with NCCL; tests substitute a CPU backend (gloo) with the same calls.
    """

    def __init__(self, shard, rank: int, world: int, max_sends: int, max_payload: int, backend):
        self.shard, self.rank, self.world = shard, rank, world
        self.wire_bytes = shard.wire_bytes(max_sends, max_payload)
        self.backend = backend
        self.send_buf = backend.alloc(self.wire_bytes)
        self.recv_buf = backend.alloc(self.wire_bytes * world) if world > 1 else self.send_buf

    def export(self, sender, group, prio, typ, lens, payload_off, payload, ts=None) -> None:
        self.shard.export_group_batch(sender, group, prio, typ, lens, payload_off, payload,
                                      self.backend.ptr(self.send_buf), self.wire_bytes, ts)

    def export_mixed(self, sender, kind, target, list_off, list_idx, prio, typ, lens, payload_off, payload, ts=None,
                     seq_base: int = 0) -> None:
        """Mixed batch in call order: kind 0 = p2p (target receiver), 1 = group, 2 = broadcast list."""
        self.shard.export_mixed_batch(sender, kind, target, list_off, list_idx, prio, typ, lens, payload_off, payload,
                                      self.backend.ptr(self.send_buf), self.wire_bytes, ts, seq_base)

    def exchange(self) -> None:
        if self.world > 1:
            self.backend.all_gather(self.recv_buf, self.send_buf)

    def import_all(self) -> int:
        return self.shard.import_wire_batches(self.world, self.backend.ptr(self.recv_buf), self.wire_bytes)

    def step(self, sender, group, prio, typ, lens, payload_off, payload, ts=None) -> int:
        self.export(sender, group, prio, typ, lens, payload_off, payload, ts)
        self.exchange()
        return self.import_all()


class PeerExchange:
    """Peer-memory transport: no collective moves message bytes and none is used as a barrier.

    Every rank exports into its own CUDA-IPC-shared buffer (two of them, alternating per step) whose last 128 bytes
    hold two counters, `ready` and `done` (include/swarmdb_b200.h).  Ranks synchronise through those flags, on
    their streams, never on the host:
      export      waits until every peer has finished importing the step that used this buffer before (done >= step-2),
                  copies the wire batch, publishes ready = step
      import_all  the import's first kernel spins until every source's ready >= step (peer flags polled over NVLink),
                  then the import + fan-out kernels pull descriptors and payloads straight out of the exporting GPUs'
                  memory; afterwards done = step
      prefetch    optional, between an export and its import_all: the flag wait and the descriptor pull of the NEXT
                  step run on a second stream beside whatever is enqueued afterwards (the receive of the current
                  step); import_all then only places, fans out and indexes.  Pipelined producers call
                  export(k+1); prefetch(); receive(k); import_all().
    """

    def __init__(self, shard, rank: int, world: int, max_sends: int, max_payload: int, device, stream=None):
        import torch
        import torch.distributed as dist
        self.shard, self.rank, self.world = shard, rank, world
        # the shard's copies, kernels and flag updates all run on this one stream
        self.stream = stream if stream is not None else torch.cuda.Stream(device)
        shard.set_stream(self.stream.cuda_stream)
        self.wire_bytes = shard.wire_bytes(max_sends, max_payload)
        self.mine = [shard.wire_alloc(self.wire_bytes) for _ in range(2)]          # (ptr, ipc handle); zero-filled: ready = done = 0
        handles = [None] * world
        if world > 1:
            dist.all_gather_object(handles, [h for _, h in self.mine])
        self.ptrs = [[0] * world for _ in range(2)]
        self.opened = []
        for b in range(2):
            for r in range(world):
                if r == rank:
                    self.ptrs[b][r] = self.mine[b][0]
                else:
                    p = shard.wire_open(handles[r][b])
                    self.ptrs[b][r] = p
                    self.opened.append(p)
        self.step_no = 0                       # steps completed; the next one is step_no + 1 and uses buffer (step_no + 1) & 1
        self._published = 0                    # last step whose export this rank published
        self._prefetched = 0                   # last step handed to the shard's prefetch stream

    @property
    def next_step(self) -> int:
        return self.step_no + 1

    @property
    def cur(self) -> int:
        return self.next_step & 1

    def _begin_export(self) -> int:
        k = self.next_step
        if self._published >= k:
            raise RuntimeError(f"step {k} was already exported; import it before exporting again")
        if k > 2:                              # peers read this buffer during step k - 2: wait (on the stream) until they are done
            self.shard.wire_wait_done(self.ptrs[k & 1], self.wire_bytes, k - 2)
        return k

    def export(self, sender, group, prio, typ, lens, payload_off, payload, ts=None) -> None:
        k = self._begin_export()
        self.shard.export_group_batch(sender, group, prio, typ, lens, payload_off, payload,
                                      self.mine[k & 1][0], self.wire_bytes, ts)
        self.shard.wire_publish(self.mine[k & 1][0], self.wire_bytes, k)
        self._published = k

    def export_mixed(self, sender, kind, target, list_off, list_idx, prio, typ, lens, payload_off, payload, ts=None,
                     seq_base: int = 0) -> None:
        k = self._begin_export()
        self.shard.export_mixed_batch(sender, kind, target, list_off, list_idx, prio, typ, lens, payload_off, payload,
                                      self.mine[k & 1][0], self.wire_bytes, ts, seq_base)
        self.shard.wire_publish(self.mine[k & 1][0], self.wire_bytes, k)
        self._published = k

    def republish(self) -> None:
        """Benchmarks with device-resident inputs: the buffer of this parity already holds a wire batch (exported
        before the timed region); declare it ready for the next step without copying anything."""
        k = self.next_step
        if self._published >= k:
            return
        self.shard.wire_publish(self.mine[k & 1][0], self.wire_bytes, k)
        self._published = k

    def prefetch(self) -> None:
        """Start the next step's flag wait + descriptor pull on the shard's prefetch stream (this rank's own export of
        that step must be published already: every rank waits for every source, itself included)."""
        k = self.next_step
        if self._published < k:
            raise RuntimeError("prefetch before this rank exported the step")
        if self._prefetched < k:
            self.shard.import_prefetch(self.ptrs[k & 1], self.wire_bytes, k)
            self._prefetched = k

    def exchange(self) -> None:
        return None                            # nothing to do: import_all waits for the sources' flags on the device

    def import_all(self) -> None:
        k = self.next_step
        self.shard.import_wire_ptrs_async(self.ptrs[k & 1], self.wire_bytes, k)
        self.step_no = k

    def step(self, *batch, ts=None) -> None:
        self.export(*batch, ts=ts)
        self.import_all()

    def close(self) -> None:
        if not self.mine:
            return
        self.stream.synchronize()
        if self.world > 1:
            import torch.distributed as dist
            dist.barrier()                     # host-level: nobody is still reading this rank's buffers
        for p in self.opened:
            self.shard.wire_close(p, True)
        for p, _ in self.mine:
            self.shard.wire_close(p, False)
        self.opened, self.mine = [], []


class TorchCudaBackend:
    """Wire buffers in CUDA memory, exchanged with NCCL (torch.distributed) on ONE stream shared with the shard
    (pass the shard so its copies/kernels and the collective are ordered against each other)."""

    def __init__(self, device, shard=None, stream=None):
        import torch
        self.torch, self.device = torch, device
        self.stream = stream if stream is not None else torch.cuda.Stream(device)
        if shard is not None:
            shard.set_stream(self.stream.cuda_stream)

    def alloc(self, nbytes: int):
        with self.torch.cuda.stream(self.stream):          # zero-fill ordered before the first export into it
            return self.torch.zeros(nbytes, dtype=self.torch.uint8, device=self.device)

    def ptr(self, t) -> int:
        return t.data_ptr()

    def all_gather(self, out, inp) -> None:
        import torch.distributed as dist
        with self.torch.cuda.stream(self.stream):
            dist.all_gather_into_tensor(out, inp)


def run_sharded_bench(args, rank: int, world: int, local_rank: int, wl):
    """N-GPU arm of bench.py (torchrun, one rank per GPU): c3 = c2's workload with the 1M agents
    hash-sharded over the ranks; every rank ingests 65,536 group sends per step (weak scaling),
    all-gathers the wire batches over NVLink and drains the agents it owns."""
    import json
    import os
    import time

    import torch
    import torch.distributed as dist

    from ._native import HDR_DTYPE, RECV_OWNED, Shard

    dev = torch.device("cuda", local_rank)
    stream = torch.cuda.Stream()
    K, W = args.steps, args.warmup
    per_rank_msgs = wl.S * wl.F                     # routed messages each rank's sends produce
    recv_cap = per_rank_msgs * 2 + (1 << 16)        # a shard receives ~1/world of world x that, hash imbalance aside
    # every agent receives from the sends of ALL ranks: mean pending per step = world x 4.19, sized with headroom
    mean_pending = world * wl.S * wl.F / wl.A
    ring_slots = 64
    while ring_slots < 3 * mean_pending + 32:
        ring_slots *= 2
    ring_slots = int(os.environ.get("SDB_RING_SLOTS", ring_slots))
    shard = Shard(max_agents=wl.A, ring_slots=ring_slots, arena_bytes=1 << 33,
                  max_payload_bytes=wl.L, max_groups=1 << 14, member_pool_entries=wl.A + 1024, max_batch_sends=wl.S,
                  max_batch_payload=wl.S * wl.L, max_recv_records=recv_cap, max_recv_payload=recv_cap * wl.L,
                  device=local_rank, shard_id=rank, num_shards=world, fanout_variant=args.variant)
    shard.set_stream(stream.cuda_stream)
    smap = shard_map_numbered("agent_", 7, wl.A, world)
    shard.set_agent_shards(smap)
    local_agents = np.nonzero(smap == rank)[0].astype(np.uint32)
    shard.register(local_agents)
    for g in range(wl.G):
        shard.create_group(g, wl.members(g))
    shard.sync()
    transport = os.environ.get("SDB_XSHARD", "peer")
    with torch.cuda.stream(stream):
        if transport == "peer":
            ex = PeerExchange(shard, rank, world, wl.S, wl.S * wl.L, dev, stream=stream)
        else:
            ex = ShardExchange(shard, rank, world, wl.S, wl.S * wl.L, TorchCudaBackend(dev, shard, stream))
        # each rank draws its own slice of the global batch: advance the generators by rank
        for _ in range(rank):
            wl.batch()
        n_distinct = 2
        batches = []
        for _ in range(n_distinct):
            batches.append(wl.batch())
            for _ in range(world - 1):
                wl.batch()
        # device-resident inputs: wire batches exported once, before the timed region
        wires = []
        if transport == "peer":
            for k, b in enumerate(batches):                 # batch k lives in this rank's export buffer k (no flags yet)
                shard.export_group_batch(*b, ex.mine[k][0], ex.wire_bytes)
            torch.cuda.synchronize(); dist.barrier()
        else:
            for b in batches:
                ex.export(*b)
                torch.cuda.synchronize()
                wires.append(ex.send_buf.clone())

        phase_ev = []
        # cross-step pipelining (peer transport): while step k's receive runs, the flag wait and the descriptor pull of
        # step k + 1 run on the shard's prefetch stream (PeerExchange.prefetch)
        pipelined = transport == "peer" and world > 1 and os.environ.get("SDB_PIPELINE", "1") != "0"

        def device_step(i, timed=False, start_next=True):
            evs = [torch.cuda.Event(enable_timing=True) for _ in range(5)] if timed else None
            if timed:
                evs[0].record(stream)
            if transport != "peer":
                ex.send_buf.copy_(wires[i % n_distinct], non_blocking=True)   # HBM -> HBM staging of this step's input
            if timed:
                evs[1].record(stream)
            if transport == "peer":
                ex.republish()                              # this step's (pre-exported) wire batch is ready: flag only
            else:
                ex.exchange()
            if timed:
                evs[2].record(stream)
            ex.import_all()
            if pipelined and start_next:
                ex.republish()                              # the next step's pre-exported wire batch: flag only
                ex.prefetch()
            if timed:
                evs[3].record(stream)
            # SDB_RECV_OWNED: the device-resident list of the agents this shard owns (no index upload, 1/world of the slots)
            shard.receive_batch(None, 100, RECV_OWNED, copy_out=False, wait=False)    # enqueued only: counted on the device
            if timed:
                evs[4].record(stream)
                phase_ev.append(evs)

        for i in range(W):
            device_step(i)
        st0 = shard.stats()
        launches0 = st0["kernel_launches"]
        shard.profile(True)
        from bench import ALG_BYTES_FANOUT, ClockSampler, hbm_peak, parity_report, traffic_note, workload_c3
        clocks = ClockSampler(local_rank); clocks.start()
        dist.barrier(); torch.cuda.synchronize()
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record(stream)
        for i in range(K):
            device_step(W + i, timed=True)
        ev1.record(stream)
        torch.cuda.synchronize(); dist.barrier()
        clk = clocks.stop()
        ms = ev0.elapsed_time(ev1)
        prof = shard.profile_read(); shard.profile(False)
        names = ["stage_input", "exchange", "import", "receive"]
        phases = {n: float(np.mean([e[k].elapsed_time(e[k + 1]) for e in phase_ev])) for k, n in enumerate(names)}
        st_end = shard.stats()
        launches = st_end["kernel_launches"] - launches0
        delivered = st_end["delivered"] - st0["delivered"]
        assert st_end["ring_overflow"] == 0, f"ring overflow on rank {rank}: {st_end['ring_overflow']} records (ring_slots={ring_slots})"
        sustained = None
        Ks = int(getattr(args, "sustained_steps", 0) or 0)
        if Ks > 0:                                          # the same step for a few hundred milliseconds, timed as one block
            clocks_s = ClockSampler(local_rank); clocks_s.start()
            dist.barrier(); torch.cuda.synchronize()
            ev0.record(stream)
            for i in range(Ks):
                device_step(W + K + i)
            ev1.record(stream)
            torch.cuda.synchronize(); dist.barrier()
            sustained = {"steps": Ks, "ms": ev0.elapsed_time(ev1), "clocks": clocks_s.stop()}
            assert shard.stats()["ring_overflow"] == 0
        if pipelined:                                       # the step prefetched by the last timed one: import it, start no other
            device_step(W + K + Ks, start_next=False)
            torch.cuda.synchronize()

        # ---- e2e: host buffers in (export H2D), results out (D2H into pinned buffers)
        pin_hdr = torch.empty(recv_cap * 32, dtype=torch.uint8, pin_memory=True).numpy().view(HDR_DTYPE)
        pin_pay = torch.empty(recv_cap * wl.L, dtype=torch.uint8, pin_memory=True).numpy()
        pinned = []
        for b in batches:
            t = torch.empty(b[6].nbytes, dtype=torch.uint8, pin_memory=True); t.numpy()[:] = b[6]
            pinned.append(b[:6] + (t.numpy(),))
        Ke = max(1, min(K, 8))

        def e2e_step(i):
            ex.step(*pinned[i % n_distinct])
            _, hdr, _ = shard.receive_batch(None, 100, RECV_OWNED, copy_out=True, out_hdr=pin_hdr, out_payload=pin_pay)
            return len(hdr)

        e2e_step(0); e2e_step(1)
        dist.barrier(); torch.cuda.synchronize()
        t0 = time.perf_counter()
        got = 0
        for i in range(Ke):
            got += e2e_step(i)
        torch.cuda.synchronize(); dist.barrier()
        e2e_ms = (time.perf_counter() - t0) * 1e3

        # ---- content parity on the real transport (outside every timed region): two verified steps with a FRESH
        # export each (both export buffers in use), every shard digests the streams of the agents it owns on the
        # device, rank 0 compares the union with ONE oracle queue fed all ranks' batches in (step, rank) order
        while shard.receive_batch(None, 100, 0, copy_out=False)[1]:
            pass
        shard.digest_reset()
        seq_base = shard.stats()["next_seq"]
        p_delivered = 0
        for step in range(wl.PARITY_STEPS):
            ex.step(*wl.parity_batch(step, rank))
            _, tt, _ = shard.receive_batch(None, 100, RECV_OWNED if step % 2 == 0 else 0, copy_out=False)
            shard.digest_fold()
            p_delivered += tt
        while True:
            _, tt, _ = shard.receive_batch(None, 100, 0, copy_out=False)
            shard.digest_fold()
            if tt == 0:
                break
            p_delivered += tt
        dg = shard.digest_read()
        foreign_ok = not dg[smap != rank].any()
        dsum = torch.from_numpy(dg.view(np.int64).copy()).to(dev)
        dist.all_reduce(dsum)                                # owners are disjoint: the sum is the union
        pstat = torch.tensor([p_delivered, 0 if foreign_ok else 1, seq_base], dtype=torch.int64, device=dev)
        pmax = pstat.clone(); dist.all_reduce(pmax, op=dist.ReduceOp.MAX)
        dist.all_reduce(pstat)

    t = torch.tensor([ms, float(delivered), e2e_ms, float(got), float(launches), sustained["ms"] if sustained else 0.0],
                     dtype=torch.float64, device=dev)
    mx = t.clone(); dist.all_reduce(mx, op=dist.ReduceOp.MAX)
    sm = t.clone(); dist.all_reduce(sm, op=dist.ReduceOp.SUM)
    if rank == 0:
        ms_max, e2e_max = float(mx[0]), float(mx[2])
        total_delivered, total_got = float(sm[1]), float(sm[3])
        assert int(total_delivered) == K * per_rank_msgs * world, (total_delivered, K * per_rank_msgs * world)
        parity = parity_report(dsum.cpu().numpy().view(np.uint64), int(pstat[0]), wl, world, seq_base,
                               f"{transport} transport, fresh export per step, {world} GPUs")
        if int(pstat[1]) or int(pmax[2]) * world != int(pstat[2]):
            parity["match"] = False
            parity["note"] = "a shard delivered to agents it does not own, or sequence bases diverged across ranks"
        peak, peak_src = hbm_peak()
        from bench import ALG_BYTES_GATHER, ALG_OWN_GATHER
        from ._native import shared_payload_enabled
        gat_ms, gat_n = prof.get("recv_gather", (0.0, 0))
        gat_avg = gat_ms / max(gat_n, 1)
        local_msgs = delivered / K
        achieved = ALG_BYTES_GATHER * local_msgs / (gat_avg * 1e-3) / 1e9 if gat_n else 0.0
        step_alg = (ALG_BYTES_FANOUT + 1 + ALG_BYTES_GATHER) * local_msgs
        line = {
            "metric": "messages/sec routed (send->receive) at 1M agents, 64-way fanout",
            "value": total_delivered / (ms_max * 1e-3), "unit": "messages/s", "n_gpus": world, "steps": K, "warmup": W,
            "ms_per_step": ms_max / K, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "u8", "data": "synthetic",
            "config": {"workload": workload_c3(world),
                       "transport": transport,
                       "transport_detail": ("peer memory: import/fan-out kernels pull descriptors and payloads from the "
                                            "exporting GPUs over NVLink" if transport == "peer"
                                            else "wire batches all-gathered over NCCL/NVLink"),
                       "timed_region": "flag wait + import (localize, fan-out, index) + receive; the wire batches "
                                       "are exported to HBM before the timed region (device-resident inputs, like N=1's "
                                       "staged batches); the export (host descriptor build + H2D) is inside `e2e` only",
                       "pipelined": ("the flag wait + descriptor pull of step k+1 run on a second stream beside step k's receive "
                                     "(sdb_import_prefetch); every step still does all of its work inside the timed region"
                                     if pipelined else False),
                       "l2": "inputs larger than L2 (each shard writes and reads back ~1.2 GB of records per step)",
                       "parallelism": f"shard{world}", "ring_slots": ring_slots},
            "clocks": clk,
            "sustained": ({"steps": Ks, "ms_per_step": float(mx[5]) / Ks, "unit": "messages/s",
                           "value": Ks * per_rank_msgs * world / (float(mx[5]) * 1e-3), "clocks": sustained["clocks"]}
                          if sustained else None),
            "e2e": {"value": total_got / (e2e_max * 1e-3), "unit": "messages/s",
                    "h2d_bytes_per_step": (wl.S * wl.L + wl.S * 64) * world,
                    "d2h_bytes_per_step": int(total_got / Ke * (32 + wl.L)) + wl.A * 4, "steps": Ke,
                    "ms_per_step": e2e_max / Ke},
            "gpu_launches": int(float(sm[4])),
            "roofline": {"kernel": "k_recv_gather_tma (dominant: %.0f %% of rank 0's step)" % (100 * gat_avg / (ms_max / K)),
                         "bound": "hbm", "achieved": achieved, "peak": peak, "unit": "GB/s",
                         "frac": achieved / peak, "traffic": traffic_note("k_recv_gather_bytes_per_launch"), "peak_source": peak_src,
                         "algorithmic_bytes_per_msg": ALG_BYTES_GATHER, "msgs_per_launch": local_msgs,
                         "ms_per_launch": gat_avg, "step_frac": step_alg / ((ms_max / K) * 1e-3) / 1e9 / peak,
                         "note": "rank 0's shard (the traffic figure is the N=1 capture); SURVEY 8(d) bytes per message, see the N=1 "
                                 "line's roofline.own_layout for the shared-payload accounting",
                         "own_layout_gather_frac": (ALG_OWN_GATHER * local_msgs / (gat_avg * 1e-3) / 1e9 / peak
                                                    if (gat_n and shared_payload_enabled()) else None)},
            "kernels": {k: {"ms_per_launch": v[0] / v[1], "launches": v[1]} for k, v in prof.items() if v[1]},
            "phases_ms_rank0": phases,
            "parity": parity,
            "cpu_baseline": None,
        }
        print(json.dumps(line), flush=True)
    if transport == "peer":
        torch.cuda.synchronize(); dist.barrier()
        ex.close()
    shard.close()
    dist.destroy_process_group()


# ------------------------------------------------------------------------------------------------
# SPMD front-end over the sharded queue: the SwarmsDB surface, one process per GPU
# ------------------------------------------------------------------------------------------------
def composite_seq(round_no: int, rank: int, local: int = 0) -> int:
    """Sequence number a rank can assign on its own at send time: (round, rank, local) order is exactly
    the import order of the wire batches (rank-major inside one collective flush)."""
    return (round_no << 40) | (rank << 32) | local


class ShardedSwarmsDB(SwarmsDB):
    """The reference's surface for a multi-GPU deployment (one process per GPU, like the reference's
    independent gunicorn workers, api.py:66, but sharing ONE queue):

      * registry and group calls (`register_agent(s)`, `deregister_agent`, `add_agent_group`) are
        REPLICATED - every rank makes them identically and in the same order (agent indices must agree);
      * `send_message` / `send_to_group` / `broadcast_message` are LOCAL - each rank ingests its own
        traffic and returns message ids immediately (composite sequence numbers);
      * `flush()` is COLLECTIVE - every rank calls it; wire batches are exchanged and imported;
      * `receive_messages(agent)` is LOCAL to the rank that owns the agent
        (`shard_of_agent(agent_id, world)`), and returns what earlier flushes delivered;
      * device lookups by id (`get_message` / `get_messages` / `delete_message(s)` with include_device=True,
        `receive_matching(..., message_ids=)`) are LOCAL, with no collective: each rank reads the queues of the agents
        it owns, so a message queued for an agent of another rank is found (or deleted) on that rank.
    """

    def __init__(self, rank: int, world: int, *a, exchange_factory=None, shard=None, **k):
        g = k.get("gpu_config") or GpuConfig()
        if g.id_nonce is None and not g.deterministic_ids:
            g = dataclasses.replace(g, deterministic_ids=True)       # ids must agree across ranks
        g = dataclasses.replace(g, shard_id=rank, num_shards=world)
        if g.lease_records or g.lease_max_deliveries:
            self._no_leases()
        if g.dedup_entries:
            self._no_dedup()
        if g.arena_relocate:
            raise NotImplementedError("ShardedSwarmsDB does not retry refused flushes (GpuConfig.arena_relocate): an "
                                      "asynchronous import that does not fit is dropped whole; call relocate_pinned instead")
        k["gpu_config"] = g
        super().__init__(*a, _shard=shard, **k)
        self.rank, self.world = rank, world
        self._round = 1
        self._next_seq = self._b_first_seq = composite_seq(1, rank)
        self._map_dirty = True
        self._replicated = 0
        self._seen_overflow = 0
        self._round_msgs = []
        g2 = self.gpu_config
        self.exchange = (exchange_factory or self._default_exchange)(self.shard, rank, world, max(g2.flush_threshold, 1),
                                                                      max(1 << 22, 2 * (g2.max_payload_bytes + 31)))

    def _default_exchange(self, shard_, rank_, world_, max_sends, max_payload):
        import torch
        dev = torch.device("cuda", self.gpu_config.device)      # the shard's device, not whatever is current
        torch.cuda.set_device(dev)
        return PeerExchange(shard_, rank_, world_, max_sends, max_payload, dev)

    def owner(self, agent_id: str) -> int:
        return shard_of_agent(agent_id, self.world)

    # ---- replicated calls: the only place where new agent indices may be created
    def _index(self, agent_id: str) -> int:
        i = self._agent_idx.get(agent_id)
        if i is None:
            if not self._replicated:
                raise KeyError(f"agent {agent_id!r} is unknown on rank {self.rank}: in a sharded deployment agents are "
                               f"introduced by register_agent(s) / add_agent_group, called identically on every rank")
            i = super()._index(agent_id)
            self._map_dirty = True
        return i

    def register_agent(self, agent_id: str) -> None:
        self._replicated += 1
        try:
            super().register_agent(agent_id)
        finally:
            self._replicated -= 1

    def register_agents(self, agent_ids):
        self._replicated += 1
        try:
            return super().register_agents(list(agent_ids))
        finally:
            self._replicated -= 1

    def add_agent_group(self, group_name: str, agent_ids) -> None:
        self._replicated += 1
        try:
            self._push_shard_map()
            super().add_agent_group(group_name, agent_ids)
        finally:
            self._replicated -= 1

    create_group = add_agent_group

    def _push_shard_map(self) -> None:
        if self._map_dirty and self._agent_name:
            self.shard.set_agent_shards(shard_map_for_names(self._agent_name, self.world))
            self._map_dirty = False

    def _sync_group(self, group_name: str) -> int:
        self._push_shard_map()              # ownership must be known before the group is filtered
        return super()._sync_group(group_name)

    # ---- local sends: every agent they name must already be known everywhere
    def _require_known(self, *agent_ids) -> None:
        for a in agent_ids:
            if a is not None and a not in self._agent_idx:
                raise KeyError(f"agent {a!r} must be registered (on every rank) before it is used in a send")

    def send_message(self, sender_id, content, receiver_id=None, message_type=None, priority=None, metadata=None,
                     visible_to=None, **kw):
        if kw.get("dedup_id") is not None:
            self._no_dedup()
        if kw.get("supersede"):
            self._no_supersede()
        self._require_known(sender_id, receiver_id, *(visible_to or []))
        return super().send_message(sender_id, content, receiver_id, message_type or MessageType.CHAT,
                                    priority if priority is not None else MessagePriority.NORMAL, metadata, visible_to, **kw)

    def broadcast_message(self, sender_id, content, *a, dedup_id=None, supersede=False, **kw):
        if dedup_id is not None:
            self._no_dedup()
        if supersede:
            self._no_supersede()
        return super().broadcast_message(sender_id, content, *a, **kw)

    def send_to_group(self, sender_id, group_name, content, message_type=None, priority=None, metadata=None,
                      dedup_id=None, supersede=False):
        if dedup_id is not None:
            self._no_dedup()
        if supersede:
            self._no_supersede()
        self._require_known(sender_id)
        return super().send_to_group(sender_id, group_name, content, message_type or MessageType.CHAT,
                                     priority if priority is not None else MessagePriority.NORMAL, metadata)

    # ---- collective flush: export (local) -> exchange (collective) -> import (local)
    def flush(self) -> None:
        try:
            self._flush_export()
            self.exchange.exchange()
        except Exception as e:
            self._fail_round(e)
            raise
        self._flush_import()
        self._apply_queue_caps()                 # on the agents this rank owns (RECV_OWNED): no collective
        self.sync_llm_backends()

    # ---- one balancer for all shards (SURVEY 8e): every rank picks from its own copy of the table; the per-backend
    # load changes each rank made since the last flush are summed across ranks (256 values) and applied everywhere
    def register_llm_backends(self, backend_ids, weights=None, loads=None) -> None:
        """REPLICATED (every rank, identically)."""
        super().register_llm_backends(backend_ids, weights, loads)
        self._be_weights = np.asarray(weights if weights is not None else [1] * len(backend_ids), np.uint32)
        self._be_synced = np.asarray(loads if loads is not None else [0] * len(backend_ids), np.int64).copy()

    def _all_reduce_i64(self, x: np.ndarray) -> np.ndarray:
        import torch
        import torch.distributed as dist
        if self.world == 1 or not dist.is_initialized():
            return x
        dev = torch.device("cuda", self.gpu_config.device) if dist.get_backend() == "nccl" else torch.device("cpu")
        t = torch.from_numpy(np.ascontiguousarray(x, np.int64)).to(dev)
        dist.all_reduce(t)
        return t.cpu().numpy()

    def sync_llm_backends(self) -> None:
        """COLLECTIVE (part of flush): after it every rank's table holds base + the sum of all ranks' changes."""
        if not getattr(self, "_backend_name", None) or not hasattr(self, "_be_synced"):
            return
        local = self.shard.backend_loads().astype(np.int64)
        total = self._be_synced + self._all_reduce_i64(local - self._be_synced)
        total = np.maximum(total, 0)
        self.shard.set_backends(self._be_weights, total.astype(np.uint64))
        self._be_synced = total

    def refresh_llm_backend_loads(self):
        """COLLECTIVE: backlog of the agents assigned to each backend, summed over the shards that own them."""
        self.shard.backend_loads_from_queues()
        total = self._all_reduce_i64(self.shard.backend_loads().astype(np.int64))
        self.shard.set_backends(self._be_weights, total.astype(np.uint64))
        self._be_synced = total
        return self.llm_backend_loads()

    def _fail_round(self, e: Exception) -> None:
        for m in self._round_msgs:
            m.status = MessageStatus.FAILED
            m.metadata["error"] = str(e)
        self._round_msgs = []

    def _flush_export(self) -> None:
        self._push_shard_map()
        self._round_msgs = self._b_msgs
        try:
            payload = np.frombuffer(bytes(self._b_payload) + bytes(32), dtype=np.uint8)
            self.exchange.export_mixed(
                np.asarray(self._b_sender, np.uint32), np.asarray(self._b_kind, np.uint8),
                np.asarray(self._b_target, np.uint32), np.asarray(self._b_list_off, np.uint64),
                np.asarray(self._b_list_idx, np.uint32), np.asarray(self._b_prio, np.uint8),
                np.asarray(self._b_type, np.uint8), np.asarray(self._b_len, np.uint16),
                np.asarray(self._b_off, np.uint64), payload, np.asarray(self._b_ts, np.float64),
                seq_base=composite_seq(self._round, self.rank))
        finally:
            self._round += 1
            self._next_seq = composite_seq(self._round, self.rank)
            self._reset_buffer()

    def _flush_import(self) -> None:
        try:
            self.exchange.import_all()
            lost = self.shard.stats()["ring_overflow"] - self._seen_overflow
            if lost > 0:
                self._seen_overflow += lost
                raise SdbError(-4, f"{lost} message(s) not enqueued on shard {self.rank}: a receiver's ring is full "
                                   f"(GpuConfig.ring_slots={self.gpu_config.ring_slots})")
        except Exception as e:
            self._fail_round(e)
            raise
        self._round_msgs = []

    def _after_send(self) -> None:
        # no automatic flush: it is a collective; the caller decides when every rank flushes
        if len(self._b_sender) >= self.gpu_config.flush_threshold:
            raise RuntimeError("send buffer full: call flush() (collectively) more often or raise flush_threshold")

    # ---- local receive on the owner
    def receive_messages(self, agent_id: str, max_messages: int = 100, timeout: float = 1.0, max_bytes: Optional[int] = None,
                         max_tokens: Optional[int] = None):
        if self.owner(agent_id) != self.rank:
            raise ValueError(f"agent {agent_id!r} lives on shard {self.owner(agent_id)}, not on rank {self.rank}")
        if agent_id not in self._agent_idx:
            return []
        return self._receive_local(agent_id, max_messages, max_bytes, max_tokens)

    def _prepare_receive(self, agent_id: str) -> bool:
        """receive_matching runs on the owner rank, locally (no collective), like receive_messages."""
        if self.owner(agent_id) != self.rank:
            raise ValueError(f"agent {agent_id!r} lives on shard {self.owner(agent_id)}, not on rank {self.rank}")
        return agent_id in self._agent_idx

    def _pre_read(self) -> None:
        return None                              # reads see what earlier collective flushes delivered

    def peek_messages(self, agent_id: str, max_messages: int = 100, max_bytes: Optional[int] = None,
                      max_tokens: Optional[int] = None):
        if self.owner(agent_id) != self.rank:
            raise ValueError(f"agent {agent_id!r} lives on shard {self.owner(agent_id)}, not on rank {self.rank}")
        if agent_id not in self._agent_idx:
            return []
        return super().peek_messages(agent_id, max_messages, max_bytes, max_tokens)

    def deregister_agent(self, agent_id: str, purge: bool = False) -> None:
        """REPLICATED, like register_agent (the registry must agree on every rank); purge=True drops the agent's
        queued messages on the rank that owns it (the other ranks hold none)."""
        super().deregister_agent(agent_id, purge)

    # ---- retention is LOCAL: each rank expires (and archives) what its own agents hold, no collective
    def _expire_scope(self, agent_ids):
        self._push_shard_map()
        if agent_ids is None:
            return None, RECV_OWNED
        return super()._expire_scope([a for a in agent_ids if self.owner(a) == self.rank])

    # ---- queue snapshots and requeue: a sharded deployment needs per-rank files, owned-agent restores and the composite
    # round moved past the restored ids; until that exists these refuse instead of restoring every agent on every rank
    def save_queue_snapshot(self, path):
        raise NotImplementedError("ShardedSwarmsDB does not write queue snapshots yet; a rank can restore its share of a "
                                  "single-shard snapshot with Shard.restore_compact(..., RECV_OWNED)")

    def load_queue_snapshot(self, path):
        raise NotImplementedError("ShardedSwarmsDB does not load queue snapshots yet (see save_queue_snapshot)")

    def requeue_batch_compact(self, counts, entries, sends, payload, agent_idx):
        raise NotImplementedError("ShardedSwarmsDB does not requeue yet: restored ids must stay below the composite "
                                  "sequence numbers of later rounds")

    # ---- leased receives redeliver with the original ids, which meets the composite-round numbering as requeue does
    def _no_dedup(self):
        raise NotImplementedError("ShardedSwarmsDB does not deduplicate sends yet (GpuConfig.dedup_entries, dedup_id): "
                                  "a key must be checked on the rank that numbers the send, before the exchange")

    def _no_supersede(self, *args, **kwargs):
        raise NotImplementedError("ShardedSwarmsDB does not supersede sends yet (supersede=True, supersede_pending): a "
                                  "rank does not know which agents other ranks' superseding sends reached, and host "
                                  "records live on the sending rank")

    supersede_pending = _no_supersede

    def _no_leases(self, *args, **kwargs):
        raise NotImplementedError("ShardedSwarmsDB does not lease yet: redelivered ids must stay below the composite "
                                  "sequence numbers of later rounds (see requeue_batch_compact)")

    receive_messages_leased = receive_batch_leased = settle_leases = _no_leases

    def receive_matching(self, agent_id: str, max_messages: int = 100, *, leased: bool = False, **kw):
        """SwarmsDB.receive_matching on the owner rank; leased=True is refused like every lease call."""
        if leased:
            self._no_leases()
        return super().receive_matching(agent_id, max_messages, **kw)
    ack_messages = nack_messages = extend_leases = redeliver_expired = _no_leases
    dead_letters = redrive_dead_letters = _no_leases

    def close(self) -> None:
        """Collective like flush(): every rank closes.  Buffered sends are NOT flushed here (a flush is a collective
        the caller schedules); the exchange's buffers are released only after their last reader is done."""
        if self._closed:
            return
        try:
            if self.auto_save:
                self.save_message_history()
        finally:
            try:
                if hasattr(self.exchange, "close"):
                    self.exchange.close()
            finally:
                self.shard.close()
                self._closed = True


def make_sharded_swarmsdb(rank: int, world: int, exchange_factory=None, shard=None, **kw) -> ShardedSwarmsDB:
    """Factory kept for callers that pass everything by keyword: `ShardedSwarmsDB(rank, world, ...)`."""
    return ShardedSwarmsDB(rank, world, exchange_factory=exchange_factory, shard=shard, **kw)
