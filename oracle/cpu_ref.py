"""ctypes wrapper over oracle/cpu_ref.c (ORACLE - TEST INFRASTRUCTURE ONLY).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
import this module.  `build()` compiles the C restatement with gcc into oracle/_build/.
"""
from __future__ import annotations

import ctypes as C
import subprocess
from pathlib import Path
from typing import Optional, Tuple

import numpy as np

_DIR = Path(__file__).resolve().parent
_SRC = _DIR / "cpu_ref.c"
_LIB = _DIR / "_build" / "liboracle.so"

HDR_DTYPE = np.dtype([("seq", "<u8"), ("timestamp", "<f8"), ("sender", "<u4"), ("receiver", "<u4"),
                      ("group", "<u4"), ("len", "<u2"), ("prio", "u1"), ("type", "u1")])
assert HDR_DTYPE.itemsize == 32


def build(force: bool = False) -> Path:
    if force or not _LIB.exists() or _LIB.stat().st_mtime < _SRC.stat().st_mtime:
        _LIB.parent.mkdir(exist_ok=True)
        subprocess.check_call(["gcc", "-O2", "-fPIC", "-shared", "-pthread", "-Wall", "-o", str(_LIB), str(_SRC)])
    return _LIB


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(str(build()))
        L = _lib
        vp, u32, u64 = C.c_void_p, C.c_uint32, C.c_uint64
        L.orc_create.restype = vp; L.orc_create.argtypes = [u32, u32]
        L.orc_destroy.argtypes = [vp]
        L.orc_register.argtypes = [vp, u32]
        L.orc_create_group.restype = C.c_int; L.orc_create_group.argtypes = [vp, u32, u32, vp]
        L.orc_create_group_pos.restype = C.c_int; L.orc_create_group_pos.argtypes = [vp, u32, u32, vp, vp]
        L.orc_set_next_seq.argtypes = [vp, u64]
        L.orc_get_next_seq.restype = u64; L.orc_get_next_seq.argtypes = [vp]
        L.orc_send_group_seq.argtypes = [vp, u32] + [vp] * 9
        L.orc_send_batch.restype = u64; L.orc_send_batch.argtypes = [vp, u32] + [vp] * 8
        L.orc_send_group_batch.restype = u64; L.orc_send_group_batch.argtypes = [vp, u32] + [vp] * 9
        L.orc_send_list_batch.restype = u64; L.orc_send_list_batch.argtypes = [vp, u32] + [vp] * 9
        L.orc_receive_batch.restype = u64; L.orc_receive_batch.argtypes = [vp, u32, vp, u32, u32, vp, vp, vp, vp]
        L.orc_pending.restype = u64; L.orc_pending.argtypes = [vp, u32]
        L.orc_set_backends.argtypes = [vp, u32, vp, vp]
        L.orc_get_backend_loads.argtypes = [vp, vp]
        L.orc_select_backend_batch.argtypes = [vp, u32, vp, u32, u64, vp]
        L.orc_log2_table.argtypes = [vp]
        L.orc_agent_loads.argtypes = [vp, u32, vp, vp]
        L.orc_digest_enable.argtypes = [vp]
        L.orc_digest_read.argtypes = [vp, u32, vp, vp]
        L.orc_mt_group_roundtrip.restype = u64
        L.orc_mt_group_roundtrip.argtypes = [vp, u32, u32] + [vp] * 7 + [u32, vp, vp]
    return _lib


def _p(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _arr(x, dt) -> np.ndarray:
    return np.ascontiguousarray(x, dtype=dt)


def log2_table() -> np.ndarray:
    """The 257-entry Q24 table of log2(1 + i/256) behind the weighted-random pick (mode 1)."""
    out = np.zeros(257, np.uint32)
    lib().orc_log2_table(_p(out))
    return out


class CpuOracle:
    """Index-level oracle with the same batch surface as swarmdb_b200._native.Shard."""

    def __init__(self, max_agents: int, max_groups: int = 1) -> None:
        self._h = lib().orc_create(max_agents, max_groups)
        self.max_agents = max_agents

    def close(self) -> None:
        if self._h:
            lib().orc_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def register(self, idx) -> None:
        for a in np.atleast_1d(idx):
            lib().orc_register(self._h, int(a))

    def create_group(self, g: int, members) -> None:
        m = _arr(members, np.uint32)
        assert lib().orc_create_group(self._h, g, len(m), _p(m)) == 0

    def create_group_pos(self, g: int, members, pos) -> None:
        m, p = _arr(members, np.uint32), _arr(pos, np.uint32)
        assert lib().orc_create_group_pos(self._h, g, len(m), _p(m), _p(p)) == 0

    @property
    def next_seq(self) -> int:
        return lib().orc_get_next_seq(self._h)

    @next_seq.setter
    def next_seq(self, v: int) -> None:
        lib().orc_set_next_seq(self._h, v)

    def send_group_seq(self, sender, group, prio, typ, lens, payload_off, payload, seq0, ts=None) -> None:
        s, g = _arr(sender, np.uint32), _arr(group, np.uint32)
        prio, typ, lens, po, pl, ts = self._common(len(s), prio, typ, lens, payload_off, payload, ts)
        q = _arr(seq0, np.uint64)
        lib().orc_send_group_seq(self._h, len(s), _p(s), _p(g), _p(prio), _p(typ), _p(lens), _p(po), _p(pl), _p(ts), _p(q))

    @staticmethod
    def _common(n, prio, typ, lens, payload_off, payload, ts):
        prio = _arr(prio if prio is not None else np.ones(n), np.uint8)
        typ = _arr(typ if typ is not None else np.zeros(n), np.uint8)
        lens = _arr(lens, np.uint16)
        payload_off = _arr(payload_off, np.uint64)
        payload = _arr(payload, np.uint8)
        ts = None if ts is None else _arr(ts, np.float64)
        return prio, typ, lens, payload_off, payload, ts

    def send_batch(self, sender, receiver, prio, typ, lens, payload_off, payload, ts=None) -> int:
        s, r = _arr(sender, np.uint32), _arr(receiver, np.uint32)
        prio, typ, lens, po, pl, ts = self._common(len(s), prio, typ, lens, payload_off, payload, ts)
        return lib().orc_send_batch(self._h, len(s), _p(s), _p(r), _p(prio), _p(typ), _p(lens), _p(po), _p(pl), _p(ts))

    def send_group_batch(self, sender, group, prio, typ, lens, payload_off, payload, ts=None) -> Tuple[int, int]:
        s, g = _arr(sender, np.uint32), _arr(group, np.uint32)
        prio, typ, lens, po, pl, ts = self._common(len(s), prio, typ, lens, payload_off, payload, ts)
        routed = C.c_uint64(0)
        base = lib().orc_send_group_batch(self._h, len(s), _p(s), _p(g), _p(prio), _p(typ), _p(lens), _p(po), _p(pl),
                                          _p(ts), C.cast(C.byref(routed), C.c_void_p))
        return base, routed.value

    def send_list_batch(self, sender, list_off, list_idx, prio, typ, lens, payload_off, payload, ts=None) -> int:
        s = _arr(sender, np.uint32)
        lo, li = _arr(list_off, np.uint64), _arr(list_idx, np.uint32)
        prio, typ, lens, po, pl, ts = self._common(len(s), prio, typ, lens, payload_off, payload, ts)
        return lib().orc_send_list_batch(self._h, len(s), _p(s), _p(lo), _p(li), _p(prio), _p(typ), _p(lens), _p(po),
                                         _p(pl), _p(ts))

    def receive_batch(self, agents, max_messages: int, flags: int = 0, rec_cap: int = 1 << 20, pay_cap: int = 1 << 28):
        if agents is None:
            n, a = 0, None
            counts = np.zeros(self.max_agents, np.uint32)
        else:
            a = _arr(agents, np.uint32)
            n = len(a)
            counts = np.zeros(n, np.uint32)
        hdr = np.zeros(rec_cap, HDR_DTYPE)
        pay = np.zeros(pay_cap, np.uint8)
        pb = C.c_uint64(0)
        total = lib().orc_receive_batch(self._h, n, _p(a), max_messages, flags, _p(counts), _p(hdr), _p(pay),
                                        C.cast(C.byref(pb), C.c_void_p))
        return counts, hdr[:total].copy(), pay[:pb.value].copy()

    def agent_loads(self, agents=None, n=None) -> np.ndarray:
        """Restatement of sdb_agent_loads: inbox size / unread count / priority histogram per agent."""
        dt = np.dtype([("received", "<u4"), ("pending", "<u4"), ("pending_by_prio", "<u4", (4,)), ("pending_granules", "<u4"),
                       ("reserved", "<u4")])
        if agents is None:
            a, cnt = None, int(n if n is not None else self.max_agents)
        else:
            a = _arr(agents, np.uint32)
            cnt = len(a)
        out = np.zeros(cnt, dt)
        lib().orc_agent_loads(self._h, cnt, _p(a), _p(out))
        return out

    def queue_stats(self, n=None) -> dict:
        ld = self.agent_loads(None, n)
        pend = ld["pending"].astype(np.int64)
        deepest = int(pend.max()) if len(pend) else 0
        return {"agents_with_pending": int((pend > 0).sum()), "pending": int(pend.sum()),
                "pending_by_prio": [int(x) for x in ld["pending_by_prio"].astype(np.int64).sum(axis=0)] if len(pend) else [0, 0, 0, 0],
                "pending_granules": int(ld["pending_granules"].astype(np.int64).sum()),
                "received": int(ld["received"].astype(np.int64).sum()), "max_pending": deepest,
                "max_pending_agent": int(np.argmax(pend)) if deepest else 0}

    def digest_enable(self) -> None:
        """Start (or restart from zero) folding every delivered record into per-agent stream digests."""
        lib().orc_digest_enable(self._h)

    def digest_read(self, agents=None) -> np.ndarray:
        if agents is None:
            n, a = self.max_agents, None
        else:
            a = _arr(agents, np.uint32)
            n = len(a)
        out = np.zeros(n, np.uint64)
        lib().orc_digest_read(self._h, n, _p(a), _p(out))
        return out

    def receive_counts(self, agents, max_messages: int, flags: int = 0) -> Tuple[np.ndarray, int]:
        """Receive without materialising the records (at-scale runs: digests carry the content)."""
        if agents is None:
            n, a = 0, None
            counts = np.zeros(self.max_agents, np.uint32)
        else:
            a = _arr(agents, np.uint32)
            n = len(a)
            counts = np.zeros(n, np.uint32)
        total = lib().orc_receive_batch(self._h, n, _p(a), max_messages, flags, _p(counts), None, None, None)
        return counts, int(total)

    def pending(self, a: int) -> int:
        return lib().orc_pending(self._h, a)

    def set_backends(self, weight, load0=None) -> None:
        w = _arr(weight, np.uint32)
        l0 = None if load0 is None else _arr(load0, np.uint64)
        lib().orc_set_backends(self._h, len(w), _p(w), _p(l0))
        self._nb = len(w)

    def backend_loads(self) -> np.ndarray:
        out = np.zeros(self._nb, np.uint64)
        lib().orc_get_backend_loads(self._h, _p(out))
        return out

    def select_backends(self, n_req: int, cost=None, mode: int = 0, seed: int = 0) -> np.ndarray:
        c = None if cost is None else _arr(cost, np.uint32)
        out = np.zeros(n_req, np.uint32)
        lib().orc_select_backend_batch(self._h, n_req, _p(c), mode, seed, _p(out))
        return out

    def mt_group_roundtrip(self, threads, sender, group, prio, typ, lens, payload_off, payload, max_messages=100):
        s, g = _arr(sender, np.uint32), _arr(group, np.uint32)
        prio, typ, lens, po, pl, _ = self._common(len(s), prio, typ, lens, payload_off, payload, None)
        drained, csum = C.c_uint64(0), C.c_uint64(0)
        routed = lib().orc_mt_group_roundtrip(self._h, threads, len(s), _p(s), _p(g), _p(prio), _p(typ), _p(lens), _p(po),
                                              _p(pl), max_messages, C.cast(C.byref(drained), C.c_void_p),
                                              C.cast(C.byref(csum), C.c_void_p))
        return routed, drained.value, csum.value
