"""The input contract of the five receive-family calls of the C ABI, table-driven.

sdb_receive_batch, sdb_receive_compact, sdb_expire, sdb_receive_where and sdb_restore_compact each check their
arguments in their own order.  Every row below is one call through the raw ABI with its expected return code.  For a
refusal the test checks that the call's scalar outputs read as the header says after a refusal (0; restore's
seq_end_out the next sequence number), that stats() and agent_loads() did not move, and that a following normal
receive still equals the CPU oracle.  Rows with SDB_OK pin the calls that accept a request with nothing to do before
they look at the output buffers.
"""
import ctypes as C

import numpy as np
import pytest

from tests.test_gpu_shared_layout import _payloads

pytestmark = pytest.mark.gpu

OK, EINVAL, ECAPACITY, EOUTPUT = 0, -1, -6, -8
A, L, REC_CAP = 256, 256, 64          # max_recv_records = 64 and room for 64 maximum-size payloads
SENTINEL = 0xDEADBEEF


class Outs:
    """Sentinel-filled scalar outputs and host buffers of one call."""

    def __init__(self, n=A):
        from swarmdb_b200._native import ENTRY_DTYPE, HDR_DTYPE, SEND_DTYPE
        self.total, self.n_sends, self.pbytes = C.c_uint64(SENTINEL), C.c_uint64(SENTINEL), C.c_uint64(SENTINEL)
        self.restored, self.seq_end = C.c_uint64(SENTINEL), C.c_uint64(SENTINEL)
        self.counts = np.zeros(n, np.uint32)
        self.hdr = np.zeros(REC_CAP, HDR_DTYPE)
        self.ent, self.snd = np.zeros(REC_CAP, ENTRY_DTYPE), np.zeros(REC_CAP, SEND_DTYPE)
        self.pay = np.zeros(REC_CAP * L, np.uint8)

    @staticmethod
    def ref(x):
        return C.cast(C.byref(x), C.c_void_p)


def _batch(g, o, agents, mx=4, flags=0, hdr_cap=REC_CAP, pay_cap=REC_CAP * L, n=None):
    from swarmdb_b200._native import _p
    a = None if agents is None else np.asarray(agents, np.uint32)
    n = (0 if a is None else len(a)) if n is None else n
    rc = g._L.sdb_receive_batch(g._h, n, _p(a), mx, flags, _p(o.counts), _p(o.hdr), hdr_cap, _p(o.pay), pay_cap,
                                o.ref(o.total), o.ref(o.pbytes))
    return rc, ("total", "pbytes")


def _compact(g, o, agents, mx=4, flags=0, ent_cap=REC_CAP, snd_cap=REC_CAP, pay_cap=REC_CAP * L):
    from swarmdb_b200._native import _p
    a = None if agents is None else np.asarray(agents, np.uint32)
    rc = g._L.sdb_receive_compact(g._h, 0 if a is None else len(a), _p(a), mx, flags, _p(o.counts), _p(o.ent), ent_cap,
                                  _p(o.snd), snd_cap, _p(o.pay), pay_cap, o.ref(o.total), o.ref(o.n_sends), o.ref(o.pbytes))
    return rc, ("total", "n_sends", "pbytes")


def _expire(g, o, agents, flags=0, ent_cap=REC_CAP, snd_cap=REC_CAP, pay_cap=REC_CAP * L, archive=True, cutoff=-1.0):
    from swarmdb_b200._native import _p
    a = None if agents is None else np.asarray(agents, np.uint32)
    ent, snd, pay = (o.ent, o.snd, o.pay) if archive else (None, None, None)
    rc = g._L.sdb_expire(g._h, 0 if a is None else len(a), _p(a), cutoff, flags, _p(o.counts), _p(ent), ent_cap,
                         _p(snd), snd_cap, _p(pay), pay_cap, o.ref(o.total), o.ref(o.n_sends), o.ref(o.pbytes))
    return rc, ("total", "n_sends", "pbytes")


def _where(g, o, agents, mx=4, flags=0, filt=None, hdr_cap=REC_CAP, pay_cap=REC_CAP * L, outputs=True):
    from swarmdb_b200._native import _p, make_filter
    a = None if agents is None else np.asarray(agents, np.uint32)
    f = make_filter() if filt is None else filt
    hdr, pay = (o.hdr, o.pay) if outputs else (None, None)
    rc = g._L.sdb_receive_where(g._h, 0 if a is None else len(a), _p(a), mx, flags, C.byref(f), _p(o.counts), _p(hdr),
                                hdr_cap, _p(pay), pay_cap, o.ref(o.total), o.ref(o.pbytes))
    return rc, ("total", "pbytes")


def _restore(g, o, agents, counts, n_ent, n_snd=1, pay_bytes=0, flags=0, null=()):
    from swarmdb_b200._native import ENTRY_DTYPE, SEND_DTYPE, _p
    a = None if "agents" in null else np.asarray(agents, np.uint32)
    c = None if "counts" in null else np.asarray(counts, np.uint32)
    ent = None if "entries" in null else np.zeros(max(n_ent, 1), ENTRY_DTYPE)
    snd = None if "sends" in null else np.zeros(max(n_snd, 1), SEND_DTYPE)
    pay = None if "payload" in null else np.zeros(max(pay_bytes, 1), np.uint8)
    rc = g._L.sdb_restore_compact(g._h, len(agents), _p(a), _p(c), _p(ent), n_ent, _p(snd), n_snd, _p(pay), pay_bytes,
                                  flags, o.ref(o.restored), o.ref(o.seq_end))
    return rc, ("restored",)


def _filter(**kw):
    from swarmdb_b200._native import make_filter
    f = make_filter()
    for k, v in kw.items():
        setattr(f, k, v)
    return f


def _cases():
    from swarmdb_b200._native import EXPIRE_ALL, RECV_ASYNC, RECV_OWNED, RECV_PEEK, RECV_PRIORITY, WHERE_DROP
    many = np.arange(20)                            # more than 8 agents: the bulk path of sdb_receive_batch
    few = np.arange(3)                              # the latency path's shape
    rep = [5, 9, 5]
    return [
        # sdb_receive_batch
        ("batch eoutput hdr_cap", EOUTPUT, lambda g, o: _batch(g, o, many, hdr_cap=0)),
        ("batch eoutput payload_cap", EOUTPUT, lambda g, o: _batch(g, o, many, pay_cap=L - 1)),
        ("batch eoutput latency shape", EOUTPUT, lambda g, o: _batch(g, o, few, hdr_cap=0)),
        ("batch out of range", EINVAL, lambda g, o: _batch(g, o, [1, A])),
        ("batch repeated", EINVAL, lambda g, o: _batch(g, o, rep)),
        ("batch repeated latency shape", EINVAL, lambda g, o: _batch(g, o, rep, flags=RECV_PRIORITY)),
        ("batch n_agents > max_agents", EINVAL, lambda g, o: _batch(g, o, np.arange(A), n=A + 1)),
        ("batch async with host outputs", EINVAL, lambda g, o: _batch(g, o, many, flags=RECV_ASYNC)),
        ("batch no agents before eoutput", OK, lambda g, o: _batch(g, o, [], hdr_cap=0)),
        ("batch max_messages 0 before einval", OK, lambda g, o: _batch(g, o, rep, mx=0)),
        # sdb_receive_compact
        ("compact eoutput entry_cap", EOUTPUT, lambda g, o: _compact(g, o, many, ent_cap=0)),
        ("compact eoutput send_cap", EOUTPUT, lambda g, o: _compact(g, o, many, snd_cap=0)),
        ("compact eoutput payload_cap", EOUTPUT, lambda g, o: _compact(g, o, None, pay_cap=L - 1)),
        ("compact out of range", EINVAL, lambda g, o: _compact(g, o, [0, A + 7])),
        ("compact repeated", EINVAL, lambda g, o: _compact(g, o, rep)),
        ("compact async", EINVAL, lambda g, o: _compact(g, o, many, flags=RECV_ASYNC)),
        ("compact no agents before eoutput", OK, lambda g, o: _compact(g, o, [], ent_cap=0)),
        ("compact max_messages 0 before einval", OK, lambda g, o: _compact(g, o, rep, mx=0)),
        # sdb_expire
        ("expire bad flags", EINVAL, lambda g, o: _expire(g, o, many, flags=RECV_PRIORITY)),
        ("expire async", EINVAL, lambda g, o: _expire(g, o, many, flags=RECV_ASYNC | EXPIRE_ALL)),
        ("expire eoutput entry_cap", EOUTPUT, lambda g, o: _expire(g, o, many, ent_cap=0)),
        ("expire eoutput before the empty list", EOUTPUT, lambda g, o: _expire(g, o, [], ent_cap=0, snd_cap=0)),
        ("expire eoutput payload_cap", EOUTPUT, lambda g, o: _expire(g, o, None, pay_cap=L - 1, flags=RECV_PEEK)),
        ("expire out of range", EINVAL, lambda g, o: _expire(g, o, [A], archive=False)),
        ("expire repeated", EINVAL, lambda g, o: _expire(g, o, rep, flags=EXPIRE_ALL, archive=False)),
        ("expire empty list, drop", OK, lambda g, o: _expire(g, o, [], archive=False)),
        # sdb_receive_where
        ("where struct_bytes", EINVAL, lambda g, o: _where(g, o, many, filt=_filter(struct_bytes=8))),
        ("where unknown fields", EINVAL, lambda g, o: _where(g, o, many, filt=_filter(fields=512))),
        ("where async", EINVAL, lambda g, o: _where(g, o, many, flags=RECV_ASYNC)),
        ("where bad flags", EINVAL, lambda g, o: _where(g, o, many, flags=EXPIRE_ALL)),
        ("where keyword too long", EINVAL, lambda g, o: _where(g, o, many, filt=_filter(fields=128, keyword_len=257))),
        ("where null keyword", EINVAL, lambda g, o: _where(g, o, many, filt=_filter(fields=128, keyword_len=3))),
        ("where drop with outputs", EINVAL, lambda g, o: _where(g, o, many, flags=WHERE_DROP)),
        ("where eoutput hdr_cap", EOUTPUT, lambda g, o: _where(g, o, many, hdr_cap=0)),
        ("where eoutput payload_cap", EOUTPUT, lambda g, o: _where(g, o, None, pay_cap=L - 1, flags=RECV_OWNED)),
        ("where out of range", EINVAL, lambda g, o: _where(g, o, [A + 1])),
        ("where repeated", EINVAL, lambda g, o: _where(g, o, rep, flags=WHERE_DROP, outputs=False)),
        ("where no agents before eoutput", OK, lambda g, o: _where(g, o, [], hdr_cap=0)),
        # sdb_restore_compact
        ("restore bad flags", EINVAL, lambda g, o: _restore(g, o, [1], [1], 1, flags=RECV_PEEK)),
        ("restore null agents", EINVAL, lambda g, o: _restore(g, o, [1], [1], 1, null=("agents",))),
        ("restore null counts", EINVAL, lambda g, o: _restore(g, o, [1], [1], 1, null=("counts",))),
        ("restore null entries", EINVAL, lambda g, o: _restore(g, o, [1], [1], 1, null=("entries",))),
        ("restore null payload", EINVAL, lambda g, o: _restore(g, o, [1], [1], 1, pay_bytes=32, null=("payload",))),
        ("restore out of range", EINVAL, lambda g, o: _restore(g, o, [A], [1], 1)),
        ("restore repeated", EINVAL, lambda g, o: _restore(g, o, [2, 2], [1, 1], 2)),
        ("restore sum(count)", EINVAL, lambda g, o: _restore(g, o, [1, 2], [1, 1], 3)),
        ("restore entries over capacity", ECAPACITY, lambda g, o: _restore(g, o, [1], [REC_CAP + 1], REC_CAP + 1)),
        ("restore sends over capacity", ECAPACITY, lambda g, o: _restore(g, o, [1], [1], 1, n_snd=REC_CAP + 1)),
        ("restore payload over capacity", ECAPACITY, lambda g, o: _restore(g, o, [1], [1], 1, pay_bytes=REC_CAP * L + 32)),
        ("restore no agents", OK, lambda g, o: _restore(g, o, [], [], 0, n_snd=0)),
    ]


def test_receive_calls_input_contract():
    from oracle.cpu_ref import CpuOracle
    from swarmdb_b200._native import Shard
    rng = np.random.default_rng(17)
    g = Shard(max_agents=A, ring_slots=256, arena_bytes=1 << 24, max_payload_bytes=L, max_recv_records=REC_CAP,
              max_recv_payload=REC_CAP * L)
    c = CpuOracle(A, 1)
    idx = np.arange(A, dtype=np.uint32)
    g.register(idx); c.register(idx)
    n = 6000
    s, r, prio = rng.integers(0, A, n), rng.integers(0, A, n), rng.integers(0, 4, n)
    lens, off, buf = _payloads(rng, n, L)
    assert g.send_batch(s, r, prio, None, lens, off, buf) == c.send_batch(s, r, prio, None, lens, off, buf)
    cases = _cases()
    assert len({name for name, _, _ in cases}) == len(cases)
    for k, (name, want, call) in enumerate(cases):
        loads0 = g.agent_loads(idx)
        st0 = g.stats()
        o = Outs()
        rc, scalars = call(g, o)
        assert rc == want, (name, rc, g._L.sdb_last_error(g._h))
        for f in scalars:
            assert getattr(o, f).value == 0, (name, f)
        if "restored" in scalars:
            assert o.seq_end.value == st0["next_seq"], name
        assert g.stats() == st0, name
        loads1 = g.agent_loads(idx)
        for f in loads0.dtype.names:
            assert np.array_equal(loads1[f], loads0[f]), (name, f)
        # the handle still serves: a normal receive equals the oracle's
        sel = ((np.arange(4) * 61 + 7 * k) % A).astype(np.uint32)
        cg, hg, pg = g.receive_batch(sel, 2)
        cc, hc, pc = c.receive_batch(sel, 2)
        assert np.array_equal(cg, cc) and hg.tobytes() == hc.tobytes() and pg.tobytes() == pc.tobytes(), name
        assert len(hg) > 0, name
    g.close(); c.close()
