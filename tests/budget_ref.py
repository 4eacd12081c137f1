"""Byte-budget receive model (TESTS ONLY): the rule of include/swarmdb_b200.h (sdb_receive_budget) stated literally.

An agent's take is the longest prefix of its delivery order with at most max_messages records and
sum(pad32(len)) <= max_agent_bytes (0: no byte limit), or its first record alone when that one is larger.  A call lays
the takes out agent by agent in list order; an agent whose take does not fit the record or the byte capacity stays
queued with every later agent, except the first agent in the output, which takes the longest prefix of its take that
fits both.  Delivery order comes from a RingModel window (tests/ring_ref.py): live slots in stream order, or stably
sorted by priority (highest first) for a priority receive.
"""
from __future__ import annotations


def pad32(n: int) -> int:
    return (int(n) + 31) & ~31


def delivery_order(model, a, prio_of, priority: bool):
    """Live seqs of agent `a` in the order a receive delivers them."""
    live = model.live_seqs(a)
    if priority:
        live = sorted(live, key=lambda s: -int(prio_of[s]))       # stable: arrival order within a level
    return live


def prefix(sizes, max_records: int, max_bytes) -> int:
    """Records of the longest prefix of `sizes` (payload lengths) with at most max_records records and padded bytes
    <= max_bytes (None: no limit), the first record taken alone when it is larger."""
    n, used = 0, 0
    for ln in sizes[:max_records]:
        p = pad32(ln)
        if max_bytes is not None and used + p > max_bytes and n > 0:
            break
        used += p
        n += 1
    return n


def agent_take(sizes, max_messages: int, max_agent_bytes: int) -> int:
    return prefix(sizes, max_messages, max_agent_bytes or None)


def call_counts(orders, max_messages: int, max_agent_bytes: int, rec_cap: int, byte_cap: int):
    """Per-agent record counts of one budget call; `orders` holds each listed agent's payload lengths in delivery
    order, in list order."""
    out, recs, used, closed = [], 0, 0, False
    for sizes in orders:
        k = agent_take(sizes, max_messages, max_agent_bytes)
        b = sum(pad32(x) for x in sizes[:k])
        if closed or k == 0:
            out.append(0)
            continue
        if recs + k <= rec_cap and used + b <= byte_cap:
            out.append(k)
            recs += k
            used += b
            continue
        closed = True
        if recs == 0:                                    # first in the output: the prefix of its take that fits
            k = prefix(sizes[:k], rec_cap, byte_cap)
            out.append(k)
            recs += k
            used += sum(pad32(x) for x in sizes[:k])
        else:
            out.append(0)
    return out


def take_from_model(model, agents, lens, prios, max_messages, max_agent_bytes, priority, rec_cap, byte_cap):
    """call_counts over the agents' RingModel windows (lens / prios: seq -> payload length / priority)."""
    orders = [[lens[s] for s in delivery_order(model, a, prios, priority)] for a in agents]
    return call_counts(orders, max_messages, max_agent_bytes, rec_cap, byte_cap)
