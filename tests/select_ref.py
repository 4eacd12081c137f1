"""Filtered and leased receives by budget (TESTS ONLY): the take rule of include/swarmdb_b200.h
(sdb_receive_where_budget, sdb_receive_leased_select) composed from tests/where_ref.py, tests/budget_ref.py and
tests/tokens_ref.py.

An agent's take is computed over its pending records that match the filter, in delivery order: the shortest of
max_messages, the byte take (budget_ref.agent_take) and the token take (tokens_ref.token_take).  The call is then the
filtered receive (where_ref.where_select) with each agent's max_messages lowered to its take, so its capacity rule -
records only, the first agent in the output giving its first rec_cap - applies on top.  where_match reads keywords
from the untagged content bytes, so keyword filters are modelled here on records without TYPEF_TOKENS only.
"""
from __future__ import annotations

from tests.budget_ref import agent_take
from tests.tokens_ref import token_take, weight
from tests.where_ref import RECV_PRIORITY, where_match


def take(recs, max_messages: int, max_agent_bytes: int, max_agent_tokens: int) -> int:
    """recs: (payload length, token weight) of an agent's matches in delivery order."""
    return min(max_messages, agent_take([ln for ln, _ in recs], max_messages, max_agent_bytes),
               token_take([w for _, w in recs], max_agent_tokens))


def matches(recs, flags: int, filt):
    """Positions of the matching records of one agent's model queue [(header, padded payload)], in delivery order."""
    m = [i for i, (h, p) in enumerate(recs) if filt is None or where_match(h, p, filt)]
    if flags & RECV_PRIORITY:
        m.sort(key=lambda i: -int(recs[i][0]["prio"]))                # stable: stream order within a level
    return m


def record_cost(h, padded: bytes):
    """(payload length, token weight) of one record."""
    return int(h["len"]), weight(int(h["type"]), padded[:int(h["len"])])


def select(state, agents, max_messages: int, max_agent_bytes: int, max_agent_tokens: int, flags: int, filt,
           rec_cap: int):
    """Per-agent counts and [(agent, position)] in output order of one call on a model queue {agent: [(header, padded
    payload)]}, with where_select's capacity rule."""
    counts, chosen, total, cut = [], [], 0, False
    for a in agents:
        recs = state.get(int(a), [])
        m = matches(recs, flags, filt)
        k = take([record_cost(*recs[i]) for i in m], max_messages, max_agent_bytes, max_agent_tokens)
        n = 0 if cut else k
        if not cut and k and total + k > rec_cap:
            n, cut = (rec_cap if total == 0 else 0), True
        counts.append(n)
        chosen += [(int(a), i) for i in m[:n]]
        total += n
    return counts, chosen
