"""Token-budget receive model (TESTS ONLY): the rule of include/swarmdb_b200.h (sdb_receive_tokens) stated literally.

A record weighs the little-endian u32 at the start of its payload when its type carries TYPEF_TOKENS and its len is at
least 4, and 0 otherwise.  An agent's token take is the longest prefix of its delivery order whose weights sum to at
most max_agent_tokens (0: no token limit), or its first record alone when that one is heavier.  The call is then the
byte-budget call (tests/budget_ref.py) with each agent's max_messages lowered to its token take: both takes are
prefixes of one delivery order, so the joint take is the shorter of the two, and the call's capacity and truncation
rule apply on top.
"""
from __future__ import annotations

from tests.budget_ref import call_counts as budget_call_counts

TYPEF_TOKENS = 0x40


def weight(typ: int, payload: bytes) -> int:
    """Token weight of one record: its type byte and its payload bytes (at least len of them)."""
    if int(typ) & TYPEF_TOKENS and len(payload) >= 4:
        return int.from_bytes(bytes(payload[:4]), "little")
    return 0


def token_take(weights, max_agent_tokens: int) -> int:
    """Records of the longest prefix of `weights` whose sum is <= max_agent_tokens (0: all), the first one alone when
    it is heavier."""
    if not max_agent_tokens:
        return len(weights)
    n, used = 0, 0
    for w in weights:
        if used + w > max_agent_tokens and n > 0:
            break
        used += w
        n += 1
    return n


def call_counts(orders, max_messages: int, max_agent_bytes: int, max_agent_tokens: int, rec_cap: int, byte_cap: int):
    """Per-agent record counts of one token call; `orders` holds each listed agent's (payload length, weight) pairs in
    delivery order, in list order."""
    cut = []
    for recs in orders:
        k = min(max_messages, token_take([w for _, w in recs], max_agent_tokens))
        cut.append([ln for ln, _ in recs[:k]])
    return budget_call_counts(cut, max_messages, max_agent_bytes, rec_cap, byte_cap)


def token_sums(orders):
    """Pending token weight of each agent (sdb_pending_tokens)."""
    return [sum(w for _, w in recs) for recs in orders]
