"""The byte-budget receive model (tests/budget_ref.py) on hand-made ring windows: limits on and next to record
boundaries, oversized first records, zero-length payloads, tombstoned slots, priority order and first-agent truncation
by records, by bytes and by both."""
from tests.budget_ref import agent_take, call_counts, delivery_order, take_from_model
from tests.ring_ref import RingModel

BIG = 1 << 40


def test_limit_on_a_record_boundary_and_one_byte_short():
    sizes = [100, 32, 1, 64]                      # padded: 128, 32, 32, 64
    assert agent_take(sizes, 100, 192) == 3       # 128 + 32 + 32 == 192 exactly
    assert agent_take(sizes, 100, 191) == 2
    assert agent_take(sizes, 100, 256) == 4
    assert agent_take(sizes, 100, 255) == 3
    assert agent_take(sizes, 2, 256) == 2         # the record limit binds first
    assert agent_take(sizes, 100, 0) == 4         # 0: no byte limit


def test_oversized_first_record_is_taken_alone():
    assert agent_take([4000, 10], 100, 100) == 1
    assert agent_take([4000, 10], 100, 31) == 1
    assert agent_take([10, 4000], 100, 100) == 1  # only the first record may exceed the limit
    assert agent_take([], 100, 100) == 0


def test_zero_length_payloads_take_no_bytes():
    assert agent_take([0, 0, 0, 33, 0], 100, 1) == 3
    assert agent_take([0, 0, 0, 33, 0], 100, 64) == 5
    assert agent_take([0] * 10, 4, 1) == 4


def test_tombstoned_slots_are_skipped_and_priority_order_is_stable():
    m = RingModel(16)
    m.append(0, [1, 2, 3, 4, 5])
    m.retire(0, [2, 4])
    lens = {1: 64, 2: 5000, 3: 40, 4: 5000, 5: 10}
    prios = {1: 0, 2: 3, 3: 2, 4: 3, 5: 2}
    assert delivery_order(m, 0, prios, False) == [1, 3, 5]
    assert delivery_order(m, 0, prios, True) == [3, 5, 1]
    assert take_from_model(m, [0], lens, prios, 100, 96, False, BIG, BIG) == [1]    # 64; 64 more does not fit
    assert take_from_model(m, [0], lens, prios, 100, 160, False, BIG, BIG) == [3]   # 64 + 64 + 32
    assert take_from_model(m, [0], lens, prios, 100, 96, True, BIG, BIG) == [2]     # 64 + 32; 64 more does not fit
    assert take_from_model(m, [0], lens, prios, 100, 128, True, BIG, BIG) == [2]
    assert take_from_model(m, [0], lens, prios, 100, 160, True, BIG, BIG) == [3]


def test_call_capacity_truncates_whole_agents_after_the_first():
    orders = [[32] * 4, [32] * 4, [32] * 4]
    assert call_counts(orders, 100, 0, BIG, BIG) == [4, 4, 4]
    assert call_counts(orders, 100, 0, 8, BIG) == [4, 4, 0]          # by records
    assert call_counts(orders, 100, 0, BIG, 255) == [4, 0, 0]        # by bytes: the second agent would reach 256
    assert call_counts(orders, 100, 0, 7, 256) == [4, 0, 0]          # by both
    assert call_counts([[], [32] * 4, [32]], 100, 0, BIG, 64) == [0, 2, 0]   # first in the output: its prefix


def test_first_agent_truncation_by_records_bytes_and_both():
    sizes = [[100, 100, 100, 100, 100]]           # padded 128 each
    assert call_counts(sizes, 100, 0, 3, BIG) == [3]
    assert call_counts(sizes, 100, 0, BIG, 300) == [2]
    assert call_counts(sizes, 100, 0, 2, 300) == [2]
    assert call_counts(sizes, 100, 0, 3, 300) == [2]
    assert call_counts(sizes, 100, 0, 1, 300) == [1]
    assert call_counts(sizes, 100, 384, 5, 300) == [2]  # the per-agent take (3), then the call's byte capacity


def test_later_agents_stay_queued_even_when_they_would_fit():
    orders = [[32], [32] * 10, [0]]
    assert call_counts(orders, 100, 0, 5, BIG) == [1, 0, 0]
    assert call_counts(orders, 100, 64, 5, BIG) == [1, 2, 1]
