"""The library's environment switches select other kernels (INTEGRATION.md).  They are read once per process, so each
setting runs a subset of the GPU parity suites in its own pytest process, chosen so that the kernel the switch
selects is exercised, and must still equal the oracle.

  SDB_SHARED_PAYLOAD=0  one payload copy per recipient for group batches above the pull threshold
  SDB_GATHER_TMA=0      LSU gather (k_recv_gather) also for bulk receives of 4096 records and more
  SDB_GATHER_LDGSTS=1   cp.async gather (k_recv_gather_cpa): bound >= 4096, records <= 544 bytes
  SDB_P2P_TMA=0         point-to-point enqueue without the TMA bulk copies
  SDB_PLAN_TICKET=0     stream-order receive plan without the ticketed look-back
  SDB_OVERLAP_INDEX=1   index build of pure group batches on a side stream beside the fan-out
"""
import os
import signal
import subprocess
import sys
from pathlib import Path

import pytest

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parents[1]
PARITY = "tests/test_gpu_parity.py"
SHARED = "tests/test_gpu_shared_layout.py"
PATHS = "tests/test_gpu_receive_paths.py"

MATRIX = {
    "SDB_SHARED_PAYLOAD=0": [SHARED + "::test_shared_records_through_the_small_receive_path",
                             SHARED + "::test_shared_records_through_the_latency_server",
                             SHARED + "::test_shared_records_through_the_bulk_gathers",
                             PARITY + "::test_ring_overflow_is_reported_not_silent",
                             PARITY + "::test_group_fanout_parity"],
    "SDB_GATHER_TMA=0": [SHARED + "::test_shared_records_through_the_bulk_gathers",
                         PARITY + "::test_priority_receive_matches_oracle_and_equal_priority_is_fifo",
                         PARITY + "::test_group_fanout_parity"],
    "SDB_GATHER_LDGSTS=1": [SHARED + "::test_shared_records_through_the_bulk_gathers",
                            SHARED + "::test_shared_batches_across_the_2_pow_32_handle_wrap",
                            PARITY + "::test_priority_receive_matches_oracle_and_equal_priority_is_fifo",
                            PARITY + "::test_broadcast_batches_owner_computes_index_equals_oracle"],
    "SDB_P2P_TMA=0": [PARITY + "::test_p2p_then_drain",
                      PARITY + "::test_ranked_p2p_enqueue_many_per_receiver_and_staged_resubmit",
                      PARITY + "::test_many_records_for_one_agent_in_one_batch"],
    "SDB_PLAN_TICKET=0": [PARITY + "::test_p2p_then_drain",
                          PARITY + "::test_receive_capacity_truncates_by_whole_agents_without_loss",
                          SHARED + "::test_shared_records_through_the_bulk_gathers",
                          PATHS + "::test_plan_warps_mix_empty_simple_holey_and_truncated_agents"],
    "SDB_OVERLAP_INDEX=1": [SHARED + "::test_shared_records_through_the_bulk_gathers",
                            SHARED + "::test_shared_batches_wrap_a_small_arena",
                            PARITY + "::test_group_fanout_parity"],
}


@pytest.mark.parametrize("setting", sorted(MATRIX))
def test_switch_keeps_parity(setting):
    name, value = setting.split("=")
    env = dict(os.environ)
    env[name] = value
    cmd = [sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider", *MATRIX[setting]]
    # own process group: on a timeout the whole group is killed, so nothing is left running
    p = subprocess.Popen(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                         start_new_session=True)
    try:
        out, _ = p.communicate(timeout=600)
    except subprocess.TimeoutExpired:
        os.killpg(p.pid, signal.SIGKILL)
        out, _ = p.communicate()
        pytest.fail(f"{setting}: timed out\n{out[-4000:]}")
    assert p.returncode == 0, f"{setting}:\n{out[-6000:]}"
    assert " passed" in out and "skipped" not in out, out[-2000:]
