"""The library's one environment switch, SDB_SHARED_PAYLOAD=0, keeps one payload copy per recipient for group batches
above the pull threshold (INTEGRATION.md).  It is read once per process, so the matrix runs a subset of the GPU parity
suites in its own pytest process, chosen so that the layout the switch selects is exercised, and must still equal the
oracle.
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

MATRIX = {
    "SDB_SHARED_PAYLOAD=0": [SHARED + "::test_shared_records_through_the_small_receive_path",
                             SHARED + "::test_shared_records_through_the_latency_server",
                             SHARED + "::test_shared_records_through_the_bulk_gathers",
                             PARITY + "::test_ring_overflow_is_reported_not_silent",
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
