"""The 32-bit counters without a GPU: a host build of flag_reached and ll_seq_next (kernels.cuh), a
simulation of the host's launch schedule across the epoch wrap, and the parser of
B200MPI_SCRUB_EVERY / B200MPI_EPOCH_START / B200MPI_LL_SEQ_START (hostutil.h)."""
import os
import re
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def wrap_test():
    exe = os.path.join(tempfile.mkdtemp(prefix="b200mpi-wrap-"), "wrap_test")
    subprocess.check_call(["/usr/local/cuda/bin/nvcc", "-std=c++17", "-O2", "-gencode", "arch=compute_90a,code=sm_90a", "-o", exe,
                           os.path.join(ROOT, "tests", "cpp", "wrap_test.cu"), "-cudart", "static"])
    return exe


def test_counters_schedule_and_parser(wrap_test):
    """flag_reached at lags 0, 1, 2^31 - 1, 2^31 and leads 1, 2^31 - 1, across 0; ll_seq_next never 0 and
    reporting every crossing of 2^32 once, from +1 and from a +2 resync; > 3 * 2^20 launches from starts
    1, 2^29, 2^31 and 2^32 (minus 40 strides) with resyncs and a skipped scrub, no row or counter ever
    looking ahead, the launch ending on 0 always the scrub; the clamp and the rejections of the parser."""
    out = subprocess.run([wrap_test], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "wrap ok" in out.stdout, out.stdout + out.stderr


@pytest.mark.parametrize("period", [1 << 16, 1 << 21])
def test_unclamped_scrub_period_lets_a_counter_look_ahead(wrap_test, period):
    """The same schedule with a scrub period above kScrubEvery (what B200MPI_SCRUB_EVERY allowed before
    it was clamped): some slot row or ring counter looks ahead of the value a launch waits for."""
    out = subprocess.run([wrap_test, "--period", str(period)], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    m = re.search(r"period %d: (\d+) rows or counters looked ahead, (\d+) scrubs ran" % period, out.stdout)
    assert m and int(m.group(1)) > 0, out.stdout
    if period >= 1 << 21:  # the 20-bit epoch index never matches: the scrub never runs
        assert int(m.group(2)) == 0, out.stdout
    assert "ahead: " in out.stdout
