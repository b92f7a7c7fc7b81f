"""The chunk rule of the pipelined host-slice collectives without a GPU: a host build of
pipe_chunk_elems (hostutil.h), and the chunk counts each rank of the mixed-pinning worlds of
test_gpu_buffer_kinds.py launches under the previous rule and under this one."""
import os
import subprocess
import tempfile

import pytest

import _kinds_worker as K

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ES = {"f32": 4, "f64": 8, "i64": 8}


@pytest.fixture(scope="module")
def pipe_chunk_test():
    exe = os.path.join(tempfile.mkdtemp(prefix="b200mpi-pipe-chunk-"), "pipe_chunk_test")
    for cxx in ("/usr/bin/g++", "g++", os.environ.get("CXX", "c++")):
        try:
            r = subprocess.run([cxx, "-std=c++17", "-O1", "-pthread", "-o", exe, os.path.join(ROOT, "tests", "cpp", "pipe_chunk_test.cpp")],
                               capture_output=True, text=True)
        except FileNotFoundError:
            continue
        if r.returncode == 0:
            return exe
    raise AssertionError("cannot build pipe_chunk_test: %s" % r.stderr[-2000:])


def test_chunk_rule(pipe_chunk_test):
    """Positive multiples of 4096 elements; in a multi-rank world independent of whether the rank
    bounces; a bouncing rank and a world of one keep the previous rule."""
    out = subprocess.run([pipe_chunk_test], capture_output=True, text=True, timeout=60)
    assert out.returncode == 0 and "pipe_chunk ok" in out.stdout, out.stdout + out.stderr


@pytest.mark.parametrize("n", [2, 3, 4, 8])
def test_mixed_pinning_worlds_launch_alike_only_under_the_new_rule(pipe_chunk_test, n):
    """For every call of part hostpipe, the chunk launches of each rank: under the previous rule a
    bouncing rank and a pinned, registered or direct rank of the same call disagree in every world
    (the GPU test would wait for the watchdog there), under the new rule all agree."""
    knobs = dict(K.PIPE_KNOBS)
    calls = K.pipe_calls(n)
    args = [str(knobs["pipe_chunk_bytes"]), str(knobs["bounce_chunk_bytes"])]
    for _, _, dn, count, rows, _ in calls:
        args += [str(ES[dn]), str(rows), str(n), str(count)]
    out = subprocess.run([pipe_chunk_test] + args, capture_output=True, text=True, timeout=60)
    assert out.returncode == 0, out.stdout + out.stderr
    lines = out.stdout.splitlines()
    assert len(lines) == len(calls), out.stdout
    diverged = 0
    for (i, coll, dn, count, rows, extra), line in zip(calls, lines):
        old_b, old_d, new_b, new_d = [int(x.split("=")[1]) for x in line.split() if "=" in x]
        bounce = [K.pipe_bounces(n, r, K.PIPE_MEMS[(r + i) % len(K.PIPE_MEMS)]) for r in range(n)]
        old = [old_b if b else old_d for b in bounce]
        new = [new_b if b else new_d for b in bounce]
        print("n=%d %s %s %s count=%d: bounce per rank %s, chunks old %s new %s" % (n, coll, extra, dn, count, bounce, old, new))
        assert len(set(new)) == 1, (coll, dn, count, new)
        diverged += len(set(old)) > 1
    assert diverged > 0, "no call of the mixed-pinning world of %d diverged under the previous rule" % n
