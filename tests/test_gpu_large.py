"""GPU tests of collectives past the 32-bit boundaries (run on an H100: pytest -m gpu).  The rank
processes run _large_worker.py.  Scenario 'high' places every buffer of _footprint_worker's calls at
planned heap offsets above, across and below 2^32 in a 4.5 GiB heap per rank; scenario 'long' moves
messages of 4 GiB and more (element indices past 2^31) in a world of two with a 9 GiB heap per rank,
and a 4 GiB local copy in a world of one.  When the box has fewer GPUs than ranks, the ranks share
device 0.  Before each world the test checks that the device memory and host memory it needs are
free, and skips naming the shortfall when they are not."""
import os
import subprocess
import threading
import time

import pytest

import _large_worker as LW
from _launch import assert_world_ok, run_world
from test_gpu_worlds import assert_nothing_skipped, need_gpus

pytestmark = pytest.mark.gpu
WORKER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_large_worker.py")
GiB = 1 << 30
CONTEXT = GiB  # a rank's CUDA context, its stream and the torch-free worker on top of its heap
HOST_HIGH = 2 * GiB  # per rank: the footprint worker's images and host views
HOST_LONG = 10 * GiB  # per rank: a 4 GiB pinned or pageable message and the windows the threads hold


def mem_available():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def gpu_memory(field):
    """nvidia-smi's `field` (memory.free, memory.used) of every GPU, in bytes; this process holds no CUDA context."""
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + field, "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout
    return [int(x) << 20 for x in out.split() if x.strip().isdigit()]


def need_memory(n, heap, host, what):
    """Skip (reported as SKIPPED) unless every GPU the ranks use has room for the ranks placed on it
    (rank r runs on device r % GPUs) and `host` bytes of host memory are available."""
    try:
        free = gpu_memory("memory.free")
    except Exception:  # noqa: BLE001
        free = []
    if not free:
        pytest.skip("%s needs a CUDA device" % what)
    short = []
    for d in range(min(n, len(free))):
        need = len(range(d, n, len(free))) * (heap + CONTEXT)
        if free[d] < need:
            short.append("device %d: %.1f GiB free, %.1f GiB needed" % (d, free[d] / GiB, need / GiB))
    avail = mem_available()
    if avail < host:
        short.append("host memory: %.1f GiB available, %.1f GiB needed" % (avail / GiB, host / GiB))
    if short:
        pytest.skip("%s: %s" % (what, "; ".join(short)))


class PeakMemory:
    """The most device memory in use on any GPU while the world runs, above what was in use on that
    GPU when it started (so other work already on a shared GPU is not counted), in MiB."""

    def __enter__(self):
        self.base = gpu_memory("memory.used")
        self.peak, self.stop = 0, threading.Event()
        self.thread = threading.Thread(target=self._poll, daemon=True)
        self.thread.start()
        return self

    def _poll(self):
        while not self.stop.is_set():
            try:
                now = gpu_memory("memory.used")
                self.peak = max([self.peak] + [(u - b) >> 20 for u, b in zip(now, self.base)])
            except Exception:  # noqa: BLE001
                pass
            self.stop.wait(1.0)

    def __exit__(self, *exc):
        self.stop.set()
        self.thread.join()


def world(n, scenario, parts, heap, host, timeout=900):
    """The library's own watchdog applies: 120 s, or 600 s when ranks time-slice one GPU."""
    need_memory(n, heap, host, "a world of %d with a %.1f GiB heap per rank" % (n, heap / GiB))
    t0 = time.time()
    with PeakMemory() as pm:
        res = run_world(n, scenario, args=["--parts", parts], timeout=timeout, worker=WORKER, env={"B200MPI_HEAP_BYTES": str(heap)})
    assert_world_ok(res)
    print("world of %d, %s %s: %.0f s, peak device memory of the world %d MiB" % (n, scenario, parts, time.time() - t0, pm.peak))
    return res


@pytest.mark.parametrize("n", [2, 3, 4])
def test_buffers_above_across_and_below_4_gib_of_heap(n):
    """Every P2P collective, Send / Receive and Isend / Wait with rank 0's buffers above 2^32, rank 1's
    send across it and its recv below, ranks 2 and 3 below: guards, out-of-place sends and the oracle
    in the order of the kernel that ran, as in test_gpu_footprint.py."""
    res = world(n, "high", "reductions,bytes,v,p2p", LW.HIGH_HEAP, n * HOST_HIGH)
    for r in res:
        print("rank %d: slots at heap offsets %s, staging probe at %s, %d buffers placed %s, %d calls checked %s, seconds %s" % (
            r["rank"], r["slots"], r["probe"], r["placed"], r["sides"], r["checked"], r["by_part"], r["seconds"]))
    assert res[0]["sides"].get("above") and not res[0]["sides"].get("below"), res[0]["sides"]
    assert res[1]["sides"].get("straddles") and res[1]["sides"].get("below"), res[1]["sides"]
    assert all(not r["sides"].get("above") and not r["sides"].get("straddles") for r in res[2:])


def test_switch_paths_above_4_gib_of_heap():
    """NVLS Allreduce, Reduce, ReduceScatter and both NVLS Bcasts with every rank's buffers at the
    same offsets above 2^32.  Ranks sharing one GPU cannot bind a multicast object: SKIPPED there."""
    have = need_gpus(2, "multimem (NVLS) kernels")
    n = 4 if have >= 4 else 2
    res = world(n, "high", "nvls", LW.HIGH_HEAP, n * HOST_HIGH)
    assert all(r["nvls"] for r in res), "multicast mapping was not set up on a multi-GPU box"
    assert_nothing_skipped(res)


@pytest.mark.parametrize("parts", ["allreduce", "reduce", "bytes", "v", "p2p", "hostpipe"])
def test_messages_past_4_gib_in_a_world_of_two(parts):
    """Every byte of 4-8 GiB messages, guards and sends included, against the plain two-rank reference
    (_large_worker.part_long_<parts>): Allreduce with the two-shot, TMA two-shot and ring kernels and
    Reduce; ReduceScatter, Scan, Exscan and ReduceScatterv; both P2P Bcasts, push and ring Allgather
    and Alltoall; Gatherv, Scatterv, Allgatherv and Alltoallv; Send / Receive from heap and pageable
    memory and Isend / Wait; the pinned and pageable host-slice pipeline."""
    res = world(2, "long", parts, LW.LONG_HEAP, 2 * HOST_LONG)
    for r in res:
        print("rank %d: %d calls checked, seconds %s, heap peak %.2f GiB (buffers %.2f GiB): %s" % (
            r["rank"], r["checked"], r["seconds"], r["heap_peak"] / GiB, r["buffer_peak"] / GiB, "; ".join(r["calls"])))
        assert r["heap_peak"] <= LW.LONG_HEAP - LW.RESERVED


def test_local_copy_past_4_gib_in_a_world_of_one():
    """An out-of-place Allreduce of 4 GiB + 20 bytes in a world of one: copy_local_kernel with send and
    recv 16-byte aligned, copy_bytes_kernel with recv 4 bytes off."""
    res = world(1, "long", "local", LW.LONG_HEAP, HOST_LONG)
    print("%d calls checked, seconds %s: %s" % (res[0]["checked"], res[0]["seconds"], "; ".join(res[0]["calls"])))
