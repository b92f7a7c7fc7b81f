"""The restated reference programs (examples/helloworld.cpp, examples/bounce.cpp) on the C++ facade
(mpi_b200/cpp/mpi.hpp), launched by the native gompirun (mpirun/gompirun.cpp)."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "examples", "bin")


@pytest.fixture(scope="module", autouse=True)
def _build_examples():
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "examples")])


def test_gompirun_appends_flags_after_user_args():
    """gompirun.go:77-83: user args, then -mpi-addr <own> -mpi-alladdr <list>; ports from :6000."""
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    out = subprocess.run([os.path.join(BIN, "gompirun"), "3", "/bin/echo", "hi", "-x"], capture_output=True, text=True, env=env, timeout=60)
    lines = sorted(out.stdout.strip().splitlines())
    assert out.returncode == 0 and len(lines) == 3
    for i, line in enumerate(lines):
        assert re.match(r"hi -x -mpi-addr :600%d -mpi-alladdr :6000,:6001,:6002( -mpi-gpu \d+)?$" % i, line), line


def test_gompirun_argument_errors_and_child_failure():
    g = os.path.join(BIN, "gompirun")
    assert subprocess.run([g], capture_output=True).returncode == 2
    assert subprocess.run([g, "x", "/bin/true"], capture_output=True).returncode == 2
    assert subprocess.run([g, "0", "/bin/true"], capture_output=True).returncode == 2
    assert subprocess.run([g, "9", "/bin/true"], capture_output=True).returncode == 2
    assert subprocess.run([g, "2", "/bin/false"], capture_output=True).returncode == 1  # reference ignores it; we report it


def test_cpp_facade_refuses_data_calls_without_a_device():
    """-mpi-gpu -2 = control plane only: Init works, Send/Receive report the missing device."""
    out = subprocess.run([os.path.join(BIN, "helloworld"), "-mpi-gpu", "-2"], capture_output=True, text=True, timeout=60)
    assert "Hello world, I'm node 0 in a land with 1 nodes" in out.stdout
    assert out.returncode == 1 and "no CPU data path" in out.stderr


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 2, 4])
def test_helloworld_cpp(n):
    env = dict(os.environ, GOMPIRUN_BASE_PORT=str(6100 + 10 * n), B200MPI_HEAP_BYTES=str(256 << 20), B200MPI_WATCHDOG_S="90")
    out = subprocess.run([os.path.join(BIN, "gompirun"), str(n), os.path.join(BIN, "helloworld"), "-mpi-inittimeout", "60s"],
                         capture_output=True, text=True, env=env, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    for r in range(n):
        assert "Hello world, I'm node %d in a land with %d nodes" % (r, n) in out.stdout
        assert 'I, node %d, received a message: "I\'m just node %d talking to myself"' % (r, r) in out.stdout
        for s in range(n):
            if s != r:
                assert 'I, node %d, received a message: "Hello node %d, I\'m node %d"' % (r, r, s) in out.stdout


@pytest.mark.gpu
def test_bounce_cpp():
    env = dict(os.environ, GOMPIRUN_BASE_PORT="6200", B200MPI_HEAP_BYTES=str(512 << 20), B200MPI_WATCHDOG_S="90")
    out = subprocess.run([os.path.join(BIN, "gompirun"), "2", os.path.join(BIN, "bounce"), "-mpi-inittimeout", "60s"],
                         capture_output=True, text=True, env=env, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr  # non-zero if any round trip came back different
    assert "Number of nodes =  2" in out.stdout
    assert "Average float64 trip time in us between node 0 and 1" in out.stdout
    assert "message not the same" not in out.stderr


def test_cpp_facade_host_logic():
    """mpi.hpp on a CPU-only box: flags, durations, Register-once, pre-Init answers."""
    import tempfile
    exe = os.path.join(tempfile.mkdtemp(prefix="b200mpi-facade-"), "facade_test")
    lib = os.path.join(ROOT, "mpi_b200", "lib")
    subprocess.check_call([os.environ.get("CXX", "g++"), "-std=c++17", "-O1", "-o", exe, os.path.join(ROOT, "tests", "cpp", "facade_test.cpp"),
                           "-L" + lib, "-lb200mpi", "-Wl,-rpath," + lib, "-pthread"])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert out.returncode == 0 and "facade ok" in out.stdout, out.stdout + out.stderr


def test_heap_allocator_unit():
    """First-fit sub-allocator of the device heap: granules, reuse, coalescing, exhaustion, stress."""
    import tempfile
    exe = os.path.join(tempfile.mkdtemp(prefix="b200mpi-heap-"), "heap_alloc_test")
    subprocess.check_call(["/usr/local/cuda/bin/nvcc", "-std=c++17", "-O1", "-o", exe, os.path.join(ROOT, "tests", "cpp", "heap_alloc_test.cpp"),
                           os.path.join(ROOT, "mpi_b200", "csrc", "heap.cpp"), os.path.join(ROOT, "mpi_b200", "csrc", "ctrl.cpp"), "-cudart", "static", "-lpthread"])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and "heap allocator ok" in out.stdout, out.stdout + out.stderr


def test_ownership_arithmetic_unit():
    """kernels.cuh Owner (shared by two-shot, TMA two-shot, NVLS, hybrid, scatter+multicast Bcast): every
    vector owned exactly once for every (count, block shift, world size); LL lane layout."""
    import tempfile
    exe = os.path.join(tempfile.mkdtemp(prefix="b200mpi-owner-"), "owner_test")
    subprocess.check_call(["/usr/local/cuda/bin/nvcc", "-std=c++17", "-O1", "-gencode", "arch=compute_90a,code=sm_90a", "-o", exe,
                           os.path.join(ROOT, "tests", "cpp", "owner_test.cu"), "-cudart", "static"])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "owner ok" in out.stdout, out.stdout + out.stderr

