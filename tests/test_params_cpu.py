"""The tuning knobs of b200mpi_set_param / b200mpi_get_param: every knob the header lists reads back
what it was set to, through its clamp; a B200MPI_* override at Init goes through the same clamp;
read-only and unknown names fail.  The library's state is global, so every case runs in a process of
its own.  The CPU cases use a control-plane-only world of one; the GPU cases bind cuda:0."""
import json
import os
import re
import subprocess
import sys

import pytest

from mpi_b200 import _lib as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

INT_MAX = 2**31 - 1
LANES = 2097152  # ll_cells(1) * 8: the LL lane capacity of a world of one (kernels.cuh)
FLAG = "flag"    # any non-zero value reads back as 1
# knob -> (lo, hi) of its clamp (None: unbounded on that side), or FLAG
CLAMPS = {
    "twoshot_unroll": FLAG,
    "nvls_unroll": (-2**31, INT_MAX),
    "nvls_min_ranks": (-2**31, INT_MAX),
    "nvls_max_blocks": (1, INT_MAX),
    "oneshot_max_bytes": (None, None),
    "ll_max_bytes": (0, LANES),
    "stage_chunk": (4096, None),
    "pipe_min_bytes": (None, None),
    "pipe_chunk_bytes": (65536, None),
    "bounce_chunk_bytes": (65536, None),
    "host_threads": (0, INT_MAX),
    "own_block_bytes": (4096, None),
    "hybrid_p2p_permille": (0, 900),
    "hybrid_p2p_blocks": (0, INT_MAX),
    "hybrid_min_bytes": (0, None),
    "bcast_nvls2": FLAG,
    "bcast_nvls_min": (0, None),
    "allgather_nvls_min": (0, None),
    "host_register": FLAG,
    "p2p_fast": FLAG,
    "watchdog_ms": (1, None),
}
READ_ONLY = ["sm_count", "shared_device", "epoch", "ll_seq"]
LADDER = [-1, 0, 1, 900, 901, 4095, 4096, 65535, 65536, 2**31 - 1, 2**31, 2**40]


def expected(name, v):
    c = CLAMPS[name]
    if c == FLAG:
        return int(v != 0)
    lo, hi = c
    if lo is not None:
        v = max(v, lo)
    if hi is not None:
        v = min(v, hi)
    return v


def header_names(fn):
    """The quoted names in the comment right above `int <fn>(` in include/b200mpi.h."""
    text = open(os.path.join(ROOT, "include", "b200mpi.h")).read()
    m = re.search(r"/\*((?:[^*]|\*(?!/))*)\*/\s*int " + fn + r"\(", text)
    assert m, fn
    return re.findall(r'"([a-z0-9_]+)"', m.group(1))


PRELUDE = (
    "import ctypes, json, os, sys\n"
    "from mpi_b200 import _lib as L\n"
    "lib = L.load()\n"
    "def get(name):\n"
    "    v = ctypes.c_int64(-12345)\n"
    "    rc = lib.b200mpi_get_param(name.encode(), ctypes.byref(v))\n"
    "    return [rc, v.value, L.last_error() if rc else '']\n"
    "def put(name, value):\n"
    "    rc = lib.b200mpi_set_param(name if name is None else name.encode(), value)\n"
    "    return [rc, L.last_error() if rc else '']\n")


def run(code, env=None, timeout=120):
    """Runs PRELUDE + code in a fresh interpreter with no B200MPI_* variables but `env`; returns the
    JSON object the code prints last."""
    e = {k: v for k, v in os.environ.items() if not k.startswith("B200MPI_")}
    e["PYTHONPATH"] = ROOT
    e.update(env or {})
    p = subprocess.run([sys.executable, "-c", PRELUDE + code], capture_output=True, text=True, cwd=ROOT, env=e, timeout=timeout)
    assert p.returncode == 0, p.stdout + p.stderr
    return json.loads(p.stdout.strip().splitlines()[-1])


CONTROL_ONLY = "assert lib.b200mpi_init(b'', b'', b'', 0, -2) == 0, L.last_error()\n"


def test_header_lists_the_knobs_this_file_pins():
    assert sorted(header_names("b200mpi_set_param")) == sorted(CLAMPS)
    assert sorted(header_names("b200mpi_get_param")) == sorted(READ_ONLY)


def test_before_init_both_entries_fail():
    out = run("print(json.dumps({'get': get('stage_chunk'), 'put': put('stage_chunk', 1)}))\n")
    assert out["get"][0] == L.ERR_NOT_INIT and "Init" in out["get"][2]
    assert out["put"][0] == L.ERR_NOT_INIT and "Init" in out["put"][1]


@pytest.fixture(scope="module")
def ladder():
    """{knob: [[set rc, get rc, value read back] per LADDER value]} from one control-only world."""
    return run(CONTROL_ONLY + (
        "names = %r\n"
        "ladder = %r\n"
        "out = {}\n"
        "for n in names:\n"
        "    out[n] = []\n"
        "    for v in ladder:\n"
        "        s = put(n, v)\n"
        "        out[n].append([s[0]] + get(n)[:2])\n"
        "lib.b200mpi_finalize()\n"
        "print(json.dumps(out))\n") % (sorted(CLAMPS), LADDER))


@pytest.mark.parametrize("name", sorted(CLAMPS))
def test_knob_reads_back_its_clamped_value(ladder, name):
    got = ladder[name]
    want = [[0, 0, expected(name, v)] for v in LADDER]
    assert got == want, list(zip(LADDER, got, want))


def test_read_only_unknown_and_null_fail():
    out = run(CONTROL_ONLY + (
        "ro = %r\n"
        "res = {'put_' + n: put(n, 1) for n in ro + ['no_such_knob']}\n"
        "res.update({'get_' + n: get(n) for n in ro + ['no_such_knob']})\n"
        "res['put_null'] = put(None, 1)\n"
        "res['get_null_name'] = lib.b200mpi_get_param(None, ctypes.byref(ctypes.c_int64()))\n"
        "res['get_null_result'] = [lib.b200mpi_get_param(b'stage_chunk', None), L.last_error()]\n"
        "print(json.dumps(res))\n") % READ_ONLY)
    for n in READ_ONLY + ["no_such_knob"]:
        assert out["put_" + n] == [L.ERR_ARG, "set_param: unknown parameter '%s'" % n]
    for n in READ_ONLY:
        assert out["get_" + n][0] == 0
    assert out["get_epoch"][1] == 1 and out["get_ll_seq"][1] == 0 and out["get_shared_device"][1] == 0
    assert out["get_no_such_knob"] == [L.ERR_ARG, -12345, "get_param: unknown parameter 'no_such_knob'"]
    assert out["put_null"] == [L.ERR_ARG, "set_param: unknown parameter ''"]
    assert out["get_null_name"] == L.ERR_ARG
    assert out["get_null_result"] == [L.ERR_ARG, "get_param: NULL result pointer"]


# (variable, value, knob, value read back): an override goes through the knob's clamp and is read
# with strtoll base 0
ENV_CASES = [
    ("B200MPI_STAGE_CHUNK", "-5", "stage_chunk", 4096),
    ("B200MPI_STAGE_CHUNK", "0x20000", "stage_chunk", 131072),
    ("B200MPI_ONESHOT_MAX", "65536", "oneshot_max_bytes", 65536),
    ("B200MPI_LL_MAX", "-1", "ll_max_bytes", 0),
    ("B200MPI_LL_MAX", "4096", "ll_max_bytes", 4096),
    ("B200MPI_LL_MAX", str(2**40), "ll_max_bytes", LANES),
    ("B200MPI_HYBRID_PERMILLE", "-3", "hybrid_p2p_permille", 0),
    ("B200MPI_HYBRID_PERMILLE", "250", "hybrid_p2p_permille", 250),
    ("B200MPI_HYBRID_PERMILLE", "5000", "hybrid_p2p_permille", 900),
    ("B200MPI_HOST_THREADS", "0x10", "host_threads", 16),
    ("B200MPI_HOST_THREADS", "-2", "host_threads", 0),
    ("B200MPI_HOST_THREADS", str(2**40), "host_threads", INT_MAX),
    ("B200MPI_HOST_REGISTER", "1", "host_register", 1),
    ("B200MPI_P2P_FAST", "0", "p2p_fast", 0),
]


@pytest.mark.parametrize("var,value,knob,want", ENV_CASES, ids=["%s=%s" % (c[0][8:], c[1]) for c in ENV_CASES])
def test_environment_override_is_clamped(var, value, knob, want):
    out = run(CONTROL_ONLY + "print(json.dumps(get(%r)))\n" % knob, env={var: value})
    assert out[:2] == [0, want], out


HOST_REGISTER_ON_OFF = "res = [put('host_register', 1), put('host_register', 0), get('host_register')]\n"


def test_host_register_off_in_a_control_only_world():
    """host_register can be switched on and off in a control-only world (test_gpu_control_only_world_
    creates_no_cuda_context checks that this makes no CUDA call)."""
    out = run(CONTROL_ONLY + HOST_REGISTER_ON_OFF + "print(json.dumps(res + [lib.b200mpi_finalize()]))\n")
    assert out == [[0, ""], [0, ""], [0, 0, ""], 0], out


# ---- GPU: a data-plane world of one on cuda:0 ------------------------------------------------------

DATA_PLANE = "assert lib.b200mpi_init(b'', b'', b'', 0, 0) == 0, L.last_error()\n"

# What get_param reports after a plain Init of a world of one on its own GPU (sm_count is checked
# against the device).
DEFAULTS = {
    "twoshot_unroll": 1, "nvls_unroll": 2, "nvls_min_ranks": 4, "nvls_max_blocks": 48,
    "oneshot_max_bytes": 256 << 10, "ll_max_bytes": 256 << 10, "stage_chunk": 32 << 20,
    "pipe_min_bytes": 8 << 20, "pipe_chunk_bytes": 16 << 20, "bounce_chunk_bytes": 4 << 20,
    "host_threads": 8, "own_block_bytes": 1 << 20, "hybrid_p2p_permille": 0, "hybrid_p2p_blocks": 0,
    "hybrid_min_bytes": 32 << 20, "bcast_nvls2": 1, "bcast_nvls_min": -1, "allgather_nvls_min": -1,
    "host_register": 0, "p2p_fast": 1, "watchdog_ms": 120000,
    "shared_device": 0, "epoch": 1, "ll_seq": 0,
}


@pytest.mark.gpu
def test_gpu_defaults_of_a_world_of_one():
    out = run(DATA_PLANE + (
        "res = {n: get(n) for n in %r}\n"
        "import torch\n"
        "res['device_sms'] = torch.cuda.get_device_properties(0).multi_processor_count\n"
        "res['finalize'] = lib.b200mpi_finalize()\n"
        "print(json.dumps(res))\n") % (sorted(DEFAULTS) + ["sm_count"]))
    assert out["finalize"] == 0
    assert out["sm_count"][:2] == [0, out["device_sms"]]
    assert {n: out[n][:2] for n in DEFAULTS} == {n: [0, v] for n, v in DEFAULTS.items()}


@pytest.mark.gpu
def test_gpu_environment_overrides_take_effect():
    env = {"B200MPI_P2P_FAST": "0", "B200MPI_LL_MAX": "4096", "B200MPI_HYBRID_PERMILLE": "250",
           "B200MPI_STAGE_CHUNK": "1048576", "B200MPI_ONESHOT_MAX": "65536", "B200MPI_HOST_THREADS": "3",
           "B200MPI_HOST_REGISTER": "1"}
    want = {"p2p_fast": 0, "ll_max_bytes": 4096, "hybrid_p2p_permille": 250, "stage_chunk": 1048576,
            "oneshot_max_bytes": 65536, "host_threads": 3, "host_register": 1}
    out = run(DATA_PLANE + "res = {n: get(n)[:2] for n in %r}\nres['finalize'] = lib.b200mpi_finalize()\n"
              "print(json.dumps(res))\n" % sorted(want), env=env)
    assert out == dict({n: [0, v] for n, v in want.items()}, finalize=0)


@pytest.mark.gpu
def test_gpu_control_only_world_creates_no_cuda_context():
    """A control-only world promises not to touch the GPU: leaving host_register mode with an empty
    registration cache, and Finalize, make no CUDA call, so device 0's primary context stays inactive."""
    out = run(CONTROL_ONLY + HOST_REGISTER_ON_OFF + (
        "cu = ctypes.CDLL('libcuda.so.1')\n"
        "def primary_ctx_active():\n"
        "    dev, flags, active = ctypes.c_int(), ctypes.c_uint(), ctypes.c_int(-1)\n"
        "    assert cu.cuInit(0) == 0 and cu.cuDeviceGet(ctypes.byref(dev), 0) == 0\n"
        "    assert cu.cuDevicePrimaryCtxGetState(dev, ctypes.byref(flags), ctypes.byref(active)) == 0\n"
        "    return active.value\n"
        "res.append(primary_ctx_active())\n"
        "res.append(lib.b200mpi_finalize())\n"
        "res.append(primary_ctx_active())\n"
        "print(json.dumps(res))\n"))
    assert out == [[0, ""], [0, ""], [0, 0, ""], 0, 0, 0], out


ALLREDUCE = (
    "import numpy as np\n"
    "from oracle import oracle as O\n"
    "def allreduce_host(x, y):\n"  # y outlives any registration of it
    "    y[:] = 0\n"
    "    rc = lib.b200mpi_allreduce(x.ctypes.data, y.ctypes.data, x.size, L.F32, L.SUM, L.HOST)\n"
    "    return rc, bool(np.array_equal(y, O.allreduce([x])))\n")


@pytest.mark.gpu
def test_gpu_host_register_off_drops_the_cache():
    """A pageable Allreduce from pipe_min_bytes up registers its buffers in host_register mode; leaving
    the mode unregisters them, and the same buffers then go through the bounce ring."""
    out = run(DATA_PLANE + ALLREDUCE + (
        "cu = ctypes.CDLL('libcuda.so.1')\n"
        "def host_registered(a):\n"   # CU_POINTER_ATTRIBUTE_MEMORY_TYPE == CU_MEMORYTYPE_HOST
        "    t = ctypes.c_uint(0)\n"
        "    rc = cu.cuPointerGetAttribute(ctypes.byref(t), ctypes.c_int(2), ctypes.c_uint64(a.ctypes.data))\n"
        "    return rc == 0 and t.value == 1\n"
        "x = O.fill(np.float32, 0xB2000001, (16 << 20) // 4)\n"
        "y = np.zeros_like(x)\n"
        "res = {'before': host_registered(x) or host_registered(y), 'on': put('host_register', 1)}\n"
        "res['first'] = allreduce_host(x, y)\n"
        "res['registered'] = host_registered(x) and host_registered(y)\n"
        "res['off'] = put('host_register', 0)\n"
        "res['after_off'] = host_registered(x) or host_registered(y)\n"
        "res['second'] = allreduce_host(x, y)\n"
        "res['finalize'] = lib.b200mpi_finalize()\n"
        "print(json.dumps(res))\n"))
    assert out == {"before": False, "on": [0, ""], "first": [0, True], "registered": True, "off": [0, ""],
                   "after_off": False, "second": [0, True], "finalize": 0}, out


@pytest.mark.gpu
def test_gpu_failed_init_then_a_working_world():
    """Init fails after binding the device (a bad B200MPI_EPOCH_START); the teardown leaves nothing
    behind that stops the next Init, whose world of one then computes."""
    out = run(ALLREDUCE + (
        "res = {'bad': [lib.b200mpi_init(b'', b'', b'', 0, 0), L.last_error()], 'rank': lib.b200mpi_rank()}\n"
        "del os.environ['B200MPI_EPOCH_START']\n"
        "res['good'] = lib.b200mpi_init(b'', b'', b'', 0, 0)\n"
        "h = O.fill(np.float32, 0xB2000002, 4099)\n"
        "res['allreduce'] = allreduce_host(h, np.zeros_like(h))\n"
        "send, recv = ctypes.c_void_p(), ctypes.c_void_p()\n"
        "x = O.fill(np.float32, 0xB2000003, 1 << 16)\n"
        "y = np.zeros_like(x)\n"
        "assert lib.b200mpi_alloc(x.nbytes, ctypes.byref(send)) == 0 and lib.b200mpi_alloc(x.nbytes, ctypes.byref(recv)) == 0\n"
        "assert lib.b200mpi_memcpy(send, x.ctypes.data, x.nbytes, 0) == 0\n"
        "rc = lib.b200mpi_allreduce(send, recv, x.size, L.F32, L.SUM, L.DEVICE)\n"
        "assert lib.b200mpi_memcpy(y.ctypes.data, recv, x.nbytes, 1) == 0\n"
        "res['allreduce_heap'] = [rc, bool(np.array_equal(y, O.allreduce([x])))]\n"
        "res['finalize'] = lib.b200mpi_finalize()\n"
        "print(json.dumps(res))\n"), env={"B200MPI_EPOCH_START": "2"})
    assert out["bad"][0] == L.ERR_ARG and "B200MPI_EPOCH_START" in out["bad"][1], out
    assert out["rank"] == -1
    assert {k: out[k] for k in ("good", "allreduce", "allreduce_heap", "finalize")} == {
        "good": 0, "allreduce": [0, True], "allreduce_heap": [0, True], "finalize": 0}, out
