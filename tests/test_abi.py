"""The C-ABI library loads on a box without a GPU and exports exactly what include/b200mpi.h
declares; before Init the facade answers like the reference (Rank -1, Size 0, mpi.go:110-118);
and without a device the product fails loudly instead of falling back to anything."""
import ctypes
import os
import re
import subprocess
import sys

import pytest

import mpi_b200 as mpi
from mpi_b200 import _lib as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    text = open(os.path.join(ROOT, "include", "b200mpi.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(b200mpi_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    names = header_symbols()
    assert len(names) >= 30
    lib = ctypes.CDLL(mpi.LIB_PATH)
    for nm in names:
        assert hasattr(lib, nm), "%s declared in b200mpi.h but not exported" % nm
    assert sorted(L.SYMBOLS) == names, "python binding and header disagree"
    out = subprocess.run(["nm", "-D", "--defined-only", mpi.LIB_PATH], capture_output=True, text=True).stdout
    exported = sorted(set(re.findall(r" T (b200mpi_[a-z0-9_]+)", out)))
    assert exported == names, "library exports symbols the header does not declare (or vice versa)"


def test_header_is_plain_c():
    """The boundary is a C ABI: the header must compile as C99 with nothing but libc headers."""
    import tempfile
    src = os.path.join(tempfile.mkdtemp(prefix="b200mpi-hdr-"), "t.c")
    with open(src, "w") as f:
        f.write('#include "b200mpi.h"\nint main(void) { return b200mpi_rank() == -1 && B200MPI_MAX_RANKS == 8 ? 0 : 1; }\n')
    exe = src[:-2]
    lib = os.path.join(ROOT, "mpi_b200", "lib")
    subprocess.check_call(["gcc", "-std=c99", "-pedantic", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), src, "-o", exe,
                           "-L" + lib, "-lb200mpi", "-Wl,-rpath," + lib])
    assert subprocess.run([exe]).returncode == 0  # links against the real library and answers like the reference before Init


def test_no_link_time_dependency_on_libcuda_or_torch():
    out = subprocess.run(["ldd", mpi.LIB_PATH], capture_output=True, text=True).stdout
    assert "libcuda.so" not in out and "torch" not in out and "nccl" not in out


def test_library_contains_sm_90a_code_only():
    out = subprocess.run(["cuobjdump", "--list-elf", mpi.LIB_PATH], capture_output=True, text=True).stdout
    archs = set(re.findall(r"sm_(\d+a?)", out))
    assert archs == {"90a"}, archs


def test_before_init_matches_reference_conventions():
    lib = mpi.load()
    assert lib.b200mpi_version() == 200
    assert mpi.Rank() == -1 and mpi.Size() == 0  # mpi.go:110-118
    assert lib.b200mpi_device() == -1
    p = ctypes.c_void_p()
    assert lib.b200mpi_alloc(16, ctypes.byref(p)) == L.ERR_NOT_INIT
    assert lib.b200mpi_barrier() == L.ERR_NOT_INIT
    assert lib.b200mpi_allreduce(None, None, 0, L.F32, L.SUM, L.HOST) == L.ERR_NOT_INIT
    assert lib.b200mpi_send(None, 0, L.U8, 0, 0, L.HOST) == L.ERR_NOT_INIT
    assert "Init" in L.last_error()
    assert lib.b200mpi_finalize() == L.ERR_NOT_INIT


def _has_gpu():
    try:
        return subprocess.run(["nvidia-smi", "-L"], capture_output=True, text=True, timeout=20).stdout.count("GPU ") > 0
    except Exception:  # noqa: BLE001
        return False


@pytest.mark.skipif(_has_gpu(), reason="box has a GPU")
def test_init_without_a_device_fails_loudly():
    code = (
        "import mpi_b200 as mpi\n"
        "try:\n"
        "    mpi.Init()\n"
        "    print('INIT-OK')\n"
        "except mpi.MpiError as e:\n"
        "    print('CODE', e.code, e.message)\n")
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=ROOT,
                         env=dict(os.environ, PYTHONPATH=ROOT)).stdout
    assert "CODE -10" in out and "no CPU fallback" in out, out


@pytest.mark.skipif(_has_gpu(), reason="box has a GPU")
def test_failed_init_leaves_the_library_reusable():
    code = (
        "from mpi_b200 import _lib as L\n"
        "lib = L.load()\n"
        "rc1 = lib.b200mpi_init(b'', b'', b'', 0, -1)\n"      # no device -> fails, state must be reset
        "r1 = (lib.b200mpi_rank(), lib.b200mpi_size())\n"
        "rc2 = lib.b200mpi_init(b'', b'', b'', 0, -2)\n"      # control plane only -> works
        "r2 = (lib.b200mpi_rank(), lib.b200mpi_size())\n"
        "rc3 = lib.b200mpi_init(b'', b'', b'', 0, -2)\n"      # Init twice -> error
        "rc4 = lib.b200mpi_finalize()\n"
        "print(rc1, r1, rc2, r2, rc3, rc4, lib.b200mpi_rank())\n")
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=ROOT, env=dict(os.environ, PYTHONPATH=ROOT)).stdout
    assert out.split() == ["-10", "(-1,", "0)", "0", "(0,", "1)", "-1", "0", "-1"], out


def test_product_does_not_import_the_oracle():
    """oracle/ is test infrastructure: nothing under mpi_b200/ may reference it."""
    for dirpath, _, files in os.walk(os.path.join(ROOT, "mpi_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".h", ".hpp")):
                text = open(os.path.join(dirpath, f), errors="replace").read()
                assert "import oracle" not in text and "from oracle" not in text and "liboracle" not in text, os.path.join(dirpath, f)
