"""GPU tests of the local device copy (copy_local_kernel, run on an H100: pytest -m gpu).

A world of one rank turns Allreduce, Allgather and Gather into a device-to-device copy of the send
buffer.  Every check here is bit-exact against the input: all 256 (src, dst) byte offsets modulo 16
at small sizes (so both the aligned path and the misaligned fallback run), sizes around one CTA's
share, one grid's worth and the 8 MiB from which the one-pass kernel is used, 256 MiB + 48 bytes and
1 GiB; in place must leave the buffer as it was;
torch device tensors (not in the library's heap) go through the same copy.  The checks run in a
child process so that the library's state never leaks into other tests."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VEC = 16
CTA_BYTES = 512 * VEC   # bytes one CTA of copy_local_kernel moves (kLocalCopyThreads vectors)
GRID_BYTES = 132 * CTA_BYTES
MIN_BYTES = 8 << 20     # kLocalCopyMinBytes: smaller copies stay on copy_bytes_kernel
SIZES = [0, 1, 15, 16, 17, CTA_BYTES - 16, CTA_BYTES, CTA_BYTES + 16, GRID_BYTES - 16, GRID_BYTES + 16,
         MIN_BYTES - 16, MIN_BYTES, MIN_BYTES + 17, 4 * MIN_BYTES + 16]
BIG = (256 << 20) + 48


def pattern(n, seed):
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8)


def run_checks():
    sys.path.insert(0, ROOT)
    import mpi_b200 as mpi
    mpi.api._reset_for_tests(mpi.Cuda(Gpu=0))
    mpi.Init()
    fails = []
    try:
        src = mpi.Alloc(BIG + 64, np.uint8)
        dst = mpi.Alloc(BIG + 64, np.uint8)

        def check(name, coll, n, so, do, dtype=np.uint8):
            it = np.dtype(dtype).itemsize
            x = pattern(n * it, n * 257 + so * 17 + do)
            src[so:so + n * it].copy_from_host(x)
            dst[do:do + n * it + 16].copy_from_host(np.full(n * it + 16, 0xA5, dtype=np.uint8))
            s = mpi.api.DeviceSlice(n, dtype, src.ptr + so, owner=False)
            d = mpi.api.DeviceSlice(n, dtype, dst.ptr + do, owner=False)
            if coll == "allreduce":
                mpi.Allreduce(s, d)
            elif coll == "allgather":
                mpi.Allgather(s, d)
            else:
                mpi.Gather(s, d, 0)
            got = dst[do:do + n * it + 16].to_host()
            if not (np.array_equal(got[:n * it], x) and np.all(got[n * it:] == 0xA5)):
                fails.append("%s n=%d src+%d dst+%d" % (name, n, so, do))

        # every byte alignment pair at small sizes, u8 through Allgather and Gather
        for n in (1, 15, 17, 100, 4099):
            for so in range(16):
                for do in range(16):
                    check("allgather", "allgather", n, so, do)
        for n in SIZES:
            for so, do in ((0, 0), (3, 3), (5, 0), (0, 9)):
                check("gather", "gather", n, so, do)
                check("allgather", "allgather", n, so, do)
                # float32: byte offsets that are multiples of 4, aligned and misaligned mod 16
                check("allreduce", "allreduce", n // 4, 4 * (so % 4), 4 * (do % 4), np.float32)
        for so, do in ((0, 0), (7, 7), (0, 8)):
            check("allgather_big", "allgather", BIG, so, do)
        check("allreduce_big", "allreduce", BIG // 4, 0, 0, np.float32)

        # in place: a no-op
        x = pattern(GRID_BYTES + 16, 99)
        src[0:GRID_BYTES + 16].copy_from_host(x)
        b = src[3:GRID_BYTES + 3]
        mpi.Allgather(b, b)
        if not np.array_equal(src[0:GRID_BYTES + 16].to_host(), x):
            fails.append("in place changed the buffer")
        src.free()
        dst.free()

        # one 1 GiB copy
        gib = 1 << 30
        a = mpi.Alloc(gib // 4, np.float32)
        r = mpi.Alloc(gib // 4, np.float32)
        block = 1 << 24
        for lo in range(0, gib // 4, block):
            a[lo:lo + block].copy_from_host(np.arange(lo, lo + block, dtype=np.float32))
        mpi.Allreduce(a, r)
        for lo in range(0, gib // 4, block):
            if not np.array_equal(r[lo:lo + block].to_host(), np.arange(lo, lo + block, dtype=np.float32)):
                fails.append("1 GiB copy differs in block at %d" % lo)
                break
        a.free()
        r.free()

        # torch device tensors: not in the heap, the copy still runs on this GPU
        import torch
        for n, so, do in ((GRID_BYTES + 16, 0, 0), (CTA_BYTES + 1, 1, 1), (4099, 2, 11)):
            ts = torch.from_numpy(pattern(n + 16, n)).cuda()
            td = torch.full((n + 32,), 0xA5, dtype=torch.uint8, device="cuda")
            torch.cuda.synchronize()
            s = mpi.api.DeviceSlice(n, np.uint8, ts.data_ptr() + so, owner=False)
            d = mpi.api.DeviceSlice(n, np.uint8, td.data_ptr() + do, owner=False)
            mpi.Allgather(s, d)
            got = td.cpu().numpy()
            want = ts.cpu().numpy()[so:so + n]
            if not (np.array_equal(got[do:do + n], want) and np.all(got[:do] == 0xA5) and np.all(got[do + n:] == 0xA5)):
                fails.append("torch n=%d src+%d dst+%d" % (n, so, do))
    finally:
        mpi.Finalize()
    if fails:
        print("FAIL " + "; ".join(fails[:20]))
        return 1
    print("local copy ok")
    return 0


@pytest.mark.gpu
def test_local_copy_bit_exact_world_of_one():
    env = dict(os.environ, B200MPI_HEAP_BYTES=str((3 << 30) + (768 << 20)))
    out = subprocess.run([sys.executable, os.path.abspath(__file__)], capture_output=True, text=True, timeout=900, env=env, cwd=ROOT)
    assert out.returncode == 0 and "local copy ok" in out.stdout, out.stdout[-4000:] + out.stderr[-4000:]


if __name__ == "__main__":
    sys.exit(run_checks())
