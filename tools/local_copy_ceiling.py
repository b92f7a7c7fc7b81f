#!/usr/bin/env python
"""tools/local_copy_ceiling.py -- what a read-S / write-S stream reaches on this GPU, next to the
library's world-of-1 Allreduce (a local device copy, the call bench.py --gpus 1 times).

    python tools/local_copy_ceiling.py [--sizes 268435456,1073741824] [--iters 200] [--rounds 3] [--out FILE]

One process, one GPU.  Prints the card's name, power limit and max SM clock, then for every round
and size one line per item:

    allreduce   b200mpi_allreduce_async(float32, sum) on heap buffers, world of 1   read S + write S
    torch_copy  dst.copy_(src), the CUDA driver's device-to-device copy             read S + write S
    torch_sum   src.sum(), read-only                                                  read S
    torch_zero  dst.zero_(), write-only                                               write S

Each item is timed with CUDA events over --iters back-to-back launches after a warm-up; the line
gives the HBM bytes the item needs (from the shapes), the time per launch and that traffic's share
of the H100 SXM data sheet's 3.35 TB/s.  The order of the items alternates between rounds, so the
spread between rounds shows drift as well as noise.  torch is a measuring stick here only; it is
never on the library's path.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_PEAK_GBS = 3350.0  # H100 SXM HBM3, data sheet


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        out = "nvidia-smi failed: %s" % e
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="%d,%d" % (256 << 20, 1 << 30), help="bytes, comma separated")
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the lines as JSON here")
    args = ap.parse_args()
    sizes = [int(s) for s in args.sizes.split(",") if s]
    if args.iters < 200:
        ap.error("--iters must be at least 200")
    os.environ.setdefault("B200MPI_HEAP_BYTES", str(2 * max(sizes) + (768 << 20)))

    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this script measures the GPU and has no CPU fallback")
    import mpi_b200 as mpi
    from mpi_b200 import _lib as L
    lib = L.load()
    mpi.api._reset_for_tests(mpi.Cuda(Gpu=0))
    mpi.Init()
    info = card()
    print("# card: %s" % info, flush=True)
    rows = []
    try:
        for S in sizes:
            count = S // 4
            send = mpi.Alloc(count, np.float32)
            recv = mpi.Alloc(count, np.float32)
            tsrc = torch.rand(count, device="cuda", dtype=torch.float32)
            tdst = torch.empty_like(tsrc)

            def lib_item():
                def step():
                    if lib.b200mpi_allreduce_async(send.ptr, recv.ptr, count, L.F32, L.SUM):
                        raise RuntimeError(L.last_error())
                for _ in range(args.warmup):
                    step()
                if lib.b200mpi_stream_sync():
                    raise RuntimeError(L.last_error())
                ms = ctypes.c_float(0)
                lib.b200mpi_timer_start()
                for _ in range(args.iters):
                    step()
                if lib.b200mpi_timer_stop(ctypes.byref(ms)):
                    raise RuntimeError(L.last_error())
                return ms.value / args.iters

            def torch_item(fn):
                def run():
                    for _ in range(args.warmup):
                        fn()
                    torch.cuda.synchronize()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(args.iters):
                        fn()
                    e1.record()
                    e1.synchronize()
                    return e0.elapsed_time(e1) / args.iters
                return run

            items = [("allreduce", 2 * S, lib_item), ("torch_copy", 2 * S, torch_item(lambda: tdst.copy_(tsrc))),
                     ("torch_sum", S, torch_item(lambda: tsrc.sum())), ("torch_zero", S, torch_item(lambda: tdst.zero_()))]
            for rnd in range(args.rounds):
                for name, hbm, fn in (items if rnd % 2 == 0 else items[::-1]):
                    ms = fn()
                    row = {"round": rnd, "bytes": S, "item": name, "hbm_bytes": hbm, "ms": ms,
                           "hbm_gbs": hbm / (ms * 1e-3) / 1e9, "algbw_gbs": S / (ms * 1e-3) / 1e9,
                           "of_peak": hbm / (ms * 1e-3) / 1e9 / HBM_PEAK_GBS, "card": info}
                    rows.append(row)
                    print("%-10s S=%-11d round %d  %8.4f ms  hbm %7.1f GB/s  algbw %7.1f GB/s  %.3f of 3.35 TB/s"
                          % (name, S, rnd, ms, row["hbm_gbs"], row["algbw_gbs"], row["of_peak"]), flush=True)
            send.free()
            recv.free()
            del tsrc, tdst
            torch.cuda.empty_cache()
    finally:
        mpi.Finalize()
    if args.out:
        with open(args.out, "w") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
