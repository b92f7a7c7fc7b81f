#!/usr/bin/env python
"""Size x algorithm sweep of every collective and of Send/Receive (SURVEY.md 8(d) tables).

Run one process per rank, either under torchrun or under the gompirun-style launcher:
    python -m torch.distributed.run --nproc-per-node N tools/sweep.py [--out FILE]
    python -m mpi_b200.launcher N tools/sweep.py [--out FILE]
Rank 0 appends one JSON line per (collective, algorithm, size) to --out (default
gpurun_out/sweep_n<N>.jsonl).  Device-resident heap buffers; time = CUDA events on the library
stream over back-to-back launches, max over ranks; `t_call_us` = wall clock of one blocking call.
busbw conventions as nccl-tests (allreduce 2(n-1)/n, allgather (n-1)/n of the total, bcast 1).
Inputs are rank-constant (x_r[i] = r+1) so every result is verified exactly in O(1) reads.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

import bench  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--max-bytes", type=int, default=1 << 30)
    ap.add_argument("--min-bytes", type=int, default=1 << 10)
    ap.add_argument("--colls", default="allreduce,bcast,allgather,p2p")
    ap.add_argument("--algos", default="oneshot,twoshot,ring,nvls,smem")
    ap.add_argument("--blocks", default="")
    ap.add_argument("--params", default="", help="name=value;name=value passed to b200mpi_set_param")
    ap.add_argument("--tag", default="")
    ap.add_argument("--param-sets", default="", help="a=1,b=2|a=3,b=4 : the allreduce sweep is repeated for every set")
    ap.add_argument("--sizes", default="", help="explicit byte sizes, comma separated")
    args, rest = ap.parse_known_args()
    if "RANK" in os.environ:
        rank, world, local, addr, addrs = bench.world_from_env(None)
        gpu = local
    else:
        sys.argv = [sys.argv[0]] + rest
        rank = world = None
        addr, addrs, gpu = "", [], None
    os.environ.setdefault("B200MPI_HEAP_BYTES", str(3 * args.max_bytes + (512 << 20)))
    import mpi_b200 as mpi
    from mpi_b200 import _lib as L
    lib = L.load()
    mpi.api._reset_for_tests(mpi.Cuda(Addr=addr, Addrs=addrs, Timeout=120 * 10**9, Gpu=gpu))
    mpi.Init()
    rank, n = mpi.Rank(), mpi.Size()
    out_path = args.out or os.path.join(ROOT, "gpurun_out", "sweep_n%d.jsonl" % n)
    if rank == 0:
        os.makedirs(os.path.dirname(out_path), exist_ok=True)
    info = (ctypes.c_size_t(), ctypes.c_size_t(), ctypes.c_int())
    lib.b200mpi_heap_info(ctypes.byref(info[0]), ctypes.byref(info[1]), ctypes.byref(info[2]))
    nvls = bool(info[2].value)
    params = {}
    for kv in [x for x in args.params.split(";") if x]:
        k, v = kv.split("=")
        params[k] = int(v)
        if lib.b200mpi_set_param(k.encode(), int(v)):
            raise RuntimeError(L.last_error())
    ALGOS = {"auto": 0, "oneshot": 1, "twoshot": 2, "ring": 3, "nvls": 4, "smem": 5, "ll": 6, "hybrid": 7}

    def emit(d):
        if rank == 0:
            d.update({"n": n, "nvls_available": nvls, "params": params, "tag": args.tag})
            with open(out_path, "a") as f:
                f.write(json.dumps(d) + "\n")
            print(json.dumps(d), flush=True)

    def maxr(v):
        a = np.array([v], dtype=np.float64)
        o = np.zeros(1, dtype=np.float64)
        mpi.Allreduce(a, o, mpi.MAX)
        return float(o[0])

    def timed(fn_async, iters, warm):
        for _ in range(warm):
            fn_async()
        if lib.b200mpi_stream_sync():
            raise RuntimeError(L.last_error())
        mpi.Barrier()
        ms = ctypes.c_float()
        lib.b200mpi_timer_start()
        for _ in range(iters):
            fn_async()
        if lib.b200mpi_timer_stop(ctypes.byref(ms)):
            raise RuntimeError(L.last_error())
        return maxr(ms.value * 1e-3 / iters)

    def iters_for(b):
        return (50, 10) if b <= (1 << 20) else (20, 5) if b <= (64 << 20) else (8, 3)

    sizes = []
    b = args.min_bytes
    while b <= args.max_bytes:
        sizes.append(b)
        b *= 2
    if args.sizes:
        sizes = [int(x) for x in args.sizes.split(",")]
    param_sets = [dict((kv.split("=")[0], int(kv.split("=")[1])) for kv in ps.split(",") if kv) for ps in args.param_sets.split("|") if ps] or [{}]
    colls = args.colls.split(",")
    maxc = args.max_bytes // 4
    blocks_list = [int(x) for x in args.blocks.split(",") if x] or [0]

    if "allreduce" in colls:
        send = mpi.Alloc(maxc, np.float32).copy_from_host(np.full(maxc, rank + 1, dtype=np.float32))
        recv = mpi.Alloc(maxc, np.float32)
        want = np.float32(n * (n + 1) // 2)
        for ps in param_sets:
          for k, v in ps.items():
            params[k] = v
            if lib.b200mpi_set_param(k.encode(), int(v)):
                raise RuntimeError(L.last_error())
          for algo in args.algos.split(","):
              if algo in ("nvls", "hybrid") and not nvls:
                  continue
              if n == 1 and algo != "twoshot":
                  continue
              lib.b200mpi_set_algo(L.COLL_ALLREDUCE, ALGOS[algo])
              for nb in blocks_list:
                  lib.b200mpi_set_max_blocks(nb)
                  for S in sizes:
                      if algo == "oneshot" and S > (8 << 20):
                          continue
                      if algo == "ll" and S > (256 << 10):
                          continue
                      if algo == "hybrid" and S < (1 << 20):
                          continue
                      cnt = S // 4
                      it, wm = iters_for(S)
                      t = timed(lambda: lib.b200mpi_allreduce_async(send.ptr, recv.ptr, cnt, L.F32, L.SUM), it, wm)
                      t0 = time.perf_counter()
                      for _ in range(5):
                          lib.b200mpi_allreduce(send.ptr, recv.ptr, cnt, L.F32, L.SUM, L.DEVICE)
                      tc = maxr((time.perf_counter() - t0) / 5)
                      probe = np.concatenate([recv[:min(cnt, 64)].to_host(), recv[max(cnt - 64, 0):cnt].to_host(), recv[cnt // 2:cnt // 2 + 1].to_host()])
                      ok = bool(np.all(probe == want))
                      emit({"coll": "allreduce", "dtype": "f32", "algo": algo, "bytes": S, "t_us": t * 1e6, "t_call_us": tc * 1e6,
                            "algbw_gbs": S / t / 1e9, "busbw_gbs": S / t / 1e9 * (2 * (n - 1) / n if n > 1 else 1), "ok": ok, "max_blocks": nb, "pset": dict(ps),
                            "algo_used": L.ALGO_NAMES.get(lib.b200mpi_get_algo(L.COLL_ALLREDUCE, cnt, L.F32))})
        lib.b200mpi_set_algo(L.COLL_ALLREDUCE, 0)
        lib.b200mpi_set_max_blocks(0)
        send.free()
        recv.free()

    if "link" in colls and n > 1:
        # raw NVLink rates of the copy kernel between neighbours: the roofline of the P2P collectives
        names = {0: "all ranks pull from rank+1", 1: "all ranks push to rank+1", 2: "rank 0 pulls from rank 1 (one direction busy)",
                 3: "rank 0 pushes to rank 1 (one direction busy)", 4: "all ranks pull and push at once"}
        for S in (64 << 20, 256 << 20):
            for mode in range(5):
                ms = ctypes.c_float()
                if lib.b200mpi_link_probe(S, mode, 10, ctypes.byref(ms)):
                    raise RuntimeError(L.last_error())
                t = maxr(ms.value * 1e-3)
                per_dir = (2 if mode == 4 else 1) * S / t / 1e9 if t > 0 else 0.0
                emit({"coll": "link", "algo": names[mode], "mode": mode, "bytes": S, "t_us": t * 1e6, "gbs_per_direction": per_dir, "busbw_gbs": per_dir, "ok": True})

    if "latency" in colls and n > 1:
        # blocking-call latency of small Allreduce (what a Go caller sees per call): device-resident and
        # pinned-host buffers, every algorithm incl. the experimental LL path; median of 200 calls
        hin, hout = ctypes.c_void_p(), ctypes.c_void_p()
        lib.b200mpi_host_alloc(1 << 16, ctypes.byref(hin))
        lib.b200mpi_host_alloc(1 << 16, ctypes.byref(hout))
        ctypes.memset(hin.value, 0, 1 << 16)
        dsend = mpi.Alloc(1 << 14, np.float32).copy_from_host(np.full(1 << 14, rank + 1, dtype=np.float32))
        drecv = mpi.Alloc(1 << 14, np.float32)
        for algo in ("auto", "oneshot", "twoshot", "nvls", "ll"):
            if algo == "nvls" and not nvls:
                continue
            lib.b200mpi_set_algo(L.COLL_ALLREDUCE, ALGOS[algo])
            for S in (8, 1024, 32768):
                cnt = S // 4
                for kind, sp, rp, mk in (("device", dsend.ptr, drecv.ptr, L.DEVICE), ("host", hin, hout, L.HOST)):
                    ts = []
                    for i in range(220):
                        mpi.Barrier() if i % 50 == 0 else None
                        t0 = time.perf_counter()
                        rc = lib.b200mpi_allreduce(sp, rp, cnt, L.F32, L.SUM, mk)
                        ts.append(time.perf_counter() - t0)
                        if rc:
                            raise RuntimeError(L.last_error())
                    ts = sorted(ts[20:])
                    emit({"coll": "latency", "dtype": "f32", "algo": algo, "kind": kind, "bytes": S, "t_call_us_median": maxr(ts[len(ts) // 2]) * 1e6,
                          "t_call_us_p10": maxr(ts[len(ts) // 10]) * 1e6, "t_us": maxr(ts[len(ts) // 2]) * 1e6, "busbw_gbs": 0.0, "ok": True})
        lib.b200mpi_set_algo(L.COLL_ALLREDUCE, 0)
        lib.b200mpi_host_free(hin)
        lib.b200mpi_host_free(hout)
        dsend.free()
        drecv.free()

    if "bcast" in colls and n > 1:
        buf = mpi.Alloc(maxc, np.float32)
        for algo in ("oneshot", "twoshot", "nvls", "nvls_root"):
            if algo.startswith("nvls") and not nvls:
                continue
            lib.b200mpi_set_param(b"bcast_nvls2", 0 if algo == "nvls_root" else 1)
            lib.b200mpi_set_algo(L.COLL_BCAST, ALGOS["nvls" if algo == "nvls_root" else algo])
            for S in sizes:
                if algo == "oneshot" and S > (64 << 20):
                    continue
                cnt = S // 4
                buf[:cnt].copy_from_host(np.full(cnt, 7.0 if rank == 0 else -1.0, dtype=np.float32)) if S <= (64 << 20) else None
                it, wm = iters_for(S)
                t = timed(lambda: lib.b200mpi_bcast_async(buf.ptr, cnt, L.F32, 0), it, wm)
                probe = np.concatenate([buf[:min(cnt, 64)].to_host(), buf[max(cnt - 64, 0):cnt].to_host()])
                ok = bool(np.all(probe == 7.0)) if S <= (64 << 20) else None
                emit({"coll": "bcast", "dtype": "f32", "algo": algo, "bytes": S, "t_us": t * 1e6, "algbw_gbs": S / t / 1e9, "busbw_gbs": S / t / 1e9, "ok": ok})
        lib.b200mpi_set_algo(L.COLL_BCAST, 0)
        buf.free()

    if "allgather" in colls and n > 1:
        per_max = min(args.max_bytes // n, 128 << 20)
        send = mpi.Alloc(per_max // 8, np.int64).copy_from_host(np.full(per_max // 8, rank + 1, dtype=np.int64))
        recv = mpi.Alloc(per_max // 8 * n, np.int64)
        for algo in ("oneshot", "ring", "nvls"):
            if algo == "nvls" and not nvls:
                continue
            lib.b200mpi_set_algo(L.COLL_ALLGATHER, ALGOS[algo])
            for S in [s for s in sizes if s <= per_max] + [1000000 * 8]:
                if S > per_max:
                    continue
                cnt = S // 8
                it, wm = iters_for(S * n)
                t = timed(lambda: lib.b200mpi_allgather_async(send.ptr, recv.ptr, cnt, L.I64), it, wm)
                got = recv[:cnt * n].to_host() if S * n <= (64 << 20) else None
                ok = bool(all(np.all(got[r * cnt:(r + 1) * cnt] == r + 1) for r in range(n))) if got is not None else None
                tot = S * n
                emit({"coll": "allgather", "dtype": "i64", "algo": "push" if algo == "oneshot" else algo, "bytes_per_rank": S, "bytes": tot, "t_us": t * 1e6,
                      "algbw_gbs": tot / t / 1e9, "busbw_gbs": tot / t / 1e9 * (n - 1) / n, "ok": ok})
        lib.b200mpi_set_algo(L.COLL_ALLGATHER, 0)
        send.free()
        recv.free()

    rooted = [c for c in ("gather", "scatter", "allgatherv") if c in colls]
    if rooted and n > 1:
        # One algorithm each, blocking calls only: time = events around back-to-back calls, max over
        # ranks.  Roofline: the busiest NVLink direction of any GPU (root's ingress for Gather, its
        # egress for Scatter, for Allgatherv the larger of a rank's egress (n-1)*c_r and its
        # ingress total-c_r) at 450 GB/s per direction (H100 SXM data sheet).
        per_max = min(args.max_bytes // n, 128 << 20)
        big = mpi.Alloc(per_max // 4 * n, np.float32)
        small = mpi.Alloc(per_max // 4, np.float32).copy_from_host(np.full(per_max // 4, rank + 1, dtype=np.float32))
        link = 450e9
        for coll in rooted:
            shapes = ("uniform", "skewed") if coll == "allgatherv" else ("uniform",)
            for shape in shapes:
                for S in [s for s in sizes if 4 * n <= s <= per_max]:
                    cnt = S // 4  # elements per rank (uniform); skewed: rank n-1 carries half of n*cnt
                    counts = [cnt] * n if shape == "uniform" else [cnt * n // (2 * (n - 1))] * (n - 1) + [cnt * n - cnt * n // (2 * (n - 1)) * (n - 1)]
                    if max(counts) > per_max // 4:
                        continue
                    total = sum(counts)
                    tab = (ctypes.c_size_t * n)(*counts)
                    if coll == "gather":
                        call = lambda: lib.b200mpi_gather(small.ptr, big.ptr, cnt, L.F32, 0, L.DEVICE)  # noqa: E731
                        link_bytes = max(total - counts[0], max(counts))
                    elif coll == "scatter":
                        call = lambda: lib.b200mpi_scatter(big.ptr, small.ptr, cnt, L.F32, 0, L.DEVICE)  # noqa: E731
                        link_bytes = max(total - counts[0], max(counts))
                    else:
                        call = lambda: lib.b200mpi_allgatherv(small.ptr, big.ptr, tab, L.F32, L.DEVICE)  # noqa: E731
                        link_bytes = max(max(c * (n - 1), total - c) for c in counts)
                    if coll == "scatter" and rank == 0:
                        big[:total].copy_from_host(np.repeat(np.arange(1, n + 1, dtype=np.float32), cnt))
                    it, wm = iters_for(total * 4)

                    def blocking():
                        if call():
                            raise RuntimeError(L.last_error())
                    t = timed(blocking, it, wm)
                    ok = True  # checked where this rank's recv was written, up to 64 MiB
                    if coll == "scatter":
                        ok = cnt > (16 << 20) or bool(np.all(small[:cnt].to_host() == rank + 1))
                    elif coll == "allgatherv" or rank == 0:
                        ok = total > (16 << 20) or bool(np.array_equal(big[:total].to_host(), np.repeat(np.arange(1, n + 1, dtype=np.float32), counts)))
                    ok = maxr(0.0 if ok else 1.0) == 0.0
                    emit({"coll": coll, "dtype": "f32", "algo": shape, "root": 0 if coll != "allgatherv" else None, "counts": counts, "bytes": total * 4,
                          "t_us": t * 1e6, "algbw_gbs": total * 4 / t / 1e9, "link_bytes": link_bytes * 4,
                          "link_roofline_share": link_bytes * 4 / link / t, "ok": ok})
        big.free()
        small.free()

    exchange = [c for c in ("alltoall", "alltoallv") if c in colls]
    if exchange and n > 1:
        # S = bytes of every rank's send.  Alltoallv runs a uniform table and a skewed one (half of
        # every rank's send to its right neighbour, the rest evenly to the others).  Roofline per GPU:
        # the larger of its egress sum_{j!=i} S_i[j] and its ingress sum_{k!=i} R_i[k], the busiest GPU
        # over 450 GB/s per direction (H100 SXM data sheet).  Block (i -> j) holds i*n + j + 1.
        per_max = min(args.max_bytes, 512 << 20)
        sbuf = mpi.Alloc(per_max // 4, np.float32)
        rbuf = mpi.Alloc(per_max // 4, np.float32)
        link = 450e9
        for coll in exchange:
            shapes = ("uniform", "skewed") if coll == "alltoallv" else ("uniform",)
            for shape in shapes:
                for S in [s for s in sizes if 4 * n <= s <= per_max // 2]:
                    cnt = S // 4 // n
                    if shape == "uniform":
                        m = [[cnt] * n for _ in range(n)]
                    else:
                        half, rest = cnt * n // 2, (cnt * n - cnt * n // 2) // (n - 1)
                        m = [[half if j == (i + 1) % n else rest for j in range(n)] for i in range(n)]
                    scounts, rcounts = m[rank], [m[k][rank] for k in range(n)]
                    sbuf[:sum(scounts)].copy_from_host(np.repeat(np.arange(rank * n + 1, rank * n + n + 1, dtype=np.float32), scounts))
                    stab, rtab = (ctypes.c_size_t * n)(*scounts), (ctypes.c_size_t * n)(*rcounts)
                    if coll == "alltoall":
                        call = lambda: lib.b200mpi_alltoall(sbuf.ptr, rbuf.ptr, cnt, L.F32, L.DEVICE)  # noqa: E731
                    else:
                        call = lambda: lib.b200mpi_alltoallv(sbuf.ptr, stab, rbuf.ptr, rtab, L.F32, L.DEVICE)  # noqa: E731
                    link_bytes = max(max(sum(m[i]) - m[i][i], sum(m[k][i] for k in range(n)) - m[i][i]) for i in range(n))
                    it, wm = iters_for(S)

                    def blocking():
                        if call():
                            raise RuntimeError(L.last_error())
                    t = timed(blocking, it, wm)
                    want = np.repeat(np.arange(n, dtype=np.float32) * n + rank + 1, rcounts)
                    ok = sum(rcounts) * 4 > (64 << 20) or bool(np.array_equal(rbuf[:sum(rcounts)].to_host(), want))
                    ok = maxr(0.0 if ok else 1.0) == 0.0
                    emit({"coll": coll, "dtype": "f32", "algo": shape, "counts": scounts, "bytes": sum(scounts) * 4,
                          "t_us": t * 1e6, "algbw_gbs": sum(scounts) * 4 / t / 1e9, "link_bytes": link_bytes * 4,
                          "link_roofline_share": link_bytes * 4 / link / t, "ok": ok})
        sbuf.free()
        rbuf.free()

    prefix = [c for c in ("scan", "exscan") if c in colls]
    if prefix:
        # One algorithm, blocking calls: time = events around back-to-back calls, max over ranks.  Both
        # move the bytes of a two-shot Allreduce of the same size: per GPU (n-1)/n*S read from peers and
        # (n-1)/n*S pushed to them, so the bound is 2(n-1)/n*S at 450 GB/s per direction (H100 SXM data
        # sheet), and a two-shot Allreduce of the same size is timed in the same run next to each.
        if n < 2 or L.get_param("shared_device"):
            emit({"coll": "scan", "ok": True, "note": "fewer than two NVLink-connected GPUs (ranks %s): Scan / Exscan bandwidth not measured"
                  % ("share one GPU" if n > 1 else "= 1")})
        else:
            per_max = min(args.max_bytes, 512 << 20)
            send = mpi.Alloc(per_max // 4, np.float32).copy_from_host(np.full(per_max // 4, rank + 1, dtype=np.float32))
            recv = mpi.Alloc(per_max // 4, np.float32)
            link = 450e9
            lib.b200mpi_set_algo(L.COLL_ALLREDUCE, ALGOS["twoshot"])
            for S in [s for s in sizes if s <= per_max]:
                cnt = S // 4
                it, wm = iters_for(S)
                bound = 2 * (n - 1) / n * S / link
                t_ar = timed(lambda: lib.b200mpi_allreduce_async(send.ptr, recv.ptr, cnt, L.F32, L.SUM), it, wm)
                for coll in prefix:
                    fn = lib.b200mpi_exscan if coll == "exscan" else lib.b200mpi_scan

                    def blocking():
                        if fn(send.ptr, recv.ptr, cnt, L.F32, L.SUM, L.DEVICE):
                            raise RuntimeError(L.last_error())
                    recv[:min(cnt, 64)].copy_from_host(np.full(min(cnt, 64), -1, dtype=np.float32))
                    t = timed(blocking, it, wm)
                    # x_r = r + 1: rank r holds (r+1)(r+2)/2 after Scan, r(r+1)/2 after Exscan (rank 0: untouched)
                    k = rank if coll == "exscan" else rank + 1
                    want = np.float32(k * (k + 1) // 2) if k else np.float32(-1)
                    probe = recv[:min(cnt, 64)].to_host()
                    ok = maxr(0.0 if bool(np.all(probe == want)) else 1.0) == 0.0
                    emit({"coll": coll, "dtype": "f32", "algo": "owner", "bytes": S, "t_us": t * 1e6, "algbw_gbs": S / t / 1e9,
                          "link_bytes": 2 * (n - 1) / n * S, "link_roofline_share": bound / t,
                          "twoshot_allreduce_t_us": t_ar * 1e6, "vs_twoshot_allreduce": t_ar / t, "ok": ok})
            lib.b200mpi_set_algo(L.COLL_ALLREDUCE, 0)
            send.free()
            recv.free()

    if "reduce_scatterv" in colls:
        # One algorithm, blocking calls: time = events around back-to-back calls, max over ranks.  S =
        # bytes of every rank's send.  Three tables: uniform (timed next to the P2P ReduceScatter of the
        # same size), a balanced split of an indivisible count, and a skewed one (rank 0 holds half).
        # Rank j reads its block c_j from n-1 peers and n-1 peers read theirs from it, so the per-GPU
        # bound is the larger of ingress (n-1)*c_j and egress total - c_j, the busiest GPU over 450 GB/s
        # per direction (H100 SXM data sheet).  x_r = r + 1, so every result element is n(n+1)/2.
        if n < 2 or L.get_param("shared_device"):
            emit({"coll": "reduce_scatterv", "ok": True, "note": "fewer than two NVLink-connected GPUs (ranks %s): ReduceScatterv bandwidth not measured"
                  % ("share one GPU" if n > 1 else "= 1")})
        else:
            per_max = min(args.max_bytes, 512 << 20)
            send = mpi.Alloc(per_max // 4 + n, np.float32).copy_from_host(np.full(per_max // 4 + n, rank + 1, dtype=np.float32))
            recv = mpi.Alloc(per_max // 4 + n, np.float32)
            link = 450e9
            want = np.float32(n * (n + 1) // 2)
            lib.b200mpi_set_algo(L.COLL_REDUCE_SCATTER, ALGOS["twoshot"])
            for S in [s for s in sizes if 4 * n <= s <= per_max]:
                cnt = S // 4 // n
                odd = cnt * n + 1  # not a multiple of n
                tables = {"uniform": [cnt] * n,
                          "balanced": [odd // n + (1 if r < odd % n else 0) for r in range(n)],
                          "skewed": [cnt * n // 2] + [(cnt * n - cnt * n // 2) // (n - 1)] * (n - 1)}
                it, wm = iters_for(S)
                t_rs = timed(lambda: lib.b200mpi_reduce_scatter_async(send.ptr, recv.ptr, cnt, L.F32, L.SUM), it, wm)
                for shape, counts in tables.items():
                    total = sum(counts)
                    tab = (ctypes.c_size_t * n)(*counts)

                    def blocking():
                        if lib.b200mpi_reduce_scatterv(send.ptr, recv.ptr, tab, L.F32, L.SUM, L.DEVICE):
                            raise RuntimeError(L.last_error())
                    k = min(counts[rank], 64)
                    recv[:k].copy_from_host(np.full(k, -1, dtype=np.float32))
                    t = timed(blocking, it, wm)
                    ok = maxr(0.0 if bool(np.all(recv[:k].to_host() == want)) else 1.0) == 0.0
                    link_bytes = 4 * max(max((n - 1) * c, total - c) for c in counts)
                    row = {"coll": "reduce_scatterv", "dtype": "f32", "algo": shape, "counts": counts, "bytes": total * 4, "t_us": t * 1e6,
                           "algbw_gbs": total * 4 / t / 1e9, "link_bytes": link_bytes, "link_roofline_share": link_bytes / link / t, "ok": ok}
                    if shape == "uniform":
                        row.update({"reduce_scatter_t_us": t_rs * 1e6, "vs_reduce_scatter": t_rs / t})
                    emit(row)
            lib.b200mpi_set_algo(L.COLL_REDUCE_SCATTER, 0)
            send.free()
            recv.free()

    if "allreduce_loc" in colls:
        # MAXLOC / MINLOC, one algorithm (the two-shot body over 16-byte pairs).  Two numbers:
        # - the blocking-call latency of one pair (median of 200 calls, max over ranks) next to a 16-byte
        #   Allreduce under AUTO (the LL path) and under forced one-shot: whether pairs need a latency path;
        # - 64 MiB of pairs per rank as a share of the two-shot link bound 2(n-1)/n*S at 450 GB/s per
        #   direction (H100 SXM data sheet), time = events around back-to-back blocking calls.
        # x_r = (r, loc r): MAXLOC ends on (n-1, n-1) everywhere.
        if n < 2 or L.get_param("shared_device"):
            emit({"coll": "allreduce_loc", "ok": True, "note": "fewer than two NVLink-connected GPUs (ranks %s): AllreduceLoc not measured"
                  % ("share one GPU" if n > 1 else "= 1")})
        else:
            big = (64 << 20) // 16
            pairs = np.zeros(big, dtype=mpi.LOC_F64)
            pairs["val"], pairs["loc"] = rank, rank
            send = mpi.Alloc(big, mpi.LOC_F64).copy_from_host(pairs)
            recv = mpi.Alloc(big, mpi.LOC_F64)
            plain = mpi.Alloc(4, np.float32).copy_from_host(np.full(4, rank + 1, dtype=np.float32))
            plain_out = mpi.Alloc(4, np.float32)

            def median_call(call):
                ts = []
                for i in range(220):
                    mpi.Barrier() if i % 50 == 0 else None
                    t0 = time.perf_counter()
                    if call():
                        raise RuntimeError(L.last_error())
                    ts.append(time.perf_counter() - t0)
                return maxr(sorted(ts[20:])[100])
            row = {"coll": "allreduce_loc", "dtype": "f64", "algo": "twoshot", "bytes": 16,
                   "t_call_us_median": median_call(lambda: lib.b200mpi_allreduce_loc(send.ptr, recv.ptr, 1, L.F64, L.MAX, L.DEVICE)) * 1e6}
            for algo in ("auto", "oneshot"):
                lib.b200mpi_set_algo(L.COLL_ALLREDUCE, ALGOS[algo])
                row["allreduce_16B_%s_t_call_us_median" % algo] = median_call(
                    lambda: lib.b200mpi_allreduce(plain.ptr, plain_out.ptr, 4, L.F32, L.MAX, L.DEVICE)) * 1e6
            lib.b200mpi_set_algo(L.COLL_ALLREDUCE, 0)
            row["ok"] = maxr(0.0 if recv[:1].to_host()["loc"][0] == n - 1 else 1.0) == 0.0
            emit(row)
            S = big * 16

            def blocking():
                if lib.b200mpi_allreduce_loc(send.ptr, recv.ptr, big, L.F64, L.MAX, L.DEVICE):
                    raise RuntimeError(L.last_error())
            it, wm = iters_for(S)
            t = timed(blocking, it, wm)
            got = recv[:64].to_host()
            ok = maxr(0.0 if bool(np.all(got["loc"] == n - 1) and np.all(got["val"] == n - 1)) else 1.0) == 0.0
            bound = 2 * (n - 1) / n * S / 450e9
            emit({"coll": "allreduce_loc", "dtype": "f64", "algo": "twoshot", "bytes": S, "t_us": t * 1e6, "algbw_gbs": S / t / 1e9,
                  "link_bytes": 2 * (n - 1) / n * S, "link_roofline_share": bound / t, "ok": ok})
            for b in (send, recv, plain, plain_out):
                b.free()

    rma = [c for c in ("put", "get", "accumulate") if c in colls]
    if rma:
        # One-sided calls, blocking, heap origins, one window of max_bytes per rank; time = events around
        # back-to-back calls, max over ranks.  Put and Get move S one way between rank and rank + 1, so
        # every GPU sends (Put) or receives (Get) S: the bound is S over 450 GB/s per direction (H100 SXM
        # data sheet).  Also the blocking latency of one 8-byte Put (median of 200 calls), and f32, f64 and
        # i64 SUM Accumulate next to Put of the same size: uncontended (into rank + 1) and contended (every
        # rank into rank 0, whose ingress then carries (n-1)*S: that is the bound there).
        if n < 2 or L.get_param("shared_device"):
            emit({"coll": "rma", "ok": True, "note": "fewer than two NVLink-connected GPUs (ranks %s): Put, Get and Accumulate not measured"
                  % ("share one GPU" if n > 1 else "= 1")})
        else:
            per_max = min(args.max_bytes, 1 << 30)
            wmem = mpi.Alloc(per_max, np.uint8)
            # finite, normal origin values for every dtype read from it: f64 1.0, as f32 0.0 and 1.875
            org = mpi.Alloc(per_max // 8, np.float64).copy_from_host(np.ones(per_max // 8))
            w = mpi.WinCreate(wmem)
            nxt = (rank + 1) % n
            link = 450e9

            def rma_call(fn, *a):
                def call():
                    if fn(*a):
                        raise RuntimeError(L.last_error())
                return call
            ts = []
            for i in range(220):
                mpi.Barrier() if i % 50 == 0 else None
                t0 = time.perf_counter()
                rma_call(lib.b200mpi_put, org.ptr, 1, L.F64, nxt, 0, w.id, L.DEVICE)()
                ts.append(time.perf_counter() - t0)
            w.Fence()
            emit({"coll": "put", "dtype": "f64", "bytes": 8, "t_call_us_median": maxr(sorted(ts[20:])[100]) * 1e6, "ok": True})
            for S in [s for s in sizes if s <= per_max]:
                it, wm = iters_for(S)
                t_put = None
                for coll in [c for c in ("put", "get") if c in rma]:
                    fn = lib.b200mpi_put if coll == "put" else lib.b200mpi_get
                    t = timed(rma_call(fn, org.ptr, S, L.U8, nxt, 0, w.id, L.DEVICE), it, wm)
                    w.Fence()
                    t_put = t if coll == "put" else t_put
                    emit({"coll": coll, "dtype": "u8", "bytes": S, "t_us": t * 1e6, "algbw_gbs": S / t / 1e9,
                          "link_roofline_share": S / link / t, "ok": True})
                if "accumulate" in rma:
                    for dn, code, es in (("f32", L.F32, 4), ("f64", L.F64, 8), ("i64", L.I64, 8)):
                        for shape, target in (("uncontended", nxt), ("contended", 0)):
                            t = timed(rma_call(lib.b200mpi_accumulate, org.ptr, S // es, code, L.SUM, target, 0, w.id, L.DEVICE), it, wm)
                            w.Fence()
                            bound = S / link if shape == "uncontended" else (n - 1) * S / link
                            row = {"coll": "accumulate", "dtype": dn, "algo": shape, "bytes": S, "t_us": t * 1e6,
                                   "algbw_gbs": S / t / 1e9, "link_roofline_share": bound / t, "ok": True}
                            if t_put is not None:
                                row["vs_put"] = t_put / t
                            emit(row)
            w.Free()
            wmem.free()
            org.free()

    passive = [c for c in ("lock", "fetch_and_op", "get_accumulate") if c in colls]
    if passive:
        # Passive target, blocking calls on a window of rank + 1 (medians of 200 calls after 20, max over
        # ranks): an uncontended Lock + Unlock pair; one i64 Fetch_and_op SUM next to the 8-byte Put of the
        # same window; every rank's Fetch_and_op on rank 0's counter at once, as operations per second
        # over the world; and f64 Get_accumulate SUM of 64 MiB (heap origin and result) next to Accumulate.
        card = {}
        try:  # a read-only query: the numbers belong next to the card and its power limit
            q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(lib.b200mpi_device())],
                               capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
            card = {"gpu": q[0], "power_limit": q[1]} if len(q) == 2 else {}
        except (OSError, subprocess.SubprocessError):
            pass

        def pemit(d):
            emit(dict(d, **card))
        if n < 2 or L.get_param("shared_device"):
            pemit({"coll": "passive", "ok": True, "note": "fewer than two NVLink-connected GPUs (ranks %s): Lock, Fetch_and_op and "
                  "Get_accumulate not measured" % ("share one GPU" if n > 1 else "= 1")})
        else:
            S = 64 << 20
            wmem = mpi.Alloc(S // 8, np.float64).copy_from_host(np.zeros(S // 8))
            org = mpi.Alloc(S // 8, np.float64).copy_from_host(np.ones(S // 8))
            res = mpi.Alloc(S // 8, np.float64)
            w = mpi.WinCreate(wmem)
            nxt = (rank + 1) % n
            one = np.ones(1, dtype=np.int64)
            old = np.zeros(1, dtype=np.int64)

            def median_of(call):
                ts = []
                for i in range(220):
                    mpi.Barrier() if i % 50 == 0 else None
                    t0 = time.perf_counter()
                    if call():
                        raise RuntimeError(L.last_error())
                    ts.append(time.perf_counter() - t0)
                return maxr(sorted(ts[20:])[100])
            if "lock" in passive:
                t = median_of(lambda: lib.b200mpi_win_lock(L.LOCK_EXCLUSIVE, nxt, w.id) or lib.b200mpi_win_unlock(nxt, w.id))
                pemit({"coll": "lock", "algo": "exclusive_uncontended", "t_pair_us_median": t * 1e6, "ok": True})
            if "fetch_and_op" in passive:
                t = median_of(lambda: lib.b200mpi_fetch_and_op(one.ctypes.data, old.ctypes.data, L.I64, L.SUM, nxt, 0, w.id))
                t_put = median_of(lambda: lib.b200mpi_put(org.ptr, 1, L.F64, nxt, 1, w.id, L.DEVICE))
                pemit({"coll": "fetch_and_op", "dtype": "i64", "algo": "uncontended", "t_call_us_median": t * 1e6,
                      "put_8B_t_call_us_median": t_put * 1e6, "ok": True})
                mpi.Barrier()
                calls = 2000
                t0 = time.perf_counter()
                for _ in range(calls):
                    if lib.b200mpi_fetch_and_op(one.ctypes.data, old.ctypes.data, L.I64, L.SUM, 0, 2, w.id):
                        raise RuntimeError(L.last_error())
                dt = maxr(time.perf_counter() - t0)
                mpi.Barrier()
                final = np.zeros(1, dtype=np.int64)
                lib.b200mpi_fetch_and_op(None, final.ctypes.data, L.I64, L.NO_OP, 0, 2, w.id)
                pemit({"coll": "fetch_and_op", "dtype": "i64", "algo": "contended", "ops_per_s": n * calls / dt,
                      "ok": bool(final[0] == n * calls)})
            if "get_accumulate" in passive:
                it, wm = iters_for(S)

                def ga():
                    if lib.b200mpi_get_accumulate(org.ptr, res.ptr, S // 8, L.F64, L.SUM, nxt, 0, w.id, L.DEVICE):
                        raise RuntimeError(L.last_error())

                def acc():
                    if lib.b200mpi_accumulate(org.ptr, S // 8, L.F64, L.SUM, nxt, 0, w.id, L.DEVICE):
                        raise RuntimeError(L.last_error())
                t_ga = timed(ga, it, wm)
                t_acc = timed(acc, it, wm)
                pemit({"coll": "get_accumulate", "dtype": "f64", "bytes": S, "t_us": t_ga * 1e6, "algbw_gbs": S / t_ga / 1e9,
                      "accumulate_t_us": t_acc * 1e6, "vs_accumulate": t_acc / t_ga, "ok": True})
            w.Fence()
            w.Free()
            for b in (wmem, org, res):
                b.free()

    if "pscw" in colls:
        # One epoch of a ring neighbour exchange (medians of 200 epochs after 20, max over ranks): every
        # rank Posts to and Starts on {left, right}, Puts S bytes into each, then Completes and Waits;
        # beside it the same Puts closed by one win_fence.  S = 8 B and 1 MiB.
        card = {}
        try:  # a read-only query: the numbers belong next to the card and its power limit
            q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(lib.b200mpi_device())],
                               capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
            card = {"gpu": q[0], "power_limit": q[1]} if len(q) == 2 else {}
        except (OSError, subprocess.SubprocessError):
            pass
        if n < 2 or L.get_param("shared_device"):
            emit(dict({"coll": "pscw", "ok": True, "note": "fewer than two NVLink-connected GPUs (ranks %s): the PSCW and fence "
                       "neighbour-exchange epochs not measured" % ("share one GPU" if n > 1 else "= 1")}, **card))
        else:
            left, right = (rank - 1) % n, (rank + 1) % n
            nbrs = sorted({left, right})
            for S in (8, 1 << 20):
                e = S // 8
                wmem = mpi.Alloc(2 * e, np.float64).copy_from_host(np.zeros(2 * e))
                org = mpi.Alloc(e, np.float64).copy_from_host(np.full(e, rank + 1.0))
                w = mpi.WinCreate(wmem)

                def put_both():
                    # slot 0 of the right neighbour holds its left's data, slot 1 of the left its right's
                    for t, slot in ((right, 0), (left, 1)):
                        if lib.b200mpi_put(org.ptr, e, L.F64, t, slot * e, w.id, L.DEVICE):
                            raise RuntimeError(L.last_error())

                def pscw_epoch():
                    w.Post(nbrs)
                    w.Start(nbrs)
                    put_both()
                    w.Complete()
                    w.Wait()

                def fence_epoch():
                    put_both()
                    w.Fence()

                res = {}
                for name, epoch in (("pscw", pscw_epoch), ("fence", fence_epoch)):
                    mpi.Barrier()
                    ts = []
                    for i in range(220):
                        t0 = time.perf_counter()
                        epoch()
                        ts.append(time.perf_counter() - t0)
                    res[name] = maxr(sorted(ts[20:])[100])
                    w.Fence()
                    got = wmem.to_host()
                    ok = bool(np.all(got[:e] == left + 1.0) and np.all(got[e:] == right + 1.0))
                    res[name + "_ok"] = bool(maxr(0.0 if ok else 1.0) == 0.0)
                emit(dict({"coll": "pscw", "bytes": S, "t_epoch_us_median": res["pscw"] * 1e6,
                           "fence_t_epoch_us_median": res["fence"] * 1e6, "fence_over_pscw": res["fence"] / res["pscw"],
                           "ok": res["pscw_ok"] and res["fence_ok"]}, **card))
                w.Free()
                wmem.free()
                org.free()

    if "p2p" in colls and n > 1:
        # bounce (examples/bounce/bounce.go:85-138): even sends, odd returns; device-resident float64
        maxp = min(args.max_bytes, 256 << 20)
        msg = mpi.Alloc(maxp // 8, np.float64).copy_from_host(np.arange(maxp // 8, dtype=np.float64))
        rcv = mpi.Alloc(maxp // 8, np.float64)
        even = rank % 2 == 0
        peer = rank + 1 if even else rank - 1
        ladder = sorted(set([0, 8, 80, 800, 8000, 80000, 800000, 8000000, 1 << 20, 16 << 20, maxp]))
        for S in ladder:
            if peer >= n or S > maxp:
                continue
            cnt = S // 8
            reps = 100 if S <= (1 << 20) else 10
            for phase in range(2):  # 0 warm-up, 1 timed
                mpi.Barrier()
                t0 = time.perf_counter()
                for _ in range(reps if phase else 3):
                    if even:
                        mpi.Send(msg[:cnt], peer, 0)
                        mpi.Receive(rcv[:cnt], peer, 0)
                    else:
                        mpi.Receive(rcv[:cnt], peer, 0)
                        mpi.Send(rcv[:cnt], peer, 0)
                dt = (time.perf_counter() - t0) / reps
            dt = maxr(dt)
            ok = bool(np.array_equal(rcv[:min(cnt, 256)].to_host(), np.arange(min(cnt, 256), dtype=np.float64))) if cnt else True
            emit({"coll": "bounce", "dtype": "f64", "algo": "pull", "bytes": S, "round_trip_us": dt * 1e6, "algbw_gbs": (2 * S / dt / 1e9) if S else 0.0,
                  "busbw_gbs": (2 * S / dt / 1e9) if S else 0.0, "ok": ok, "reps": reps})
        # host-slice ping-pong at the headline 1 MiB float64 point (what an unmodified Go caller does)
        h = np.arange(131072, dtype=np.float64)
        hr = np.zeros(131072, dtype=np.float64)
        if peer < n:
            for phase in range(2):
                mpi.Barrier()
                t0 = time.perf_counter()
                for _ in range(20 if phase else 3):
                    if even:
                        mpi.Send(h, peer, 1)
                        hr = mpi.Receive(hr, peer, 1)
                    else:
                        hr = mpi.Receive(hr, peer, 1)
                        mpi.Send(hr, peer, 1)
                dt = (time.perf_counter() - t0) / 20
            dt = maxr(dt)
            emit({"coll": "bounce_host", "dtype": "f64", "algo": "staged", "bytes": 1 << 20, "round_trip_us": dt * 1e6, "ok": bool(np.array_equal(hr, h))})
        msg.free()
        rcv.free()
    mpi.Barrier()
    mpi.Finalize()


if __name__ == "__main__":
    main()
