"""Launch a world of N rank processes the way mpirun/gompirun does (one process per rank, the two
-mpi-* flags appended after the program's own arguments; /root/reference/mpirun/gompirun/gompirun.go:77-89)
and collect what each rank reports."""
import json
import os
import socket
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "_worker.py")


def free_ports(n):
    """n consecutive free TCP ports with the same number of digits (sorted order == rank order).
    Every one of them is bound once here, so a port some other process holds is never handed out."""
    for _ in range(400):
        s = socket.socket()
        s.bind(("127.0.0.1", 0))
        base = s.getsockname()[1]
        s.close()
        if not (20000 <= base <= 60000 - n):
            continue
        held = []
        try:
            for i in range(n):
                t = socket.socket()
                t.setsockopt(socket.SOL_SOCKET, socket.SO_REUSEADDR, 1)
                t.bind(("127.0.0.1", base + i))
                held.append(t)
        except OSError:
            continue
        finally:
            for t in held:
                t.close()
        if len(held) == n:
            return [base + i for i in range(n)]
    raise RuntimeError("no run of %d free ports found" % n)


def run_world(n, scenario, args=(), env=None, timeout=600, gpus_shared=True, extra_flags=(), per_rank_env=None, worker=None):
    """worker: the rank program (default WORKER, _worker.py)."""
    ports = free_ports(n)
    addrs = ["127.0.0.1:%d" % p for p in ports]
    procs = []
    outs = []
    e = dict(os.environ)
    e.setdefault("B200MPI_HEAP_BYTES", str(256 << 20))
    e["PYTHONPATH"] = ROOT + os.pathsep + e.get("PYTHONPATH", "")
    if env:
        e.update(env)
    for r in range(n):
        out = tempfile.NamedTemporaryFile("w+", suffix=".rank%d.json" % r, delete=False)
        outs.append(out.name)
        out.close()
        er = dict(e)
        if per_rank_env:
            er.update(per_rank_env(r))
        cmd = [sys.executable, worker or WORKER, scenario, "--out", outs[r]] + list(args) + list(extra_flags) + [
            "-mpi-addr", addrs[r], "-mpi-alladdr", ",".join(addrs), "-mpi-inittimeout", "60s"]
        procs.append(subprocess.Popen(cmd, env=er, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    # A rank that fails leaves its peers blocked in a collective: give them a short grace period,
    # then stop the world (exact PIDs we started, never by pattern).
    import time
    deadline = time.time() + timeout
    first_fail = None
    while True:
        codes = [p.poll() for p in procs]
        if all(c is not None for c in codes):
            break
        now = time.time()
        if first_fail is None and any(c not in (None, 0) for c in codes):
            first_fail = now
        if now > deadline or (first_fail is not None and now - first_fail > 5.0):
            for p in procs:
                if p.poll() is None:
                    p.kill()
            break
        time.sleep(0.05)
    results = []
    for r, p in enumerate(procs):
        log, _ = p.communicate()
        if p.returncode is not None and p.returncode < 0:
            log += "\n[launcher] killed (timeout %ss or a peer failed)" % timeout
        try:
            with open(outs[r]) as f:
                res = json.load(f)
        except Exception:
            res = {"ok": False, "error": "no result file"}
        res["rank"] = r
        res["returncode"] = p.returncode
        res["log"] = log
        results.append(res)
        os.unlink(outs[r])
    return results


def assert_world_ok(results):
    bad = [r for r in results if not r.get("ok") or r.get("returncode") != 0]
    if bad:
        msg = []
        for r in bad:
            msg.append("rank %s rc=%s error=%s\n%s" % (r.get("rank"), r.get("returncode"), r.get("error"), (r.get("log") or "")[-3000:]))
        raise AssertionError("\n".join(msg))
