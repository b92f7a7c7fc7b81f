#!/usr/bin/env python
"""Turn tools/sweep.py JSON lines into markdown tables (bus bandwidth GB/s and time us per size).

    python tools/report.py sweep_n8.jsonl [more.jsonl ...] [--coll allreduce]

One table per (file, collective): rows = message size, columns = algorithm (and parameter set / block
cap when a sweep varied them).  Values failing the sweep's own result check are marked with '!'.
"""
import argparse
import json
import sys


def load(path):
    with open(path) as f:
        return [json.loads(line) for line in f if line.strip()]


def column_key(r):
    key = r.get("algo", "?")
    ps = r.get("pset") or {}
    if ps:
        key += " " + ",".join("%s=%s" % kv for kv in sorted(ps.items()))
    if r.get("max_blocks"):
        key += " blocks=%d" % r["max_blocks"]
    if r.get("tag"):
        key += " [%s]" % r["tag"]
    return key


def table(rows, coll):
    rows = [r for r in rows if r.get("coll") == coll]
    if not rows:
        return None
    cols, sizes = [], []
    for r in rows:
        k = column_key(r)
        if k not in cols:
            cols.append(k)
        if r["bytes"] not in sizes:
            sizes.append(r["bytes"])
    sizes.sort()
    out = ["| bytes | " + " | ".join(cols) + " |", "|---|" + "---|" * len(cols)]
    for s in sizes:
        cells = []
        for k in cols:
            m = [r for r in rows if r["bytes"] == s and column_key(r) == k]
            if not m:
                cells.append("")
                continue
            r = m[-1]
            if "round_trip_us" in r:
                cells.append("%.1f us rt" % r["round_trip_us"])
            else:
                cells.append("%.1f (%.1f)%s" % (r["busbw_gbs"], r["t_us"], "" if r.get("ok") in (True, None) else " !"))
        out.append("| %d | %s |" % (s, " | ".join(cells)))
    return "\n".join(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("files", nargs="+")
    ap.add_argument("--coll", default="")
    a = ap.parse_args()
    for path in a.files:
        rows = load(path)
        n = rows[0].get("n") if rows else "?"
        colls = [a.coll] if a.coll else sorted({r["coll"] for r in rows})
        for c in colls:
            t = table(rows, c)
            if t:
                print("### %s — %s, %s ranks: busbw GB/s (time us)\n\n%s\n" % (path, c, n, t))
    return 0


if __name__ == "__main__":
    sys.exit(main())
