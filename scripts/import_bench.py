"""ImportBulkRelationships against the other ways to fill a store with named relationships, on one GPU.

For a named workload store (every object named as workloads.object_name names it; duplicates dropped) it reports one
JSON line per method, each into a fresh engine:
  import     zg_import_relationships in calls of --call relationships: wall time, and the last call's split into the
             device steps (names, sort, duplicates, from device events) and the host's (interning, store and index,
             publish)
  writes     zg_write_relationships CREATEs in calls of 1 000 (what a resync through WriteRelationships does): a timed
             prefix of --write-prefix relationships, extrapolated linearly to the whole store and labelled so
  load       zg_intern_objects_packed + zg_load_tuples + zg_publish (ids, no SpiceDB semantics)
and after each the time of the first write (one CREATE), which builds the host relationship index when the method
left it behind. The card's name and power limit come from nvidia-smi in the same run.

    python scripts/import_bench.py --workload cfg2 --scale 1.0
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

import zgpu  # noqa: E402
from spicedb_kubeapi_proxy_b200 import workloads  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def classes(w):
    """The workload's relationships by class, duplicates dropped: {(res_type, rel, subj_type, srel): (res, subj)}."""
    out = {}
    for g in w.groups:
        srel = "*" if g.wildcard else (g.srel or "")
        k = (g.res_type, g.rel, g.subj_type, srel)
        r, s = out.get(k, (np.zeros(0, np.uint64), np.zeros(0, np.uint64)))
        out[k] = (np.concatenate([r, g.res.astype(np.uint64)]), np.concatenate([s, g.subj.astype(np.uint64)]))
    for k, (r, s) in out.items():
        key = np.unique((r << np.uint64(32)) | s)
        out[k] = ((key >> np.uint64(32)).astype(np.int64), (key & np.uint64(0xFFFFFFFF)).astype(np.int64))
    return out


def names(t, ids):
    return [workloads.object_name(t, int(i)) for i in ids]


def import_groups(cls, lo, hi):
    """The relationships [lo, hi) in class order, as import groups."""
    gs, at = [], 0
    for (rt, rel, st, srel), (r, s) in cls.items():
        a, b = max(lo - at, 0), min(hi - at, r.size)
        if a < b:
            subj = ["*"] * (b - a) if srel == "*" else names(st, s[a:b])
            gs.append((rt, rel, st, "" if srel == "*" else srel, names(rt, r[a:b]), subj, None))
        at += r.size
    return gs


def first_write(e):
    t0 = time.perf_counter()
    e.write_relationships([(1, "%s:first_write_probe#%s@%s:%s" % probe, 0)])
    return (time.perf_counter() - t0) * 1e3


probe = None


def main():
    global probe
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cfg2")
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--call", type=int, default=1 << 20, help="relationships per import call")
    ap.add_argument("--write-prefix", type=int, default=200_000, help="relationships timed through the write path")
    ap.add_argument("--methods", default="import,writes,load")
    a = ap.parse_args()
    w = workloads.by_name(a.workload, scale=a.scale)
    cls = classes(w)
    total = sum(r.size for r, _ in cls.values())
    rt, rel, st, srel = next(k for k in cls if k[3] == "")
    probe = (rt, rel, st, names(st, [0])[0])
    base = {"workload": a.workload, "scale": a.scale, "relationships": total, "card": card()}
    for m in a.methods.split(","):
        e = zgpu.Engine(w.schema, device=0)
        if m == "import":
            parts, t0 = {}, time.perf_counter()
            for lo in range(0, total, a.call):
                gs = import_groups(cls, lo, lo + a.call)
                t1 = time.perf_counter()
                e.import_relationships(gs)
                parts["calls_ms"] = parts.get("calls_ms", 0.0) + (time.perf_counter() - t1) * 1e3
            wall = (time.perf_counter() - t0) * 1e3
            print(json.dumps({**base, "method": "import", "call": a.call, "wall_ms": round(wall, 1),
                              "in_calls_ms": round(parts["calls_ms"], 1),
                              "last_call_ms": {k: round(v, 2) for k, v in e.import_last_times().items()},
                              "first_write_ms": round(first_write(e), 2)}), flush=True)
        elif m == "writes":
            n = min(a.write_prefix, total)
            gs = import_groups(cls, 0, n)
            rels = [("%s:%s#%s@%s:%s" % (g[0], r, g[1], g[2], s)) + ("#" + g[3] if g[3] else "")
                    for g in gs for r, s in zip(g[4], g[5])]
            t0 = time.perf_counter()
            for i in range(0, n, 1000):
                e.write_relationships([(1, r, 0) for r in rels[i:i + 1000]])
            ms = (time.perf_counter() - t0) * 1e3
            print(json.dumps({**base, "method": "writes", "timed_relationships": n, "timed_ms": round(ms, 1),
                              "extrapolated_ms" if n < total else "wall_ms": round(ms * total / max(n, 1), 1),
                              "first_write_ms": round(first_write(e), 2)}), flush=True)
        elif m == "load":
            t0 = time.perf_counter()
            workloads.intern_names(w, e)
            w.load_into(e)
            e.publish()
            ms = (time.perf_counter() - t0) * 1e3
            print(json.dumps({**base, "method": "load", "wall_ms": round(ms, 1), "first_write_ms": round(first_write(e), 2)}),
                  flush=True)
        e.close()


if __name__ == "__main__":
    main()
