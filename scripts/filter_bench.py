"""Relationship filters: the device path (csrc/filter.cuh, answered from the resident CSR) against the host scan
(Store::match) on the same engine and the same store. One JSON line.

Per workload (cfg4 and cfg3 at --scale): bulk load + publish, then the wall time of
  * the first zg_read_relationships after the bulk load (the device path builds no host index),
  * zg_read_relationships exact, by resource, by subject and by (type, relation),
  * a write whose precondition fails (ZG_EPRECOND: the precondition's cost alone, nothing is applied),
  * zg_write_relationships with 1 update + 1 exact-match precondition (the proxy's write), device path,
  * zg_delete_relationships by resource, device path (the rows are put back outside the timed window),
each as median and p99 after warm-up. The host scan is forced by leaving the store dirty (one relationship loaded again
and not published), and timed on the same filters; its first call also builds the store's index and is reported apart.
Every timed answer is compared between the paths. The successful write and the delete publish, which ends the dirty
state, so their host-scan times are not measured. Power limit and clocks are read in the same run.

  python scripts/filter_bench.py [--scale 1.0] [--iters 200] [--host-iters 5]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import zgpu  # noqa: E402
from spicedb_kubeapi_proxy_b200 import workloads  # noqa: E402

NAMED = 64  # objects per type that get a name at least: filters name objects by string, the rest of the store stays numeric


def _stat(ts):
    a = np.sort(np.asarray(ts)) * 1e3
    return {"median_ms": round(float(np.median(a)), 4), "p99_ms": round(float(a[min(a.size - 1, int(a.size * 0.99))]), 4), "n": int(a.size)}


def _timed(fn, iters, warm):
    for _ in range(warm):
        fn()
    ts, out = [], None
    for _ in range(iters):
        t0 = time.perf_counter()
        out = fn()
        ts.append(time.perf_counter() - t0)
    return _stat(ts), out


def _oid(name):
    """Dense id of an object from how a read prints it: its workload name (letters, then the id) or the bare id."""
    return int("".join(ch for ch in name if ch.isdigit()))


def _gpu_state():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks.mem"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    except OSError:
        return {}
    return dict(zip(q.split(","), [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")])) if r.returncode == 0 else {}


def run(w, iters, host_iters):
    # a relationship from the group with the most relationships whose two objects have the lowest ids: names are
    # interned densely from id 0, so every type gets names up to there
    g = max((g for g in w.groups if not g.wildcard), key=lambda g: g.res.size)
    i = int(np.argmin(np.maximum(g.res, g.subj)))
    named = max(NAMED, int(max(g.res[i], g.subj[i])) + 1)
    e = zgpu.Engine(w.schema, device=0)
    for t, n in sorted(workloads.object_counts(w).items()):
        e.intern_packed(t, [workloads.object_name(t, k) for k in range(min(n, named))])
    w.load_into(e)
    e.publish()
    rt, st = g.res_type, g.subj_type
    rid, sid = workloads.object_name(rt, int(g.res[i])), workloads.object_name(st, int(g.subj[i]))
    exact = {"res_type": rt, "res_id": rid, "rel": g.rel, "subj_type": st, "subj_id": sid, "subj_rel": g.srel or "..."}
    per_rel = {}
    for q in w.groups:
        per_rel[(q.res_type, q.rel)] = per_rel.get((q.res_type, q.rel), 0) + q.res.size
    small_type, small_rel = min(per_rel, key=per_rel.get)  # the (type, relation) with the fewest relationships
    reads = {"exact": exact, "by_resource": {"res_type": rt, "res_id": rid}, "by_subject": {"subj_type": st, "subj_id": sid},
             "by_type_relation": {"res_type": small_type, "rel": small_rel}}
    rel_text = f"{rt}:{rid}#{g.rel}@{st}:{sid}" + (f"#{g.srel}" if g.srel else "")
    out = {"workload": w.name, "relationships": int(e.stats()["tuples"]), "device": {}, "host_scan": {}, "answers": {}}

    def failing_write():
        try:
            e.write_relationships([(0, rel_text, 0)], [(zgpu._lib.PRECOND_MUST_NOT_MATCH, exact)])
        except zgpu.ZgpuError as x:
            return x.code
        return 0

    t0 = time.perf_counter()
    first = e.read_relationships(**reads["by_resource"])
    out["device"]["first_read_after_bulk_load_ms"] = round((time.perf_counter() - t0) * 1e3, 4)
    dev_answers = {}
    for name, f in reads.items():
        # a large answer is mostly rendered text on either path: few repetitions
        n_it = iters if name != "by_type_relation" else host_iters
        out["device"]["read_" + name], dev_answers[name] = _timed(lambda: e.read_relationships(**f), n_it, 2)
        out["answers"][name] = len(dev_answers[name])
    assert first == dev_answers["by_resource"]
    out["device"]["failing_precondition"], code = _timed(failing_write, iters, 5)
    assert code == -5, code
    # the proxy's write: 1 update + 1 exact-match precondition; a relationship to a named subject the resource does not
    # have yet is touched and deleted in turn
    have = set(dev_answers["by_resource"])
    fresh = next(r for r in (f"{rt}:{rid}#{g.rel}@{st}:{workloads.object_name(st, k)}" + (f"#{g.srel}" if g.srel else "")
                             for k in range(named)) if r not in have)
    turn = [0]

    def write():
        e.write_relationships([(0 if turn[0] % 2 == 0 else 2, fresh, 0)], [(zgpu._lib.PRECOND_MUST_MATCH, exact)])
        turn[0] += 1

    out["device"]["write_1_update_1_precondition"], _ = _timed(write, iters + iters % 2, 6)
    rows = e.read_relationships(**reads["by_resource"])
    assert rows == dev_answers["by_resource"]
    # delete by resource; the rows are put back (interned TOUCH + publish) outside the timed window
    ups = np.zeros(len(rows), dtype=zgpu.UPDATE_DTYPE)
    for j, r in enumerate(rows):
        a_rt, a_rid, a_rel, a_st, a_sid, a_srel = zgpu._lib.split_rel(r)
        ups["res"][j], ups["rel"][j], ups["stype"][j] = _oid(a_rid), e.slot_id(a_rt, a_rel), e.type_id(a_st)
        ups["srel"][j] = zgpu.SREL_WILDCARD if a_sid == "*" else e.slot_id(a_st, a_srel) if a_srel else zgpu.SREL_NONE
        ups["subj"][j] = 0 if a_sid == "*" else _oid(a_sid)
    ts = []
    for _ in range(max(iters // 4, 3)):
        t0 = time.perf_counter()
        n_del = e.delete_relationships(reads["by_resource"])
        ts.append(time.perf_counter() - t0)
        assert n_del == len(rows), (n_del, len(rows))
        e.apply_updates(ups)
        e.publish()
    out["device"]["delete_by_resource"] = _stat(ts[1:])
    assert e.read_relationships(**reads["by_resource"]) == rows
    c = e.filter_counters()
    assert c["host_filters"] == 0, c
    out["device"]["counters"] = c

    # the host scan on the same store: one relationship loaded again and left unpublished
    t = np.zeros(1, dtype=zgpu.TUPLE_DTYPE)
    t["res"], t["subj"], t["rel"], t["stype"] = int(g.res[i]), int(g.subj[i]), e.slot_id(rt, g.rel), e.type_id(st)
    t["srel"] = e.slot_id(st, g.srel) if g.srel else zgpu.SREL_NONE
    e.load_tuples(t)
    rev = e.stats()["revision"]
    t0 = time.perf_counter()
    first = e.read_relationships(**reads["by_resource"])
    out["host_scan"]["first_read_builds_the_index_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
    mismatches = int(first != dev_answers["by_resource"])
    for name, f in reads.items():
        out["host_scan"]["read_" + name], ans = _timed(lambda: e.read_relationships(**f), host_iters, 1)
        mismatches += int(ans != dev_answers[name])
    out["host_scan"]["failing_precondition"], code = _timed(failing_write, host_iters, 1)
    mismatches += int(code != -5)
    c2 = e.filter_counters()
    assert c2["device_filters"] == c["device_filters"] and c2["host_filters"] > 0 and e.stats()["revision"] == rev, c2
    out["mismatches"] = mismatches
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--host-iters", type=int, default=5)
    ap.add_argument("--workloads", default="cfg4,cfg3")
    a = ap.parse_args()
    res = {"bench": "filter_bench", "scale": a.scale, "gpu": _gpu_state(), "runs": []}
    for name in a.workloads.split(","):
        res["runs"].append(run(getattr(workloads, name)(scale=a.scale), a.iters, a.host_iters))
    res["gpu_after"] = _gpu_state()
    res["mismatches"] = sum(r["mismatches"] for r in res["runs"])
    print(json.dumps(res))
    return 1 if res["mismatches"] else 0


if __name__ == "__main__":
    sys.exit(main())
