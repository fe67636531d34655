"""Pages of relationship reads on the device (csrc/filter.cuh page_*, zg_read_relationships_page) against the unpaged
zg_read_relationships of the same read. One JSON line.

Per workload (cfg4 and cfg3 at --scale): bulk load + publish, then for the (type, relation) read with the fewest
relationships (on cfg4 at scale 1.0 that read returns 2.0 M relationships) and limits 1 000 / 10 000 / 100 000:
  * the first page (no cursor): median and p99 over --iters calls, through Engine.read_relationships_page (lines,
    expirations and cursors as Python objects) and through the C call alone,
  * a drain of the whole read page by page: the time of every page (median, p99) and the total,
  * the same read through zg_read_relationships (--one-shot-iters calls),
  * zg_delete_relationships_limited with limit 1 000: a refused one (ZG_EPRECOND) and a partial one (the rows are put
    back outside the timed window).
The drained lines are compared with the one-shot read. Power limit and clocks are read in the same run.

  python scripts/read_page_bench.py [--scale 1.0] [--iters 50] [--one-shot-iters 3]"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import zgpu  # noqa: E402
from filter_bench import _gpu_state, _oid, _stat, _timed  # noqa: E402
from spicedb_kubeapi_proxy_b200 import workloads  # noqa: E402

LIMITS = (1000, 10_000, 100_000)


def _abi_page(e, flt, limit, buf):
    """The C call alone: no expirations, no cursors, no Python list of lines."""
    need, n, more = C.c_size_t(0), C.c_uint64(0), C.c_int32(0)
    rc = e._L.zg_read_relationships_page(e._h, C.byref(flt), limit, None, buf, len(buf), C.byref(need), C.byref(n), None,
                                         None, None, C.byref(more))
    assert rc == 0 and n.value == limit, rc
    return n.value


def run(w, iters, one_shot_iters):
    e = zgpu.Engine(w.schema, device=0)
    w.load_into(e)
    e.publish()
    per_rel = {}
    for q in w.groups:
        per_rel[(q.res_type, q.rel)] = per_rel.get((q.res_type, q.rel), 0) + q.res.size
    rt, rel = min(per_rel, key=per_rel.get)
    f = {"res_type": rt, "rel": rel}
    out = {"workload": w.name, "relationships": int(e.stats()["tuples"]), "read": f"{rt}#{rel}", "pages": {}}
    t0 = time.perf_counter()
    one_shot = e.read_relationships(**f)
    out["one_shot_first_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
    out["one_shot"], again = _timed(lambda: e.read_relationships(**f), one_shot_iters, 0)
    assert again == one_shot
    out["answer"] = len(one_shot)
    mismatches = 0
    flt, buf = e._filter(f), C.create_string_buffer(max(LIMITS) * 128)
    for limit in LIMITS:
        r = {}
        r["first_page"], _ = _timed(lambda: e.read_relationships_page(limit, None, **f), iters, 3)
        r["first_page_abi"], _ = _timed(lambda: _abi_page(e, flt, limit, buf), iters, 3)
        lines, ts, cursor = [], [], None
        t_all = time.perf_counter()
        while True:
            t0 = time.perf_counter()
            page, _, _, cursor, more = e.read_relationships_page(limit, cursor, **f)
            ts.append(time.perf_counter() - t0)
            lines += page
            if not more:
                break
        r["drain_total_ms"] = round((time.perf_counter() - t_all) * 1e3, 1)
        r["per_page"] = _stat(ts)
        mismatches += int(sorted(lines) != one_shot)
        out["pages"][str(limit)] = r
    # deletes with a limit: refused (more than 1 000 match), and partial (the first 1 000 go, then come back)
    def refused():
        try:
            e.delete_relationships_limited(f, limit=1000)
        except zgpu.ZgpuError as x:
            return x.code
        return 0

    out["delete_limited_refused"], code = _timed(refused, iters, 2)
    mismatches += int(code != -5)
    first = e.read_relationships_page(1000, None, **f)[0]
    ups = np.zeros(len(first), dtype=zgpu.UPDATE_DTYPE)
    for j, l in enumerate(first):
        a_rt, a_rid, a_rel, a_st, a_sid, a_srel = zgpu._lib.split_rel(l)
        ups["res"][j], ups["rel"][j], ups["stype"][j] = _oid(a_rid), e.slot_id(a_rt, a_rel), e.type_id(a_st)
        ups["srel"][j] = zgpu.SREL_WILDCARD if a_sid == "*" else e.slot_id(a_st, a_srel) if a_srel else zgpu.SREL_NONE
        ups["subj"][j] = 0 if a_sid == "*" else _oid(a_sid)
    ts = []
    for _ in range(max(iters // 5, 3)):
        t0 = time.perf_counter()
        got = e.delete_relationships_limited(f, limit=1000, allow_partial=True)
        ts.append(time.perf_counter() - t0)
        mismatches += int(got != (1000, True))
        e.apply_updates(ups)
        e.publish()
    out["delete_limited_partial_1000"] = _stat(ts[1:])
    mismatches += int(e.read_relationships_page(1000, None, **f)[0] != first)
    c = e.page_counters()
    mismatches += int(c["host_pages"] != 0)
    out["page_counters"] = c
    out["mismatches"] = mismatches
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--one-shot-iters", type=int, default=3)
    ap.add_argument("--workloads", default="cfg4,cfg3")
    a = ap.parse_args()
    res = {"bench": "read_page_bench", "scale": a.scale, "gpu": _gpu_state(), "runs": []}
    for name in a.workloads.split(","):
        res["runs"].append(run(getattr(workloads, name)(scale=a.scale), a.iters, a.one_shot_iters))
    res["gpu_after"] = _gpu_state()
    res["mismatches"] = sum(r["mismatches"] for r in res["runs"])
    print(json.dumps(res))
    return 1 if res["mismatches"] else 0


if __name__ == "__main__":
    sys.exit(main())
