"""Pages of LookupResources on the device (Device::lookup_page, zg_lookup_resources_page) against the unpaged
zg_lookup_resources of the same lookup. One JSON line.

Per workload (cfg2, cfg3, cfg4 at --scale): bulk load + publish, then for the workload's lookup with the largest answer:
  * the unpaged lookup (zg_lookup_resources; the engine clock moves by one second per call so that its answer cache
    never serves it),
  * the first page (no cursor) at limits 1, 100 and 1 000,
  * a full paging at 1 000 (every page, then the total),
each timed by the host clock around the call (the call synchronises with the device before it returns), after
--warmup calls, median and p99 over --iters. Every row reports the candidates after the cursor, the candidates
verified and the verification windows of one call (zg_lookup_page_counters). The pages are compared with the unpaged
answer. --window / --growth set ZGPU_LOOKUP_PAGE_WINDOW / ZGPU_LOOKUP_PAGE_GROWTH (the first window's floor and the
least growth factor) for the engines the run creates. Power limit and clocks are read in the same run.

  python scripts/lookup_page_bench.py [--scale 1.0] [--iters 30] [--configs cfg2,cfg3,cfg4] [--window N] [--growth G]"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import zgpu  # noqa: E402
from filter_bench import _gpu_state, _stat  # noqa: E402
from spicedb_kubeapi_proxy_b200 import workloads  # noqa: E402

LIMITS = (1, 100, 1000)


def _timed(e, fn, iters, warm):
    """-> (timing, the last answer, the page counters of the last call)."""
    ts, out, c = [], None, {}
    t_clock = int(time.time())
    for i in range(warm + iters):
        e.set_clock(t_clock + i)
        before = e.lookup_page_counters()
        t0 = time.perf_counter()
        out = fn()
        dt = time.perf_counter() - t0
        after = e.lookup_page_counters()
        c = {k: after[k] - before[k] for k in ("after_cursor", "verified", "windows")}
        if i >= warm:
            ts.append(dt)
    return _stat(ts), out, c


def run(w, iters, warm):
    e = zgpu.Engine(w.schema, device=0)
    workloads.intern_names(w, e)
    w.load_into(e)
    e.publish()
    q = max(w.lookups, key=lambda q: len(e.lookup_resources_ids(*q)))
    out = {"workload": w.name, "relationships": int(e.stats()["tuples"]), "lookup": list(map(str, q)), "rows": {}}
    st, whole, _ = _timed(e, lambda: e.lookup_resources_ids(*q), iters, warm)
    out["answer"] = int(whole.size)
    out["rows"]["unpaged"] = st
    for limit in LIMITS:
        st, page, c = _timed(e, lambda: e.lookup_resources_page(*q, limit=limit), iters, warm)
        assert np.array_equal(page[0], whole[:limit]), (w.name, limit)
        out["rows"][f"first_page_{limit}"] = {**st, **c}

    def drain():
        ids, cur, n_pages, tot = [], None, 0, {"after_cursor": 0, "verified": 0, "windows": 0}
        while True:
            b = e.lookup_page_counters()
            page, _, cur, more = e.lookup_resources_page(*q, limit=1000, after=cur)
            a = e.lookup_page_counters()
            for k in tot:
                tot[k] += a[k] - b[k]
            ids.append(page)
            n_pages += 1
            if not more:
                return np.concatenate(ids), n_pages, tot

    st, (ids, n_pages, tot), _ = _timed(e, drain, max(3, iters // 10), 1)
    assert np.array_equal(ids, whole), w.name
    out["rows"]["full_paging_1000"] = {**st, "pages": n_pages, **tot}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--configs", default="cfg2,cfg3,cfg4")
    ap.add_argument("--window", type=int, default=0, help="ZGPU_LOOKUP_PAGE_WINDOW (0: the default)")
    ap.add_argument("--growth", type=int, default=0, help="ZGPU_LOOKUP_PAGE_GROWTH (0: the default)")
    a = ap.parse_args()
    if a.window:
        os.environ["ZGPU_LOOKUP_PAGE_WINDOW"] = str(a.window)
    if a.growth:
        os.environ["ZGPU_LOOKUP_PAGE_GROWTH"] = str(a.growth)
    res = {"gpu": _gpu_state(), "scale": a.scale, "window": a.window or "default", "growth": a.growth or "default",
           "runs": [run(workloads.by_name(c, a.scale), a.iters, a.warmup) for c in a.configs.split(",")]}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
