"""Filters by resource id prefix (optional_resource_id_prefix) on the device against the host store's scan, on the named
workloads. One JSON line.

Per workload (named cfg2 at --cfg2-scale, named cfg4 at --cfg4-scale), a device engine and a host-only engine hold the
same relationships. Timed through the Python binding, median and p99 over --iters calls (the host over --host-iters):
  * a read of every relationship of one namespace (cfg2: `ns00042/`; cfg4: the documents `document00012`), with and
    without the resource type (the first call of each is timed apart; both are warmed up before either is timed,
    and the device calls are timed before the host's),
  * the first page of 100 of that read,
  * a write whose only content is a MUST_MATCH precondition on the prefix (on the device also without the type),
  * the delete of the namespace (once per engine; both engines delete the same relationships),
  * the first prefix read after a retirement (the names mirror is rebuilt), against the steady-state read.
Answers of the two engines are compared. The card's name, power limit and clocks are read in the same run.

  python scripts/prefix_filter_bench.py [--cfg2-scale 1.0] [--cfg4-scale 0.1] [--iters 20] [--host-iters 3]"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import zgpu  # noqa: E402
from filter_bench import _gpu_state, _stat, _timed  # noqa: E402
from spicedb_kubeapi_proxy_b200 import workloads  # noqa: E402

MUST_MATCH = 1


def _engine(w, **kw):
    e = zgpu.Engine(w.schema, **kw)
    workloads.intern_names(w, e)
    w.load_into(e)
    e.publish()
    return e


def run(w, rt, prefix, iters, host_iters):
    d, h = _engine(w, device=0), _engine(w, host_only=True)
    out = {"workload": w.name, "relationships": int(d.stats()["tuples"]), "prefix": prefix}
    reads = {"typed": {"res_type": rt, "res_id_prefix": prefix}, "untyped": {"res_id_prefix": prefix}}
    first = {}
    for name, f in reads.items():  # the first calls build the names mirror and size the buffers
        t0 = time.perf_counter()
        first[name] = d.read_relationships(**f)
        out[f"read_{name}_first_ms"] = round((time.perf_counter() - t0) * 1e3, 3)
    for _ in range(3):  # both shapes warm before either is timed
        for f in reads.values():
            d.read_relationships(**f)
    for name, f in reads.items():
        out[f"read_{name}_device"], got = _timed(lambda: d.read_relationships(**f), iters, 0)
        assert got == first[name], name
    for name, f in reads.items():
        out[f"read_{name}_host"], want = _timed(lambda: h.read_relationships(**f), host_iters, 0)
        assert want == first[name], name
        out["matched"] = len(want)
    f = reads["typed"]
    out["page100_device"], got = _timed(lambda: d.read_relationships_page(100, None, **f)[0], iters, 2)
    out["page100_host"], want = _timed(lambda: h.read_relationships_page(100, None, **f)[0], host_iters, 0)
    assert got == want
    pre = [(MUST_MATCH, f)]
    out["precondition_device"], _ = _timed(lambda: d.write_relationships([], pre), iters, 2)
    out["precondition_host"], _ = _timed(lambda: h.write_relationships([], pre), host_iters, 0)
    # the same count without the type: the device's scan and filter alone, without rendering lines
    pre_any = [(MUST_MATCH, reads["untyped"])]
    out["precondition_untyped_device"], _ = _timed(lambda: d.write_relationships([], pre_any), iters, 2)
    # the first read after a retirement rebuilds the names mirror
    for e in (d, h):
        e.intern(rt, "zz-unused")
        assert e.retire_unused_names() >= 1
    t0 = time.perf_counter()
    got = d.read_relationships(**f)
    out["read_after_retirement_ms"] = round((time.perf_counter() - t0) * 1e3, 3)
    assert got == h.read_relationships(**f)
    t0 = time.perf_counter()
    n_d = d.delete_relationships({"res_id_prefix": prefix})
    out["delete_device_ms"] = round((time.perf_counter() - t0) * 1e3, 3)
    t0 = time.perf_counter()
    n_h = h.delete_relationships({"res_id_prefix": prefix})
    out["delete_host_ms"] = round((time.perf_counter() - t0) * 1e3, 3)
    assert n_d == n_h == out["matched"]
    assert d.read_relationships(**f) == []
    out["prefix_counters"] = d.prefix_counters()
    assert out["prefix_counters"]["host_filters"] == 0
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cfg2-scale", type=float, default=1.0)
    ap.add_argument("--cfg4-scale", type=float, default=0.1)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--host-iters", type=int, default=3)
    a = ap.parse_args()
    res = {"gpu": _gpu_state(), "runs": [
        run(workloads.cfg2(scale=a.cfg2_scale), "pod", "ns00042/", a.iters, a.host_iters),
        run(workloads.cfg4(scale=a.cfg4_scale), "document", "document00012", a.iters, a.host_iters),
    ]}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
