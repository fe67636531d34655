"""ExpandPermissionTree on one GPU: batches of 1, 64 and 4 096 trees of a workload's checked permission.

For each batch size it prints one JSON line: trees, nodes and subjects per second (host clock around the C calls, which
end in a device synchronise, after a warm-up call; the Python trees are not built), the levels launched per call, and the per-level split of the device time into
count, scan and emit (CUDA events, the last call). With --verify, a sample of 16 trees is compared line for line with the
restatement over the workload's rows (tests/expand_oracle.py, DESIGN.md §2). The card's name and power limit come from
nvidia-smi in the same run.

    python scripts/expand_bench.py --workload cfg4 --scale 1.0
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import zgpu  # noqa: E402
from spicedb_kubeapi_proxy_b200 import workloads  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cfg4")
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--batches", default="1,64,4096")
    ap.add_argument("--seconds", type=float, default=2.0, help="timed window per batch size")
    ap.add_argument("--verify", action="store_true", help="check a sample of trees against the oracle")
    a = ap.parse_args()
    gpu = card()
    w = workloads.by_name(a.workload, scale=a.scale)
    e = zgpu.Engine(w.schema, device=0)
    w.load_into(e)
    e.publish()
    c = w.checks[0]
    res = np.unique(c.res)
    for b in (int(x) for x in a.batches.split(",")):
        reqs = np.zeros(b, dtype=zgpu._lib.EXPAND_REQUEST_DTYPE)
        reqs["perm"], reqs["res"] = e.slot_id(c.res_type, c.perm), res[np.arange(b) % res.size]
        status, _, _ = e.expand_permission_arrays(reqs)  # warm-up: module load
        out = (np.zeros(1 << 22, dtype=zgpu._lib.EXPAND_NODE_DTYPE), np.zeros(1 << 24, dtype=zgpu._lib.EXPAND_SUBJECT_DTYPE))
        e.expand_permission_arrays(reqs, out=out)  # and the answer buffers' pages
        before, calls, t0 = e.expand_counters(), 0, time.perf_counter()
        while time.perf_counter() - t0 < a.seconds or calls < 3:  # the C call into the same buffers: no Python trees
            e.expand_permission_arrays(reqs, out=out)
            calls += 1
        dt = time.perf_counter() - t0
        after = e.expand_counters()
        split = e.expand_last_times()
        d = {k: after[k] - before[k] for k in after}
        print(json.dumps({
            "workload": a.workload, "scale": a.scale, "batch": b, "calls": calls, "ms_per_call": 1e3 * dt / calls,
            "trees_per_s": d["trees"] / dt, "nodes_per_s": d["nodes"] / dt, "subjects_per_s": d["subjects"] / dt,
            "nodes_per_tree": d["nodes"] / max(d["trees"], 1), "levels_per_call": d["levels"] / calls,
            "last_call_ms_count_scan_emit": [round(float(x), 4) for x in split.sum(axis=0)],
            "last_call_ms_per_level": [[round(float(x), 4) for x in lv] for lv in split],
            "last_call_levels": int(split.shape[0]), "failed": int((status[:b] != 0).sum()),
            "card": gpu}), flush=True)
    if a.verify:  # a sample of trees line for line against the restatement over the workload's rows
        from expand_oracle import GroupRows, expand_tree, group_order, id_tree_lines, lines

        rows = GroupRows(w.schema, w.groups)
        pick = res[np.random.default_rng(0).choice(res.size, 16, replace=False)]
        trees = e.expand_permission_trees([(c.res_type, int(r), c.perm) for r in pick])
        bad = sum(id_tree_lines(t) != lines(expand_tree(rows, c.res_type, str(int(r)), c.perm, order=group_order))
                  for r, t in zip(pick, trees))
        print(json.dumps({"workload": a.workload, "scale": a.scale, "verified_trees": len(pick), "mismatches": bad}),
              flush=True)

if __name__ == "__main__":
    main()
