"""zg_retire_unused_names under the proxy's churn: the bootstrap schema with a base of --base named pod#viewer
relationships, then --cycles rounds of --churn dual writes, each a workflow taking a lock and writing an idempotency key
that expires in 24 h (interned updates + publish), releasing the lock, and a day later the keys collected. With
retirement the names are retired at the end of each round; without, they stay. One JSON line.

Per cycle and mode:
  retire_ms       wall time of the retirement call
  scan_ms         device time of mention_scan_kernel and the bitmaps' copy back (torch.profiler), taken on a second
                  call that finds nothing to retire (the same scan)
  named / free / extent   zg_name_counters out[0] / out[2] / out[3]
  caps            object capacities of workflow, activity and lock
  delta / full    merge and full publishes of the round
  ingress_ms      wall time of the first device-ingress call after the round (the mirror re-upload after a retirement)
                  and ingress_steady_ms of the next one
The card's name and power limit are read in the same run.

  python scripts/retire_bench.py [--base 10000000] [--churn 20000] [--cycles 6]"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import zgpu  # noqa: E402
from expire_bench import _gpu_state  # noqa: E402
from spicedb_kubeapi_proxy_b200 import workloads  # noqa: E402

T0 = 1_700_000_000
DAY = 86_400


def _ups(e, res_type, rel, subj_type, res, subj, exp, op):
    u = np.zeros(res.size, dtype=zgpu.UPDATE_DTYPE)
    u["res"], u["subj"], u["rel"], u["stype"], u["srel"] = res, subj, e.slot_id(res_type, rel), e.type_id(subj_type), 0xFFFF
    u["expires_at"], u["op"] = exp, op
    return u


def _scan_ms(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    us = 0.0
    for ev in prof.key_averages():
        if "mention_scan_kernel" in ev.key or "DtoH" in ev.key:
            us += getattr(ev, "self_device_time_total", 0.0) or getattr(ev, "self_cuda_time_total", 0.0)
    return us / 1e3, out


def run(base, churn, cycles, retire):
    rng = np.random.default_rng(11)
    e = zgpu.Engine(workloads.BOOTSTRAP_SCHEMA, device=0)
    n_pod, n_user = max(1, base // 4), max(1, base // 20)
    pods = e.intern_packed("pod", [f"ns{i % 1000}/pod-{i}" for i in range(n_pod)])
    users = e.intern_packed("user", [f"user-{i}" for i in range(n_user)])
    t = np.zeros(base, dtype=zgpu.TUPLE_DTYPE)
    t["res"], t["subj"] = pods[rng.integers(0, n_pod, base)], users[rng.integers(0, n_user, base)]
    t["rel"], t["stype"], t["srel"] = e.slot_id("pod", "viewer"), e.type_id("user"), 0xFFFF
    e.load_tuples(t)
    e.publish()
    probe_pods, probe_users = [f"ns{i % 1000}/pod-{i}" for i in range(64)], [f"user-{i}" for i in range(64)]
    e.check_bulk_packed_ingress("pod", "view", "user", probe_pods, probe_users)  # the mirror, built once
    rows = []
    for c in range(cycles):
        now = T0 + c * 2 * DAY
        e.set_clock(now)
        s0 = e.stats()
        wf = e.intern_packed("workflow", [f"wf-{c}-{i}" for i in range(churn)])
        act = e.intern_packed("activity", [f"{c:04d}{i:012x}" for i in range(churn)])
        lock = e.intern_packed("lock", [f"{c:04d}{i:012x}" for i in range(churn)])
        e.apply_updates(np.concatenate([_ups(e, "lock", "workflow", "workflow", lock, wf, 0, 0),
                                        _ups(e, "workflow", "idempotency_key", "activity", wf, act, now + DAY, 0)]))
        e.publish()
        e.apply_updates(_ups(e, "lock", "workflow", "workflow", lock, wf, 0, 2))
        e.publish()
        e.set_clock(now + DAY + 1)
        e.collect_expired(now + DAY)
        row = {"cycle": c}
        if retire:
            t1 = time.perf_counter()
            row["retired"] = e.retire_unused_names()
            row["retire_ms"] = (time.perf_counter() - t1) * 1e3
            row["scan_ms"], again = _scan_ms(e.retire_unused_names)
            assert again == 0
        t1 = time.perf_counter()
        e.check_bulk_packed_ingress("pod", "view", "user", probe_pods, probe_users)
        row["ingress_ms"] = (time.perf_counter() - t1) * 1e3
        t1 = time.perf_counter()
        e.check_bulk_packed_ingress("pod", "view", "user", probe_pods, probe_users)
        row["ingress_steady_ms"] = (time.perf_counter() - t1) * 1e3
        nc, s1 = e.name_counters(), e.stats()
        row.update(named=nc["named"], free=nc["free_ids"], extent=nc["id_extent"],
                   caps=[e.object_capacity(x) for x in ("workflow", "activity", "lock")],
                   delta=s1["delta_publishes"] - s0["delta_publishes"], full=s1["full_publishes"] - s0["full_publishes"])
        rows.append({k: (round(v, 3) if isinstance(v, float) else v) for k, v in row.items()})
    e.close()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", type=int, default=10_000_000)
    ap.add_argument("--churn", type=int, default=20_000)
    ap.add_argument("--cycles", type=int, default=6)
    a = ap.parse_args()
    out = {"gpu": _gpu_state(), "base": a.base, "churn": a.churn,
           "with_retirement": run(a.base, a.churn, a.cycles, True),
           "without_retirement": run(a.base, a.churn, a.cycles, False)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
