"""zg_collect_expired on the proxy's store: the bootstrap schema with --other relationships that never expire
(namespaces and pods with creators and viewers, the pods' namespaces) plus K workflow#idempotency_key@activity keys
with a 24 h expiration, half of them expired at the collection's `before`. One JSON line.

Per K (--keys, default 1 M and 10 M), median wall time over --reps of
  * a probe that finds nothing (before = the oldest key's expiration - 1): one count launch,
  * a full collection of the expired half on the device path, split into
      scan     device time of filter_expired_kernel (count + emit) and the records' copy back (torch.profiler),
      publish  the library's own timing of the merge-publish (zg_stats last_publish_ms),
      apply    the rest: records to store positions (Store::locate) and Store::apply,
  * the same collection on the host-scan path (Store::expired), taken by leaving one change unpublished; its time
    includes the full publish that change forces.
The expired keys are put back (bulk load + publish) outside the timed window. n_tuples and the snapshot's device
bytes are reported before and after a collection, with the card's name and power limit read in the same run.

  python scripts/expire_bench.py [--other 95400000] [--keys 1000000,10000000] [--reps 3]"""
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

T0 = 1_700_000_000  # the clock at which the keys were written
DAY = 86_400


def _gpu_state():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    except OSError:
        return {}
    return dict(zip(q.split(","), [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")])) if r.returncode == 0 else {}


def _tuples(e, res_type, rel, subj_type, res, subj):
    t = np.zeros(res.size, dtype=zgpu.TUPLE_DTYPE)
    t["res"], t["subj"], t["rel"], t["stype"], t["srel"] = res, subj, e.slot_id(res_type, rel), e.type_id(subj_type), 0xFFFF
    return t


def _updates(t, exp):
    u = np.zeros(t.size, dtype=zgpu.UPDATE_DTYPE)
    for f in ("res", "subj", "rel", "stype", "srel"):
        u[f] = t[f]
    u["expires_at"], u["op"] = exp, 0  # TOUCH
    return u


def _other(e, n, rng):
    """n relationships without expiration over namespaces, pods and users."""
    n_ns, n_pod, n_user = max(1, n // 200), max(1, n // 4), max(1, n // 20)
    parts, left = [], n
    for (rt, rel, st, nr, ns), share in ((("pod", "namespace", "namespace", n_pod, n_ns), 0.25),
                                         (("pod", "creator", "user", n_pod, n_user), 0.25),
                                         (("pod", "viewer", "user", n_pod, n_user), 0.3),
                                         (("namespace", "creator", "user", n_ns, n_user), 0.05),
                                         (("namespace", "viewer", "user", n_ns, n_user), 0.15)):
        k = min(left, int(n * share)) if share != 0.15 else left
        left -= k
        parts.append(_tuples(e, rt, rel, st, rng.integers(0, nr, k, dtype=np.uint32), rng.integers(0, ns, k, dtype=np.uint32)))
    return np.concatenate(parts)


def _keys(e, k):
    """k keys, one workflow and one activity each; key i expires at T0 + DAY + i % 3600 + (i odd: 2 days)."""
    i = np.arange(k, dtype=np.uint32)
    t = _tuples(e, "workflow", "idempotency_key", "activity", i, i)
    exp = (T0 + DAY + i % 3600 + (i & 1) * 2 * DAY).astype(np.uint32)
    return t, exp


def _scan_ms(fn):
    """Device time of the collection's kernels and copies back during fn(), by torch.profiler; None if unavailable."""
    try:
        import torch
        from torch.profiler import ProfilerActivity, profile
    except ImportError:
        return None, fn()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    us = 0.0
    for ev in prof.key_averages():
        if "filter_expired_kernel" in ev.key or "DtoH" in ev.key:
            us += getattr(ev, "self_device_time_total", 0.0) or getattr(ev, "self_cuda_time_total", 0.0)
    return us / 1e3, out


def run(n_other, k, reps):
    rng = np.random.default_rng(7)
    e = zgpu.Engine(workloads.BOOTSTRAP_SCHEMA, device=0)
    e.set_clock(T0)
    e.load_tuples(_other(e, n_other, rng))
    keys, kexp = _keys(e, k)
    expired = int((kexp <= T0 + DAY + 3600).sum())
    e.load_tuples(keys, kexp)
    e.publish()
    e.set_clock(T0 + 3 * DAY)
    before = T0 + DAY + 3600  # half the keys
    touch = _updates(_tuples(e, "namespace", "viewer", "user", np.zeros(1, np.uint32), np.zeros(1, np.uint32)), np.zeros(1, np.uint32))
    e.apply_updates(touch)  # builds the store's index outside the timing
    e.publish()
    out = {"n_other": n_other, "keys": k, "expired": expired}
    st = e.stats()
    out["before"] = {"n_tuples": e.num_tuples(), "snapshot_bytes": st["snapshot_bytes"]}
    probe = []
    for _ in range(max(5, reps)):
        t0 = time.perf_counter()
        n = e.collect_expired(T0 + DAY - 1)
        probe.append(time.perf_counter() - t0)
        assert n == 0
    out["probe_ms"] = round(float(np.median(probe)) * 1e3, 4)
    back = _updates(keys[kexp <= before], kexp[kexp <= before])

    def put_back():  # TOUCHes through the store's index: the next collection does not rebuild it
        e.apply_updates(back)
        e.publish()

    # one untimed collection under the profiler for the scan's device time (the profiler's start-up would swamp a
    # timed call), then the timed ones
    s, n = _scan_ms(lambda: e.collect_expired(before))
    assert n == expired, (n, expired)
    st = e.stats()
    out["after"] = {"n_tuples": e.num_tuples(), "snapshot_bytes": st["snapshot_bytes"]}
    put_back()
    total, pub, scan, host = [], [], [s] if s is not None else [], []
    for _ in range(reps):
        t0 = time.perf_counter()
        n = e.collect_expired(before)
        total.append(time.perf_counter() - t0)
        assert n == expired, (n, expired)
        pub.append(e.stats()["last_publish_ms"])
        put_back()
    # host-scan path: one change left unpublished (a TOUCH of a relationship without expiration)
    for _ in range(reps):
        e.apply_updates(touch)
        fc = e.filter_counters()["host_filters"]
        t0 = time.perf_counter()
        n = e.collect_expired(before)
        host.append(time.perf_counter() - t0)
        assert n == expired and e.filter_counters()["host_filters"] == fc + 1
        put_back()
    ms = lambda a: round(float(np.median(a)) * 1e3, 3)  # noqa: E731
    out["collect_ms"] = ms(total)
    out["publish_ms"] = round(float(np.median(pub)), 3)
    out["scan_ms"] = round(float(np.median(scan)), 3) if scan else None
    out["apply_ms"] = round(out["collect_ms"] - out["publish_ms"] - (out["scan_ms"] or 0.0), 3)
    out["host_path_ms"] = ms(host)
    out["filter_counters"] = e.filter_counters()
    e.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--other", type=int, default=95_400_000)
    ap.add_argument("--keys", default="1000000,10000000")
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    res = {"gpu": _gpu_state(), "runs": [run(a.other, int(k), a.reps) for k in a.keys.split(",")]}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
