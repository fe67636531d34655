"""LookupSubjects on a sharded handle (zg_config.n_shards with ZG_FLAG_HANDLE_SUBJECTS), against the multi-engine
driver (dist.DeviceShardedLookup.lookup_subjects over LocalDeviceTransport) and a replica engine, on the same seeded
resources.

One process, S virtual shards on ONE GPU: this measures what the in-process exchange (walk entries written into their
owners' inboxes through peer memory, both verifications on the handle's check protocol) costs against the Python
driver and a replica, not multi-GPU scaling. Workloads: cfg3 namespace#view, cfg4 document#view and
document#restricted_view, subjects of type user, ZG_WILDCARDS_INCLUDE. One call per lookup (median / p99); the
handle's walk levels, host waits and inbox entries per lookup. Every timed answer is compared with the replica's.
Prints one JSON line with the GPU name and its enforced power limit, read in the same run.

    python scripts/handle_subjects_bench.py [--shards 4] [--resources 200] [--scale 0.1]
"""
import argparse, json, os, sys, threading, time
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import zgpu
from spicedb_kubeapi_proxy_b200 import dist as zdist, workloads

ap = argparse.ArgumentParser()
ap.add_argument("--shards", type=int, default=4, help="virtual shards on one GPU")
ap.add_argument("--resources", type=int, default=200, help="lookups per workload")
ap.add_argument("--scale", type=float, default=0.1)
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--verify-chunk", type=int, default=1 << 12, help="candidates per check_bulk call of the driver")
ap.add_argument("--subq-cap", type=int, default=1 << 24, help="zg_config.subquery_capacity of every shard")
a = ap.parse_args()


def gpu_info():
    try:
        import pynvml as nv
        nv.nvmlInit()
        h = nv.nvmlDeviceGetHandleByIndex(int(os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0] or 0))
        name = nv.nvmlDeviceGetName(h)
        return {"gpu": name.decode() if isinstance(name, bytes) else name,
                "power_limit_w": nv.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0}
    except Exception as ex:  # noqa: BLE001  (reported beside the numbers)
        import torch
        return {"gpu": torch.cuda.get_device_name(0), "power_limit_w": None, "nvml_error": repr(ex)}


def pct(x, q):
    return round(float(np.percentile(x, q)), 3) if len(x) else None


def same(x, y):
    return x is not None and y is not None and np.array_equal(x[0], y[0]) and x[1] == y[1] and np.array_equal(x[2], y[2])


def run(w, cases):
    import torch

    S = a.shards
    replica = zgpu.Engine(w.schema, device=0)
    handle = zgpu.Engine(w.schema, device=0, n_shards=S, handle_subjects=True, subquery_capacity=a.subq_cap)
    ts = zdist.LocalDeviceTransport.cluster(S)
    engines = [zgpu.Engine(w.schema, device=0, shard_rank=r, shard_count=S, subquery_capacity=a.subq_cap) for r in range(S)]
    for e in [replica, handle] + engines:
        w.load_into(e)
        e.publish()
        e.set_clock(int(time.time()))
    lks = [zdist.DeviceShardedLookup(engines[r], ts[r], verify_chunk=a.verify_chunk) for r in range(S)]
    e0 = engines[0]
    reqs = [(e0.type_id(rt), r, e0.slot_id(rt, p), e0.type_id(st), zgpu.SREL_NONE, zgpu._lib.WILDCARDS_INCLUDE) for rt, r, p, st in cases]

    def driver():
        """rank 0 brings one lookup per call, the other ranks none -> (ms per call, answers)."""
        times, got, errs = [], [], []

        def rank(r):
            try:
                for q in reqs:
                    t0 = time.perf_counter()
                    ans = lks[r].lookup_subjects([q] if r == 0 else [])
                    if r == 0:
                        torch.cuda.synchronize()
                        times.append((time.perf_counter() - t0) * 1e3)
                        got.append(ans[0])
            except Exception as ex:  # noqa: BLE001
                errs.append(repr(ex))
                ts[r]._s["bar"].abort()

        th = [threading.Thread(target=rank, args=(r,)) for r in range(S)]
        [x.start() for x in th]
        [x.join() for x in th]
        if errs:
            raise RuntimeError(errs[0])
        return times, got

    def singles(e):
        times, out = [], []
        for rt, r, p, st in cases:
            t0 = time.perf_counter()
            out.append(e.lookup_subjects_ids(rt, r, p, st, cap=1 << 20))  # one call: no ZG_E2BIG retry
            times.append((time.perf_counter() - t0) * 1e3)
        return times, out

    res = {"lookups": len(cases) - a.warmup}
    c0 = handle.handle_subjects_counters()
    ht, hans = singles(handle)
    c1 = handle.handle_subjects_counters()
    dt, dans = driver()
    rt_, rans = singles(replica)
    res["mismatches_vs_replica"] = sum(int(not same(h, r)) + int(not same(d, r)) for h, d, r in zip(hans, dans, rans))
    for name, t in (("handle", ht), ("driver", dt), ("replica", rt_)):
        res[f"{name}_ms_median"], res[f"{name}_ms_p99"] = pct(t[a.warmup:], 50), pct(t[a.warmup:], 99)
    assert c1["lookups"] - c0["lookups"] == len(cases)
    res["handle_counters_per_lookup"] = {k: round((c1[k] - c0[k]) / len(cases), 2) for k in c1 if k != "lookups"}
    res["answer_ids"] = int(sum(len(x[0]) + len(x[2]) for x in rans))
    for e in [replica, handle] + engines:
        e.close()
    return res


def main():
    rng = np.random.default_rng(11)
    result = {"shards": a.shards, "scale": a.scale}
    mismatches = 0
    specs = [("cfg3", workloads.cfg3(scale=a.scale), [("namespace", "view")]),
             ("cfg4", workloads.cfg4(scale=a.scale), [("document", "view"), ("document", "restricted_view")])]
    for name, w, perms in specs:
        cases = []
        for rt, p in perms:
            c = next(c for c in w.checks if c.res_type == rt)
            res = rng.permutation(np.unique(c.res))[: a.resources // len(perms)]
            cases += [(rt, int(r), p, c.subj_type) for r in res]
        print(f"{name}: {len(cases)} lookups", file=sys.stderr, flush=True)
        result[name] = run(w, cases)
        mismatches += result[name]["mismatches_vs_replica"]
    result.update(mismatches_vs_replica=mismatches, **gpu_info())
    print(json.dumps(result))


if __name__ == "__main__":
    main()
