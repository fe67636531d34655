"""LookupResources on a sharded handle (zg_config.n_shards with ZG_FLAG_HANDLE_LOOKUPS), against the multi-engine
driver (dist.DeviceShardedLookup over LocalDeviceTransport) and a replica engine, on the same seeded lookups.

One process, S virtual shards on ONE GPU: this measures what the in-process exchange (frontier and answer keys
through peer memory, candidates verified by the handle's check protocol) costs against the Python driver and a
replica, not multi-GPU scaling. Workloads: cfg2 pod#view, cfg3 namespace#view, cfg4 document#view and
document#restricted_view. Per path: one call per lookup (median / p99) and all the lookups at once (the handle and
the replica: one thread per lookup, so that the batcher forms groups of up to 64; the driver: one call). Every
timed answer is compared with the replica's. Both clocks are pinned, one second apart for the two phases, so that
no answer of the first phase is served from the lookup cache in the second. Prints one JSON line with the GPU name
and its enforced power limit, read in the same run.

    python scripts/handle_lookup_bench.py [--shards 4] [--subjects 300] [--scale 0.1]
"""
import argparse, json, os, sys, threading, time
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import zgpu
from spicedb_kubeapi_proxy_b200 import dist as zdist, workloads

ap = argparse.ArgumentParser()
ap.add_argument("--shards", type=int, default=4, help="virtual shards on one GPU")
ap.add_argument("--subjects", type=int, default=300)
ap.add_argument("--scale", type=float, default=0.1, help="cfg3 and cfg4 scale; cfg2 uses 4x of it")
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


def users_of(w):
    return max(int(g.subj.max()) + 1 for g in w.groups if g.subj_type == "user" and not g.wildcard and g.subj.size)


def pct(x, q):
    return round(float(np.percentile(x, q)), 3) if len(x) else None


def singles(fn, cases):
    """-> (ms per call, answers) of fn(case) called once per case."""
    times, out = [], []
    for c in cases:
        t0 = time.perf_counter()
        out.append(fn(c))
        times.append((time.perf_counter() - t0) * 1e3)
    return times, out


def concurrent(fn, cases):
    """-> (ms from the release of one thread per case until the last answer, answers)."""
    out, errs = [None] * len(cases), []
    gate = threading.Barrier(len(cases) + 1)

    def run(i):
        try:
            gate.wait()
            out[i] = fn(cases[i])
        except Exception as ex:  # noqa: BLE001
            errs.append(repr(ex))

    th = [threading.Thread(target=run, args=(i,)) for i in range(len(cases))]
    [x.start() for x in th]
    gate.wait()
    t0 = time.perf_counter()
    [x.join() for x in th]
    ms = (time.perf_counter() - t0) * 1e3
    if errs:
        raise RuntimeError(errs[0])
    return ms, out


def run(w, cases):
    import torch

    S = a.shards
    replica = zgpu.Engine(w.schema, device=0)
    handle = zgpu.Engine(w.schema, device=0, n_shards=S, handle_lookups=True, subquery_capacity=a.subq_cap)
    ts = zdist.LocalDeviceTransport.cluster(S)
    engines = [zgpu.Engine(w.schema, device=0, shard_rank=r, shard_count=S, subquery_capacity=a.subq_cap) for r in range(S)]
    for e in [replica, handle] + engines:
        w.load_into(e)
        e.publish()
    lks = [zdist.DeviceShardedLookup(engines[r], ts[r], verify_chunk=a.verify_chunk) for r in range(S)]
    e0 = engines[0]
    reqs = [(e0.type_id(rt), e0.slot_id(rt, p), e0.type_id("user"), u, zgpu.SREL_NONE) for rt, p, u in cases]
    T = int(time.time())

    def clock(t):
        for e in [replica, handle] + engines:
            e.set_clock(t)

    def driver(batches):
        """DeviceShardedLookup: rank 0 brings each batch, the other ranks none -> (ms per batch, answers per batch)."""
        times, got, errs = [], [], []

        def rank(r):
            try:
                for b in batches:
                    t0 = time.perf_counter()
                    ans = lks[r].lookup_resources(b if r == 0 else [])
                    if r == 0:
                        torch.cuda.synchronize()
                        times.append((time.perf_counter() - t0) * 1e3)
                        got.append(ans)
            except Exception as ex:  # noqa: BLE001
                errs.append(repr(ex))
                ts[r]._s["bar"].abort()

        th = [threading.Thread(target=rank, args=(r,)) for r in range(S)]
        [x.start() for x in th]
        [x.join() for x in th]
        if errs:
            raise RuntimeError(errs[0])
        return times, got

    lookup = lambda e: (lambda c: e.lookup_resources_ids(c[0], c[1], "user", c[2]))  # noqa: E731
    res, mism = {"lookups": len(cases) - a.warmup}, 0
    # one call per lookup
    clock(T)
    c0 = handle.handle_lookup_counters()
    ht, hans = singles(lookup(handle), cases)
    c1 = handle.handle_lookup_counters()
    dt, dans = driver([[q] for q in reqs])
    rt_, rans = singles(lookup(replica), cases)
    for h, d, r in zip(hans, dans, rans):
        mism += int(not np.array_equal(h, r)) + int(d[0] is None or not np.array_equal(d[0], r))
    for name, t in (("handle", ht), ("driver", dt), ("replica", rt_)):
        res[f"{name}_ms_median"], res[f"{name}_ms_p99"] = pct(t[a.warmup:], 50), pct(t[a.warmup:], 99)
    res["handle_counters_per_lookup"] = {k: round((c1[k] - c0[k]) / len(cases), 2) for k in c1}
    # all at once
    clock(T + 1)
    res["replica_all_at_once_ms"], rall = concurrent(lookup(replica), cases)
    res["handle_all_at_once_ms"], hall = concurrent(lookup(handle), cases)
    t, dall = driver([reqs])
    res["driver_all_in_one_call_ms"] = t[0]
    for h, d, r in zip(hall, dall[0], rall):
        mism += int(not np.array_equal(h, r)) + int(d is None or not np.array_equal(d, r))
    for k in ("replica_all_at_once_ms", "handle_all_at_once_ms", "driver_all_in_one_call_ms"):
        res[k] = round(res[k], 3)
    res["answer_ids"] = int(sum(len(x) for x in rans))
    res["mismatches_vs_replica"] = mism
    for e in [replica, handle] + engines:
        e.close()
    return res


def main():
    rng = np.random.default_rng(11)
    result = {"shards": a.shards, "scale": a.scale}
    mismatches = 0
    specs = [("cfg2", workloads.cfg2(scale=min(1.0, 4 * a.scale)), [("pod", "view")]),
             ("cfg3", workloads.cfg3(scale=a.scale), [("namespace", "view")]),
             ("cfg4", workloads.cfg4(scale=a.scale), [("document", "view"), ("document", "restricted_view")])]
    for name, w, perms in specs:
        users = rng.permutation(users_of(w))[: a.subjects // len(perms)]  # distinct: no answer comes from the cache
        cases = [(rt, p, int(u)) for rt, p in perms for u in users]
        print(f"{name}: {len(cases)} lookups", file=sys.stderr, flush=True)
        result[name] = run(w, cases)
        mismatches += result[name]["mismatches_vs_replica"]
    result.update(mismatches_vs_replica=mismatches, **gpu_info())
    print(json.dumps(result))


if __name__ == "__main__":
    main()
