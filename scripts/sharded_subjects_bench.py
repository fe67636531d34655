"""LookupSubjects on the object-hash sharded store (dist.DeviceShardedLookup.lookup_subjects), against a replica engine.

One process: W virtual shards on ONE GPU (LocalDeviceTransport, one thread per shard). That measures the protocol's
overhead (levels, exchanges, the two sharded verifications), not multi-GPU scaling. Under torch.distributed.run: one
process per GPU (TorchDeviceTransport over NCCL). Workloads: cfg3 namespace#view, cfg4 document#view and
document#restricted_view, for user subjects of a few hundred seeded resources. Every answer (ids, wildcard entry,
exclusions) is compared with the replica's zg_lookup_subjects. Prints one JSON line with the GPU name and its enforced
power limit, read in the same run.

    python scripts/sharded_subjects_bench.py [--world 4] [--resources 200] [--scale 0.1]
    torchrun --nproc-per-node 2 scripts/sharded_subjects_bench.py --resources 200
"""
import argparse, json, os, sys, threading, time
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import zgpu
from spicedb_kubeapi_proxy_b200 import dist as zdist, workloads

ap = argparse.ArgumentParser()
ap.add_argument("--world", type=int, default=4, help="virtual shards on one GPU (ignored under torch.distributed)")
ap.add_argument("--resources", type=int, default=200)
ap.add_argument("--scale", type=float, default=0.1, help="workload scale of cfg3 and cfg4")
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--verify-chunk", type=int, default=1 << 12, help="candidates per sharded check_bulk call")
ap.add_argument("--subq-cap", type=int, default=1 << 24, help="zg_config.subquery_capacity of the shards")
a = ap.parse_args()

STATS = ("levels", "candidates", "entries_sent", "admitted", "nowild_verified", "fallbacks", "halvings")


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


def same(got, want):
    return got is not None and np.array_equal(got[0], want[0]) and got[1] == want[1] and np.array_equal(got[2], want[2])


def compare(w, cases, answers, dev):
    """-> (replica times in ms, mismatches) for the per-lookup answers."""
    replica = zgpu.Engine(w.schema, device=dev)
    w.load_into(replica)
    replica.publish()
    rtimes, mism = [], 0
    for i, (rt, r, p) in enumerate(cases):
        t0 = time.perf_counter()
        want = replica.lookup_subjects_ids(rt, r, p, "user")
        rtimes.append((time.perf_counter() - t0) * 1e3)
        mism += int(not same(answers[i], want))
    return rtimes, mism, replica


def summary(cases, times, rtimes, mism, stats):
    n = len(cases) - a.warmup
    t, rt_ = times[a.warmup:], rtimes[a.warmup:]
    per = {k: round(stats[k] / max(n, 1), 2) for k in STATS}  # rank 0's counts per timed lookup
    return {"lookups": n, "sharded_ms_median": pct(t, 50), "sharded_ms_p99": pct(t, 99), "replica_ms_median": pct(rt_, 50),
            "replica_ms_p99": pct(rt_, 99), "mismatches_vs_replica": mism, "rank0_per_lookup": per}


def single_process(w, cases):
    """W virtual shards in threads; rank 0 asks every lookup, one call per lookup, then all of them in one call."""
    import torch

    world = a.world
    ts = zdist.LocalDeviceTransport.cluster(world)
    engines = [zgpu.Engine(w.schema, device=0, shard_rank=r, shard_count=world, subquery_capacity=a.subq_cap)
               for r in range(world)]
    for e in engines:
        w.load_into(e)
        e.publish()
    lks = [zdist.DeviceShardedLookup(engines[r], ts[r], verify_chunk=a.verify_chunk) for r in range(world)]
    e0 = engines[0]
    reqs = [(e0.type_id(rt), r, e0.slot_id(rt, p), e0.type_id("user"), zgpu.SREL_NONE, 0) for rt, r, p in cases]
    times, answers, errs, batch = [], [None] * len(reqs), [], []

    def rank(r):
        try:
            for i, q in enumerate(reqs):
                if i == a.warmup and r == 0:
                    for k in lks[0].stats:
                        lks[0].stats[k] = 0
                t0 = time.perf_counter()
                got = lks[r].lookup_subjects([q] if r == 0 else [])
                if r == 0:
                    torch.cuda.synchronize()
                    times.append((time.perf_counter() - t0) * 1e3)
                    answers[i] = got[0]
            if r == 0:
                stats.update(lks[0].stats)
            t0 = time.perf_counter()
            got = lks[r].lookup_subjects(reqs if r == 0 else [])
            if r == 0:
                batch.extend([(time.perf_counter() - t0) * 1e3, got])
        except Exception as ex:  # noqa: BLE001
            errs.append(repr(ex))
            ts[r]._s["bar"].abort()

    stats = {}
    th = [threading.Thread(target=rank, args=(r,)) for r in range(world)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    if errs:
        raise RuntimeError(errs[0])
    rtimes, mism, replica = compare(w, cases, answers, 0)
    for i, (rt, r, p) in enumerate(cases):
        mism += int(not same(batch[1][i], replica.lookup_subjects_ids(rt, r, p, "user")))
    out = summary(cases, times, rtimes, mism, stats)
    out["sharded_all_in_one_call_ms"] = round(batch[0], 3)
    return out


def multi_process(w, cases):
    import torch
    import torch.distributed as tdist

    if not tdist.is_initialized():
        tdist.init_process_group("nccl")
    r, world = tdist.get_rank(), tdist.get_world_size()
    torch.cuda.set_device(r % torch.cuda.device_count())
    dev = torch.cuda.current_device()
    e = zgpu.Engine(w.schema, device=dev, shard_rank=r, shard_count=world, subquery_capacity=a.subq_cap)
    w.load_into(e)
    e.publish()
    lk = zdist.DeviceShardedLookup(e, zdist.TorchDeviceTransport(), verify_chunk=a.verify_chunk)
    reqs = [(e.type_id(rt), res, e.slot_id(rt, p), e.type_id("user"), zgpu.SREL_NONE, 0) for rt, res, p in cases]
    times, answers = [], []
    for i, q in enumerate(reqs):
        if i == a.warmup:
            for k in lk.stats:
                lk.stats[k] = 0
        tdist.barrier()
        t0 = time.perf_counter()
        got = lk.lookup_subjects([q] if r == 0 else [])
        if r == 0:
            times.append((time.perf_counter() - t0) * 1e3)
            answers.append(got[0])
    out = None
    if r == 0:
        rtimes, mism, _ = compare(w, cases, answers, dev)
        out = summary(cases, times, rtimes, mism, lk.stats)
    tdist.barrier()
    return out, world


def main():
    distributed = "RANK" in os.environ and "WORLD_SIZE" in os.environ
    rng = np.random.default_rng(13)
    result = {"transport": "TorchDeviceTransport (nccl)" if distributed else "LocalDeviceTransport (virtual shards, one GPU)"}
    mismatches = 0
    specs = [("cfg3", workloads.cfg3(scale=a.scale), [("namespace", "view")]),
             ("cfg4", workloads.cfg4(scale=a.scale), [("document", "view"), ("document", "restricted_view")])]
    world = a.world
    for name, w, perms in specs:
        rt = perms[0][0]
        res = np.unique(np.concatenate([g.res for g in w.groups if g.res_type == rt and g.res.size]))
        picked = rng.choice(res, size=min(a.resources, res.size), replace=False)
        cases = [(rt, int(r), p) for _, p in perms for r in picked[: a.resources // len(perms)]]
        print(f"{name}: {len(cases)} lookups", file=sys.stderr, flush=True)
        if distributed:
            res_, world = multi_process(w, cases)
        else:
            res_ = single_process(w, cases)
        if res_ is not None:
            result[name] = res_
            mismatches += res_["mismatches_vs_replica"]
    if not distributed or int(os.environ["RANK"]) == 0:
        result.update(world=world, scale=a.scale, mismatches_vs_replica=mismatches, **gpu_info())
        print(json.dumps(result))


if __name__ == "__main__":
    main()
