"""LookupResources on the object-hash sharded store (dist.DeviceShardedLookup), against a replica engine.

One process: W virtual shards on ONE GPU (LocalDeviceTransport, one thread per shard). That measures the protocol's
overhead (levels, exchanges, the sharded verification), not multi-GPU scaling. Under torch.distributed.run: one
process per GPU (TorchDeviceTransport over NCCL). Workloads: cfg2 pod#view, cfg3 namespace#view, cfg4 document#view
and document#restricted_view, each for a few hundred seeded users. Every answer is compared with the replica's.
Prints one JSON line with the GPU name and its enforced power limit, read in the same run.

    python scripts/sharded_lookup_bench.py [--world 4] [--subjects 300] [--scale 0.1]
    torchrun --nproc-per-node 2 scripts/sharded_lookup_bench.py --subjects 300
"""
import argparse, json, os, sys, threading, time
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import zgpu
from spicedb_kubeapi_proxy_b200 import dist as zdist, workloads

ap = argparse.ArgumentParser()
ap.add_argument("--world", type=int, default=4, help="virtual shards on one GPU (ignored under torch.distributed)")
ap.add_argument("--subjects", type=int, default=300)
ap.add_argument("--scale", type=float, default=0.1, help="cfg4 scale; cfg2 and cfg3 use 4x and 1x of it")
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--verify-chunk", type=int, default=1 << 12, help="candidates per sharded check_bulk call")
ap.add_argument("--subq-cap", type=int, default=1 << 24, help="zg_config.subquery_capacity of the shards")
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


def single_process(w, cases):
    """W virtual shards in threads; rank 0 asks every lookup, one call per lookup, then all of them in one call."""
    import torch

    world = a.world
    replica = zgpu.Engine(w.schema, device=0)
    w.load_into(replica)
    replica.publish()
    ts = zdist.LocalDeviceTransport.cluster(world)
    engines = [zgpu.Engine(w.schema, device=0, shard_rank=r, shard_count=world, subquery_capacity=a.subq_cap)
               for r in range(world)]
    for e in engines:
        w.load_into(e)
        e.publish()
    lks = [zdist.DeviceShardedLookup(engines[r], ts[r], verify_chunk=a.verify_chunk) for r in range(world)]
    e0 = engines[0]
    reqs = [(e0.type_id(rt), e0.slot_id(rt, p), e0.type_id("user"), u, zgpu.SREL_NONE) for rt, p, u in cases]
    times, answers, errs = [], [None] * len(reqs), []

    def rank(r, batch):
        try:
            for i, q in enumerate(reqs):
                if i == a.warmup and r == 0:
                    for k in lks[0].stats:
                        lks[0].stats[k] = 0
                t0 = time.perf_counter()
                got = lks[r].lookup_resources([q] if r == 0 else [])
                if r == 0:
                    torch.cuda.synchronize()
                    times.append((time.perf_counter() - t0) * 1e3)
                    answers[i] = got[0]
            t0 = time.perf_counter()
            got = lks[r].lookup_resources(reqs if r == 0 else [])
            if r == 0:
                batch.append((time.perf_counter() - t0) * 1e3)
                batch.append(got)
        except Exception as ex:  # noqa: BLE001
            errs.append(repr(ex))
            ts[r]._s["bar"].abort()

    batch = []
    th = [threading.Thread(target=rank, args=(r, batch)) for r in range(world)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    if errs:
        raise RuntimeError(errs[0])
    rtimes, mism = [], 0
    for i, (rt, p, u) in enumerate(cases):
        t0 = time.perf_counter()
        want = replica.lookup_resources_ids(rt, p, "user", u)
        rtimes.append((time.perf_counter() - t0) * 1e3)
        mism += int(answers[i] is None or not np.array_equal(answers[i], want))
        mism += int(batch[1][i] is None or not np.array_equal(batch[1][i], want))
    st = dict(lks[0].stats)  # the timed single lookups and the all-in-one call
    n = len(cases) - a.warmup
    t = times[a.warmup:]
    rt_ = rtimes[a.warmup:]
    return {"lookups": n, "sharded_ms_median": pct(t, 50), "sharded_ms_p99": pct(t, 99),
            "replica_ms_median": pct(rt_, 50), "replica_ms_p99": pct(rt_, 99),
            "sharded_all_in_one_call_ms": round(batch[0], 3), "answer_ids": int(sum(len(x) for x in answers if x is not None)),
            "mismatches_vs_replica": mism, "rank0_stats": st}


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
    reqs = [(e.type_id(rt), e.slot_id(rt, p), e.type_id("user"), u, zgpu.SREL_NONE) for rt, p, u in cases]
    times, answers = [], []
    for i, q in enumerate(reqs):
        tdist.barrier()
        t0 = time.perf_counter()
        got = lk.lookup_resources([q] if r == 0 else [])
        if r == 0:
            times.append((time.perf_counter() - t0) * 1e3)
            answers.append(got[0])
    out = None
    if r == 0:
        replica = zgpu.Engine(w.schema, device=dev)
        w.load_into(replica)
        replica.publish()
        rtimes, mism = [], 0
        for i, (rt, p, u) in enumerate(cases):
            t0 = time.perf_counter()
            want = replica.lookup_resources_ids(rt, p, "user", u)
            rtimes.append((time.perf_counter() - t0) * 1e3)
            mism += int(answers[i] is None or not np.array_equal(answers[i], want))
        t, rt_ = times[a.warmup:], rtimes[a.warmup:]
        out = {"lookups": len(t), "sharded_ms_median": pct(t, 50), "sharded_ms_p99": pct(t, 99),
               "replica_ms_median": pct(rt_, 50), "replica_ms_p99": pct(rt_, 99), "mismatches_vs_replica": mism,
               "rank0_stats": dict(lk.stats)}
    tdist.barrier()
    return out, world


def main():
    distributed = "RANK" in os.environ and "WORLD_SIZE" in os.environ
    rng = np.random.default_rng(11)
    result = {"transport": "TorchDeviceTransport (nccl)" if distributed else "LocalDeviceTransport (virtual shards, one GPU)"}
    mismatches = 0
    specs = [("cfg2", workloads.cfg2(scale=min(1.0, 4 * a.scale)), [("pod", "view")]),
             ("cfg3", workloads.cfg3(scale=a.scale), [("namespace", "view")]),
             ("cfg4", workloads.cfg4(scale=a.scale), [("document", "view"), ("document", "restricted_view")])]
    world = a.world
    for name, w, perms in specs:
        users = rng.integers(0, users_of(w), a.subjects)
        cases = [(rt, p, int(u)) for rt, p in perms for u in users[: a.subjects // len(perms)]]
        print(f"{name}: {len(cases)} lookups", file=sys.stderr, flush=True)
        if distributed:
            res, world = multi_process(w, cases)
        else:
            res = single_process(w, cases)
        if res is not None:
            result[name] = res
            mismatches += res["mismatches_vs_replica"]
    if not distributed or int(os.environ["RANK"]) == 0:
        result.update(world=world, scale=a.scale, mismatches_vs_replica=mismatches, **gpu_info())
        print(json.dumps(result))


if __name__ == "__main__":
    main()
