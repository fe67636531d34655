"""The sharded handle (zg_config.n_shards) against the two other ways to answer the same batch: cfg4 on S virtual shards of
ONE GPU, batches of 1 M checks, three paths over the same shards and the same batch:
  handle   one engine holding the S shards, zg_check_bulk (in-process exchange through device memory)
  dist     dist.DeviceShardedChecker over LocalDeviceTransport on S one-shard engines (one thread per shard)
  replica  one engine holding the whole store
Every path's answers are compared; a mismatch fails the run. Also: levels and host round trips per batch, the wall time
of a 1 000-update write on the handle (the first after the bulk load, then a steady-state one), and the GPU name and enforced power limit read in the same run. One JSON line.
Virtual shards share one card, so this measures the protocol's cost, not multi-GPU scaling or peer traffic.

    python scripts/sharded_handle_bench.py [--scale 1.0] [--shards 4] [--iters 10]
"""
import argparse, json, os, sys, threading, time
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import zgpu
from spicedb_kubeapi_proxy_b200 import _lib, dist as zdist, workloads

ap = argparse.ArgumentParser()
ap.add_argument("--scale", type=float, default=1.0, help="cfg4 scale: 1.0 = 95.4 M relationships")
ap.add_argument("--shards", type=int, default=4)
ap.add_argument("--batch", type=int, default=1 << 20)
ap.add_argument("--iters", type=int, default=10)
ap.add_argument("--warmup", type=int, default=2)
ap.add_argument("--subq-cap", type=int, default=1 << 24, help="zg_config.subquery_capacity of every engine")
ap.add_argument("--out", default="", help="also write the JSON line to this file")
a = ap.parse_args()


def gpu_info():
    try:
        import pynvml as nv
        nv.nvmlInit()
        h = nv.nvmlDeviceGetHandleByIndex(0)
        name = nv.nvmlDeviceGetName(h)
        return {"gpu": name.decode() if isinstance(name, bytes) else name,
                "power_limit_w": nv.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0}
    except Exception as ex:  # noqa: BLE001  (reported beside the numbers)
        import torch
        return {"gpu": torch.cuda.get_device_name(0), "power_limit_w": None, "nvml_error": repr(ex)}


def stats_ms(x):
    return {"median": round(float(np.median(x)), 3), "p99": round(float(np.percentile(x, 99)), 3)}


def main():
    import torch

    S = a.shards
    t0 = time.perf_counter()
    w = workloads.cfg4(scale=a.scale)
    handle = zgpu.Engine(w.schema, device=0, n_shards=S, subquery_capacity=a.subq_cap)
    replica = zgpu.Engine(w.schema, device=0, subquery_capacity=a.subq_cap)
    shards = [zgpu.Engine(w.schema, device=0, shard_rank=r, shard_count=S, subquery_capacity=a.subq_cap) for r in range(S)]
    for e in [handle, replica] + shards:
        w.load_into(e)
        e.publish()
    load_s = time.perf_counter() - t0
    items = w.check_items(handle, zgpu.CHECK_DTYPE)[: a.batch]
    n = items.size
    pinned = _lib.PinnedArray((n,), zgpu.CHECK_DTYPE)
    pinned.array[:] = items
    out_h, out_r = _lib.PinnedArray((n,), np.uint8), _lib.PinnedArray((n,), np.uint8)

    ts = zdist.LocalDeviceTransport.cluster(S)
    checkers = [zdist.DeviceShardedChecker(shards[r], ts[r]) for r in range(S)]
    bounds = [zdist.shard_bounds(n, r, S) for r in range(S)]
    d_slices = [torch.from_numpy(np.ascontiguousarray(items[lo:hi]).view(np.uint8).copy()).cuda() for lo, hi in bounds]
    got_d = [None] * S

    def dist_batch():
        errs = []

        def run(r):
            try:
                got_d[r] = checkers[r].check_bulk(d_slices[r], bounds[r][1] - bounds[r][0])
            except Exception as ex:  # noqa: BLE001
                errs.append(repr(ex))
                ts[r]._s["bar"].abort()

        th = [threading.Thread(target=run, args=(r,)) for r in range(S)]
        [x.start() for x in th]
        [x.join() for x in th]
        torch.cuda.synchronize()
        if errs:
            raise RuntimeError(errs)
        return np.concatenate([g.cpu().numpy() for g in got_d])

    paths = {
        "handle": lambda: handle.check_bulk(pinned.array, out_h.array),
        "dist": dist_batch,
        "replica": lambda: replica.check_bulk(pinned.array, out_r.array),
    }
    answers = {k: np.array(f(), copy=True) for k, f in paths.items()}  # first call of each path: warm-up as well
    for _ in range(max(0, a.warmup - 1)):
        for f in paths.values():
            f()
    ms = {k: [] for k in paths}
    for _ in range(a.iters):  # alternating paths, each timed to its answers on the host
        for k, f in paths.items():
            t = time.perf_counter()
            f()
            ms[k].append((time.perf_counter() - t) * 1e3)
    st = handle.stats()
    levels, round_trips, subq = st["last_levels"], st["last_round_trips"], st["last_subqueries"]
    identical = bool(np.array_equal(answers["handle"], answers["replica"]) and np.array_equal(answers["dist"], answers["replica"]))
    # 1 000-update writes: TOUCH of banned relationships on documents of the batch, merged into every shard. The first
    # write after a bulk load also builds the host relationship index (DESIGN.md §8), on the handle as on a replica;
    # the second is the steady-state write.
    def write(k):
        up = np.zeros(1000, dtype=zgpu.UPDATE_DTYPE)
        up["res"] = items["res"][k * 1000:(k + 1) * 1000]
        up["subj"] = np.arange(1000) % 97
        up["rel"], up["stype"], up["srel"], up["op"] = handle.slot_id("document", "banned"), handle.type_id("user"), zgpu.SREL_NONE, _lib.OP_TOUCH
        t = time.perf_counter()
        handle.apply_updates(up)
        handle.publish()
        ms = (time.perf_counter() - t) * 1e3
        replica.apply_updates(up), replica.publish()
        return ms

    first_write_ms = write(0)
    d0 = handle.stats()["delta_publishes"]
    write_ms = write(1)
    merged = handle.stats()["delta_publishes"] - d0
    after_identical = bool(np.array_equal(handle.check_bulk(pinned.array), replica.check_bulk(pinned.array)))
    res = {"bench": "sharded_handle", "workload": "cfg4", "scale": a.scale, "relationships": int(replica.stats()["tuples"]),
           "shards": S, "virtual_shards_on_one_gpu": True, "batch": n, "iters": a.iters,
           "ms_per_batch": {k: stats_ms(v) for k, v in ms.items()},
           "levels_per_batch": int(levels), "host_round_trips_per_batch": int(round_trips), "subqueries_per_batch": int(subq),
           "dist_levels": int(checkers[0].stats["levels"]),
           "write_1000_updates_ms": round(write_ms, 3), "write_shards_merged": int(merged),
           "first_write_after_load_ms": round(first_write_ms, 3),
           "answers_identical": identical, "answers_identical_after_write": after_identical,
           "has_fraction": round(float((answers["replica"] == zgpu.HAS_PERMISSION).mean()), 4), "load_s": round(load_s, 1)}
    res.update(gpu_info())
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")
    if not (identical and after_identical):
        sys.exit(1)


if __name__ == "__main__":
    main()
