"""String ingress on the host vs on the device, on named cfg2 / cfg3 / cfg4 stores (users u%07d, pods ns%05d/p%07d,
other types <type>%07d: workloads.object_name). One JSON line per (workload, batch size):
  host_resolve_ms        zg_resolve_checks_packed, wall (median), and the host threads it uses
  dev_resolve_ms         zg_resolve_checks_packed_device, CUDA events, ids already on the device (median)
  packed_ms / ingress_ms zg_check_bulk_packed vs zg_check_bulk_packed_ingress, wall, median and p99 after warm-up;
                         the answers of every timed call are compared
  cold_sync_ms, mirror_bytes, write_sync_ms   the first call's sync of every name, and the sync after a write of
                         1 000 updates that name new objects (a 1-item device resolve, wall)
plus the GPU's name and power limit, read in the same run.

    python scripts/ingress_bench.py [--workloads cfg2,cfg3,cfg4] [--cfg4-scale 0.05] [--steps 20] [--warmup 3]
"""
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

BATCHES = (1_000, 10_000, 100_000, 1_000_000)


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        name, power = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
        return name, power
    except Exception as ex:  # noqa: BLE001
        return "unknown", repr(ex)


def stats(ts):
    a = np.array(ts) * 1e3
    return round(float(np.median(a)), 4), round(float(np.percentile(a, 99)), 4)


def run(name, scale, steps, warmup, info):
    import torch

    w = workloads.by_name(name, scale=scale)
    e = zgpu.Engine(w.schema, device=0)
    L = e._L
    t0 = time.perf_counter()
    n_names = workloads.intern_names(w, e)
    w.load_into(e)
    e.publish()
    setup_s = time.perf_counter() - t0
    c = w.checks[0]
    rt, perm, st = c.res_type.encode(), c.perm.encode(), c.subj_type.encode()
    big = max(BATCHES)
    reps = -(-big // c.res.size)
    res_all = np.tile(c.res, reps)[:big]
    sub_all = np.tile(c.subj, reps)[:big]
    res_names = [workloads.object_name(c.res_type, int(i)) for i in res_all]
    sub_names = [workloads.object_name(c.subj_type, int(i)) for i in sub_all]
    s = torch.cuda.Stream()

    # cold sync: the first device-ingress call mirrors every name
    one_blob, one_off = e.pack_ids(res_names[:1])
    d1, d1o = torch.frombuffer(bytearray(one_blob), dtype=torch.uint8).cuda(), torch.from_numpy(one_off.view(np.int32)).cuda()
    d1out = torch.zeros(16, dtype=torch.uint8, device="cuda")
    one_subj = sub_names[0].encode()

    def dev1():
        t = time.perf_counter()
        e._ck(L.zg_resolve_checks_packed_device(e._h, rt, perm, st, b"", d1.data_ptr(), d1o.data_ptr(), one_subj, None, 1,
                                                d1out.data_ptr(), s.cuda_stream))
        return time.perf_counter() - t

    cold = dev1()
    mirror_bytes = e.ingress_counters()["device_bytes"]
    idle = min(dev1() for _ in range(5))
    rel = next(g for g in w.groups if not g.srel and not g.wildcard)  # a write that names a new resource and subject
    e.write_relationships([(0, "%s:bench-new-%d#%s@%s:bench-newsubj-%d" % (rel.res_type, i, rel.rel, rel.subj_type, i), 0)
                           for i in range(1000)])
    e.publish()
    after_write = dev1()
    hw = os.cpu_count() or 1
    for n in BATCHES:
        blob, off = e.pack_ids(res_names[:n])
        sblob, soff = e.pack_ids(sub_names[:n])
        out_items = np.zeros(n, dtype=zgpu.CHECK_DTYPE)
        a_packed, a_ing = np.empty(n, dtype=np.uint8), np.empty(n, dtype=np.uint8)

        def host_resolve():
            e._ck(L.zg_resolve_checks_packed(e._h, rt, perm, st, b"", blob, off.ctypes.data, sblob, soff.ctypes.data, n,
                                             out_items.ctypes.data))

        def packed():
            e._ck(L.zg_check_bulk_packed(e._h, rt, perm, st, b"", blob, off.ctypes.data, sblob, soff.ctypes.data, n,
                                         a_packed.ctypes.data))

        def ingress():
            e._ck(L.zg_check_bulk_packed_ingress(e._h, rt, perm, st, b"", blob, off.ctypes.data, sblob, soff.ctypes.data, n,
                                                 a_ing.ctypes.data))

        db = torch.frombuffer(bytearray(blob), dtype=torch.uint8).cuda()
        do = torch.from_numpy(off.view(np.int32)).cuda()
        dsb = torch.frombuffer(bytearray(sblob), dtype=torch.uint8).cuda()
        dso = torch.from_numpy(soff.view(np.int32)).cuda()
        dout = torch.zeros(n * 16, dtype=torch.uint8, device="cuda")
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

        def dev_resolve():
            with torch.cuda.stream(s):
                ev0.record(s)
                e._ck(L.zg_resolve_checks_packed_device(e._h, rt, perm, st, b"", db.data_ptr(), do.data_ptr(),
                                                        dsb.data_ptr(), dso.data_ptr(), n, dout.data_ptr(), s.cuda_stream))
                ev1.record(s)
            ev1.synchronize()
            return ev0.elapsed_time(ev1) / 1e3

        def wall(fn):
            t = time.perf_counter()
            fn()
            return time.perf_counter() - t

        for _ in range(warmup):
            host_resolve(), dev_resolve(), packed(), ingress()
        host_t = [wall(host_resolve) for _ in range(steps)]
        dev_t = [dev_resolve() for _ in range(steps)]
        same_items = dout.cpu().numpy().view(zgpu.CHECK_DTYPE).tobytes() == out_items.tobytes()
        p_t, i_t, mismatches = [], [], 0
        for _ in range(steps):
            p_t.append(wall(packed))
            i_t.append(wall(ingress))
            mismatches += int((a_packed != a_ing).sum())
        pm, pp = stats(p_t)
        im, ip = stats(i_t)
        line = {
            "bench": "ingress", "workload": name, "scale": scale, "batch": n, "names": n_names,
            "gpu": info[0], "power_limit": info[1],
            "host_resolve_ms": stats(host_t)[0], "host_threads": int(min(n // 16384, hw, 16)) or 1,
            "dev_resolve_ms": stats(dev_t)[0], "items_identical": bool(same_items),
            "packed_ms": pm, "packed_p99_ms": pp, "ingress_ms": im, "ingress_p99_ms": ip, "answer_mismatches": mismatches,
            "cold_sync_ms": round(cold * 1e3, 3), "idle_call_ms": round(idle * 1e3, 4),
            "write_sync_ms": round(after_write * 1e3, 4), "mirror_bytes": int(mirror_bytes),
            "setup_s": round(setup_s, 1), "steps": steps, "warmup": warmup,
        }
        print(json.dumps(line), flush=True)
    e.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="cfg2,cfg3,cfg4")
    ap.add_argument("--cfg4-scale", type=float, default=0.05)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    info = gpu_info()
    for name in a.workloads.split(","):
        run(name, a.cfg4_scale if name == "cfg4" else 1.0, a.steps, a.warmup, info)


if __name__ == "__main__":
    main()
