"""LookupSubjects on the BASELINE workloads: per-call wall time (host clock around the synchronous call), median
and p99, candidates verified, answer size and fallbacks, for cfg4 (`document#view`, `document#restricted_view`)
and cfg3 (`namespace#view`) over seeded resources. Every timed answer is checked against zg_check_bulk: listed
subjects check HAS, excluded ones NO, every other subject HAS exactly when the wildcard entry is present.
Prints one JSON line with the GPU name and its enforced power limit, read in the same run.

    python scripts/lookup_subjects_bench.py [--scale 1.0] [--resources 300] [--warmup 5]
"""
import argparse, json, os, sys, time
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import zgpu
from spicedb_kubeapi_proxy_b200 import workloads
from lookup_subjects_oracle import property_violations

ap = argparse.ArgumentParser()
ap.add_argument("--scale", type=float, default=1.0)
ap.add_argument("--cfg3-scale", type=float, default=1.0)
ap.add_argument("--resources", type=int, default=300)
ap.add_argument("--warmup", type=int, default=5)
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


def n_of(w, t):
    return max(int(max(g.res.max() if g.res_type == t and g.res.size else -1,
                       g.subj.max() if g.subj_type == t and not g.wildcard and g.subj.size else -1)) + 1 for g in w.groups)


def run(w, res_type, perms, scale):
    e = zgpu.Engine(w.schema)
    w.load_into(e)
    e.publish()
    n_res, n_users = n_of(w, res_type), n_of(w, "user")
    rng = np.random.default_rng(2024)
    res = rng.choice(n_res, size=min(a.resources, n_res), replace=False)
    out = []
    for perm in perms:
        for r in res[:a.warmup]:
            e.lookup_subjects_ids(res_type, int(r), perm, "user")
        wall, verified, size, fell, wild, bad = [], [], [], 0, 0, 0
        for r in res:
            c0 = e.lookup_subjects_counters()
            t0 = time.perf_counter()
            ids, w_, ex = e.lookup_subjects_ids(res_type, int(r), perm, "user")
            wall.append((time.perf_counter() - t0) * 1e3)
            c1 = e.lookup_subjects_counters()
            verified.append(c1["items_verified"] - c0["items_verified"])
            fell += c1["fallbacks"] - c0["fallbacks"]
            size.append(len(ids) + len(ex))
            wild += int(w_)
            bad += len(property_violations(e.check_bulk, zgpu.CHECK_DTYPE, int(r), e.slot_id(res_type, perm),
                                           e.type_id("user"), zgpu.SREL_NONE, n_users, ids, w_, ex)) > 0
        out.append({"workload": w.name, "scale": scale, "tuples": int(e.stats()["tuples"]), "permission": f"{res_type}#{perm}",
                    "calls": len(res), "wall_ms_median": float(np.median(wall)), "wall_ms_p99": float(np.percentile(wall, 99)),
                    "verified_median": float(np.median(verified)), "verified_max": int(max(verified)),
                    "answer_median": float(np.median(size)), "answer_max": int(max(size)), "wildcard_answers": wild,
                    "fallbacks": int(fell), "property_failures": int(bad)})
    del e
    return out


rows = run(workloads.cfg4(scale=a.scale), "document", ["view", "restricted_view"], a.scale)
rows += run(workloads.by_name("cfg3", a.cfg3_scale), "namespace", ["view"], a.cfg3_scale)
print(json.dumps({**gpu_info(), "results": rows, "ok": all(r["property_failures"] == 0 for r in rows)}))
