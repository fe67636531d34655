"""WriteRelationships-sized updates against the full cfg3 store, touching group#member and team#member (the classes of
its closure index, so every publish rebuilds the index): wall and device time of the write plus publish. Prints one
JSON line with the GPU name and its enforced power limit, read in the same run.

    python scripts/index_write_bench.py [--scale 1.0] [--writes 5] [--updates 1000]
"""
import argparse, json, os, sys, time
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import zgpu
from spicedb_kubeapi_proxy_b200 import workloads

ap = argparse.ArgumentParser()
ap.add_argument("--scale", type=float, default=1.0)
ap.add_argument("--writes", type=int, default=5)
ap.add_argument("--updates", type=int, default=1000)
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


def updates(e, w, rng, n):
    """n updates of group#member@user, team#member@group#member and namespace#viewer@team#member (the lean kernel's
    range records): half deletes of loaded relationships, half inserts of new pairings between existing objects (one
    update per relationship)."""
    ups = np.zeros(n, dtype=zgpu.UPDATE_DTYPE)
    gs = w.groups[:2] + [g for g in w.groups if (g.res_type, g.rel, g.subj_type) == ("namespace", "viewer", "team")]
    for i in range(n):
        g = gs[int(rng.integers(0, len(gs)))]
        ups["rel"][i], ups["stype"][i] = e.slot_id(g.res_type, g.rel), e.type_id(g.subj_type)
        ups["srel"][i] = zgpu.SREL_NONE if g.srel is None else e.slot_id(g.subj_type, g.srel)
        k = int(rng.integers(0, g.res.size))
        if rng.random() < 0.5:
            ups["res"][i], ups["subj"][i], ups["op"][i] = g.res[k], g.subj[k], 2
        else:
            ups["res"][i], ups["subj"][i], ups["op"][i] = g.res[int(rng.integers(0, g.res.size))], g.subj[k], 0
    key = np.stack([ups["rel"], ups["res"], ups["stype"], ups["srel"], ups["subj"]], axis=1)
    return ups[np.sort(np.unique(key, axis=0, return_index=True)[1])]


w = workloads.cfg3(scale=a.scale)
e = zgpu.Engine(w.schema)
w.load_into(e)
t0 = time.perf_counter(); e.publish(); full_wall = time.perf_counter() - t0
full_dev = e.stats()["last_publish_ms"]
rng = np.random.default_rng(3)
# the first write after a bulk load also builds the host relationship index (Store::ensure_index): timed on its own
t0 = time.perf_counter(); e.apply_updates(updates(e, w, rng, 4)); e.publish()
first_write_wall = time.perf_counter() - t0
wall, dev = [], []
for i in range(a.writes):
    ups = updates(e, w, rng, a.updates)
    t0 = time.perf_counter(); e.apply_updates(ups); e.publish(); wall.append((time.perf_counter() - t0) * 1e3)
    dev.append(e.stats()["last_publish_ms"])
st = e.stats()
out = {**gpu_info(), "store_tuples": int(st["tuples"]), "updates_per_write": a.updates, "wall_ms": wall, "device_ms": dev,
       "delta_publishes": int(st["delta_publishes"]), "full_rebuild_device_ms": full_dev,
       "full_rebuild_wall_ms": full_wall * 1e3, "first_write_after_load_wall_ms": first_write_wall * 1e3}
if hasattr(e, "closure_index_counters"):
    out["closure_index"] = e.closure_index_counters()
if hasattr(e, "flat_record_info"):
    out["flat_records"] = e.flat_record_info(0)  # build_us: the last rebuild, after the last write
print(json.dumps(out))
