"""WriteRelationships-sized updates against the full cfg4 store: wall and device time of the incremental publish
(csrc/delta.cuh) next to a rebuild. Under `ncu -k regex:delta_ --metrics gpu__time_duration.sum` it gives the
per-kernel split.

    python scripts/write_bench.py [--scale 1.0] [--writes 8] [--updates 1000]
"""
import argparse, json, os, sys, time
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import zgpu
from spicedb_kubeapi_proxy_b200 import workloads
from test_gpu_parity import _random_updates

ap = argparse.ArgumentParser()
ap.add_argument("--scale", type=float, default=1.0)
ap.add_argument("--writes", type=int, default=8)
ap.add_argument("--updates", type=int, default=1000)
a = ap.parse_args()
w = workloads.cfg4(scale=a.scale)
e = zgpu.Engine(w.schema)
w.load_into(e)
t0 = time.perf_counter(); e.publish(); full_wall = time.perf_counter() - t0
full_dev = e.stats()["last_publish_ms"]
rng = np.random.default_rng(3)
# the first write after a bulk load also builds the host relationship index (Store::ensure_index): timed on its own
t0 = time.perf_counter(); e.apply_updates(_random_updates(zgpu, e, w, rng, 4, new_objects=False)); e.publish()
first_write_wall = time.perf_counter() - t0
wall, dev, apply_ms = [], [], []
for i in range(a.writes):
    ups = _random_updates(zgpu, e, w, rng, a.updates, new_objects=(i % 2 == 1))
    t0 = time.perf_counter(); e.apply_updates(ups); t1 = time.perf_counter(); e.publish(); t2 = time.perf_counter()
    apply_ms.append((t1 - t0) * 1e3); wall.append((t2 - t0) * 1e3); dev.append(e.stats()["last_publish_ms"])
st = e.stats()
print(json.dumps({"store_tuples": int(st["tuples"]), "updates_per_write": a.updates, "wall_ms": wall, "apply_ms": apply_ms,
                  "device_ms": dev, "delta_publishes": int(st["delta_publishes"]), "full_publishes": int(st["full_publishes"]),
                  "full_rebuild_device_ms": full_dev, "full_rebuild_wall_ms": full_wall * 1e3,
                  "first_write_after_load_wall_ms": first_write_wall * 1e3}))
