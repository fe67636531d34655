"""Where a check kernel's warp spends its cycles, per phase, on the BASELINE workloads cfg3 and cfg4 (full size by
default): admission, root visit, two-level meet, one-level meet and pop loop (the visits exclude the meets inside
them). Runs the batch device-resident as bench.py does (L2 flushed before every step) and divides each phase's
warp-cycle total by the checks answered. Needs a library built with the counters:

    scripts/build_variant.sh phase "-DZG_PHASE_CLOCKS=1"
    ZGPU_LIB=spicedb-kubeapi-proxy_b200/variants/libzgpu_phase.so python scripts/phase_clocks.py [--steps 20]

The counters cost time themselves, so the rate printed beside them is not the library's rate. Prints one JSON line
with the GPU name and its enforced power limit, read in the same run.
"""
import argparse, json, os, sys
import numpy as np
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import zgpu
from spicedb_kubeapi_proxy_b200 import workloads

ap = argparse.ArgumentParser()
ap.add_argument("--scale", type=float, default=1.0)
ap.add_argument("--steps", type=int, default=20)
ap.add_argument("--workloads", default="cfg3,cfg4")
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
        return {"gpu": torch.cuda.get_device_name(0), "power_limit_w": None, "nvml_error": repr(ex)}


def run(name):
    w = workloads.by_name(name, a.scale)
    e = zgpu.Engine(w.schema)
    w.load_into(e)
    e.publish()
    items = w.check_items(e, zgpu.CHECK_DTYPE)
    n = items.size
    d_items = torch.from_numpy(items.view(np.uint8).copy()).cuda()
    d_out = torch.zeros(n, dtype=torch.uint8, device="cuda")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    stream = torch.cuda.current_stream()
    for _ in range(3):
        e.check_bulk_device(d_items.data_ptr(), n, d_out.data_ptr(), stream.cuda_stream)
    torch.cuda.synchronize()
    c0 = e.phase_clocks()
    ms = 0.0
    for _ in range(a.steps):
        flush.zero_()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record(stream)
        e.check_bulk_device(d_items.data_ptr(), n, d_out.data_ptr(), stream.cuda_stream)
        t1.record(stream)
        torch.cuda.synchronize()
        ms += t0.elapsed_time(t1)
    c1 = e.phase_clocks()
    per = {k: (c1[k] - c0[k]) / (n * a.steps) for k in c0}
    total = sum(per.values())
    out = {"workload": name, "scale": a.scale, "checks_per_step": n, "steps": a.steps,
           "warp_cycles_per_check": {k: round(v, 1) for k, v in per.items()},
           "share": {k: round(v / total, 4) if total else 0.0 for k, v in per.items()},
           "mchecks_s_with_counters": round(n * a.steps / ms / 1e3, 1)}
    del e
    return out


rows = [run(x) for x in a.workloads.split(",")]
print(json.dumps({**gpu_info(), "lib": os.path.basename(os.environ.get("ZGPU_LIB", "libzgpu.so")), "results": rows}))
