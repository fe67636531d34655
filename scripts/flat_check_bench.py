"""cfg3 with the lean flat-check kernel on and off (ZGPU_FLAT_CHECK=0), device-resident, timed like bench.py's
headline (CUDA events around zg_check_bulk_device, L2 flushed outside the events). Prints one JSON line per
configuration, then, with --profile, the per-kernel device times of a run of its own under torch.profiler.

  python scripts/flat_check_bench.py [--steps 200] [--scale 1.0] [--libs NAME=PATH ...] [--sig-words 8,16] [--profile]

--libs runs the same measurement over other builds of the library (scripts/build_variant.sh, e.g. the lean kernel's
launch bounds -DZG_FLAT_MIN_BLOCKS=6, or the parent commit's library), each in a child process (ZGPU_LIB). Every
configuration's answers are compared with the first one's."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def measure(args):
    import numpy as np
    import torch

    import zgpu
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.cfg3(scale=args.scale)
    eng = zgpu.Engine(w.schema, device=0)
    w.load_into(eng)
    eng.publish()
    items = w.check_items(eng, zgpu.CHECK_DTYPE)
    n = items.size
    d_items = torch.from_numpy(items.view(np.uint8).copy()).cuda()
    d_out = torch.zeros(n, dtype=torch.uint8, device="cuda")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    stream = torch.cuda.current_stream()

    def step():
        eng.check_bulk_device(d_items.data_ptr(), n, d_out.data_ptr(), stream.cuda_stream)

    alg = eng.count_alg_bytes(items) / n
    for _ in range(10):
        flush.zero_()
        step()
    torch.cuda.synchronize()
    st0 = eng.stats()
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
    for a, b in evs:
        flush.zero_()
        a.record(stream)
        step()
        b.record(stream)
    torch.cuda.synchronize()
    ms = sorted(a.elapsed_time(b) for a, b in evs)
    st1 = eng.stats()
    res = {"flat_check": os.environ.get("ZGPU_FLAT_CHECK", "1"), "flat_records": os.environ.get("ZGPU_FLAT_RECORDS", "1"),
           "lib": os.environ.get("ZGPU_LIB", "default"),
           "sig_words": os.environ.get("ZGPU_CLOSURE_SIG_WORDS", "chosen"), "checks": n,
           "mean_ms": sum(ms) / len(ms), "median_ms": ms[len(ms) // 2], "min_ms": ms[0],
           "mchecks_per_s": n / (sum(ms) / len(ms)) / 1e3, "alg_bytes_per_check": round(alg, 2),
           "launches_per_step": (st1["launches"] - st0["launches"]) / args.steps,
           "flat_slots": st1["flat_slots"], "residual_per_step": (st1["flat_residual"] - st0["flat_residual"]) / args.steps,
           "answers_sha": __import__("hashlib").sha1(d_out.cpu().numpy().tobytes()).hexdigest()[:16]}
    if hasattr(eng, "flat_record_info"):
        try:
            res["records"] = eng.flat_record_info(0)
        except Exception as ex:  # no records in this configuration
            res["records"] = repr(ex)[:80]
    if args.profile:
        from torch.profiler import ProfilerActivity, profile

        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(20):
                flush.zero_()
                step()
            torch.cuda.synchronize()
        kern = {}
        for e in prof.key_averages():
            if "check_kernel" in e.key or "flat_check" in e.key or "memset" in e.key.lower():
                kern[e.key[:60]] = {"calls": e.count, "avg_us": round(e.device_time_total / max(e.count, 1), 2)}
        res["kernels"] = kern
    print(json.dumps(res), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--libs", nargs="*", default=[], help="NAME=PATH of other library builds to measure")
    ap.add_argument("--sig-words", default="", help="comma-separated ZGPU_CLOSURE_SIG_WORDS values to compare")
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        return measure(args)
    try:
        print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True).stdout.strip(), flush=True)
    except OSError:
        pass
    confs = [{}, {"ZGPU_FLAT_CHECK": "0"}, {"ZGPU_FLAT_RECORDS": "0"}]
    confs += [{"ZGPU_LIB": p.split("=", 1)[1]} for p in args.libs]
    confs += [{"ZGPU_CLOSURE_SIG_WORDS": x} for x in args.sig_words.split(",") if x]
    base = [sys.executable, os.path.abspath(__file__), "--child", "--steps", str(args.steps), "--scale", str(args.scale)]
    shas = []
    for c in confs:
        env = dict(os.environ, **c)
        r = subprocess.run(base, env=env, capture_output=True, text=True)
        line = (r.stdout.strip().splitlines() or [""])[-1]
        print(line if r.returncode == 0 else f"{c}: failed {r.stderr[-2000:]}", flush=True)
        if r.returncode == 0:
            shas.append(json.loads(line)["answers_sha"])
    if args.profile:
        for c in confs[:3]:
            r = subprocess.run(base + ["--profile"], env=dict(os.environ, **c), capture_output=True, text=True)
            print((r.stdout.strip().splitlines() or [""])[-1] if r.returncode == 0 else r.stderr[-2000:], flush=True)
    print(json.dumps({"answers_identical": len(set(shas)) == 1, "configs": len(shas), "time": time.time()}), flush=True)


if __name__ == "__main__":
    main()
