"""BASELINE config 5 replayed at the C ABI: many concurrent clients, each submitting one
list-sized CheckBulkPermissions (the post-filter shape, pkg/authz/postfilter.go:127-134) and one
LookupResources (the pre-filter shape, pkg/authz/lookups.go:65) against the cfg4 store.
The true end-to-end path (Go HTTP handlers) cannot run here (no Go toolchain); this drives the
same library entry points from threads (ctypes releases the GIL inside the calls).

    python scripts/cfg5_replay.py [--scale 1.0] [--clients 1000] [--items 10000] [--rounds 2] [--devices 8]

--devices N: ONE engine handle owning N GPUs (zg_config.n_devices: a replica per device, every bulk call and every
batch of lookups split across them) -- BASELINE config 5 names 8 GPUs behind the proxy's single client.
A third phase runs both shapes at once (the proxy's pre-filter goroutine runs concurrently with the list request,
pkg/authz/responsefilterer.go:165-183).
"""
import argparse, json, os, sys, threading, time
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import zgpu
from spicedb_kubeapi_proxy_b200 import workloads

ap = argparse.ArgumentParser()
ap.add_argument("--scale", type=float, default=1.0)
ap.add_argument("--clients", type=int, default=1000)
ap.add_argument("--items", type=int, default=10000)
ap.add_argument("--rounds", type=int, default=2)
ap.add_argument("--devices", type=int, default=1)
ap.add_argument("--cold", action="store_true", help="no untimed warm-up round (first-use costs inside the timed phases)")
a = ap.parse_args()

w = workloads.cfg4(scale=a.scale)
e = zgpu.Engine(w.schema, device=0, n_devices=a.devices)
w.load_into(e)
e.publish()
base = w.check_items(e, zgpu.CHECK_DTYPE)
rng = np.random.default_rng(5)
n_users = int(max(g.subj.max() for g in w.groups if g.subj_type == "user" and not g.wildcard)) + 1
n_docs = int(max(g.res.max() for g in w.groups if g.res_type == "document")) + 1
view = e.slot_id("document", "view")

def make_list(user):  # one user lists 10k documents: one post-filter item per document
    it = np.zeros(a.items, dtype=zgpu.CHECK_DTYPE)
    it["res"] = rng.integers(0, n_docs, a.items)
    it["subj"] = user
    it["perm"], it["stype"], it["srel"] = view, e.type_id("user"), 0xFFFF
    return it

users = rng.integers(0, n_users, a.clients)
lists = [make_list(int(u)) for u in users]
ref = [e.check_bulk(l) for l in lists[:4]]  # single-caller answers for a spot check
# ---- native client threads (tests/cabi/loadgen.c): Python threads would spend the run fighting over the GIL
import ctypes as C
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "spicedb-kubeapi-proxy_b200")
lg_so = os.path.join(ROOT, "tests", "cabi", "libloadgen.so")
subprocess.run(["gcc", "-O2", "-shared", "-fPIC", "-std=c11", "-D_GNU_SOURCE", "-I", os.path.join(ROOT, "include"),
                os.path.join(ROOT, "tests", "cabi", "loadgen.c"), "-o", lg_so,
                # the library this process already loaded (ZGPU_LIB selects a tuning variant)
                os.environ.get("ZGPU_LIB") or os.path.join(PKG, "libzgpu.so"), "-Wl,-rpath," + PKG, "-lpthread"], check=True)
LG = C.CDLL(lg_so)


class Client(C.Structure):
    _fields_ = [("e", C.c_void_p), ("items", C.c_void_p), ("n_items", C.c_uint64), ("out", C.c_void_p), ("rounds", C.c_int),
                ("do_lookup", C.c_int), ("res_type", C.c_uint16), ("perm", C.c_uint16), ("stype", C.c_uint16),
                ("subj", C.c_uint32), ("ids", C.c_void_p), ("ids_cap", C.c_uint64), ("n_found", C.c_uint64), ("rc", C.c_int)]


LG.loadgen_run.restype = C.c_double
LG.loadgen_run.argtypes = [C.POINTER(Client), C.c_int, C.c_int]
all_items = np.ascontiguousarray(np.stack(lists))          # clients x items
all_out = np.zeros((a.clients, a.items), dtype=np.uint8)
ids_cap = max(1 << 16, int(n_docs * 0.06))  # a lookup returns ~3 % of the documents (the wildcard ones) + the user's own
all_ids = np.empty((a.clients, ids_cap), dtype=np.uint32)  # untouched pages cost nothing
doc_t, user_t = e.type_id("document"), e.type_id("user")


def run_phase(mode, users):
    cl = (Client * a.clients)()
    for i in range(a.clients):
        cl[i].e = e._h
        cl[i].items = all_items[i].ctypes.data
        cl[i].n_items = a.items
        cl[i].out = all_out[i].ctypes.data
        cl[i].rounds = a.rounds if mode == 0 else 1
        cl[i].do_lookup = 1
        cl[i].res_type, cl[i].perm, cl[i].stype, cl[i].subj = doc_t, view, user_t, int(users[i])
        cl[i].ids, cl[i].ids_cap = all_ids[i].ctypes.data, ids_cap
    s0 = e.stats()
    dt = LG.loadgen_run(cl, a.clients, mode)
    s1 = e.stats()
    assert dt > 0 and all(c.rc == 0 for c in cl), [c.rc for c in cl if c.rc][:5]
    return dt, s0, s1, [int(c.n_found) for c in cl]


if not a.cold:  # first-use costs (pinned staging on every device, thread stacks) stay out of the timed phases
    run_phase(0, users)
    run_phase(1, rng.integers(0, n_users, a.clients))
dt_c, c0, c1, _ = run_phase(0, users)
kept = (all_out == 2).sum(axis=1)
errors = [i for i in range(4) if not np.array_equal(all_out[i], ref[i])]
dt_l, l0, l1, found = run_phase(1, rng.integers(0, n_users, a.clients))  # fresh subjects: nothing from the answer cache
dt_m, m0, m1, _ = run_phase(2, rng.integers(0, n_users, a.clients))
lists_done = a.clients * a.rounds
print(json.dumps({
    "workload": f"cfg5 replay at the C ABI on {w.note}", "clients": a.clients, "items_per_list": a.items, "rounds": a.rounds,
    "postfilter": {"filtered_lists_per_s": lists_done / dt_c, "Mchecks_per_s": lists_done * a.items / dt_c / 1e6,
                   "wall_s": dt_c, "kept_per_list_mean": float(np.mean(kept)), "parity_spot_check_ok": not errors,
                   "kernel_launches": c1["launches"] - c0["launches"],
                   "coalesced": {"requests": c1["coalesced_requests"] - c0["coalesced_requests"],
                                 "launches": c1["coalesced_launches"] - c0["coalesced_launches"]}},
    "prefilter": {"lookups_per_s": a.clients / dt_l, "wall_s": dt_l, "results_per_lookup_mean": float(np.mean(found)),
                  "results_per_s_M": float(np.sum(found)) / dt_l / 1e6, "kernel_launches": l1["launches"] - l0["launches"],
                  "batches": l1["lookup_batches"] - l0["lookup_batches"],
                  "lookups_in_batches": l1["lookups_batched"] - l0["lookups_batched"]},
    "clients_are": "native threads (tests/cabi/loadgen.c)", "warm_up_round": not a.cold,
    "mixed": {"filtered_lists_per_s": a.clients / dt_m, "wall_s": dt_m,
              "what": "per client: one LookupResources + one 10k-item bulk check, all clients at once"},
    "devices": int(m1["devices"]), "store_tuples": int(m1["tuples"]),
    "note": "post-filter: one 10k-item zg_check_bulk per list, concurrent callers coalesced by the library's batcher; "
            "pre-filter: one zg_lookup_resources per client, concurrent calls answered up to 64 per launch sequence "
            "(multi-source reverse walk + one verification launch). The clients are native threads calling the C ABI; the Go HTTP "
            "path cannot run here."}))
