"""Shared cases and driver of the sharded LookupResources tests (dist.DeviceShardedLookup): under the kernel emulator
in test_shard_lookup_emulation.py, on the GPU in test_gpu_sharded_lookup.py."""
from __future__ import annotations

import random
import threading
import traceback

import numpy as np

import randgen
from golden_runner import split_rel

SREL_NONE, SREL_WILDCARD = 0xFFFF, 0xFFFE
TUPLE_DTYPE = np.dtype([("res", "<u4"), ("subj", "<u4"), ("rel", "<u2"), ("stype", "<u2"), ("srel", "<u2"), ("flags", "<u2")])


def intern(rels):
    """(type, name) -> id in order of first appearance, resource before subject: the same on every shard."""
    names = {}
    for r in rels:
        rt, rid, _rel, st, sid, _srel = split_rel(r)
        for key in ((rt, rid), (st, sid)):
            if key[1] != "*" and key not in names:
                names[key] = sum(1 for k in names if k[0] == key[0])
    return names


def load(engine, rels, names, expires=None):
    """Writes rels (strings, optional {rel: expires_at}) with the given interning into an engine (or emulated one)."""
    t = np.zeros(len(rels), dtype=TUPLE_DTYPE)
    ex = np.zeros(len(rels), dtype=np.uint32)
    for i, r in enumerate(rels):
        rt, rid, rel, st, sid, srel = split_rel(r)
        t["res"][i], t["rel"][i], t["stype"][i] = names[(rt, rid)], engine.slot_id(rt, rel), engine.type_id(st)
        if sid == "*":
            t["srel"][i], t["subj"][i] = SREL_WILDCARD, 0
        else:
            t["srel"][i] = engine.slot_id(st, srel) if srel else SREL_NONE
            t["subj"][i] = names[(st, sid)]
        ex[i] = (expires or {}).get(r, 0)
    engine.load_tuples(t, ex if expires else None)


def request(engine, names, q):
    """(res_type, perm, subj_type, subj_id, subj_rel) names -> the id tuple DeviceShardedLookup takes."""
    rt, perm, st, sid, srel = q
    return (engine.type_id(rt), engine.slot_id(rt, perm), engine.type_id(st), names[(st, sid)],
            engine.slot_id(st, srel) if srel else SREL_NONE)


def oracle_answer(o, q, now=0):
    """Sorted resource names, or None where the lookup fails (a candidate hits the depth cap)."""
    from oracle.pyoracle import OracleError

    rt, perm, st, sid, srel = q
    try:
        return sorted(o.lookup_resources(rt, perm, st, sid, srel, now=now))
    except OracleError:
        return None


def names_of(names, res_type, ids):
    inv = {i: n for (t, n), i in names.items() if t == res_type}
    return None if ids is None else sorted(inv[int(i)] for i in ids)


def random_lookups(rng, model, rels, n):
    """n lookups over the written objects: plain users and userset subjects (type:object#relation-or-permission)."""
    objs = sorted({(t, i) for (t, i) in intern(rels) if t != "user"})
    users = sorted({i for (t, i) in intern(rels) if t == "user"})
    out = []
    tn = [t for t in model["tnames"] if model["types"][t]["rels"] or model["types"][t]["perms"]]
    for _ in range(n):
        t = rng.choice(tn)
        d = model["types"][t]
        name = rng.choice(list(d["rels"]) + list(d["perms"]))
        if users and (rng.random() < 0.7 or not objs):
            out.append((t, name, "user", rng.choice(users), ""))
        elif objs:
            st, sid = rng.choice(objs)
            sd = model["types"][st]
            out.append((t, name, st, sid, rng.choice(list(sd["rels"]) + list(sd["perms"]))))
    return out


def random_case(seed, fixed=None, n_lookups=12):
    rng = random.Random(seed)
    if fixed:
        schema = randgen.FIXED_SCHEMAS[fixed]
        model = randgen.model_from_schema(schema)
    else:
        schema, model = randgen.random_schema(rng)
    rels = randgen.random_relationships(rng, model, n_obj=6, n_user=5, density=0.35)
    return schema, rels, random_lookups(rng, model, rels, n_lookups)


def deal(items, world, skip_rank=None):
    """Requests dealt unevenly over the ranks (rank r gets about (r + 1) shares); skip_rank brings none."""
    pattern = [r for r in range(world) if r != skip_rank for _ in range(r + 1)]
    out = [[] for _ in range(world)]
    for i, x in enumerate(items):
        out[pattern[i % len(pattern)]].append(x)
    return out


def run_sharded(engines, transports, reqs_per_rank, walk_cap=1 << 16):
    """dist.DeviceShardedLookup on every rank (one thread each) -> (answers per rank, stats of every rank)."""
    from spicedb_kubeapi_proxy_b200 import dist as zdist

    world = len(engines)
    out, stats, errs = [None] * world, [None] * world, []

    def run(r):
        try:
            lk = zdist.DeviceShardedLookup(engines[r], transports[r], walk_cap=walk_cap)
            out[r] = lk.lookup_resources(reqs_per_rank[r])
            stats[r] = lk.stats
        except Exception:  # noqa: BLE001
            errs.append(traceback.format_exc())
            transports[r]._s["bar"].abort()

    th = [threading.Thread(target=run, args=(r,)) for r in range(world)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    assert not errs, errs[0]
    return out, stats
