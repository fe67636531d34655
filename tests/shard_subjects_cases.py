"""Shared cases and driver of the sharded LookupSubjects tests (dist.DeviceShardedLookup.lookup_subjects): under the
kernel emulator in test_shard_subjects_emulation.py, on the GPU in test_gpu_sharded_subjects.py. Relationships are
loaded with shard_lookup_cases' interning, the same on every shard."""
from __future__ import annotations

import random
import threading
import traceback

import randgen
import shard_lookup_cases as slc
from lookup_subjects_oracle import EXCLUDE, INCLUDE, COracleSubjects, DepthError, subject_queries

NEVER_WRITTEN = 1 << 20  # a resource id above every written one: no relationship names it


def request(engine, names, q, option):
    """(res_type, res_id, perm, subj_type, subj_rel) names -> the id tuple lookup_subjects takes."""
    rt, rid, perm, st, srel = q
    return (engine.type_id(rt), names.get((rt, rid), NEVER_WRITTEN), engine.slot_id(rt, perm), engine.type_id(st),
            engine.slot_id(st, srel) if srel else slc.SREL_NONE, option)


def names_of(names, subj_type, answer):
    """(ids, wildcard, excluded) -> (sorted names, wildcard, sorted names); None stays None."""
    if answer is None:
        return None
    inv = {i: n for (t, n), i in names.items() if t == subj_type}
    ids, wild, ex = answer
    return sorted(inv[int(i)] for i in ids), wild, sorted(inv[int(i)] for i in ex)


# A wildcard behind a hop to another shard: doc:d#view reaches folder:f's `user:*` through `parent`, and d and f land
# on different shards (fx takes folder id 0, so d = doc 0 and f = folder 1). The no-wildcards verification must hold in
# the sub-query that d's owner raises to f's owner too; otherwise bob, an editor but not a member2, would be listed.
REMOTE_WILD = """
definition user {}
definition folder {
  relation viewer: user | user:*
  permission view = viewer
}
definition doc {
  relation parent: folder
  relation editor: user
  relation member2: user
  permission view = parent->view + (editor & member2)
}
"""
REMOTE_WILD_RELS = ["folder:fx#viewer@user:alice", "doc:d#parent@folder:f", "folder:f#viewer@user:*", "doc:d#editor@user:bob"]
REMOTE_WILD_QUERIES = [("doc", "d", "view", "user", ""), ("folder", "f", "view", "user", ""), ("folder", "fx", "view", "user", "")]


def oracle(schema, rels, expires=None):
    c = COracleSubjects(schema)
    for r in rels:
        c.touch(r, (expires or {}).get(r, 0))
    return c


def oracle_answer(c, q, option, now=0):
    try:
        return c.lookup_subjects(*q, wildcards=option, now=now)
    except DepthError:
        return None


def random_case(seed, fixed=None, n_obj=5):
    """A random (or fixed) schema, its relationships, and LookupSubjects queries with plain and userset subject types
    (o{n_obj} is a never-written resource)."""
    rng = random.Random(seed)
    if fixed:
        schema = randgen.FIXED_SCHEMAS[fixed]
        model = randgen.model_from_schema(schema)
    else:
        schema, model = randgen.random_schema(rng)
    rels = randgen.random_relationships(rng, model, n_obj=n_obj, n_user=4, density=0.35)
    return schema, rels, subject_queries(model, rng, n_obj, per_type=1)


def with_options(queries):
    """Every query with both wildcard options."""
    return [(q, opt) for q in queries for opt in (INCLUDE, EXCLUDE)]


def run_sharded(engines, transports, reqs_per_rank, walk_cap=1 << 16):
    """dist.DeviceShardedLookup.lookup_subjects on every rank (one thread each) -> (answers per rank, stats of every rank)."""
    from spicedb_kubeapi_proxy_b200 import dist as zdist

    world = len(engines)
    out, stats, errs = [None] * world, [None] * world, []

    def run(r):
        try:
            lk = zdist.DeviceShardedLookup(engines[r], transports[r], walk_cap=walk_cap)
            out[r] = lk.lookup_subjects(reqs_per_rank[r])
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


def strings_case(cluster, schema, rels, lookups, world, expires=None, now=0, walk_cap=1 << 16, skip_rank=None):
    """Every (query, option) of `lookups` through the sharded driver, dealt unevenly over the ranks; cluster(schema,
    world, loader, now) -> (engines, transports). -> (answers by name, the oracle's, stats of every rank)."""
    names = slc.intern(rels)
    engines, ts = cluster(schema, world, lambda e: slc.load(e, rels, names, expires), now)
    idx = slc.deal(list(range(len(lookups))), world, skip_rank)
    reqs = [[request(engines[0], names, *lookups[i]) for i in idx[r]] for r in range(world)]
    out, stats = run_sharded(engines, ts, reqs, walk_cap)
    got = [None] * len(lookups)
    for r in range(world):
        for j, i in enumerate(idx[r]):
            got[i] = names_of(names, lookups[i][0][3], out[r][j])
    c = oracle(schema, rels, expires)
    return got, [oracle_answer(c, q, opt, now) for q, opt in lookups], stats


def agree(got, want, lookups):
    for q, a, b in zip(lookups, got, want):
        assert a == b, f"{q}: sharded={a} oracle={b}"
