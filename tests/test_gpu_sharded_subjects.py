"""LookupSubjects on the object-hash sharded store on the GPU: dist.DeviceShardedLookup.lookup_subjects with the real
kernels over W virtual shards of one GPU (LocalDeviceTransport), W in {2, 3, 4}, against the C oracle and against a
replica engine's zg_lookup_subjects (ids, wildcard entry and exclusions compared exactly)."""
import os
import random

import numpy as np
import pytest

import randgen
import shard_lookup_cases as slc
import shard_subjects_cases as cases
from lookup_subjects_oracle import EXCLUDE, INCLUDE

pytestmark = pytest.mark.gpu

WORLDS = [2, 3, 4]


@pytest.fixture(scope="module")
def zg():
    import zgpu

    return zgpu


def _cluster_fn(zg):
    def cluster(schema, world, loader, now=0):
        from spicedb_kubeapi_proxy_b200 import dist as zdist

        ts = zdist.LocalDeviceTransport.cluster(world)
        engines = [zg.Engine(schema, device=0, shard_rank=r, shard_count=world) for r in range(world)]
        for e in engines:
            loader(e)
            e.publish()
            if now:
                e.set_clock(now)
        return engines, ts

    return cluster


def _case(zg, *a, **k):
    return cases.strings_case(_cluster_fn(zg), *a, **k)


@pytest.mark.parametrize("world", WORLDS)
def test_hand_table(zg, world):
    from test_lookup_subjects import HAND, HAND_EXPIRES, HAND_RELS, HAND_TABLE

    lookups = cases.with_options([q for q, _, _ in HAND_TABLE])
    got, want, stats = _case(zg, HAND, HAND_RELS, lookups, world, expires=HAND_EXPIRES, now=100)
    cases.agree(got, want, lookups)
    for (q, opt, expect) in HAND_TABLE:
        assert got[lookups.index((q, opt))] == (None if expect == "EDEPTH" else expect), q
    assert sum(s["entries_sent"] for s in stats) > 0


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("world", WORLDS)
def test_random_and_fixed_schemas(zg, seed, world):
    fixed = sorted(randgen.FIXED_SCHEMAS)[seed % len(randgen.FIXED_SCHEMAS)] if seed % 2 else None
    schema, rels, queries = cases.random_case(9700 + seed, fixed=fixed)
    lookups = cases.with_options(queries)
    cases.agree(*_case(zg, schema, rels, lookups, world)[:2], lookups)


@pytest.mark.parametrize("world", WORLDS)
def test_expiry_at_two_clocks(zg, world):
    from lookup_subjects_oracle import subject_queries
    from test_lookup_subjects import EXP_SCHEMA

    rng = random.Random(9800)
    model = randgen.model_from_schema(EXP_SCHEMA)
    rels = randgen.random_relationships(rng, model, n_obj=6, n_user=5, density=0.4)
    expires = {r: rng.choice([50, 150]) for r in rels if rng.random() < 0.5}
    lookups = cases.with_options(subject_queries(model, rng, 6, per_type=3))
    answers = []
    for now in (100, 200):
        got, want, _ = _case(zg, EXP_SCHEMA, rels, lookups, world, expires=expires, now=now)
        cases.agree(got, want, lookups)
        answers.append(got)
    assert answers[0] != answers[1]


@pytest.mark.parametrize("world", WORLDS)
def test_overflow_halves_then_falls_back_to_every_owned_subject(zg, world):
    schema, rels, queries = cases.random_case(9900, fixed="nesting")
    lookups = cases.with_options(queries)
    got, want, stats = _case(zg, schema, rels, lookups, world, walk_cap=1)
    cases.agree(got, want, lookups)
    assert sum(s["halvings"] for s in stats) > 0 and sum(s["fallbacks"] for s in stats) > 0


@pytest.mark.parametrize("world", WORLDS)
def test_more_than_one_round_uneven_ranks_one_empty(zg, world):
    schema, rels, queries = cases.random_case(10000, n_obj=6)
    lookups = (cases.with_options(queries) * 13)[:150]
    got, want, stats = _case(zg, schema, rels, lookups, world, skip_rank=1)
    cases.agree(got, want, lookups)
    assert stats[0]["rounds"] >= 3


@pytest.mark.parametrize("world", WORLDS)
def test_no_wildcards_holds_in_the_sub_queries_raised_to_other_shards(zg, world):
    """doc:d#view reaches a `user:*` only through folder:f, owned by another shard: the no-wildcards verification
    must hold in the pass that evaluates the raised sub-query there, or bob (editor, not member2) is listed."""
    names = slc.intern(cases.REMOTE_WILD_RELS)
    assert names[("doc", "d")] % world != names[("folder", "f")] % world
    lookups = cases.with_options(cases.REMOTE_WILD_QUERIES)
    got, want, stats = _case(zg, cases.REMOTE_WILD, cases.REMOTE_WILD_RELS, lookups, world)
    cases.agree(got, want, lookups)
    assert got[:2] == [([], True, []), ([], False, [])]
    assert sum(s["nowild_verified"] for s in stats) > 0


def _replica_agrees(engines, ts, replica, lookups):
    """lookups: (res_type, res id, perm, subj_type, option) -> the sharded answers equal the replica's, exactly."""
    e0 = engines[0]
    per_rank = slc.deal(lookups, len(engines))
    reqs = [[(e0.type_id(rt), int(r), e0.slot_id(rt, p), e0.type_id(st), slc.SREL_NONE, opt) for rt, r, p, st, opt in per_rank[k]]
            for k in range(len(engines))]
    out, stats = cases.run_sharded(engines, ts, reqs, walk_cap=1 << 22)
    for k in range(len(engines)):
        for (rt, r, p, st, opt), got in zip(per_rank[k], out[k]):
            ids, wild, ex = replica.lookup_subjects_ids(rt, int(r), p, st, wildcards=opt)
            assert got is not None, (rt, r, p, st, opt)
            assert np.array_equal(got[0], ids) and got[1] == wild and np.array_equal(got[2], ex), (rt, r, p, st, opt)
    return stats


def _workload_lookups(w, n, seed):
    rng = np.random.default_rng(seed)
    out = []
    for c in w.checks[:2]:
        for r in rng.choice(np.unique(c.res), size=min(n, np.unique(c.res).size), replace=False):
            out += [(c.res_type, int(r), c.perm, c.subj_type, opt) for opt in (INCLUDE, EXCLUDE)]
    return out


@pytest.mark.parametrize("wl,scale", [("cfg2", 0.002), ("cfg3", 0.002), ("cfg4", 0.001)])
@pytest.mark.parametrize("world", WORLDS)
def test_workloads_agree_with_a_replica(zg, wl, scale, world):
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.by_name(wl, scale)
    replica = zg.Engine(w.schema, device=0)
    w.load_into(replica)
    replica.publish()
    engines, ts = _cluster_fn(zg)(w.schema, world, w.load_into)
    stats = _replica_agrees(engines, ts, replica, _workload_lookups(w, 8, 5))
    assert sum(s["entries_sent"] for s in stats) > 0


def test_cfg4_agrees_with_a_replica_at_the_full_size_scale(zg):
    """cfg4 at the scale of test_gpu_fullsize.py (ZGPU_FULLSIZE_SCALE): a seeded sample of documents, view and
    restricted_view, both wildcard options."""
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.cfg4(scale=float(os.environ.get("ZGPU_FULLSIZE_SCALE", "0.25")))
    replica = zg.Engine(w.schema, device=0)
    w.load_into(replica)
    replica.publish()
    engines, ts = _cluster_fn(zg)(w.schema, 2, w.load_into)
    rng = np.random.default_rng(11)
    docs = np.unique(np.concatenate([c.res for c in w.checks if c.res_type == "document"]))
    lookups = [("document", int(r), p, "user", opt) for p in ("view", "restricted_view")
               for r in rng.choice(docs, size=12, replace=False) for opt in (INCLUDE, EXCLUDE)]
    _replica_agrees(engines, ts, replica, lookups)


def test_answers_follow_write_relationships_on_every_shard(zg):
    """1 000 write_relationships updates applied to the replica and to every shard: the sharded answers move with
    them. Every engine sees the same writes in the same order, so the interned ids agree."""
    from lookup_subjects_oracle import subject_queries

    rng = random.Random(10100)
    schema = randgen.FIXED_SCHEMAS["nesting"]
    model = randgen.model_from_schema(schema)
    rels = randgen.random_relationships(rng, model, n_obj=30, n_user=20, density=0.15)
    pool = randgen.random_relationships(rng, model, n_obj=30, n_user=20, density=0.15)
    ups = [((zg._lib.OP_DELETE if rng.random() < 0.3 else zg._lib.OP_TOUCH), r, 0) for _ in range(10)
           for r in rng.sample(pool, 100)]
    queries = [q for q in subject_queries(model, rng, 30, per_type=4) if not q[4]]

    def load(e):
        e.write_relationships([(zg._lib.OP_TOUCH, r, 0) for r in rels])

    replica = zg.Engine(schema, device=0)
    load(replica)
    replica.publish()
    engines, ts = _cluster_fn(zg)(schema, 3, load)
    for e in [replica] + engines:
        for i in range(0, len(ups), 100):
            e.write_relationships(ups[i:i + 100])
        e.publish()
    lookups = [(rt, replica.find(rt, rid), p, st, opt) for rt, rid, p, st, _ in queries for opt in (INCLUDE, EXCLUDE)]
    _replica_agrees(engines, ts, replica, [q for q in lookups if q[1] != 0xFFFFFFFF])


def test_lookup_subjects_on_a_sharded_engine_is_still_refused(zg):
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.cfg4(scale=0.0002)
    e = zg.Engine(w.schema, device=0, shard_rank=0, shard_count=2)
    w.load_into(e)
    e.publish()
    c = w.checks[0]
    with pytest.raises(zg._lib.ZgpuError) as ex:
        e.lookup_subjects_ids(c.res_type, int(c.res[0]), c.perm, c.subj_type)
    assert ex.value.code == -1  # ZG_EINVAL
    with pytest.raises(zg._lib.ZgpuError) as ex:
        e.lookup_subjects_str(c.res_type, "0", c.perm, c.subj_type)
    assert ex.value.code == -1
    replica = zg.Engine(w.schema, device=0)
    w.load_into(replica)
    replica.publish()
    for call in (lambda: replica.shard_subjects_candidates_dev(False, 0, 0), lambda: replica.shard_pass_nowild_dev(0, 0, 0)):
        with pytest.raises(zg._lib.ZgpuError) as ex:
            call()
        assert ex.value.code == -1 and "use zg_lookup_subjects" in str(ex.value)
