"""LookupResources on the object-hash sharded store on the GPU: dist.DeviceShardedLookup with the real kernels over
W virtual shards of one GPU (LocalDeviceTransport), W in {2, 3, 4}, against the C oracle and a replica engine."""
import os
import random

import numpy as np
import pytest

import shard_lookup_cases as cases

pytestmark = pytest.mark.gpu

WORLDS = [2, 3, 4]


@pytest.fixture(scope="module")
def zg():
    import zgpu

    return zgpu


def _cluster(zg, schema, world, loader, now=None):
    from spicedb_kubeapi_proxy_b200 import dist as zdist

    ts = zdist.LocalDeviceTransport.cluster(world)
    engines = [zg.Engine(schema, device=0, shard_rank=r, shard_count=world) for r in range(world)]
    for e in engines:
        loader(e)
        e.publish()
        if now is not None:
            e.set_clock(now)
    return engines, ts


def _strings_case(zg, schema, rels, lookups, world, expires=None, now=None, walk_cap=1 << 20, skip_rank=None):
    from oracle.pyoracle import Oracle

    o = Oracle(schema)
    for r in rels:
        o.touch(r, (expires or {}).get(r, 0))
    names = cases.intern(rels)
    engines, ts = _cluster(zg, schema, world, lambda e: cases.load(e, rels, names, expires), now)
    idx = cases.deal(list(range(len(lookups))), world, skip_rank)
    reqs = [[cases.request(engines[0], names, lookups[i]) for i in idx[r]] for r in range(world)]
    out, stats = cases.run_sharded(engines, ts, reqs, walk_cap)
    got = [None] * len(lookups)
    for r in range(world):
        for j, i in enumerate(idx[r]):
            got[i] = cases.names_of(names, lookups[i][0], out[r][j])
    return got, [cases.oracle_answer(o, q, now or 0) for q in lookups], stats


def _agree(got, want, lookups):
    for q, a, b in zip(lookups, got, want):
        assert a == b, f"{q}: sharded={a} oracle={b}"


@pytest.mark.parametrize("wl,scale", [("cfg2", 0.002), ("cfg3", 0.002), ("cfg4", 0.001)])
@pytest.mark.parametrize("world", WORLDS)
def test_workloads(zg, wl, scale, world):
    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.by_name(wl, scale)
    o = Oracle(w.schema)
    w.load_into(o)
    engines, ts = _cluster(zg, w.schema, world, w.load_into)
    rng = np.random.default_rng(5)
    n_users = max(int(g.subj.max()) + 1 for g in w.groups if g.subj_type == "user" and not g.wildcard and g.subj.size)
    rt, perm = w.lookups[0][:2]
    lookups = list(w.lookups) + [(rt, perm, "user", int(u)) for u in rng.integers(0, n_users, 12)]
    e0 = engines[0]
    per_rank = cases.deal(lookups, world)
    reqs = [[(e0.type_id(a), e0.slot_id(a, p), e0.type_id(s), u, cases.SREL_NONE) for a, p, s, u in per_rank[r]]
            for r in range(world)]
    out, stats = cases.run_sharded(engines, ts, reqs)
    for r in range(world):
        for q, a in zip(per_rank[r], out[r]):
            assert a is not None and np.array_equal(a, o.lookup_resources_ids(*q)), f"{wl} {q}"


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("world", WORLDS)
def test_random_and_fixed_schemas(zg, seed, world):
    import randgen

    fixed = sorted(randgen.FIXED_SCHEMAS)[seed] if seed < len(randgen.FIXED_SCHEMAS) and seed % 2 else None
    schema, rels, lookups = cases.random_case(9100 + seed, fixed=fixed)
    _agree(*_strings_case(zg, schema, rels, lookups, world)[:2], lookups)


@pytest.mark.parametrize("world", WORLDS)
def test_userset_subject_itself_when_check_says_so(zg, world):
    from test_oracle_random import SELF_LOOKUPS, SELF_RELS, SELF_SCHEMA

    lookups = [q for q, _ in SELF_LOOKUPS if q[3] != "9"]  # a never-written subject is answered by the string path only
    got, want, _ = _strings_case(zg, SELF_SCHEMA, SELF_RELS, lookups, world)
    _agree(got, want, lookups)
    assert got[0] == ["3", "5"] and got[2] == ["5"] and got[4] == []


@pytest.mark.parametrize("world", WORLDS)
def test_expiry_at_two_clocks(zg, world):
    import randgen
    from test_lookup_subjects import EXP_SCHEMA

    rng = random.Random(9300)
    model = randgen.model_from_schema(EXP_SCHEMA)
    rels = randgen.random_relationships(rng, model, n_obj=6, n_user=5, density=0.4)
    expires = {r: rng.choice([50, 150]) for r in rels if rng.random() < 0.5}
    lookups = cases.random_lookups(rng, model, rels, 10)
    answers = []
    for now in (100, 200):
        got, want, _ = _strings_case(zg, EXP_SCHEMA, rels, lookups, world, expires=expires, now=now)
        _agree(got, want, lookups)
        answers.append(got)
    assert answers[0] != answers[1]


@pytest.mark.parametrize("world", WORLDS)
def test_depth_cap_fails_only_that_lookup(zg, world):
    from test_oracle_random import CHAIN

    rels = [f"group:g{i}#member@group:g{i+1}#member" for i in range(55)] + ["group:g55#member@user:deep"]
    rels += ["group:x#member@user:v", "folder:f0#viewer@user:v", "folder:f1#parent@folder:f0"]
    lookups = [("group", "member", "user", "deep", ""), ("group", "member", "user", "v", ""),
               ("folder", "view", "user", "v", "")]
    got, want, _ = _strings_case(zg, CHAIN, rels, lookups, world)
    assert got[0] is None  # as zg_lookup_resources: ZG_EDEPTH
    _agree(got[1:], want[1:], lookups[1:])


@pytest.mark.parametrize("world", WORLDS)
def test_overflow_halves_then_verifies_every_owned_resource(zg, world):
    schema, rels, lookups = cases.random_case(9400, fixed="nesting", n_lookups=10)
    got, want, stats = _strings_case(zg, schema, rels, lookups, world, walk_cap=2)
    _agree(got, want, lookups)
    assert sum(s["halvings"] for s in stats) > 0 and sum(s["fallbacks"] for s in stats) > 0


@pytest.mark.parametrize("world", WORLDS)
def test_more_than_one_round_uneven_ranks_one_empty(zg, world):
    schema, rels, lookups = cases.random_case(9500, n_lookups=150)
    got, want, stats = _strings_case(zg, schema, rels, lookups, world, skip_rank=1)
    _agree(got, want, lookups)
    assert stats[0]["rounds"] >= 3


def _replica_agrees(zg, engines, ts, replica, lookups):
    e0 = engines[0]
    per_rank = cases.deal(lookups, len(engines))
    reqs = [[(e0.type_id(a), e0.slot_id(a, p), e0.type_id(s), u, cases.SREL_NONE if sr is None else e0.slot_id(s, sr))
             for a, p, s, u, sr in per_rank[r]] for r in range(len(engines))]
    out, _ = cases.run_sharded(engines, ts, reqs)
    for r in range(len(engines)):
        for (a, p, s, u, sr), got in zip(per_rank[r], out[r]):
            assert got is not None and np.array_equal(got, replica.lookup_resources_ids(a, p, s, u, sr)), (a, p, s, u, sr)


def test_cfg4_agrees_with_a_replica_at_the_full_size_scale(zg):
    """cfg4 at the scale of test_gpu_fullsize.py (ZGPU_FULLSIZE_SCALE): view, restricted_view and a userset subject."""
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.cfg4(scale=float(os.environ.get("ZGPU_FULLSIZE_SCALE", "0.25")))
    replica = zg.Engine(w.schema, device=0)
    w.load_into(replica)
    replica.publish()
    engines, ts = _cluster(zg, w.schema, 2, w.load_into)
    users = [u for _, _, _, u in w.lookups]
    lookups = [("document", p, "user", u, None) for p in ("view", "restricted_view") for u in users]
    lookups += [("document", "view", "group", g, "member") for g in (0, 1, 7)]
    _replica_agrees(zg, engines, ts, replica, lookups)


def test_answers_follow_write_relationships_on_every_shard(zg):
    """1 000 write_relationships updates applied to the replica and to every shard: the sharded answers move with
    them. Every engine sees the same writes in the same order, so the interned ids agree."""
    import randgen

    rng = random.Random(9600)
    schema = randgen.FIXED_SCHEMAS["nesting"]
    model = randgen.model_from_schema(schema)
    rels = randgen.random_relationships(rng, model, n_obj=30, n_user=20, density=0.15)
    pool = randgen.random_relationships(rng, model, n_obj=30, n_user=20, density=0.15)
    # ten writes of 100 distinct relationships each (a write may name a relationship once)
    ups = [((zg._lib.OP_DELETE if rng.random() < 0.3 else zg._lib.OP_TOUCH), r, 0) for _ in range(10)
           for r in rng.sample(pool, 100)]
    lookups = cases.random_lookups(rng, model, rels, 24)

    def load(e):
        e.write_relationships([(zg._lib.OP_TOUCH, r, 0) for r in rels])

    replica = zg.Engine(schema, device=0)
    load(replica)
    replica.publish()
    engines, ts = _cluster(zg, schema, 3, load)
    for e in [replica] + engines:
        for i in range(0, len(ups), 100):
            e.write_relationships(ups[i:i + 100])
        e.publish()
    per_rank = cases.deal(lookups, 3)
    reqs = [[(replica.type_id(a), replica.slot_id(a, p), replica.type_id(s), replica.find(s, sid),
              replica.slot_id(s, sr) if sr else cases.SREL_NONE) for a, p, s, sid, sr in per_rank[r]] for r in range(3)]
    out, _ = cases.run_sharded(engines, ts, reqs)
    for r in range(3):
        for (a, p, s, sid, sr), got in zip(per_rank[r], out[r]):
            want = replica.lookup_resources_ids(a, p, s, replica.find(s, sid), sr or None)
            assert got is not None and np.array_equal(got, want), (a, p, s, sid, sr)


def test_lookup_resources_on_a_sharded_engine_is_still_refused(zg):
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.cfg2(scale=0.001)
    e = zg.Engine(w.schema, device=0, shard_rank=0, shard_count=2)
    w.load_into(e)
    e.publish()
    rt, perm, st, u = w.lookups[0]
    with pytest.raises(zg._lib.ZgpuError) as ex:
        e.lookup_resources_ids(rt, perm, st, u)
    assert ex.value.code == -1  # ZG_EINVAL
    replica = zg.Engine(w.schema, device=0)
    w.load_into(replica)
    replica.publish()
    with pytest.raises(zg._lib.ZgpuError) as ex:
        replica.shard_lookup_candidates_dev(False, 0, 0)
    assert ex.value.code == -1


@pytest.mark.parametrize("world", WORLDS)
def test_undecidable_self_membership_is_left_out_as_on_a_replica(zg, world):
    """doc:x#safe@doc:x#viewer cannot be decided (a 56-link `banned` chain): left out, the lookup still answered --
    what zg_lookup_resources does on a replica engine loaded the same way."""
    from test_oracle_random import SELF_SCHEMA

    rels = ["doc:x#banned@doc:c0#viewer"] + [f"doc:c{i}#viewer@doc:c{i + 1}#viewer" for i in range(55)]
    rels += ["doc:c55#viewer@user:a", "doc:y#viewer@user:b"]
    lookups = [("doc", "safe", "doc", "x", "viewer"), ("doc", "view", "doc", "x", "viewer"), ("doc", "view", "user", "b", "")]
    got, want, _ = _strings_case(zg, SELF_SCHEMA, rels, lookups, world)
    _agree(got, want, lookups)
    assert got == [[], ["x"], ["y"]]
    replica = zg.Engine(SELF_SCHEMA, device=0)
    replica.write_relationships([(zg._lib.OP_TOUCH, r, 0) for r in rels])
    assert replica.lookup_resources_str("doc", "safe", "doc", "x", "viewer") == []
