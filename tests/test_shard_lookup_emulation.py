"""LookupResources on the object-hash sharded store under the CPU kernel emulator: the product's own driver
(dist.DeviceShardedLookup) over 2 and 3 emulated shards, every answer against the C oracle. The round's kernels
(mrbfs_expand_kernel, the self-membership and exhaustive-fill kernels, the answer keys, the routing home, the split)
run emulated; the candidates are verified by the emulated sharded check protocol."""
import os
import random
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))

import shard_lookup_cases as cases  # noqa: E402


def _cluster(schema, world, loader, now=0):
    import torch

    import emu_shard_lookup as esl
    import zgpu  # noqa: F401
    from spicedb_kubeapi_proxy_b200 import dist as zdist

    ts = zdist.LocalDeviceTransport.cluster(world, device=torch.device("cpu"))
    engines = [esl.EmuEngine(schema, shard_rank=r, shard_count=world) for r in range(world)]
    for e in engines:
        loader(e)
        e.publish()
        e.shard_opts.now = now
    return engines, ts


def _strings_case(schema, rels, lookups, world, expires=None, now=0, walk_cap=1 << 16, skip_rank=None):
    """Every lookup through the sharded driver, dealt over the ranks; -> (answers by name, oracle's, stats)."""
    from oracle.pyoracle import Oracle

    o = Oracle(schema)
    for r in rels:
        o.touch(r, (expires or {}).get(r, 0))
    names = cases.intern(rels)
    engines, ts = _cluster(schema, world, lambda e: cases.load(e, rels, names, expires), now)
    idx = cases.deal(list(range(len(lookups))), world, skip_rank)
    reqs = [[cases.request(engines[0], names, lookups[i]) for i in idx[r]] for r in range(world)]
    out, stats = cases.run_sharded(engines, ts, reqs, walk_cap)
    got = [None] * len(lookups)
    for r in range(world):
        for j, i in enumerate(idx[r]):
            got[i] = cases.names_of(names, lookups[i][0], out[r][j])
    want = [cases.oracle_answer(o, q, now) for q in lookups]
    return got, want, stats


def _agree(got, want, lookups):
    for q, a, b in zip(lookups, got, want):
        assert a == b, f"{q}: sharded={a} oracle={b}"


@pytest.mark.parametrize("wl,scale", [("cfg2", 0.0005), ("cfg3", 0.002), ("cfg4", 0.001)])
@pytest.mark.parametrize("world", [2, 3])
def test_workloads(wl, scale, world):
    import zgpu  # noqa: F401
    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.by_name(wl, scale)
    o = Oracle(w.schema)
    w.load_into(o)
    engines, ts = _cluster(w.schema, world, w.load_into)
    rng = np.random.default_rng(5)
    n_users = max(int(g.subj.max()) + 1 for g in w.groups if g.subj_type == "user" and not g.wildcard and g.subj.size)
    lookups = list(w.lookups) + [(w.lookups[0][0], w.lookups[0][1], "user", int(u)) for u in rng.integers(0, n_users, 6)]
    e0 = engines[0]
    per_rank = cases.deal(lookups, world)
    reqs = [[(e0.type_id(rt), e0.slot_id(rt, perm), e0.type_id(st), u, cases.SREL_NONE) for rt, perm, st, u in per_rank[r]]
            for r in range(world)]
    out, stats = cases.run_sharded(engines, ts, reqs)
    for r in range(world):
        for q, a in zip(per_rank[r], out[r]):
            assert a is not None and np.array_equal(a, o.lookup_resources_ids(*q)), f"{wl} {q}"
    assert sum(s["candidates"] for s in stats) > 0 and stats[0]["levels"] >= 2


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("world", [2, 3])
def test_random_schemas(seed, world):
    schema, rels, lookups = cases.random_case(8100 + seed)
    _agree(*_strings_case(schema, rels, lookups, world)[:2], lookups)


@pytest.mark.parametrize("name", sorted(__import__("randgen").FIXED_SCHEMAS))
def test_fixed_schemas(name):
    schema, rels, lookups = cases.random_case(8200, fixed=name)
    _agree(*_strings_case(schema, rels, lookups, 3)[:2], lookups)


def test_userset_subject_itself_when_check_says_so():
    from test_oracle_random import SELF_LOOKUPS, SELF_RELS, SELF_SCHEMA

    lookups = [q for q, _ in SELF_LOOKUPS if q[3] != "9"]  # a never-written subject is answered by the string path only
    for world in (2, 3):
        got, want, _ = _strings_case(SELF_SCHEMA, SELF_RELS, lookups, world)
        _agree(got, want, lookups)
    # doc:5#editor is in doc:5#view by itself; doc:7#viewer is banned from doc:7#safe
    assert got[0] == ["3", "5"] and got[2] == ["5"] and got[4] == []


def test_expiry_at_two_clocks():
    from test_lookup_subjects import EXP_SCHEMA

    import randgen

    rng = random.Random(8300)
    model = randgen.model_from_schema(EXP_SCHEMA)
    rels = randgen.random_relationships(rng, model, n_obj=6, n_user=5, density=0.4)
    expires = {r: rng.choice([50, 150]) for r in rels if rng.random() < 0.5}
    lookups = cases.random_lookups(rng, model, rels, 10)
    answers = []
    for now in (100, 200):
        got, want, _ = _strings_case(EXP_SCHEMA, rels, lookups, 3, expires=expires, now=now)
        _agree(got, want, lookups)
        answers.append(got)
    assert answers[0] != answers[1]


def test_depth_cap_fails_only_that_lookup():
    from test_oracle_random import CHAIN

    rels = [f"group:g{i}#member@group:g{i+1}#member" for i in range(55)] + ["group:g55#member@user:deep"]
    rels += ["group:x#member@user:v", "folder:f0#viewer@user:v", "folder:f1#parent@folder:f0"]
    lookups = [("group", "member", "user", "deep", ""), ("group", "member", "user", "v", ""),
               ("folder", "view", "user", "v", "")]
    got, want, _ = _strings_case(CHAIN, rels, lookups, 2)
    # g0 .. g4 are more than 50 dispatches from user:deep: the engine fails that LookupResources (ZG_EDEPTH, as
    # zg_lookup_resources does) where the oracle leaves the undecidable candidates out
    assert got[0] is None and set(want[0]) == {f"g{i}" for i in range(5, 56)}
    _agree(got[1:], want[1:], lookups[1:])
    assert got[1] == ["x"] and got[2] == ["f0", "f1"]


def test_overflow_halves_then_verifies_every_owned_resource():
    schema, rels, lookups = cases.random_case(8400, fixed="nesting", n_lookups=10)
    want = _strings_case(schema, rels, lookups, 3)[1]
    got, _, stats = _strings_case(schema, rels, lookups, 3, walk_cap=2)
    _agree(got, want, lookups)
    assert sum(s["halvings"] for s in stats) > 0 and sum(s["fallbacks"] for s in stats) > 0


def test_more_than_one_round_uneven_ranks_one_empty():
    schema, rels, lookups = cases.random_case(8500, n_lookups=150)
    got, want, stats = _strings_case(schema, rels, lookups, 3, skip_rank=1)
    _agree(got, want, lookups)
    assert stats[0]["rounds"] >= 3


def test_undecidable_self_membership_is_left_out_as_on_a_replica():
    """doc:x#safe@doc:x#viewer: view holds (self-membership) but `banned` is a 56-link chain, so the check cannot be
    decided. The replica asks Check about the subject's own object and leaves it out unless HAS; so does the shard."""
    from test_oracle_random import SELF_SCHEMA

    rels = ["doc:x#banned@doc:c0#viewer"] + [f"doc:c{i}#viewer@doc:c{i + 1}#viewer" for i in range(55)]
    rels += ["doc:c55#viewer@user:a", "doc:y#viewer@user:b"]
    lookups = [("doc", "safe", "doc", "x", "viewer"), ("doc", "view", "doc", "x", "viewer"), ("doc", "view", "user", "b", "")]
    for world in (2, 3):
        got, want, _ = _strings_case(SELF_SCHEMA, rels, lookups, world)
        _agree(got, want, lookups)
        assert got == [[], ["x"], ["y"]]
