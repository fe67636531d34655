"""LookupSubjects on the object-hash sharded store under the CPU kernel emulator: the product's own driver
(dist.DeviceShardedLookup.lookup_subjects) over 2 and 3 emulated shards, every answer against the C oracle
(tests/lookup_subjects_oracle.py COracleSubjects) with both wildcard options. The round's kernels (the expand, the
routing to the owners, the admission, the exhaustive fill, the verdicts, the answer keys, the routing home, the split)
run emulated; the candidates are verified by the emulated sharded check protocol, the second time with no_wildcards."""
import os
import random
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))

import randgen  # noqa: E402
import shard_subjects_cases as cases  # noqa: E402
from lookup_subjects_oracle import INCLUDE  # noqa: E402
from test_lookup_subjects import EXP_SCHEMA, HAND, HAND_EXPIRES, HAND_RELS, HAND_TABLE  # noqa: E402


def _cluster(schema, world, loader, now=0):
    import torch

    import emu_shard_subjects as ess
    import zgpu  # noqa: F401
    from spicedb_kubeapi_proxy_b200 import dist as zdist

    ts = zdist.LocalDeviceTransport.cluster(world, device=torch.device("cpu"))
    engines = [ess.EmuEngine(schema, shard_rank=r, shard_count=world) for r in range(world)]
    for e in engines:
        loader(e)
        e.publish()
        e.shard_opts.now = now
    return engines, ts


def _case(*a, **k):
    return cases.strings_case(_cluster, *a, **k)


@pytest.mark.parametrize("world", [2, 3])
def test_hand_table(world):
    """Wildcard exclusions, the EXCLUDE option, a userset subject type, the depth cap (None), an expired wildcard,
    a never-written resource and the fenced divergence row d4, each with both options."""
    lookups = cases.with_options([q for q, _, _ in HAND_TABLE])
    got, want, stats = _case(HAND, HAND_RELS, lookups, world, expires=HAND_EXPIRES, now=100)
    cases.agree(got, want, lookups)
    for (q, opt, expect) in HAND_TABLE:
        assert got[lookups.index((q, opt))] == (None if expect == "EDEPTH" else expect), q
    assert sum(s["entries_sent"] for s in stats) > 0  # the walk crossed shards
    assert sum(s["nowild_verified"] for s in stats) > 0


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("world", [2, 3])
def test_random_schemas(seed, world):
    schema, rels, queries = cases.random_case(8600 + seed)
    lookups = cases.with_options(queries)
    cases.agree(*_case(schema, rels, lookups, world)[:2], lookups)


@pytest.mark.parametrize("name", sorted(randgen.FIXED_SCHEMAS))
def test_fixed_schemas(name):
    schema, rels, queries = cases.random_case(8700, fixed=name)
    lookups = cases.with_options(queries)
    cases.agree(*_case(schema, rels, lookups, 3)[:2], lookups)


@pytest.mark.parametrize("world", [2, 3])
def test_no_wildcards_holds_in_the_sub_queries_raised_to_other_shards(world):
    """doc:d#view reaches a `user:*` only through folder:f, owned by another shard: the no-wildcards verification
    must hold in the pass that evaluates the raised sub-query there, or bob (editor, not member2) is listed."""
    import shard_lookup_cases as slc

    names = slc.intern(cases.REMOTE_WILD_RELS)
    assert names[("doc", "d")] % world != names[("folder", "f")] % world
    lookups = cases.with_options(cases.REMOTE_WILD_QUERIES)
    got, want, stats = _case(cases.REMOTE_WILD, cases.REMOTE_WILD_RELS, lookups, world)
    cases.agree(got, want, lookups)
    assert got[:2] == [([], True, []), ([], False, [])]
    assert sum(s["nowild_verified"] for s in stats) > 0


def test_admission_admits_each_object_once_per_lookup():
    """Every object is admitted by its owner once per lookup: the shards together admit exactly the objects a
    replica's forward walk marks, and verify exactly the items it verifies (the probe and the resource itself
    included); entries crossed shards."""
    import emu_shard_subjects as ess
    import emu_subjects as E
    import shard_lookup_cases as slc

    schema, rels, queries = cases.random_case(8800, fixed="nesting", n_obj=8)
    lookups = [(q, INCLUDE) for q in queries]
    got, want, stats = _case(schema, rels, lookups, 3)
    cases.agree(got, want, lookups)
    names = slc.intern(rels)
    walker = ess.EmuEngine(schema)  # unsharded, loaded with the shards' interning
    slc.load(walker, rels, names)
    walker.publish()
    marked = sum(walker.replica_marks(*cases.request(walker, names, q, INCLUDE)[:5]) for q, _ in lookups)
    assert sum(s["admitted"] for s in stats) == marked > 0
    replica = E.EmuEngine(schema)
    replica.write_rels(rels, __import__("golden_runner").split_rel)
    replica.publish()
    verified = sum(replica.lookup_subjects(*q)[3].get("verified", 0) for q, _ in lookups)
    assert sum(s["candidates"] for s in stats) == verified > 0
    assert sum(s["entries_sent"] for s in stats) > 0 and sum(s["fallbacks"] for s in stats) == 0


def test_expiry_at_two_clocks():
    rng = random.Random(8900)
    model = randgen.model_from_schema(EXP_SCHEMA)
    rels = randgen.random_relationships(rng, model, n_obj=6, n_user=5, density=0.4)
    expires = {r: rng.choice([50, 150]) for r in rels if rng.random() < 0.5}
    lookups = cases.with_options(__import__("lookup_subjects_oracle").subject_queries(model, rng, 6, per_type=3))
    answers = []
    for now in (100, 200):
        got, want, _ = _case(EXP_SCHEMA, rels, lookups, 3, expires=expires, now=now)
        cases.agree(got, want, lookups)
        answers.append(got)
    assert answers[0] != answers[1]


def test_overflow_halves_then_falls_back_to_every_owned_subject():
    schema, rels, queries = cases.random_case(9000, fixed="nesting")
    lookups = cases.with_options(queries)
    got, want, stats = _case(schema, rels, lookups, 3, walk_cap=1)
    cases.agree(got, want, lookups)
    assert sum(s["halvings"] for s in stats) > 0 and sum(s["fallbacks"] for s in stats) > 0
    # the hand table's wildcard rows through the fallback too
    lookups = cases.with_options([q for q, _, _ in HAND_TABLE])
    got, want, stats = _case(HAND, HAND_RELS, lookups, 2, expires=HAND_EXPIRES, now=100, walk_cap=1)
    cases.agree(got, want, lookups)
    assert sum(s["fallbacks"] for s in stats) > 0


def test_more_than_one_round_uneven_ranks_one_empty():
    schema, rels, queries = cases.random_case(9100, n_obj=6)
    lookups = (cases.with_options(queries) * 13)[:150]
    assert len(lookups) > 2 * 64
    got, want, stats = _case(schema, rels, lookups, 3, skip_rank=1)
    cases.agree(got, want, lookups)
    assert stats[0]["rounds"] >= 3


def test_answers_are_ascending_uint32():
    schema, rels, queries = cases.random_case(9200, fixed="docs")
    names = __import__("shard_lookup_cases").intern(rels)
    engines, ts = _cluster(schema, 2, lambda e: __import__("shard_lookup_cases").load(e, rels, names))
    reqs = [[cases.request(engines[0], names, q, INCLUDE) for q in queries], []]
    out, _ = cases.run_sharded(engines, ts, reqs)
    assert out[1] == []
    for a in out[0]:
        assert a is not None
        for arr in (a[0], a[2]):
            assert arr.dtype == np.uint32 and np.all(np.diff(arr.astype(np.int64)) > 0)
