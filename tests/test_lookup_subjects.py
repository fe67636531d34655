"""LookupSubjects on the CPU: the two oracle restatements against each other, a hand table of the semantics
(wildcard exclusions, the EXCLUDE option, userset self-membership, the depth cap, the fenced divergence from
SpiceDB), the launch sequence of device.cu under the kernel emulator against the oracle (forward walk and the
every-object fallback), and the C ABI's refusals on a host-only engine."""
import os
import random
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))

import randgen  # noqa: E402
from golden_runner import split_rel  # noqa: E402
from lookup_subjects_oracle import (  # noqa: E402
    EXCLUDE, INCLUDE, COracleSubjects, DepthError, mini_lookup_subjects, property_violations, subject_queries)
from oracle.mini_oracle import MiniOracle  # noqa: E402


def _ask(fn, *a, **k):
    try:
        return fn(*a, **k)
    except DepthError:
        return "EDEPTH"


def _both(schema, rels, expires=None):
    c, m = COracleSubjects(schema), MiniOracle(schema)
    for r in rels:
        ex = (expires or {}).get(r, 0)
        c.touch(r, ex)
        m.write(r, ex)
    return c, m


def _oracles_agree(schema, rels, queries, now=0, expires=None):
    c, m = _both(schema, rels, expires)
    for q in queries:
        for opt in (INCLUDE, EXCLUDE):
            a = _ask(c.lookup_subjects, *q, wildcards=opt, now=now)
            b = _ask(mini_lookup_subjects, m, c.seen, *q, wildcards=opt, now=now)
            assert a == b, f"{q} opt={opt}: C={a} mini={b}\n{schema}\n" + "\n".join(rels)


@pytest.mark.parametrize("seed", range(25))
def test_oracles_agree_random_schemas(seed):
    rng = random.Random(7000 + seed)
    schema, model = randgen.random_schema(rng)
    rels = randgen.random_relationships(rng, model, n_obj=5, n_user=4, density=0.35)
    _oracles_agree(schema, rels, subject_queries(model, rng, 5))


@pytest.mark.parametrize("name", sorted(randgen.FIXED_SCHEMAS))
@pytest.mark.parametrize("seed", range(3))
def test_oracles_agree_fixed_schemas(name, seed):
    rng = random.Random(7100 + seed)
    schema = randgen.FIXED_SCHEMAS[name]
    model = randgen.model_from_schema(schema)
    rels = randgen.random_relationships(rng, model, n_obj=5, n_user=5, density=0.3)
    _oracles_agree(schema, rels, subject_queries(model, rng, 5))


EXP_SCHEMA = """
use expiration
definition user {}
definition group { relation member: user with expiration | group#member with expiration }
definition doc {
  relation viewer: user with expiration | user:* with expiration | group#member with expiration
  relation banned: user with expiration
  permission view = viewer - banned
}
"""


@pytest.mark.parametrize("seed", range(6))
def test_oracles_agree_with_expiration(seed):
    rng = random.Random(7200 + seed)
    model = randgen.model_from_schema(EXP_SCHEMA)
    rels = randgen.random_relationships(rng, model, n_obj=5, n_user=5, density=0.4)
    expires = {r: rng.choice([50, 150]) for r in rels if rng.random() < 0.5}
    _oracles_agree(EXP_SCHEMA, rels, subject_queries(model, rng, 5, per_type=3), now=100, expires=expires)


HAND = """
use expiration
definition user {}
definition group { relation member: user | group#member }
definition doc {
  relation viewer: user | user:* | group#member
  relation editor: user | user:*
  relation banned: user
  relation banned2: user
  relation member2: user
  relation temp: user:* with expiration
  permission view = viewer - banned
  permission view2 = viewer - (banned & banned2)
  permission both = viewer & member2
  permission diverge = (viewer & member2) + editor
  permission temp_view = temp
}
"""
HAND_RELS = [
    "doc:d1#viewer@user:*", "doc:d1#viewer@user:alice", "doc:d1#banned@user:bob",
    "doc:d2#viewer@user:*", "doc:d2#viewer@user:alice", "doc:d2#banned@user:bob", "doc:d2#banned@user:carol",
    "doc:d2#banned2@user:carol",
    "doc:d3#viewer@user:*", "doc:d3#member2@user:dave",
    "doc:d4#viewer@user:*", "doc:d4#editor@user:*", "doc:d4#member2@user:erin",
    "group:g1#member@group:g2#member", "group:g2#member@user:frank",
    # d5: a wildcard viewer and a group chain deeper than the dispatch cap: Check HAS through `*`, the
    # no-wildcards check of `deep` cannot be decided -- not listed, and not a failure
    "doc:d5#viewer@user:*", "doc:d5#viewer@group:c0#member",
] + [f"group:c{i}#member@group:c{i + 1}#member" for i in range(55)] + ["group:c55#member@user:deep"] + [
    "doc:d6#temp@user:*",
]
HAND_EXPIRES = {"doc:d6#temp@user:*": 50}
HAND_TABLE = [
    # (resource, perm, subject type, subject relation, option) -> (concrete, wildcard, excluded) or "EDEPTH"
    (("doc", "d1", "view", "user", ""), INCLUDE, (["alice"], True, ["bob"])),  # {*, alice} - {bob}
    (("doc", "d1", "view", "user", ""), EXCLUDE, (["alice"], False, [])),
    (("doc", "d2", "view2", "user", ""), INCLUDE, (["alice"], True, ["carol"])),  # {*} - (banned & banned2)
    (("doc", "d3", "both", "user", ""), INCLUDE, (["dave"], False, [])),  # viewer & member2, viewer = {*}
    (("doc", "d4", "diverge", "user", ""), INCLUDE, ([], True, [])),  # the fenced divergence (DESIGN §2)
    (("group", "g1", "member", "group", "member"), INCLUDE, (["g1", "g2"], False, [])),  # userset: itself
    (("group", "g1", "member", "user", ""), INCLUDE, (["frank"], False, [])),
    (("group", "c0", "member", "user", ""), INCLUDE, "EDEPTH"),  # depth cap
    (("doc", "d5", "viewer", "user", ""), INCLUDE, ([], True, [])),  # nowild ERROR is not a failure
    (("doc", "d6", "temp_view", "user", ""), INCLUDE, ([], False, [])),  # expired wildcard
    (("doc", "nope", "view", "user", ""), INCLUDE, ([], False, [])),  # never-written resource
]


@pytest.mark.parametrize("i", range(len(HAND_TABLE)))
def test_hand_table_both_oracles(i):
    q, opt, want = HAND_TABLE[i]
    c, m = _both(HAND, HAND_RELS, HAND_EXPIRES)
    assert _ask(c.lookup_subjects, *q, wildcards=opt, now=100) == want
    assert _ask(mini_lookup_subjects, m, c.seen, *q, wildcards=opt, now=100) == want


def test_fenced_divergence_describes_the_same_set():
    """SpiceDB lists erin concretely beside `*` for (viewer & member2) + editor with viewer = editor = {*}; this
    engine lists only `*`. Both answers describe the same set: every subject has the permission."""
    c, _ = _both(HAND, HAND_RELS)
    for s in ("erin", "zed", "alice"):
        assert c.o.check("doc", "d4", "diverge", "user", s) == 2
    assert c.lookup_subjects("doc", "d4", "diverge", "user") == ([], True, [])


# ---- the launch sequence under the kernel emulator ---------------------------------------------------------

@pytest.fixture(scope="module")
def emu():
    import emu_subjects as E  # tests/emu/emu_subjects.cc: the emulator driver plus LookupSubjects' sequence

    E.lib()
    return E


def _emu_vs_oracle(emu, schema, rels, queries, now=0, expires=None, walk_caps=(1 << 16, 2)):
    c = COracleSubjects(schema)
    for r in rels:
        c.touch(r, (expires or {}).get(r, 0))
    e = emu.EmuEngine(schema)
    e.write_rels(rels, split_rel)
    if expires:
        t = np.zeros(len(expires), dtype=emu.TUPLE_DTYPE)
        for i, r in enumerate(expires):
            rt, rid, rel, st, sid, srel = split_rel(r)
            t["rel"][i], t["stype"][i] = e.slot_id(rt, rel), e.type_id(st)
            t["res"][i] = e._id(rt, rid, True)
            t["srel"][i], t["subj"][i] = (emu.SREL_WILDCARD, 0) if sid == "*" else (
                e.slot_id(st, srel) if srel else emu.SREL_NONE, e._id(st, sid, True))
        e.load_tuples(t, np.array(list(expires.values()), dtype=np.uint32))
    e.publish()
    opts = emu.default_opts(now=now)
    for q in queries:
        for opt in (INCLUDE, EXCLUDE):
            want = _ask(c.lookup_subjects, *q, wildcards=opt, now=now)
            # the walk with both options; the overflow and the forced fallback with INCLUDE (the emulator is slow)
            for force in (False, True) if opt == INCLUDE else (False,):
                for cap in (walk_caps if opt == INCLUDE else walk_caps[:1]) if not force else (0,):
                    try:
                        ids, wild, ex, _ = e.lookup_subjects(*q, include_wildcard=opt == INCLUDE, force_fallback=force,
                                                             walk_cap=cap or 16, opts=opts)
                        got = (sorted(ids), wild, sorted(ex))
                    except RuntimeError as err:
                        assert str(err) == "EDEPTH", err
                        got = "EDEPTH"
                    assert got == want, f"{q} opt={opt} fallback={force} cap={cap}: emu={got} oracle={want}"


def test_emulator_hand_table(emu):
    queries = [q for q, _, _ in HAND_TABLE]
    _emu_vs_oracle(emu, HAND, HAND_RELS, queries, now=100, expires=HAND_EXPIRES)


@pytest.mark.parametrize("name", ["nesting", "docs", "deep_nonpure"])  # cfg3, cfg4 at small scale
def test_emulator_fixed_schemas(emu, name):
    rng = random.Random(7300)
    schema = randgen.FIXED_SCHEMAS[name]
    model = randgen.model_from_schema(schema)
    rels = randgen.random_relationships(rng, model, n_obj=6, n_user=5, density=0.3)
    _emu_vs_oracle(emu, schema, rels, subject_queries(model, rng, 6, per_type=1))


@pytest.mark.parametrize("seed", range(6))
def test_emulator_random_schemas(emu, seed):
    rng = random.Random(7400 + seed)
    schema, model = randgen.random_schema(rng)
    rels = randgen.random_relationships(rng, model, n_obj=5, n_user=4, density=0.35)
    _emu_vs_oracle(emu, schema, rels, subject_queries(model, rng, 5, per_type=1))


@pytest.mark.parametrize("wl", ["cfg3", "cfg4"])
def test_emulator_workloads_property(emu, wl):
    """The BASELINE shapes, scaled down: walk and fallback agree, and the answer has the defining property
    against the oracle's Check."""
    import zgpu  # noqa: F401  (registers the package for the workload generators)
    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.by_name(wl, 0.0002 if wl == "cfg4" else 0.002)
    e, o = emu.EmuEngine(w.schema), Oracle(w.schema)
    w.load_into(e), w.load_into(o)
    e.publish()
    n_users = max(int(g.subj.max()) + 1 for g in w.groups if g.subj_type == "user" and not g.wildcard and g.subj.size)
    rt = w.checks[0].res_type
    n_res = max(int(g.res.max()) + 1 for g in w.groups if g.res_type == rt and g.res.size)
    rng = np.random.default_rng(5)
    for perm in [c.perm for c in w.checks][:2]:
        for r in rng.choice(n_res, size=4, replace=False):
            a = e.lookup_subjects_ids(e.type_id(rt), r, e.slot_id(rt, perm), e.type_id("user"))
            b = e.lookup_subjects_ids(e.type_id(rt), r, e.slot_id(rt, perm), e.type_id("user"), force_fallback=True)
            assert [list(x) for x in a[:3:2]] == [list(x) for x in b[:3:2]] and a[1] == b[1]
            assert not a[3]["fell_back"] and b[3]["fell_back"] and a[3]["verified"] <= b[3]["verified"]
            bad = property_violations(o.check_bulk, emu.CHECK_DTYPE, r, o.slot_id(rt, perm), o.type_id("user"),
                                      emu.SREL_NONE, n_users, a[0], a[1], a[2])
            assert not bad, (wl, perm, r, bad)


# ---- C ABI refusals (host-only engine: no GPU needed) -----------------------------------------------------

def test_host_only_engine_refuses_and_bad_arguments_are_einval():
    import zgpu

    e = zgpu.Engine(HAND, host_only=True)
    e.write_relationships([(zgpu._lib.OP_TOUCH, r, 0) for r in HAND_RELS[:3]])
    with pytest.raises(zgpu.ZgpuError) as ei:
        e.lookup_subjects_str("doc", "d1", "view", "user")
    assert ei.value.code == -4
    with pytest.raises(zgpu.ZgpuError) as ei:
        e.lookup_subjects_ids("doc", 0, "view", "user")
    assert ei.value.code == -4
    for args, kw in [(("nodoc", "d1", "view", "user"), {}), (("doc", "d1", "nope", "user"), {}),
                     (("doc", "d1", "view", "nouser"), {}), (("doc", "d1", "view", "user", "nope"), {}),
                     (("doc", "d1", "view", "user"), {"wildcards": 7})]:
        with pytest.raises(zgpu.ZgpuError) as ei:
            e.lookup_subjects_str(*args, **kw)
        assert ei.value.code == -1, args
    for args, kw in [(("doc", 0, "nope", "user"), {}), (("doc", 0, "view", "nouser"), {}),
                     (("doc", 0, "view", "user"), {"wildcards": 2})]:
        with pytest.raises(zgpu.ZgpuError) as ei:
            e.lookup_subjects_ids(*args, **kw)
        assert ei.value.code == -1, args
