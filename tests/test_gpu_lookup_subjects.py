"""LookupSubjects on the GPU, through the C ABI: bit-exact against the oracle's definition on the random and fixed
schemas of the check parity tests, the forward walk against the every-object fallback (ZGPU_NO_RBFS=1), answers
after incremental writes, the ZG_E2BIG retry, the client mirror, and cfg4 at the full-size tests' scale through
the answer's defining property."""
import ctypes as C
import os
import random

import numpy as np
import pytest

import randgen
from lookup_subjects_oracle import EXCLUDE, INCLUDE, COracleSubjects, DepthError, property_violations, subject_queries
from test_lookup_subjects import HAND, HAND_EXPIRES, HAND_RELS, HAND_TABLE

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def zg():
    import zgpu

    return zgpu


def _load(zg, schema, rels, now=0, expires=None, **kw):
    c, e = COracleSubjects(schema), zg.Engine(schema, **kw)
    if now:
        e.set_clock(now)
    ups = []
    for r in rels:
        ex = (expires or {}).get(r, 0)
        c.touch(r, ex)
        ups.append((zg._lib.OP_TOUCH, r, ex))
    for i in range(0, len(ups), 1000):
        e.write_relationships(ups[i:i + 1000])
    e.publish()
    return e, c


def _engine_answer(zg, e, q, opt):
    try:
        ids, wild, ex = e.lookup_subjects_str(*q, wildcards=opt)
    except zg.ZgpuError as err:
        assert err.code == -9, err
        return "EDEPTH"
    return sorted(ids), wild, sorted(ex)


def _compare(zg, e, c, queries, now=0):
    for q in queries:
        for opt in (INCLUDE, EXCLUDE):
            try:
                want = c.lookup_subjects(*q, wildcards=opt, now=now)
            except DepthError:
                want = "EDEPTH"
            got = _engine_answer(zg, e, q, opt)
            assert got == want, f"{q} opt={opt}: gpu={got} oracle={want}\n{c.schema}\n" + "\n".join(c.rels)


@pytest.mark.parametrize("seed", range(30))
def test_random_schemas_random_graphs(zg, seed):
    rng = random.Random(seed)
    schema, model = randgen.random_schema(rng)
    rels = randgen.random_relationships(rng, model, n_obj=6, n_user=5, density=0.35)
    e, c = _load(zg, schema, rels)
    _compare(zg, e, c, subject_queries(model, rng, 6))


@pytest.mark.parametrize("name", sorted(randgen.FIXED_SCHEMAS))
@pytest.mark.parametrize("seed", range(3))
def test_fixed_schemas_random_graphs(zg, name, seed):
    rng = random.Random(500 + seed)
    schema = randgen.FIXED_SCHEMAS[name]
    model = randgen.model_from_schema(schema)
    rels = randgen.random_relationships(rng, model, n_obj=7, n_user=6, density=0.3)
    e, c = _load(zg, schema, rels)
    _compare(zg, e, c, subject_queries(model, rng, 7, per_type=3))


def test_hand_table(zg):
    e, c = _load(zg, HAND, HAND_RELS, now=100, expires=HAND_EXPIRES)
    for q, opt, want in HAND_TABLE:
        assert _engine_answer(zg, e, q, opt) == want, q
    _compare(zg, e, c, [q for q, _, _ in HAND_TABLE], now=100)


@pytest.mark.parametrize("seed", range(6))
def test_walk_and_exhaustive_fallback_agree(zg, seed, monkeypatch):
    rng = random.Random(900 + seed)
    schema, model = (randgen.FIXED_SCHEMAS["docs"], randgen.model_from_schema(randgen.FIXED_SCHEMAS["docs"])) \
        if seed % 2 else randgen.random_schema(rng)
    rels = randgen.random_relationships(rng, model, n_obj=8, n_user=6, density=0.3)
    queries = subject_queries(model, rng, 8, per_type=3)
    walk, c = _load(zg, schema, rels)
    monkeypatch.setenv("ZGPU_NO_RBFS", "1")
    scan, _ = _load(zg, schema, rels)
    for q in queries:
        for opt in (INCLUDE, EXCLUDE):
            assert _engine_answer(zg, walk, q, opt) == _engine_answer(zg, scan, q, opt), q
    _compare(zg, scan, c, queries)


def test_answers_follow_incremental_writes(zg):
    rng = random.Random(77)
    schema = randgen.FIXED_SCHEMAS["docs"]
    model = randgen.model_from_schema(schema)
    rels = randgen.random_relationships(rng, model, n_obj=8, n_user=6, density=0.3)
    e, c = _load(zg, schema, rels)
    queries = subject_queries(model, rng, 8, per_type=3)
    _compare(zg, e, c, queries)
    for round_ in range(3):
        more = randgen.random_relationships(random.Random(100 + round_), model, n_obj=8, n_user=6, density=0.1)
        gone = rng.sample(sorted(c.rels), 5)
        ups = [(zg._lib.OP_TOUCH, r, 0) for r in more] + [(zg._lib.OP_DELETE, r, 0) for r in gone if r not in more]
        e.write_relationships(ups)
        for r in more:
            c.touch(r)
        for r in gone:
            if r not in more:
                c.delete(r)
        _compare(zg, e, c, queries)


def test_e2big_reports_both_sizes_and_the_retry_answers(zg):
    e, c = _load(zg, HAND, HAND_RELS)
    L = e._L
    p, st = e.slot_id("doc", "view"), e.type_id("user")
    res = L.zg_find_object(e._h, e.type_id("doc"), b"d1")
    n, nx, w = C.c_uint64(0), C.c_uint64(0), C.c_int32(0)
    rc = L.zg_lookup_subjects(e._h, p, res, st, zg.SREL_NONE, 0, None, 0, C.byref(n), None, 0, C.byref(nx), C.byref(w))
    assert rc == -7 and (n.value, nx.value, w.value) == (1, 1, 1)
    ids, ex = np.zeros(n.value, np.uint32), np.zeros(nx.value, np.uint32)
    rc = L.zg_lookup_subjects(e._h, p, res, st, zg.SREL_NONE, 0, ids.ctypes.data, n.value, C.byref(n), ex.ctypes.data,
                              nx.value, C.byref(nx), C.byref(w))
    assert rc == 0
    got = e.lookup_subjects_ids("doc", res, "view", "user", cap=0)
    assert list(got[0]) == list(ids) and got[1] and list(got[2]) == list(ex)
    assert e.lookup_subjects_str("doc", "d1", "view", "user", cap=2) == (["alice"], True, ["bob"])


def test_client_mirror_gives_the_engine_answers(zg):
    Cl = zg.client
    cl = Cl.PermissionsClient(HAND, HAND_RELS)
    for q, opt, want in HAND_TABLE:
        if want == "EDEPTH":
            with pytest.raises(Cl.RpcError):
                list(cl.LookupSubjects(Cl.LookupSubjectsRequest(Cl.ObjectReference(q[0], q[1]), q[2], q[3], q[4])))
            continue
        req = Cl.LookupSubjectsRequest(Cl.ObjectReference(q[0], q[1]), q[2], q[3], q[4],
                                       Cl.WILDCARD_OPTION_EXCLUDE_WILDCARDS if opt == EXCLUDE else Cl.WILDCARD_OPTION_UNSPECIFIED)
        resp = list(cl.LookupSubjects(req))
        concrete = sorted(r.subject.subject_object_id for r in resp if r.subject.subject_object_id != "*")
        wild = [r for r in resp if r.subject.subject_object_id == "*"]
        excluded = sorted(x.subject_object_id for r in wild for x in r.excluded_subjects)
        if q[1] == "d6":
            continue  # the client's engine runs on the wall clock: the expired wildcard is a clock question
        assert (concrete, bool(wild), excluded) == want, q


def test_cfg4_full_size_sampled_resources_have_the_property(zg):
    from spicedb_kubeapi_proxy_b200 import workloads

    scale = float(os.environ.get("ZGPU_FULLSIZE_SCALE", "0.25"))
    w = workloads.cfg4(scale=scale)
    e = zg.Engine(w.schema)
    w.load_into(e)
    e.publish()
    n_users = max(int(g.subj.max()) + 1 for g in w.groups if g.subj_type == "user" and not g.wildcard and g.subj.size)
    n_docs = max(int(g.res.max()) + 1 for g in w.groups if g.res_type == "document" and g.res.size)
    rng = np.random.default_rng(11)
    ut = e.type_id("user")
    for perm in ("view", "restricted_view"):
        p = e.slot_id("document", perm)
        for r in rng.choice(n_docs, size=6, replace=False):
            ids, wild, ex = e.lookup_subjects_ids("document", int(r), perm, "user")
            bad = property_violations(e.check_bulk, zg.CHECK_DTYPE, int(r), p, ut, zg.SREL_NONE, n_users, ids, wild, ex)
            assert not bad, (perm, int(r), wild, len(ids), len(ex), bad)
