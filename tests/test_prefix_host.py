"""Filters by resource id prefix (optional_resource_id_prefix) on host-only engines (Store::match, Store::page): the
match rule against a restatement, every validation error, the cursor rules, deletes and preconditions with their watch
feed, expiry, retirement and id reuse, ids without a name, and the client's field."""
import ctypes as C
import random

import pytest

import filter_cases as cases
import randgen
from golden_runner import split_rel

EINVAL, EPRECOND = -1, -5
TOUCH = 0
MUST_MATCH, MUST_NOT_MATCH = 1, 2


@pytest.fixture(scope="module")
def zg():
    import zgpu

    return zgpu


def _engine(zg, schema, rels, expires=None, now=0):
    e = zg.Engine(schema, host_only=True)
    if now:
        e.set_clock(now)
    ups = [(TOUCH, r, (expires or {}).get(r, 0)) for r in rels]
    for i in range(0, len(ups), 1000):
        e.write_relationships(ups[i:i + 1000])
    return e


def _drain(e, limit, **f):
    out, cursor = [], None
    while True:
        lines, _, _, cursor, more = e.read_relationships_page(limit, cursor, **f)
        out += lines
        if not more:
            return out


def _restrict(lines, prefix):
    return [l for l in lines if split_rel(l)[1].startswith(prefix)]


def _prefixes(rels, rng, n=3):
    """Every proper prefix of a few sampled resource names, a prefix nobody has."""
    names = sorted({split_rel(r)[1] for r in rels})
    out = {"zz-nobody-"}
    for name in rng.sample(names, min(n, len(names))):
        out.update(name[:k] for k in range(1, len(name)))
    return sorted(out)


@pytest.mark.parametrize("name", sorted(randgen.FIXED_SCHEMAS) + ["exp"])
def test_prefix_matches_restatement(zg, name):
    rng = random.Random(4242)
    schema = cases.EXP_SCHEMA if name == "exp" else randgen.FIXED_SCHEMAS[name]
    rels = randgen.random_relationships(rng, randgen.model_from_schema(schema), n_obj=12, n_user=6, density=0.3)
    expires = {r: rng.choice([50, 150]) for r in rels if rng.random() < 0.5} if name == "exp" else None
    e = _engine(zg, schema, rels, expires, now=100 if expires else 0)
    prefixes = _prefixes(rels, rng)
    n = 0
    for f in cases.filters_for(rels, split_rel, rng, samples=2):
        if f.get("res_id"):
            continue
        try:
            base = e.read_relationships(**f)
        except zg.ZgpuError:
            continue
        base_k = _drain(e, 1000, **f)
        for p in rng.sample(prefixes, min(4, len(prefixes))):
            got = e.read_relationships(**f, res_id_prefix=p)
            assert got == _restrict(base, p), (f, p)
            # pages: the unprefixed page order restricted to the prefix
            lim = rng.choice([1, 2, 7])
            assert _drain(e, lim, **f, res_id_prefix=p) == _restrict(base_k, p), (f, p, lim)
            n += 1
    assert n > 10
    # without a resource type: every type's resources with the prefix
    every = e.read_relationships()
    for p in prefixes:
        assert e.read_relationships(res_id_prefix=p) == _restrict(every, p)
    c = e.prefix_counters()
    assert c["host_filters"] > 0 and c["device_filters"] == 0


def test_validation(zg):
    schema = randgen.FIXED_SCHEMAS["docs"]
    e = _engine(zg, schema, ["document:a/b#viewer@user:u0", "document:a|c#viewer@user:u1"])
    for bad in ["*", "a*", "a b", "é", "a.b", "x" * 1025, "a\tb"]:
        with pytest.raises(zg.ZgpuError) as ex:
            e.read_relationships(res_type="document", res_id_prefix=bad)
        assert ex.value.code == EINVAL, bad
    for ok in ["a", "a/", "a|", "x" * 1024, "a-_=+|/Z9"]:
        e.read_relationships(res_type="document", res_id_prefix=ok)
    assert e.read_relationships(res_id_prefix="a/") == ["document:a/b#viewer@user:u0"]
    assert e.read_relationships(res_id_prefix="A") == []  # case-sensitive
    with pytest.raises(zg.ZgpuError) as ex:  # res_id and a prefix together
        e.read_relationships(res_type="document", res_id="a/b", res_id_prefix="a")
    assert ex.value.code == EINVAL
    with pytest.raises(zg.ZgpuError) as ex:  # relation still needs the type
        e.read_relationships(rel="viewer", res_id_prefix="a")
    assert ex.value.code == EINVAL
    for call in (lambda f: e.read_relationships_page(3, **f), lambda f: e.delete_relationships(f),
                 lambda f: e.delete_relationships_limited(f, limit=1),
                 lambda f: e.write_relationships([], [(MUST_MATCH, f)])):
        with pytest.raises(zg.ZgpuError) as ex:
            call({"res_type": "document", "res_id_prefix": "a*"})
        assert ex.value.code == EINVAL
    assert e.num_tuples() == 2


def _raw_page(zg, e, filt, prefix, limit, after=None):
    """zg_read_relationships_page or its _ex form, called directly: (lines, cursors, next)."""
    from spicedb_kubeapi_proxy_b200 import _lib

    L = e._L
    cap = 1 << 16
    buf = C.create_string_buffer(cap)
    need, n, more = C.c_size_t(0), C.c_uint64(0), C.c_int32(0)
    curs = C.create_string_buffer(limit * _lib.READ_CURSOR_BYTES)
    nxt = C.create_string_buffer(_lib.READ_CURSOR_BYTES)
    f = e._filter(filt)
    a = None if after is None else C.create_string_buffer(after, _lib.READ_CURSOR_BYTES)
    if prefix is False:
        rc = L.zg_read_relationships_page(e._h, C.byref(f), limit, a, buf, cap, C.byref(need), C.byref(n), None, curs,
                                          nxt, C.byref(more))
    else:
        fx = _lib._FilterEx(f, None if prefix is None else prefix.encode())
        rc = L.zg_read_relationships_page_ex(e._h, C.byref(fx), limit, a, buf, cap, C.byref(need), C.byref(n), None, curs,
                                             nxt, C.byref(more))
    if rc:
        raise zg.ZgpuError(rc, "")
    return buf.value.decode().split("\n")[:-1], curs.raw, nxt.raw


def test_cursor_rules(zg):
    schema = randgen.FIXED_SCHEMAS["docs"]
    rels = [f"document:ns{i}/d{j}#viewer@user:u{k}" for i in range(3) for j in range(3) for k in range(2)]
    e = _engine(zg, schema, rels)
    flt = {"res_type": "document"}
    # an unprefixed filter through the _ex call (NULL or "") gives the old call's bytes
    old = _raw_page(zg, e, flt, False, 4)
    assert _raw_page(zg, e, flt, None, 4) == old
    assert _raw_page(zg, e, flt, "", 4) == old
    assert e.read_relationships_page(4, **flt)[3] == old[2]
    lines, _, _, cur, more = e.read_relationships_page(2, res_id_prefix="ns1/", **flt)
    assert lines == sorted(r for r in rels if r.startswith("document:ns1/"))[:2] and more
    for other in ({"res_id_prefix": "ns2/"}, {"res_id_prefix": "ns1"}, {}):
        with pytest.raises(zg.ZgpuError) as ex:
            e.read_relationships_page(2, cur, **flt, **other)
        assert ex.value.code == EINVAL, other
    with pytest.raises(zg.ZgpuError) as ex:  # an unprefixed cursor with a prefix
        e.read_relationships_page(2, old[2], **flt, res_id_prefix="ns1/")
    assert ex.value.code == EINVAL
    assert e.read_relationships_page(10, cur, **flt, res_id_prefix="ns1/")[0] == \
        sorted(r for r in rels if r.startswith("document:ns1/"))[2:]


def test_deletes_preconditions_and_watch(zg):
    schema = randgen.FIXED_SCHEMAS["docs"]
    rels = [f"document:ns{i}/d{j}#viewer@user:u{k}" for i in range(3) for j in range(3) for k in range(2)]
    rels += ["org:ns1/o#member@user:u0"]
    e = _engine(zg, schema, rels)
    rev = e.stats()["revision"]
    with pytest.raises(zg.ZgpuError) as ex:
        e.write_relationships([(TOUCH, "document:x#viewer@user:u0", 0)], [(MUST_NOT_MATCH, {"res_id_prefix": "ns1/"})])
    assert ex.value.code == EPRECOND
    with pytest.raises(zg.ZgpuError) as ex:
        e.write_relationships([(TOUCH, "document:x#viewer@user:u0", 0)], [(MUST_MATCH, {"res_id_prefix": "ns9/"})])
    assert ex.value.code == EPRECOND
    e.write_relationships([(TOUCH, "document:x#viewer@user:u0", 0)], [(MUST_MATCH, {"res_id_prefix": "ns1/"}),
                                                                       (MUST_NOT_MATCH, {"res_id_prefix": "ns9/"})])
    with pytest.raises(zg.ZgpuError) as ex:  # refused: more than the limit
        e.delete_relationships_limited({"res_type": "document", "res_id_prefix": "ns0/"}, limit=5)
    assert ex.value.code == EPRECOND
    n, partial = e.delete_relationships_limited({"res_type": "document", "res_id_prefix": "ns0/"}, limit=4,
                                                allow_partial=True)
    assert (n, partial) == (4, True)
    left0 = sorted(r for r in rels if r.startswith("document:ns0/"))[4:]
    assert e.read_relationships(res_id_prefix="ns0/") == left0
    # every type: the org goes with the documents
    assert e.delete_relationships({"res_id_prefix": "ns1/"}) == 7
    assert e.read_relationships(res_id_prefix="ns1") == []
    feed, _ = e.watch_read(rev)
    deleted = sorted(r for _, op, r, _ in feed if op == "DELETE")
    assert deleted == sorted(sorted(r for r in rels if r.startswith("document:ns0/"))[:4] +
                             [r for r in rels if ":ns1/" in r])


def test_expiry_two_clocks(zg):
    schema = cases.EXP_SCHEMA
    rels = [f"doc:team{i}/d{j}#viewer@user:u{j}" for i in range(2) for j in range(4)]
    expires = {r: 150 for r in rels[::2]}
    e = _engine(zg, schema, rels, expires, now=100)
    assert e.read_relationships(res_id_prefix="team1/") == sorted(r for r in rels if "team1/" in r)
    e.set_clock(200)
    assert e.read_relationships(res_id_prefix="team1/") == sorted(r for r in rels[1::2] if "team1/" in r)
    # deletes include expired relationships
    assert e.delete_relationships({"res_id_prefix": "team0/"}) == 4


def test_retirement_reuse_and_numeric_ids(zg):
    import numpy as np

    schema = randgen.FIXED_SCHEMAS["docs"]
    e = _engine(zg, schema, ["document:keep/b#viewer@user:u0"])
    old_id = e.intern("document", "old/a")  # no relationship (and no watch change) mentions it
    assert e.retire_unused_names() == 1
    assert e.read_relationships(res_id_prefix="old") == []
    e.write_relationships([(TOUCH, "document:new/c#viewer@user:u0", 0)])
    assert e.find("document", "new/c") == old_id  # the id is reused, and matches by its new name
    assert e.read_relationships(res_id_prefix="new/") == ["document:new/c#viewer@user:u0"]
    assert e.read_relationships(res_id_prefix="old") == []
    # ids a bulk load uses without a name never match, even where their printed id has the prefix
    t = np.zeros(1, dtype=zg.TUPLE_DTYPE)
    t["res"], t["subj"] = 123, e.find("user", "u0")
    t["rel"], t["stype"], t["srel"] = e.slot_id("document", "viewer"), e.type_id("user"), zg.SREL_NONE
    e.load_tuples(t)
    assert "document:123#viewer@user:u0" in e.read_relationships(res_type="document")
    assert e.read_relationships(res_id_prefix="1") == []


def test_client_field(zg):
    from spicedb_kubeapi_proxy_b200 import client as v1

    flt = v1.RelationshipFilter("document", optional_relation="viewer")
    assert "res_id_prefix" not in flt.fields()  # unprefixed dicts are unchanged
    assert v1.RelationshipFilter("document", optional_resource_id_prefix="ns1/").fields()["res_id_prefix"] == "ns1/"

    class Stub:  # records what the client hands the engine
        def __init__(self):
            self.calls = []

        def read_relationships(self, **f):
            self.calls.append(("read", f))
            return []

        def delete_relationships(self, f, pre):
            self.calls.append(("delete", f, pre))
            return 0

    stub = Stub()
    schema = randgen.FIXED_SCHEMAS["docs"]
    c = v1.PermissionsClient(schema, [], engine=zg.Engine(schema, host_only=True))
    c.engine = stub
    list(c.ReadRelationships(v1.ReadRelationshipsRequest(v1.RelationshipFilter(optional_resource_id_prefix="ns1/"))))
    c.DeleteRelationships(v1.DeleteRelationshipsRequest(
        v1.RelationshipFilter(optional_resource_id_prefix="ns2/"),
        [v1.Precondition(v1.PRECONDITION_MUST_MATCH, v1.RelationshipFilter(optional_resource_id_prefix="ns2/"))]))
    assert stub.calls[0] == ("read", {"res_type": "", "res_id": "", "rel": "", "res_id_prefix": "ns1/"})
    assert stub.calls[1][1]["res_id_prefix"] == "ns2/" and stub.calls[1][2][0][1]["res_id_prefix"] == "ns2/"
    # and over a real engine
    rels = ["document:ns1/a#viewer@user:u0", "document:ns2/b#viewer@user:u0"]
    c = v1.PermissionsClient(schema, rels, engine=zg.Engine(schema, host_only=True))
    got = [r.relationship.text() for r in c.ReadRelationships(
        v1.ReadRelationshipsRequest(v1.RelationshipFilter(optional_resource_id_prefix="ns2/")))]
    assert got == ["document:ns2/b#viewer@user:u0"]
