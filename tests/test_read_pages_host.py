"""Pages of relationship reads on host-only engines (Store::page): paging concatenates to the unpaged read in the page
order K, cursors resume anywhere, a foreign cursor is ZG_EINVAL, and deletes with a limit refuse, delete a part, or
delete everything, with the counts and the watch feed of zg_delete_relationships."""
import random

import pytest

import filter_cases as cases
import randgen
from golden_runner import split_rel
from page_keys import class_positions, page_key

EINVAL, EPRECOND = -1, -5
TOUCH = 0


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
        lines, exp, curs, cursor, more = e.read_relationships_page(limit, cursor, **f)
        assert len(lines) == len(exp) == len(curs) and len(lines) <= limit
        assert not more or len(lines) == limit
        if lines:
            assert curs[-1] == cursor
        out += lines
        if not more:
            return out


@pytest.mark.parametrize("name", sorted(randgen.FIXED_SCHEMAS) + ["exp"])
def test_pages_concatenate_in_key_order(zg, name):
    rng = random.Random(9950)
    schema = cases.EXP_SCHEMA if name == "exp" else randgen.FIXED_SCHEMAS[name]
    rels = randgen.random_relationships(rng, randgen.model_from_schema(schema), n_obj=6, n_user=6, density=0.4)
    expires = {r: rng.choice([50, 150]) for r in rels if rng.random() < 0.5} if name == "exp" else None
    e = _engine(zg, schema, rels, expires, now=100 if expires else 0)
    pos = class_positions(schema)
    for i, f in enumerate(cases.filters_for(rels, split_rel, rng, samples=3)):
        try:
            want = e.read_relationships(**f)
        except Exception as ex:  # noqa: BLE001 -- an invalid filter is refused by both calls alike
            with pytest.raises(type(ex)):
                e.read_relationships_page(1, **f)
            continue
        for limit in ((1, 2, 7, 1000) if i % 5 == 0 else (3,)):
            got = _drain(e, limit, **f)
            assert sorted(got) == want, (f, limit)
            keys = [page_key(e, pos, g) for g in got]
            assert keys == sorted(keys) and len(set(keys)) == len(keys), (f, limit)
    c = e.page_counters()
    assert c["host_pages"] > 0 and c["device_pages"] == 0


def test_cursors_and_expirations(zg):
    schema = cases.EXP_SCHEMA
    rels = [f"doc:d{i}#viewer@user:u{j}" for i in range(4) for j in range(3)] + ["doc:d1#viewer@user:*", "doc:d2#banned@user:u1"]
    expires = {"doc:d1#viewer@user:u2": 150, "doc:d3#viewer@user:u0": 50}
    e = _engine(zg, schema, rels, expires, now=100)
    lines, exp, curs, nxt, more = e.read_relationships_page(100, res_type="doc")
    assert more is False and "doc:d3#viewer@user:u0" not in lines and len(lines) == len(rels) - 1
    assert exp[lines.index("doc:d1#viewer@user:u2")] == 150 and sum(exp) == 150
    # resuming after every line gives the rest of the read
    for i, c in enumerate(curs):
        assert _rest(e, c) == lines[i + 1:]
    # an empty page keeps the cursor
    l2, _, _, n2, m2 = e.read_relationships_page(5, nxt, res_type="doc")
    assert l2 == [] and n2 == nxt and m2 is False
    # another filter, another schema, or bytes that are no cursor: ZG_EINVAL
    for bad in (lambda: e.read_relationships_page(5, curs[0], res_type="doc", rel="viewer"),
                lambda: e.read_relationships_page(5, b"\0" * 32, res_type="doc"),
                lambda: e.read_relationships_page(0, None, res_type="doc")):
        with pytest.raises(zg.ZgpuError) as ex:
            bad()
        assert ex.value.code == EINVAL
    # the key does not depend on the engine: another engine with the same schema and ids resumes it alike
    assert _rest(_engine(zg, schema, rels, expires, now=100), curs[3]) == lines[4:]
    e.load_schema(schema)
    with pytest.raises(zg.ZgpuError) as ex:
        e.read_relationships_page(5, curs[0], res_type="doc")
    assert ex.value.code == EINVAL


def _rest(e, cursor):
    out = []
    while True:
        lines, _, _, cursor, more = e.read_relationships_page(3, cursor, res_type="doc")
        out += lines
        if not more:
            return out


def test_delete_with_a_limit(zg):
    schema = randgen.FIXED_SCHEMAS["docs"]
    rels = [f"document:d{i}#viewer@user:u{j}" for i in range(5) for j in range(4)] + ["org:o#member@user:u0"]
    a, b = _engine(zg, schema, rels), _engine(zg, schema, rels)
    f = {"res_type": "document", "rel": "viewer"}
    with pytest.raises(zg.ZgpuError) as ex:
        a.delete_relationships_limited(f, limit=19)
    assert ex.value.code == EPRECOND and "more than 19 relationships" in str(ex.value)
    assert a.read_relationships() == sorted(rels) and a.watch_read(0) == b.watch_read(0)
    first = _drain(a, 1000, **f)[:7]
    assert a.delete_relationships_limited(f, limit=7, allow_partial=True) == (7, True)
    assert a.read_relationships() == sorted(set(rels) - set(first))
    assert a.delete_relationships_limited(f, limit=13) == (13, False)
    assert a.delete_relationships_limited(f, limit=5) == (0, False)
    assert a.read_relationships() == ["org:o#member@user:u0"]
    # limit 0 is zg_delete_relationships; the feed holds the same DELETEs in the same order
    assert b.delete_relationships_limited(f) == (20, False)
    assert sorted(c[1:] for c in a.watch_read(0)[0]) == sorted(c[1:] for c in b.watch_read(0)[0])
    # preconditions are checked first
    with pytest.raises(zg.ZgpuError) as ex:
        a.delete_relationships_limited({"res_type": "org"}, [(1, {"res_type": "document"})], limit=1, allow_partial=True)
    assert ex.value.code == EPRECOND
    assert a.read_relationships() == ["org:o#member@user:u0"]


def test_client_mirror(zg):
    from spicedb_kubeapi_proxy_b200 import client as v1

    schema = randgen.FIXED_SCHEMAS["docs"]
    rels = [f"document:d{i}#viewer@user:u{j}" for i in range(3) for j in range(3)] + ["org:o#member@user:u0"]
    c = v1.PermissionsClient(schema, rels, engine=zg.Engine(schema, host_only=True))
    flt = v1.RelationshipFilter("document", optional_relation="viewer")
    whole = [r.relationship.text() for r in c.ReadRelationships(v1.ReadRelationshipsRequest(flt))]
    assert whole == sorted(r for r in rels if r.startswith("document:"))
    first = list(c.ReadRelationships(v1.ReadRelationshipsRequest(flt, optional_limit=4)))
    assert len(first) == 4 and all(r.after_result_cursor for r in first)
    rest = list(c.ReadRelationships(v1.ReadRelationshipsRequest(flt, optional_cursor=first[-1].after_result_cursor)))
    assert sorted(r.relationship.text() for r in first + rest) == whole
    exported = list(c.ExportBulkRelationships(v1.ExportBulkRelationshipsRequest(optional_limit=4)))
    assert [len(x.relationships) for x in exported] == [4, 4, 2]
    assert sorted(r.text() for x in exported for r in x.relationships) == sorted(rels)
    with pytest.raises(v1.RpcError) as ex:
        c.DeleteRelationships(v1.DeleteRelationshipsRequest(flt, optional_limit=5))
    assert ex.value.code == "FAILED_PRECONDITION"
    got = c.DeleteRelationships(v1.DeleteRelationshipsRequest(flt, optional_limit=5, optional_allow_partial_deletions=True))
    assert got == 5 and got.deletion_progress == v1.DELETION_PROGRESS_PARTIAL
    got = c.DeleteRelationships(v1.DeleteRelationshipsRequest(flt))
    assert got == 4 and got.deletion_progress == v1.DELETION_PROGRESS_COMPLETE
