"""zg_import_relationships on host-only engines (the host path, which the device path is compared against): ids, names,
reads and the watch feed equal those of the same relationships written in the same order through
zg_write_relationships; the first failing relationship's code and message; nothing changes on failure; duplicates in
the call and against the store; freed ids reused lowest first; the feed's cap; the client's Export -> Import round
trip."""
import random
import re

import pytest

import filter_cases as cases

EINVAL, EEXIST, EPRECOND = -1, -2, -5  # include/zgpu.h
NO_OBJECT = 0xFFFFFFFF
CREATE = 1

PLAIN_SCHEMA = """
definition user {}
definition team { relation member: user | team#member }
definition repo {
  relation reader: user | user:* | team#member
  relation admin: user
  permission read = reader + admin
}
"""


@pytest.fixture(scope="module")
def zg():
    import zgpu

    return zgpu


def _engine(zg, schema=cases.EXP_SCHEMA, clock=100):
    e = zg.Engine(schema, host_only=True)
    e.set_clock(clock)
    return e


def _exp_rels(rng, n, prefix=""):
    """Relationship texts with expirations on EXP_SCHEMA: users, wildcards and group usersets, names shared between
    the subject and resource columns (group:gN is both), grouped by class."""
    out = []
    for _ in range(n):
        k = rng.random()
        exp = rng.choice([0, 0, 500, 50])  # 50 is expired at clock 100, not collected
        if k < 0.4:
            out.append((f"doc:{prefix}d{rng.randrange(40)}#viewer@user:{prefix}u{rng.randrange(30)}", exp))
        elif k < 0.5:
            out.append((f"doc:{prefix}d{rng.randrange(40)}#viewer@user:*", exp))
        elif k < 0.7:
            out.append((f"doc:{prefix}d{rng.randrange(40)}#viewer@group:{prefix}g{rng.randrange(8)}#member", exp))
        elif k < 0.85:
            out.append((f"group:{prefix}g{rng.randrange(8)}#member@user:{prefix}u{rng.randrange(30)}", exp))
        else:
            out.append((f"doc:{prefix}d{rng.randrange(40)}#banned@user:{prefix}u{rng.randrange(30)}", exp))
    seen, uniq = set(), []
    for r, x in out:
        if r not in seen:
            seen.add(r)
            uniq.append((r, x))
    return uniq


def _call_order(zg, rels):
    """The relationships in the order an import of Engine.import_groups(rels) takes them."""
    return [(f"{rt}:{rid}#{r}@{st}:{sid}" + (f"#{sr}" if sr else ""), x)
            for rt, r, st, sr, res, subj, ex in zg.Engine.import_groups(rels)
            for rid, sid, x in zip(res, subj, ex if ex is not None else [0] * len(res))]


def _write(zg, e, rels):
    for i in range(0, len(rels), 1000):
        e.write_relationships([(CREATE, r, x) for r, x in rels[i:i + 1000]])


def _split(r):
    from spicedb_kubeapi_proxy_b200._lib import split_rel

    return split_rel(r)


def _ids(zg, e, rels):
    ids = {}
    for r, _ in rels:
        rt, rid, _, st, sid, _ = _split(r)
        ids[(rt, rid)] = e.find(rt, rid)
        if sid != "*":
            ids[(st, sid)] = e.find(st, sid)
    return ids


def _feed(e, since):
    return [(op, text, x) for _, op, text, x in e.watch_read(since)[0]]


def _same_as_writes(zg, schema, batches, clock=100):
    """Imports each batch into one engine and writes it (in the import's call order) into another; compares ids,
    names, reads and the feed after every batch."""
    imp, wr = _engine(zg, schema, clock), _engine(zg, schema, clock)
    r0i, r0w = imp.stats()["revision"], wr.stats()["revision"]
    every = []
    for rels in batches:
        assert imp.import_relationships(imp.import_groups(rels)) == len(rels)
        order = _call_order(zg, rels)
        _write(zg, wr, order)
        every += order
        assert _ids(zg, imp, every) == _ids(zg, wr, every)
        assert imp.read_relationships() == wr.read_relationships()
        assert _feed(imp, r0i) == _feed(wr, r0w)
        assert imp.name_counters()["id_extent"] == wr.name_counters()["id_extent"]
    assert imp.stats()["revision"] == r0i + len(batches)
    return imp, wr


def test_ids_reads_and_feed_equal_the_write_path(zg):
    rng = random.Random(7)
    _same_as_writes(zg, cases.EXP_SCHEMA, [_exp_rels(rng, 300), _exp_rels(rng, 300, "n"), _exp_rels(rng, 200, "m")])


def test_counters(zg):
    e = _engine(zg)
    e.import_relationships(e.import_groups([("doc:a#viewer@user:u", 0), ("doc:b#viewer@user:u", 0)]))
    c = e.import_counters()
    assert c == {"device": 0, "host": 1, "relationships": 2, "names_found": 0, "names_new": 3}
    e.import_relationships(e.import_groups([("doc:a#banned@user:u", 0)]))
    c = e.import_counters()
    assert c["host"] == 2 and c["relationships"] == 3 and c["names_found"] == 2 and c["names_new"] == 3


def _body(err):
    """An error's message without its "update <i>" / "relationship <i>" prefix."""
    return re.sub(r"^zgpu error -?\d+: (update|relationship) \d+", "", str(err))


BAD = [  # (schema, relationship text, expires_at)
    (PLAIN_SCHEMA, "nope:x#reader@user:a", 0),
    (PLAIN_SCHEMA, "repo:x#reader@nope:a", 0),
    (PLAIN_SCHEMA, "repo:x#nope@user:a", 0),
    (PLAIN_SCHEMA, "repo:x#read@user:a", 0),
    (PLAIN_SCHEMA, "repo:x!#reader@user:a", 0),
    (PLAIN_SCHEMA, "repo:*#reader@user:a", 0),
    (PLAIN_SCHEMA, "repo:" + "x" * 1025 + "#reader@user:a", 0),
    (PLAIN_SCHEMA, "repo:x#reader@user:a b", 0),
    (PLAIN_SCHEMA, "repo:x#reader@team:*#member", 0),
    (PLAIN_SCHEMA, "repo:x#reader@team:t#nope", 0),
    (PLAIN_SCHEMA, "repo:x#admin@user:*", 0),
    (PLAIN_SCHEMA, "repo:x#reader@team:t", 0),
    (PLAIN_SCHEMA, "repo:x#reader@user:a", 500),
    (cases.EXP_SCHEMA, "doc:x#banned@user:*", 0),
]


@pytest.mark.parametrize("case", range(len(BAD)))
@pytest.mark.parametrize("where", ["start", "middle", "end"])
def test_first_failure_is_the_write_paths(zg, case, where):
    schema, bad, exp = BAD[case]
    good = [(f"repo:g{i}#reader@user:u{i}", 0) if schema is PLAIN_SCHEMA else (f"doc:g{i}#viewer@user:u{i}", 0)
            for i in range(6)]
    at = {"start": 0, "middle": 3, "end": 6}[where]
    rels = good[:at] + [(bad, exp)] + good[at:] + [good[0]]  # a later duplicate must not be the one reported
    wr = _engine(zg, schema)
    with pytest.raises(zg.ZgpuError) as want:
        for r, x in rels:
            wr.write_relationships([(CREATE, r, x)])
    imp = _engine(zg, schema)
    groups = [(*_lit(r), [_split(r)[1]], [_split(r)[4]], [x] if x else None) for r, x in rels]
    with pytest.raises(zg.ZgpuError) as got:
        imp.import_relationships(groups)
    assert got.value.code == want.value.code
    assert re.match(rf"zgpu error -?\d+: relationship {at}\b", str(got.value)), str(got.value)
    assert _body(got.value) == _body(want.value)
    assert _state(imp) == _state(_engine(zg, schema))


def _lit(r):
    rt, _, rel, st, _, srel = _split(r)
    return rt, rel, st, srel


def _state(e):
    return (e.read_relationships(), e.stats()["revision"], e.name_counters(), _feed(e, 0))


def test_failure_changes_nothing(zg):
    rng = random.Random(3)
    e = _engine(zg)
    e.import_relationships(e.import_groups(_exp_rels(rng, 200)))
    before = _state(e)
    fresh = [(f"doc:new{i}#viewer@user:newu{i}", 0) for i in range(50)]
    for bad in (("doc:d0!#viewer@user:x", 0), (fresh[10][0], 0), ("doc:x#banned@user:*", 0)):
        with pytest.raises(zg.ZgpuError):
            e.import_relationships(e.import_groups(fresh + [bad]) if bad[0] not in dict(fresh)
                                   else e.import_groups(fresh) + e.import_groups([bad]))
        assert _state(e) == before
        assert e.find("doc", "new0") == NO_OBJECT and e.find("user", "newu0") == NO_OBJECT


def test_duplicates(zg):
    e = _engine(zg)
    e.write_relationships([(CREATE, "doc:a#viewer@user:u", 0), (CREATE, "doc:b#viewer@user:*", 0),
                           (CREATE, "doc:c#viewer@user:old", 50)])  # expired at clock 100, not collected
    for rels, at in (([("doc:z#viewer@user:u", 0), ("doc:a#viewer@user:u", 500)], 1),
                     ([("doc:b#viewer@user:*", 0)], 0),
                     ([("doc:n#viewer@user:n", 0), ("doc:c#viewer@user:old", 0)], 1),
                     ([("doc:n#viewer@user:n", 0), ("doc:m#viewer@user:n", 0), ("doc:n#viewer@user:n", 0)], 2),
                     ([("doc:w#viewer@user:*", 0), ("doc:w#viewer@user:*", 0)], 1)):
        with pytest.raises(zg.ZgpuError) as ex:
            e.import_relationships(e.import_groups(rels))
        assert ex.value.code == EEXIST
        assert f"relationship {at}: relationship already exists" in str(ex.value)
    assert e.find("doc", "n") == NO_OBJECT


def _updates(zg, e, rows):
    """zg_apply_updates of doc:d<i>#viewer@user:u<i> for rows of (op, i), then a publish."""
    import numpy as np

    u = np.zeros(len(rows), dtype=zg.UPDATE_DTYPE)
    for k, (op, i) in enumerate(rows):
        u[k]["res"], u[k]["subj"], u[k]["rel"] = e.intern("doc", f"d{i}"), e.intern("user", f"u{i}"), e.slot_id("doc", "viewer")
        u[k]["stype"], u[k]["srel"], u[k]["op"] = e.type_id("user"), 0xFFFF, op
    e.apply_updates(u)
    e.publish()


def test_freed_ids_reused_lowest_first(zg):
    engines = []
    for use_import in (True, False):
        e = _engine(zg)
        # interned updates record nothing in the watch feed, which would keep the deleted names
        _updates(zg, e, [(0, i) for i in range(20)])
        _updates(zg, e, [(2, 3), (2, 11)])
        assert e.retire_unused_names() == 4
        rels = [("doc:x#viewer@user:y", 0), ("doc:z#viewer@user:u0", 0), ("doc:q#viewer@user:w", 0)]
        if use_import:
            e.import_relationships(e.import_groups(rels))
        else:
            _write(zg, e, rels)
        engines.append(e)
    for t, n in (("doc", "x"), ("doc", "z"), ("doc", "q"), ("user", "y"), ("user", "w")):
        assert engines[0].find(t, n) == engines[1].find(t, n)
    assert engines[0].find("user", "y") in (3, 11) and engines[0].name_counters()["free_ids"] == 0


def test_import_past_the_feed_cap_moves_the_floor(zg):
    e = _engine(zg, PLAIN_SCHEMA)
    e.write_relationships([(CREATE, "repo:r#reader@user:first", 0)])
    r0 = e.stats()["revision"]
    n = (1 << 20) + 5
    e.import_relationships([("repo", "reader", "user", "", [f"r{i}" for i in range(n)], ["u"] * n, None)])
    r1 = e.stats()["revision"]
    assert r1 == r0 + 1
    with pytest.raises(zg.ZgpuError) as ex:
        e.watch_read(r0)
    assert ex.value.code == EPRECOND
    assert e.watch_read(r1)[0] == []
    assert e.num_tuples() == n + 1


def test_client_export_then_import(zg):
    from spicedb_kubeapi_proxy_b200 import client as v1

    rng = random.Random(11)
    src = v1.PermissionsClient(cases.EXP_SCHEMA, engine=_engine(zg))
    src.engine.import_relationships(src.engine.import_groups(_exp_rels(rng, 400)))
    exported = list(src.ExportBulkRelationships(v1.ExportBulkRelationshipsRequest(optional_limit=97)))
    dst = v1.PermissionsClient(cases.EXP_SCHEMA, engine=_engine(zg))
    resp = dst.ImportBulkRelationships(v1.ImportBulkRelationshipsRequest(p.relationships) for p in exported)
    assert resp.num_loaded == sum(len(p.relationships) for p in exported)
    again = list(dst.ExportBulkRelationships(v1.ExportBulkRelationshipsRequest(optional_limit=97)))
    # the same relationships; the page order follows the ids, which the import hands out in its own call order
    flat = lambda pages: sorted((r.text(), r.optional_expires_at) for p in pages for r in p.relationships)  # noqa: E731
    assert flat(again) == flat(exported) and len(flat(again)) == len(set(flat(again)))
    with pytest.raises(v1.RpcError) as ex:
        dst.ImportBulkRelationships([v1.ImportBulkRelationshipsRequest(exported[0].relationships[:1])])
    assert ex.value.code == "ALREADY_EXISTS"
    with pytest.raises(v1.RpcError) as ex:
        dst.ImportBulkRelationships([v1.ImportBulkRelationshipsRequest([v1.Relationship.parse("doc:x#nope@user:y")])])
    assert ex.value.code == "INVALID_ARGUMENT"


def test_empty_import_publishes_once(zg):
    e = _engine(zg)
    r0 = e.stats()["revision"]
    assert e.import_relationships([]) == 0
    assert e.import_relationships([("doc", "viewer", "user", "", [], [], None)]) == 0
    assert e.stats()["revision"] == r0 + 2 and e.read_relationships() == []
