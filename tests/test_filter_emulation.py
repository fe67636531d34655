"""The relationship-filter kernels (csrc/filter.cuh) under the CPU kernel emulator, against Store::match over the same
store: every combination of set and unset filter fields over the fixed and random schemas, wildcard classes, userset
subjects, expirations at two clocks, ids never written and ids beyond the snapshot's tables, empty rows, a row longer
than one block's share, several launches per filter, and the count launch against the emit launch."""
import os
import random
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))

import filter_cases as cases  # noqa: E402
import randgen  # noqa: E402


def _engine(schema, rels, expires=None):
    import emu_filter
    import zgpu  # noqa: F401
    from spicedb_kubeapi_proxy_b200._lib import split_rel

    e = emu_filter.EmuEngine(schema)
    e.write_rels(rels, split_rel) if expires is None else _write_expiring(e, rels, expires, split_rel)
    e.publish()
    return e, split_rel


def _write_expiring(e, rels, expires, split_rel):
    import emu_filter

    t = np.zeros(len(rels), dtype=emu_filter.TUPLE_DTYPE)
    for i, r in enumerate(rels):
        rt, rid, rel, st, sid, srel = split_rel(r)
        t["rel"][i], t["stype"][i], t["res"][i] = e.slot_id(rt, rel), e.type_id(st), e._id(rt, rid, True)
        if sid == "*":
            t["srel"][i] = emu_filter.SREL_WILDCARD
        else:
            t["srel"][i] = e.slot_id(st, srel) if srel else emu_filter.SREL_NONE
            t["subj"][i] = e._id(st, sid, True)
    e.load_tuples(t, np.array([expires.get(r, 0) for r in rels], dtype=np.uint32))


def _agree(e, filters, now=0, **kw):
    """Every filter: emit == Store::match, the count launch == the emit launch == their number."""
    shapes = set()
    for f in filters:
        x = e.resolve(f)
        if x is None:
            continue
        want = e.host_match(x, now)
        got, info = e.device_match(x, now, **kw)
        assert got == want, (f, now)
        assert info["count"] == info["emitted"] == len(want), (f, info)
        shapes.add(info["shape"])
    return shapes


@pytest.mark.parametrize("name", sorted(randgen.FIXED_SCHEMAS))
def test_fixed_schemas(name):
    rng = random.Random(9100)
    schema = randgen.FIXED_SCHEMAS[name]
    model = randgen.model_from_schema(schema)
    rels = randgen.random_relationships(rng, model, n_obj=5, n_user=5, density=0.4)
    e, split_rel = _engine(schema, rels)
    filters = cases.filters_for(rels, split_rel, rng, samples=2)
    assert _agree(e, filters) == {0, 1, 2}
    # the emulated answers are also what the statement of the filter says, not only what Store::match says
    parts = [split_rel(r) for r in rels]
    for f in filters[:40]:
        x = e.resolve(f)
        if x is not None:
            assert len(e.device_match(x)[0]) == sum(cases.matches(f, p) for p in parts), f


@pytest.mark.parametrize("seed", range(3))
def test_random_schemas(seed):
    rng = random.Random(9200 + seed)
    schema, model = randgen.random_schema(rng)
    rels = randgen.random_relationships(rng, model, n_obj=4, n_user=4, density=0.4)
    e, split_rel = _engine(schema, rels)
    # one selected class per launch: a filter that selects several classes appends behind one count
    _agree(e, cases.filters_for(rels, split_rel, rng, samples=2), max_sel=1 + seed % 2)


@pytest.mark.parametrize("now", [0, 100, 200])
def test_expirations(now):
    """Half of the relationships expire at 50 or 150: clock 0 ignores expirations (what a delete by filter matches),
    100 and 200 drop what has expired by then; the emitted expirations are the store's."""
    rng = random.Random(9300)
    model = randgen.model_from_schema(cases.EXP_SCHEMA)
    rels = randgen.random_relationships(rng, model, n_obj=5, n_user=5, density=0.4)
    rels += ["doc:o0#viewer@user:*", "doc:o1#viewer@user:*"]
    expires = {r: rng.choice([50, 150]) for r in rels if rng.random() < 0.5}
    expires["doc:o1#viewer@user:*"] = 150
    e, split_rel = _engine(cases.EXP_SCHEMA, rels, expires)
    assert _agree(e, cases.filters_for(rels, split_rel, rng, samples=3), now=now) == {0, 1, 2}


def test_ids_beyond_the_tables_and_empty_rows():
    schema = randgen.FIXED_SCHEMAS["docs"]
    rels = ["document:d0#viewer@user:u0", "document:d0#viewer@user:*", "document:d2#owner@group:g0#member",
            "group:g0#member@user:u1"]
    e, split_rel = _engine(schema, rels)
    import emu_filter
    doc, user = e.type_id("document"), e.type_id("user")
    for res in (2, 3, 10 ** 6, 0xFFFFFFF0):  # ids nobody wrote: inside the row tables' spare capacity, and beyond them
        x = emu_filter.Filter(doc, -1, -1, 1, res, 0, 0, 0, 0, emu_filter.SREL_NONE)
        assert e.device_match(x)[0] == e.host_match(x) == []
    for subj in (5, 10 ** 6, 0xFFFFFFF0):
        x = emu_filter.Filter(-1, -1, user, 0, 0, 1, subj, 0, 0, emu_filter.SREL_NONE)
        assert e.device_match(x)[0] == e.host_match(x) == []
        x = emu_filter.Filter(doc, -1, user, 1, 0, 1, subj, 0, 0, emu_filter.SREL_NONE)
        assert e.device_match(x)[0] == e.host_match(x) == []
    # a concrete id does not match the wildcard relationship, "*" matches only it
    x = e.resolve({"res_type": "document", "res_id": "d0", "subj_type": "user", "subj_id": "u0"})
    assert len(e.device_match(x)[0]) == 1
    x = e.resolve({"res_type": "document", "subj_type": "user", "subj_id": "*"})
    got = e.device_match(x)[0]
    assert len(got) == 1 and got[0][4] == emu_filter.SREL_WILDCARD and got == e.host_match(x)


def test_long_row_is_spread_over_the_grid():
    """An organisation with 700 members: more than the 64 threads of one emulated block take in a step, read by
    resource, by (type, relation) and, from the other side, by one member."""
    schema = randgen.FIXED_SCHEMAS["docs"]
    rels = [f"org:big#member@user:u{i}" for i in range(700)] + ["org:small#member@user:u3"]
    e, split_rel = _engine(schema, rels)
    for f in ({"res_type": "org", "res_id": "big"}, {"res_type": "org", "rel": "member"}, {"subj_type": "user", "subj_id": "u3"},
              {"res_type": "org", "res_id": "big", "subj_type": "user", "subj_id": "u699"}, {}):
        x = e.resolve(f)
        for grid in (1, 3):
            got, info = e.device_match(x, grid=grid)
            assert got == e.host_match(x) and info["count"] == len(got), f
            assert e.device_match(x, grid=grid, emit=False)[1]["count"] == len(got), f
    assert len(e.device_match(e.resolve({"res_type": "org", "res_id": "big"}))[0]) == 700
