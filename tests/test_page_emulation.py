"""The page kernels (csrc/filter.cuh page_window_kernel, page_count_kernel, page_emit_kernel, page_subject_kernel) and
their host side (page_walk, page_merge) under the CPU kernel emulator, against Store::page over the same store and
against a restatement in Python: every match sorted by the key K = (resource type, resource, class position, subject)
and cut after the cursor. Every filter shape, limits 1, 2, 31, 32, 33 and 1000, cursors at a row's last entry, at an
empty row, at an object past the tables' capacity and between types, expirations at two clocks, and windows that must
grow."""
import os
import random
import sys

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))

import filter_cases as cases  # noqa: E402
import randgen  # noqa: E402

LIMITS = (1, 2, 31, 32, 33, 1000)


def _engine(schema, rels, expires=None):
    import emu_page
    import zgpu  # noqa: F401
    from spicedb_kubeapi_proxy_b200._lib import split_rel
    from test_filter_emulation import _write_expiring

    e = emu_page.EmuEngine(schema)
    e.write_rels(rels, split_rel) if expires is None else _write_expiring(e, rels, expires, split_rel)
    e.publish()
    return e, split_rel


def _restated(e, x, now, after, want):
    rows = sorted(e.host_match(x, now), key=e.key)  # host_match rows: (res, subj, rel, stype, srel, flags, expires)
    rows = [r[:5] + (r[6],) for r in rows if after is None or e.key(r) > tuple(after)]
    return rows[:want]


def _page(e, x, limit, now=0, after=None, **kw):
    """One page on both paths and the restatement; -> (rows, cursor of the last row, more, info)."""
    want = limit + 1
    got, info = e.device_page(x, want, now, after, **kw)
    assert got == e.host_page(x, want, now, after) == _restated(e, x, now, after, want), (limit, after)
    return got[:limit], (e.key(got[limit - 1]) if len(got) >= limit else None), len(got) > limit, info


def _drain(e, x, limit, now=0, **kw):
    """Pages until the end: their concatenation is every match in K order, each exactly once."""
    rows, after, infos = [], None, []
    while True:
        page, last, more, info = _page(e, x, limit, now, after, **kw)
        rows += page
        infos.append(info)
        if not more:
            break
        after = last
    assert rows == _restated(e, x, now, None, 10 ** 6)
    return rows, infos


def _filters(e, rels, split_rel, rng, samples):
    out = []
    for f in cases.filters_for(rels, split_rel, rng, samples=samples):
        x = e.resolve(f)
        if x is not None:
            out.append(x)
    return out


@pytest.mark.parametrize("name", sorted(randgen.FIXED_SCHEMAS))
def test_fixed_schemas(name):
    rng = random.Random(9700)
    schema = randgen.FIXED_SCHEMAS[name]
    rels = randgen.random_relationships(rng, randgen.model_from_schema(schema), n_obj=5, n_user=5, density=0.4)
    e, split_rel = _engine(schema, rels)
    filters = _filters(e, rels, split_rel, rng, samples=2)
    shapes = set()
    for i, x in enumerate(filters):
        shapes.add(0 if x.has_res else 1 if (x.has_subj or x.subj_wildcard) else 2)
        for limit in (LIMITS if i % 8 == 0 else (7, 1000)):
            _drain(e, x, limit)
    assert shapes == {0, 1, 2}


@pytest.mark.parametrize("seed", range(3))
def test_random_schemas(seed):
    rng = random.Random(9800 + seed)
    schema, model = randgen.random_schema(rng)
    rels = randgen.random_relationships(rng, model, n_obj=4, n_user=4, density=0.4)
    e, split_rel = _engine(schema, rels)
    for i, x in enumerate(_filters(e, rels, split_rel, rng, samples=2)):
        _drain(e, x, (1, 7, 33)[i % 3])


@pytest.mark.parametrize("now", [100, 200])
def test_expirations(now):
    """Half of the relationships expire at 50 or 150: the windows of the scan shape come up short and grow, and the
    expirations on every page are the store's."""
    rng = random.Random(9900)
    rels = randgen.random_relationships(rng, randgen.model_from_schema(cases.EXP_SCHEMA), n_obj=6, n_user=6, density=0.5)
    rels += ["doc:o0#viewer@user:*", "doc:o1#viewer@user:*"]
    expires = {r: rng.choice([50, 150]) for r in rels if rng.random() < 0.5}
    e, split_rel = _engine(cases.EXP_SCHEMA, rels, expires)
    for x in _filters(e, rels, split_rel, rng, samples=3)[::2]:
        for limit in (1, 32):
            _drain(e, x, limit, now=now)
    # clock 0 (a limited delete): expired relationships are matched too
    x = e.resolve({"res_type": "doc"})
    assert len(_drain(e, x, 5, now=0)[0]) == len({r for r in rels if r.startswith("doc:")})


def test_cursors_at_edges():
    schema = randgen.FIXED_SCHEMAS["docs"]
    rels = ["document:d0#viewer@user:u0", "document:d0#viewer@user:u1", "document:d0#viewer@user:*",
            "document:d2#owner@group:g0#member", "document:d2#viewer@user:u1", "group:g0#member@user:u1",
            "org:o0#member@user:u0"]
    e, split_rel = _engine(schema, rels)
    doc, user = e.type_id("document"), e.type_id("user")
    everything = e.resolve({})
    keys = [e.key(r) for r in _restated(e, everything, 0, None, 100)]
    u1 = e.resolve({"subj_type": "user", "subj_id": "u1"})
    d0 = e.resolve({"res_type": "document", "res_id": "d0"})
    scan = e.resolve({"res_type": "document"})
    cursors = keys + [
        (doc, keys[1][1], keys[1][2], 0xFFFFFFFF),  # the last subject a row can hold
        (doc, 1, 0, 0),                              # an object with empty rows
        (doc, 0xFFFFFFF0, 0, 0),                     # past the tables' capacity
        (doc, 0, 0xFFFF, 0),                         # past the type's last class
        (user, 0, 0, 0),                             # a type with no relations, between two that have some
        (0xFFFF, 0, 0, 0),                           # past every type
    ]
    for after in cursors:
        for x in (everything, u1, d0, scan):
            for limit in (1, 2, 1000):
                _page(e, x, limit, after=after)


def test_windows_grow():
    """A type with two relations: paging one of them sizes the first window from the offsets of both, so it comes up
    short and grows; a row longer than a tile's share, a single long row, and limits across its 32-entry steps."""
    schema = randgen.FIXED_SCHEMAS["docs"]
    rels = [f"document:d{i}#owner@user:u{i % 7}" for i in range(300)]
    rels += [f"document:d{i}#viewer@user:u{j}" for i in range(0, 300, 37) for j in range(3)]
    rels += [f"org:big#member@user:u{i}" for i in range(100)]
    e, split_rel = _engine(schema, rels)
    x = e.resolve({"res_type": "document", "rel": "viewer"})
    for limit in (1, 2, 7):
        _, infos = _drain(e, x, limit)
        assert max(i["windows"] for i in infos) > 1
        assert max(i["max_tiles"] for i in infos) > 1
    for f in ({"res_type": "org", "res_id": "big"}, {"res_type": "org", "rel": "member"}, {"subj_type": "user", "subj_id": "u3"}):
        for limit in (31, 32, 33):
            _drain(e, e.resolve(f), limit, grid=3)
